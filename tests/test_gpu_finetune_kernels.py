"""The fine-tuning kernels one by one against float64 torch: eat_ce_loss against F.cross_entropy (ex_esc50.py:103-118,
ex_dcase20.py:108-123), eat_bce_masked_loss against the expression of ex_openmic.py:101-121 and eat_mixstyle against
the reference's mixstyle (helpers/utils.py:101-121), each fed the same lambda and permutation."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from efficientat_b200._lib import lib

pytestmark = pytest.mark.gpu


def _st():
    return torch.cuda.current_stream().cuda_stream


def _ce_reference(z, y, rn, lam):
    """ex_esc50.py:103-118 in float64 (y: class indices or probability rows)"""
    if rn is None:
        return F.cross_entropy(z, y, reduction="none").mean()
    bs = z.shape[0]
    return (F.cross_entropy(z, y, reduction="none") * lam.reshape(bs) +
            F.cross_entropy(z, y[rn], reduction="none") * (1. - lam.reshape(bs))).mean()


@pytest.mark.parametrize("C", [1, 10, 50, 200, 527, 4099])
@pytest.mark.parametrize("B", [1, 3, 64])
@pytest.mark.parametrize("target", ["index", "prob"])
@pytest.mark.parametrize("mix", [False, True])
def test_ce_loss_matches_cross_entropy(C, B, target, mix):
    g = torch.Generator().manual_seed(C * 1000 + B)
    z = torch.randn(B, C, generator=g, dtype=torch.float64) * 4 + 2
    if target == "index":
        y = torch.randint(0, C, (B,), generator=g)
    else:                                                       # rows that do not sum to 1 (S != 1 in the gradient)
        y = torch.rand(B, C, generator=g, dtype=torch.float64) * 2.0 / C
        y[:, 0] += 0.3
    rn = torch.randperm(B, generator=g) if mix else None
    lam = (torch.rand(B, generator=g, dtype=torch.float64) * 0.5 + 0.5) if mix else None
    zd = z.float().cuda()
    yd = y.int().cuda() if target == "index" else y.float().cuda()
    rn_d = rn.int().cuda() if mix else None
    lam_d = lam.float().cuda() if mix else None
    dz = torch.empty(B, C, device="cuda")
    acc = torch.zeros(1, device="cuda", dtype=torch.float64)
    lib().ce_loss(zd.data_ptr(), yd.data_ptr() if target == "index" else 0, yd.data_ptr() if target == "prob" else 0,
                  rn_d.data_ptr() if mix else 0, lam_d.data_ptr() if mix else 0, B, C, dz.data_ptr(), acc.data_ptr(), _st())
    # the reference is evaluated on the fp32-rounded logits' float64 values, so the comparison measures the kernel only
    zr32 = zd.double().cpu().requires_grad_(True)
    want = _ce_reference(zr32, y, rn, lam)
    want.backward()
    got = acc.item()
    assert abs(got - want.item()) <= 1e-5 * max(abs(want.item()), 1e-6), (got, want.item())
    ref_g = zr32.grad
    row_max = ref_g.abs().amax(dim=1, keepdim=True).clamp_min(1e-30)
    err = ((dz.double().cpu() - ref_g).abs() / row_max).max().item()
    assert err <= 1e-5, err


def test_ce_loss_large_logits_keep_relative_accuracy():
    """lse - z for logits around 1e3 with a small loss: no cancellation of lse against z"""
    B, C = 4, 50
    z = torch.full((B, C), 1000.0, dtype=torch.float64)
    z[:, 7] = 1012.0
    y = torch.full((B,), 7, dtype=torch.long)
    want = F.cross_entropy(z, y)
    zd, yd = z.float().cuda(), y.int().cuda()
    acc = torch.zeros(1, device="cuda", dtype=torch.float64)
    lib().ce_loss(zd.data_ptr(), yd.data_ptr(), 0, 0, 0, B, C, 0, acc.data_ptr(), _st())
    assert abs(acc.item() - want.item()) <= 1e-5 * want.item(), (acc.item(), want.item())


def test_ce_loss_index_out_of_range_gives_nan_and_empty_batch_is_noop():
    z = torch.randn(3, 10, device="cuda")
    y = torch.tensor([1, 10, 2], device="cuda", dtype=torch.int32)
    acc = torch.zeros(1, device="cuda", dtype=torch.float64)
    lib().ce_loss(z.data_ptr(), y.data_ptr(), 0, 0, 0, 3, 10, 0, acc.data_ptr(), _st())
    assert np.isnan(acc.item())
    acc.zero_()
    lib().ce_loss(z.data_ptr(), y.data_ptr(), 0, 0, 0, 0, 10, 0, acc.data_ptr(), _st())
    assert acc.item() == 0.0


def _openmic_reference(z, batch, rn, lam):
    """ex_openmic.py:101-121, float64"""
    bs = z.shape[0]
    y_mask = batch[:, 20:]
    y = (batch[:, :20] > 0.5).double()
    if rn is not None:
        y_mix = y * lam.reshape(bs, 1) + y[rn] * (1. - lam.reshape(bs, 1))
    else:
        y_mix = y
    samples_loss = F.binary_cross_entropy_with_logits(z, y_mix, reduction="none")
    return (y_mask.double() * samples_loss).mean()


@pytest.mark.parametrize("B", [1, 5, 64])
@pytest.mark.parametrize("mix", [False, True])
def test_bce_masked_loss_matches_openmic_expression(B, mix):
    g = torch.Generator().manual_seed(B + 100 * mix)
    C = 20
    z = torch.randn(B, C, generator=g, dtype=torch.float64) * 3
    batch = torch.rand(B, 2 * C, generator=g, dtype=torch.float64)          # soft targets: binarised by the loss
    batch[:, C:] = (batch[:, C:] > 0.4).double()                             # the 0/1 mask of observed labels
    rn = torch.randperm(B, generator=g) if mix else None
    lam = (torch.rand(B, generator=g, dtype=torch.float64) * 0.5 + 0.5) if mix else None
    zd, bd = z.float().cuda(), batch.float().cuda()
    rn_d = rn.int().cuda() if mix else None
    lam_d = lam.float().cuda() if mix else None
    zr = zd.double().cpu().requires_grad_(True)
    want = _openmic_reference(zr, bd.double().cpu(), rn, lam_d.double().cpu() if mix else None)
    want.backward()
    dz = torch.empty(B, C, device="cuda")
    acc = torch.zeros(1, device="cuda", dtype=torch.float64)
    lib().bce_masked_loss(zd.data_ptr(), bd.data_ptr(), 2 * C, bd[:, C:].data_ptr(), 2 * C,
                          rn_d.data_ptr() if mix else 0, lam_d.data_ptr() if mix else 0, B, C, dz.data_ptr(),
                          acc.data_ptr(), _st())
    assert abs(acc.item() - want.item()) <= 2e-6 * max(1.0, abs(want.item())), (acc.item(), want.item())
    assert (dz.double().cpu() - zr.grad).abs().max().item() <= 1e-5 * zr.grad.abs().max().item() + 1e-12


def _mixstyle_reference(x, lmda, perm, eps=1e-6):
    """helpers/utils.py:106-119 with the draws given"""
    f_mu = x.mean(dim=[1, 3], keepdim=True)
    f_var = x.var(dim=[1, 3], keepdim=True)
    f_sig = (f_var + eps).sqrt()
    x_normed = (x - f_mu) / f_sig
    f_mu_perm, f_sig_perm = f_mu[perm], f_sig[perm]
    mu_mix = f_mu * lmda + f_mu_perm * (1 - lmda)
    sig_mix = f_sig * lmda + f_sig_perm * (1 - lmda)
    return x_normed * sig_mix + mu_mix


def _run_mixstyle(x, lmda, perm, eps=1e-6):
    B, _, F_, T = x.shape
    out = torch.empty_like(x)
    stats = torch.empty(2 * B * F_, device=x.device)
    perm_d, lam_d = perm.int().cuda(), lmda.reshape(B).float().cuda()
    lib().mixstyle(x.data_ptr(), perm_d.data_ptr(), lam_d.data_ptr(), eps, stats.data_ptr(), out.data_ptr(), B, F_, T, _st())
    return out


@pytest.mark.parametrize("B,F_,T", [(6, 128, 501), (1, 128, 101), (4, 64, 2), (3, 7, 1000), (64, 128, 33)])
def test_mixstyle_matches_reference(B, F_, T):
    g = torch.Generator().manual_seed(B * T + F_)
    # log-mel-like rows: a mean around -1 and a spread of ~0.2 (the case where E[x^2] - E[x]^2 would cancel)
    x = (torch.randn(B, 1, F_, 1, generator=g) * 0.3 - 1.0) + torch.randn(B, 1, F_, T, generator=g) * 0.2
    x[0, 0, 0] = 5.0                                            # a constant row: sigma = sqrt(eps)
    lmda = torch.distributions.Beta(0.4, 0.4).sample((B, 1, 1, 1))
    perm = torch.randperm(B, generator=g)
    xd = x.cuda()
    got = _run_mixstyle(xd, lmda, perm).double().cpu()
    want = _mixstyle_reference(xd.double().cpu(), lmda.double(), perm)
    err = (got - want).abs().max().item()
    assert err <= 1e-5 * max(1.0, want.abs().max().item()), err


def test_mixstyle_helper_draws_like_the_reference():
    """helpers.utils.mixstyle consumes np.random.rand, Beta(alpha, alpha).sample((B,1,1,1)) and torch.randperm(B) in
    the reference's order: the same seeds give the reference's output and (perm, lambda)"""
    from torch.distributions.beta import Beta

    from efficientat_b200.helpers.utils import mixstyle
    B, F_, T = 5, 16, 40
    x = torch.randn(B, 1, F_, T, generator=torch.Generator().manual_seed(3)) * 0.5 - 2.0
    np.random.seed(11)
    torch.manual_seed(12)
    out, perm, lmda = mixstyle(x.cuda(), p=1.0, alpha=0.4, mix_labels=True)
    np.random.seed(11)
    torch.manual_seed(12)
    assert not np.random.rand() > 1.0
    want_l = Beta(0.4, 0.4).sample((B, 1, 1, 1))
    want_p = torch.randperm(B)
    assert torch.equal(perm.cpu(), want_p) and torch.equal(lmda.cpu(), want_l)
    want = _mixstyle_reference(x.double(), want_l.double(), want_p)
    assert (out.double().cpu() - want).abs().max().item() <= 1e-5 * want.abs().max().item()
    xc = x.cuda()
    assert mixstyle(xc, p=0.0) is xc                            # skipped (rand() > p): x itself comes back
    with pytest.raises(NotImplementedError):
        mixstyle(x.cuda().requires_grad_(True), p=1.0)
