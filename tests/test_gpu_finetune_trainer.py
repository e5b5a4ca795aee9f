"""FineTuneTrainer.step against the loop bodies of the four fine-tuning scripts written with autograd around this
package's model (ex_esc50.py:98-126, ex_dcase20.py:98-131, ex_fsd50k.py:97-125, ex_openmic.py:97-127): torch ops for
the augmentation and the loss, loss.backward(), torch.optim.Adam and LambdaLR.  Same mel jitter draws, same mixup /
MixStyle draws.  mn04 and dymn04 at B = 5, eager and CUDA graph; the bounds and their rationale are those of
tests/test_gpu_train_step.py::test_trainer_step_matches_reference_loop_with_autograd, with DyMN's noisier updates bounded
separately (see below).  Measured on an H100 80GB HBM3 at a 700 W power limit, worst over the 20 cases (mn04 / dymn04):
step-1 loss 2.0e-6 / 3.1e-6 relative, steps 1-3 3.3e-5 / 6.7e-5; whole update vector 1.8e-2 / 5.0e-2 relative L2; worst
tightly bounded tensor 0.13 / 0.15; worst loosely bounded tensor 0.71 / 0.75."""
import contextlib
import io

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from efficientat_b200.helpers.utils import exp_warmup_linear_down
from efficientat_b200.synth import set_bn_stats, synth_state_, synth_waveform
from tests.util import NETS, golden, report

pytestmark = pytest.mark.gpu

B = 5
# (script, loss mode, classes, target form, mixup, mixstyle_p)
CASES = {"esc50": ("ce", 50, "prob", True, 0.0), "dcase20": ("ce", 10, "index", True, 0.0),
         "dcase20_mixstyle": ("ce", 10, "index", True, 1.0), "fsd50k": ("bce", 200, "multi", True, 0.0),
         "openmic": ("bce_masked", 20, "masked", True, 0.0)}


def _build(tag, num_classes):
    kind, width, _, _ = NETS[tag]
    if kind == "mn":
        from efficientat_b200.models.mn.model import get_model
    else:
        from efficientat_b200.models.dymn.model import get_model
    torch.manual_seed(0)
    with contextlib.redirect_stdout(io.StringIO()):
        m = get_model(width_mult=width, num_classes=num_classes, verbose=False)
    synth_state_(m, seed=7)
    g = golden(tag)
    m = set_bn_stats(m, g["cal_rm"], g["cal_rv"]).cuda()
    for mod in m.modules():
        if isinstance(mod, torch.nn.Dropout):
            mod.p = 0.0
    return m


def _mel():
    from efficientat_b200.models.preprocess import AugmentMelSTFT
    with contextlib.redirect_stdout(io.StringIO()):
        return AugmentMelSTFT(freqm=0, timem=0).cuda()


def _targets(form, C, seed):
    g = torch.Generator().manual_seed(seed)
    if form == "index":
        return torch.randint(0, C, (B,), generator=g)
    if form == "prob":                                         # one-hot rows, one blended as by waveform mixing
        y = F.one_hot(torch.randint(0, C, (B,), generator=g), C).float()
        y[1] = 0.7 * y[1] + 0.3 * y[2]
        return y
    if form == "multi":
        return (torch.rand(B, C, generator=g) < 0.05).float()
    y = torch.rand(B, 2 * C, generator=g)                       # OpenMIC: soft targets | 0/1 mask
    y[:, C:] = (y[:, C:] > 0.3).float()
    return y


def _mixstyle_torch(x, p, alpha, eps=1e-6):
    """the reference's MixStyle as torch ops on the device, with its host draws in its order"""
    if np.random.rand() > p:
        return x
    bs = x.size(0)
    mu = x.mean(dim=[1, 3], keepdim=True)
    sig = (x.var(dim=[1, 3], keepdim=True) + eps).sqrt()
    lmda = torch.distributions.Beta(alpha, alpha).sample((bs, 1, 1, 1)).to(x.device)
    perm = torch.randperm(bs).to(x.device)
    return (x - mu) / sig * (sig * lmda + sig[perm] * (1 - lmda)) + mu * lmda + mu[perm] * (1 - lmda)


def _script_loss(mode, y_hat, y, rn, lam):
    """the loss statements of the scripts' loops (rn is None: no mixup)"""
    bs = y_hat.shape[0]
    if mode == "ce":
        if rn is None:
            return F.cross_entropy(y_hat, y, reduction="none").mean()
        return (F.cross_entropy(y_hat, y, reduction="none") * lam.reshape(bs) +
                F.cross_entropy(y_hat, y[rn], reduction="none") * (1. - lam.reshape(bs))).mean()
    if mode == "bce_masked":
        y_mask = y[:, 20:]
        y = (y[:, :20] > 0.5).float()
    if rn is not None:
        y = y * lam.reshape(bs, 1) + y[rn] * (1. - lam.reshape(bs, 1))
    loss = F.binary_cross_entropy_with_logits(y_hat, y, reduction="none")
    if mode == "bce_masked":
        loss = y_mask.float() * loss
    return loss.mean()


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("tag", ["mn04", "dymn04"])
@pytest.mark.parametrize("case", list(CASES))
def test_finetune_step_matches_script_loop_with_autograd(case, tag, graph):
    from efficientat_b200.finetune import FineTuneTrainer
    mode, C, form, mix, ms_p = CASES[case]
    sched = exp_warmup_linear_down(2, 4, 1, 0.1)
    wave = synth_waveform(B, 32000, seed=3).cuda()
    y = _targets(form, C, seed=4).cuda()
    draws = [(torch.randperm(B, generator=torch.Generator().manual_seed(10 + i)),
              torch.rand(B, generator=torch.Generator().manual_seed(20 + i)) * 0.5 + 0.5) for i in range(3)]

    # ---- the script's loop body (autograd around this package's modules)
    model, mel = _build(tag, C), _mel()
    model.train(); mel.train()
    p_before = {n: p.detach().clone() for n, p in model.named_parameters()}
    opt = torch.optim.Adam(model.parameters(), lr=4e-4)
    lr_sched = torch.optim.lr_scheduler.LambdaLR(opt, sched)
    ref_losses, gnorm = [], {}
    torch.manual_seed(77)
    np.random.seed(78)
    for i, (rn, lam) in enumerate(draws):
        x = mel(wave).unsqueeze(1)
        if ms_p > 0:
            x = _mixstyle_torch(x, ms_p, 0.4)
            rn_d = lam_d = None
        else:
            lam_d, rn_d = lam.cuda(), rn.cuda()
            x = x * lam_d.reshape(B, 1, 1, 1) + x[rn_d] * (1. - lam_d.reshape(B, 1, 1, 1))
        y_hat, _ = model(x)
        loss = _script_loss(mode, y_hat, y, rn_d, lam_d)
        loss.backward()
        if i == 0:
            gnorm = {n: p.grad.norm().item() for n, p in model.named_parameters()}
        opt.step()
        opt.zero_grad()
        lr_sched.step()
        ref_losses.append(loss.item())
    ref_delta = {n: (p.detach() - p_before[n]) for n, p in model.named_parameters()}

    # ---- trainer
    model2, mel2 = _build(tag, C), _mel()
    tr = FineTuneTrainer(model2, mel2, loss=mode, lr=4e-4, mixup_alpha=0.3 if mix else 0.0, mixstyle_p=ms_p,
                         cuda_graph=graph, schedule=sched)
    torch.manual_seed(77)
    np.random.seed(78)
    losses = []
    for i, (rn, lam) in enumerate(draws):
        tr.set_epoch(i)
        out = tr.step(wave, y) if ms_p > 0 else tr.step(wave, y, perm=rn, lam=lam)
        assert out.dtype == torch.float64 and out.is_cuda and out.dim() == 0
        losses.append(out.item())
    # step 1 pins the loss kernels (same logits up to the network's own fp32 noise); steps 2-3 follow two Adam updates,
    # whose sign-like first steps amplify that noise (see the update bounds below)
    err1 = abs(losses[0] - ref_losses[0]) / abs(ref_losses[0])
    err = max(abs(a - r) / abs(r) for a, r in zip(losses, ref_losses))
    assert err1 <= 1e-5 and err <= 2e-4, (losses, ref_losses)
    gmax = max(gnorm.values())
    skipped = 0
    num = den = 0.0
    ratios = {}
    for n, p in model2.named_parameters():
        if gnorm[n] < 1e-5 * gmax:
            skipped += 1
            continue
        d = p.detach() - p_before[n]
        diff, ref_n = (d - ref_delta[n]).norm().item(), max(ref_delta[n].norm().item(), 1e-12)
        num += diff ** 2
        den += ref_n ** 2
        ratios[n] = diff / ref_n
    total = (num / den) ** 0.5
    # Adam's first steps move every element by ~lr * sign(g), so an element whose gradient is within the fp32 noise of
    # the step flips its whole update.  Loosely bounded (1.5: the sign of the update is right on most of the tensor)
    # are the tensors where that decides the comparison: small vectors (<= 64 elements, e.g. one BatchNorm of mn04's
    # early blocks, measured up to 0.81), tensors whose gradient is below 1e-3 of the largest, and DyMN's
    # attention-logit layers (".residuals.", O(1e-6) gradients; tests/test_gpu_dymn.py gives their norms 0.2-0.3 in
    # one step).  A wrong learning rate, schedule factor or loss scale moves every tensor and the total.
    loose = {n for n, p in model2.named_parameters() if n in ratios and
             (".residuals." in n or gnorm[n] < 1e-3 * gmax or p.numel() <= 64)}
    tight = {n: r for n, r in ratios.items() if n not in loose}
    worst = max(tight, key=tight.get)
    worst_loose = max((ratios[n] for n in loose), default=0.0)
    report(f"[parity] finetune {case} {tag} graph={graph}: loss rel err step 1 {err1:.2e}, steps 1-3 {err:.2e}; update rel err "
           f"{total:.2e}, worst tensor {tight[worst]:.2e} ({worst}), worst loose {worst_loose:.2e} ({len(loose)}), "
           f"{skipped} zero-gradient tensors skipped")
    assert tight[worst] <= 0.3, (worst, tight[worst], gnorm[worst])
    assert worst_loose <= 1.5, worst_loose
    assert total <= (5e-2 if tag.startswith("mn") else 0.1), total
    assert skipped < 40


def test_finetune_trainer_rejects_bad_inputs():
    from efficientat_b200.finetune import FineTuneTrainer
    model, mel = _build("mn04", 10), _mel()
    wave = synth_waveform(2, 32000, seed=3).cuda()
    with pytest.raises(ValueError):
        FineTuneTrainer(model, mel, loss="mse")
    with pytest.raises(ValueError):
        FineTuneTrainer(model, mel, loss="bce", mixstyle_p=0.5)
    tr = FineTuneTrainer(model, mel, loss="ce")
    with pytest.raises(ValueError):
        tr.step(wave, torch.zeros(2, device="cuda"))                     # float class indices
    with pytest.raises(ValueError):
        tr.step(wave, torch.zeros(2, 11, device="cuda"))                 # wrong class count
    with pytest.raises(RuntimeError):
        tr.step(wave, torch.zeros(2, dtype=torch.long))                  # targets on the host
    tr = FineTuneTrainer(_build("mn04", 20), mel, loss="bce_masked")
    with pytest.raises(ValueError):
        tr.step(wave, torch.zeros(2, 20, device="cuda"))                 # targets without the mask half
