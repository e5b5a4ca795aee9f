"""The DyMN kernels one by one against float64 torch restatements of the DyMN expressions (reference
models/dymn/dy_block.py, line numbers next to each section), at batch sizes other than two; a DyMN training step at
B = 5 against the fp64 oracle (oracle/net_oracle.py) under both GEMM routes and in bf16 storage; and the C-ABI argument
checks that fire before any launch (no GPU needed).

Every backward reference is autograd of the forward expression.  Tolerances, stated again at each assertion:
  - fp32 element-wise outputs: per element 1e-6 of |ref| plus a floor of 1e-6 of the magnitude of the terms that
    make it up (1e-5 for the k*k-term depthwise outputs), which covers cancellation;
  - reductions (pooled means, sums over pixels or samples, BatchNorm sums): tol * sum |terms| per entry (_close_sum);
  - GEMM outputs in fp32 storage: 2e-4 of the tensor's max (bf16x3 products, as tests/test_gpu_gemm.py);
  - bf16 storage: against fp64 from the bf16-rounded inputs; one output rounding is 2^-8 of |ref| per element, GEMMs
    keep 2e-2 of the max.
"""
import pytest
import torch
import torch.nn.functional as Fn

from efficientat_b200._lib import EatError, lib
from tests import dymn_util as du
from tests.util import report

RELU, HS = 1, 2
F32, BF16 = 0, 1
DT = {F32: torch.float32, BF16: torch.bfloat16}
BF16_REL = 2.0 ** -8


def _st():
    return torch.cuda.current_stream().cuda_stream


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _p(t):
    return 0 if t is None else t.data_ptr()


def _close(got, ref, tol, what):
    """GEMM outputs: max error within tol of the tensor's max"""
    err = (got.double() - ref.double()).abs().max().item()
    scale = ref.double().abs().max().item()
    assert err <= tol * scale + 1e-12, f"{what}: max error {err:.3e} vs scale {scale:.3e}"
    return err / max(scale, 1e-30)


def _close_sum(got, ref, mag, tol, what):
    """reductions: each entry within tol of the sum of the magnitudes of its terms"""
    err = (got.double() - ref.double()).abs()
    bound = tol * mag.double() + 1e-30
    worst = (err / bound).max().item()
    assert bool((err <= bound).all()), f"{what}: worst error / bound {worst:.3f}"
    return worst


def _close_elem(got, ref, rel, floor, what):
    """element-wise outputs: |got - ref| <= rel * |ref| + floor (floor: a scalar or a per-element magnitude)"""
    err = (got.double() - ref.double()).abs()
    bound = rel * ref.double().abs() + floor
    worst = (err / bound).max().item()
    assert bool((err <= bound).all()), f"{what}: worst error / bound {worst:.3f}"
    return worst


# ------------------------------------------------------------------------------------------------ DyReLU-B * CoordAtt
# p = max(u a1 + b1, u a2 + b2) * ca_f * ca_t, u = z * scale + shift, (a1, a2, b1, b2) = (2 theta - 1) * lam + init
# (dy_block.py:157-188, 195-201, 400-402)
DY_ACT_CASES = [  # (B, Fo, To, C)
    (1, 64, 1, 16),        # one output column, the widest Fo
    (3, 5, 31, 72),        # partial 32-column block, partial 32-channel chunk
    (5, 8, 33, 120),       # two column blocks, the second with one column
    (3, 16, 101, 184),
    (1, 64, 250, 200),
    (5, 2, 250, 16),
]


def _dy_inputs(B, Fo, To, C, dtype, seed):
    g = _gen(seed)
    r = lambda *s: torch.randn(*s, device="cuda", generator=g)
    u = lambda *s: torch.rand(*s, device="cuda", generator=g)
    d = dict(z=r(B, Fo, To, C), scale=u(C) + 0.5, shift=r(C) * 0.3, theta=u(B, C, 4), lam=torch.tensor(
        [1.0, 1.0, 0.5, 0.5], device="cuda"), init=torch.tensor([1.0, 0.0, 0.0, 0.0], device="cuda"),
        ca_f=u(B, Fo, C), ca_t=u(B, To, C), dp=r(B, Fo, To, C))
    d["z"] = d["z"].to(DT[dtype])
    d["dp"] = d["dp"].to(DT[dtype])
    # keep every pixel away from the kink of the max (|l1 - l2| >= 1e-3): there fp32 and fp64 may pick different
    # branches, and the gradient jumps
    for _ in range(4):
        co = _coef(d)
        uu = _u(d)
        near = (uu * co[:, None, None, :, 0] + co[:, None, None, :, 2] - uu * co[:, None, None, :, 1]
                - co[:, None, None, :, 3]).abs() < 1e-3
        if not bool(near.any()):
            break
        d["z"] = torch.where(near, (d["z"].float() + 0.37).to(DT[dtype]), d["z"])
    return d


def _coef(d):
    return (2 * d["theta"].double() - 1) * d["lam"].double() + d["init"].double()     # [B, C, 4]


def _u(d):
    return d["z"].double() * d["scale"].double() + d["shift"].double()


def _dy_act_ref(u, co, caf, cat):
    a1, a2, b1, b2 = (co[:, None, None, :, j] for j in range(4))
    return torch.maximum(u * a1 + b1, u * a2 + b2) * caf[:, :, None, :] * cat[:, None, :, :]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [F32, BF16], ids=["f32", "bf16"])
@pytest.mark.parametrize("case", DY_ACT_CASES, ids=lambda c: "B{}_Fo{}_To{}_C{}".format(*c))
def test_dy_act_fwd_bwd_match_fp64(case, dtype):
    B, Fo, To, C = case
    L, st = lib(), _st()
    d = _dy_inputs(B, Fo, To, C, dtype, seed=B * 1000 + Fo * 10 + To + C)
    P = [d[n].data_ptr() for n in ("scale", "shift", "theta", "lam", "init", "ca_f", "ca_t")]
    out = torch.full_like(d["z"], float("nan"))
    L.dy_act_fwd(d["z"].data_ptr(), out.data_ptr(), dtype, *P, B, Fo, To, C, st)

    u = _u(d).requires_grad_(True)
    co = _coef(d).requires_grad_(True)
    caf = d["ca_f"].double().requires_grad_(True)
    cat = d["ca_t"].double().requires_grad_(True)
    ref = _dy_act_ref(u, co, caf, cat)
    # fp32: a few roundings of terms of size |u a| + |b| before the two gate products; bf16: one output rounding more
    q = d["ca_f"].double()[:, :, None, :] * d["ca_t"].double()[:, None, :, :]
    mag = (u.detach().abs() * co.detach()[:, None, None, :, :2].abs().amax(-1)
           + co.detach()[:, None, None, :, 2:].abs().amax(-1)) * q
    rel = 1e-6 if dtype == F32 else BF16_REL
    w_fwd = _close_elem(out, ref.detach(), rel, 1e-6 * mag + 1e-30, "dy_act_fwd")

    # backward: dcaf / dcoef accumulate onto what is there, dcat / du are overwritten
    g = _gen(7)
    dcaf0 = torch.randn(B, Fo, C, device="cuda", generator=g)
    dcoef0 = torch.randn(B, C, 4, device="cuda", generator=g)
    dcaf, dcoef = dcaf0.clone(), dcoef0.clone()
    dcat = torch.full((B, To, C), float("nan"), device="cuda")
    du = torch.full_like(d["z"], float("nan"))
    L.dy_act_bwd(d["dp"].data_ptr(), d["z"].data_ptr(), du.data_ptr(), dtype, *P, dcaf.data_ptr(), dcat.data_ptr(),
                 dcoef.data_ptr(), B, Fo, To, C, st)
    gp = d["dp"].double()
    ref.backward(gp)
    # magnitudes of the terms of each reduction: dr = g ca_f ca_t goes to the selected branch's (a, b)
    a1, a2, b1, b2 = (co.detach()[:, None, None, :, j] for j in range(4))
    uu = u.detach()
    l1, l2 = uu * a1 + b1, uu * a2 + b2
    sel = l1 >= l2
    r = torch.where(sel, l1, l2)
    dr = (gp * q).abs()
    m_caf = (gp * r * d["ca_t"].double()[:, None, :, :]).abs().sum(2) + dcaf0.double().abs()
    m_cat = (gp * r * d["ca_f"].double()[:, :, None, :]).abs().sum(1)
    m_coef = torch.stack([(dr * uu.abs() * sel).sum((1, 2)), (dr * uu.abs() * ~sel).sum((1, 2)),
                          (dr * sel).sum((1, 2)), (dr * ~sel).sum((1, 2))], -1) + dcoef0.double().abs()
    # reductions in fp32 over at most Fo (per thread) and To (across the CTA) terms: 1e-5 of sum |terms|
    w_caf = _close_sum(dcaf, dcaf0.double() + caf.grad, m_caf, 1e-5, "dcaf")
    w_cat = _close_sum(dcat, cat.grad, m_cat, 1e-5, "dcat")
    w_coef = _close_sum(dcoef, dcoef0.double() + co.grad, m_coef, 1e-5, "dcoef")
    # du = dr * (selected slope): one product chain; bf16 adds one output rounding
    w_du = _close_elem(du, u.grad, rel, 1e-6 * dr * co.detach()[:, None, None, :, :2].abs().amax(-1) + 1e-30, "du")
    report(f"[kernel] dy_act {case} {'bf16' if dtype else 'f32'}: worst error/bound fwd {w_fwd:.2f} du {w_du:.2f} "
           f"dcaf {w_caf:.2f} dcat {w_cat:.2f} dcoef {w_coef:.2f}")


# ------------------------------------------------------------------------------------------------ ContextGen pooling
# out[b] = [mean over T of x[b, f] | mean over F of x[b, :, t]]  (dy_block.py:236-240); backward added onto dx
CTX_CASES = [(2, 7, 13, 16), (3, 64, 1, 24), (1, 1, 50, 72), (5, 32, 101, 72), (4, 40, 250, 16)]   # (B, F, T, C)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [F32, BF16], ids=["f32", "bf16"])
@pytest.mark.parametrize("case", CTX_CASES, ids=lambda c: "B{}_F{}_T{}_C{}".format(*c))
def test_ctx_pool_fwd_bwd_match_fp64(case, dtype):
    B, F, T, C = case
    if dtype == BF16 and C % 8:
        pytest.skip("bf16 ContextGen pooling takes channel counts that are multiples of 8")
    L, st = lib(), _st()
    g = _gen(B + F + T + C)
    x = torch.randn(B, F, T, C, device="cuda", generator=g).to(DT[dtype])
    out = torch.full((B, F + T, C), float("nan"), device="cuda")
    L.ctx_pool(x.data_ptr(), dtype, out.data_ptr(), B, F, T, C, st)
    xd = x.double().requires_grad_(True)
    ref = torch.cat([xd.mean(2), xd.mean(1)], 1)
    mag = torch.cat([xd.detach().abs().mean(2), xd.detach().abs().mean(1)], 1)
    w_f = _close_sum(out, ref.detach(), mag, 1e-5, "ctx_pool")          # means in fp32: 1e-5 of mean |terms|

    dg = torch.randn(B, F + T, C, device="cuda", generator=g)
    dx0 = torch.randn(B, F, T, C, device="cuda", generator=g).to(DT[dtype])
    dx = dx0.clone()
    L.ctx_pool_bwd(dg.data_ptr(), dx.data_ptr(), dtype, B, F, T, C, st)
    ref.backward(dg.double())
    rdx = dx0.double() + xd.grad
    # three terms per element: 1e-6 of their magnitude in fp32, plus one bf16 rounding of the result
    mag_dx = dx0.double().abs() + dg.double()[:, :F, None, :].abs() / T + dg.double()[:, None, F:, :].abs() / F
    w_b = _close_elem(dx, rdx, 1e-6 if dtype == F32 else BF16_REL, 1e-6 * mag_dx + 1e-30, "ctx_pool_bwd")
    report(f"[kernel] ctx_pool {case} {'bf16' if dtype else 'f32'}: worst error/bound fwd {w_f:.2f} bwd {w_b:.2f}")


# ------------------------------------------------------------------------------------------------ sequence pooling
# rows [row0, row0 + L) of in [B, Ltot, H] -> AvgPool(3, stride, pad 1, count_include_pad) or a copy (stride 1),
# optionally act(x * scale + shift) on load  (dy_block.py:227-233, 249)
SEQ_CASES = [  # (B, Ltot, row0, L, H, stride, affine)
    (1, 1, 0, 1, 32, 1, False), (3, 5, 2, 3, 40, 1, True), (2, 165, 64, 101, 32, 1, True),
    (1, 1, 0, 1, 32, 2, False), (3, 2, 0, 2, 40, 2, True), (2, 7, 4, 3, 32, 2, False),
    (3, 165, 0, 64, 56, 2, True), (3, 165, 64, 101, 56, 2, True), (5, 300, 64, 101, 120, 2, False),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", SEQ_CASES, ids=lambda c: "B{}_Ltot{}_row{}_L{}_H{}_s{}{}".format(*c[:6], "_aff" if c[6] else ""))
def test_seq_pool_fwd_bwd_match_fp64(case):
    B, Ltot, row0, L_, H, s, aff = case
    L, st = lib(), _st()
    g = _gen(Ltot + row0 + L_ + H + s)
    x = torch.randn(B, Ltot, H, device="cuda", generator=g)
    sc = torch.rand(H, device="cuda", generator=g) + 0.5 if aff else None
    sh = torch.randn(H, device="cuda", generator=g) * 0.3 if aff else None
    Lo = (L_ - 1) // s + 1
    out = torch.full((B, Lo, H), float("nan"), device="cuda")
    L.seq_pool(x.data_ptr(), out.data_ptr(), B, Ltot, row0, L_, H, s, _p(sc), _p(sh), HS if aff else 0, st)
    # the reference runs on the CPU: torch's CUDA avg_pool1d backward on the transposed (channels-last) view of this
    # layout gives wrong gradients for the last window
    rows = x.double().cpu()[:, row0:row0 + L_]
    tmag = rows.abs()
    if aff:
        pre = rows * sc.double().cpu() + sh.double().cpu()
        tmag = 2 * ((rows * sc.double().cpu()).abs() + sh.double().cpu().abs())   # |x sc| + |sh|, hardswish slope <= 1.5
        rows = Fn.hardswish(pre)
    rows = rows.requires_grad_(True)

    def pool(v):
        if s == 1:
            return v
        return Fn.avg_pool1d(v.transpose(1, 2).contiguous(), 3, s, 1, count_include_pad=True).transpose(1, 2)
    ref = pool(rows)
    assert ref.shape == out.shape
    # at most three terms per output: 1e-6 of their magnitude (with the affine + hardswish on load: of the magnitude of
    # the pre-activation terms, whose rounding hardswish carries over near its zero at -3)
    w_f = _close_elem(out.cpu(), ref.detach(), 1e-6, 1e-6 * pool(tmag) + 1e-30, "seq_pool")

    dout = torch.randn(B, Lo, H, device="cuda", generator=g)
    dsrc = torch.full((B, Ltot, H), 12345.0, device="cuda")          # rows outside the window keep this sentinel
    L.seq_pool_bwd(dout.data_ptr(), dsrc.data_ptr(), B, Ltot, row0, L_, H, s, st)
    ref.backward(dout.double().cpu())
    keep = torch.ones(Ltot, dtype=torch.bool, device="cuda")
    keep[row0:row0 + L_] = False
    assert bool((dsrc[:, keep] == 12345.0).all()), "seq_pool_bwd wrote outside rows [row0, row0 + L)"
    # at most three terms per entry (the backward stops before the affine + activation, which the caller differentiates)
    w_b = _close_elem(dsrc[:, row0:row0 + L_].cpu(), rows.grad, 1e-6,
                      1e-6 * pool_t_abs(dout.double().cpu().abs(), L_, s) + 1e-30, "seq_pool_bwd")
    report(f"[kernel] seq_pool {case}: worst error/bound fwd {w_f:.2f} bwd {w_b:.2f}")


def pool_t_abs(dabs, L_, s):
    """transposed pooling of |dout|: the magnitude of the terms of each dsrc entry"""
    if s == 1:
        return dabs
    v = torch.zeros(dabs.shape[0], L_, dabs.shape[2], dtype=dabs.dtype, device=dabs.device, requires_grad=True)
    out = Fn.avg_pool1d(v.transpose(1, 2).contiguous(), 3, s, 1, count_include_pad=True).transpose(1, 2)
    (gv,) = torch.autograd.grad(out, v, dabs)
    return gv


# ------------------------------------------------------------------------------------------------ DynamicConv attention
# att = softmax((h_c Wr^T + br) / T)  (dy_block.py:104-107); backward: dWr, dbr, dh_c accumulated
ATT_CASES = [(B, H, k, T) for (B, H), k, T in zip([(1, 32), (4, 56), (5, 120), (9, 128), (9, 56), (5, 32), (4, 128),
                                                  (1, 120)], [1, 2, 3, 4, 4, 3, 2, 1], [30.0, 1.0] * 4)]


@pytest.mark.gpu
@pytest.mark.parametrize("case", ATT_CASES, ids=lambda c: "B{}_H{}_k{}_T{:g}".format(*c))
def test_dyconv_att_fwd_bwd_match_fp64(case):
    B, H, k, T = case
    L, st = lib(), _st()
    g = _gen(B * 100 + H + k)
    hc = torch.randn(B, H, device="cuda", generator=g)
    wr = torch.randn(k, H, device="cuda", generator=g) / H ** 0.5 * 4
    br = torch.randn(k, device="cuda", generator=g)
    att = torch.full((B, k), float("nan"), device="cuda")
    L.dyconv_att(hc.data_ptr(), wr.data_ptr(), br.data_ptr(), T, att.data_ptr(), B, H, k, st)
    hd, wd, bd = (t.double().requires_grad_(True) for t in (hc, wr, br))
    ref = torch.softmax((hd @ wd.t() + bd) / T, -1)
    # each logit is an fp32 dot product over H: its error is a few ulp of sum |w h|, and exp turns the logit error into
    # a relative error of att
    lmag = ((hc.double().abs() @ wr.double().abs().t()) + br.double().abs()) / T
    w_f = _close_elem(att, ref.detach(), 1e-6, 1e-5 * ref.detach() * lmag.amax(1, keepdim=True) + 1e-30, "dyconv_att")

    datt = torch.randn(B, k, device="cuda", generator=g)
    dwr0, dbr0, dhc0 = (torch.randn(*s, device="cuda", generator=g) for s in ((k, H), (k,), (B, H)))
    dwr, dbr, dhc = dwr0.clone(), dbr0.clone(), dhc0.clone()
    att_in = ref.detach().float()
    L.dyconv_att_bwd(datt.data_ptr(), att_in.data_ptr(), T, hc.data_ptr(), wr.data_ptr(), dwr.data_ptr(), dbr.data_ptr(),
                     dhc.data_ptr(), B, H, k, st)
    (ref * datt.double()).sum().backward()
    a = att_in.double()
    dl_mag = a * (datt.double().abs() + (a * datt.double().abs()).sum(1, keepdim=True)) / T        # |terms| of dlogit
    # sums over the samples (atomics) and over the kernels: 1e-5 of sum |terms|
    w_wr = _close_sum(dwr, dwr0.double() + wd.grad, dl_mag.t() @ hc.double().abs() + dwr0.double().abs(), 1e-5, "dWr")
    w_br = _close_sum(dbr, dbr0.double() + bd.grad, dl_mag.sum(0) + dbr0.double().abs(), 1e-5, "dbr")
    w_hc = _close_sum(dhc, dhc0.double() + hd.grad, dl_mag @ wr.double().abs() + dhc0.double().abs(), 1e-5, "dh_c")
    report(f"[kernel] dyconv_att {case}: worst error/bound att {w_f:.2f} dWr {w_wr:.2f} dbr {w_br:.2f} dh_c {w_hc:.2f}")


# ------------------------------------------------------------------------------------------------ depthwise weight mix
# wt[b, tap, c] = sum_j att[b, j] W[j, c, tap]  (dy_block.py:111-117)
@pytest.mark.gpu
@pytest.mark.parametrize("ksize", [3, 5])
def test_dyconv_mix_dw_matches_fp64(ksize):
    L, st = lib(), _st()
    g = _gen(ksize)
    for B, C, k in [(1, 16, 4), (2, 72, 4), (3, 13, 1), (5, 120, 3), (7, 200, 2), (9, 960, 4)]:
        W = torch.randn(k, C, ksize * ksize, device="cuda", generator=g)
        att = torch.softmax(torch.randn(B, k, device="cuda", generator=g), 1)
        wt = torch.full((B, ksize * ksize, C), float("nan"), device="cuda")
        L.dyconv_mix_dw(W.data_ptr(), att.data_ptr(), wt.data_ptr(), B, C, ksize, k, st)
        ref = torch.einsum("bj,jct->btc", att.double(), W.double())
        mag = torch.einsum("bj,jct->btc", att.double(), W.double().abs())
        _close_sum(wt, ref, mag, 1e-6, f"dyconv_mix_dw B{B} C{C} k{k}")        # <= 4 fp32 products: 1e-6 of sum |terms|


# ------------------------------------------------------------------------------------------------ element-wise backward
# dpre = dcoef * lam * 2 s (1 - s) (dy_block.py:157-160, 179); out = g * s (1 - s); transpose
@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 12, 4 * 200 * 4 + 3, 132 * 16 * 256 + 1001, 3 * 132 * 16 * 256 + 7])
def test_elementwise_backward_kernels_match_fp64(n):
    L, st = lib(), _st()
    g = _gen(n % 1000)
    dc, s, lam = torch.randn(n, device="cuda", generator=g), torch.rand(n, device="cuda", generator=g), \
        torch.tensor([1.0, 1.0, 0.5, 0.5], device="cuda")
    out = torch.full((n,), float("nan"), device="cuda")
    L.dyrelu_coef_bwd(dc.data_ptr(), s.data_ptr(), lam.data_ptr(), out.data_ptr(), n, st)
    sd = s.double()
    ref = dc.double() * lam.double().repeat((n + 3) // 4)[:n] * 2 * sd * (1 - sd)
    _close_elem(out, ref, 1e-6, 1e-30, "dyrelu_coef_bwd")               # a product of five factors: 1e-6 relative
    out.fill_(float("nan"))
    L.sigmoid_bwd(dc.data_ptr(), s.data_ptr(), out.data_ptr(), n, st)
    _close_elem(out, dc.double() * sd * (1 - sd), 1e-6, 1e-30, "sigmoid_bwd")


@pytest.mark.gpu
def test_transpose_is_exact():
    L, st = lib(), _st()
    g = _gen(3)
    for R, Cc in [(1, 1), (4, 4), (37, 53), (1000, 33), (33, 1000), (240, 40), (8, 960)]:
        x = torch.randn(R, Cc, device="cuda", generator=g)
        y = torch.full((Cc, R), float("nan"), device="cuda")
        L.transpose_f32(x.data_ptr(), y.data_ptr(), R, Cc, st)
        assert torch.equal(y, x.t()), (R, Cc)


# ------------------------------------------------------------------------------------------------ DynamicConv bank grads
# dW[k] += sum_b att[b, k] S[b];  datt[b, k] = <S[b], W[k]>  (autograd of the mix W_b = sum_k att[b, k] W[k])
DYMN20_WIDEST = 1920 * 320          # dymn20: the 1920-channel expansion projected to 320 channels


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 2, 3, 4, 5, 8, 13])
def test_dyn_wgrad_mix_matches_fp64(B):
    """B = 4, 8 take only the four-sample main loop, 1-3 only the tail, 5 and 13 both"""
    L, st = lib(), _st()
    g = _gen(B)
    worst = [0.0, 0.0]
    for k in (1, 2, 3, 4):
        for n in (4, 4 * 2501, DYMN20_WIDEST):
            S = torch.randn(B, n, device="cuda", generator=g)
            att = torch.softmax(torch.randn(B, k, device="cuda", generator=g), 1)
            W = torch.randn(k, n, device="cuda", generator=g)
            dW0 = torch.randn(k, n, device="cuda", generator=g)
            dW = dW0.clone()
            datt = torch.full((B, k), float("nan"), device="cuda")
            L.dyn_wgrad_mix(S.data_ptr(), att.data_ptr(), W.data_ptr(), dW.data_ptr(), datt.data_ptr(), B, n, k, st)
            Wd = W.double().requires_grad_(True)
            ad = att.double().requires_grad_(True)
            (torch.einsum("bk,kn->bn", ad, Wd) * S.double()).sum().backward()
            # dW: B fp32 products per entry added to the prefill; datt: a sum over n products; both 1e-5 of sum |terms|
            worst[0] = max(worst[0], _close_sum(dW, dW0.double() + Wd.grad, att.double().t() @ S.double().abs()
                                                + dW0.double().abs(), 1e-5, f"dW k{k} n{n}"))
            worst[1] = max(worst[1], _close_sum(datt, ad.grad, S.double().abs() @ W.double().abs().t(), 1e-5,
                                                f"datt k{k} n{n}"))
    report(f"[kernel] dyn_wgrad_mix B={B}: worst error/bound dW {worst[0]:.2f} datt {worst[1]:.2f}")


# ------------------------------------------------------------------------------------------------ DynamicConv 1x1 GEMM
# C = epi(A_b . (sum_j att[b, j] W_j)^T) per sample (dy_block.py:103-131), register-staged kernel (below ~400 rows
# per sample in the engine)
DYN_CASES = [  # (B, rps, N, K, nk)
    (64, 28, 24, 72, 4), (9, 37, 40, 16, 3), (33, 104, 72, 24, 2), (5, 399, 16, 120, 1), (64, 104, 200, 80, 4),
    (2, 37, 8, 8, 4), (17, 399, 112, 480, 3),
]


def _dyn_ref(A, W, att, rps):
    B = att.shape[0]
    Wb = torch.einsum("bj,jnk->bnk", att.double(), W.double())
    return torch.einsum("brk,bnk->brn", A.double().view(B, rps, -1), Wb).reshape(A.shape[0], -1)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [F32, BF16], ids=["f32", "bf16"])
@pytest.mark.parametrize("case", DYN_CASES, ids=lambda c: "B{}_rps{}_N{}_K{}_k{}".format(*c))
def test_pw_tc_dyn_fwd_matches_fp64(case, dtype):
    B, rps, N, K, nk = case
    L, st = lib(), _st()
    g = _gen(B + rps + N + K)
    M = B * rps
    A = torch.randn(M, K, device="cuda", generator=g).to(DT[dtype])
    W = torch.randn(nk, N, K, device="cuda", generator=g) / K ** 0.5
    att = torch.softmax(torch.randn(B, nk, device="cuda", generator=g), 1)
    sc = torch.stack([torch.rand(N, device="cuda", generator=g) + 0.5, torch.randn(N, device="cuda", generator=g) * 0.1])
    res = torch.randn(M, N, device="cuda", generator=g).to(DT[dtype])
    raw = _dyn_ref(A, W, att, rps)
    tol = 2e-4 if dtype == F32 else 2e-2          # bf16x3 products / one bf16 operand rounding (test_gpu_gemm.py)
    worst = 0.0
    for variant in ("stats", "scale_act", "scale_res"):
        C = torch.full((M, N), float("nan"), device="cuda").to(DT[dtype])
        stats = torch.zeros(2, N, device="cuda", dtype=torch.float64) if variant == "stats" else None
        s0, s1, act, r = (0, 0, 0, None) if variant == "stats" else (sc[0].data_ptr(), sc[1].data_ptr(),
                                                                    HS if variant == "scale_act" else 0,
                                                                    res if variant == "scale_res" else None)
        L.pw_tc_dyn_fwd(A.data_ptr(), dtype, W.data_ptr(), att.data_ptr(), nk, C.data_ptr(), M, N, K, rps, 0, 0, 0, s0, s1,
                        act, _p(r), _p(stats[0]) if stats is not None else 0, _p(stats[1]) if stats is not None else 0, st)
        ref = raw
        if variant != "stats":
            ref = ref * sc[0].double() + sc[1].double()
        if variant == "scale_act":
            ref = Fn.hardswish(ref)
        if variant == "scale_res":
            ref = ref + res.double()
        worst = max(worst, _close(C, ref, tol, f"pw_tc_dyn_fwd {variant}"))
        if stats is not None:     # fp64 sums of the fp32 results: the GEMM's own error, 1e-3 of the largest sum (3e-2 bf16)
            stol = 1e-3 if dtype == F32 else 3e-2
            _close(stats[0], raw.sum(0), stol, "stat_sum")
            _close(stats[1], (raw * raw).sum(0), stol, "stat_sq")
    report(f"[kernel] pw_tc_dyn_fwd {case} {'bf16' if dtype else 'f32'}: max error / max |ref| {worst:.2e}")
    # the input BatchNorm + activation on load is not offered with dynamic weights: refused, not silently ignored
    C = torch.empty(M, N, device="cuda").to(DT[dtype])
    isc, ish = torch.ones(K, device="cuda"), torch.zeros(K, device="cuda")
    with pytest.raises(EatError, match=r"code 3\): .*not instantiated for DynamicConv"):
        L.pw_tc_dyn_fwd(A.data_ptr(), dtype, W.data_ptr(), att.data_ptr(), nk, C.data_ptr(), M, N, K, rps, isc.data_ptr(),
                        ish.data_ptr(), RELU, 0, 0, 0, 0, 0, 0, st)


# ------------------------------------------------------------------------------------------------ per-sample weight grads
# S[b] = G_b^T . X_b  (the DynamicConv 1x1 weight gradient before the bank mix)
PS_CASES = [  # (B, rps, N, K)
    (1, 37, 24, 72), (3, 101, 64, 16), (7, 37, 40, 120), (3, 4000, 72, 24), (7, 101, 200, 80),
    (64, 6464, 64, 16),     # dymn10 block 2 at B = 64: four splits per sample, each walks more 64-row blocks than
                            # the ring has stages, and the last split of each sample is shorter than the others
]
GUARD = 256


def _persample_check(S, G, X, B, rps, N, K, tol, what):
    body = S[: B * N * K].view(B, N, K)
    assert bool((S[B * N * K:] == -777.0).all()), f"{what}: wrote past the last sample's slice"
    ref = torch.einsum("brn,brk->bnk", G.double().view(B, rps, N), X.double().view(B, rps, K))
    worst = 0.0
    for b in range(B):            # each sample on its own scale
        worst = max(worst, _close(body[b], ref[b], tol, f"{what} sample {b}"))
    return worst


def _guarded(B, N, K):
    S = torch.zeros(B * N * K + GUARD, device="cuda")
    S[B * N * K:] = -777.0
    return S


@pytest.mark.gpu
@pytest.mark.parametrize("case", PS_CASES, ids=lambda c: "B{}_rps{}_N{}_K{}".format(*c))
def test_persample_wgrad_matches_fp64(case):
    B, rps, N, K = case
    L, st = lib(), _st()
    g = _gen(B * 7 + rps + N + K)
    M = B * rps
    G = torch.randn(M, N, device="cuda", generator=g)
    X = torch.randn(M, K, device="cuda", generator=g)
    S = _guarded(B, N, K)                           # fp32: the TMA kernel through the entry point the engine calls
    L.pw_tc_wgrad_persample(G.data_ptr(), X.data_ptr(), F32, S.data_ptr(), M, N, K, rps, st)
    w32 = _persample_check(S, G, X, B, rps, N, K, 2e-4, "pw_tc_wgrad_persample f32")
    S = _guarded(B, N, K)                           # the same kernel called directly in per-sample mode
    L.pw_tma_wgrad(G.data_ptr(), X.data_ptr(), S.data_ptr(), M, N, K, 0, 0, 0, 0, rps, 1, st)
    wt = _persample_check(S, G, X, B, rps, N, K, 2e-4, "pw_tma_wgrad per_sample")
    Gb, Xb = G.bfloat16(), X.bfloat16()             # bf16 storage: the register-staged wgmma kernel
    S = _guarded(B, N, K)
    L.pw_tc_wgrad_persample(Gb.data_ptr(), Xb.data_ptr(), BF16, S.data_ptr(), M, N, K, rps, st)
    wb = _persample_check(S, Gb, Xb, B, rps, N, K, 2e-2, "pw_tc_wgrad_persample bf16")
    report(f"[kernel] per-sample wgrad {case}: max error / max |ref| f32 {w32:.2e} tma {wt:.2e} bf16 {wb:.2e}")


# ------------------------------------------------------------------------------------------------ depthwise, per sample
# DynamicConv depthwise (dy_block.py:111-131) with per-sample tap-major tables wt [B][k*k][C]; forward with BN affine +
# DyReLU-B + CoordAtt (eval, dy_block.py:172-201) or raw output + BatchNorm sums (training, input BN + act on load);
# data gradient (+ residual) and weight gradient per sample
DW_CASES = [(k, s, B) for (k, s), B in zip([(3, 1), (3, 2), (5, 1), (5, 2)] * 2, [1, 3, 5, 3, 5, 1, 3, 5])]
DW_SHAPE = {1: (13, 37, 24), 3: (16, 33, 72), 5: (9, 20, 40)}      # B -> (F, T, C)


def _dw_tables(B, C, k, g, pad=8):
    kk = k * k
    bstride = kk * C + pad                                        # a gap between the tables: the stride is honoured
    buf = torch.full((B * bstride + GUARD,), float("nan"), device="cuda")
    w = torch.randn(B, kk, C, device="cuda", generator=g) / k
    for b in range(B):
        buf[b * bstride: b * bstride + kk * C] = w[b].flatten()
    return buf, bstride, w


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [F32, BF16], ids=["f32", "bf16"])
@pytest.mark.parametrize("case", DW_CASES, ids=lambda c: "k{}_s{}_B{}".format(*c))
def test_dw_conv_dy_fwd_matches_fp64(case, dtype):
    k, s, B = case
    F, T, C = DW_SHAPE[B]
    L, st = lib(), _st()
    g = _gen(k * 10 + s + B)
    Fo, To = (F - 1) // s + 1, (T - 1) // s + 1
    x = torch.randn(B, F, T, C, device="cuda", generator=g).to(DT[dtype])
    buf, bstride, w = _dw_tables(B, C, k, g)
    d = _dy_inputs(B, Fo, To, C, F32, seed=k + s + B)
    rel = 1e-6 if dtype == F32 else BF16_REL
    wd = w.double()
    conv = du.conv_ps(x.double(), wd, k, s)
    cmag = du.conv_ps(x.double().abs(), wd.abs(), k, s)
    # eval form: BN affine + DyReLU-B + CoordAtt on the conv output
    out = torch.full((B, Fo, To, C), float("nan"), device="cuda").to(DT[dtype])
    L.dw_conv_fwd_dy(x.data_ptr(), buf.data_ptr(), bstride, out.data_ptr(), dtype, B, F, T, C, k, s, 0, 0, 0,
                     d["scale"].data_ptr(), d["shift"].data_ptr(), d["theta"].data_ptr(), d["lam"].data_ptr(),
                     d["init"].data_ptr(), d["ca_f"].data_ptr(), d["ca_t"].data_ptr(), 0, 0, st)
    co = _coef(d)
    u = conv * d["scale"].double() + d["shift"].double()
    ref = _dy_act_ref(u, co, d["ca_f"].double(), d["ca_t"].double())
    q = d["ca_f"].double()[:, :, None, :] * d["ca_t"].double()[:, None, :, :]
    mag = ((cmag * d["scale"].double() + d["shift"].double().abs()) * co[:, None, None, :, :2].abs().amax(-1)
           + co[:, None, None, :, 2:].abs().amax(-1)) * q
    # k*k fp32 products then the epilogue: 1e-5 of the magnitude of the terms; bf16 adds one output rounding
    w_e = _close_elem(out, ref, rel, 1e-5 * mag + 1e-30, "dw_conv_fwd_dy eval")
    # training form: the input's BatchNorm + activation on load, raw output, fp64 BatchNorm sums of the output
    isc = torch.rand(C, device="cuda", generator=g) + 0.5
    ish = torch.randn(C, device="cuda", generator=g) * 0.3
    out.fill_(float("nan"))
    stats = torch.zeros(2, C, device="cuda", dtype=torch.float64)
    L.dw_conv_fwd_dy(x.data_ptr(), buf.data_ptr(), bstride, out.data_ptr(), dtype, B, F, T, C, k, s, isc.data_ptr(),
                     ish.data_ptr(), HS, 0, 0, 0, 0, 0, 0, 0, stats[0].data_ptr(), stats[1].data_ptr(), st)
    xf = Fn.hardswish(x.double() * isc.double() + ish.double())
    raw = du.conv_ps(xf, wd, k, s)
    rmag = du.conv_ps(xf.abs(), wd.abs(), k, s)
    w_t = _close_elem(out, raw, rel, 1e-5 * rmag + 1e-30, "dw_conv_fwd_dy training")
    # BatchNorm sums over B*Fo*To fp32 values (of the unrounded result): 1e-5 of sum |terms|
    w_s = _close_sum(stats[0], raw.sum((0, 1, 2)), rmag.sum((0, 1, 2)), 1e-5, "stat_sum")
    w_q = _close_sum(stats[1], (raw * raw).sum((0, 1, 2)), (rmag * rmag).sum((0, 1, 2)), 1e-5, "stat_sq")
    report(f"[kernel] dw_conv_fwd_dy {case} {'bf16' if dtype else 'f32'}: worst error/bound eval {w_e:.2f} "
           f"training {w_t:.2f} sums {w_s:.2f} / {w_q:.2f}")


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [F32, BF16], ids=["f32", "bf16"])
@pytest.mark.parametrize("case", DW_CASES, ids=lambda c: "k{}_s{}_B{}".format(*c))
def test_dw_conv_per_sample_backward_matches_fp64(case, dtype):
    k, s, B = case
    F, T, C = DW_SHAPE[B]
    L, st = lib(), _st()
    g = _gen(k * 100 + s * 10 + B)
    Fo, To = (F - 1) // s + 1, (T - 1) // s + 1
    kk = k * k
    x = torch.randn(B, F, T, C, device="cuda", generator=g).to(DT[dtype])
    dz = torch.randn(B, Fo, To, C, device="cuda", generator=g).to(DT[dtype])
    isc = torch.rand(C, device="cuda", generator=g) + 0.5
    ish = torch.randn(C, device="cuda", generator=g) * 0.3
    # weight gradient: per-sample slices dw[b] [C, k, k] at stride C*k*k, a guard after the last one
    dw = torch.zeros(B * C * kk + GUARD, device="cuda")
    dw[B * C * kk:] = -777.0
    L.dw_conv_wgrad(dz.data_ptr(), x.data_ptr(), isc.data_ptr(), ish.data_ptr(), RELU, dw.data_ptr(), C * kk, dtype, B, F,
                    T, C, k, s, st)
    assert bool((dw[B * C * kk:] == -777.0).all()), "dw_conv_wgrad wrote past the last sample's slice"
    xf = torch.relu(x.double() * isc.double() + ish.double())
    wv = torch.zeros(B, kk, C, dtype=torch.float64, device="cuda", requires_grad=True)
    (du.conv_ps(xf, wv, k, s) * dz.double()).sum().backward()
    wabs = torch.zeros(B, kk, C, dtype=torch.float64, device="cuda", requires_grad=True)
    (du.conv_ps(xf.abs(), wabs, k, s) * dz.double().abs()).sum().backward()
    to_ck = lambda t: t.permute(0, 2, 1).reshape(B, C * kk)                 # [B, k*k, C] -> [B, C*k*k] (dw [C,1,k,k])
    # a sum over Fo*To products per entry, fp32: 1e-5 of sum |terms|
    w_w = _close_sum(dw[: B * C * kk].view(B, C * kk), to_ck(wv.grad), to_ck(wabs.grad), 1e-5, "dw_conv_wgrad")
    # data gradient with per-sample tables (+ residual)
    buf, bstride, w = _dw_tables(B, C, k, g)
    worst = 0.0
    for with_res in (False, True):
        res = torch.randn(B, F, T, C, device="cuda", generator=g).to(DT[dtype]) if with_res else None
        din = torch.full((B, F, T, C), float("nan"), device="cuda").to(DT[dtype])
        L.dw_conv_dgrad(dz.data_ptr(), buf.data_ptr(), bstride, _p(res), din.data_ptr(), dtype, B, F, T, C, k, s, st)
        xv = torch.zeros(B, F, T, C, dtype=torch.float64, device="cuda", requires_grad=True)
        (du.conv_ps(xv, w.double(), k, s) * dz.double()).sum().backward()
        xa = torch.zeros(B, F, T, C, dtype=torch.float64, device="cuda", requires_grad=True)
        (du.conv_ps(xa, w.double().abs(), k, s) * dz.double().abs()).sum().backward()
        ref, mag = xv.grad, xa.grad
        if res is not None:
            ref, mag = ref + res.double(), mag + res.double().abs()
        # at most k*k products per element: 1e-5 of their magnitude, plus one bf16 output rounding
        worst = max(worst, _close_elem(din, ref, 1e-6 if dtype == F32 else BF16_REL, 1e-5 * mag + 1e-30,
                                       f"dw_conv_dgrad res={with_res}"))
    report(f"[kernel] dw per-sample backward {case} {'bf16' if dtype else 'f32'}: worst error/bound wgrad {w_w:.2f} "
           f"dgrad {worst:.2f}")


# ------------------------------------------------------------------------------------------------ C-ABI argument checks
def test_dymn_entry_points_reject_bad_arguments_before_any_launch():
    L = lib()
    fake = 4096                                                   # never dereferenced: validation comes first
    with pytest.raises(EatError, match=r"code 3\): .*1\.\.4 kernels"):
        L.dyconv_att_bwd(fake, fake, 30.0, fake, fake, fake, fake, fake, 4, 64, 5, 0)
    with pytest.raises(EatError, match=r"code 3\): .*1\.\.4 kernels"):
        L.dyconv_att_bwd(fake, fake, 30.0, fake, fake, fake, fake, fake, 4, 64, 0, 0)
    with pytest.raises(EatError, match=r"code 3\): .*1\.\.4 kernels"):
        L.dyconv_att(fake, fake, fake, 30.0, fake, 4, 64, 5, 0)
    for stride in (0, -2):
        with pytest.raises(EatError, match=r"code 1\): .*stride must be at least 1"):
            L.seq_pool(fake, fake, 2, 165, 64, 101, 32, stride, 0, 0, 0, 0)
        with pytest.raises(EatError, match=r"code 1\): .*stride must be at least 1"):
            L.seq_pool_bwd(fake, fake, 2, 165, 64, 101, 32, stride, 0)
    for Ltot, row0, L_ in ((164, 64, 101), (165, -1, 10), (165, 0, 0)):
        with pytest.raises(EatError, match=r"code 1\): .*must lie inside \[0, Ltot\)"):
            L.seq_pool(fake, fake, 2, Ltot, row0, L_, 32, 2, 0, 0, 0, 0)
        with pytest.raises(EatError, match=r"code 1\): .*must lie inside \[0, Ltot\)"):
            L.seq_pool_bwd(fake, fake, 2, Ltot, row0, L_, 32, 1, 0)
    with pytest.raises(EatError, match=r"code 3\): .*1\.\.4 kernels"):
        L.dyn_wgrad_mix(fake, fake, fake, fake, fake, 5, 4096, 5, 0)
    with pytest.raises(EatError, match=r"code 1\): .*multiple of 4"):
        L.dyn_wgrad_mix(fake, fake, fake, fake, fake, 5, 4098, 4, 0)
    for S, W, dW in ((fake + 4, fake, fake), (fake, fake + 8, fake), (fake, fake, fake + 12)):
        with pytest.raises(EatError, match=r"code 1\): .*16-byte aligned"):
            L.dyn_wgrad_mix(S, fake, W, dW, fake, 5, 4096, 4, 0)
    with pytest.raises(EatError, match=r"code 1\): .*multiple of 4"):
        L.dy_act_fwd(fake, fake, 0, fake, fake, fake, fake, fake, fake, fake, 3, 8, 33, 70, 0)
    with pytest.raises(EatError, match=r"code 1\): .*multiple of 4"):
        L.dy_act_bwd(fake, fake, fake, 0, fake, fake, fake, fake, fake, fake, fake, fake, fake, fake, 3, 8, 33, 70, 0)
    with pytest.raises(EatError, match=r"code 1\): .*M must be B \* rows_per_sample"):
        L.pw_tc_dyn_fwd(fake, 0, fake, fake, 4, fake, 5 * 37 + 1, 24, 72, 37, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0)
    with pytest.raises(EatError, match=r"code 1\): .*M must be B \* rows_per_sample"):
        L.pw_tc_dyn_fwd(fake, 0, fake, fake, 4, fake, 5 * 37, 24, 72, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0)


# ------------------------------------------------------------------------------------------------ training step at B = 5
TRAIN_B, TRAIN_FRAMES = 5, 201
TRAIN_ROUTES, BOUNDS = du.TRAIN_ROUTES, du.BOUNDS
_ORACLE = {}


def _train_inputs():
    return du.train_inputs(TRAIN_B, TRAIN_FRAMES)


def _oracle(tag, temperature):
    """fp64 oracle training step (CPU, autograd): loss, logits, gradients, BatchNorm buffers after the step, eval
    logits (the golden state's BatchNorm buffers were calibrated on other clips, and on these the eval-mode network
    saturates, logits ~1e10: calibrated on this batch); cached per tag for the routes that share it"""
    if tag not in _ORACLE:
        _ORACLE[tag] = du.oracle_step(tag, temperature, *_train_inputs())
    return _ORACLE[tag]


def _engine_step(tag, precision, gemm, dyn_tma_min_rps=None):
    return du.engine_step(tag, precision, gemm, *_train_inputs(), dyn_tma_min_rps=dyn_tma_min_rps)


@pytest.mark.gpu
@pytest.mark.parametrize("route", list(TRAIN_ROUTES))
@pytest.mark.parametrize("tag", ["dymn04", "dymn10"])
def test_dymn_train_step_b5_matches_fp64_oracle(tag, route):
    """One DyMN training step at B = 5 (not a multiple of four), 201 frames, dropout off, against autograd through the
    fp64 oracle: loss, logits, every BatchNorm running statistic and EVERY full gradient tensor.
    Routes: gemm 'simt' (exact fp32 everywhere, DynamicConv in the reference's order); 'auto' with every DynamicConv 1x1
    on the TMA kernels (dyn_tma_min_rps = 0) and with every one on the register-staged kernels (dyn_tma_min_rps huge).

    Measured on an H100 80GB HBM3 over three runs each (fp32 atomics make runs differ), dymn04 / dymn10:
      simt:  gradient relative L2 <= 6.6e-4 / 3.1e-3 (attention-logit layers 2.9e-3 / 7.5e-3), norms <= 2.7e-5 / 4.6e-4
             (3.2e-3), logits 4.4e-6, BatchNorm buffers 8.7e-8;
      auto:  relative L2 <= 2.3e-2 / 6.9e-2 (attention-logit layers 3.5e-2 / 9.5e-2), norms <= 7.4e-3 / 1.8e-2 (7.5e-2),
             logits 8.8e-5, BatchNorm buffers 2.4e-6, both DynamicConv routes alike.
    The norm bounds are the batch-2 golden bands of tests/test_gpu_dymn.py (5e-3 / 2e-2 simt, 3e-2 / 0.2 auto) or
    tighter, with no tensor exempt; relative L2 over the whole tensor is the stricter measure and gets about twice the
    worst figure.  The one analytically-zero gradient (a BatchNorm bias whose shift the next training-mode BatchNorm
    removes; fp64 gives 1e-9 of the gradient norm) is bounded against the whole gradient's norm (measured 1.5e-9)."""
    gemm, min_rps = TRAIN_ROUTES[route]
    ref = _oracle(tag, du.temperature(tag))
    model, loss, logits = _engine_step(tag, "fp32", gemm, min_rps)
    du.check_train_step(f"{tag} B={TRAIN_B} train", route, model, loss, logits, ref)


@pytest.mark.gpu
@pytest.mark.parametrize("tag", ["dymn04", "dymn10"])
def test_dymn_eval_b5_matches_fp64_oracle(tag):
    """eval forward at B = 5, exact-fp32 route: logits within 1e-4 of the fp64 oracle"""
    from tests.util import build_model
    ref = _oracle(tag, du.temperature(tag))
    spec, _ = _train_inputs()
    model = build_model(tag)
    with torch.no_grad():
        for k, v in model.state_dict().items():
            if k in ref["cal"]:
                v.copy_(ref["cal"][k])
    model = model.cuda().eval()
    model.engine().gemm_impl = "simt"
    with torch.no_grad():
        logits, _ = model(spec.cuda())
    err = (logits.double().cpu() - ref["eval_logits"]).abs().max().item()
    report(f"[parity] {tag} B={TRAIN_B} eval gemm=simt: logit max-abs err {err:.2e} "
           f"(logits up to {ref['eval_logits'].abs().max().item():.2e})")
    assert err < 1e-4                                # measured 2.6e-5 / 1.3e-5 (dymn04 / dymn10)


@pytest.mark.gpu
def test_dymn_bf16_train_step_b5_against_fp64_oracle():
    """bf16 activation storage, dymn04, B = 5: the whole gradient's cosine against the fp64 oracle and every tensor's
    relative L2.  Coarse bounds: bf16 rounds every stored activation to 2^-9, and the BatchNorm backward of this
    calibrated synthetic state amplifies rounding by ~1e3-1e4 (the exact-fp32 route turns 6e-8 into 3e-3).  Measured on
    an H100 80GB HBM3 over three runs: cosine 0.940-0.945, logits 4.3e-2, classifier gradients <= 1.9e-2, out_c BatchNorm
    3.4e-2; from the out_c conv on, every tensor 0.2-0.6 (median 0.42, max 1.1 / 1.6; attention-logit layers up to 5.2).
    The error appears at the last BatchNorm's backward and stays level through the network instead of growing in any
    one DyMN layer: amplified rounding, not a kernel defect (the kernels alone pass the bf16 cases above)."""
    tag = "dymn04"
    ref = _oracle(tag, du.temperature(tag))
    model, loss, logits = _engine_step(tag, "bf16", "auto")
    rel, zero, _ = du.grad_errors(du.grads_of(model), ref)
    names = [n for n, _ in model.named_parameters()]
    g = torch.cat([dict(model.named_parameters())[n].grad.detach().double().cpu().flatten() for n in names])
    r = torch.cat([ref["grads"][n].flatten() for n in names])
    cos = Fn.cosine_similarity(g, r, dim=0).item()
    lerr = (logits - ref["logits"]).abs().max().item()
    res_rel = max(v for n, v in rel.items() if ".residuals." in n)
    oth = sorted(((v, n) for n, v in rel.items() if ".residuals." not in n), reverse=True)
    report(f"[parity] {tag} B={TRAIN_B} bf16 train: loss {abs(loss - ref['loss']):.2e}, logits {lerr:.2e}, cosine "
           f"{cos:.6f}, grad rel-L2 max {oth[0][0]:.2e} ({oth[0][1]}), median {oth[len(oth) // 2][0]:.2e}, "
           f"attention-logit layers {res_rel:.2e}")
    head = max(v for n, v in rel.items() if n.startswith("classifier."))
    report(f"[parity] {tag} B={TRAIN_B} bf16 train: classifier gradients rel-L2 max {head:.2e}")
    assert cos > 0.9
    assert lerr < 0.1
    assert head < 5e-2
    assert oth[len(oth) // 2][0] < 0.6 and oth[0][0] < 3.0 and res_rel < 10.0
