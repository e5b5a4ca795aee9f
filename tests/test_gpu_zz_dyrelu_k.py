"""DyReLU-B with M = 1, 3, 4 linear pieces on the GPU: each entry point that takes M against float64 torch autograd of
the DyReLU-B expression (reference models/dymn/dy_block.py:157-188, 195-201), eval parity with the reference's goldens
(tests/golden/make_golden_dyrelu_k.py), a B = 5 training step against the fp64 oracle of tests/dyrelu_util.py with a
planted defect that must be caught, and the trainers.

Tolerances, as tests/test_gpu_zz_dymn_kernels.py states them: fp32 element-wise outputs within 1e-6 of |ref| plus a
floor of 1e-6 (1e-5 for the k*k-term depthwise outputs) of the magnitude of their terms; sums within 1e-5 of the sum of
the magnitudes of their terms; bf16 storage adds one output rounding (2^-8 of |ref|)."""
import contextlib
import io

import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

from efficientat_b200._lib import lib
from tests import dyrelu_util as du
from tests.util import fmap_digest, golden, report, topk_match

F32, BF16 = 0, 1
DT = {F32: torch.float32, BF16: torch.bfloat16}
BF16_REL = 2.0 ** -8
PIECES = [1, 3, 4]


def _st():
    return torch.cuda.current_stream().cuda_stream


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _close_elem(got, ref, rel, floor, what):
    err = (got.double() - ref.double()).abs()
    bound = rel * ref.double().abs() + floor
    worst = (err / bound).max().item()
    assert bool((err <= bound).all()), f"{what}: worst error / bound {worst:.3f}"
    return worst


def _close_sum(got, ref, mag, tol, what):
    err = (got.double() - ref.double()).abs()
    bound = tol * mag.double() + 1e-30
    worst = (err / bound).max().item()
    assert bool((err <= bound).all()), f"{what}: worst error / bound {worst:.3f}"
    return worst


def _buffers(M):
    lam = torch.tensor([1.0] * M + [0.5] * M, device="cuda")
    init = torch.tensor([1.0] + [0.0] * (2 * M - 1), device="cuda")
    return lam, init


def _coef(theta, lam, init):
    return (2 * theta.double() - 1) * lam.double() + init.double()              # [B, C, 2M]


def _pieces(u, co, M):
    """[B, Fo, To, C, M] lines a_m u + b_m; u [B, Fo, To, C], co [B, C, 2M]"""
    return u.unsqueeze(-1) * co[:, None, None, :, :M] + co[:, None, None, :, M:]


def _dyrelu(u, co, M):
    return _pieces(u, co, M).max(-1)[0]


def _away_from_kinks(z, scale, shift, co, M, dtype, margin=1e-3):
    """moves every pixel whose two largest pieces lie within margin of each other: there fp32 and fp64 may pick different
    pieces and the gradient jumps"""
    for _ in range(8):
        if M == 1:
            return z
        lines = _pieces(z.double() * scale.double() + shift.double(), co, M)
        top = lines.topk(2, -1)[0]
        near = (top[..., 0] - top[..., 1]) < margin
        if not bool(near.any()):
            return z
        z = torch.where(near, (z.float() + 0.37).to(DT[dtype]), z)
    raise AssertionError("could not move the inputs away from the kinks")


# ------------------------------------------------------------------------------------------------ dy_act_fwd/bwd_m
ACT_CASES = [(1, 1, 1, 16), (5, 7, 33, 72), (37, 3, 9, 24), (5, 1, 250, 40)]   # (B, Fo, To, C): odd, 1, partial blocks


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [F32, BF16], ids=["f32", "bf16"])
@pytest.mark.parametrize("M", PIECES)
@pytest.mark.parametrize("case", ACT_CASES, ids=lambda c: "B{}_Fo{}_To{}_C{}".format(*c))
def test_dy_act_m_matches_fp64(case, M, dtype):
    B, Fo, To, C = case
    L, st = lib(), _st()
    g = _gen(B * 131 + Fo * 17 + To + C + M)
    r = lambda *s: torch.randn(*s, device="cuda", generator=g)
    u_ = lambda *s: torch.rand(*s, device="cuda", generator=g)
    scale, shift = u_(C) + 0.5, r(C) * 0.3
    theta, (lam, init) = u_(B, C, 2 * M), _buffers(M)
    ca_f, ca_t = u_(B, Fo, C), u_(B, To, C)
    co0 = _coef(theta, lam, init)
    z = _away_from_kinks(r(B, Fo, To, C).to(DT[dtype]), scale, shift, co0, M, dtype)
    dp = r(B, Fo, To, C).to(DT[dtype])
    P = [t.data_ptr() for t in (scale, shift, theta, lam, init, ca_f, ca_t)]
    out = torch.full_like(z, float("nan"))
    L.dy_act_fwd_m(z.data_ptr(), out.data_ptr(), dtype, *P, M, B, Fo, To, C, st)
    u = (z.double() * scale.double() + shift.double()).requires_grad_(True)
    co = co0.clone().requires_grad_(True)
    caf, cat = ca_f.double().requires_grad_(True), ca_t.double().requires_grad_(True)
    ref = _dyrelu(u, co, M) * caf[:, :, None, :] * cat[:, None, :, :]
    q = ca_f.double()[:, :, None, :] * ca_t.double()[:, None, :, :]
    mag = (u.detach().abs().unsqueeze(-1) * co0[:, None, None, :, :M].abs() + co0[:, None, None, :, M:].abs()).amax(-1) * q
    rel = 1e-6 if dtype == F32 else BF16_REL
    w_f = _close_elem(out, ref.detach(), rel, 1e-6 * mag + 1e-30, f"dy_act_fwd_m M={M}")
    # backward: dcaf / dcoef accumulate onto what is there, dcat / du are overwritten
    dcaf0, dcoef0 = r(B, Fo, C), r(B, C, 2 * M)
    dcaf, dcoef = dcaf0.clone(), dcoef0.clone()
    dcat = torch.full((B, To, C), float("nan"), device="cuda")
    du = torch.full_like(z, float("nan"))
    L.dy_act_bwd_m(dp.data_ptr(), z.data_ptr(), du.data_ptr(), dtype, *P, dcaf.data_ptr(), dcat.data_ptr(),
                   dcoef.data_ptr(), M, B, Fo, To, C, st)
    ref.backward(dp.double())
    # magnitudes of the terms of each gradient (same expression with |.|)
    ua, coa = u.detach().abs(), co0.abs()
    dpa, qa = dp.double().abs(), q
    lines = _pieces(u.detach(), co0, M)
    sel = torch.nn.functional.one_hot(lines.argmax(-1), M).double()     # the piece each pixel's gradient goes to
    # a slope is (2 theta - 1) lam + init in fp32, as the reference computes it: for piece 0 (init 1) with theta near 0
    # that sum cancels, so the slope's error is relative to the magnitude of its terms, not to its value
    tmag = ((2 * theta.double() - 1).abs() * lam.double() + init.double().abs())[:, None, None, :, :M]
    slope = (sel * tmag).sum(-1)
    w_u = _close_elem(du, u.grad, rel, 1e-6 * dpa * qa * slope + 1e-30, f"dy_act_bwd_m du M={M}")
    rmag = (ua.unsqueeze(-1) * coa[:, None, None, :, :M] + coa[:, None, None, :, M:]).amax(-1)
    w_cf = _close_sum(dcaf, dcaf0.double() + caf.grad, dcaf0.double().abs() + (dpa * rmag * ca_t.double()[:, None]).sum(2),
                      1e-5, "dcaf")
    w_ct = _close_sum(dcat, cat.grad, (dpa * rmag * ca_f.double()[:, :, None]).sum(1), 1e-5, "dcat")
    gd = (dpa * qa).unsqueeze(-1) * sel
    cmag = torch.cat([(gd * ua.unsqueeze(-1)).sum((1, 2)), gd.sum((1, 2))], -1)            # [B, C, 2M]
    w_co = _close_sum(dcoef, dcoef0.double() + co.grad, dcoef0.double().abs() + cmag, 1e-5, "dcoef")
    report(f"[kernel] dy_act_m M={M} {case} {'bf16' if dtype else 'f32'}: worst error/bound fwd {w_f:.2f} du {w_u:.2f} "
           f"dcaf {w_cf:.2f} dcat {w_ct:.2f} dcoef {w_co:.2f}")


@pytest.mark.gpu
@pytest.mark.parametrize("M", PIECES)
def test_dyrelu_coef_bwd_m_matches_fp64(M):
    B, C = 5, 40
    g = _gen(M)
    dcoef = torch.randn(B, C, 2 * M, device="cuda", generator=g)
    s = torch.rand(B, C, 2 * M, device="cuda", generator=g)
    lam, _ = _buffers(M)
    out = torch.full_like(s, float("nan"))
    lib().dyrelu_coef_bwd_m(dcoef.data_ptr(), s.data_ptr(), lam.data_ptr(), out.data_ptr(), s.numel(), M, _st())
    ref = dcoef.double() * lam.double() * 2 * s.double() * (1 - s.double())
    _close_elem(out, ref, 1e-6, 1e-30, f"dyrelu_coef_bwd_m M={M}")


@pytest.mark.gpu
@pytest.mark.parametrize("M", [3, 4])
def test_tie_goes_to_lowest_piece(M):
    """pieces 1 and 2 identical (same slope and offset) and above the others at every pixel: the whole gradient goes to
    piece 1, none to piece 2"""
    B, Fo, To, C = 2, 3, 5, 8
    L, st = lib(), _st()
    lam, init = _buffers(M)
    # coefficients (a_m, b_m) = (1, 0), (0.5, 0.25), (0.5, 0.25), (1, -0.5): for u < -0.5 pieces 1 and 2 tie at the max
    want = torch.tensor([1.0, 0.5, 0.5, 1.0][:M] + [0.0, 0.25, 0.25, -0.5][:M], device="cuda")
    theta = (((want - init) / lam + 1) / 2).expand(B, C, 2 * M).contiguous()     # 0, 0.5, 0.75, 1: exact in fp32
    co = _coef(theta, lam, init)
    assert torch.equal(co[..., 1], co[..., 2]) and torch.equal(co[..., M + 1], co[..., M + 2])
    z = -torch.rand(B, Fo, To, C, device="cuda", generator=_gen(5)) - 0.5      # u = z < -0.5: piece 0 loses to 1 / 2
    one, zero = torch.ones(C, device="cuda"), torch.zeros(C, device="cuda")
    ca_f, ca_t = torch.ones(B, Fo, C, device="cuda"), torch.ones(B, To, C, device="cuda")
    lines = _pieces(z.double(), co, M)
    assert bool((lines[..., 1] == lines.max(-1)[0]).all()) and bool((lines[..., 2] == lines[..., 1]).all())
    dp = torch.ones_like(z)
    P = [t.data_ptr() for t in (one, zero, theta, lam, init, ca_f, ca_t)]
    dcaf, dcoef = torch.zeros(B, Fo, C, device="cuda"), torch.zeros(B, C, 2 * M, device="cuda")
    dcat, du = torch.empty(B, To, C, device="cuda"), torch.empty_like(z)
    L.dy_act_bwd_m(dp.data_ptr(), z.data_ptr(), du.data_ptr(), F32, *P, dcaf.data_ptr(), dcat.data_ptr(), dcoef.data_ptr(),
                   M, B, Fo, To, C, st)
    n = Fo * To
    assert torch.allclose(dcoef[..., M + 1], torch.full_like(dcoef[..., 0], float(n)))
    assert bool((dcoef[..., 2] == 0).all()) and bool((dcoef[..., M + 2] == 0).all())
    assert torch.allclose(dcoef[..., 1], z.sum((1, 2)), rtol=1e-6)
    assert torch.allclose(du, torch.full_like(du, 0.5))


# ------------------------------------------------------------------------------------------------ depthwise + epilogue
DW_CASES = [(3, 1, 1, (1, 1, 16)), (3, 2, 5, (13, 37, 24)), (5, 1, 37, (9, 7, 16)), (5, 2, 5, (7, 1, 40)),
            (3, 1, 37, (5, 11, 8)), (5, 1, 1, (17, 33, 72))]        # (k, stride, B, (F, T, C)); F, T odd, including 1


def _conv_ps(x, w, k, s):
    """x [B, F, T, C], w [B, k*k, C] -> per-sample depthwise conv, NHWC out"""
    B, F, T, C = x.shape
    wc = w.permute(0, 2, 1).reshape(B * C, 1, k, k)
    y = Fn.conv2d(x.permute(0, 3, 1, 2).reshape(1, B * C, F, T), wc, None, s, (k - 1) // 2, 1, B * C)
    return y.view(B, C, y.shape[2], y.shape[3]).permute(0, 2, 3, 1)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [F32, BF16], ids=["f32", "bf16"])
@pytest.mark.parametrize("M", PIECES)
@pytest.mark.parametrize("case", DW_CASES, ids=lambda c: "k{}_s{}_B{}_F{}_T{}_C{}".format(*c[:3], *c[3]))
def test_dw_conv_fwd_dy_m_matches_fp64(case, M, dtype):
    k, s, B, (F, T, C) = case
    if dtype == BF16 and C % 8:
        C += 4
    L, st = lib(), _st()
    g = _gen(k * 1000 + s * 100 + B + M)
    Fo, To = (F - 1) // s + 1, (T - 1) // s + 1
    kk = k * k
    x = torch.randn(B, F, T, C, device="cuda", generator=g).to(DT[dtype])
    w = torch.randn(B, kk, C, device="cuda", generator=g) / k
    bstride = kk * C + 8                                         # a gap between the tables: the stride is honoured
    buf = torch.full((B * bstride + 256,), float("nan"), device="cuda")
    for b in range(B):
        buf[b * bstride: b * bstride + kk * C] = w[b].flatten()
    scale = torch.rand(C, device="cuda", generator=g) + 0.5
    shift = torch.randn(C, device="cuda", generator=g) * 0.3
    theta, (lam, init) = torch.rand(B, C, 2 * M, device="cuda", generator=g), _buffers(M)
    ca_f = torch.rand(B, Fo, C, device="cuda", generator=g)
    ca_t = torch.rand(B, To, C, device="cuda", generator=g)
    co = _coef(theta, lam, init)
    conv = _conv_ps(x.double(), w.double(), k, s)
    cmag = _conv_ps(x.double().abs(), w.double().abs(), k, s)
    out = torch.full((B, Fo, To, C), float("nan"), device="cuda").to(DT[dtype])
    L.dw_conv_fwd_dy_m(x.data_ptr(), buf.data_ptr(), bstride, out.data_ptr(), dtype, B, F, T, C, k, s, 0, 0, 0,
                       scale.data_ptr(), shift.data_ptr(), theta.data_ptr(), lam.data_ptr(), init.data_ptr(),
                       ca_f.data_ptr(), ca_t.data_ptr(), M, 0, 0, st)
    u = conv * scale.double() + shift.double()
    q = ca_f.double()[:, :, None, :] * ca_t.double()[:, None, :, :]
    ref = _dyrelu(u, co, M) * q
    umag = cmag * scale.double() + shift.double().abs()
    mag = (umag.unsqueeze(-1) * co[:, None, None, :, :M].abs() + co[:, None, None, :, M:].abs()).amax(-1) * q
    rel = 1e-6 if dtype == F32 else BF16_REL
    w_e = _close_elem(out, ref, rel, 1e-5 * mag + 1e-30, f"dw_conv_fwd_dy_m eval M={M}")
    # training form: input BatchNorm + Hardswish on load, raw output and fp64 statistics (does not depend on M)
    isc = torch.rand(C, device="cuda", generator=g) + 0.5
    ish = torch.randn(C, device="cuda", generator=g) * 0.3
    out.fill_(float("nan"))
    stats = torch.zeros(2, C, device="cuda", dtype=torch.float64)
    L.dw_conv_fwd_dy_m(x.data_ptr(), buf.data_ptr(), bstride, out.data_ptr(), dtype, B, F, T, C, k, s, isc.data_ptr(),
                       ish.data_ptr(), 2, 0, 0, 0, 0, 0, 0, 0, M, stats[0].data_ptr(), stats[1].data_ptr(), st)
    xf = Fn.hardswish(x.double() * isc.double() + ish.double())
    raw = _conv_ps(xf, w.double(), k, s)
    rmag = _conv_ps(xf.abs(), w.double().abs(), k, s)
    w_t = _close_elem(out, raw, rel, 1e-5 * rmag + 1e-30, "dw_conv_fwd_dy_m training")
    w_s = _close_sum(stats[0], raw.sum((0, 1, 2)), rmag.sum((0, 1, 2)), 1e-5, "stat_sum")
    report(f"[kernel] dw_conv_fwd_dy_m M={M} {case} {'bf16' if dtype else 'f32'}: worst error/bound eval {w_e:.2f} "
           f"training {w_t:.2f} sums {w_s:.2f}")


# ------------------------------------------------------------------------------------------------ eval parity
@pytest.mark.gpu
@pytest.mark.parametrize("gemm", ["simt", "auto"])
@pytest.mark.parametrize("M", PIECES)
def test_eval_matches_reference_vectors(M, gemm):
    g = golden(du.tag(M))
    model = du.build_model(M).cuda().eval()
    model.engine().gemm_impl = gemm
    spec, _ = du.net_inputs()
    with torch.no_grad():
        logits, feat = model(spec.cuda())
        _, _, fmaps = model.engine().forward(spec.cuda(), return_fmaps=True)
    logits, feat = logits.cpu().numpy(), feat.cpu().numpy()
    lerr = np.abs(logits - g["eval_logits"]).max()
    report(f"[parity] dymn04 dyrelu_k={M} eval gemm={gemm}: logits max error {lerr:.2e}")
    assert lerr <= 1e-3
    assert np.abs(feat - g["eval_feat"]).max() <= 1e-3
    assert topk_match(logits, g["eval_logits"], 10, tie_tol=1e-5)
    d = fmap_digest([f.float().cpu() for f in fmaps])
    assert np.abs(d - g["eval_fmaps"]).max() < 1e-3 * max(1.0, np.abs(g["eval_fmaps"]).max())


# ------------------------------------------------------------------------------------------------ training step, B = 5
B_STEP, FRAMES = 5, 201
# the bounds of tests/test_gpu_zz_dymn_kernels.py for dymn04: (relative L2, relative error of the norm) for the
# attention-logit layers (`*.residuals.0.*`) and for all other tensors (coef_net included), and the logits' max-abs error
BOUNDS = {"simt": dict(res=(2e-2, 1e-2), other=(1e-2, 2e-3), logits=5e-5),
          "auto": dict(res=(0.25, 0.2), other=(0.15, 3e-2), logits=5e-4)}
# With four pieces this state and batch are ill-conditioned in fp32: the same network in plain fp32 torch differs from
# fp64 by up to 3.1e-2 relative L2 and 1.2e-2 in a gradient norm (32 tensors beyond 2e-3), because fp32 rounding moves
# pixels to another piece where two lie close (for M = 3: 3.3e-3 and 1.5e-3).  The engine measured 3.5e-2 / 8.4e-3 (simt)
# and 8.2e-2 / 3.3e-2 (auto) on an H100; M = 4 gets bounds of about twice that
BOUNDS_M4 = {"simt": dict(res=(7e-2, 4e-2), other=(7e-2, 2.5e-2), logits=5e-5),
             "auto": dict(res=(0.3, 0.25), other=(0.2, 6e-2), logits=5e-4)}
_ORACLE = {}


def _step_inputs():
    return du.net_inputs(B_STEP, 1 + (FRAMES - 1) * 320)


def _oracle_step(M, pieces_used=None):
    key = (M, pieces_used)
    if key in _ORACLE:
        return _ORACLE[key]
    model = du.build_model(M)
    params = [k for k, _ in model.named_parameters()]
    sd = {k: (v.double() if v.is_floating_point() else v).clone() for k, v in model.state_dict().items()}
    for k in params:
        sd[k].requires_grad_(True)
    spec, y = _step_inputs()
    logits, _ = du.dymn_forward(sd, spec.double(), M, training=True,
                                temperature=float(model.layers[0].depth_conv.temperature), pieces_used=pieces_used)
    loss = Fn.binary_cross_entropy_with_logits(logits, y.double())
    loss.backward()
    _ORACLE[key] = dict(loss=loss.item(), logits=logits.detach(), grads={k: sd[k].grad.detach() for k in params})
    return _ORACLE[key]


def _engine_step(M, gemm):
    model = du.build_model(M).cuda().train()
    eng = model.engine()
    eng.gemm_impl = gemm
    model.classifier[4].p = 0.0
    eng.dropout_p = 0.0
    spec, y = _step_inputs()
    logits, _ = model(spec.cuda())
    loss = Fn.binary_cross_entropy_with_logits(logits, y.cuda())
    loss.backward()
    return model, loss.item(), logits.detach().double().cpu()


def _check_step(what, bd, model, loss, logits, ref):
    total = torch.sqrt(sum((g * g).sum() for g in ref["grads"].values())).item()
    lerr = (logits - ref["logits"]).abs().max().item()
    bad, worst, coef = [], 0.0, 0.0
    for n, p in model.named_parameters():
        g, r = p.grad.detach().double().cpu(), ref["grads"][n]
        e = (g - r).norm().item()
        if r.norm().item() <= 1e-9 * total:                  # analytically zero: against the whole gradient's norm
            if e > 1e-7 * total:
                bad.append(f"{n}: {e / total:.2e} of the gradient norm")
            continue
        rel, nrm = e / r.norm().item(), abs(g.norm().item() - r.norm().item()) / r.norm().item()
        brel, bnorm = bd["res" if ".residuals." in n else "other"]
        if ".residuals." not in n:
            worst = max(worst, rel)
        if ".coef_net." in n:
            coef = max(coef, rel)
        if rel > brel or nrm > bnorm:
            bad.append(f"{n}: relative L2 {rel:.2e} (bound {brel:.0e}), norm {nrm:.2e} (bound {bnorm:.0e})")
    report(f"[parity] {what}: loss {abs(loss - ref['loss']):.2e}, logits {lerr:.2e}, grad rel-L2 max {worst:.2e}, "
           f"coef_net {coef:.2e}")
    assert abs(loss - ref["loss"]) < 1e-5 * max(1.0, abs(ref["loss"])), (loss, ref["loss"])
    assert lerr < bd["logits"], lerr
    assert not bad, "\n".join(bad)


@pytest.mark.gpu
@pytest.mark.parametrize("gemm", ["simt", "auto"])
@pytest.mark.parametrize("M", PIECES)
def test_train_step_matches_fp64_oracle(M, gemm):
    """dymn04 with M pieces, B = 5, 201 frames, dropout off: loss, logits and every gradient tensor (the coef_net layers
    included) against autograd through the fp64 oracle, with the dymn04 bounds of tests/test_gpu_zz_dymn_kernels.py"""
    model, loss, logits = _engine_step(M, gemm)
    _check_step(f"dymn04 dyrelu_k={M} B={B_STEP} train gemm={gemm}", (BOUNDS_M4 if M == 4 else BOUNDS)[gemm], model, loss,
                logits, _oracle_step(M))


@pytest.mark.gpu
@pytest.mark.parametrize("M", [3, 4])
def test_planted_defect_is_caught(M):
    """an oracle that keeps only M - 1 of the M pieces lands outside the bounds"""
    model, loss, logits = _engine_step(M, "simt")
    with pytest.raises(AssertionError):
        _check_step(f"dymn04 dyrelu_k={M} planted defect (M - 1 pieces)", (BOUNDS_M4 if M == 4 else BOUNDS)["simt"], model,
                    loss, logits,
                    _oracle_step(M, pieces_used=M - 1))


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("M", PIECES)
def test_precisions_agree(M, precision):
    """eval and one training step in both storage precisions: finite everywhere, logits within the precision's band of
    the fp64 oracle, and in fp32 a coef_net gradient as well"""
    spec, y = _step_inputs()
    model = du.build_model(M, precision=precision).cuda().eval()
    with torch.no_grad():
        ev, _ = model(spec.cuda())
    ref = _oracle_step(M)
    model.train()
    model.classifier[4].p = 0.0
    model.engine().dropout_p = 0.0
    logits, _ = model(spec.cuda())
    loss = Fn.binary_cross_entropy_with_logits(logits, y.cuda())
    loss.backward()
    assert bool(torch.isfinite(ev).all()) and np.isfinite(loss.item())
    tol = 5e-4 if precision == "fp32" else 0.15            # bf16 storage: measured 8.0e-2 (M = 4) on an H100
    assert (logits.detach().double().cpu() - ref["logits"]).abs().max().item() < tol
    assert all(bool(torch.isfinite(p.grad).all()) for p in model.parameters())
    if precision == "fp32":
        # bf16 storage rounds every activation to 2^-8, and with pieces close to each other that moves many pixels to
        # another piece (a coef_net gradient measured 0.68 relative L2 off fp64 for M = 3 and 4): bf16 is held to its
        # logits band above
        g = model.layers[3].depth_act.coef_net[0].weight.grad.double().cpu()
        r = ref["grads"]["layers.3.depth_act.coef_net.0.weight"]
        assert ((g - r).norm() / r.norm()).item() < 0.15


# ------------------------------------------------------------------------------------------------ trainers
def _trainer(cls, M, graph, **kw):
    from efficientat_b200.models.preprocess import AugmentMelSTFT
    model = du.build_model(M).cuda()
    with contextlib.redirect_stdout(io.StringIO()):
        mel = AugmentMelSTFT(freqm=0, timem=0).cuda()
    model.classifier[4].p = 0.0
    return model, cls(model, mel, cuda_graph=graph, **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("M", PIECES)
def test_audioset_trainer_graph_equals_eager(M):
    from efficientat_b200.synth import synth_labels, synth_waveform
    from efficientat_b200.train import AudioSetTrainer
    B = 5
    wave = synth_waveform(B, 64000, seed=31).cuda()
    y = synth_labels(B, 527, seed=32).cuda()
    teacher = synth_labels(B, 527, seed=33).cuda()
    perm, lam = torch.tensor([1, 2, 3, 4, 0]), torch.full((B,), 0.7)
    losses, deltas = [], []
    for graph in (False, True):
        model, tr = _trainer(AudioSetTrainer, M, graph, lr=4e-4, kd_lambda=0.1, mixup_alpha=0.3)
        start = tr.flat_p.detach().clone()
        losses.append([tr.step(wave, y, teacher, perm=perm, lam=lam).sum().item() for _ in range(2)])  # 2nd: a replay
        deltas.append(tr.flat_p.detach() - start)
    # as tests/test_gpu_zz_dilated.py: the first loss agrees up to summation order, the total update in relative L2
    # (Adam's sign-like first steps flip noise-level elements; twice dymn04's band of tests/test_gpu_finetune_trainer.py,
    # as pieces close to each other make more of them flip)
    assert all(np.isfinite(v) for run in losses for v in run)
    assert abs(losses[0][0] - losses[1][0]) <= 1e-6 * abs(losses[0][0])
    assert abs(losses[0][1] - losses[1][1]) <= 1e-4 * abs(losses[0][1])
    assert ((deltas[0] - deltas[1]).norm() / deltas[0].norm()).item() <= 0.2     # measured up to 0.11 (M = 3)


@pytest.mark.gpu
@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("M", PIECES)
def test_finetune_trainer_ce_step(M, graph):
    from efficientat_b200.finetune import FineTuneTrainer
    from efficientat_b200.synth import synth_waveform
    B = 5
    wave = synth_waveform(B, 64000, seed=41).cuda()
    y = torch.tensor([3, 1, 526, 0, 3], device="cuda")
    model, tr = _trainer(FineTuneTrainer, M, graph, loss="ce", lr=4e-4, mixup_alpha=0.0)
    before = tr.flat_p.detach().clone()
    losses = [tr.step(wave, y).item() for _ in range(2)]
    assert all(np.isfinite(losses)) and losses[1] < losses[0]
    assert (tr.flat_p - before).abs().max().item() > 0
