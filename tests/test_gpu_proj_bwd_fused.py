"""eat_pw_proj_bwd_fused: the project stage's backward in one pass (BN3-backward apply on load, data and weight gradient of
the 1x1 conv from the same tile, the depthwise BatchNorm's backward sums in the epilogue) against a float64 reference
built from the expressions and against the passes it replaces (eat_bn_bwd_apply, eat_pw_tc_wgrad with the BN2 affine
and activation applied on load, eat_pw_tma_fwd with w_trans = 1, eat_bn_bwd_reduce on (dp, z2)); the engine with and
without it; the stem weight gradient with the stem BatchNorm's backward apply on load against the apply pass plus the
plain weight gradient; and the host-side planner and argument checks (no GPU needed).
Tolerances: dp and dW as tests/test_gpu_pw_bwd_fused.py (against fp64 2e-4 of the tensor's max; against the passes dp
2e-5, dW 1e-4); the sums s1 / s2 1e-4 of the sum of the magnitudes of their terms."""
import contextlib
import ctypes
import io

import pytest
import torch
import torch.nn.functional as Fn

from efficientat_b200._lib import EatError, lib

RELU, HS = 1, 2
CASES = [  # (M, cexp, cout, act)
    (4032, 16, 16, RELU),                  # mn10 block 1 channels (one half-empty k-block); M not a multiple of 128
    (3000, 64, 24, RELU),                  # block 2
    (5001, 72, 24, RELU),                  # block 3: partial 32-channel box
    (2000, 128, 32, HS),                   # four full k-blocks, a full dz3 box
    (1000, 120, 16, HS),                   # four k-blocks, the last one partial
    (77, 72, 24, HS),                      # one partial tile
    (132 * 5 * 128 + 77, 72, 24, HS),      # several tiles per CTA (both rings come round), last tile partial
]


def _st():
    return torch.cuda.current_stream().cuda_stream


def _act(v, a):
    if a == RELU:
        return v.clamp_min(0)
    return v * (v + 3).clamp(0, 6) / 6


def _dact(v, a):
    if a == RELU:
        return (v > 0).to(v.dtype)
    return torch.where(v < -3, torch.zeros_like(v), torch.where(v <= 3, (2 * v + 3) / 6, torch.ones_like(v)))


def _inputs(M, cexp, cout, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    r = lambda *sh: torch.randn(*sh, device="cuda", generator=g)
    u = lambda *sh: torch.rand(*sh, device="cuda", generator=g)
    return dict(dy=r(M, cout), z3=r(M, cout), z2=r(M, cexp), w=r(cout, cexp) / cout ** 0.5,
                scale3=u(cout) + 0.5, shift3=r(cout) * 0.3, mean3=r(cout) * 0.2, invstd3=u(cout) + 0.5,
                c1=r(cout) * 0.1, c2=r(cout) * 0.1,
                scale2=u(cexp) + 0.5, shift2=r(cexp) * 0.3, mean2=r(cexp) * 0.2, invstd2=u(cexp) + 0.5)


def _reference(d, act):
    """-> dp, dW, s1, s2 and the magnitudes sum |terms| of s1 and s2, in fp64"""
    D = {n: v.double() for n, v in d.items()}
    dz = D["scale3"] * (D["dy"] - D["c1"] - (D["z3"] - D["mean3"]) * D["invstd3"] * D["c2"])
    u = D["z2"] * D["scale2"] + D["shift2"]
    dp = dz @ D["w"]
    dw = dz.t() @ _act(u, act)
    g = dp * _dact(u, act)
    t2 = g * (D["z2"] - D["mean2"]) * D["invstd2"]
    return dp, dw, g.sum(0), t2.sum(0), g.abs().sum(0), t2.abs().sum(0)


def _fused(d, M, cexp, cout, act):
    dp = torch.full((M, cexp), float("nan"), device="cuda")
    dw = torch.zeros(cout, cexp, device="cuda")
    s = torch.zeros(2, cexp, device="cuda", dtype=torch.float64)
    lib().pw_proj_bwd_fused(d["dy"].data_ptr(), d["z3"].data_ptr(), d["scale3"].data_ptr(), d["shift3"].data_ptr(),
                            d["mean3"].data_ptr(), d["invstd3"].data_ptr(), d["c1"].data_ptr(), d["c2"].data_ptr(),
                            d["z2"].data_ptr(), d["scale2"].data_ptr(), d["shift2"].data_ptr(), d["mean2"].data_ptr(),
                            d["invstd2"].data_ptr(), act, d["w"].data_ptr(), dp.data_ptr(), dw.data_ptr(), s[0].data_ptr(),
                            s[1].data_ptr(), 0, M, cexp, cout, _st())
    return dp, dw, s[0], s[1]


def _chain(d, M, cexp, cout, act):
    """the passes the fused kernel replaces: BN3 apply, weight-gradient GEMM (BN2 + activation on load), data-gradient
    GEMM, BN2-backward reduce"""
    L, st = lib(), _st()
    dz = torch.empty_like(d["z3"])
    L.bn_bwd_apply(d["dy"].data_ptr(), 0, 0, d["z3"].data_ptr(), d["scale3"].data_ptr(), d["shift3"].data_ptr(),
                   d["mean3"].data_ptr(), d["invstd3"].data_ptr(), 0, d["c1"].data_ptr(), d["c2"].data_ptr(), dz.data_ptr(),
                   0, 1, M, cout, st)
    dw = torch.zeros(cout, cexp, device="cuda")
    L.pw_tc_wgrad(dz.data_ptr(), 0, d["z2"].data_ptr(), 0, dw.data_ptr(), 0, M, cout, cexp, d["scale2"].data_ptr(),
                  d["shift2"].data_ptr(), act, 0, 1, st)
    dp = torch.empty(M, cexp, device="cuda")
    ws = torch.empty(cexp * ((cout + 31) // 32) * 128, device="cuda", dtype=torch.uint8)
    L.pw_tma_fwd(dz.data_ptr(), d["w"].data_ptr(), 1, dp.data_ptr(), M, cexp, cout, 0, 0, 0, 0, 1, 0, 0, 0, 0, 0, 0,
                 ws.data_ptr(), ws.numel(), st)
    s = torch.zeros(2, cexp, device="cuda", dtype=torch.float64)
    L.bn_bwd_reduce(dp.data_ptr(), 0, 0, d["z2"].data_ptr(), d["scale2"].data_ptr(), d["shift2"].data_ptr(),
                    d["mean2"].data_ptr(), d["invstd2"].data_ptr(), act, 0, 1, M, cexp, s[0].data_ptr(), s[1].data_ptr(), st)
    return dp, dw, s[0], s[1]


def _close(got, ref, tol, what):
    err = (got.double() - ref.double()).abs().max().item()
    scale = ref.double().abs().max().item()
    assert err <= tol * scale + 1e-12, f"{what}: max error {err:.3e} vs scale {scale:.3e}"


def _close_sum(got, ref, mag, tol, what):
    err = (got.double() - ref.double()).abs()
    bound = tol * mag.double() + 1e-9
    assert bool((err <= bound).all()), f"{what}: worst error / bound {(err / bound).max().item():.3f}"


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=lambda c: "M{}_cexp{}_cout{}_{}".format(*c[:3], "hs" if c[3] == HS else "relu"))
def test_fused_matches_fp64_and_the_separate_passes(case):
    M, cexp, cout, act = case
    d = _inputs(M, cexp, cout, seed=M + cexp + cout)
    dp, dw, s1, s2 = _fused(d, M, cexp, cout, act)
    rdp, rdw, rs1, rs2, m1, m2 = _reference(d, act)
    _close(dp, rdp, 2e-4, "dp vs fp64")
    _close(dw, rdw, 2e-4, "dW vs fp64")
    _close_sum(s1, rs1, m1, 1e-4, "s1 vs fp64")
    _close_sum(s2, rs2, m2, 1e-4, "s2 vs fp64")
    cdp, cdw, cs1, cs2 = _chain(d, M, cexp, cout, act)
    _close(dp, cdp, 2e-5, "dp vs passes")
    _close(dw, cdw, 1e-4, "dW vs passes")
    _close_sum(s1, cs1, m1, 1e-4, "s1 vs passes")
    _close_sum(s2, cs2, m2, 1e-4, "s2 vs passes")


@pytest.mark.gpu
def test_engine_step_with_and_without_the_fused_project_backward():
    """one mn10 training step (16 clips of 1000 frames) with the fused and with the separate project-stage backward (and the
    stem BatchNorm's backward apply on load in the stem weight gradient, or as its own pass),
    bounded as test_gpu_pw_bwd_fused.py's engine test: the whole gradient's relative L2 distance between the routes must
    stay within 3x the old route's run-to-run distance (floor 2e-4) and below 5e-3, and the direction must agree to 1e-5."""
    from efficientat_b200.models.mn.model import get_model
    from efficientat_b200.synth import synth_labels, synth_state_, synth_waveform

    B, T = 16, 1000
    spec = synth_waveform(B, 128 * T, seed=21, std=0.7).view(B, 1, 128, T).cuda()
    y = synth_labels(B, 527, seed=5).cuda()

    def grads(fused):
        torch.manual_seed(0)
        with contextlib.redirect_stdout(io.StringIO()):
            model = synth_state_(get_model(width_mult=1.0, verbose=False), seed=7).cuda().train()
        model.classifier[4].p = 0.0
        eng = model.engine()
        eng.dropout_p = 0.0
        eng.proj_bwd_fused = fused
        eng.stem_bwd_fused = fused
        logits, _ = model(spec)
        Fn.binary_cross_entropy_with_logits(logits, y).backward()
        return torch.cat([p.grad.detach().double().flatten() for p in model.parameters()])

    old, old2, new = grads(False), grads(False), grads(True)
    spread = ((old2 - old).norm() / old.norm()).item()
    cross = ((new - old).norm() / old.norm()).item()
    assert cross <= min(3 * max(spread, 2e-4), 5e-3), f"fused vs passes {cross:.2e}, passes run to run {spread:.2e}"
    assert torch.nn.functional.cosine_similarity(old, new, dim=0) > 1 - 1e-5


def _mn10_project_stages(B=256, F=64, T=501):
    """(block, M, cexp, cout, has SE) of every mn10 block, 128 mel bins x 1001 frames (stem output 64 x 501)"""
    from efficientat_b200.models.mn.model import get_model
    with contextlib.redirect_stdout(io.StringIO()):
        model = get_model(width_mult=1.0, verbose=False)
    out = []
    for i, m in enumerate(list(model.features)[1:-1]):
        c = m.cnf
        pad = (c.kernel - 1) // 2
        F, T = (F + 2 * pad - c.kernel) // c.stride + 1, (T + 2 * pad - c.kernel) // c.stride + 1
        out.append((i + 1, B * F * T, c.expanded_channels, c.out_channels, bool(c.use_se)))
    return out


def test_planner_takes_blocks_1_to_3_and_fits_shared_memory():
    L = lib()
    plan = (ctypes.c_int * 4)()
    stages = _mn10_project_stages()
    assert [s[0] for s in stages] == list(range(1, 16))
    assert [s[0] for s in stages if s[4]] == [4, 5, 6, 11, 12, 13, 14, 15]
    for blk, M, cexp, cout, _ in stages:
        if blk <= 3:
            L.pw_proj_bwd_plan(M, cexp, cout, ctypes.addressof(plan))
            splits, rows, nstages, smem = list(plan)
            assert 1 <= splits <= 132 and rows % 128 == 0 and splits * rows >= M
            assert 3 <= nstages and smem <= 227 * 1024, (blk, list(plan))
        else:   # block 4 and every SE block: wider than one 32-channel dz3 box (and the engine never asks for SE blocks)
            with pytest.raises(EatError, match=r"code 3\): .*cout <= 32 and cexp <= 128"):
                L.pw_proj_bwd_plan(M, cexp, cout, ctypes.addressof(plan))
    L.pw_proj_bwd_plan(300, 72, 24, ctypes.addressof(plan))
    assert list(plan)[:2] == [3, 128]
    for M, cexp, cout, _ in CASES:
        L.pw_proj_bwd_plan(M, cexp, cout, ctypes.addressof(plan))


def test_cabi_rejects_unsupported_arguments_before_any_launch():
    L = lib()
    fake = 4096                                                   # never dereferenced: validation comes first

    def call(dtype=0, act=RELU, cexp=72, cout=24, M=1000, dy=fake, dp=fake, s1=fake):
        L.pw_proj_bwd_fused(dy, fake, fake, fake, fake, fake, fake, fake, fake, fake, fake, fake, fake, act, fake, dp, fake,
                            s1, fake, dtype, M, cexp, cout, 0)

    with pytest.raises(EatError, match=r"code 3\): .*fp32 storage only"):
        call(dtype=1)
    with pytest.raises(EatError, match=r"code 3\): .*relu or hardswish"):
        call(act=0)
    with pytest.raises(EatError, match=r"code 3\): .*cout <= 32 and cexp <= 128"):
        call(cout=40)
    with pytest.raises(EatError, match=r"code 3\): .*cout <= 32 and cexp <= 128"):
        call(cexp=240)
    with pytest.raises(EatError, match=r"code 1\): .*multiples of 4"):
        call(cexp=70)
    with pytest.raises(EatError, match=r"code 1\): .*are required"):
        call(dy=0)
    with pytest.raises(EatError, match=r"code 1\): .*16-byte aligned"):
        call(dp=fake + 4)
    with pytest.raises(EatError, match=r"code 1\): .*8-byte aligned"):
        call(s1=fake + 4)
    with pytest.raises(EatError, match=r"code 1\): .*negative M"):
        call(M=-1)
    call(M=0)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(4, 128, 1001, 16, 2), (3, 37, 50, 16, 2), (2, 20, 33, 8, 1)],
                         ids=lambda s: "B{}_F{}_T{}_C{}_s{}".format(*s))
def test_stem_wgrad_apply_on_load_matches_the_apply_pass(shape):
    """eat_stem_wgrad with z (dz0 computed on load, hardswish) against eat_bn_bwd_apply + eat_stem_wgrad on the stored dz0:
    the same fp32 products, so 1e-5 of the largest weight-gradient entry"""
    B, F, T, C, s = shape
    L, st = lib(), _st()
    Fo, To = (F - 1) // s + 1, (T - 1) // s + 1
    g = torch.Generator(device="cuda").manual_seed(B * F + T)
    r = lambda *sh: torch.randn(*sh, device="cuda", generator=g)
    u = lambda *sh: torch.rand(*sh, device="cuda", generator=g)
    x, dy, z = r(B, F, T), r(B, Fo, To, C), r(B, Fo, To, C)
    bn = [u(C) + 0.5, r(C) * 0.3, r(C) * 0.2, u(C) + 0.5]
    c12 = [r(C) * 0.1, r(C) * 0.1]
    P = [t.data_ptr() for t in bn]
    dz = torch.empty_like(z)
    L.bn_bwd_apply(dy.data_ptr(), 0, 0, z.data_ptr(), *P, HS, c12[0].data_ptr(), c12[1].data_ptr(), dz.data_ptr(), 0, 1,
                   B * Fo * To, C, st)
    ref, got = torch.zeros(C, 1, 3, 3, device="cuda"), torch.zeros(C, 1, 3, 3, device="cuda")
    L.stem_wgrad(dz.data_ptr(), 0, x.data_ptr(), ref.data_ptr(), B, F, T, C, s, 0, 0, 0, 0, 0, 0, 0, 0, st)
    L.stem_wgrad(dy.data_ptr(), 0, x.data_ptr(), got.data_ptr(), B, F, T, C, s, z.data_ptr(), *P, HS, c12[0].data_ptr(),
                 c12[1].data_ptr(), st)
    _close(got, ref, 1e-5, "stem dW apply on load vs apply pass")


def test_stem_wgrad_apply_on_load_rejects_what_it_does_not_take():
    L = lib()
    fake = 4096                                                   # never dereferenced: validation comes first
    with pytest.raises(EatError, match=r"code 3\): .*apply on load needs fp32"):
        L.stem_wgrad(fake, 1, fake, fake, 2, 128, 1001, 16, 2, fake, fake, fake, fake, fake, HS, fake, fake, 0)
    with pytest.raises(EatError, match=r"code 3\): .*apply on load needs fp32"):
        L.stem_wgrad(fake, 0, fake, fake, 2, 128, 1001, 16, 3, fake, fake, fake, fake, fake, HS, fake, fake, 0)
    with pytest.raises(EatError, match=r"code 1\): .*needs scale, shift"):
        L.stem_wgrad(fake, 0, fake, fake, 2, 128, 1001, 16, 2, fake, fake, 0, fake, fake, HS, fake, fake, 0)
