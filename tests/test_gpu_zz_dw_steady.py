"""The depthwise kernels in the launch regime the benchmark runs them in: several work units per thread slot, segments of
several rows (so a segment boundary falls inside a sample and the register window restarts there), walks that cross from
one sample to the next, every prefetch-ring depth, partial last channel chunks, and the tile kernel with several tiles per
CTA.  At B = 2 every thread walks at most one unit of one or two rows, so the batch-2 files (test_gpu_dw.py) never reach
this state; the cases here are chosen with the launch planner itself (eat_dw_plan), and the CPU test below asserts what
each one reaches.

Every kernel result is compared with float64 torch (F.conv2d with groups = C and its autograd):
  - per-output results (forward output, din): at most 25 taps summed in an order the walk does not change, so the
    batch-2 bounds stay: fp32 1e-5 of the output scale (din 2e-5), bf16 2e-2.  More is a walk defect, not rounding;
  - long sums (the batch statistics, the SE pool sums, dW): |error| <= SUM_ULPS * 2^-24 * sum |terms| per channel (per
    sample and channel for pool and per-sample dW), where the terms are the conv of |input| with |w| (their squares for
    the sum of squares) or |dz| * |xf(in)|;
  - the variance eat_bn_finalize derives from the kernel's sums, on an input with mean >> std (4 + 0.25 randn), is no
    further from fp64 than 2x what torch.var_mean in fp32 (the reference's own BatchNorm precision) gets on the same
    fp32 output, both saved as an fp32 invstd (measured on an H100: 1.3-2.2e-7 against torch's 3.9-4.9e-7 at mean/std
    up to 24; with unshifted fp32 per-thread sums the kernel was at 3.8e-6 to 1.1e-5).
Without a GPU, test_bounds_see_walk_defects plants walk defects in an fp64 reference of one steady-state case per kind
(forward, weight gradient, stride-2 data gradient, and a per-sample plan): the rows at each segment start without their
first input row, one unit per thread dropped, and a sample's top halo read from the previous sample (the per-sample
plan never crosses samples, so only the dropped unit applies there).  Each must lie >= 10x outside its bound.

References are built in chunks of <= 32 samples with fp64 sums.  The largest case, B = 256 at mn10 block 2 (64 x 500 x 64
input, 2.1 GB in fp32), asserts its peak device memory below 8 GiB; measured on an H100: 4.15 GiB.
"""
import ctypes

import pytest
import torch
import torch.nn.functional as Fn

from efficientat_b200._lib import lib
from tests.steady_util import dw_plan as _plan, out_hw as _out_hw
from tests.util import bn_variance_check, report

NONE, RELU, HS = 0, 1, 2
F32, BF16 = 0, 1
DT = {F32: torch.float32, BF16: torch.bfloat16}
U = 2.0 ** -24
# long-sum bound, in units of 2^-24 * sum |terms|.  Measured on an H100 80GB HBM3 (700 W): statistics <= 8.8, SE pool
# <= 6.0, dW <= 6.6 (fused backward: dW 3.0, BN1 sums 0.9); a planted dropped unit sits >= 2700x above the bound
SUM_ULPS = 64
TOL = {F32: 1e-5, BF16: 2e-2}     # forward output, of the output scale
TOL_DIN = {F32: 2e-5, BF16: 2e-2}
EPS = 1e-3                        # nn.BatchNorm2d(eps=1e-3), models/mn/model.py:114
CHUNK = 32

# (B, F, T, C, k, stride): F x T is the layer's input.  mn10 at 10 s (1000 frames): block 2 64x500 -> 32x250 (stride 2),
# the 8x63 layers (C = 480 / 672 / 960) and the 4x32 5x5 layers (C = 960) at the bench's B = 256
FWD = [(16, 64, 100, 16, 3, 1),         # chunks of <= 32 channels: the three-row ring
       (32, 64, 500, 64, 3, 2), (32, 32, 250, 72, 5, 2), (32, 16, 126, 516, 3, 1),
       (16, 8, 63, 2688, 5, 2),         # mn40 block 13: 5x5 stride 2 at 112 vectors per chunk, ring off (depth 0)
       (256, 8, 63, 960, 3, 1), (256, 4, 32, 960, 5, 1)]
FWD_STATS_BENCH = (256, 64, 500, 64, 3, 2)      # mn10 block 2 at the bench's batch: the statistics' longest walk
EVAL = [(32, 16, 126, 516, 3, 1), (64, 32, 250, 72, 3, 1), (256, 8, 63, 672, 3, 1)]       # slide kernel, per sample
EVAL_TILE = [(64, 32, 250, 72, 5, 2), (256, 16, 125, 120, 5, 1), (16, 16, 126, 480, 5, 1)]  # 5x5 eval: tile kernel
DGRAD = [(32, 32, 250, 72, 3, 1), (32, 16, 125, 120, 5, 1),                   # stride 1, slide kernel (5x5: C <= 256)
         (16, 16, 126, 480, 5, 1), (256, 4, 32, 960, 5, 1),                   # stride 1, 5x5, C > 256: tile kernel
         (32, 32, 250, 72, 5, 2), (16, 16, 126, 516, 3, 2), (16, 16, 126, 520, 3, 2), (256, 8, 63, 672, 5, 2)]
DGRAD_PS = [(32, 32, 250, 72, 3, 1), (64, 32, 250, 72, 5, 2), (256, 8, 63, 960, 5, 2)]    # per-sample weight tables
WGRAD = [(16, 32, 250, 72, 3, 1), (32, 16, 125, 120, 5, 1), (64, 64, 500, 64, 3, 2), (16, 16, 126, 520, 5, 1),
         (256, 8, 63, 960, 3, 1)]
WGRAD_PS = [(64, 8, 63, 200, 3, 1), (16, 16, 125, 120, 5, 1), (256, 4, 32, 960, 5, 1)]
DIL = [(256, 8, 63, 480, 3), (256, 8, 63, 960, 5)]                            # the dilated tail at B = 256


def _st():
    return torch.cuda.current_stream().cuda_stream


def _p(t):
    return 0 if t is None else t.data_ptr()


def _act(x, code):
    return torch.relu(x) if code == RELU else (Fn.hardswish(x) if code == HS else x)


def _ids(cases):
    return ["B{}_F{}_T{}_C{}_k{}_s{}".format(*c) for c in cases]


def _ring_depth(dtype, C, k, s):
    """the prefetch-ring depth the forward / stride-1 data-gradient kernel takes (eat_dw_ring_depth)"""
    d = ctypes.c_int(-1)
    lib().dw_ring_depth(dtype, C, k, s, ctypes.addressof(d))
    return d.value


# ------------------------------------------------------------------------------------------------ the cases reach it
def _slide_cases():
    """(kind, per_sample, dtype, case) of every slide-kernel launch the GPU tests make"""
    out = []
    for dt in (F32, BF16):
        out += [(0, 0, dt, c) for c in FWD + [FWD_STATS_BENCH] + [c for c in DGRAD if c[5] == 1 and not
                                                                   (c[4] == 5 and c[3] > 256)]]
        out += [(0, 1, dt, c) for c in EVAL]
        out += [(2, 0, dt, c) for c in DGRAD if c[5] == 2] + [(2, 1, dt, c) for c in DGRAD_PS if c[5] == 2]
        out += [(1, 0, dt, c) for c in WGRAD if not (dt == BF16 and c[4] == 5)]
        out += [(1, 1, dt, c) for c in WGRAD_PS if not (dt == BF16 and c[4] == 5)]
    return [(kind, ps, dt, c) for kind, ps, dt, c in out if c[3] % (8 if dt == BF16 else 4) == 0]


def test_cases_reach_the_steady_state():
    got = {}
    for kind, ps, dt, c in _slide_cases():
        pl = _plan(kind, dt, *c, per_sample=ps)
        g = got.setdefault(kind, dict(max_slot={}, seg_inside=0, crosses=0, ps_one_group=0, partial=0, rings=set(),
                                      b256=0))
        g["max_slot"][dt] = max(g["max_slot"].get(dt, 0), pl["per_slot"])
        g["seg_inside"] += 1 < pl["seg"] < pl["rows"] and pl["per_slot"] >= 2
        g["crosses"] += pl["crosses"] and pl["per_slot"] >= 2
        g["ps_one_group"] += bool(ps) and pl["groups"] == 1
        g["partial"] += pl["partial"]
        g["b256"] += c[0] == 256
        if kind == 0:
            g["rings"].add(_ring_depth(dt, c[3], c[4], c[5]))
    for kind, g in sorted(got.items()):
        report(f"[plan] dw kind {kind}: largest units per thread slot "
               + ", ".join(f"{'fp32' if dt == F32 else 'bf16'} {v:.1f}" for dt, v in sorted(g["max_slot"].items()))
               + f"; cases with a segment boundary inside a sample {g['seg_inside']}, crossing samples {g['crosses']}, "
               f"per-sample with one group {g['ps_one_group']}, partial chunk {g['partial']}, rings {sorted(g['rings'])}")
        assert min(g["max_slot"].values()) >= 8, (kind, g)
        assert g["seg_inside"] and g["crosses"] and g["ps_one_group"] and g["partial"] and g["b256"], (kind, g)
    assert got[0]["rings"] == {0, 2, 3}, got[0]["rings"]
    # chunks of <= 32 channels take three rows; 5x5 stride 2 with wide chunks has no room for two: mn40 block 13
    assert _ring_depth(F32, 16, 3, 1) == 3 and _ring_depth(F32, 2688, 5, 2) == 0 and _ring_depth(F32, 960, 3, 1) == 2
    # tile kernel: every CTA strides over several tiles of its chunk
    for B, F, T, C, k, s in EVAL_TILE + [c for c in DGRAD if c[4] == 5 and c[5] == 1 and c[3] > 256]:
        pl = _plan(4, F32, B, F, T, C, k, s)
        report(f"[plan] dw tile {(B, F, T, C, k, s)}: {pl['tiles']} tiles per chunk and sample, {pl['groups']} CTAs")
        if pl["tiles"] > 1:
            assert pl["groups"] < pl["tiles"], (B, F, T, C, k, s, pl)
    assert any(_plan(4, F32, *c)["tiles"] >= 4 * _plan(4, F32, *c)["groups"] for c in EVAL_TILE)


# ------------------------------------------------------------------------------------------------ fp64 references
def _xf(x, sc, act):
    a = x.double()
    return a if sc is None else _act(a * sc[0].double() + sc[1].double(), act)


def _conv(a, w, k, s, groups=None, dil=1):
    """a [B, F, T, C] fp64 -> depthwise conv [B, Fo, To, C]"""
    C = a.shape[3]
    return Fn.conv2d(a.permute(0, 3, 1, 2), w, None, s, (k - 1) // 2 * dil, dil, groups or C).permute(0, 2, 3, 1)


def _setup(B, F, T, C, k, dtype, seed, dc=False):
    if C % (8 if dtype == BF16 else 4):
        pytest.skip("bf16 storage needs C a multiple of 8")
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, F, T, C, device="cuda", generator=g)
    if dc:
        x.mul_(0.25).add_(4.0)
    x = x.to(DT[dtype])
    w = torch.randn(C, 1, k, k, device="cuda", generator=g) * 0.3
    wt = torch.empty(k * k, C, device="cuda")
    lib().dw_repack(w.data_ptr(), wt.data_ptr(), C, k, _st())
    sc = torch.rand(2, C, device="cuda", generator=g) + 0.5
    sc[1] -= 1.0
    return g, x, w, wt, sc


def _check_sum(got, ref, mag, what):
    """long sum: |got - ref| <= SUM_ULPS * 2^-24 * mag per entry; returns the worst |error| / (2^-24 mag)"""
    ulps = ((got.double() - ref).abs() / (U * mag + 1e-300)).max().item()
    assert ulps <= SUM_ULPS, f"{what}: error {ulps:.1f} x 2^-24 sum|terms| (bound {SUM_ULPS})"
    return ulps


def _fwd_run(x, wt, dtype, B, F, T, C, k, s, in_act=-1, sc=None, eval_act=None, dil=1):
    L = lib()
    Fo, To = (F, T) if dil == 2 else _out_hw(F, T, k, s)
    out = torch.full((B, Fo, To, C), float("nan"), device="cuda", dtype=DT[dtype])
    if eval_act is None:
        stats = torch.zeros(2, C, device="cuda", dtype=torch.float64)
        xs = (sc[0].data_ptr(), sc[1].data_ptr(), max(in_act, 0)) if in_act >= 0 else (0, 0, 0)
        tail = (0, 0, 0, 0, stats[0].data_ptr(), stats[1].data_ptr())
    else:
        stats = torch.zeros(B, C, device="cuda")                      # pool
        xs = (0, 0, 0)
        tail = (sc[0].data_ptr(), sc[1].data_ptr(), eval_act, stats.data_ptr(), 0, 0)
    if dil == 2:
        L.dw_conv_fwd_dil(x.data_ptr(), wt.data_ptr(), out.data_ptr(), dtype, B, F, T, C, k, 1, 2, *xs, *tail, _st())
    else:
        L.dw_conv_fwd(x.data_ptr(), wt.data_ptr(), out.data_ptr(), dtype, B, F, T, C, k, s, *xs, *tail, _st())
    return out, stats


def _check_fwd_train(x, w, wt, sc, dtype, case, in_act, dil=1):
    B, F, T, C, k, s = case
    out, stats = _fwd_run(x, wt, dtype, *case, in_act=in_act, sc=sc, dil=dil)
    err = scale = 0.0
    ref = torch.zeros(2, C, device="cuda", dtype=torch.float64)
    mag = torch.zeros_like(ref)
    for b0 in range(0, B, CHUNK):
        a = _xf(x[b0:b0 + CHUNK], sc if in_act >= 0 else None, max(in_act, 0))
        conv, cmag = _conv(a, w.double(), k, s, dil=dil), _conv(a.abs(), w.double().abs(), k, s, dil=dil)
        err = max(err, (out[b0:b0 + CHUNK].double() - conv).abs().max().item())
        scale = max(scale, conv.abs().max().item())
        ref += torch.stack([conv.sum((0, 1, 2)), (conv * conv).sum((0, 1, 2))])
        mag += torch.stack([cmag.sum((0, 1, 2)), (cmag * cmag).sum((0, 1, 2))])
        del a, conv, cmag
    assert err <= TOL[dtype] * scale, f"output: error {err:.3e} vs scale {scale:.3e}"
    u_s = _check_sum(stats[0], ref[0], mag[0], "stat_sum")
    u_q = _check_sum(stats[1], ref[1], mag[1], "stat_sq")
    return out, stats, ref, err / scale, u_s, u_q


@pytest.mark.gpu
@pytest.mark.parametrize("in_act", [-1, NONE, RELU, HS], ids=["no_xf", "xf_none", "xf_relu", "xf_hs"])
@pytest.mark.parametrize("dtype", [F32, BF16], ids=["f32", "bf16"])
@pytest.mark.parametrize("case", FWD, ids=_ids(FWD))
def test_forward_training(case, dtype, in_act):
    _, x, w, wt, sc = _setup(*case[:4], case[4], dtype, seed=sum(case) + in_act)
    _, _, _, e, u_s, u_q = _check_fwd_train(x, w, wt, sc, dtype, case, in_act)
    report(f"[kernel] dw fwd train {case} {dtype} xf{in_act}: output {e:.2e} of scale, stat_sum {u_s:.1f} / "
           f"stat_sq {u_q:.1f} x 2^-24 sum|terms|")


@pytest.mark.gpu
@pytest.mark.parametrize("case", [FWD[1], FWD[5], FWD_STATS_BENCH], ids=_ids([FWD[1], FWD[5], FWD_STATS_BENCH]))
def test_forward_statistics_keep_the_variance(case):
    """input 4 + 0.25 randn through the producing layer's BatchNorm + Hardswish: the conv output's mean is many times
    its std, where E[x^2] - E[x]^2 cancels"""
    B, F, T, C, k, s = case
    torch.cuda.reset_peak_memory_stats()
    _, x, w, wt, sc = _setup(B, F, T, C, k, F32, seed=7 + B, dc=True)
    out, stats, ref, e, u_s, u_q = _check_fwd_train(x, w, wt, sc, F32, case, HS)
    del x
    Fo, To = _out_hw(F, T, k, s)
    report(f"[kernel] dw fwd train dc {case}: output {e:.2e}, stat_sum {u_s:.1f} / stat_sq {u_q:.1f} x 2^-24 sum|terms|")
    bn_variance_check(out, stats, ref, B * Fo * To, C, EPS, f"dw fwd train dc {case}")
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    report(f"[kernel] dw fwd train dc {case}: peak device memory {peak:.2f} GiB")
    assert peak < 8, f"peak device memory {peak:.2f} GiB"


@pytest.mark.gpu
@pytest.mark.parametrize("act", [NONE, RELU, HS], ids=["none", "relu", "hs"])
@pytest.mark.parametrize("dtype", [F32, BF16], ids=["f32", "bf16"])
@pytest.mark.parametrize("case", EVAL + EVAL_TILE, ids=_ids(EVAL + EVAL_TILE))
def test_forward_eval_with_pool(case, dtype, act):
    B, F, T, C, k, s = case
    _, x, w, wt, sc = _setup(B, F, T, C, k, dtype, seed=100 + sum(case) + act)
    out, pool = _fwd_run(x, wt, dtype, *case, sc=sc, eval_act=act)
    err = scale = 0.0
    ulps = 0.0
    for b0 in range(0, B, CHUNK):
        a = x[b0:b0 + CHUNK].double()
        y = _act(_conv(a, w.double(), k, s) * sc[0].double() + sc[1].double(), act)
        err = max(err, (out[b0:b0 + CHUNK].double() - y).abs().max().item())
        scale = max(scale, y.abs().max().item())
        # terms of the pool sum: the activated outputs, each within 1.5 x its conv's rounding of the fp64 value
        mag = (_conv(a.abs(), w.double().abs(), k, s) * sc[0].double() + sc[1].double().abs()).sum((1, 2)) * 1.5
        ulps = max(ulps, _check_sum(pool[b0:b0 + CHUNK], y.sum((1, 2)), mag, "pool"))
        del a, y, mag
    assert err <= TOL[dtype] * scale, f"output: error {err:.3e} vs scale {scale:.3e}"
    report(f"[kernel] dw fwd eval {case} {dtype} act{act}: output {err / scale:.2e} of scale, pool {ulps:.1f} x 2^-24")


def _grads_ref(x, sc, w, dz, k, s, per_sample=False, wps=None, dil=1):
    """fp64 autograd of the depthwise conv of xf(x) (shared w, or per-sample tables wps [B, C, 1, k, k]):
    (d input, dW, sum |dz| * |xf| per weight entry)"""
    Bc, _, _, C = x.shape
    a = _xf(x, sc, HS)
    if wps is not None or per_sample:
        # one sample of Bc * C channels: channel b * C + c is sample b's channel c, with its own weight table
        flat = lambda t: t.permute(1, 2, 0, 3).reshape(1, t.shape[1], t.shape[2], Bc * C)
        wv = (wps.double() if wps is not None else w.double().expand(Bc, *w.shape)).reshape(Bc * C, 1, k, k)
        wv = wv.clone().requires_grad_(True)
        ar = flat(a).requires_grad_(True)
        ga, gw = torch.autograd.grad(_conv(ar, wv, k, s, dil=dil), (ar, wv), flat(dz.double()))
        wa = wv.detach().abs().requires_grad_(True)
        gmag = torch.autograd.grad(_conv(flat(a.abs()), wa, k, s, dil=dil), wa, flat(dz.double().abs()))[0]
        ga = ga.reshape(ga.shape[1], ga.shape[2], Bc, C).permute(2, 0, 1, 3)
        return ga, gw.reshape(Bc, C, 1, k, k), gmag.reshape(Bc, C, 1, k, k)
    ar = a.clone().requires_grad_(True)
    wd = w.double().clone().requires_grad_(True)
    ga, gw = torch.autograd.grad(_conv(ar, wd, k, s, dil=dil), (ar, wd), dz.double())
    wa = w.double().abs().clone().requires_grad_(True)
    gmag = torch.autograd.grad(_conv(a.abs(), wa, k, s, dil=dil), wa, dz.double().abs())[0]
    return ga, gw, gmag


def _check_dgrad(case, dtype, with_res, per_sample, dil=1):
    B, F, T, C, k, s = case
    L = lib()
    g, x, w, wt, sc = _setup(B, F, T, C, k, dtype, seed=200 + sum(case) + with_res + 2 * per_sample)
    Fo, To = (F, T) if dil == 2 else _out_hw(F, T, k, s)
    dz = torch.randn(B, Fo, To, C, device="cuda", generator=g).to(DT[dtype])
    res = torch.randn(B, F, T, C, device="cuda", generator=g).to(DT[dtype]) if with_res else None
    wps = wtps = None
    if per_sample:
        wps = torch.randn(B, C, 1, k, k, device="cuda", generator=g) * 0.3
        wtps = torch.empty(B, k * k, C, device="cuda")
        for b in range(B):
            L.dw_repack(wps[b].data_ptr(), wtps[b].data_ptr(), C, k, _st())
    din = torch.full((B, F, T, C), float("nan"), device="cuda", dtype=DT[dtype])
    if dil == 2:
        L.dw_conv_dgrad_dil(dz.data_ptr(), wt.data_ptr(), _p(res), din.data_ptr(), dtype, B, F, T, C, k, 1, 2, _st())
    else:
        L.dw_conv_dgrad(dz.data_ptr(), (wtps if per_sample else wt).data_ptr(), k * k * C if per_sample else 0, _p(res),
                        din.data_ptr(), dtype, B, F, T, C, k, s, _st())
    err = scale = 0.0
    for b0 in range(0, B, CHUNK):
        sl = slice(b0, b0 + CHUNK)
        # the data gradient of the conv itself: the input transform is the identity here
        ga = _grads_ref(x[sl], None, w, dz[sl], k, s, wps=None if wps is None else wps[sl], dil=dil)[0]
        want = ga + (res[sl].double() if res is not None else 0)
        err = max(err, (din[sl].double() - want).abs().max().item())
        scale = max(scale, want.abs().max().item())
        del ga, want
    assert err <= TOL_DIN[dtype] * scale, f"din: error {err:.3e} vs scale {scale:.3e}"
    return err / scale


@pytest.mark.gpu
@pytest.mark.parametrize("with_res", [False, True], ids=["plain", "res"])
@pytest.mark.parametrize("dtype", [F32, BF16], ids=["f32", "bf16"])
@pytest.mark.parametrize("case", DGRAD, ids=_ids(DGRAD))
def test_dgrad(case, dtype, with_res):
    e = _check_dgrad(case, dtype, with_res, False)
    report(f"[kernel] dw dgrad {case} {dtype} res={with_res}: din {e:.2e} of scale")


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [F32, BF16], ids=["f32", "bf16"])
@pytest.mark.parametrize("case", DGRAD_PS, ids=_ids(DGRAD_PS))
def test_dgrad_per_sample_weights(case, dtype):
    e = _check_dgrad(case, dtype, case[5] == 1, True)
    report(f"[kernel] dw dgrad per-sample {case} {dtype}: din {e:.2e} of scale")


def _check_wgrad(case, dtype, per_sample, dil=1):
    B, F, T, C, k, s = case
    L = lib()
    g, x, w, wt, sc = _setup(B, F, T, C, k, dtype, seed=300 + sum(case) + per_sample)
    Fo, To = (F, T) if dil == 2 else _out_hw(F, T, k, s)
    dz = torch.randn(B, Fo, To, C, device="cuda", generator=g).to(DT[dtype])
    dw = torch.zeros((B if per_sample else 1) * C * k * k, device="cuda")
    if dil == 2:
        L.dw_conv_wgrad_dil(dz.data_ptr(), x.data_ptr(), sc[0].data_ptr(), sc[1].data_ptr(), HS, dw.data_ptr(), dtype,
                            B, F, T, C, k, 1, 2, _st())
    else:
        L.dw_conv_wgrad(dz.data_ptr(), x.data_ptr(), sc[0].data_ptr(), sc[1].data_ptr(), HS, dw.data_ptr(),
                        C * k * k if per_sample else 0, dtype, B, F, T, C, k, s, _st())
    ref = torch.zeros(B if per_sample else 1, C, 1, k, k, device="cuda", dtype=torch.float64)
    mag = torch.zeros_like(ref)
    for b0 in range(0, B, CHUNK):
        sl = slice(b0, b0 + CHUNK)
        _, gw, gm = _grads_ref(x[sl], sc, w, dz[sl], k, s, per_sample=per_sample, dil=dil)
        if per_sample:
            ref[sl], mag[sl] = gw, gm
        else:
            ref[0] += gw
            mag[0] += gm
        del gw, gm
    return _check_sum(dw.view_as(ref), ref, mag, "dW")


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [F32, BF16], ids=["f32", "bf16"])
@pytest.mark.parametrize("case", WGRAD, ids=_ids(WGRAD))
def test_wgrad(case, dtype):
    if dtype == BF16 and case[4] == 5:
        pytest.skip("the bf16 5x5 weight gradient runs on the tile kernel (test_gpu_dw.py)")
    ulps = _check_wgrad(case, dtype, False)
    report(f"[kernel] dw wgrad {case} {dtype}: dW {ulps:.1f} x 2^-24 sum|terms|")


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [F32, BF16], ids=["f32", "bf16"])
@pytest.mark.parametrize("case", WGRAD_PS, ids=_ids(WGRAD_PS))
def test_wgrad_per_sample(case, dtype):
    if dtype == BF16 and case[4] == 5:
        pytest.skip("the bf16 5x5 weight gradient runs on the tile kernel (test_gpu_dw.py)")
    ulps = _check_wgrad(case, dtype, True)
    report(f"[kernel] dw wgrad per-sample {case} {dtype}: dW {ulps:.1f} x 2^-24 sum|terms|")


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [F32, BF16], ids=["f32", "bf16"])
@pytest.mark.parametrize("case", DIL, ids=["B{}_F{}_T{}_C{}_k{}".format(*c) for c in DIL])
def test_dilated_tail(case, dtype):
    """eat_dw_conv_fwd_dil (training and eval), eat_dw_conv_dgrad_dil and eat_dw_conv_wgrad_dil at the bench's batch"""
    B, F, T, C, k = case
    c6 = (B, F, T, C, k, 1)
    _, x, w, wt, sc = _setup(B, F, T, C, k, dtype, seed=400 + C + k)
    _, _, _, e, u_s, u_q = _check_fwd_train(x, w, wt, sc, dtype, c6, HS, dil=2)
    out, pool = _fwd_run(x, wt, dtype, *c6, sc=sc, eval_act=HS, dil=2)
    err = scale = pu = 0.0
    for b0 in range(0, B, CHUNK):
        a = x[b0:b0 + CHUNK].double()
        y = _act(_conv(a, w.double(), k, 1, dil=2) * sc[0].double() + sc[1].double(), HS)
        err = max(err, (out[b0:b0 + CHUNK].double() - y).abs().max().item())
        scale = max(scale, y.abs().max().item())
        mag = (_conv(a.abs(), w.double().abs(), k, 1, dil=2) * sc[0].double() + sc[1].double().abs()).sum((1, 2)) * 1.5
        pu = max(pu, _check_sum(pool[b0:b0 + CHUNK], y.sum((1, 2)), mag, "pool"))
    assert err <= TOL[dtype] * scale, f"eval output: error {err:.3e} vs scale {scale:.3e}"
    del x, out
    e_d = _check_dgrad(c6, dtype, True, False, dil=2)
    u_w = _check_wgrad(c6, dtype, False, dil=2)
    report(f"[kernel] dw dilated {case} {dtype}: train output {e:.2e}, stats {u_s:.1f} / {u_q:.1f}, eval output "
           f"{err / scale:.2e}, pool {pu:.1f}, din {e_d:.2e}, dW {u_w:.1f} x 2^-24")


@pytest.mark.gpu
def test_bwd_fused_at_the_bench_batch():
    """eat_dw_conv_bwd_fused (the bench's default depthwise backward) at B = 256, mn10 block 13 (8x63, C = 672, 5x5
    stride 2, SE, expand), against the fp64 expressions of test_gpu_dw_bwd_fused.py.  din per output; dW and the
    expand BatchNorm's sums per channel against 2^-24 sum |terms|, the terms built from |dz| and |xf| (dW) and from
    |din terms| * act' (the sums)"""
    from tests.test_gpu_dw_bwd_fused import HS as FHS, _act as _fact, _dact, _fused, _inputs, _reference
    B, F, T, C, k, s = 256, 8, 63, 672, 5, 2
    d = _inputs(B, F, T, C, k, s, True, True, seed=5)
    din, dw, sums = _fused(d, B, F, T, C, k, s, FHS)
    rdin, rdw, rsums = _reference(d, k, s, FHS)
    err = (din.double() - rdin).abs().max().item()
    scale = rdin.abs().max().item()
    assert err <= TOL_DIN[F32] * scale, f"din: error {err:.3e} vs scale {scale:.3e}"
    del din, rdin
    D = {n: (v.double() if torch.is_tensor(v) else v) for n, v in d.items()}
    g = D["dp"] * D["gate"][:, None, None, :] + D["dpool"][:, None, None, :]
    dz = D["scale"] * (g * _dact(D["z2"] * D["scale"] + D["shift"], FHS) - D["c1"]
                       - (D["z2"] - D["mean"]) * D["invstd"] * D["c2"])
    u = D["x"] * D["in_scale"] + D["in_shift"]
    xf = _fact(u, FHS).abs().permute(0, 3, 1, 2).requires_grad_(True)
    wa = D["w"].abs().requires_grad_(True)
    gx, gw = torch.autograd.grad(Fn.conv2d(xf, wa, None, s, (k - 1) // 2, 1, C), (xf, wa), dz.abs().permute(0, 3, 1, 2))
    g1mag = gx.permute(0, 2, 3, 1) * _dact(u, FHS).abs()
    smag = torch.stack([g1mag.sum((0, 1, 2)), D["zinvstd"] * (g1mag * (D["x"] - D["zmean"]).abs()).sum((0, 1, 2))])
    u_w = _check_sum(dw, rdw, gw, "dW")
    u_s = _check_sum(sums, rsums, smag, "BN1 sums")
    report(f"[kernel] dw bwd fused B=256: din {err / scale:.2e} of scale, dW {u_w:.1f}, BN1 sums {u_s:.1f} x 2^-24")


# ------------------------------------------------------------------------------------------------ the bounds see defects
# No GPU: each defect a walk could plausibly have is planted in an fp64 reference of a steady-state case, and its
# distance from the clean result must be >= 10x the bound the GPU tests above apply.
def _cpu(B, F, T, C, k, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, F, T, C, generator=g, dtype=torch.float64), torch.randn(C, 1, k, k, generator=g,
                                                                                 dtype=torch.float64) * 0.3


def _seg_starts(pl):
    return range(pl["seg"], pl["rows"], pl["seg"])


def _first_units(pl, B, rows, cols, per_sample=False):
    """mask [B, rows, cols] of the output pixels in the first unit of every thread slot: unit g = (sample, segment,
    strip) in flat order (per sample for a per-sample plan), thread slot g mod gstep"""
    b = torch.arange(B)[:, None, None] * (0 if per_sample else 1)
    r = torch.arange(rows)[None, :, None]
    c = torch.arange(cols)[None, None, :]
    return b * pl["units1"] + (r // pl["seg"]) * -(-cols // pl["P"]) + c // pl["P"] < pl["gstep"]


def test_bounds_see_walk_defects():
    # kind 0: forward (the statistics), mn10 block 13 at B = 16: 2.6 units per slot, 2-row segments of 4, flat walk
    B, F, T, C, k, s = 16, 8, 63, 672, 5, 2
    pl = _plan(0, F32, B, F, T, C, k, s)
    assert pl["per_slot"] >= 2 and 1 < pl["seg"] < pl["rows"] and pl["crosses"]
    x, w = _cpu(B, F, T, C, k, 1)
    x = 4.0 + 0.25 * x
    conv = _conv(x, w, k, s)
    cmag = _conv(x.abs(), w.abs(), k, s)
    scale = conv.abs().max().item()
    pad = (k - 1) // 2
    halo = crossing = 0.0
    for fo in _seg_starts(pl):                                           # segment start without its first input row
        xh = x.clone()
        xh[:, fo * s - pad] = 0
        halo = max(halo, (_conv(xh, w, k, s)[:, fo] - conv[:, fo]).abs().max().item())
    xc = Fn.pad(x, (0, 0, 0, 0, pad, 0))                                 # top halo read from the previous sample
    xc[1:, :pad] = x[:-1, -pad:]
    crossing = (Fn.conv2d(xc.permute(0, 3, 1, 2), w, None, s, (0, pad), 1, C).permute(0, 2, 3, 1)[:, 0]
                - conv[:, 0]).abs()[1:].max().item()
    drop = _first_units(pl, B, *conv.shape[1:3])[..., None].double()   # one unit per thread missing from the sums
    mag = torch.stack([cmag.sum((0, 1, 2)), (cmag * cmag).sum((0, 1, 2))])
    dev = torch.stack([(conv * drop).sum((0, 1, 2)), (conv * conv * drop).sum((0, 1, 2))]).abs()
    stat = (dev / (SUM_ULPS * U * mag)).amax(1)
    # kind 0, per-sample plan (eval with the SE pool): one unit per thread missing from a sample's pool sums
    Bp, Fp, Tp, Cp = 64, 32, 250, 72
    pp = _plan(0, F32, Bp, Fp, Tp, Cp, 3, 1, per_sample=1)
    assert pp["per_slot"] >= 2 and 1 < pp["seg"] < pp["rows"]
    xp, wp = _cpu(Bp, Fp, Tp, Cp, 3, 5)
    xp = 4.0 + 0.25 * xp
    yp, ymag = _conv(xp, wp, 3, 1), _conv(xp.abs(), wp.abs(), 3, 1)
    mp = _first_units(pp, Bp, Fp, Tp, per_sample=True)[..., None].double()
    pool = ((yp * mp).sum((1, 2)).abs() / (SUM_ULPS * U * 1.5 * ymag.sum((1, 2)))).max().item()
    # kind 1: weight gradient, mn10 block 5 (32 x 250, C = 72, 3x3) at B = 16: 2.9 units per slot, 4-row segments
    B1, F1, T1, C1, k1, s1 = 16, 32, 250, 72, 3, 1
    p1 = _plan(1, F32, B1, F1, T1, C1, k1, s1)
    assert p1["per_slot"] >= 2 and 1 < p1["seg"] < p1["rows"]
    x1, w1 = _cpu(B1, F1, T1, C1, k1, 2)
    dz1 = torch.randn(B1, F1, T1, C1, generator=torch.Generator().manual_seed(3), dtype=torch.float64)

    def wg(xx, dd):
        wd = w1.clone().requires_grad_(True)
        return torch.autograd.grad(_conv(xx, wd, k1, s1), wd, dd)[0]
    gw, gmag = wg(x1, dz1), wg(x1.abs(), dz1.abs())
    bound1 = SUM_ULPS * U * gmag
    m1 = _first_units(p1, B1, F1, T1)[..., None].double()
    wdrop = ((wg(x1, dz1 * m1)).abs() / bound1).max().item()
    whalo = 0.0
    for fo in _seg_starts(p1):
        xh = x1.clone()
        xh[:, fo - 1] = 0
        dm = torch.zeros_like(dz1)
        dm[:, fo] = dz1[:, fo]
        whalo = max(whalo, ((wg(xh, dm) - wg(x1, dm)).abs() / bound1).max().item())
    assert p1["crosses"]                         # the top halo row of a sample read from the previous sample
    xc1 = Fn.pad(x1, (0, 0, 0, 0, 1, 1))
    xc1[1:, 0] = x1[:-1, -1]
    wd = w1.clone().requires_grad_(True)
    gwc = torch.autograd.grad(Fn.conv2d(xc1.permute(0, 3, 1, 2), wd, None, 1, (0, 1), 1, C1), wd,
                              dz1.permute(0, 3, 1, 2))[0]
    wcross = ((gwc - gw).abs() / bound1).max().item()
    # kind 2: stride-2 data gradient, mn10 block 13 (din 8 x 63, C = 672, 5x5) at B = 16: 2-pair segments of 4 pairs
    p2 = _plan(2, F32, 16, 8, 63, 672, 5, 2)
    assert p2["per_slot"] >= 2 and 1 < p2["seg"] < p2["rows"] and p2["crosses"]
    dz2, w2 = _cpu(16, 4, 32, 672, 5, 4)

    def dg(dd):
        return Fn.conv_transpose2d(dd.permute(0, 3, 1, 2), w2, None, 2, 2, (1, 0), 672).permute(0, 2, 3, 1)
    din = dg(dz2)
    assert din.shape[1:3] == (8, 63)
    dscale = din.abs().max().item()
    dhalo = 0.0
    for m0 in _seg_starts(p2):                   # the first dz row of the pair's window (m0 - 1 for 5x5) left out
        dh = dz2.clone()
        dh[:, m0 - 1] = 0
        dhalo = max(dhalo, (dg(dh)[:, 2 * m0:2 * m0 + 2] - din[:, 2 * m0:2 * m0 + 2]).abs().max().item())
    m2 = _first_units(p2, 16, p2["rows"], 63).repeat_interleave(2, 1)[..., None].double()   # one unit per thread unstored
    ddrop = (din * m2).abs().max().item()
    dc = dz2.clone()                             # din rows 0, 1 of a sample reading the previous sample's last dz row
    dcross = (dg(torch.cat([dz2[:-1, -1:], dc[1:]], 1))[:, 2:4] - din[1:, :2]).abs().max().item()
    ratios = {"fwd halo": halo / (TOL[F32] * scale), "fwd crossing": crossing / (TOL[F32] * scale),
              "stat_sum dropped unit": stat[0].item(), "stat_sq dropped unit": stat[1].item(),
              "pool dropped unit (per-sample plan)": pool, "dW dropped unit": wdrop, "dW halo": whalo,
              "dW crossing": wcross, "din halo": dhalo / (TOL_DIN[F32] * dscale),
              "din dropped unit": ddrop / (TOL_DIN[F32] * dscale), "din crossing": dcross / (TOL_DIN[F32] * dscale)}
    report("[defect] dw walk: " + ", ".join(f"{n} {r:.0f}x" for n, r in ratios.items()))
    for n, r in ratios.items():
        assert r >= 10, f"{n}: the bound is only {r:.1f}x below the defect"
