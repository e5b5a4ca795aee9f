"""The 1x1 GEMMs in the launch regime the benchmark runs them in: hundreds of 128-row tiles per CTA or split, with the
batch statistics, the weight gradient and the fused backward's dW kept across all of them and the TMA rings going round
hundreds of times.  The cases are mn10 at the benchmark's B = 256 with 10 s clips (mn40 at B = 64, dymn20 at B = 128),
their shapes taken from the models; the launch planners (eat_pw_tma_plan, eat_pw_wgrad_plan, eat_pw_bwd_plan,
eat_pw_proj_bwd_plan) tell what each one reaches and the CPU test below asserts it.

Every kernel result is compared with float64 torch:
  - the statistics of eat_pw_tma_fwd / eat_pw_tma_dyn_fwd (fp32 storage) against fp64 sums of the kernel's own output C
    (prefilled with NaN, so a tile the walk never stores poisons the reference), so that only summation error counts
    (test_gpu_gemm.py bounds the bf16x3 products): |error| <= SUM_ULPS * 2^-24 * sum |C| per column (sum C^2 for the
    sum of squares).  The bf16-storage kernel (eat_pw_tc_fwd, pw_wgmma.cu) sums its fp32 accumulators before the bf16
    store: its sums against fp64 of the product of the same bf16 operands, bounded by SUM_ULPS * 2^-24 * the sums of
    |A| |W|;
  - the variance eat_bn_finalize derives from those sums, on an output with mean/std from 4 to 24 per column (45 for
    dymn20's per-sample kernels), is no further from fp64 than 2x what torch.var_mean in fp32 gets on the same output,
    both saved as an fp32 invstd (the criterion of test_gpu_zz_dw_steady.py).  For the bf16-storage kernel the reference
    is the exact product, which its fp32 accumulators only approximate, so the factor is 4;
  - weight gradients (eat_pw_tma_wgrad on 128-row blocks with each input transform and per sample, wgrad_narrow.cu
    through eat_pw_tc_wgrad, the fused kernels' dW) and the project kernel's BN2 sums:
    |error| <= (C_PROD + SUM_ULPS * 2^-24) * sum |terms| per entry, with g and xf(x) positive (mean >> std) so that a
    dropped tile shows against sum |terms|; C_PROD covers the bf16x3 products and the tensor core's fp32 accumulation
    over one flush window (0 for the exact fp32 narrow kernel).  dX / dp per output, 2e-4 of the tensor's max;
  - eat_bn_bwd_reduce's sums: |error| <= SUM_ULPS * 2^-24 * sum |terms| per channel.
Measured on an H100 80GB HBM3 (700 W).  Variance relative error, kernel / torch.var_mean in fp32, per case: fp32
storage 0.06-0.43 (1.1-2.3e-7); bf16 storage 0.69, 2.23, 2.55 (mn10 blocks 2, 3, 7).  Before the kernels summed as
their comments now state (unshifted per-lane fp32 sums in pw_tma.cu, per-warp fp32 partials across tiles in
pw_wgmma.cu) they were at 1.4e-5-1.0e-4 (fp32) and 1.4-2.3e-5 (bf16).  Statistics sums <= 0.2 (fp32), <= 3.0 (bf16),
reduce <= 0.9, narrow dW 20 x 2^-24 sum |terms|; tensor-core dW and sums <= 280 x 2^-24 = 1.7e-5 of sum |terms|
(wgrad 1.4-1.7e-5, per sample 8.2e-6, fused 1.1-1.7e-5).  Before the weight-gradient kernels flushed their
accumulators every 4,096 rows / 32 tiles, the same cases were at 1.5e-4 (wgrad), 6.6e-5 (per sample) and 3.6e-4
(fused, mn10 block 2), within 6x of a dropped tile.

Without a GPU, test_bounds_see_tile_defects plants the defects a tile walk could have (a tile per CTA or block per
split dropped, one counted twice, a 16-row slab's statistics dropped, a sample's rows attributed to the next sample) in
fp64 references built on the CPU with the rows per CTA / split of the largest case of each family; each lies >= 10x
outside its bound.  References are built in chunks with fp64 sums; peak device memory is asserted below 8 GiB (measured
<= 5.4 GiB).
"""
import contextlib
import ctypes
import io

import pytest
import torch

from efficientat_b200._lib import lib
from tests.steady_util import (C_PROD, HS, RELU, SMS, SUM_ULPS, U, check_prod as _check_prod, chunks as _chunks,
                               dc as _dc, fwd_operands as _fwd_operands, tma_plan as _tma_plan, ulps as _ulps,
                               wgrad_ref as _wgrad_ref)
from tests.util import bn_variance_check, report

TOL_OUT = 2e-4                    # dX / dp of the fused kernels, of the tensor's max
EPS = 1e-3                        # nn.BatchNorm2d(eps=1e-3)
GIB = 2.0 ** 30


def _st():
    return torch.cuda.current_stream().cuda_stream


def _p(t):
    return 0 if t is None else t.data_ptr()


# ------------------------------------------------------------------------------------------------ shapes from the models
def _mn_blocks(width, B, F=64, T=500):
    """(block, rows at the block's input, rows after its depthwise conv, cin, cexp, cout, activation) of every MN block,
    128 mel bins x 1000 frames (stem output 64 x 500)"""
    from efficientat_b200.models.mn.model import get_model
    with contextlib.redirect_stdout(io.StringIO()):
        model = get_model(width_mult=width, verbose=False)
    out = []
    for i, m in enumerate(list(model.features)[1:-1]):
        c = m.cnf
        Mi = B * F * T
        pad = (c.kernel - 1) // 2
        F, T = (F + 2 * pad - c.kernel) // c.stride + 1, (T + 2 * pad - c.kernel) // c.stride + 1
        out.append((i + 1, Mi, B * F * T, c.input_channels, c.expanded_channels, c.out_channels,
                    HS if c.use_hs else RELU))
    return out


def _dymn_blocks(width, F=64, T=500):
    """(layer, rows per sample at the input, after the depthwise conv, cin, cexp, cout) of every DyMN layer"""
    from efficientat_b200.models.dymn.model import get_model
    with contextlib.redirect_stdout(io.StringIO()):
        model = get_model(width_mult=width, verbose=False)
    out = []
    for i, blk in enumerate(model.layers):
        c = blk.cnf
        Pi = F * T
        pad = (c.kernel - 1) // 2
        F, T = (F + 2 * pad - c.kernel) // c.stride + 1, (T + 2 * pad - c.kernel) // c.stride + 1
        out.append((i, Pi, F * T, c.input_channels, c.expanded_channels, c.out_channels))
    return out


def _mn10(block, B=256):
    return next(b for b in _mn_blocks(1.0, B) if b[0] == block)


def _fwd_cases():
    """(name, M, N, K, rows per sample (0: one matrix)) of the training-forward statistics cases: expand layers"""
    out = []
    for blk in (2, 3, 7):                       # 3 and 4 share a shape; 7: N = 240, two N tiles
        _, M, _, cin, cexp, _, _ = _mn10(blk)
        out.append((f"mn10_b{blk}_B256", M, cexp, cin, 0))
    _, M, _, cin, cexp, _, _ = next(b for b in _mn_blocks(4.0, 64) if b[0] == 2)
    out.append(("mn40_b2_B64", M, cexp, cin, 0))
    li, P, _, cin, cexp, _ = next(b for b in _dymn_blocks(2.0) if b[4] != b[3])     # first dymn20 layer with an expand
    out.append((f"dymn20_l{li}_B128", 128 * P, cexp, cin, P))
    return out


def _wgrad_cases():
    """(name, M, N, K, rows per sample of the gate / per-sample mode, per_sample) of eat_pw_tma_wgrad: mn10 block 2's
    expand (dW [64, 16], N <= 64, K <= 32: 128-row blocks) and dymn20's first project (dW [cout, cexp] per sample)"""
    _, M, _, cin, cexp, _, _ = _mn10(2)
    li, _, P, _, cexp_d, cout_d = _dymn_blocks(2.0)[0]
    return [("mn10_b2_B256", M, cexp, cin, 64 * 500, 0),
            (f"dymn20_l{li}_proj_B128_per_sample", 128 * P, cout_d, cexp_d, P, 1)]


def _narrow_case():
    """mn10 block 1's project at B = 256: dW [16, 16] (N * K <= 512: wgrad_narrow.cu)"""
    _, _, M, _, cexp, cout, act = _mn10(1)
    return M, cout, cexp, act


def _expand_cases():
    """(name, M, cexp, cin, act, residual) for eat_pw_conv_bwd_fused: mn10 blocks 2-4, and block 3 with M not a
    multiple of 128"""
    out = []
    for blk in (2, 3, 4):
        _, M, Mo, cin, cexp, cout, act = _mn10(blk)
        out.append((f"mn10_b{blk}", M, cexp, cin, act, cin == cout and Mo == M))
    n, M, cexp, cin, act, res = out[1]
    out.append((n + "_ragged", M - 51, cexp, cin, act, res))
    return out


def _project_cases():
    """(name, M, cexp, cout, act) for eat_pw_proj_bwd_fused: mn10 blocks 1-3 (M after the depthwise conv)"""
    return [(f"mn10_b{b}", _mn10(b)[2], _mn10(b)[4], _mn10(b)[5], _mn10(b)[6]) for b in (1, 2, 3)]


def _reduce_cases():
    """(P, C, act) of eat_bn_bwd_reduce on the expand BatchNorms of mn10 blocks 2 and 3 at B = 256"""
    return [(_mn10(b)[1] // 256, _mn10(b)[4], _mn10(b)[6]) for b in (2, 3)]


# ------------------------------------------------------------------------------------------------ planners
def _wg_plan(M, N, K, rps=0, per_sample=0):
    pl = (ctypes.c_int * 6)()
    lib().pw_wgrad_plan(M, N, K, rps, per_sample, SMS, ctypes.addressof(pl))
    return dict(zip(("mb", "tiles", "splits", "rows", "sps", "stages"), list(pl)))


def _fused_plan(proj, M, cexp, cn):
    pl = (ctypes.c_int * 4)()
    (lib().pw_proj_bwd_plan if proj else lib().pw_bwd_plan)(M, cexp, cn, ctypes.addressof(pl))
    return dict(zip(("ctas", "rows", "stages", "smem"), list(pl)))


def _narrow_slabs_per_cta(M):
    """wgrad_narrow.cu's launch: 64-row slabs, grid min(slabs, 4 x 132), CTA b takes slabs b, b + grid, ..."""
    slabs = -(-M // 64)
    return -(-slabs // min(slabs, 4 * SMS))


def test_cases_reach_the_steady_state():
    fwd = {n: _tma_plan(M, N, K, rps) for n, M, N, K, rps in _fwd_cases()}
    for n, pl in fwd.items():
        report(f"[plan] pw_tma fwd {n}: N tile {pl['BN']} x {pl['n_tiles']}, {pl['m_tiles']} M tiles on {pl['grid']} "
               f"CTAs, up to {pl['per_cta']} M tiles per CTA")
    assert max(pl["per_cta"] for pl in fwd.values()) >= 400, fwd
    assert any(pl["n_tiles"] == 2 for pl in fwd.values())
    # eat_pw_tma_wgrad at the benchmark's M: mn10 block 2's expand (dW [64, 16]) on 128-row blocks, and dymn20's first
    # project per sample (dW [cout, cexp] of 32,000 rows per sample) in more than one split per sample
    _, M, _, cin, cexp, _, _ = _mn10(2)
    p0 = _wg_plan(M, cexp, cin)
    li, _, P, _, cexp_d, cout_d = _dymn_blocks(2.0)[0]
    p1 = _wg_plan(128 * P, cout_d, cexp_d, P, 1)
    for n, pl in (("mn10_b2_B256", p0), (f"dymn20_l{li}_proj_B128_per_sample", p1)):
        report(f"[plan] pw_tma_wgrad {n}: MB {pl['mb']}, {pl['tiles']} dW tiles x {pl['splits']} splits of {pl['rows']} "
               f"rows ({pl['sps']} per sample), {pl['stages']} stages")
    assert p0["mb"] == 128 and p0["rows"] // 128 >= 100 and p0["splits"] * p0["rows"] >= M, p0
    assert p1["mb"] == 64 and p1["sps"] > 1 and p1["splits"] == 128 * p1["sps"] and p1["sps"] * p1["rows"] >= P, p1
    M, N, K, _ = _narrow_case()
    assert N * K <= 512 and _narrow_slabs_per_cta(M) >= 100
    for proj, cases in ((False, _expand_cases()), (True, _project_cases())):
        for n, M, cexp, cn, *_ in cases:
            pl = _fused_plan(proj, M, cexp, cn)
            report(f"[plan] pw {'proj' if proj else 'conv'}_bwd_fused {n}: M {M}, {pl['ctas']} CTAs x "
                   f"{pl['rows'] // 128} tiles, {pl['stages']} stages")
            assert pl["rows"] // 128 >= 100, (n, pl)
    assert any(M % 128 for _, M, *_ in _expand_cases())


# ------------------------------------------------------------------------------------------------ helpers
def _check(got, ref, mag, what):
    u = _ulps(got, ref, mag)
    assert u <= SUM_ULPS, f"{what}: error {u:.1f} x 2^-24 sum|terms| (bound {SUM_ULPS})"
    return u


def _peak(what):
    peak = torch.cuda.max_memory_allocated() / GIB
    report(f"[kernel] pw {what}: peak device memory {peak:.2f} GiB")
    assert peak < 8, f"{what}: peak device memory {peak:.2f} GiB"


# ------------------------------------------------------------------------------------------------ forward statistics
@pytest.mark.gpu
@pytest.mark.parametrize("case", _fwd_cases(), ids=lambda c: c[0])
def test_forward_statistics_at_the_bench_batch(case):
    name, M, N, K, rps = case
    L = lib()
    torch.cuda.reset_peak_memory_stats()
    g = torch.Generator(device="cuda").manual_seed(M % 9973 + N)
    A, W, att = _fwd_operands(M, N, K, rps, g)
    C = torch.full((M, N), float("nan"), device="cuda")          # rows the walk never stores poison the reference
    stats = torch.zeros(2, N, device="cuda", dtype=torch.float64)
    if rps:
        ws = torch.empty((M // rps) * N * ((K + 31) // 32) * 128, device="cuda", dtype=torch.uint8)
        L.pw_tma_dyn_fwd(A.data_ptr(), W.data_ptr(), att.data_ptr(), W.shape[0], 0, C.data_ptr(), M, N, K, rps, 0, 0, 0,
                         0, stats[0].data_ptr(), stats[1].data_ptr(), ws.data_ptr(), ws.numel(), _st())
        del ws
    else:
        L.pw_tma_fwd(A.data_ptr(), W.data_ptr(), 0, C.data_ptr(), M, N, K, 0, 0, 0, 0, 1, 0, 0, 0, 0,
                     stats[0].data_ptr(), stats[1].data_ptr(), 0, 0, _st())
    del A
    ref = torch.zeros(2, N, device="cuda", dtype=torch.float64)
    mag = torch.zeros(N, device="cuda", dtype=torch.float64)
    for m0, m1 in _chunks(M, N):
        c = C[m0:m1].double()
        ref += torch.stack([c.sum(0), (c * c).sum(0)])
        mag += c.abs().sum(0)
        del c
    u_s = _ulps(stats[0], ref[0], mag)
    u_q = _ulps(stats[1], ref[1], ref[1])
    report(f"[kernel] pw_tma fwd stats {name} (M {M}, N {N}, K {K}): stat_sum {u_s:.1f} / stat_sq {u_q:.1f} "
           f"x 2^-24 sum|terms|")
    bn_variance_check(C, stats, ref, M, N, EPS, f"pw_tma fwd stats {name}")
    assert u_s <= SUM_ULPS and u_q <= SUM_ULPS, (u_s, u_q)
    _peak(f"fwd stats {name}")


@pytest.mark.gpu
@pytest.mark.parametrize("case", [c for c in _fwd_cases() if c[0].startswith("mn10")], ids=lambda c: c[0])
def test_forward_statistics_bf16_storage(case):
    """eat_pw_tc_fwd with bf16 activations (pw_wgmma.cu): statistics of the fp32 accumulators, against fp64 of the
    product of the same bf16 operands; the variance against torch.var_mean of that product rounded to fp32"""
    name, M, N, K, _ = case
    torch.cuda.reset_peak_memory_stats()
    g = torch.Generator(device="cuda").manual_seed(M % 9973 + N + 1)
    A, W, _ = _fwd_operands(M, N, K, 0, g)
    A = A.bfloat16()
    Wb = W.bfloat16().double()
    C = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    stats = torch.zeros(2, N, device="cuda", dtype=torch.float64)
    lib().pw_tc_fwd(A.data_ptr(), 1, W.data_ptr(), 0, C.data_ptr(), 1, M, N, K, 0, 0, 0, 0, 1, 0, 0, 0, 0,
                    stats[0].data_ptr(), stats[1].data_ptr(), _st())
    del C
    ref = torch.zeros(2, N, device="cuda", dtype=torch.float64)
    mag = torch.zeros(2, N, device="cuda", dtype=torch.float64)
    P32 = torch.empty(M, N, device="cuda")
    for m0, m1 in _chunks(M, N):
        a = A[m0:m1].double()
        c, cm = a @ Wb.t(), a.abs() @ Wb.abs().t()
        P32[m0:m1] = c
        ref += torch.stack([c.sum(0), (c * c).sum(0)])
        mag += torch.stack([cm.sum(0), (cm * cm).sum(0)])
        del a, c, cm
    del A
    u_s = _ulps(stats[0], ref[0], mag[0])
    u_q = _ulps(stats[1], ref[1], mag[1])
    report(f"[kernel] pw_tc fwd bf16 stats {name}: stat_sum {u_s:.1f} / stat_sq {u_q:.1f} x 2^-24 sum|terms|")
    bn_variance_check(P32, stats, ref, M, N, EPS, f"pw_tc fwd bf16 stats {name}", factor=4)
    assert u_s <= SUM_ULPS and u_q <= SUM_ULPS, (u_s, u_q)
    _peak(f"fwd bf16 stats {name}")


# ------------------------------------------------------------------------------------------------ weight gradients
WGRAD_XF = [("none", None), ("bn_relu", RELU), ("bn_hs", HS), ("gate", "gate")]


@pytest.mark.gpu
@pytest.mark.parametrize("xf", WGRAD_XF, ids=lambda x: x[0])
def test_wgrad_128_row_blocks(xf):
    """eat_pw_tma_wgrad at mn10 block 2's expand, B = 256: MB = 128, ~31k rows per split; g and xf(x) positive"""
    name, M, N, K, rps, _ = _wgrad_cases()[0]
    torch.cuda.reset_peak_memory_stats()
    g = torch.Generator(device="cuda").manual_seed(11 + len(xf[0]))
    G, X = _dc((M, N), g), _dc((M, K), g)
    sc = gate = None
    act = 0
    if xf[1] in (RELU, HS):
        sc = torch.stack([torch.rand(K, device="cuda", generator=g) + 0.5, torch.randn(K, device="cuda", generator=g) * 0.1])
        act = xf[1]
    elif xf[1] == "gate":
        gate = torch.rand(M // rps, K, device="cuda", generator=g) + 0.5
    dW = torch.zeros(N, K, device="cuda")
    lib().pw_tma_wgrad(G.data_ptr(), X.data_ptr(), dW.data_ptr(), M, N, K, _p(sc[0] if sc is not None else None),
                       _p(sc[1] if sc is not None else None), act, _p(gate), rps, 0, _st())
    ref, mag = _wgrad_ref(G, X, sc, act, gate, rps, False)
    u = _check_prod(dW[None], ref, mag, f"dW {name} {xf[0]}")
    report(f"[kernel] pw_tma_wgrad MB=128 {name} {xf[0]}: dW {u:.0f} x 2^-24 sum|terms| ({u * U:.2e} relative)")
    _peak(f"wgrad {name} {xf[0]}")


@pytest.mark.gpu
def test_wgrad_per_sample():
    """eat_pw_tma_wgrad per sample at dymn20's B = 128 x 32,000 rows: two splits per sample"""
    name, M, N, K, rps, _ = _wgrad_cases()[1]
    torch.cuda.reset_peak_memory_stats()
    g = torch.Generator(device="cuda").manual_seed(12)
    G, X = _dc((M, N), g), _dc((M, K), g)
    S = torch.zeros(M // rps, N, K, device="cuda")
    lib().pw_tma_wgrad(G.data_ptr(), X.data_ptr(), S.data_ptr(), M, N, K, 0, 0, 0, 0, rps, 1, _st())
    ref, mag = _wgrad_ref(G, X, None, 0, None, rps, True)
    u = _check_prod(S, ref, mag, f"S {name}")
    report(f"[kernel] pw_tma_wgrad per sample {name}: S {u:.0f} x 2^-24 sum|terms| ({u * U:.2e} relative)")
    _peak(f"wgrad per sample {name}")


@pytest.mark.gpu
def test_wgrad_narrow_long_reduction(monkeypatch):
    """wgrad_narrow.cu (exact fp32 FMAs) through eat_pw_tc_wgrad at mn10 block 1's project, B = 256; fp32 launches take
    it when EAT_WG_NARROW is set (the default is eat_pw_tma_wgrad)"""
    monkeypatch.setenv("EAT_WG_NARROW", "1")
    M, N, K, act = _narrow_case()
    torch.cuda.reset_peak_memory_stats()
    g = torch.Generator(device="cuda").manual_seed(13)
    G, X = _dc((M, N), g), _dc((M, K), g)
    sc = torch.stack([torch.rand(K, device="cuda", generator=g) + 0.5, torch.randn(K, device="cuda", generator=g) * 0.1])
    dW = torch.zeros(N, K, device="cuda")
    lib().pw_tc_wgrad(G.data_ptr(), 0, X.data_ptr(), 0, dW.data_ptr(), 0, M, N, K, sc[0].data_ptr(), sc[1].data_ptr(),
                      act, 0, 1, _st())
    ref, mag = _wgrad_ref(G, X, sc, act, None, 1, False)
    u = _check_prod(dW[None], ref, mag, "dW narrow", 0.0)
    report(f"[kernel] wgrad_narrow M {M} N {N} K {K}: dW {u:.1f} x 2^-24 sum|terms|")
    _peak("wgrad narrow")


# ------------------------------------------------------------------------------------------------ fused backward
def _act(v, a):
    return v.clamp_min(0) if a == RELU else v * (v + 3).clamp(0, 6) / 6


@pytest.mark.gpu
@pytest.mark.parametrize("case", _expand_cases(), ids=lambda c: c[0])
def test_expand_bwd_fused_at_the_bench_batch(case):
    name, M, cexp, cin, act, res = case
    torch.cuda.reset_peak_memory_stats()
    g = torch.Generator(device="cuda").manual_seed(M % 9973 + cexp)
    da, z, x = _dc((M, cexp), g), _dc((M, cexp), g), _dc((M, cin), g)
    t = _bn_tables(cexp, g)
    w = torch.randn(cexp, cin, device="cuda", generator=g) / cexp ** 0.5
    r = torch.randn(M, cin, device="cuda", generator=g) if res else None
    dx = torch.full((M, cin), float("nan"), device="cuda")
    dw = torch.zeros(cexp, cin, device="cuda")
    lib().pw_conv_bwd_fused(da.data_ptr(), z.data_ptr(), t["scale"].data_ptr(), t["shift"].data_ptr(),
                            t["mean"].data_ptr(), t["invstd"].data_ptr(), act, t["c1"].data_ptr(), t["c2"].data_ptr(),
                            x.data_ptr(), w.data_ptr(), _p(r), dx.data_ptr(), dw.data_ptr(), 0, M, cexp, cin, _st())
    D = {k: v.double() for k, v in t.items()}
    rdw = torch.zeros(cexp, cin, device="cuda", dtype=torch.float64)
    mag = torch.zeros_like(rdw)
    err = scale = 0.0
    for m0, m1 in _chunks(M, 2 * cexp + cin):
        zz = z[m0:m1].double()
        dz = D["scale"] * (da[m0:m1].double() * _dact(zz * D["scale"] + D["shift"], act) - D["c1"]
                           - (zz - D["mean"]) * D["invstd"] * D["c2"])
        del zz
        want = dz @ w.double()
        if r is not None:
            want += r[m0:m1].double()
        err = max(err, (dx[m0:m1].double() - want).abs().max().item())
        scale = max(scale, want.abs().max().item())
        xx = x[m0:m1].double()
        rdw += dz.t() @ xx
        mag += dz.abs().t() @ xx.abs()
        del dz, want, xx
    assert err <= TOL_OUT * scale, f"dX: error {err:.3e} vs scale {scale:.3e}"
    u = _check_prod(dw, rdw, mag, f"dW {name}")
    report(f"[kernel] pw_conv_bwd_fused {name} (M {M}): dX {err / scale:.2e} of scale, dW {u:.0f} x 2^-24 sum|terms| "
           f"({u * U:.2e} relative)")
    _peak(f"conv_bwd_fused {name}")


@pytest.mark.gpu
@pytest.mark.parametrize("case", _project_cases(), ids=lambda c: c[0])
def test_project_bwd_fused_at_the_bench_batch(case):
    name, M, cexp, cout, act = case
    torch.cuda.reset_peak_memory_stats()
    g = torch.Generator(device="cuda").manual_seed(M % 9973 + cout)
    dy, z3, z2 = _dc((M, cout), g), _dc((M, cout), g), _dc((M, cexp), g)
    t3, t2 = _bn_tables(cout, g), _bn_tables(cexp, g)
    w = torch.rand(cout, cexp, device="cuda", generator=g) / cout ** 0.5        # positive: dp > 0
    dp = torch.full((M, cexp), float("nan"), device="cuda")
    dw = torch.zeros(cout, cexp, device="cuda")
    s = torch.zeros(2, cexp, device="cuda", dtype=torch.float64)
    lib().pw_proj_bwd_fused(dy.data_ptr(), z3.data_ptr(), t3["scale"].data_ptr(), t3["shift"].data_ptr(),
                            t3["mean"].data_ptr(), t3["invstd"].data_ptr(), t3["c1"].data_ptr(), t3["c2"].data_ptr(),
                            z2.data_ptr(), t2["scale"].data_ptr(), t2["shift"].data_ptr(), t2["mean"].data_ptr(),
                            t2["invstd"].data_ptr(), act, w.data_ptr(), dp.data_ptr(), dw.data_ptr(), s[0].data_ptr(),
                            s[1].data_ptr(), 0, M, cexp, cout, _st())
    D3 = {k: v.double() for k, v in t3.items()}
    D2 = {k: v.double() for k, v in t2.items()}
    rdw = torch.zeros(cout, cexp, device="cuda", dtype=torch.float64)
    wmag = torch.zeros_like(rdw)
    rs = torch.zeros(2, cexp, device="cuda", dtype=torch.float64)
    smag = torch.zeros_like(rs)
    err = scale = 0.0
    for m0, m1 in _chunks(M, 2 * cout + 3 * cexp):
        zz = z3[m0:m1].double()
        dz = D3["scale"] * (dy[m0:m1].double() - D3["c1"] - (zz - D3["mean"]) * D3["invstd"] * D3["c2"])
        del zz
        want = dz @ w.double()
        err = max(err, (dp[m0:m1].double() - want).abs().max().item())
        scale = max(scale, want.abs().max().item())
        z2d = z2[m0:m1].double()
        u = z2d * D2["scale"] + D2["shift"]
        xf = _act(u, act)
        rdw += dz.t() @ xf
        wmag += dz.abs().t() @ xf.abs()
        gg = want * _dact(u, act)
        t2s = gg * (z2d - D2["mean"]) * D2["invstd"]
        rs += torch.stack([gg.sum(0), t2s.sum(0)])
        smag += torch.stack([gg.abs().sum(0), t2s.abs().sum(0)])
        del dz, want, z2d, u, xf, gg, t2s
    assert err <= TOL_OUT * scale, f"dp: error {err:.3e} vs scale {scale:.3e}"
    u_w = _check_prod(dw, rdw, wmag, f"dW {name}")
    # the BN2 sums take dp from the bf16x3 products: each term carries their error
    u_s1 = _check_prod(s[0], rs[0], smag[0], f"s1 {name}")
    u_s2 = _check_prod(s[1], rs[1], smag[1], f"s2 {name}")
    report(f"[kernel] pw_proj_bwd_fused {name} (M {M}): dp {err / scale:.2e} of scale, dW {u_w:.0f}, s1 {u_s1:.0f}, "
           f"s2 {u_s2:.0f} x 2^-24 sum|terms|")
    _peak(f"proj_bwd_fused {name}")


def _dact(v, a):
    if a == RELU:
        return (v > 0).to(v.dtype)
    return torch.where(v < -3, torch.zeros_like(v), torch.where(v <= 3, (2 * v + 3) / 6, torch.ones_like(v)))


def _bn_tables(C, g):
    u = lambda: torch.rand(C, device="cuda", generator=g)
    r = lambda: torch.randn(C, device="cuda", generator=g)
    # scale, shift, mean, invstd of a BatchNorm whose input is 4 + 0.25 randn; c1 / c2 small, so that dz > 0
    return dict(scale=u() + 0.5, shift=r() * 0.3, mean=4.0 + r() * 0.02, invstd=3.0 + u() * 2, c1=r() * 0.1,
                c2=r() * 0.1)


# ------------------------------------------------------------------------------------------------ BatchNorm-backward reduce
@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [0, 1], ids=["f32", "bf16"])
@pytest.mark.parametrize("case", _reduce_cases(), ids=lambda c: f"P{c[0]}_C{c[1]}")
def test_bn_bwd_reduce_at_the_bench_batch(case, dtype):
    P, C, act = case
    B = 256
    torch.cuda.reset_peak_memory_stats()
    g = torch.Generator(device="cuda").manual_seed(P + C + dtype)
    dt = torch.bfloat16 if dtype else torch.float32
    gA, z = _dc((B, P, C), g).to(dt), _dc((B, P, C), g).to(dt)
    t = _bn_tables(C, g)
    s = torch.zeros(2, C, device="cuda", dtype=torch.float64)
    lib().bn_bwd_reduce(gA.data_ptr(), 0, 0, z.data_ptr(), t["scale"].data_ptr(), t["shift"].data_ptr(),
                        t["mean"].data_ptr(), t["invstd"].data_ptr(), act, dtype, B, P, C, s[0].data_ptr(),
                        s[1].data_ptr(), _st())
    D = {k: v.double() for k, v in t.items()}
    ref = torch.zeros(2, C, device="cuda", dtype=torch.float64)
    mag = torch.zeros_like(ref)
    bs = max(1, (1 << 24) // (P * C))
    for b0 in range(0, B, bs):
        zz = z[b0:b0 + bs].double()
        dy = gA[b0:b0 + bs].double() * _dact(zz * D["scale"] + D["shift"], act)
        t2 = dy * (zz - D["mean"]) * D["invstd"]
        ref += torch.stack([dy.sum((0, 1)), t2.sum((0, 1))])
        mag += torch.stack([dy.abs().sum((0, 1)), t2.abs().sum((0, 1))])
        del zz, dy, t2
    u1 = _check(s[0], ref[0], mag[0], "s1")
    u2 = _check(s[1], ref[1], mag[1], "s2")
    report(f"[kernel] bn_bwd_reduce B {B} P {P} C {C} {'bf16' if dtype else 'fp32'}: s1 {u1:.1f} / s2 {u2:.1f} "
           f"x 2^-24 sum|terms|")
    _peak(f"bn_bwd_reduce P {P} C {C}")


# ------------------------------------------------------------------------------------------------ the bounds see defects
# No GPU: the defects a tile walk could have, planted in an fp64 reference built on the CPU with the tiles per CTA of the
# largest statistics case (two CTAs' worth of rows: every CTA carries the same defect, so its share of a sum does not
# depend on the number of CTAs).  Each must lie >= 10x outside the bound the GPU tests above apply.
def _sep(delta, bound):
    return (delta.abs() / bound).max().item()


def _cpu_dc(shape, g):
    return torch.randn(*shape, generator=g, dtype=torch.float64) * 0.25 + 4.0


def test_bounds_see_tile_defects():
    g = torch.Generator().manual_seed(3)
    ratios = {}
    # training-forward statistics: mn10 block 2 at B = 256, 485 M tiles per CTA, 8 consumer warps of 16 rows per tile
    _, M, N, K, _ = _fwd_cases()[0]
    tiles = _tma_plan(M, N, K)["per_cta"]
    A = torch.randn(2 * tiles * 128, K, generator=g, dtype=torch.float64)
    A[:, 0] = 1.0
    W = torch.randn(N, K, generator=g, dtype=torch.float64) / K ** 0.5
    W[:, 0] = torch.linspace(4.0, 24.0, N, dtype=torch.float64) * W[:, 1:].norm(dim=1)
    C = (A @ W.t()).view(2, tiles, 128, N)
    terms = torch.stack([C, C * C])                                          # [2 sums, CTA, tile, row, N]
    bound = SUM_ULPS * U * torch.stack([C.abs().sum((0, 1, 2)), (C * C).sum((0, 1, 2))])
    ratios["stats: tile dropped"] = _sep(terms[:, :, 0].sum((1, 2)), bound)
    ratios["stats: tile counted twice"] = _sep(terms[:, :, 1].sum((1, 2)), bound)
    ratios["stats: 16-row slab dropped"] = _sep(terms[:, :, 2, :16].sum((1, 2)), bound)
    # eat_pw_tma_wgrad, 128-row blocks: one split of mn10 block 2 at B = 256 (two splits' worth of rows)
    _, M, N, K, rps, _ = _wgrad_cases()[0]
    pl = _wg_plan(M, N, K)
    blocks = pl["rows"] // pl["mb"]
    G, X = _cpu_dc((2, blocks, pl["mb"], N), g), _cpu_dc((2, blocks, pl["mb"], K), g)
    bound = (C_PROD + SUM_ULPS * U) * torch.einsum("sbrn,sbrk->nk", G, X)      # every term positive
    ratios["wgrad MB=128: block dropped"] = _sep(torch.einsum("srn,srk->nk", G[:, 0], X[:, 0]), bound)
    ratios["wgrad MB=128: block counted twice"] = _sep(torch.einsum("srn,srk->nk", G[:, 1], X[:, 1]), bound)
    # per sample: dymn20 at 32,000 rows per sample in 64-row blocks; a block of one sample's rows attributed to the next
    # sample moves that block out of one sample's S and into the other's
    _, M, N, K, rps, _ = _wgrad_cases()[1]
    mb = _wg_plan(M, N, K, rps, 1)["mb"]
    Gs, Xs = _cpu_dc((2, rps, N), g), _cpu_dc((2, rps, K), g)
    bound = (C_PROD + SUM_ULPS * U) * torch.einsum("brn,brk->bnk", Gs, Xs)
    last = torch.einsum("rn,rk->nk", Gs[0, -mb:], Xs[0, -mb:])
    ratios["wgrad per sample: block dropped"] = _sep(torch.einsum("rn,rk->nk", Gs[0, :mb], Xs[0, :mb]), bound[0])
    ratios["wgrad per sample: rows attributed to the next sample"] = min(_sep(last, bound[0]), _sep(last, bound[1]))
    # wgrad_narrow: one 64-row slab per CTA dropped (exact fp32: no product term)
    M, N, K, _ = _narrow_case()
    slabs = _narrow_slabs_per_cta(M)
    Gn, Xn = _cpu_dc((slabs, 64, N), g), _cpu_dc((slabs, 64, K), g)
    bound = SUM_ULPS * U * torch.einsum("srn,srk->nk", Gn, Xn)
    ratios["wgrad narrow: slab dropped"] = _sep(torch.einsum("rn,rk->nk", Gn[0], Xn[0]), bound)
    # fused backward: dW of the expand kernel (mn10 block 2), dW and the BN2 sum s1 of the project kernel (block 1), one
    # CTA's tiles; the terms are positive as in the GPU tests
    for proj, (n, M, cexp, cn, *_) in ((False, _expand_cases()[0]), (True, _project_cases()[0])):
        tiles = _fused_plan(proj, M, cexp, cn)["rows"] // 128
        dz, xf = _cpu_dc((tiles, 128, cn if proj else cexp), g), _cpu_dc((tiles, 128, cexp if proj else cn), g)
        bound = (C_PROD + SUM_ULPS * U) * torch.einsum("trn,trk->nk", dz, xf)
        what = "proj" if proj else "expand"
        ratios[f"{what} fused dW: tile dropped"] = _sep(torch.einsum("rn,rk->nk", dz[0], xf[0]), bound)
        ratios[f"{what} fused dW: tile counted twice"] = _sep(torch.einsum("rn,rk->nk", dz[1], xf[1]), bound)
        if proj:
            bound = (C_PROD + SUM_ULPS * U) * xf.sum((0, 1))                   # g = dp * act' > 0, terms like xf
            ratios["proj fused s1: tile dropped"] = _sep(xf[0].sum(0), bound)
    report("[defect] pw tile walk: " + ", ".join(f"{n} {r:.0f}x" for n, r in ratios.items()))
    for n, r in ratios.items():
        assert r >= 10, f"{n}: the bound is only {r:.1f}x below the defect"
