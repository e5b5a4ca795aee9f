"""eat_pw_tma_wgrad (wgrad_tma.cu) with hi and lo in separate boxes: one of G and X is the m operand (128 channels per
CTA), the other the n operand (an exact-width n tile of up to 128 channels), three bf16 products into one accumulator.
Every 1x1 weight-gradient shape of mn10 at the benchmark's B = 256 (expand, project and the last conv, 10 s clips), the
wide layers of mn40 at B = 64 and dymn20's per-sample project layers at B = 128, plus ragged channel counts down to 4,
against float64 at the criterion of test_gpu_zz_pw_steady.py: |error| <= (C_PROD + SUM_ULPS * 2^-24) * sum |terms| per
entry, g and xf(x) positive so that a dropped block shows against sum |terms|.

The CPU test asserts what the planner reaches at those shapes: both orientations, more than one n tile, more than one
split, and splits longer than the 4,096-row flush window (so the flush runs inside a split, not only at its end).
"""
import ctypes

import pytest
import torch

from efficientat_b200._lib import lib
from tests.test_gpu_zz_pw_steady import (HS, RELU, SMS, U, _check_prod, _dc, _dymn_blocks, _mn_blocks, _p, _peak, _st,
                                         _wgrad_ref)
from tests.util import report

FLUSH_ROWS = 4096
XFS = ("none", "bn_relu", "bn_hs", "gate", "bn_hs_gate")


def _shapes(width, B, blocks):
    """(name, M, N, K, rows per sample) of the expand and project weight gradients of the MN blocks, and the last conv"""
    out = []
    bl = _mn_blocks(width, B)
    for blk, Mi, Mo, cin, cexp, cout, _ in bl:
        if blk not in blocks:
            continue
        if cexp != cin:
            out.append((f"mn{int(width * 10)}_b{blk}_expand", Mi, cexp, cin, Mi // B))
        out.append((f"mn{int(width * 10)}_b{blk}_project", Mo, cout, cexp, Mo // B))
    _, _, Mo, _, _, cout, _ = bl[-1]
    out.append((f"mn{int(width * 10)}_last_conv", Mo, cout * 6, cout, Mo // B))
    return out


def _cases():
    """(name, M, N, K, rows per sample, transform): every mn10 shape that runs on this kernel in the training step
    (blocks 4-15 and the last conv) with the transforms taken in turn, mn40's wide blocks, ragged and tiny channel counts"""
    out = []
    for i, (n, M, N, K, rps) in enumerate(_shapes(1.0, 256, range(4, 16)) + _shapes(4.0, 64, (13, 15))):
        out.append((n, M, N, K, rps, XFS[i % len(XFS)]))
    for N, K in ((4, 8), (8, 4), (24, 40), (200, 184), (960, 240), (112, 672)):
        out.append((f"ragged_{N}x{K}", 100003 // 8 * 8 - 4, N, K, 1250, "bn_hs_gate"))
    return out


def _plan(M, N, K, rps=0, per_sample=0):
    pl = (ctypes.c_int * 6)()
    lib().pw_wgrad_plan(M, N, K, rps, per_sample, SMS, ctypes.addressof(pl))
    return dict(zip(("mb", "tiles", "splits", "rows", "sps", "stages"), list(pl)))


def test_planner_reaches_the_pair_layout_regime():
    plans = {c[0]: (c, _plan(c[1], c[2], c[3])) for c in _cases()}
    for n, (c, pl) in plans.items():
        report(f"[plan] pw_tma_wgrad {n} M={c[1]} N={c[2]} K={c[3]}: MB {pl['mb']}, {pl['tiles']} dW tiles x "
               f"{pl['splits']} splits of {pl['rows']} rows, {pl['stages']} stages")
        assert pl["splits"] * pl["rows"] >= c[1] and pl["stages"] >= 2, (n, pl)
    wide = {n: v for n, v in plans.items() if n.startswith("mn10_b1") or n == "mn10_last_conv"}
    # 128 x BN tiles: mn10 block 12's expand dW [672, 112] is 6 tiles (it was 11 x 2 = 22 tiles of 64 x 64)
    assert plans["mn10_b12_expand"][1]["tiles"] == 6, plans["mn10_b12_expand"]
    assert all(pl["splits"] > 1 for _, pl in wide.values()), wide
    assert any(pl["rows"] > FLUSH_ROWS for c, pl in plans.values() if c[0].startswith("mn10"))
    assert max(pl["tiles"] for _, pl in plans.values()) > 6
    # dymn20's per-sample projects: splits never straddle samples
    for li, _, P, _, cexp, cout in _dymn_blocks(2.0)[::5]:
        pl = _plan(128 * P, cout, cexp, P, 1)
        assert pl["splits"] == 128 * pl["sps"] and pl["sps"] * pl["rows"] >= P, (li, pl)


def _operands(M, N, K, rps, xf, g):
    G, X = _dc((M, N), g), _dc((M, K), g)
    sc = gate = None
    act = 0
    if xf.startswith("bn"):
        sc = torch.stack([torch.rand(K, device="cuda", generator=g) + 0.5, torch.randn(K, device="cuda", generator=g) * 0.1])
        act = HS if "hs" in xf else RELU
    if xf.endswith("gate"):
        gate = torch.rand(M // rps + 1, K, device="cuda", generator=g) + 0.5
    return G, X, sc, act, gate


@pytest.mark.gpu
@pytest.mark.parametrize("case", _cases(), ids=lambda c: f"{c[0]}-{c[5]}")
def test_wgrad_pairs_against_fp64(case):
    name, M, N, K, rps, xf = case
    torch.cuda.reset_peak_memory_stats()
    g = torch.Generator(device="cuda").manual_seed(M % 1000 + N + K)
    G, X, sc, act, gate = _operands(M, N, K, rps, xf, g)
    dW = torch.zeros(N, K, device="cuda")
    lib().pw_tma_wgrad(G.data_ptr(), X.data_ptr(), dW.data_ptr(), M, N, K, _p(sc[0] if sc is not None else None),
                       _p(sc[1] if sc is not None else None), act, _p(gate), rps, 0, _st())
    ref, mag = _wgrad_ref(G, X, sc, act, gate, rps, False)
    u = _check_prod(dW[None], ref, mag, f"dW {name} {xf}")
    report(f"[kernel] pw_tma_wgrad {name} {xf}: dW {u:.0f} x 2^-24 sum|terms| ({u * U:.2e} relative)")
    _peak(f"wgrad pairs {name} {xf}")


@pytest.mark.gpu
@pytest.mark.parametrize("li", [0, 7, 14])
def test_wgrad_pairs_per_sample(li):
    """per-sample mode at dymn20's B = 128: S_b = G_b^T X_b for every sample"""
    _, _, P, _, cexp, cout = _dymn_blocks(2.0)[li]
    B = 128
    M = B * P
    torch.cuda.reset_peak_memory_stats()
    g = torch.Generator(device="cuda").manual_seed(20 + li)
    G, X = _dc((M, cout), g), _dc((M, cexp), g)
    S = torch.zeros(B, cout, cexp, device="cuda")
    lib().pw_tma_wgrad(G.data_ptr(), X.data_ptr(), S.data_ptr(), M, cout, cexp, 0, 0, 0, 0, P, 1, _st())
    ref, mag = _wgrad_ref(G, X, None, 0, None, P, True)
    u = _check_prod(S, ref, mag, f"S dymn20 layer {li}")
    report(f"[kernel] pw_tma_wgrad per sample dymn20 layer {li} B={B}: S {u:.0f} x 2^-24 sum|terms|")
    _peak(f"wgrad pairs per sample {li}")
