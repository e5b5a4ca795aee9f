"""Helpers shared by the steady-state test files (tests/test_gpu_zz_dw_steady.py, test_gpu_zz_pw_steady.py,
test_gpu_zz_dymn_steady.py): the launch planners' views of a case, the long-sum bounds and the fp64 references of the 1x1
GEMMs' weight gradients."""
import ctypes

import torch

from efficientat_b200._lib import lib

RELU, HS = 1, 2
F32, BF16 = 0, 1
U = 2.0 ** -24
SMS = 132                         # H100 SXM
# long-sum bound in units of 2^-24 * sum |terms| (measured on an H100 80GB HBM3 at 700 W: <= 20 without products)
SUM_ULPS = 64
# the bf16x3 products and the tensor core's fp32 accumulation over one flush window of the weight-gradient kernels, of
# sum |terms| (measured <= 1.7e-5); planted defects sit >= 20x above the bound
C_PROD = 1e-4


def out_hw(F, T, k, s):
    pad = (k - 1) // 2
    return (F + 2 * pad - k) // s + 1, (T + 2 * pad - k) // s + 1


def dw_plan(kind, dtype, B, F, T, C, k, s, per_sample=0):
    """eat_dw_plan -> what the walk reaches: units per thread slot, segment rows vs rows, whether a thread's walk crosses
    a sample boundary (flat plan, gy clipped below the CTAs that would give every slot one unit), partial last chunk"""
    plan = (ctypes.c_int * 6)()
    lib().dw_plan(kind, dtype, B, F, T, C, k, s, per_sample, ctypes.addressof(plan))
    chunks, cvc, seg, groups, gy, P = list(plan)
    if kind == 4:
        return dict(chunks=chunks, tiles=seg, groups=groups, gy=gy)
    Fo, To = out_hw(F, T, k, s)
    rows, cols = ((F + 1) // 2, T) if kind == 2 else (Fo, To)
    V = 2 if (kind == 1 and k == 5) else (8 if dtype == BF16 else 4)
    ppb = 128 // cvc
    units1 = -(-cols // P) * -(-rows // seg)                   # units of one sample
    slots = groups * ppb * (1 if per_sample else gy)
    units = units1 * (1 if per_sample else B)
    return dict(chunks=chunks, cvc=cvc, seg=seg, rows=rows, groups=groups, gy=gy, P=P, ppb=ppb, units1=units1,
                gstep=slots, per_slot=units / slots, crosses=not per_sample and gy < -(-units // ppb),
                partial=(C // V) % cvc != 0)


def tma_plan(M, N, K, rps=0):
    pl = (ctypes.c_int * 5)()
    lib().pw_tma_plan(M, N, K, rps, 1, SMS, ctypes.addressof(pl))
    return dict(zip(("BN", "n_tiles", "m_tiles", "grid", "per_cta"), list(pl)))


def chunks(M, cols, budget=1 << 25):
    step = max(128, budget // max(cols, 1))
    return [(m, min(M, m + step)) for m in range(0, M, step)]


def dc(shape, g, device="cuda"):
    """4 + 0.25 randn: positive, mean >> std"""
    return torch.randn(*shape, device=device, generator=g).mul_(0.25).add_(4.0)


def ulps(got, ref, mag):
    """worst |got - ref| in units of 2^-24 mag"""
    return ((got.double() - ref).abs() / (U * mag + 1e-300)).max().item()


def check_prod(got, ref, mag, what, c_prod=C_PROD):
    """|got - ref| <= (c_prod + SUM_ULPS * 2^-24) * mag per entry; returns the worst error in units of 2^-24 mag"""
    u = ((got.double() - ref).abs() / (U * mag + 1e-300)).max().item()
    assert u <= c_prod / U + SUM_ULPS, f"{what}: error {u:.0f} x 2^-24 sum|terms| (bound {c_prod / U + SUM_ULPS:.0f})"
    return u


def fwd_operands(M, N, K, rps, g, dyn_k=4):
    """A [M, K] with a constant first column, W [N, K] (dyn: [dyn_k, N, K] + softmax attention): column n of C has
    mean r_n * s_n and std s_n, r_n from 4 to 24"""
    A = torch.randn(M, K, device="cuda", generator=g)
    A[:, 0] = 1.0
    nw = dyn_k if rps else 1
    W = torch.randn(nw, N, K, device="cuda", generator=g) / K ** 0.5
    s = W[0, :, 1:].norm(dim=1)
    W[:, :, 0] = torch.linspace(4.0, 24.0, N, device="cuda") * s
    att = torch.softmax(torch.randn(M // rps, dyn_k, device="cuda", generator=g), 1) if rps else None
    return A, (W if rps else W[0].contiguous()), att


def _xf(x, sc, act, gate, rps, m0):
    a = x.double()
    if sc is not None:
        a = a * sc[0].double() + sc[1].double()
        a = a.clamp_min(0) if act == RELU else (a * (a + 3).clamp(0, 6) / 6 if act == HS else a)
    if gate is not None:
        rows = torch.arange(m0, m0 + x.shape[0], device=x.device) // rps
        a = a * gate.double()[rows]
    return a


def wgrad_ref(G, X, sc, act, gate, rps, per_sample):
    """fp64 dW ([1, N, K], per sample [B, N, K]) and sum |g| |xf| per entry, in chunks"""
    M, N = G.shape
    K = X.shape[1]
    nb = M // rps if per_sample else 1
    ref = torch.zeros(nb, N, K, device="cuda", dtype=torch.float64)
    mag = torch.zeros_like(ref)
    spans = [(b * rps, (b + 1) * rps) for b in range(nb)] if per_sample else chunks(M, N + K)
    for m0, m1 in spans:
        gg, xx = G[m0:m1].double(), _xf(X[m0:m1], sc, act, gate, rps, m0)
        i = m0 // rps if per_sample else 0
        ref[i] += gg.t() @ xx
        mag[i] += gg.abs().t() @ xx.abs()
        del gg, xx
    return ref, mag
