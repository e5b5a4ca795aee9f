"""Per-layer benchmark of the project stage's backward at the mn10 shapes of every block without SE (fp32): the five passes
(BN3-backward reduce and apply, weight-gradient GEMM with BN2 + activation on load, data-gradient GEMM, BN2-backward
reduce on (dp, z2)) against the BN3 reduce plus eat_pw_proj_bwd_fused, L2 flushed before every timed call.  Prints
algorithmic bytes and GB/s of both and checks that they agree (dp 2e-5 and dW 1e-4 of the tensor's max, BN2 sums 1e-4 of
their largest entry); blocks the fused kernel does not take print the five passes only.  Then the stem: the
BatchNorm-backward apply pass plus the weight gradient against eat_stem_wgrad with the apply on load.  One JSON summary
line at the end."""
import argparse
import contextlib
import ctypes
import io
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from efficientat_b200._lib import EatError, lib  # noqa: E402
from efficientat_b200.models.mn.model import get_model  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=256)
ap.add_argument("--frames", type=int, default=1001, help="spectrogram frames (a 10 s clip at 32 kHz, hop 320)")
ap.add_argument("--reps", type=int, default=5)
a = ap.parse_args()


def conv_out(n, k, s):
    return (n + 2 * ((k - 1) // 2) - k) // s + 1


def layers():
    """(block, rows per sample, cexp, cout, act) of each project stage without SE, mn10 with a 128-bin spectrogram"""
    with contextlib.redirect_stdout(io.StringIO()):
        model = get_model(width_mult=1.0, verbose=False)
    F, T = conv_out(128, 3, 2), conv_out(a.frames, 3, 2)
    out = []
    for i, m in enumerate(list(model.features)[1:-1]):
        c = m.cnf
        F, T = conv_out(F, c.kernel, c.stride), conv_out(T, c.kernel, c.stride)
        if not c.use_se:
            out.append((i + 1, F * T, c.expanded_channels, c.out_channels, 2 if c.use_hs else 1))
    return out


L = lib()
st = torch.cuda.current_stream().cuda_stream
flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")


def timeit(fn):
    fn()
    ts = []
    for _ in range(a.reps):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return sorted(ts)[len(ts) // 2]


def close(x, y, tol):
    return (x.double() - y.double()).abs().max().item() <= tol * y.double().abs().max().item() + 1e-12


B = a.batch
tot = {"chain_ms": 0.0, "fused_ms": 0.0, "chain_gb": 0.0, "fused_gb": 0.0}
fused_blocks = []
all_ok = True
plan = (ctypes.c_int * 4)()
for blk, P, cexp, cout, act in layers():
    M = B * P
    try:
        L.pw_proj_bwd_plan(M, cexp, cout, ctypes.addressof(plan))
        takes = True
    except EatError:
        takes = False
    g = torch.Generator(device="cuda").manual_seed(blk)
    r = lambda *sh: torch.randn(*sh, device="cuda", generator=g)
    u = lambda *sh: torch.rand(*sh, device="cuda", generator=g)
    dy, z3, z2 = r(M, cout), r(M, cout), r(M, cexp)
    w = r(cout, cexp) / cout ** 0.5
    bn3 = [u(cout) + 0.5, r(cout) * 0.3, r(cout) * 0.2, u(cout) + 0.5]      # scale, shift, mean, invstd
    bn2 = [u(cexp) + 0.5, r(cexp) * 0.3, r(cexp) * 0.2, u(cexp) + 0.5]
    c12 = [r(cout) * 0.1, r(cout) * 0.1]
    s3 = torch.zeros(2, cout, device="cuda", dtype=torch.float64)
    dz3 = torch.empty_like(z3)
    dp_c, dp_f = torch.empty(M, cexp, device="cuda"), torch.empty(M, cexp, device="cuda")
    dw_c, dw_f = torch.zeros(cout, cexp, device="cuda"), torch.zeros(cout, cexp, device="cuda")
    s2_c, s2_f = (torch.zeros(2, cexp, device="cuda", dtype=torch.float64) for _ in range(2))
    ws = torch.empty(cexp * ((cout + 31) // 32) * 128, device="cuda", dtype=torch.uint8)
    P3, P2 = [t.data_ptr() for t in bn3], [t.data_ptr() for t in bn2]

    def bn3_reduce():
        L.bn_bwd_reduce(dy.data_ptr(), 0, 0, z3.data_ptr(), *P3, 0, 0, 1, M, cout, s3[0].data_ptr(), s3[1].data_ptr(), st)

    def chain():
        bn3_reduce()
        L.bn_bwd_apply(dy.data_ptr(), 0, 0, z3.data_ptr(), *P3, 0, c12[0].data_ptr(), c12[1].data_ptr(), dz3.data_ptr(),
                       0, 1, M, cout, st)
        L.pw_tc_wgrad(dz3.data_ptr(), 0, z2.data_ptr(), 0, dw_c.data_ptr(), 0, M, cout, cexp, P2[0], P2[1], act, 0, 1, st)
        L.pw_tma_fwd(dz3.data_ptr(), w.data_ptr(), 1, dp_c.data_ptr(), M, cexp, cout, 0, 0, 0, 0, 1, 0, 0, 0, 0, 0, 0,
                     ws.data_ptr(), ws.numel(), st)
        L.bn_bwd_reduce(dp_c.data_ptr(), 0, 0, z2.data_ptr(), *P2, act, 0, 1, M, cexp, s2_c[0].data_ptr(),
                        s2_c[1].data_ptr(), st)

    def fused():
        bn3_reduce()
        L.pw_proj_bwd_fused(dy.data_ptr(), z3.data_ptr(), *P3, c12[0].data_ptr(), c12[1].data_ptr(), z2.data_ptr(), *P2,
                            act, w.data_ptr(), dp_f.data_ptr(), dw_f.data_ptr(), s2_f[0].data_ptr(), s2_f[1].data_ptr(), 0,
                            M, cexp, cout, st)

    # algorithmic bytes (fp32 elements of the tensors each pass must read or write); the BN3 reduce is in both
    To, T2 = M * cout * 4, M * cexp * 4
    b_c = 2 * To + 3 * To + (To + T2) + (To + T2) + 2 * T2
    b_f = 2 * To + 2 * To + 2 * T2
    t_c = timeit(chain)
    line = (f"block {blk:2d} M={M:8d} cexp={cexp:4d} cout={cout:3d} {'hs ' if act == 2 else 'relu'} | "
            f"chain {t_c * 1e3:8.1f} us {b_c / 1e9:6.3f} GB {b_c / t_c / 1e6:6.0f} GB/s")
    if takes:
        # agreement: one call of each from zeroed accumulators
        for t in (dw_c, dw_f, s2_c, s2_f):
            t.zero_()
        chain()
        fused()
        torch.cuda.synchronize()
        ok = (close(dp_f, dp_c, 2e-5) and close(dw_f, dw_c, 1e-4) and close(s2_f[0], s2_c[0], 1e-4)
              and close(s2_f[1], s2_c[1], 1e-4))
        all_ok &= ok
        t_f = timeit(fused)
        tot["chain_ms"] += t_c
        tot["fused_ms"] += t_f
        tot["chain_gb"] += b_c / 1e9
        tot["fused_gb"] += b_f / 1e9
        fused_blocks.append(blk)
        line += (f" | fused {t_f * 1e3:8.1f} us {b_f / 1e9:6.3f} GB {b_f / t_f / 1e6:6.0f} GB/s | x{t_c / t_f:4.2f} "
                 f"{'agree' if ok else 'MISMATCH'}")
    else:
        line += " | fused: shape not taken"
    print(line, flush=True)
    del dy, z3, z2, dz3, dp_c, dp_f
    torch.cuda.empty_cache()
# the stem: BatchNorm-backward apply pass + weight gradient on the stored dz0 against the weight gradient with the apply
# on load (hardswish); the BN reduce before both is not timed
F0, T0 = conv_out(128, 3, 2), conv_out(a.frames, 3, 2)
C0 = 16
g = torch.Generator(device="cuda").manual_seed(0)
x, dy, z = (torch.randn(*sh, device="cuda", generator=g) for sh in ((B, 128, a.frames), (B, F0, T0, C0), (B, F0, T0, C0)))
bn = [torch.rand(C0, device="cuda", generator=g) + 0.5, torch.randn(C0, device="cuda", generator=g) * 0.3,
      torch.randn(C0, device="cuda", generator=g) * 0.2, torch.rand(C0, device="cuda", generator=g) + 0.5]
c12 = [torch.randn(C0, device="cuda", generator=g) * 0.1 for _ in range(2)]
P0 = [t.data_ptr() for t in bn]
dz0 = torch.empty_like(z)
dw_c, dw_f = torch.zeros(C0, 9, device="cuda"), torch.zeros(C0, 9, device="cuda")
M0 = B * F0 * T0


def stem_chain():
    L.bn_bwd_apply(dy.data_ptr(), 0, 0, z.data_ptr(), *P0, 2, c12[0].data_ptr(), c12[1].data_ptr(), dz0.data_ptr(), 0, 1,
                   M0, C0, st)
    L.stem_wgrad(dz0.data_ptr(), 0, x.data_ptr(), dw_c.data_ptr(), B, 128, a.frames, C0, 2, 0, 0, 0, 0, 0, 0, 0, 0, st)


def stem_fused():
    L.stem_wgrad(dy.data_ptr(), 0, x.data_ptr(), dw_f.data_ptr(), B, 128, a.frames, C0, 2, z.data_ptr(), *P0, 2,
                 c12[0].data_ptr(), c12[1].data_ptr(), st)


dw_c.zero_()
dw_f.zero_()
stem_chain()
stem_fused()
torch.cuda.synchronize()
ok = close(dw_f, dw_c, 1e-5)
all_ok &= ok
t_c, t_f = timeit(stem_chain), timeit(stem_fused)
T0b, Xb = M0 * C0 * 4, B * 128 * a.frames * 4
b_c, b_f = 3 * T0b + (T0b + Xb), 2 * T0b + Xb
print(f"stem     M={M0:8d} C={C0} hs | apply + wgrad {t_c * 1e3:8.1f} us {b_c / 1e9:6.3f} GB {b_c / t_c / 1e6:6.0f} GB/s | "
      f"wgrad with apply on load {t_f * 1e3:8.1f} us {b_f / 1e9:6.3f} GB {b_f / t_f / 1e6:6.0f} GB/s | x{t_c / t_f:4.2f} "
      f"{'agree' if ok else 'MISMATCH'}", flush=True)
tot["stem_chain_ms"], tot["stem_fused_ms"] = t_c, t_f
print(json.dumps({"batch": B, "fused_blocks": fused_blocks, **{k_: round(v, 4) for k_, v in tot.items()},
                  "agree": all_ok, "device": torch.cuda.get_device_name()}))
sys.exit(0 if all_ok else 1)
