"""Per-layer benchmark of the expand stage's backward below its BatchNorm at the mn10 shapes of every block with an expand
stage (fp32): the three passes (BN1-backward apply, weight-gradient GEMM, data-gradient GEMM with the residual) against
eat_pw_conv_bwd_fused, L2 flushed before every timed call.  Prints algorithmic bytes and GB/s of both and checks that they
agree (dX 2e-5, dW 1e-4 of the tensor's max); blocks the fused kernel does not take print the three passes only.  One JSON
summary line at the end."""
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
ap.add_argument("--frames", type=int, default=1000, help="spectrogram frames (the bench's clip length)")
ap.add_argument("--reps", type=int, default=5)
a = ap.parse_args()


def conv_out(n, k, s):
    return (n + 2 * ((k - 1) // 2) - k) // s + 1


def layers():
    """(block, rows per sample, cexp, cin, act, residual) of each expand stage, mn10 with a 128-bin spectrogram"""
    with contextlib.redirect_stdout(io.StringIO()):
        model = get_model(width_mult=1.0, verbose=False)
    F, T = conv_out(128, 3, 2), conv_out(a.frames, 3, 2)
    out = []
    for i, m in enumerate(list(model.features)[1:-1]):
        c = m.cnf
        if c.expanded_channels != c.input_channels:
            out.append((i + 1, F * T, c.expanded_channels, c.input_channels, 2 if c.use_hs else 1, bool(m.use_res_connect)))
        F, T = conv_out(F, c.kernel, c.stride), conv_out(T, c.kernel, c.stride)
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


def p(t):
    return 0 if t is None else t.data_ptr()


def close(x, y, tol):
    return (x.double() - y.double()).abs().max().item() <= tol * y.double().abs().max().item() + 1e-12


B = a.batch
tot = {"chain_ms": 0.0, "fused_ms": 0.0, "chain_gb": 0.0, "fused_gb": 0.0}
fused_blocks = []
all_ok = True
plan = (ctypes.c_int * 4)()
for blk, P, cexp, cin, act, has_res in layers():
    M = B * P
    try:
        L.pw_bwd_plan(M, cexp, cin, ctypes.addressof(plan))
        takes = True
    except EatError:
        takes = False
    g = torch.Generator(device="cuda").manual_seed(blk)
    r = lambda *sh: torch.randn(*sh, device="cuda", generator=g)
    u = lambda *sh: torch.rand(*sh, device="cuda", generator=g)
    da, z, x = r(M, cexp), r(M, cexp), r(M, cin)
    w = r(cexp, cin) / cexp ** 0.5
    bn = [u(cexp) + 0.5, r(cexp) * 0.3, r(cexp) * 0.2, u(cexp) + 0.5]      # scale, shift, mean, invstd
    c12 = [r(cexp) * 0.1, r(cexp) * 0.1]
    res = r(M, cin) if has_res else None
    dz = torch.empty_like(z)
    dx_c, dx_f = torch.empty(M, cin, device="cuda"), torch.empty(M, cin, device="cuda")
    dw_c, dw_f = torch.zeros(cexp, cin, device="cuda"), torch.zeros(cexp, cin, device="cuda")
    ws = torch.empty(cin * ((cexp + 31) // 32) * 128, device="cuda", dtype=torch.uint8)

    def chain():
        L.bn_bwd_apply(da.data_ptr(), 0, 0, z.data_ptr(), *[t.data_ptr() for t in bn], act, c12[0].data_ptr(),
                       c12[1].data_ptr(), dz.data_ptr(), 0, 1, M, cexp, st)
        L.pw_tc_wgrad(dz.data_ptr(), 0, x.data_ptr(), 0, dw_c.data_ptr(), 0, M, cexp, cin, 0, 0, 0, 0, 1, st)
        L.pw_tma_fwd(dz.data_ptr(), w.data_ptr(), 1, dx_c.data_ptr(), M, cin, cexp, 0, 0, 0, 0, 1, 0, 0, 0, p(res), 0, 0,
                     ws.data_ptr(), ws.numel(), st)

    def fused():
        L.pw_conv_bwd_fused(da.data_ptr(), z.data_ptr(), *[t.data_ptr() for t in bn], act, c12[0].data_ptr(),
                            c12[1].data_ptr(), x.data_ptr(), w.data_ptr(), p(res), dx_f.data_ptr(), dw_f.data_ptr(), 0, M,
                            cexp, cin, st)

    # algorithmic bytes (fp32 elements of the tensors each pass must read or write)
    T1, Tin = M * cexp * 4, M * cin * 4
    b_c = 3 * T1 + (T1 + Tin) + (T1 + Tin + (Tin if has_res else 0))
    b_f = 2 * T1 + 2 * Tin + (Tin if has_res else 0)
    t_c = timeit(chain)
    line = (f"block {blk:2d} M={M:8d} cexp={cexp:4d} cin={cin:3d} {'hs ' if act == 2 else 'relu'} res={int(has_res)} | "
            f"chain {t_c * 1e3:8.1f} us {b_c / 1e9:6.3f} GB {b_c / t_c / 1e6:6.0f} GB/s")
    if takes:
        # agreement: one call of each from zeroed accumulators
        dw_c.zero_()
        chain()
        fused()
        torch.cuda.synchronize()
        ok = close(dx_f, dx_c, 2e-5) and close(dw_f, dw_c, 1e-4)
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
    del da, z, x, res, dz, dx_c, dx_f
    torch.cuda.empty_cache()
print(json.dumps({"batch": B, "fused_blocks": fused_blocks, **{k_: round(v, 4) for k_, v in tot.items()},
                  "agree": all_ok, "device": torch.cuda.get_device_name()}))
sys.exit(0 if all_ok else 1)
