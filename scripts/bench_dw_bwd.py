"""Per-layer benchmark of the depthwise stage's backward below its BatchNorm at the mn10 shapes of all 15 blocks (fp32):
the four separate passes (BN2-backward apply, depthwise weight gradient, data gradient, expand-BatchNorm reduce) against
eat_dw_conv_bwd_fused, L2 flushed before every timed call.  Prints algorithmic bytes and GB/s of both and checks that
they agree (din 2e-5, dW 1e-4 of the tensor's max, BN1 sums 1e-4 relative); one JSON summary line at the end."""
import argparse
import contextlib
import io
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from efficientat_b200._lib import lib  # noqa: E402
from efficientat_b200.models.mn.model import get_model  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=256)
ap.add_argument("--frames", type=int, default=1001, help="spectrogram frames (10 s at 32 kHz, hop 320)")
ap.add_argument("--reps", type=int, default=5)
a = ap.parse_args()


def conv_out(n, k, s):
    return (n + 2 * ((k - 1) // 2) - k) // s + 1


def layers():
    """(F, T, C, k, stride, act, se, expand) of each block's depthwise input, mn10 with a 128-bin spectrogram"""
    with contextlib.redirect_stdout(io.StringIO()):
        model = get_model(width_mult=1.0, verbose=False)
    feats = list(model.features)
    F, T = conv_out(128, 3, 2), conv_out(a.frames, 3, 2)
    out = []
    for m in feats[1:-1]:
        c = m.cnf
        out.append((F, T, c.expanded_channels, c.kernel, c.stride, 2 if c.use_hs else 1, bool(c.use_se),
                    c.expanded_channels != c.input_channels))
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
all_ok = True
for li, (F, T, C, k, s, act, se, expand) in enumerate(layers()):
    Fo, To = conv_out(F, k, s), conv_out(T, k, s)
    g = torch.Generator(device="cuda").manual_seed(li)
    r = lambda *sh: torch.randn(*sh, device="cuda", generator=g)
    u = lambda *sh: torch.rand(*sh, device="cuda", generator=g)
    x, dp, z2 = r(B, F, T, C), r(B, Fo, To, C), r(B, Fo, To, C)
    w = r(C, 1, k, k) * 0.3
    wt = torch.empty(k * k, C, device="cuda")
    L.dw_repack(w.data_ptr(), wt.data_ptr(), C, k, st)
    bn2 = [u(C) + 0.5, r(C) * 0.3, r(C) * 0.2, u(C) + 0.5]            # scale, shift, mean, invstd
    c12 = [r(C) * 0.1, r(C) * 0.1]
    gate, dpool = (u(B, C), r(B, C) * 0.1) if se else (None, None)
    bn1 = [u(C) + 0.5, r(C) * 0.3, r(C) * 0.2, u(C) + 0.5] if expand else [None] * 4
    res = None if expand else r(B, F, T, C)
    xact = act if expand else 0
    dz = torch.empty_like(z2)
    din_c, din_f = torch.empty_like(x), torch.empty_like(x)
    dw_c, dw_f = torch.zeros_like(w), torch.zeros_like(w)
    s_c = torch.zeros(2, C, device="cuda", dtype=torch.float64)
    s_f = torch.zeros(2, C, device="cuda", dtype=torch.float64)

    def chain():
        L.bn_bwd_apply(dp.data_ptr(), p(gate), p(dpool), z2.data_ptr(), *[t.data_ptr() for t in bn2], act,
                       c12[0].data_ptr(), c12[1].data_ptr(), dz.data_ptr(), 0, B, Fo * To, C, st)
        L.dw_conv_wgrad(dz.data_ptr(), x.data_ptr(), p(bn1[0]), p(bn1[1]), xact, dw_c.data_ptr(), 0, 0, B, F, T, C, k, s, st)
        L.dw_conv_dgrad(dz.data_ptr(), wt.data_ptr(), 0, p(res), din_c.data_ptr(), 0, B, F, T, C, k, s, st)
        if expand:
            L.bn_bwd_reduce(din_c.data_ptr(), 0, 0, x.data_ptr(), *[t.data_ptr() for t in bn1], act, 0, B, F * T, C,
                            s_c[0].data_ptr(), s_c[1].data_ptr(), st)

    def fused():
        L.dw_conv_bwd_fused(dp.data_ptr(), p(gate), p(dpool), z2.data_ptr(), *[t.data_ptr() for t in bn2], act,
                            c12[0].data_ptr(), c12[1].data_ptr(), wt.data_ptr(), x.data_ptr(), p(bn1[0]), p(bn1[1]), xact,
                            p(res), din_f.data_ptr(), dw_f.data_ptr(), p(bn1[2]), p(bn1[3]),
                            s_f[0].data_ptr() if expand else 0, s_f[1].data_ptr() if expand else 0, 0, B, F, T, C, k, s, st)

    # agreement: one call of each from zeroed accumulators
    chain()
    fused()
    torch.cuda.synchronize()
    ok = close(din_f, din_c, 2e-5) and close(dw_f, dw_c, 1e-4) and (not expand or close(s_f, s_c, 1e-4))
    all_ok &= ok
    t_c, t_f = timeit(chain), timeit(fused)
    # algorithmic bytes (fp32 elements of the tensors each pass must read or write)
    T1, T2 = B * F * T * C * 4, B * Fo * To * C * 4
    b_c = 3 * T2 + (T2 + T1) + (T2 + T1 + (T1 if res is not None else 0)) + (2 * T1 if expand else 0)
    b_f = 2 * T2 + 2 * T1 + (T1 if res is not None else 0)
    tot["chain_ms"] += t_c
    tot["fused_ms"] += t_f
    tot["chain_gb"] += b_c / 1e9
    tot["fused_gb"] += b_f / 1e9
    print(f"block {li + 1:2d} F={F:3d} T={T:4d} C={C:4d} k={k} s={s} {'hs ' if act == 2 else 'relu'} se={int(se)} "
          f"exp={int(expand)} | chain {t_c * 1e3:8.1f} us {b_c / 1e9:6.3f} GB {b_c / t_c / 1e6:6.0f} GB/s | "
          f"fused {t_f * 1e3:8.1f} us {b_f / 1e9:6.3f} GB {b_f / t_f / 1e6:6.0f} GB/s | x{t_c / t_f:4.2f} "
          f"{'agree' if ok else 'MISMATCH'}", flush=True)
print(json.dumps({"batch": B, **{k_: round(v, 4) for k_, v in tot.items()}, "agree": all_ok,
                  "device": torch.cuda.get_device_name()}))
sys.exit(0 if all_ok else 1)
