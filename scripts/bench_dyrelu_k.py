"""DyReLU-B with M = 1..4 linear pieces (get_model(dyrelu_k=M)) against M = 2: the launches that take M, and whole
AudioSetTrainer steps of dymn10 on 10 s clips.

    python scripts/bench_dyrelu_k.py [--batch 128] [--rounds 7] [--steps 5] [--baseline-lib PATH]
                                     [--out gpu_out/dyrelu_k.json]

Launches, fp32 storage, on three dymn10 10 s layer shapes: the eval depthwise conv with the DyReLU-B + CoordAtt epilogue
(eat_dw_conv_fwd_dy_m; the 5x5 layer runs in the tile kernel), and the training-path DyReLU-B * CoordAtt forward and
backward (eat_dy_act_fwd_m / eat_dy_act_bwd_m).  M = 2 goes through the same entry points.  Each launch is timed with
CUDA events with the L2 flushed before it; M and M = 2 alternate round by round and the median is reported.  With
--baseline-lib (another build of libeat_b200.so, for instance an earlier commit's) each launch alternates with the same
launch and M of that build instead, and the outputs of the two builds are compared: bit for bit, except d(ca_f) and the
coefficient gradients, which the backward sums with atomics in no fixed order (relative difference reported).
Algorithmic bytes come from the shapes: every tensor the launch must read or write once (activations, per-sample
coefficient and attention tensors, gradients).  Trainer steps: eager AudioSetTrainer steps, the
four models alternating step by step in one process.  Prints the card, its power limit and maximum SM clock."""
import argparse
import contextlib
import io
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import efficientat_b200._lib as _lib  # noqa: E402
from efficientat_b200._lib import lib  # noqa: E402

HBM = 3.35e12       # H100 SXM data-sheet HBM3 bandwidth, bytes/s
# (F, T, C, k, stride) of the depthwise input: three dymn10 layers of a 10 s clip (1000 frames)
SHAPES = [(32, 250, 72, 3, 1), (16, 125, 120, 5, 1), (8, 63, 480, 3, 1)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    return q or torch.cuda.get_device_name()


def load(path):
    """The C ABI of another build of the library, bound like lib()."""
    saved, _lib.LIB_PATH = _lib.LIB_PATH, path
    try:
        return _lib._Lib()
    finally:
        _lib.LIB_PATH = saved


def kernels(B, rounds, L, st, L0=None):
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")

    def one(fn):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1e-3

    p = lambda t: t.data_ptr()       # noqa: E731
    rows = []
    for F, T, C, k, s in SHAPES:
        Fo, To = (F - 1) // s + 1, (T - 1) // s + 1
        kk = k * k
        x = torch.randn(B, F, T, C, device="cuda")
        wt = torch.randn(B, kk, C, device="cuda") / k
        z, dp = torch.randn(B, Fo, To, C, device="cuda"), torch.randn(B, Fo, To, C, device="cuda")
        sc = torch.rand(2, C, device="cuda") + 0.5
        ca_f, ca_t = torch.rand(B, Fo, C, device="cuda"), torch.rand(B, To, C, device="cuda")
        act = B * Fo * To * C * 4
        att = (B * Fo * C + B * To * C) * 4

        def make(M, lib_):
            theta, lam, init = coef[M]
            out, du = torch.empty_like(z), torch.empty_like(z)
            dcaf, dcat = torch.zeros(B, Fo, C, device="cuda"), torch.empty(B, To, C, device="cuda")
            dcoef = torch.zeros(B, C, 2 * M, device="cuda")
            P = (p(sc[0]), p(sc[1]), p(theta), p(lam), p(init), p(ca_f), p(ca_t))
            th = B * C * 2 * M * 4
            return {
                "dw_eval": (x.numel() * 4 + act + th + att + B * kk * C * 4,
                            lambda: lib_.dw_conv_fwd_dy_m(p(x), p(wt), kk * C, p(out), 0, B, F, T, C, k, s, 0, 0, 0, *P, M,
                                                          0, 0, st), dict(out=out)),
                "act_fwd": (2 * act + th + att, lambda: lib_.dy_act_fwd_m(p(z), p(out), 0, *P, M, B, Fo, To, C, st),
                            dict(out=out)),
                "act_bwd": (3 * act + th + 2 * att + 2 * th,
                            lambda: lib_.dy_act_bwd_m(p(dp), p(z), p(du), 0, *P, p(dcaf), p(dcat), p(dcoef), M, B, Fo, To,
                                                      C, st), dict(du=du, dcat=dcat, dcaf=dcaf, dcoef=dcoef)),
            }
        # the launches take raw pointers: theta, lam and init live as long as the shape's launches
        coef = {M: (torch.rand(B, C, 2 * M, device="cuda"), torch.tensor([1.0] * M + [0.5] * M, device="cuda"),
                    torch.tensor([1.0] + [0.0] * (2 * M - 1), device="cuda")) for M in (1, 2, 3, 4)}
        base = make(2, L)
        for M in (1, 3, 4, 2):
            cur = make(M, L)
            if L0 is not None:
                base = make(M, L0)
            for name, (nbytes, fn, outs) in cur.items():
                nb2, fn2, outs2 = base[name]
                fn(), fn2()                                   # warm-up: module load, shared-memory opt-in
                same = {}
                if L0 is not None:                            # one more launch each from zeroed accumulators
                    for t in [*outs.values(), *outs2.values()]:
                        t.zero_()
                    fn(), fn2()
                    torch.cuda.synchronize()
                    for key, t in outs.items():
                        t2 = outs2[key]
                        same[key] = (bool(torch.equal(t, t2)) if key not in ("dcaf", "dcoef") else
                                     ((t - t2).abs().max() / t2.abs().max().clamp_min(1e-30)).item())
                tm, t2 = [], []
                for _ in range(rounds):
                    tm.append(one(fn))
                    t2.append(one(fn2))
                mm, m2 = sorted(tm)[rounds // 2], sorted(t2)[rounds // 2]
                other = "M=2" if L0 is None else "baseline"
                r = dict(shape=[B, F, T, C], k=k, stride=s, pieces=M, launch=name, bytes=nbytes, us=mm * 1e6,
                         GBs=nbytes / mm / 1e9, hbm_share=nbytes / mm / HBM, ratio=mm / m2)
                r["m2_us" if L0 is None else "baseline_us"] = m2 * 1e6
                r["m2_GBs" if L0 is None else "baseline_GBs"] = nb2 / m2 / 1e9
                if L0 is not None:
                    r["vs_baseline"] = same
                rows.append(r)
                print(f"[{B},{F},{T},{C}] k{k} s{s} {name:8s} M={M} {mm * 1e6:8.1f} us {nbytes / mm / 1e9:6.0f} GB/s "
                      f"({100 * nbytes / mm / HBM:4.1f} % of 3.35 TB/s) | {other} {m2 * 1e6:8.1f} us | ratio {mm / m2:.2f}"
                      + (f" | {same}" if same else ""), flush=True)
    return rows


def steps(B, n, warm):
    from efficientat_b200.models.dymn.model import get_model
    from efficientat_b200.models.preprocess import AugmentMelSTFT
    from efficientat_b200.synth import synth_labels, synth_waveform
    from efficientat_b200.train import AudioSetTrainer
    tr = {}
    for M in (2, 1, 3, 4):
        with contextlib.redirect_stdout(io.StringIO()):
            model = get_model(width_mult=1.0, dyrelu_k=M, verbose=False).cuda()
            mel = AugmentMelSTFT(freqm=0, timem=0).cuda()
        tr[M] = AudioSetTrainer(model, mel, lr=1e-4, kd_lambda=0.0, mixup_alpha=0.3)
    wave = synth_waveform(B, 320000, seed=1).cuda()
    y = synth_labels(B, 527, seed=2).cuda()
    perm, lam = torch.randperm(B), torch.full((B,), 0.7)
    times = {M: [] for M in tr}
    for i in range(warm + n):
        for M in tr:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            tr[M].step(wave, y, None, perm=perm, lam=lam)
            e1.record()
            torch.cuda.synchronize()
            if i >= warm:
                times[M].append(e0.elapsed_time(e1))
    med = {M: sorted(t)[len(t) // 2] for M, t in times.items()}
    print(f"dymn10 AudioSetTrainer step, B={B}, 10 s clips: " +
          ", ".join(f"M={M} {med[M]:.2f} ms (x{med[M] / med[2]:.3f})" for M in sorted(med)), flush=True)
    return dict(batch=B, step_ms={str(M): med[M] for M in sorted(med)})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--baseline-lib", default=None, help="another libeat_b200.so to alternate with and compare against")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_dyrelu_k.py measures on a CUDA device; none is visible")
    dev = card()
    print("device:", dev, flush=True)
    L, st = lib(), torch.cuda.current_stream().cuda_stream
    L0 = load(os.path.abspath(a.baseline_lib)) if a.baseline_lib else None
    res = dict(device=dev, kernels=kernels(a.batch, a.rounds, L, st, L0))
    if a.steps > 0:
        res["trainer"] = steps(a.batch, a.steps, a.warmup)
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
