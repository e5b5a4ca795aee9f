"""Dilated depthwise kernels (eat_dw_conv_*_dil) against the undilated 5x5 stride-1 launches on the same tensors, and
whole AudioSetTrainer steps of mn10 with and without get_model(dilated=True).

    python scripts/bench_dw_dilated.py [--batch 256] [--rounds 7] [--steps 10] [--out gpu_out/dw_dilated.json]

Kernels: the mn10 10 s tail shapes ([B, 8, 63, 672] and [B, 8, 63, 960], k = 5), each launch timed with CUDA events
with the L2 flushed before it; the dilated and the undilated launch alternate round by round and the median is
reported.  Both move the same algorithmic bytes: input + output (+ residual for the data gradient) for the forward and
data gradient, dz + input for the weight gradient.  Trainer steps: eager AudioSetTrainer steps on 10 s clips, the two
models alternating step by step in one process.  Prints the card, its power limit and maximum SM clock."""
import argparse
import contextlib
import io
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from efficientat_b200._lib import lib  # noqa: E402

HBM = 3.35e12       # H100 SXM data-sheet HBM3 bandwidth, bytes/s
SHAPES = [(8, 63, 672), (8, 63, 960)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    return q or torch.cuda.get_device_name()


def kernels(B, rounds, L, st):
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")

    def one(fn):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1e-3

    rows = []
    for F, T, C in SHAPES:
        k = 5
        x = torch.randn(B, F, T, C, device="cuda")
        w = torch.randn(C, 1, k, k, device="cuda") * 0.2
        wt = torch.empty(k * k, C, device="cuda")
        L.dw_repack(w.data_ptr(), wt.data_ptr(), C, k, st)
        out, din, res = torch.empty_like(x), torch.empty_like(x), torch.randn_like(x)
        dz = torch.randn_like(x)
        sc = torch.rand(2, C, device="cuda")
        stats = torch.zeros(2, C, device="cuda", dtype=torch.float64)
        pool = torch.zeros(B, C, device="cuda")
        dw = torch.zeros(C, 1, k, k, device="cuda")
        p = lambda t: t.data_ptr()       # noqa: E731
        el = B * F * T * C * 4
        launches = {
            "train_fwd": (el * 2,
                          lambda: L.dw_conv_fwd_dil(p(x), p(wt), p(out), 0, B, F, T, C, k, 1, 2, p(sc[0]), p(sc[1]), 2, 0, 0, 0,
                                                    0, p(stats[0]), p(stats[1]), st),
                          lambda: L.dw_conv_fwd(p(x), p(wt), p(out), 0, B, F, T, C, k, 1, p(sc[0]), p(sc[1]), 2, 0, 0, 0, 0,
                                                p(stats[0]), p(stats[1]), st)),
            "eval": (el * 2,
                     lambda: L.dw_conv_fwd_dil(p(x), p(wt), p(out), 0, B, F, T, C, k, 1, 2, 0, 0, 0, p(sc[0]), p(sc[1]), 2,
                                               p(pool), 0, 0, st),
                     lambda: L.dw_conv_fwd(p(x), p(wt), p(out), 0, B, F, T, C, k, 1, 0, 0, 0, p(sc[0]), p(sc[1]), 2, p(pool),
                                           0, 0, st)),
            "dgrad_res": (el * 3,
                          lambda: L.dw_conv_dgrad_dil(p(dz), p(wt), p(res), p(din), 0, B, F, T, C, k, 1, 2, st),
                          lambda: L.dw_conv_dgrad(p(dz), p(wt), 0, p(res), p(din), 0, B, F, T, C, k, 1, st)),
            "wgrad": (el * 2,
                      lambda: L.dw_conv_wgrad_dil(p(dz), p(x), p(sc[0]), p(sc[1]), 2, p(dw), 0, B, F, T, C, k, 1, 2, st),
                      lambda: L.dw_conv_wgrad(p(dz), p(x), p(sc[0]), p(sc[1]), 2, p(dw), 0, 0, B, F, T, C, k, 1, st)),
        }
        for name, (nbytes, dil, und) in launches.items():
            dil(), und()                                    # warm-up: module load, shared-memory opt-in
            td, tu = [], []
            for _ in range(rounds):
                td.append(one(dil))
                tu.append(one(und))
            md, mu = sorted(td)[rounds // 2], sorted(tu)[rounds // 2]
            r = dict(shape=[B, F, T, C], launch=name, bytes=nbytes, dilated_us=md * 1e6, undilated_us=mu * 1e6,
                     dilated_GBs=nbytes / md / 1e9, hbm_share=nbytes / md / HBM, ratio=md / mu)
            rows.append(r)
            print(f"[{B},{F},{T},{C}] {name:9s} dilated {md * 1e6:8.1f} us {nbytes / md / 1e9:7.0f} GB/s "
                  f"({100 * nbytes / md / HBM:4.1f} % of 3.35 TB/s) | undilated 5x5 s1 {mu * 1e6:8.1f} us | "
                  f"ratio {md / mu:.2f}", flush=True)
    return rows


def steps(B, n, warm):
    from efficientat_b200.models.mn.model import get_model
    from efficientat_b200.models.preprocess import AugmentMelSTFT
    from efficientat_b200.synth import synth_labels, synth_waveform
    from efficientat_b200.train import AudioSetTrainer
    tr = {}
    for dil in (False, True):
        with contextlib.redirect_stdout(io.StringIO()):
            model = get_model(width_mult=1.0, dilated=dil, verbose=False).cuda()
            mel = AugmentMelSTFT(freqm=0, timem=0).cuda()
        tr[dil] = AudioSetTrainer(model, mel, lr=1e-4, kd_lambda=0.0, mixup_alpha=0.3)
    wave = synth_waveform(B, 320000, seed=1).cuda()
    y = synth_labels(B, 527, seed=2).cuda()
    perm, lam = torch.randperm(B), torch.full((B,), 0.7)
    times = {False: [], True: []}
    for i in range(warm + n):
        for dil in (False, True):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            tr[dil].step(wave, y, None, perm=perm, lam=lam)
            e1.record()
            torch.cuda.synchronize()
            if i >= warm:
                times[dil].append(e0.elapsed_time(e1))
    med = {d: sorted(t)[len(t) // 2] for d, t in times.items()}
    print(f"mn10 AudioSetTrainer step, B={B}, 10 s clips: undilated {med[False]:.2f} ms, dilated {med[True]:.2f} ms "
          f"(x{med[True] / med[False]:.3f})", flush=True)
    return dict(batch=B, undilated_ms=med[False], dilated_ms=med[True])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--step-batch", type=int, default=256)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_dw_dilated.py measures on a CUDA device; none is visible")
    dev = card()
    print("device:", dev, flush=True)
    L, st = lib(), torch.cuda.current_stream().cuda_stream
    res = dict(device=dev, kernels=kernels(a.batch, a.rounds, L, st))
    if a.steps > 0:
        res["trainer"] = steps(a.step_batch, a.steps, a.warmup)
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
