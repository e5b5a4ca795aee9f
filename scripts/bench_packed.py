#!/usr/bin/env python
"""Clips of different lengths in one eval batch: clips/s of three ways to run a variable-length eval set, on the H100.

    python scripts/bench_packed.py [--clips 2048] [--batch 64] [--runs 5] [--out DIR]

Workload: --clips seeded clip lengths, log-uniform from 0.3 s to 30 s (FSD50K's range, ex_fsd50k.py
--variable_eval_length), as 128-band log-mel spectrograms at 100 frames/s; mn10 and dymn10, fp32.
  (a) B = 1 per clip: the reference's variable-length eval loop;
  (b) clips sorted by length, packed into batches of <= --batch clips, each run with `lengths`;
  (c) the same batches without `lengths`: the padded forward's cost, the floor for (b).
Timing: every shape is warmed up first; a host clock around synchronised work; the median of --runs runs.
Kernels alone at mn10's block-4 shape, batches of 64 and of 7 clips of 30 s: eat_time_pad_zero and eat_mean_len with the
L2 flushed between launches, algorithmic bytes (padding written; valid region read) over CUDA-event time.
A small batch (7 clips of 3 to 30 s, the size of a last partial bucket): ms per forward with and without `lengths`,
where eat_mean_len has the fewest CTAs (one per 32 channels and clip).
Prints one JSON line with the device name, power limit and max SM clock read in the same run."""
import argparse
import contextlib
import io
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from efficientat_b200._lib import lib  # noqa: E402
from efficientat_b200.synth import synth_state_  # noqa: E402

FPS = 100                                           # frames per second: 32 kHz, hop 320


def device_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name()


def model(kind):
    if kind == "mn10":
        from efficientat_b200.models.mn.model import get_model
    else:
        from efficientat_b200.models.dymn.model import get_model
    torch.manual_seed(0)
    with contextlib.redirect_stdout(io.StringIO()):
        m = get_model(width_mult=1.0, verbose=False)
    return synth_state_(m, seed=7).cuda().eval()


def timed(fn, runs):
    out = []
    for _ in range(runs):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        out.append(time.perf_counter() - t0)
    return statistics.median(out)


def kernel_rates(B=64, T=3000):
    """eat_time_pad_zero and eat_mean_len at mn10's block-4 shapes (stride-2 stage of 30 s clips: F=32, T/4, 72 ch.) with
    half of the clips at a quarter of the length; the L2 (50 MB) is flushed between launches"""
    L, st = lib(), torch.cuda.current_stream().cuda_stream
    F, Tn, C = 32, T // 4, 72
    x = torch.randn(B, F, Tn, C, device="cuda")
    tv = [Tn if b % 2 == 0 else Tn // 4 for b in range(B)]
    t_valid = torch.tensor(tv, dtype=torch.int32, device="cuda")
    out = torch.empty(B, C, device="cuda")
    flush = torch.empty(64 << 20, dtype=torch.uint8, device="cuda")
    pad_bytes = sum(Tn - t for t in tv) * F * C * 4
    valid_bytes = sum(tv) * F * C * 4
    res = {}
    for name, fn, nbytes in (("time_pad_zero", lambda: L.time_pad_zero(x.data_ptr(), 0, B, F, Tn, C, t_valid.data_ptr(), st),
                              pad_bytes),
                             ("mean_len", lambda: L.mean_len(x.data_ptr(), 0, out.data_ptr(), B, F, Tn, C,
                                                             t_valid.data_ptr(), st), valid_bytes)):
        ms = []
        for i in range(23):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            if i >= 3:
                ms.append(e0.elapsed_time(e1))
        t = statistics.median(ms)
        res[name] = dict(ms=round(t, 4), bytes=nbytes, tb_s=round(nbytes / t / 1e9, 3))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=2048)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--nets", default="mn10,dymn10")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_packed.py measures on the GPU; no CUDA device found")
    rng = np.random.default_rng(0)
    secs = np.exp(rng.uniform(np.log(0.3), np.log(30.0), a.clips))
    frames = [max(1, int(round(s * FPS))) for s in secs]
    order = sorted(range(a.clips), key=lambda i: frames[i])
    batches = [order[i:i + a.batch] for i in range(0, a.clips, a.batch)]
    g = torch.Generator(device="cuda").manual_seed(1)
    specs = [torch.randn(1, 1, 128, t, device="cuda", generator=g) for t in frames]
    packed = []
    for idx in batches:
        T = max(frames[i] for i in idx)
        x = torch.zeros(len(idx), 1, 128, T, device="cuda")
        for j, i in enumerate(idx):
            x[j, :, :, :frames[i]] = specs[i][0]
        packed.append((x, [frames[i] for i in idx]))
    result = dict(device=device_info(), clips=a.clips, batch=a.batch, runs=a.runs, total_seconds=round(float(secs.sum()), 1))
    for kind in a.nets.split(","):
        m = model(kind)
        ways = {"b1": lambda: [m(s) for s in specs],
                "lengths": lambda: [m(x, lengths=n) for x, n in packed],
                "padded": lambda: [m(x) for x, _ in packed]}
        with torch.no_grad():
            for fn in ways.values():
                fn()                                    # warm every shape
            r = {k: a.clips / timed(fn, a.runs) for k, fn in ways.items()}
        r = {k: round(v, 1) for k, v in r.items()}
        r["lengths_over_padded"] = round(r["padded"] / r["lengths"] - 1.0, 4)
        result[kind] = r
    small = [3000, 2600, 2100, 1700, 1200, 700, 300]
    xs = torch.randn(len(small), 1, 128, max(small), device="cuda", generator=g)
    for kind in a.nets.split(","):
        m = model(kind)
        with torch.no_grad():
            for fn in (lambda: m(xs, lengths=small), lambda: m(xs)):
                fn()
            ms = {k: round(1e3 * timed(fn, a.runs), 3)
                  for k, fn in (("lengths_ms", lambda: m(xs, lengths=small)), ("padded_ms", lambda: m(xs)))}
        result[kind + "_B7_3to30s"] = ms
    result["kernels_mn10_block4_B64_30s"] = kernel_rates()
    result["kernels_mn10_block4_B7_30s"] = kernel_rates(B=7)
    line = json.dumps(result)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_packed.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
