"""Benchmark of the waveform augmentation (gain, roll, waveform mixing; efficientat_b200/augment.py, csrc/wave_aug.cu).

1. `eat_wave_aug` at B = 256 x 10 s and B = 32 x 5 s (32 kHz) from a batch source, every row mixed and every row
   unmixed, and `eat_clip_sum` over the same batch: CUDA events over --steps launches after --warmup, median of
   --rounds.  Algorithmic bytes: a mixed row reads two source rows and writes one, 12 N bytes; an unmixed row 8 N;
   the sum reads 4 N per clip.  Set against the 3.35 TB/s HBM3 figure of NVIDIA's H100 SXM data sheet.
2. `FineTuneTrainer(loss="ce", mixup_alpha=0.3, cuda_graph=True)` at the ESC-50 shape (mn10, 5 s, 50 classes, B = 32
   and 256) with a resident store of 1 600 clips and `WaveAugment("esc50", gain_augment=12, roll=True, wavmix=True)`,
   against the same trainer fed an un-augmented batch, alternating --trials times, CUDA events; medians.  The step with
   augmentation includes its host draw.
3. The host draw, `WaveAugment.draw`, per step at B = 32 and 256 (host clock, median of --rounds).

The card's name, power limit and maximum SM clock are read in the same call.  One JSON line per result."""
import argparse
import contextlib
import io
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from efficientat_b200._lib import lib  # noqa: E402
from efficientat_b200.augment import WaveAugment  # noqa: E402
from efficientat_b200.finetune import FineTuneTrainer  # noqa: E402
from efficientat_b200.models.mn.model import get_model  # noqa: E402
from efficientat_b200.models.preprocess import AugmentMelSTFT  # noqa: E402
from efficientat_b200.synth import synth_state_  # noqa: E402

HBM = 3.35e12

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=20, help="timed launches / steps per round")
ap.add_argument("--warmup", type=int, default=3)
ap.add_argument("--rounds", type=int, default=5)
ap.add_argument("--trials", type=int, default=3)
ap.add_argument("--store-clips", type=int, default=1600)
a = ap.parse_args()


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                            "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        name, power, clock = (s.strip() for s in q.stdout.strip().split(","))
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:                                       # the numbers still stand; say what is missing
        return {"gpu": torch.cuda.get_device_name(), "power_limit": f"not read ({type(e).__name__})",
                "max_sm_clock": "not read"}


def emit(d):
    print(json.dumps(d), flush=True)


def timed(fn, n):
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(n):
        fn()
    t1.record()
    t1.synchronize()
    return t0.elapsed_time(t1) / n


def kernels(info):
    L, st = lib(), torch.cuda.current_stream().cuda_stream
    for B, seconds in ((256, 10.0), (32, 5.0)):
        N = int(seconds * 32000)
        src = torch.randn(B, N, device="cuda") * 0.1
        out = torch.empty_like(src)
        sums = torch.empty(B, device="cuda", dtype=torch.float64)
        g = torch.Generator().manual_seed(0)
        idx1 = torch.arange(B, dtype=torch.int32)
        shifts = torch.randint(-4000, 4001, (2, B), generator=g, dtype=torch.int32).cuda()
        gains = torch.full((2, B), 0.7).cuda()
        lam = (torch.rand(B, generator=g) * 0.5 + 0.5).cuda()
        L.clip_sum(src.data_ptr(), B, N, sums.data_ptr(), st)
        for mode in ("mixed", "unmixed"):
            idx2 = torch.randperm(B, generator=g).int() if mode == "mixed" else torch.full((B,), -1, dtype=torch.int32)
            i1, i2 = idx1.cuda(), idx2.cuda()

            def run():
                L.wave_aug(src.data_ptr(), sums.data_ptr(), B, N, i1.data_ptr(), i2.data_ptr(), shifts[0].data_ptr(),
                           shifts[1].data_ptr(), gains[0].data_ptr(), gains[1].data_ptr(), lam.data_ptr(),
                           out.data_ptr(), B, st)
            timed(run, a.warmup)
            ms = statistics.median(timed(run, a.steps) for _ in range(a.rounds))
            nbytes = (12 if mode == "mixed" else 8) * B * N
            emit({"bench": "wave_aug", "rows": mode, "B": B, "seconds": seconds, "kernel_us": round(ms * 1e3, 2),
                  "GB_s": round(nbytes / (ms * 1e-3) / 1e9, 1), "share_of_3.35TB_s": round(nbytes / (ms * 1e-3) / HBM, 3),
                  **info})

        def csum():
            L.clip_sum(src.data_ptr(), B, N, sums.data_ptr(), st)
        timed(csum, a.warmup)
        ms = statistics.median(timed(csum, a.steps) for _ in range(a.rounds))
        emit({"bench": "clip_sum", "B": B, "seconds": seconds, "kernel_us": round(ms * 1e3, 2),
              "GB_s": round(4 * B * N / (ms * 1e-3) / 1e9, 1), **info})
        del src, out
        torch.cuda.empty_cache()


def steps(info):
    N, C = 5 * 32000, 50
    gs = torch.Generator().manual_seed(1)
    S = a.store_clips
    store = (torch.randn(S, N, generator=gs) * 0.1).cuda()
    labels = F.one_hot(torch.arange(S) % C, C).float().cuda()
    aug = WaveAugment("esc50", gain_augment=12, roll=True, wavmix=True, source=store, labels=labels)
    for B in (32, 256):
        def build(augment):
            with contextlib.redirect_stdout(io.StringIO()):
                model = synth_state_(get_model(width_mult=1.0, num_classes=C, verbose=False), seed=3).cuda()
                mel = AugmentMelSTFT(freqm=0, timem=0).cuda()
            return FineTuneTrainer(model, mel, loss="ce", lr=6e-5, mixup_alpha=0.3, cuda_graph=True, augment=augment)
        tr_aug, tr_plain = build(aug), build(None)
        idx = torch.randperm(S, generator=gs)[:B]
        wave, y = store[idx.cuda()], labels[idx.cuda()]

        def with_aug():
            tr_aug.step(idx, None)

        def without():
            tr_plain.step(wave, y)
        timed(with_aug, a.warmup)
        timed(without, a.warmup)
        t_a, t_p = [], []
        for _ in range(a.trials):
            t_a.append(timed(with_aug, a.steps))
            t_p.append(timed(without, a.steps))
        emit({"bench": "finetune_step_wave_aug", "model": "mn10", "B": B, "seconds": 5.0, "store_clips": S,
              "with_augment_ms": round(statistics.median(t_a), 3), "without_ms": round(statistics.median(t_p), 3),
              "trials_with_ms": [round(t, 3) for t in t_a], "trials_without_ms": [round(t, 3) for t in t_p], **info})
        del tr_aug, tr_plain
        torch.cuda.empty_cache()


def host_draw(info):
    aug = WaveAugment("esc50", gain_augment=12, roll=True, wavmix=True)
    for B in (32, 256):
        ts = []
        for _ in range(a.rounds):
            t0 = time.perf_counter()
            aug.draw(np.arange(B), 1600)
            ts.append((time.perf_counter() - t0) * 1e3)
        emit({"bench": "wave_aug_host_draw", "B": B, "ms_per_step": round(statistics.median(ts), 3), **info})


def main():
    if not torch.cuda.is_available():
        raise SystemExit("bench_wave_aug.py measures on a CUDA device; none is available")
    info = card()
    kernels(info)
    host_draw(info)
    steps(info)


if __name__ == "__main__":
    main()
