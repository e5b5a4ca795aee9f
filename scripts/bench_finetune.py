"""Benchmark of the fine-tuning step at the ESC-50 shape: mn10, 5 s clips at 32 kHz (500 frames, 128 mels), 50 classes,
B = 64 and 256.

1. `FineTuneTrainer(loss="ce", cuda_graph=True)` steps (mel, mixup, captured forward + CE + backward, Adam) against the
   loop body of ex_esc50.py:98-126 on the same model class: mixup as tensor arithmetic, `model(x)` through the autograd
   Function, F.cross_entropy, loss.backward(), torch.optim.Adam, and the `.cpu()` read of the loss every step.  Both
   timed with CUDA events around --steps steps after --warmup, alternating the two --trials times; medians reported.
2. `eat_mixstyle` on [B, 1, 128, 500]: CUDA events over --steps launches, median of --rounds.  Algorithmic bytes: the
   statistics launch reads x once (its second pass over each row is served by L1/L2) and writes 8 bytes per row; the
   apply launch reads x and the statistics and writes out: 3 * 4 * B*F*T + 16 * B*F.  Set against the 3.35 TB/s HBM3
   figure of NVIDIA's H100 SXM data sheet.

The card's name, power limit and maximum SM clock are read in the same call.  One JSON line per result."""
import argparse
import contextlib
import io
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from efficientat_b200._lib import lib  # noqa: E402
from efficientat_b200.finetune import FineTuneTrainer  # noqa: E402
from efficientat_b200.helpers.utils import mixup  # noqa: E402
from efficientat_b200.models.mn.model import get_model  # noqa: E402
from efficientat_b200.models.preprocess import AugmentMelSTFT  # noqa: E402
from efficientat_b200.synth import synth_state_, synth_waveform  # noqa: E402

HBM = 3.35e12

ap = argparse.ArgumentParser()
ap.add_argument("--batches", type=int, nargs="+", default=[64, 256])
ap.add_argument("--seconds", type=float, default=5.0)
ap.add_argument("--classes", type=int, default=50)
ap.add_argument("--steps", type=int, default=10, help="timed steps / launches per trial")
ap.add_argument("--warmup", type=int, default=3)
ap.add_argument("--trials", type=int, default=3)
ap.add_argument("--rounds", type=int, default=5)
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


def build(B):
    with contextlib.redirect_stdout(io.StringIO()):
        model = synth_state_(get_model(width_mult=1.0, num_classes=a.classes, verbose=False), seed=3).cuda()
        mel = AugmentMelSTFT(freqm=0, timem=0).cuda()
    return model, mel


def timed(fn, n):
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(n):
        fn()
    t1.record()
    t1.synchronize()
    return t0.elapsed_time(t1) / n


def main():
    if not torch.cuda.is_available():
        raise SystemExit("bench_finetune.py measures on a CUDA device; none is available")
    info = card()
    n_samples = int(a.seconds * 32000)
    for B in a.batches:
        wave = synth_waveform(B, n_samples, seed=5).cuda()
        y = F.one_hot(torch.arange(B) % a.classes, a.classes).float().cuda()

        model, mel = build(B)
        tr = FineTuneTrainer(model, mel, loss="ce", lr=6e-5, mixup_alpha=0.3, cuda_graph=True)

        def ours():
            tr.step(wave, y)

        ref_model, ref_mel = build(B)
        ref_model.train(); ref_mel.train()
        opt = torch.optim.Adam(ref_model.parameters(), lr=6e-5)

        def script():                                             # ex_esc50.py:98-126
            x = ref_mel(wave).unsqueeze(1)
            rn, lam = mixup(B, 0.3)
            lam = lam.to(x.device)
            x = x * lam.reshape(B, 1, 1, 1) + x[rn] * (1. - lam.reshape(B, 1, 1, 1))
            y_hat, _ = ref_model(x)
            loss = (F.cross_entropy(y_hat, y, reduction="none") * lam.reshape(B) +
                    F.cross_entropy(y_hat, y[rn], reduction="none") * (1. - lam.reshape(B))).mean()
            loss.detach().cpu().numpy()
            loss.backward()
            opt.step()
            opt.zero_grad()

        timed(ours, a.warmup)
        timed(script, a.warmup)
        t_ours, t_ref = [], []
        for _ in range(a.trials):
            t_ours.append(timed(ours, a.steps))
            t_ref.append(timed(script, a.steps))
        mo, mr = statistics.median(t_ours), statistics.median(t_ref)
        emit({"bench": "finetune_step", "model": "mn10", "B": B, "seconds": a.seconds, "classes": a.classes,
              "trainer_graph_ms": round(mo, 3), "script_loop_ms": round(mr, 3), "speedup": round(mr / mo, 3),
              "trials_trainer_ms": [round(t, 3) for t in t_ours], "trials_script_ms": [round(t, 3) for t in t_ref],
              **info})
        del tr, model, ref_model, opt
        torch.cuda.empty_cache()

        # MixStyle on the log-mel of this batch size
        T = 1 + (n_samples - 1) // 320
        x = torch.randn(B, 1, 128, T, device="cuda") * 0.2 - 1.0
        out, stats = torch.empty_like(x), torch.empty(2 * B * 128, device="cuda")
        perm = torch.randperm(B).int().cuda()
        lam = torch.rand(B).cuda()
        st = torch.cuda.current_stream().cuda_stream

        def ms():
            lib().mixstyle(x.data_ptr(), perm.data_ptr(), lam.data_ptr(), 1e-6, stats.data_ptr(), out.data_ptr(), B, 128,
                           T, st)

        timed(ms, a.warmup)
        t = statistics.median(timed(ms, a.steps) for _ in range(a.rounds))
        nbytes = 3 * 4 * B * 128 * T + 16 * B * 128
        emit({"bench": "eat_mixstyle", "B": B, "F": 128, "T": T, "us": round(t * 1e3, 2), "alg_bytes": nbytes,
              "GB_s": round(nbytes / (t * 1e-3) / 1e9, 1), "of_hbm_peak": round(nbytes / (t * 1e-3) / HBM, 3), **info})


if __name__ == "__main__":
    np.random.seed(0)
    torch.manual_seed(0)
    main()
