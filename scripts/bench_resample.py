"""Benchmark of the polyphase resampler (efficientat_b200/resample.py, csrc/resample.cu).

1. `eat_resample_poly_fwd` and `eat_resample_poly_bwd` at B = 256 x 10 s from 44.1, 48, 22.05 and 16 kHz to 32 kHz:
   each launch after a write of 256 MB that flushes the L2, timed alone with CUDA events; median of --rounds launches.
   Algorithmic bytes: 4 (N_in + N_out) per clip, set against the 3.35 TB/s HBM3 figure of NVIDIA's H100 SXM data sheet.
2. The CPU baseline: scipy.signal.resample_poly over the same batch on every host core (one process per core, rows
   split evenly, results kept in the workers), host clock, median of --cpu-rounds.
3. End to end: eval of mel + mn10 (synthetic weights) on B = --e2e-batch clips of 10 s at 44.1 kHz already on the
   device, with Resample in front, against the same clips resampled on the host beforehand (mel + mn10 only); CUDA
   events, median of --rounds.

The card's name, power limit and maximum SM clock are read in the same call.  One JSON line per result."""
import argparse
import contextlib
import io
import json
import multiprocessing as mp
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from efficientat_b200._lib import lib  # noqa: E402
from efficientat_b200.models.mn.model import get_model  # noqa: E402
from efficientat_b200.models.preprocess import AugmentMelSTFT  # noqa: E402
from efficientat_b200.resample import Resample  # noqa: E402
from efficientat_b200.synth import synth_state_  # noqa: E402

HBM = 3.35e12

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=256)
ap.add_argument("--seconds", type=float, default=10.0)
ap.add_argument("--rounds", type=int, default=20)
ap.add_argument("--cpu-rounds", type=int, default=3)
ap.add_argument("--e2e-batch", type=int, default=64)
ap.add_argument("--skip-cpu", action="store_true")
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


def signal(B, N, sr, seed=0):
    g = torch.Generator().manual_seed(seed)
    t = torch.arange(N, dtype=torch.float64) / sr
    chirp = torch.sin(2 * torch.pi * (100 + 4000 * t / (N / sr)) * t)
    return (0.5 * chirp + 0.2 * torch.randn(B, N, generator=g, dtype=torch.float64)).float()


_FLUSH = None


def cold_ms(fn, rounds):
    """median time of fn() alone, each launch after a 256 MB write that evicts the 50 MB L2"""
    global _FLUSH
    if _FLUSH is None:
        _FLUSH = torch.empty(64 << 20, dtype=torch.float32, device="cuda")
    ts = []
    for _ in range(rounds + 2):
        _FLUSH.zero_()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        fn()
        t1.record()
        t1.synchronize()
        ts.append(t0.elapsed_time(t1))
    return statistics.median(ts[2:])


def kernels(info):
    L, st = lib(), torch.cuda.current_stream().cuda_stream
    B = a.batch
    for orig in (44100, 48000, 22050, 16000):
        rs = Resample(orig).cuda()
        N = int(orig * a.seconds)
        x = signal(B, N, orig).cuda()
        y = rs(x)
        dx = torch.empty_like(x)
        n_out = y.shape[1]
        fwd = lambda: L.resample_poly_fwd(x.data_ptr(), B, N, 0, rs.up, rs.down, rs._table.data_ptr(), rs.taps,  # noqa
                                          rs.half_len, y.data_ptr(), n_out, st)
        bwd = lambda: L.resample_poly_bwd(y.data_ptr(), B, N, rs.up, rs.down, rs._table_adj.data_ptr(), rs.taps_adj,  # noqa
                                          rs.half_len, dx.data_ptr(), n_out, st)
        nbytes = 4 * B * (N + n_out)
        for name, fn in (("fwd", fwd), ("bwd", bwd)):
            ms = cold_ms(fn, a.rounds)
            rate = nbytes / (ms * 1e-3)
            emit({"bench": f"resample_{name}", "orig_sr": orig, "new_sr": 32000, "up": rs.up, "down": rs.down,
                  "B": B, "N_in": N, "N_out": n_out, "taps_per_output": rs.taps if name == "fwd" else rs.taps_adj,
                  "ms": round(ms, 4), "algorithmic_GBps": round(rate / 1e9, 1),
                  "share_of_hbm_peak": round(rate / HBM, 3), **info})
        del x, y, dx


_ROWS = None


def _cpu_rows(span):
    import scipy.signal as ss
    lo, hi, up, down = span
    s = 0.0
    for r in range(lo, hi):
        s += float(ss.resample_poly(_ROWS[r], up, down)[0])
    return s


def cpu_baseline(info):
    global _ROWS
    cores = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else os.cpu_count()
    for orig in (44100, 48000):
        rs = Resample(orig)
        _ROWS = signal(a.batch, int(orig * a.seconds), orig).numpy()
        per = -(-a.batch // cores)
        spans = [(i, min(i + per, a.batch), rs.up, rs.down) for i in range(0, a.batch, per)]
        ts = []
        with mp.get_context("fork").Pool(min(cores, len(spans))) as pool:
            pool.map(_cpu_rows, spans[:1])                        # scipy imported in the workers
            for _ in range(a.cpu_rounds):
                t0 = time.perf_counter()
                pool.map(_cpu_rows, spans)
                ts.append(time.perf_counter() - t0)
        emit({"bench": "resample_cpu_scipy", "orig_sr": orig, "B": a.batch, "seconds": a.seconds, "host_cores": cores,
              "ms": round(statistics.median(ts) * 1e3, 1), **info})


def end_to_end(info):
    B, orig = a.e2e_batch, 44100
    with contextlib.redirect_stdout(io.StringIO()):
        model = synth_state_(get_model(width_mult=1.0, verbose=False), seed=3).cuda().eval()
        mel = AugmentMelSTFT(freqm=0, timem=0).cuda().eval()
    rs = Resample(orig).cuda()
    x = signal(B, int(orig * a.seconds), orig).cuda()
    x32 = rs(x).clone()                       # the pre-resampled batch (identical values to a host resampling's shape)

    def native():
        model(mel(rs(x)).unsqueeze(1))

    def pre():
        model(mel(x32).unsqueeze(1))
    with torch.no_grad():
        for fn in (native, pre):
            for _ in range(3):
                fn()
        res = {"native": [], "pre": []}
        for _ in range(a.rounds):                                 # alternated, so that drift hits both arms alike
            for name, fn in (("native", native), ("pre", pre)):
                torch.cuda.synchronize()
                t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0.record()
                fn()
                t1.record()
                t1.synchronize()
                res[name].append(t0.elapsed_time(t1))
    nat, pre_ms = statistics.median(res["native"]), statistics.median(res["pre"])
    emit({"bench": "resample_e2e_mn10_eval", "orig_sr": orig, "B": B, "seconds": a.seconds,
          "ms_resample_mel_mn10": round(nat, 3), "ms_mel_mn10_pre_resampled": round(pre_ms, 3),
          "clips_per_s_native": round(B / nat * 1e3, 1), "clips_per_s_pre_resampled": round(B / pre_ms * 1e3, 1), **info})


def main():
    if not torch.cuda.is_available():
        raise SystemExit("bench_resample.py measures on a CUDA device; none is available")
    info = card()
    kernels(info)
    end_to_end(info)
    if not a.skip_cpu:
        cpu_baseline(info)


if __name__ == "__main__":
    main()
