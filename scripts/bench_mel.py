"""Benchmark of the fused mel kernel (eat_mel_fwd) at every supported n_fft, B = 256 clips of 10 s at 32 kHz.

Geometry per size: 128 mels, win_length = min(800, n_fft), hop = min(320, n_fft / 2).  Each size is timed with CUDA
events over --steps launches after --warmup launches, --rounds times; the input (327 MB) does not fit in L2, so no flush
is needed.  Algorithmic bytes per clip are 4·N (waveform read) + 4·n_mels·T (log-mel written); the achieved rate is
set against the 3.35 TB/s HBM3 figure of NVIDIA's H100 SXM data sheet, with the card's name and power limit read in the
same call.

--baseline-lib PATH loads a second build of libeat_b200.so (for instance the one of an earlier commit) and, at the
sizes it supports, alternates its launches with this tree's round by round and checks that both produce the same bits
on the same seeded batch.  One JSON line per size, then a summary line; --out also writes them to a file."""
import argparse
import contextlib
import ctypes
import io
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from efficientat_b200 import _lib  # noqa: E402
from efficientat_b200.models.preprocess import AugmentMelSTFT  # noqa: E402
from efficientat_b200.synth import synth_waveform  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
SIZES = (256, 512, 1024, 2048, 4096)

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=256)
ap.add_argument("--seconds", type=float, default=10.0)
ap.add_argument("--sr", type=int, default=32000)
ap.add_argument("--steps", type=int, default=20, help="timed launches per round")
ap.add_argument("--warmup", type=int, default=3)
ap.add_argument("--rounds", type=int, default=5)
ap.add_argument("--sizes", type=int, nargs="*", default=list(SIZES))
ap.add_argument("--baseline-lib", default=None, help="another libeat_b200.so to alternate with and compare against")
ap.add_argument("--out", default=None, help="also write the JSON lines here")
a = ap.parse_args()


def load(path):
    dll = ctypes.CDLL(path)
    f = dll.eat_mel_fwd
    f.restype = ctypes.c_int
    f.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
                  ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                  ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_void_p, ctypes.c_void_p]
    dll.eat_last_error.restype = ctypes.c_char_p
    return dll


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                            "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        name, power, clock = (s.strip() for s in q.stdout.strip().split(","))
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:                                     # report what could be read, never guess
        return {"gpu": torch.cuda.get_device_name(), "power_limit": f"not read ({type(e).__name__})",
                "max_sm_clock": "not read"}


def launcher(dll, mel, x, out):
    start, length, taps, max_len = mel._filterbank(mel.fmin, mel.fmax, x.device)
    b, n = x.shape
    st = torch.cuda.current_stream().cuda_stream

    def run():
        rc = dll.eat_mel_fwd(x.data_ptr(), b, n, mel.window.data_ptr(), mel.win_length, mel.hopsize, mel.n_fft,
                             mel._twiddle.data_ptr(), start.data_ptr(), length.data_ptr(), taps.data_ptr(), max_len,
                             mel.n_mels, mel._preemph, out.data_ptr(), st)
        if rc != 0:
            raise RuntimeError(f"eat_mel_fwd failed ({rc}): {dll.eat_last_error().decode()}")
    return run


def time_round(fn):
    for _ in range(a.warmup):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.steps):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / a.steps


def main():
    assert torch.cuda.is_available(), "bench_mel.py times the CUDA kernel and needs a GPU"
    dev = torch.device("cuda")
    info = card()
    new = load(_lib.LIB_PATH)
    old = load(os.path.abspath(a.baseline_lib)) if a.baseline_lib else None
    n = int(round(a.seconds * a.sr))
    x = synth_waveform(a.batch, n, seed=0).to(dev)
    lines = []
    for n_fft in a.sizes:
        win, hop, n_mels = min(800, n_fft), min(320, n_fft // 2), 128
        with contextlib.redirect_stdout(io.StringIO()):
            mel = AugmentMelSTFT(n_mels=n_mels, sr=a.sr, win_length=win, hopsize=hop, n_fft=n_fft).to(dev).eval()
        t = 1 + (n - 1) // hop
        out_new = torch.empty(a.batch, n_mels, t, device=dev)
        runs = {"new": launcher(new, mel, x, out_new)}
        out_old = None
        if old is not None:
            out_old = torch.full_like(out_new, float("nan"))
            probe = launcher(old, mel, x, out_old)
            try:
                probe()
                runs["baseline"] = probe
            except RuntimeError as e:
                print(f"# n_fft {n_fft}: baseline library refuses it ({e})", flush=True)
        times = {k: [] for k in runs}
        for _ in range(a.rounds):                               # alternate the builds round by round
            for k, fn in runs.items():
                times[k].append(time_round(fn))
        torch.cuda.synchronize()
        nbytes = a.batch * (4 * n + 4 * n_mels * t)
        rec = dict(info, n_fft=n_fft, win_length=win, hop=hop, n_mels=n_mels, batch=a.batch, samples=n, frames=t,
                   bytes=nbytes)
        for k, ts in times.items():
            med = statistics.median(ts)
            rec[f"{k}_ms"] = round(med, 4)
            rec[f"{k}_ms_min_max"] = [round(min(ts), 4), round(max(ts), 4)]
            rec[f"{k}_GBps"] = round(nbytes / (med * 1e-3) / 1e9, 1)
            rec[f"{k}_share_of_3.35TBps"] = round(nbytes / (med * 1e-3) / HBM_BYTES_PER_S, 4)
        if "baseline" in runs:
            rec["bitwise_equal_to_baseline"] = bool(torch.equal(out_new, out_old))
            rec["max_abs_diff_to_baseline"] = (out_new - out_old).abs().max().item()
        assert torch.isfinite(out_new).all(), f"n_fft {n_fft}: non-finite output"
        line = json.dumps(rec)
        print(line, flush=True)
        lines.append(line)
        del out_new, out_old
    summary = {"bench": "mel", "gpu": info["gpu"], "power_limit": info["power_limit"],
               "ms": {json.loads(l)["n_fft"]: json.loads(l)["new_ms"] for l in lines}}
    print(json.dumps(summary), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write("\n".join(lines + [json.dumps(summary)]) + "\n")


if __name__ == "__main__":
    main()
