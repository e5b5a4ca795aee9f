"""Gradients with respect to the input spectrogram of a frozen tagger in eval(): the cost of using mn10 or dymn10 as a
differentiable loss.

    python scripts/bench_input_grad.py [--batch 64 256] [--steps 10] [--warmup 3] [--out gpu_out/input_grad.json]

For each model and batch size, 10 s clips (128 x 1001 spectrogram), fp32 storage, every parameter frozen:
- eval forward alone (input without grad: the folded-BatchNorm forward);
- forward plus input backward (input requires grad: the saving forward on running statistics, the backward down to
  the spectrogram through eat_stem_dgrad, no weight-gradient pass);
- the same from the waveform: AugmentMelSTFT forward, the model, and the backward through eat_mel_bwd;
- eat_stem_dgrad and eat_mel_bwd alone (L2 flushed, CUDA events), with their algorithmic bytes over their time:
  stem: dy and z read once, dx written once; mel: dspec and the waveform read once, dwave written once, and the
  frame-slice scratch written and read once.
Host clock around work that ends in a device synchronise, median over --steps; the models alternate step by step.
Prints the card, its power limit and maximum SM clock, read in the same call."""
import argparse
import contextlib
import ctypes
import io
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from efficientat_b200._lib import lib  # noqa: E402
from efficientat_b200.models.preprocess import AugmentMelSTFT  # noqa: E402
from efficientat_b200.synth import synth_state_  # noqa: E402

FRAMES = 1001
HBM = 3.35e12       # H100 SXM data-sheet HBM3 bandwidth, bytes/s


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    return q or torch.cuda.get_device_name()


def model(kind):
    if kind == "mn10":
        from efficientat_b200.models.mn.model import get_model
    else:
        from efficientat_b200.models.dymn.model import get_model
    with contextlib.redirect_stdout(io.StringIO()):
        m = synth_state_(get_model(width_mult=1.0, verbose=False), seed=3)
    m = m.cuda().eval()
    for p in m.parameters():
        p.requires_grad_(False)
    return m


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def events(fn, steps):
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    times = []
    for i in range(steps + 1):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        if i:
            times.append(e0.elapsed_time(e1) * 1e-3)
    return sorted(times)[len(times) // 2]


def mel_bwd(mel, B, steps):
    """eat_mel_bwd at n_fft 1024, hop 320, 128 mels, 10 s at 32 kHz (the module's eval filterbank)"""
    N = 320000
    wave = torch.randn(B, N, device="cuda") * 0.1
    x = wave.clone().requires_grad_(True)
    out = mel(x)
    saved = out.grad_fn.saved
    dspec = torch.randn_like(out)
    t = events(lambda: mel._backward(wave, dspec, saved), steps)
    need = ctypes.c_longlong()
    lib().mel_bwd_workspace(B, N, mel.hopsize, mel.n_fft, ctypes.addressof(need))
    scratch = 4 * 2 * need.value
    nbytes = 4 * (dspec.numel() + 2 * wave.numel()) + scratch
    return dict(ms=t * 1e3, bytes=nbytes, gbps=nbytes / t / 1e9, share_of_hbm=nbytes / t / HBM)


def stem_dgrad(B, steps):
    """eat_stem_dgrad at the mn10 stem shape (C = 16, stride 2), fp32, L2 flushed before each launch"""
    F, T, C = 128, FRAMES, 16
    Fo, To = (F - 1) // 2 + 1, (T - 1) // 2 + 1
    dy, z = torch.randn(B, Fo, To, C, device="cuda"), torch.randn(B, Fo, To, C, device="cuda")
    v = torch.rand(6, C, device="cuda") + 0.5
    v[4:].zero_()
    w = torch.randn(C, 1, 3, 3, device="cuda")
    dx = torch.empty(B, F, T, device="cuda")
    t = events(lambda: lib().stem_dgrad(dy.data_ptr(), 0, z.data_ptr(), *[v[j].data_ptr() for j in range(4)], 2,
                                        v[4].data_ptr(), v[5].data_ptr(), w.data_ptr(), dx.data_ptr(), B, F, T, C, 2,
                                        torch.cuda.current_stream().cuda_stream), steps)
    nbytes = 4 * (2 * dy.numel() + dx.numel())
    return dict(ms=t * 1e3, bytes=nbytes, gbps=nbytes / t / 1e9, share_of_hbm=nbytes / t / HBM)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, nargs="+", default=[64, 256])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_input_grad.py measures on a CUDA device"
    info = card()
    print(info, flush=True)
    models = {k: model(k) for k in ("mn10", "dymn10")}
    with contextlib.redirect_stdout(io.StringIO()):
        mel = AugmentMelSTFT(freqm=0, timem=0).cuda().eval()
    rows = []
    for B in a.batch:
        spec = torch.randn(B, 1, 128, FRAMES, device="cuda")
        x = spec.clone().requires_grad_(True)
        wave = (torch.randn(B, 320000, device="cuda") * 0.1).requires_grad_(True)

        def fwd(m):
            with torch.no_grad():
                m(spec)

        def fwd_bwd(m):
            out, _ = m(x)
            out.sum().backward()
            x.grad = None

        def wave_bwd(m):
            out, _ = m(mel(wave).unsqueeze(1))
            out.sum().backward()
            wave.grad = None
        res = {k: {"eval_forward": [], "forward_input_backward": [], "waveform_forward_backward": []} for k in models}
        for i in range(a.warmup + a.steps):
            for k, m in models.items():             # the models alternate step by step
                tf, tb, tw = timed(lambda: fwd(m)), timed(lambda: fwd_bwd(m)), timed(lambda: wave_bwd(m))
                if i >= a.warmup:
                    res[k]["eval_forward"].append(tf)
                    res[k]["forward_input_backward"].append(tb)
                    res[k]["waveform_forward_backward"].append(tw)
        for k in models:
            row = dict(model=k, batch=B, frames=FRAMES, card=info)
            for what, ts in res[k].items():
                row[what + "_ms"] = sorted(ts)[len(ts) // 2] * 1e3
            rows.append(row)
            print(json.dumps(row), flush=True)
        del spec, x, wave
        torch.cuda.empty_cache()
        for name, fn in (("eat_stem_dgrad", lambda: stem_dgrad(B, a.steps)), ("eat_mel_bwd", lambda: mel_bwd(mel, B, a.steps))):
            row = dict(kernel=name, batch=B, card=info, **fn())
            rows.append(row)
            print(json.dumps(row), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
