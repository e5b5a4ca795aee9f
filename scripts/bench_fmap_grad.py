"""Cost of losses on the embedding and on the feature maps in a training step of mn10 and dymn10.

    python scripts/bench_fmap_grad.py [--batch 64 256] [--steps 10] [--warmup 3] [--out results/fmap_grad.json]

For each model and batch size, 10 s clips (128 x 1001 spectrogram), fp32 storage, train(), dropout 0, through autograd
(model forward, loss, loss.backward()):
- logits:     bce(logits);
- +embedding: bce(logits) + <r, features>;
- +per-frame: bce(logits) + a per-frame linear head on the last map's frequency mean (10 outputs per frame);
- +17 maps:   bce(logits) + sum_i <R_i, fmap_i> / numel_i over all 17 maps.
Host clock around work that ends in a device synchronise, median over --steps; the four losses alternate step by step.
Then eat_fmap_grad_nhwc alone (CUDA events, L2 flushed before each launch) on the last map's shape from a contiguous
NCHW gradient, a channels-last one and a frequency-mean broadcast, each overwriting and accumulating, with its
algorithmic bytes (src read once unless broadcast, dst written once, read once more when accumulating) over its time,
against 3.35 TB/s.  Prints the card, its power limit and maximum SM clock, read in the same call."""
import argparse
import contextlib
import io
import json
import os
import subprocess
import sys
import time

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from efficientat_b200._lib import lib  # noqa: E402
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
    m = m.cuda().train()
    for mod in m.modules():
        if isinstance(mod, torch.nn.Dropout):
            mod.p = 0.0
    return m


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def fmaps_of(m, x):
    if hasattr(m, "layers"):
        return m(x, return_fmaps=True)
    return m._forward_impl(x, return_fmaps=True)


def kernel_rows(B, C, Fq, T, steps):
    """eat_fmap_grad_nhwc on a [B, C, Fq, T] map: (layout, accumulate) -> ms and GB/s"""
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    dst = torch.empty(B, Fq, T, C, device="cuda")
    srcs = {"nchw": torch.randn(B, C, Fq, T, device="cuda"),
            "channels_last": torch.randn(B, Fq, T, C, device="cuda").permute(0, 3, 1, 2),
            "freq_mean": torch.randn(B, C, 1, T, device="cuda").expand(B, C, Fq, T)}
    rows = []
    for name, src in srcs.items():
        for acc in (0, 1):
            def run():
                lib().fmap_grad_nhwc(src.data_ptr(), 0, *src.stride(), dst.data_ptr(), 0, B, C, Fq, T, acc,
                                     torch.cuda.current_stream().cuda_stream)
            times = []
            for i in range(steps + 1):
                flush.zero_()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                run()
                e1.record()
                torch.cuda.synchronize()
                if i:
                    times.append(e0.elapsed_time(e1) * 1e-3)
            t = sorted(times)[len(times) // 2]
            n = B * C * Fq * T
            src_bytes = 4 * (n // Fq if name == "freq_mean" else n)
            nbytes = src_bytes + 4 * n * (2 if acc else 1)
            rows.append(dict(kernel="eat_fmap_grad_nhwc", layout=name, accumulate=acc, shape=[B, C, Fq, T],
                             ms=t * 1e3, GBps=nbytes / t / 1e9, share_of_hbm=nbytes / t / HBM))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, nargs="+", default=[64, 256])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark needs a GPU"
    info = card()
    print(info, flush=True)
    models = {k: model(k) for k in ("mn10", "dymn10")}
    rows = []
    for B in a.batch:
        spec = torch.randn(B, 1, 128, FRAMES, device="cuda")
        y = (torch.rand(B, 527, device="cuda") < 0.05).float()
        for k, m in models.items():
            with torch.no_grad():
                _, feat = m(spec)
                _, maps = fmaps_of(m, spec)
            r = torch.randn_like(feat)
            R = [torch.randn_like(t) for t in maps]
            W = torch.randn(10, maps[-1].shape[1], device="cuda") * 0.05
            frame_y = torch.full((B, maps[-1].shape[3], 10), 0.3, device="cuda")
            m.zero_grad(set_to_none=True)

            def logits_only():
                lo, _ = m(spec)
                F.binary_cross_entropy_with_logits(lo, y).backward()

            def embedding():
                lo, fe = m(spec)
                (F.binary_cross_entropy_with_logits(lo, y) + (r * fe).sum()).backward()

            def per_frame():
                lo, mp = fmaps_of(m, spec)
                fr = mp[-1].mean(2).transpose(1, 2)
                (F.binary_cross_entropy_with_logits(lo, y)
                 + F.binary_cross_entropy_with_logits(fr @ W.T, frame_y)).backward()

            def all_maps():
                lo, mp = fmaps_of(m, spec)
                loss = F.binary_cross_entropy_with_logits(lo, y)
                for Ri, t in zip(R, mp):
                    loss = loss + (Ri * t).sum() / t.numel()
                loss.backward()
            cases = {"logits": logits_only, "embedding": embedding, "per_frame_head": per_frame, "all_17_maps": all_maps}
            res = {c: [] for c in cases}
            for i in range(a.warmup + a.steps):
                for c, fn in cases.items():             # the losses alternate step by step
                    t = timed(fn)
                    m.zero_grad(set_to_none=True)
                    if i >= a.warmup:
                        res[c].append(t)
            row = dict(model=k, batch=B, frames=FRAMES, card=info)
            for c, ts in res.items():
                row[c + "_ms"] = sorted(ts)[len(ts) // 2] * 1e3
            rows.append(row)
            print(json.dumps(row), flush=True)
            last = maps[-1].shape
            del maps, R
            torch.cuda.empty_cache()
        for row in kernel_rows(B, last[1], last[2], last[3], a.steps):
            row["card"] = info
            rows.append(row)
            print(json.dumps(row), flush=True)
        del spec
        torch.cuda.empty_cache()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
