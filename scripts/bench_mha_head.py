"""Benchmark of the multi-head attention pooling head (MN head_type='multihead_attention_pooling') at the flagship shape:
mn10, B = 256 clips of 10 s at 32 kHz (1000 frames, 128 mels), H = 4 heads, K = 527 classes.  The head sees the last conv's
output [256, 960, 4, 32]; its projection is [8192 rows, 960] x [4216, 960]^T.

1. Each new kernel and the three head GEMMs (projection, its weight and data gradient), timed with CUDA events over
   --steps launches after --warmup, --rounds times (median), on the shapes of a training step.  Algorithmic bytes
   (operands read once, results written once) and FLOPs are set against NVIDIA's H100 SXM data-sheet figures: 3.35 TB/s
   HBM3 and 989 TFLOP/s dense bf16, i.e. 330 TFLOP/s for the bf16x3 products (three bf16 MMAs per fp32-grade product)
   the fp32-storage tensor-core GEMMs use.  The bound named is the larger of bytes / bandwidth and FLOPs / rate.
2. Whole AudioSetTrainer steps (CUDA graph, as bench.py) with the mlp head and with this head, same trunk state,
   alternating the two trainers --trials times in one process; the difference of the medians is reported.
3. The head's eval logits against fp64 at that size: the fp64 expression of attention_pooling.py:40-56 evaluated on the
   engine's own last feature map (the trunk's parity is pinned elsewhere).

The card's name and power limit are read in the same call.  One JSON line per result; --out also writes them to a file."""
import argparse
import contextlib
import io
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from efficientat_b200._lib import lib  # noqa: E402
from efficientat_b200.models.mn.model import get_model  # noqa: E402
from efficientat_b200.models.preprocess import AugmentMelSTFT  # noqa: E402
from efficientat_b200.synth import synth_labels, synth_state_, synth_waveform  # noqa: E402
from efficientat_b200.train import AudioSetTrainer  # noqa: E402
from tests.mha_util import HEAD, mha_head  # noqa: E402

HBM = 3.35e12
BF16 = 989e12
BF16X3 = BF16 / 3

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=256)
ap.add_argument("--seconds", type=float, default=10.0)
ap.add_argument("--heads", type=int, default=4)
ap.add_argument("--steps", type=int, default=20, help="timed launches per round")
ap.add_argument("--warmup", type=int, default=3)
ap.add_argument("--rounds", type=int, default=5)
ap.add_argument("--trials", type=int, default=5, help="alternations of the mlp and attention-head trainers")
ap.add_argument("--train-steps", type=int, default=10, help="trainer steps per trial")
ap.add_argument("--out", default=None)
a = ap.parse_args()

lines = []


def emit(d):
    s = json.dumps(d)
    print(s, flush=True)
    lines.append(s)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                            "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        name, power, clock = (s.strip() for s in q.stdout.strip().split(","))
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:                     # the name still comes from the driver; the limit is then unknown
        return {"gpu": torch.cuda.get_device_name(), "power_limit": f"not read ({type(e).__name__})",
                "max_sm_clock": "not read"}


def time_ms(fn):
    for _ in range(a.warmup):
        fn()
    meds = []
    for _ in range(a.rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.steps):
            fn()
        e1.record()
        e1.synchronize()
        meds.append(e0.elapsed_time(e1) / a.steps)
    return statistics.median(meds)


def report(name, ms, nbytes, flops=0.0, rate=None):
    t_mem = nbytes / HBM
    t_cmp = flops / rate if rate else 0.0
    bound = "compute" if t_cmp > t_mem else "memory"
    emit({"kernel": name, "ms": round(ms, 4), "alg_bytes": int(nbytes), "alg_flops": int(flops),
          "GB_per_s": round(nbytes / ms / 1e6, 1), "TFLOP_per_s": round(flops / ms / 1e9, 1) if flops else None,
          "bound": bound, "share_of_bound": round(max(t_mem, t_cmp) * 1e3 / ms, 3)})


def main():
    if not torch.cuda.is_available():
        raise SystemExit("bench_mha_head.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    info = card()
    emit({"bench": "mha_head", **info, "batch": a.batch, "seconds": a.seconds, "heads": a.heads})
    L = lib()
    st = torch.cuda.current_stream().cuda_stream
    n = int(a.seconds * 32000)
    frames = 1 + (n - 1) // 320
    torch.manual_seed(0)
    with contextlib.redirect_stdout(io.StringIO()):
        mha = synth_state_(get_model(width_mult=1.0, head_type=HEAD, multihead_attention_heads=a.heads, verbose=False),
                           seed=7).to(dev)
        mlp = synth_state_(get_model(width_mult=1.0, verbose=False), seed=7).to(dev)
    eng = mha.engine()
    head = mha.classifier
    B, H, K = a.batch, a.heads, head.out_dim
    C = head.in_dim
    spec = synth_waveform(B, 128 * frames, seed=21, std=0.7).view(B, 1, 128, frames).to(dev)

    # ---- 3. parity of the head at this size (eval, engine's own last feature map)
    mha.eval()
    with torch.no_grad():
        logits, fmaps = mha._forward_impl(spec, return_fmaps=True)
        z = fmaps[-1]
        F_, T_ = z.shape[2], z.shape[3]
        ref = mha_head(z.double(), head.subspace_proj.weight.double(), head.subspace_proj.bias.double(),
                       head.head_weight.double(), H, K)
    err = (logits.double() - ref).abs().max().item()
    emit({"parity": "head logits vs fp64 on the engine's last feature map", "shape": list(z.shape),
          "max_abs_err": err, "ref_absmax": ref.abs().max().item()})
    del fmaps, z, ref

    # ---- 1. kernels and GEMMs on the training-step shapes
    M, N = B * T_, 2 * H * K
    zl = torch.randn(B, F_, T_, C, device=dev)
    sc = torch.stack([torch.rand(C, device=dev) + 0.5, torch.randn(C, device=dev) * 0.1])
    m = torch.empty(B, T_, C, device=dev)
    feat = torch.empty(B, C, device=dev)
    report("eat_freq_pool (BN + Hardswish on load)", time_ms(lambda: L.freq_pool(
        zl.data_ptr(), 0, sc[0].data_ptr(), sc[1].data_ptr(), 2, m.data_ptr(), feat.data_ptr(), B, F_, T_, C, st)),
        4 * (B * F_ * T_ * C + B * T_ * C + B * C))
    P = torch.empty(M, N, device=dev)
    proj = head.subspace_proj
    report("projection GEMM m.W^T+b (eat_pw_tma_fwd)", time_ms(lambda: eng._gemm(
        m, proj.weight, P, M, N, C, bias=proj.bias, a_code=0, c_code=0)), 4 * (M * C + N * C + M * N), 2.0 * M * N * C, BF16X3)
    out = torch.empty(B, K, device=dev)
    sa, r = torch.empty(B, H, K, device=dev), torch.empty(B, H, K, device=dev)
    hw = head.head_weight
    report("eat_att_pool_fwd", time_ms(lambda: L.att_pool_fwd(
        P.data_ptr(), hw.data_ptr(), head.epsilon, out.data_ptr(), sa.data_ptr(), r.data_ptr(), B, T_, H, K, st)),
        4 * (M * N + 3 * B * H * K + B * K))
    dout = torch.randn(B, K, device=dev) / (B * K)
    dP = torch.empty_like(P)
    dhw, db = torch.zeros(H, device=dev), torch.zeros(N, device=dev)
    report("eat_att_pool_bwd", time_ms(lambda: L.att_pool_bwd(
        dout.data_ptr(), P.data_ptr(), dP.data_ptr(), hw.data_ptr(), sa.data_ptr(), r.data_ptr(), head.epsilon,
        dhw.data_ptr(), db.data_ptr(), B, T_, H, K, st)), 4 * (2 * M * N + 2 * B * H * K + B * K + N))
    dW = torch.zeros(N, C, device=dev)
    report("weight gradient dP^T.m (eat_pw_tc_wgrad)", time_ms(lambda: eng._wgrad(
        dP, m, dW, None, M, N, C, g_code=0, a_code=0)), 4 * (M * N + M * C + N * C), 2.0 * M * N * C, BF16X3)
    dm = torch.empty(B, T_, C, device=dev)
    report("data gradient dP.W (eat_pw_tma_fwd, W transposed)", time_ms(lambda: eng._gemm(
        dP, proj.weight, dm, M, C, N, a_code=0, c_code=0, w_trans=True)), 4 * (M * N + N * C + M * C), 2.0 * M * N * C, BF16X3)
    gA = torch.empty_like(zl)
    report("eat_freq_pool_bwd", time_ms(lambda: L.freq_pool_bwd(
        dm.data_ptr(), 1.0 / F_, gA.data_ptr(), 0, B, F_, T_, C, st)), 4 * (B * T_ * C + B * F_ * T_ * C))
    del zl, m, P, dP, gA, dW, dm
    torch.cuda.empty_cache()

    # ---- 2. whole training steps, the two heads alternating
    with contextlib.redirect_stdout(io.StringIO()):
        mel = AugmentMelSTFT(freqm=0, timem=0).to(dev)
    wave = synth_waveform(B, n, seed=3).to(dev)
    y = synth_labels(B, K, seed=4).to(dev)
    teacher = torch.sigmoid(torch.randn(B, K, generator=torch.Generator().manual_seed(5))).to(dev)
    trainers = {name: AudioSetTrainer(model, mel, lr=8e-4, kd_lambda=0.1, mixup_alpha=0.3, cuda_graph=True)
                for name, model in (("mlp", mlp), (HEAD, mha))}
    for tr in trainers.values():
        for _ in range(3):
            tr.step(wave, y, teacher)
    torch.cuda.synchronize()
    times = {k: [] for k in trainers}
    for _ in range(a.trials):
        for name, tr in trainers.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.train_steps):
                tr.step(wave, y, teacher)
            e1.record()
            e1.synchronize()
            times[name].append(e0.elapsed_time(e1) / a.train_steps)
    med = {k: statistics.median(v) for k, v in times.items()}
    emit({"trainer_step_ms": {k: round(v, 3) for k, v in med.items()},
          "spread_ms": {k: [round(min(v), 3), round(max(v), 3)] for k, v in times.items()},
          "difference_ms": round(med[HEAD] - med["mlp"], 3),
          "difference_pct": round(100 * (med[HEAD] - med["mlp"]) / med["mlp"], 2), **info})
    for tr in trainers.values():
        tr.close()
    if a.out:
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
