"""Micro-benchmark of the wgmma weight-gradient kernel at mn10 layer shapes: dW[N,K] += G[M,N]^T . xf(A)[M,K].
    python scripts/bench_wgrad.py [--batch 256]
    python scripts/bench_wgrad.py --mn10-step [--batch 256] [--baseline-lib PATH] [--out FILE]

--mn10-step records every eat_pw_tc_wgrad launch of one eager mn10 training step at --batch clips (the 1x1 weight
gradients the fused backward kernels do not cover, the last conv included, with their real M, N, K, input transform and
SE gate), then times each launch on fresh operands with CUDA events, the L2 flushed before every launch, --rounds
rounds of --iters launches after a warm-up.  --baseline-lib loads another build of libeat_b200.so (an earlier commit's)
and alternates with it round by round on the same operands; the largest difference of dW between the two builds is
reported relative to sum |g| |xf(x)| of that entry.  Per launch and in total: time, algorithmic GB/s (4 bytes x
(M N + M K + N K)) and TFLOP/s (2 M N K).  The card's name and power limit are read in the same call."""
import argparse, ctypes, json, os, statistics, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from efficientat_b200 import _lib
from efficientat_b200._lib import lib
LAYERS = [(32000, 16, 16, 0), (32000, 16, 64, 0), (8000, 64, 24, 1), (8000, 24, 72, 0), (8000, 72, 24, 1),
          (8000, 24, 72, 0), (2000, 72, 40, 1), (2000, 40, 120, 0), (2000, 120, 40, 1), (2000, 40, 240, 0),
          (504, 240, 80, 1), (504, 80, 200, 0), (504, 200, 80, 1), (504, 80, 480, 0), (504, 480, 112, 1),
          (504, 112, 672, 0), (504, 672, 112, 1), (128, 672, 160, 1), (128, 160, 960, 0), (128, 960, 160, 1)]
ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=256)
ap.add_argument("--mn10-step", action="store_true", help="every eat_pw_tc_wgrad launch of the mn10 training step")
ap.add_argument("--rounds", type=int, default=5, help="--mn10-step: timed rounds per launch and library")
ap.add_argument("--iters", type=int, default=5, help="--mn10-step: launches per round (each after an L2 flush)")
ap.add_argument("--baseline-lib", default=None, help="--mn10-step: another libeat_b200.so to alternate with")
ap.add_argument("--out", default=None, help="--mn10-step: also write the JSON lines here")
a = ap.parse_args()


def card():
    import subprocess
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                            "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        name, power, clock = (s.strip() for s in q.stdout.strip().split(","))
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:                                     # report what could be read, never guess
        return {"gpu": torch.cuda.get_device_name(), "power_limit": f"not read ({type(e).__name__})",
                "max_sm_clock": "not read"}


def record_step_launches(batch):
    """(M, N, K, in_act, has in-transform, gate rows per sample or 0) of every eat_pw_tc_wgrad launch of one eager mn10
    training step"""
    import contextlib, io
    import bench
    from efficientat_b200.models.mn.model import get_model
    from efficientat_b200.models.preprocess import AugmentMelSTFT
    from efficientat_b200.synth import synth_state_
    from efficientat_b200.train import AudioSetTrainer
    dev = torch.device("cuda")
    torch.manual_seed(0)
    with contextlib.redirect_stdout(io.StringIO()):
        model = synth_state_(get_model(width_mult=1.0, verbose=False), seed=7).to(dev)
        mel = AugmentMelSTFT(freqm=0, timem=0).to(dev)
    trainer = AudioSetTrainer(model, mel, lr=8e-4, kd_lambda=0.1, mixup_alpha=0.3, cuda_graph=False)
    wave, y, teacher, known = (t.to(dev) for t in bench._synth_batch(batch, 0))
    L = lib()
    orig, launches = L.pw_tc_wgrad, []

    def rec(*args):
        (G, gd, A, ad, dW, db, M, N, K, isc, ish, in_act, gate, rps, st) = args
        launches.append((M, N, K, in_act, bool(isc), rps if gate else 0))
        return orig(*args)
    L.pw_tc_wgrad = rec
    try:
        trainer.step(wave, y, teacher, teacher_known=known.float())
        torch.cuda.synchronize()
    finally:
        L.pw_tc_wgrad = orig
    del trainer, model, mel
    torch.cuda.empty_cache()
    return launches


def load(path):
    dll = ctypes.CDLL(path)
    f = dll.eat_pw_tc_wgrad
    f.restype = ctypes.c_int
    f.argtypes = _lib.parse_header()["eat_pw_tc_wgrad"][1]
    dll.eat_last_error.restype = ctypes.c_char_p
    return dll


def mn10_step():
    assert torch.cuda.is_available(), "bench_wgrad.py times CUDA kernels and needs a GPU"
    info = card()
    libs = {"new": load(_lib.LIB_PATH)}
    if a.baseline_lib:
        libs["baseline"] = load(os.path.abspath(a.baseline_lib))
    launches = record_step_launches(a.batch)
    g = torch.Generator(device="cuda").manual_seed(0)
    st = torch.cuda.current_stream().cuda_stream
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
    p = lambda t: 0 if t is None else t.data_ptr()
    lines, tot = [], {k: 0.0 for k in libs}
    tot_bytes = tot_flop = 0
    for i, (M, N, K, in_act, xf, rps) in enumerate(launches):
        G = torch.randn(M, N, device="cuda", generator=g)
        X = torch.randn(M, K, device="cuda", generator=g)
        isc = torch.stack([torch.rand(K, device="cuda", generator=g) + 0.5, torch.randn(K, device="cuda", generator=g) * 0.1]) if xf else None
        gate = torch.rand((M + rps - 1) // rps, K, device="cuda", generator=g) if rps else None
        outs = {k: torch.zeros(N, K, device="cuda") for k in libs}

        def launcher(dll, dW):
            def run():
                rc = dll.eat_pw_tc_wgrad(G.data_ptr(), 0, X.data_ptr(), 0, dW.data_ptr(), None, M, N, K,
                                         p(isc[0]) if xf else 0, p(isc[1]) if xf else 0, in_act if xf else 0, p(gate),
                                         rps if rps else 1, st)
                if rc != 0:
                    raise RuntimeError(f"eat_pw_tc_wgrad failed ({rc}): {dll.eat_last_error().decode()}")
            return run
        runs = {k: launcher(dll, outs[k]) for k, dll in libs.items()}
        for k, fn in runs.items():                             # one launch into a zeroed dW: the compared result
            fn()
        torch.cuda.synchronize()
        res = {k: o.clone() for k, o in outs.items()}
        times = {k: [] for k in runs}
        for _ in range(a.rounds):                              # alternate the builds round by round
            for k, fn in runs.items():
                ts = []
                for _ in range(a.iters):
                    flush.zero_()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    fn()
                    e1.record()
                    e1.synchronize()
                    ts.append(e0.elapsed_time(e1))
                times[k].append(statistics.median(ts))
        nbytes = 4 * (M * N + M * K + N * K)
        flop = 2 * M * N * K
        rec = dict(idx=i, M=M, N=N, K=K, in_transform=xf, in_act=in_act, gate_rps=rps)
        for k, ts in times.items():
            med = statistics.median(ts)
            tot[k] += med
            rec[f"{k}_us"] = round(med * 1e3, 2)
            rec[f"{k}_us_min_max"] = [round(min(ts) * 1e3, 2), round(max(ts) * 1e3, 2)]
            rec[f"{k}_GBps"] = round(nbytes / (med * 1e-3) / 1e9, 1)
            rec[f"{k}_TFLOPs"] = round(flop / (med * 1e-3) / 1e12, 2)
        if "baseline" in runs:
            xx = X.double()
            if xf:
                xx = xx * isc[0].double() + isc[1].double()
                xx = xx.clamp_min(0) if in_act == 1 else (xx * (xx + 3).clamp(0, 6) / 6 if in_act == 2 else xx)
            if rps:
                xx = xx * gate.double()[torch.arange(M, device="cuda") // rps]
            mag = G.double().abs().t() @ xx.abs()
            rec["max_dW_diff_over_sum_abs_terms"] = ((res["new"].double() - res["baseline"].double()).abs() / (mag + 1e-300)).max().item()
            del xx, mag
        tot_bytes += nbytes
        tot_flop += flop
        line = json.dumps(rec)
        print(line, flush=True)
        lines.append(line)
        del G, X, isc, gate, outs, res
    summary = dict(info, bench="eat_pw_tc_wgrad launches of the mn10 training step, L2 flushed", batch=a.batch,
                   launches=len(launches))
    for k, t in tot.items():
        summary[f"{k}_total_ms"] = round(t, 4)
        summary[f"{k}_total_GBps"] = round(tot_bytes / (t * 1e-3) / 1e9, 1)
        summary[f"{k}_total_TFLOPs"] = round(tot_flop / (t * 1e-3) / 1e12, 2)
    print(json.dumps(summary), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write("\n".join(lines + [json.dumps(summary)]) + "\n")


if a.mn10_step:
    mn10_step()
    sys.exit(0)

L = lib(); st = torch.cuda.current_stream().cuda_stream
flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
tot = 0.0; totb = 0
for i, (rows, K, N, xf) in enumerate(LAYERS):
    M = rows * a.batch
    A = torch.randn(M, K, device="cuda"); G = torch.randn(M, N, device="cuda"); dW = torch.zeros(N, K, device="cuda")
    isc = torch.rand(2, K, device="cuda")
    args = (G.data_ptr(), 0, A.data_ptr(), 0, dW.data_ptr(), 0, M, N, K, isc[0].data_ptr() if xf else 0, isc[1].data_ptr() if xf else 0, 2 if xf else 0, 0, rows, st)
    L.pw_tc_wgrad(*args); ts = []
    for _ in range(6):
        flush.zero_(); e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); L.pw_tc_wgrad(*args); e1.record(); torch.cuda.synchronize(); ts.append(e0.elapsed_time(e1))
    ms = sorted(ts)[len(ts) // 2]; nb = M * (K + N) * 4; tot += ms; totb += nb
    print(f"{i:2d} M={M:8d} K={K:4d} N={N:4d} xf={xf}  {ms*1e3:8.1f} us  {nb/ms/1e6:8.1f} GB/s", flush=True)
print(json.dumps({"impl": "pw_tc_wgrad", "batch": a.batch, "total_ms": tot, "total_GBps": totb / tot / 1e6}))
