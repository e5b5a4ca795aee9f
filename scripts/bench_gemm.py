"""Micro-benchmark of the pointwise-conv GEMM kernels at mn10 layer shapes (B clips): time + achieved GB/s.
    python scripts/bench_gemm.py [--batch 256] [--impl pw_tc_fwd] [--dtype fp32] [--only IDX]
    python scripts/bench_gemm.py --mn10-step [--batch 256] [--baseline-lib PATH] [--out FILE]

--mn10-step records every eat_pw_tma_fwd launch of one eager mn10 training step at --batch clips (forward 1x1 convs and
the 1x1 data gradients that the fused backward kernels do not cover, with their real M, N, K, input transform, SE gate,
residual and statistics), then times each launch shape on fresh operands with CUDA events, --rounds rounds of --iters
launches after a warm-up.  --baseline-lib loads another build of libeat_b200.so (an earlier commit's) and alternates
with it round by round, on the same operands, and reports the largest output difference between the two.  Per launch and
in total: time, algorithmic GB/s (4 bytes x (M K + M N (+ M N residual) + N K)) and FLOP/s (2 M N K) against 330 TFLOP/s,
the H100 SXM data sheet's dense BF16 rate (989 TFLOP/s) over the three bf16 products of the fp32-grade GEMM.  The card's
name and power limit are read in the same call."""
import argparse, ctypes, json, os, statistics, subprocess, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from efficientat_b200 import _lib
from efficientat_b200._lib import lib

BF16X3_FLOPS = 989e12 / 3

# (rows per clip, K, N, residual, in-transform+gate)  -- mn10 forward pointwise layers
LAYERS = [(32000, 16, 16, 1, 0), (32000, 16, 64, 0, 0), (8000, 64, 24, 0, 0), (8000, 24, 72, 0, 0), (8000, 72, 24, 1, 0),
          (8000, 24, 72, 0, 0), (2000, 72, 40, 0, 1), (2000, 40, 120, 0, 0), (2000, 120, 40, 1, 1), (2000, 40, 240, 0, 0),
          (504, 240, 80, 0, 0), (504, 80, 200, 0, 0), (504, 200, 80, 1, 0), (504, 80, 480, 0, 0), (504, 480, 112, 0, 1),
          (504, 112, 672, 0, 0), (504, 672, 112, 1, 1), (128, 672, 160, 0, 1), (128, 160, 960, 0, 0), (128, 960, 160, 1, 1)]

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=256)
ap.add_argument("--impl", default="pw_tc_fwd")
ap.add_argument("--dtype", default="fp32")
ap.add_argument("--only", type=int, default=-1)
ap.add_argument("--iters", type=int, default=10)
ap.add_argument("--raw", action="store_true", help="no input transform, no epilogue, no statistics (data-gradient shape)")
ap.add_argument("--train", action="store_true", help="training-mode variant: raw output + statistics, BN+act on load")
ap.add_argument("--mn10-step", action="store_true", help="every eat_pw_tma_fwd launch of the mn10 training step")
ap.add_argument("--rounds", type=int, default=5, help="--mn10-step: timed rounds per launch shape and library")
ap.add_argument("--baseline-lib", default=None, help="--mn10-step: another libeat_b200.so to alternate with")
ap.add_argument("--out", default=None, help="--mn10-step: also write the JSON lines here")
a = ap.parse_args()


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                            "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        name, power, clock = (s.strip() for s in q.stdout.strip().split(","))
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:                                     # report what could be read, never guess
        return {"gpu": torch.cuda.get_device_name(), "power_limit": f"not read ({type(e).__name__})",
                "max_sm_clock": "not read"}


def record_step_launches(batch):
    """(w_trans, M, N, K, in_act, has in-transform, gate rows per sample or 0, epilogue act or None, residual, stats) of
    every eat_pw_tma_fwd launch of one eager mn10 training step"""
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
    orig, launches = L.pw_tma_fwd, []

    def rec(*args):
        (A, W, wt, C, M, N, K, isc, ish, in_act, gate, rps, sc, sh, act, res, s0, s1, ws, wsb, st) = args
        launches.append((wt, M, N, K, in_act, bool(isc), rps if gate else 0,
                         (act if (sc or sh or act) else None), bool(res), bool(s0)))
        return orig(*args)
    L.pw_tma_fwd = rec
    try:
        trainer.step(wave, y, teacher, teacher_known=known.float())
        torch.cuda.synchronize()
    finally:
        L.pw_tma_fwd = orig
    del trainer, model, mel
    torch.cuda.empty_cache()
    return launches


def load(path):
    dll = ctypes.CDLL(path)
    f = dll.eat_pw_tma_fwd
    f.restype = ctypes.c_int
    f.argtypes = _lib.parse_header()["eat_pw_tma_fwd"][1]
    dll.eat_last_error.restype = ctypes.c_char_p
    return dll


def mn10_step():
    assert torch.cuda.is_available(), "bench_gemm.py times CUDA kernels and needs a GPU"
    info = card()
    libs = {"new": load(_lib.LIB_PATH)}
    if a.baseline_lib:
        libs["baseline"] = load(os.path.abspath(a.baseline_lib))
    launches = record_step_launches(a.batch)
    g = torch.Generator(device="cuda").manual_seed(0)
    st = torch.cuda.current_stream().cuda_stream
    p = lambda t: 0 if t is None else t.data_ptr()
    lines, tot = [], {k: 0.0 for k in libs}
    tot_bytes = tot_flop = 0
    for i, (wt, M, N, K, in_act, xf, rps, act, res, stats) in enumerate(launches):
        A = torch.randn(M, K, device="cuda", generator=g)
        W = torch.randn(K, N, device="cuda", generator=g) / K ** 0.5 if wt else torch.randn(N, K, device="cuda", generator=g) / K ** 0.5
        isc = torch.stack([torch.rand(K, device="cuda", generator=g) + 0.5, torch.randn(K, device="cuda", generator=g) * 0.1]) if xf else None
        gate = torch.rand((M + rps - 1) // rps, K, device="cuda", generator=g) if rps else None
        sc = torch.stack([torch.rand(N, device="cuda", generator=g) + 0.5, torch.randn(N, device="cuda", generator=g) * 0.1]) if act is not None else None
        R = torch.randn(M, N, device="cuda", generator=g) if res else None
        S = torch.zeros(2, N, device="cuda", dtype=torch.float64) if stats else None
        ws = torch.empty(N * ((K + 31) // 32) * 128, device="cuda", dtype=torch.uint8)
        outs = {k: torch.empty(M, N, device="cuda") for k in libs}

        def launcher(dll, C):
            def run():
                rc = dll.eat_pw_tma_fwd(A.data_ptr(), W.data_ptr(), wt, C.data_ptr(), M, N, K, p(isc[0]) if xf else 0,
                                        p(isc[1]) if xf else 0, in_act if xf else 0, p(gate), rps if rps else 1,
                                        p(sc[0]) if sc is not None else 0, p(sc[1]) if sc is not None else 0,
                                        act or 0, p(R), p(S[0]) if S is not None else 0, p(S[1]) if S is not None else 0,
                                        ws.data_ptr(), ws.numel(), st)
                if rc != 0:
                    raise RuntimeError(f"eat_pw_tma_fwd failed ({rc}): {dll.eat_last_error().decode()}")
            return run
        runs = {k: launcher(dll, outs[k]) for k, dll in libs.items()}
        times = {k: [] for k in runs}
        for fn in runs.values():
            fn()
        for _ in range(a.rounds):                              # alternate the builds round by round
            for k, fn in runs.items():
                fn()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(a.iters):
                    fn()
                e1.record()
                e1.synchronize()
                times[k].append(e0.elapsed_time(e1) / a.iters)
        nbytes = 4 * (M * K + M * N * (2 if res else 1) + N * K)
        flop = 2 * M * N * K
        rec = dict(idx=i, M=M, N=N, K=K, w_trans=wt, in_transform=xf, gate_rps=rps, epilogue=act is not None,
                   residual=res, stats=stats)
        for k, ts in times.items():
            med = statistics.median(ts)
            tot[k] += med
            rec[f"{k}_us"] = round(med * 1e3, 2)
            rec[f"{k}_us_min_max"] = [round(min(ts) * 1e3, 2), round(max(ts) * 1e3, 2)]
            rec[f"{k}_GBps"] = round(nbytes / (med * 1e-3) / 1e9, 1)
            rec[f"{k}_TFLOPs"] = round(flop / (med * 1e-3) / 1e12, 2)
            rec[f"{k}_share_of_330TFLOPs"] = round(flop / (med * 1e-3) / BF16X3_FLOPS, 4)
        if "baseline" in runs:
            ref = outs["baseline"]
            rec["max_rel_diff_to_baseline"] = ((outs["new"] - ref).abs().max() / (ref.abs().max() + 1e-30)).item()
        tot_bytes += nbytes
        tot_flop += flop
        line = json.dumps(rec)
        print(line, flush=True)
        lines.append(line)
        del A, W, isc, gate, sc, R, S, ws, outs
    summary = dict(info, bench="pw_tma_fwd launches of the mn10 training step", batch=a.batch, launches=len(launches))
    for k, t in tot.items():
        summary[f"{k}_total_ms"] = round(t, 4)
        summary[f"{k}_total_GBps"] = round(tot_bytes / (t * 1e-3) / 1e9, 1)
        summary[f"{k}_total_TFLOPs"] = round(tot_flop / (t * 1e-3) / 1e12, 2)
        summary[f"{k}_share_of_330TFLOPs"] = round(tot_flop / (t * 1e-3) / BF16X3_FLOPS, 4)
    print(json.dumps(summary), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write("\n".join(lines + [json.dumps(summary)]) + "\n")


if a.mn10_step:
    mn10_step()
    sys.exit(0)

L = lib()
fn = getattr(L, a.impl)
td = torch.float32 if a.dtype == "fp32" else torch.bfloat16
code = 0 if a.dtype == "fp32" else 1
es = 4 if code == 0 else 2
st = torch.cuda.current_stream().cuda_stream
flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
tot_t = tot_b = 0.0
for i, (rows, K, N, res, xf) in enumerate(LAYERS):
    if a.only >= 0 and i != a.only:
        continue
    M = rows * a.batch
    A = torch.randn(M, K, device="cuda").to(td)
    W = torch.randn(N, K, device="cuda") / K ** 0.5
    C = torch.empty(M, N, device="cuda", dtype=td)
    R = torch.randn(M, N, device="cuda").to(td) if res else None
    sc = torch.rand(2, N, device="cuda")
    isc = torch.rand(2, K, device="cuda")
    gate = torch.rand(a.batch, K, device="cuda") if xf else None
    stats = torch.zeros(2, N, device="cuda", dtype=torch.float64)
    p = lambda t: 0 if t is None else t.data_ptr()
    if a.raw:
        args = (A.data_ptr(), code, W.data_ptr(), 0, C.data_ptr(), code, M, N, K, 0, 0, 0, 0, rows, 0, 0, 0, 0, 0, 0, st)
    elif a.train:
        args = (A.data_ptr(), code, W.data_ptr(), 0, C.data_ptr(), code, M, N, K, isc[0].data_ptr(), isc[1].data_ptr(), 2,
                p(gate), rows, 0, 0, 0, 0, stats[0].data_ptr(), stats[1].data_ptr(), st)
    else:
        args = (A.data_ptr(), code, W.data_ptr(), 0, C.data_ptr(), code, M, N, K, 0, 0, 0, p(gate), rows,
                sc[0].data_ptr(), sc[1].data_ptr(), 2, p(R), 0, 0, st)
    for _ in range(2):
        fn(*args)
    ts = []
    for _ in range(a.iters):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(*args); e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ms = sorted(ts)[len(ts) // 2]
    nbytes = M * K * es + M * N * es * (2 if (res and not a.train and not a.raw) else 1) + N * K * 4
    tot_t += ms; tot_b += nbytes
    print(f"{i:2d} M={M:8d} K={K:4d} N={N:4d} res={res} xf={xf}  {ms*1e3:8.1f} us  {nbytes/ms/1e6:8.1f} GB/s  "
          f"{2*M*N*K/ms/1e9:8.2f} TFLOP/s", flush=True)
print(json.dumps({"impl": a.impl, "dtype": a.dtype, "batch": a.batch, "train": a.train, "total_ms": tot_t,
                  "total_GBps": tot_b / tot_t / 1e6}))
