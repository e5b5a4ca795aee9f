"""GPU parity of the GEMM kernels through the C ABI: the wgmma pointwise-conv kernel (csrc/pw_wgmma.cu)
and the exact-fp32 CUDA-core kernel (csrc/gemm_simt.cu) against a float64 torch reference, over the layer
shapes of mn10/mn40 plus ragged edge cases (M not a multiple of 128, K / N not multiples of 64 / 16).
fp32 storage (hi/lo split, 3 MMAs): 2e-4 of the output scale.  bf16 storage: 2e-2 (bf16 operand rounding)."""
import pytest
import torch

from efficientat_b200._lib import lib

pytestmark = pytest.mark.gpu

SHAPES = [  # (M, N, K)
    (4096, 64, 16), (4000, 24, 64), (1300, 72, 24), (777, 40, 72), (2048, 120, 40), (1024, 240, 40),
    (640, 80, 240), (512, 200, 80), (384, 480, 80), (300, 112, 480), (256, 672, 112), (128, 160, 672),
    (1024, 960, 160), (130, 960, 160), (20000, 16, 16), (256, 3840, 640), (129, 8, 8),
    # N tiles wider than 128 columns (K >= 160): one ragged tile of 208, 3 x 160, one of 192, 4 x 192 with a clipped last tile
    (1000, 200, 160), (515, 480, 192), (900, 184, 200), (260, 672, 192), (700, 160, 960),
]


def _ref(A, W, in_sc, in_act, gate, rps, sc, act, res):
    a = A.double()
    if in_sc is not None:
        a = a * in_sc[0].double() + in_sc[1].double()
        a = torch.relu(a) if in_act == 1 else (torch.nn.functional.hardswish(a) if in_act == 2 else a)
    if gate is not None:
        a = a * gate.double().repeat_interleave(rps, 0)[: a.shape[0]]
    raw = a @ W.double().t()
    out = raw
    if sc is not None:
        out = out * sc[0].double() + sc[1].double()
    out = torch.relu(out) if act == 1 else (torch.nn.functional.hardswish(out) if act == 2 else out)
    if res is not None:
        out = out + res.double()
    return out, raw


def _call(fn, A, W, C, M, N, K, in_sc, in_act, gate, rps, sc, act, res, stats):
    code = 0 if A.dtype == torch.float32 else 1
    p = lambda t: 0 if t is None else t.data_ptr()
    fn(A.data_ptr(), code, W.data_ptr(), 0, C.data_ptr(), code, M, N, K, p(in_sc[0]) if in_sc is not None else 0,
       p(in_sc[1]) if in_sc is not None else 0, in_act, p(gate), rps, p(sc[0]) if sc is not None else 0,
       p(sc[1]) if sc is not None else 0, act, p(res), p(stats[0]) if stats is not None else 0,
       p(stats[1]) if stats is not None else 0, torch.cuda.current_stream().cuda_stream)


@pytest.mark.parametrize("impl", ["pw_tc_fwd", "gemm_simt_fwd"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_gemm_all_shapes_fused_epilogue(impl, dtype):
    fn = getattr(lib(), impl)
    g = torch.Generator(device="cuda").manual_seed(0)
    for idx, (M, N, K) in enumerate(SHAPES):
        A = torch.randn(M, K, device="cuda", generator=g).to(dtype)
        W = torch.randn(N, K, device="cuda", generator=g) / K ** 0.5
        variant = idx % 4
        in_sc = gate = sc = res = stats = None
        in_act = act = 0
        rps = 1
        if variant in (1, 3):
            in_sc = torch.stack([torch.rand(K, device="cuda", generator=g) + 0.5, torch.randn(K, device="cuda", generator=g) * 0.1])
            in_act = 2 if variant == 1 else 1
        if variant in (2, 3):
            rps = 37
            nb = (M + rps - 1) // rps
            gate = torch.rand(nb, K, device="cuda", generator=g)
        if variant in (0, 2):
            sc = torch.stack([torch.rand(N, device="cuda", generator=g) + 0.5, torch.randn(N, device="cuda", generator=g) * 0.1])
            act = 2 if variant == 0 else 0
            res = torch.randn(M, N, device="cuda", generator=g).to(dtype) if variant == 2 else None
        else:
            stats = torch.zeros(2, N, device="cuda", dtype=torch.float64)
        C = torch.full((M, N), float("nan"), device="cuda").to(dtype)
        _call(fn, A, W, C, M, N, K, in_sc, in_act, gate, rps, sc, act, res, stats)
        torch.cuda.synchronize()
        ref, raw = _ref(A, W, in_sc, in_act, gate, rps, sc, act, res)
        scale = ref.abs().max().item() + 1e-6
        tol = (2e-4 if impl == "pw_tc_fwd" else 2e-5) if dtype == torch.float32 else 2e-2
        err = (C.double() - ref).abs().max().item() / scale
        assert err < tol, f"{impl} {dtype} shape {(M, N, K)} variant {variant}: rel err {err}"
        if stats is not None:
            s_ref, q_ref = raw.sum(0), (raw * raw).sum(0)
            stol = 1e-3 if dtype == torch.float32 else 3e-2
            assert ((stats[0] - s_ref).abs().max() / (s_ref.abs().max() + 1e-6)).item() < stol, (M, N, K)
            assert ((stats[1] - q_ref).abs().max() / (q_ref.abs().max() + 1e-6)).item() < stol, (M, N, K)


@pytest.mark.parametrize("w_trans", [0, 1])
def test_tma_gemm_with_presplit_weights(w_trans):
    """eat_pw_tma_fwd with the weight workspace (the engine's route): weights pre-split into bf16 hi|lo rows by a prep kernel
    (epilogue scale folded; w_trans = 1: W handed over as [K, N], the data-gradient case), every variant / ragged shape."""
    L = lib()
    g = torch.Generator(device="cuda").manual_seed(5)
    st = torch.cuda.current_stream().cuda_stream
    p = lambda t: 0 if t is None else t.data_ptr()
    for idx, (M, N, K) in enumerate(SHAPES):
        if K % 4 or N % 4:
            continue
        A = torch.randn(M, K, device="cuda", generator=g)
        W = torch.randn(N, K, device="cuda", generator=g) / K ** 0.5
        variant = idx % 4
        in_sc = gate = sc = res = stats = None
        in_act = act = 0
        rps = 1
        if variant in (1, 3):
            in_sc = torch.stack([torch.rand(K, device="cuda", generator=g) + 0.5, torch.randn(K, device="cuda", generator=g) * 0.1])
            in_act = 2 if variant == 1 else 1
        if variant in (2, 3):
            rps = 37
            gate = torch.rand((M + rps - 1) // rps, K, device="cuda", generator=g)
        if variant in (0, 2):
            sc = torch.stack([torch.rand(N, device="cuda", generator=g) + 0.5, torch.randn(N, device="cuda", generator=g) * 0.1])
            act = 2 if variant == 0 else 0
            res = torch.randn(M, N, device="cuda", generator=g) if variant == 2 else None
        else:
            stats = torch.zeros(2, N, device="cuda", dtype=torch.float64)
        C = torch.full((M, N), float("nan"), device="cuda")
        Wg = W.t().contiguous() if w_trans else W
        ws = torch.empty(N * ((K + 31) // 32) * 128, device="cuda", dtype=torch.uint8)
        L.pw_tma_fwd(A.data_ptr(), Wg.data_ptr(), w_trans, C.data_ptr(), M, N, K, p(in_sc[0]) if in_sc is not None else 0,
                     p(in_sc[1]) if in_sc is not None else 0, in_act, p(gate), rps, p(sc[0]) if sc is not None else 0,
                     p(sc[1]) if sc is not None else 0, act, p(res), p(stats[0]) if stats is not None else 0,
                     p(stats[1]) if stats is not None else 0, ws.data_ptr(), ws.numel(), st)
        torch.cuda.synchronize()
        ref, raw = _ref(A, W, in_sc, in_act, gate, rps, sc, act, res)
        err = (C.double() - ref).abs().max().item() / (ref.abs().max().item() + 1e-6)
        assert err < 2e-4, f"pw_tma_fwd(ws) w_trans={w_trans} shape {(M, N, K)} variant {variant}: rel err {err}"
        if stats is not None:
            s_ref = raw.sum(0)
            assert ((stats[0] - s_ref).abs().max() / (s_ref.abs().max() + 1e-6)).item() < 1e-3, (M, N, K)


def test_tc_gemm_large_streaming_shape():
    """block-2 expand of mn10 at B=32: M = 32*64*500 rows, K = 16 -> N = 64; checks the persistent tile loop."""
    M, N, K = 32 * 64 * 500, 64, 16
    g = torch.Generator(device="cuda").manual_seed(1)
    A = torch.randn(M, K, device="cuda", generator=g)
    W = torch.randn(N, K, device="cuda", generator=g) / 4
    C = torch.empty(M, N, device="cuda")
    stats = torch.zeros(2, N, device="cuda", dtype=torch.float64)
    _call(lib().pw_tc_fwd, A, W, C, M, N, K, None, 0, None, 1, None, 0, None, stats)
    ref = A @ W.t()
    assert (C - ref).abs().max() < 1e-3
    assert ((stats[0] - ref.double().sum(0)).abs().max() / ref.double().sum(0).abs().max()) < 1e-3


def test_wgrad_and_transposed_gemm_match_torch():
    L = lib()
    g = torch.Generator(device="cuda").manual_seed(2)
    st = torch.cuda.current_stream().cuda_stream
    for (M, N, K) in [(5000, 72, 24), (256, 527, 1280), (300, 960, 160), (7, 24, 8)]:
        G = torch.randn(M, N, device="cuda", generator=g)
        A = torch.randn(M, K, device="cuda", generator=g)
        dW = torch.zeros(N, K, device="cuda")
        db = torch.zeros(N, device="cuda")
        L.gemm_simt_wgrad(G.data_ptr(), 0, A.data_ptr(), 0, dW.data_ptr(), db.data_ptr(), M, N, K, 0, 0, 0, 0, 1, st)
        ref = G.double().t() @ A.double()
        assert ((dW.double() - ref).abs().max() / ref.abs().max()).item() < 1e-4
        assert ((db.double() - G.double().sum(0)).abs().max() / G.double().sum(0).abs().max()).item() < 1e-4
        # data gradient: dA[M,K] = G[M,N] . W[N,K]  via the transposed-weight path
        W = torch.randn(N, K, device="cuda", generator=g)
        dA = torch.empty(M, K, device="cuda")
        L.gemm_simt_fwd(G.data_ptr(), 0, W.data_ptr(), 1, dA.data_ptr(), 0, M, K, N, 0, 0, 0, 0, 1, 0, 0, 0, 0, 0, 0, st)
        ref = G.double() @ W.double()
        assert ((dA.double() - ref).abs().max() / ref.abs().max()).item() < 1e-5


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_tc_wgrad_matches_torch(dtype):
    """wgmma weight gradient (MN-major operands) vs float64 torch; fused input transform + SE gate included."""
    L = lib()
    g = torch.Generator(device="cuda").manual_seed(3)
    st = torch.cuda.current_stream().cuda_stream
    code = 0 if dtype == torch.float32 else 1
    cases = [(4096, 64, 16, 0), (5000, 72, 24, 1), (3000, 24, 72, 2), (2048, 240, 40, 0), (1100, 112, 672, 3),
             (1024, 960, 160, 0), (700, 160, 960, 1), (40000, 16, 16, 2), (2000, 200, 80, 0), (1500, 8, 8, 0),
             # narrow layers with a long reduction: N*K <= 512 in fp32 storage takes the CUDA-core kernel
             # (csrc/wgrad_narrow.cu); the wider ones stay on tensor cores
             (70001, 16, 16, 0), (66000, 64, 16, 1), (65537, 24, 64, 1), (80000, 72, 24, 0), (70003, 24, 72, 1),
             (66001, 8, 8, 1), (70000, 16, 16, 2), (66003, 32, 16, 1), (65540, 16, 24, 3)]
    for (M, N, K, variant) in cases:
        G = (torch.randn(M, N, device="cuda", generator=g) * 0.1).to(dtype)
        A = torch.randn(M, K, device="cuda", generator=g).to(dtype)
        in_sc = gate = None
        in_act, rps = 0, 1
        if variant in (1, 3):
            in_sc = torch.stack([torch.rand(K, device="cuda", generator=g) + 0.5, torch.randn(K, device="cuda", generator=g) * 0.1])
            in_act = 2 if variant == 1 else 1
        if variant in (2, 3):
            rps = 53
            gate = torch.rand((M + rps - 1) // rps, K, device="cuda", generator=g)
        dW = torch.zeros(N, K, device="cuda")
        p = lambda t: 0 if t is None else t.data_ptr()
        L.pw_tc_wgrad(G.data_ptr(), code, A.data_ptr(), code, dW.data_ptr(), 0, M, N, K,
                      p(in_sc[0]) if in_sc is not None else 0, p(in_sc[1]) if in_sc is not None else 0, in_act, p(gate),
                      rps, st)
        torch.cuda.synchronize()
        a = A.double()
        if in_sc is not None:
            a = a * in_sc[0].double() + in_sc[1].double()
            a = torch.relu(a) if in_act == 1 else torch.nn.functional.hardswish(a)
        if gate is not None:
            a = a * gate.double().repeat_interleave(rps, 0)[:M]
        ref = G.double().t() @ a
        err = ((dW.double() - ref).abs().max() / (ref.abs().max() + 1e-9)).item()
        tol = 2e-4 if dtype == torch.float32 else 2e-2
        assert err < tol, f"wgrad {dtype} {(M, N, K)} variant {variant}: rel err {err}"


@pytest.mark.parametrize("w_trans", [0, 1])
def test_tma_dynamic_gemm_matches_per_sample_reference(w_trans):
    """eat_pw_tma_dyn_fwd (DynamicConv 1x1, dy_block.py:103-131): per-sample kernels sum_j att[b,j] W_j; tiles, loads and
    stores never cross a sample (3-D tensor maps) -- rows per sample that are not multiples of 128 / 32, ragged N and K,
    epilogue scale / shift / activation, residual, statistics; w_trans = 1 is the data-gradient orientation."""
    L = lib()
    g = torch.Generator(device="cuda").manual_seed(9)
    st = torch.cuda.current_stream().cuda_stream
    p = lambda t: 0 if t is None else t.data_ptr()
    for idx, (B, rps, N, K) in enumerate([(3, 500, 64, 16), (2, 2000, 24, 72), (5, 130, 200, 80), (4, 128, 112, 672), (2, 63, 8, 8),
                                          (3, 504, 960, 160), (7, 37, 40, 120),
                                          # B >= 8: several samples' tiles per CTA, per-sample kernels past the first eight
                                          (12, 101, 64, 16), (64, 28, 24, 72)]):
        M, nk = B * rps, 4
        A = torch.randn(M, K, device="cuda", generator=g)
        W = torch.randn(nk, N, K, device="cuda", generator=g) / K ** 0.5
        att = torch.softmax(torch.randn(B, nk, device="cuda", generator=g), 1)
        variant = idx % 3
        sc = res = stats = None
        act = 0
        if variant == 0:
            stats = torch.zeros(2, N, device="cuda", dtype=torch.float64)
        elif variant == 1:
            sc = torch.stack([torch.rand(N, device="cuda", generator=g) + 0.5, torch.randn(N, device="cuda", generator=g) * 0.1])
            act = 2
        else:
            sc = torch.stack([torch.rand(N, device="cuda", generator=g) + 0.5, torch.randn(N, device="cuda", generator=g) * 0.1])
            res = torch.randn(M, N, device="cuda", generator=g)
        Wg = W.transpose(1, 2).contiguous() if w_trans else W
        C = torch.full((M, N), float("nan"), device="cuda")
        ws = torch.empty(B * N * ((K + 31) // 32) * 128, device="cuda", dtype=torch.uint8)
        L.pw_tma_dyn_fwd(A.data_ptr(), Wg.data_ptr(), att.data_ptr(), nk, w_trans, C.data_ptr(), M, N, K, rps,
                         p(sc[0]) if sc is not None else 0, p(sc[1]) if sc is not None else 0, act, p(res),
                         p(stats[0]) if stats is not None else 0, p(stats[1]) if stats is not None else 0, ws.data_ptr(),
                         ws.numel(), st)
        torch.cuda.synchronize()
        Wb = torch.einsum("bj,jnk->bnk", att.double(), W.double())
        raw = torch.einsum("brk,bnk->brn", A.double().view(B, rps, K), Wb).reshape(M, N)
        ref = raw
        if sc is not None:
            ref = ref * sc[0].double() + sc[1].double()
        if act == 2:
            ref = torch.nn.functional.hardswish(ref)
        if res is not None:
            ref = ref + res.double()
        err = (C.double() - ref).abs().max().item() / (ref.abs().max().item() + 1e-6)
        assert err < 2e-4, f"pw_tma_dyn_fwd w_trans={w_trans} {(B, rps, N, K)} variant {variant}: rel err {err}"
        if stats is not None:
            s_ref, q_ref = raw.sum(0), (raw * raw).sum(0)
            assert ((stats[0] - s_ref).abs().max() / (s_ref.abs().max() + 1e-6)).item() < 1e-3
            assert ((stats[1] - q_ref).abs().max() / (q_ref.abs().max() + 1e-6)).item() < 1e-3
