"""eat_pw_tma_fwd / eat_pw_tma_dyn_fwd at every N-tile width the planner produces, against float64 torch.

N is cut into ceil(N / 128) tiles of equal width rounded up to 8 columns (N = 72 -> 72, 200 -> 2 x 104, 240 -> 2 x 120,
4216 -> 33 x 128).  The last 32-column chunk of a tile may be 8, 16 or 24 columns wide and is stored through its own
tensor map; a store that reached past it would overwrite the next tile's columns, so every multi-tile case here has such
a tail and checks every output column.  Output: 2e-4 of the output scale (bf16x3 products); batch statistics: 1e-3 of
the largest column sum."""
import pytest
import torch

from efficientat_b200._lib import lib

pytestmark = pytest.mark.gpu


def _p(t):
    return 0 if t is None else t.data_ptr()


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


def _run(M, N, K, g, *, w_trans=0, in_act=0, gate_rps=0, epi=False, act=0, res=False, stats=False):
    A = torch.randn(M, K, device="cuda", generator=g)
    W = torch.randn(N, K, device="cuda", generator=g) / K ** 0.5
    in_sc = gate = sc = R = st = None
    rps = 1
    if in_act:
        in_sc = torch.stack([torch.rand(K, device="cuda", generator=g) + 0.5, torch.randn(K, device="cuda", generator=g) * 0.1])
    if gate_rps:
        rps = gate_rps
        gate = torch.rand((M + rps - 1) // rps, K, device="cuda", generator=g)
    if epi:
        sc = torch.stack([torch.rand(N, device="cuda", generator=g) + 0.5, torch.randn(N, device="cuda", generator=g) * 0.1])
    if res:
        R = torch.randn(M, N, device="cuda", generator=g)
    if stats:
        st = torch.zeros(2, N, device="cuda", dtype=torch.float64)
    C = torch.full((M, N), float("nan"), device="cuda")
    Wg = W.t().contiguous() if w_trans else W
    ws = torch.empty(N * ((K + 31) // 32) * 128, device="cuda", dtype=torch.uint8)
    lib().pw_tma_fwd(A.data_ptr(), Wg.data_ptr(), w_trans, C.data_ptr(), M, N, K, _p(in_sc[0]) if in_sc is not None else 0,
                     _p(in_sc[1]) if in_sc is not None else 0, in_act if in_sc is not None else 0, _p(gate), rps,
                     _p(sc[0]) if sc is not None else 0, _p(sc[1]) if sc is not None else 0, act, _p(R),
                     _p(st[0]) if st is not None else 0, _p(st[1]) if st is not None else 0, ws.data_ptr(), ws.numel(),
                     torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    ref, raw = _ref(A, W, in_sc, in_act, gate, rps, sc, act, R)
    tag = f"M={M} N={N} K={K} w_trans={w_trans} in_act={in_act} gate_rps={gate_rps} epi={epi} act={act} res={res}"
    assert torch.isfinite(C).all(), f"{tag}: output columns left unwritten"
    err = (C.double() - ref).abs().max().item() / (ref.abs().max().item() + 1e-6)
    assert err < 2e-4, f"{tag}: rel err {err}"
    if st is not None:
        for got, want in ((st[0], raw.sum(0)), (st[1], (raw * raw).sum(0))):
            serr = ((got - want).abs().max() / (want.abs().max() + 1e-6)).item()
            assert serr < 1e-3, f"{tag}: statistics rel err {serr}"


# one tile at every compiled width of the raw-output kernel (8 .. 128): the tails 8 / 16 / 24 and the full chunks
@pytest.mark.parametrize("N", list(range(8, 129, 8)))
def test_single_tile_every_width(N):
    g = torch.Generator(device="cuda").manual_seed(N)
    _run(1000, N, 40, g, stats=True)
    _run(515, N, 72, g, w_trans=1, res=True)


# several tiles of equal width: (N, K) -> tiles  136 -> 2 x 72 (tail 8), 176 -> 2 x 88 (tail 24), 200 -> 2 x 104 (tail 8),
# 184 -> 2 x 96, 240 -> 2 x 120 (tail 24), 272 -> 3 x 96 (last tile 80 wide), 480 -> 4 x 120, 672 -> 6 x 112 (tail 16),
# 960 -> 8 x 120
MULTI = [(136, 24), (176, 40), (200, 80), (184, 80), (240, 40), (272, 64), (480, 80), (672, 112), (960, 160)]


@pytest.mark.parametrize("N,K", MULTI)
def test_multi_tile_raw_statistics_and_data_gradient(N, K):
    g = torch.Generator(device="cuda").manual_seed(N + K)
    _run(2000 + 37, N, K, g, stats=True)                      # training forward: raw output + batch statistics, ragged M
    _run(1300, N, K, g, w_trans=1, res=True)                  # data gradient: transposed weights + residual
    _run(777, N, K, g, in_act=2, gate_rps=504, stats=True)    # BatchNorm + Hardswish on load, SE gate, 504 rows per sample
    _run(4100, N, K, g, in_act=1, gate_rps=2016)              # ReLU on load, SE gate, 2016 rows per sample


@pytest.mark.parametrize("N,K", [(72, 24), (200, 80), (240, 40), (960, 160)])
def test_epilogue_variants_on_the_wider_instances(N, K):
    """scale / shift / activation epilogues run on the 32 / 64 / 128-column instances (N = 200 -> 2 x 128, clipped)"""
    g = torch.Generator(device="cuda").manual_seed(7 * N + K)
    _run(1000, N, K, g, epi=True, act=2)
    _run(600, N, K, g, epi=True, res=True, gate_rps=504)


def test_mha_head_projection_width():
    """the attention-pooling head's projection: N = 4216 -> 33 x 128, K = 960 (more than 160: streamed weights)"""
    g = torch.Generator(device="cuda").manual_seed(11)
    _run(300, 4216, 960, g, epi=True)
    _run(300, 960, 4216 // 8 * 8, g, w_trans=1)


@pytest.mark.parametrize("N,K", [(200, 80), (240, 40), (176, 72), (960, 160)])
def test_dynamic_conv_multi_tile(N, K):
    """eat_pw_tma_dyn_fwd with several N tiles per sample: per-sample mixed kernels, tails, statistics, residual"""
    L = lib()
    g = torch.Generator(device="cuda").manual_seed(N * K)
    st = torch.cuda.current_stream().cuda_stream
    for w_trans in (0, 1):
        for B, rps, variant in ((3, 504, 0), (5, 130, 1), (2, 2016, 2)):
            M, nk = B * rps, 4
            A = torch.randn(M, K, device="cuda", generator=g)
            W = torch.randn(nk, N, K, device="cuda", generator=g) / K ** 0.5
            att = torch.softmax(torch.randn(B, nk, device="cuda", generator=g), 1)
            sc = res = stats = None
            act = 0
            if variant == 0:
                stats = torch.zeros(2, N, device="cuda", dtype=torch.float64)
            else:
                sc = torch.stack([torch.rand(N, device="cuda", generator=g) + 0.5, torch.randn(N, device="cuda", generator=g) * 0.1])
                act = 2 if variant == 1 else 0
                res = torch.randn(M, N, device="cuda", generator=g) if variant == 2 else None
            Wg = W.transpose(1, 2).contiguous() if w_trans else W
            C = torch.full((M, N), float("nan"), device="cuda")
            ws = torch.empty(B * N * ((K + 31) // 32) * 128, device="cuda", dtype=torch.uint8)
            L.pw_tma_dyn_fwd(A.data_ptr(), Wg.data_ptr(), att.data_ptr(), nk, w_trans, C.data_ptr(), M, N, K, rps,
                             _p(sc[0]) if sc is not None else 0, _p(sc[1]) if sc is not None else 0, act, _p(res),
                             _p(stats[0]) if stats is not None else 0, _p(stats[1]) if stats is not None else 0,
                             ws.data_ptr(), ws.numel(), st)
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
            tag = f"dyn w_trans={w_trans} B={B} rps={rps} N={N} K={K} variant={variant}"
            assert torch.isfinite(C).all(), f"{tag}: output columns left unwritten"
            err = (C.double() - ref).abs().max().item() / (ref.abs().max().item() + 1e-6)
            assert err < 2e-4, f"{tag}: rel err {err}"
            if stats is not None:
                for got, want in ((stats[0], raw.sum(0)), (stats[1], (raw * raw).sum(0))):
                    assert ((got - want).abs().max() / (want.abs().max() + 1e-6)).item() < 1e-3, tag
