"""The DyMN-only kernels in the launch regime the benchmark runs them in (bench.py --model dymn10 | dymn20: B = 256 and
128 clips of 10 s, 128 mel bins x 1000 frames), and whole-network DyMN checks at large batch.  At the small batches of
test_gpu_zz_dymn_kernels.py and test_gpu_zz_dyrelu_k.py every thread of the element-wise DyReLU-B and ContextGen
kernels takes at most one vector, the 5x5 tile kernel gives every CTA one tile, and the DynamicConv gradient mixes run at
most three four-sample trips; here the grid-stride walks go round ~100 times, one CTA walks all of a sample's tiles with
one set of DyReLU-B coefficients, and the weight-gradient mix chains 256 samples.  The layer shapes come from the model
(oracle.net_oracle.block_table, dymn_context_dim); the CPU test below asserts what each case reaches, with eat_dw_plan
for the depthwise kernels and the launchers' grid formulas (restated, source line cited) for the others.

Every kernel result is compared with a float64 torch restatement of the same expression, built in slices of <= 32
samples; inputs are realistic (theta, ca_f, ca_t sigmoid outputs; attention a softmax at temperatures 30 and 1;
DyReLU-B pixels kept away from the kink of the max, as the small-batch tests do).  Bounds:
  - per-output results: |error| <= rel |ref| + c * (magnitude of the output's terms), rel = 1e-6 for fp32 storage and one
    bf16 rounding (2^-8) for bf16 storage, c = 1e-6 (1e-5 for the k*k-term depthwise outputs) -- the bounds of
    test_gpu_zz_dymn_kernels.py; more is a defect, not rounding;
  - long sums: |error| <= SUM_ULPS * 2^-24 * sum |terms| per sum, SUM_ULPS = 64, except where the kernel's fixed
    summation order makes that unreachable by argument (stated at the bound);
  - the variance eat_bn_finalize derives from the depthwise training forward's statistics, on an output with mean >> std,
    within 2x of torch.var_mean in fp32 (tests/util.py: bn_variance_check).
Every case reports its worst error / bound; peak device memory is asserted below 8 GiB.
Measured on an H100 80GB HBM3 at 700 W: the 106 GPU tests of this file run in 71 s, including the plain fp32 oracle
runs on the host CPU that the whole-network bounds use (so the figure depends on the host).

Whole network: dymn10 eval at B = 256 x 1000 frames against the fp64 oracle (exact-fp32 route and the default route),
and batch independence (the same clips at B = 4 agree with the B = 256 run); one dymn10 training step at B = 128 x 101
frames against autograd through the fp64 oracle on every route of the B = 5 test.  The B = 5 bounds are widened by the
error plain fp32 torch itself makes on the same clip or tensor and capped (see K_ROUTE); a sample-index defect planted in
the oracle at B = 128 lands >= 20x outside the bounds applied.

Without a GPU, test_bounds_see_planted_defects plants defects a large-batch walk could have in the fp64 reference of one
regime case each (theta or ca_t read from sample b + 1, a 32-column block missing from dcoef, the last four-sample trip of
dyn_wgrad_mix dropped, a tile skipped by the tile walk, a tie given to the highest DyReLU-B piece); each lies >= 20x
outside the bound the GPU test applies.
"""
import pytest
import torch
import torch.nn.functional as Fn

from efficientat_b200._lib import lib
from oracle import net_oracle as no
from tests import dymn_util as du
from tests.steady_util import (C_PROD, SMS, SUM_ULPS, U, check_prod, chunks, dc, dw_plan as _dw_plan, fwd_operands,
                               tma_plan, ulps, wgrad_ref)
from tests.util import bn_variance_check, build_model, report

RELU, HS = 1, 2
F32, BF16 = 0, 1
DT = {F32: torch.float32, BF16: torch.bfloat16}
BF16_REL = 2.0 ** -8
CHUNK = 32                        # samples per fp64 reference slice
EPS = 1e-3                        # nn.BatchNorm2d(eps=1e-3), dy_block.py
GIB = 2.0 ** 30
B_BENCH, B_STEP = 256, 128        # bench.py's default batch; the B = 128 training step of the launch trace


def _st():
    return torch.cuda.current_stream().cuda_stream


def _gen(seed, device="cuda"):
    return torch.Generator(device=device).manual_seed(seed)


def _cdiv(a, b):
    return -(-a // b)


# ------------------------------------------------------------------------------------------------ shapes from the model
def _layers(width):
    """every DyMN layer at 128 mel bins x 1000 frames (stem output 64 x 500): input / output F x T, channels, kernel,
    stride and ContextGen dimension H"""
    F, T = 64, 500
    out = []
    for i, r in enumerate(no.block_table(width)):
        k, s = r["k"], r["stride"]
        Fo, To = (F + 2 * ((k - 1) // 2) - k) // s + 1, (T + 2 * ((k - 1) // 2) - k) // s + 1
        out.append(dict(i=i, Fi=F, Ti=T, Fo=Fo, To=To, cin=r["cin"], cexp=r["cexp"], cout=r["cout"], k=k, s=s,
                        H=no.dymn_context_dim(r["cexp"], width)))
        F, T = Fo, To
    return out


D10, D20 = _layers(1.0), _layers(2.0)


def _distinct(items, key):
    seen, out = set(), []
    for it in items:
        if key(it) not in seen:
            seen.add(key(it))
            out.append(it)
    return out


def _act_shape(l):
    return l["Fo"], l["To"], l["cexp"]


def _dw_key(l):
    return l["Fi"], l["Ti"], l["cexp"], l["k"], l["s"]


# (tag, B, layer, M, dtype) of eat_dy_act_fwd_m / _bwd_m: M = 2 at every dymn10 layer shape, M = 1, 3, 4 at blocks 0, 1, 13
ACT_CASES = ([("dymn10", B_BENCH, l, 2, dt) for l in _distinct(D10, _act_shape) for dt in (F32, BF16)]
             + [("dymn10", B_BENCH, D10[i], M, dt) for i in (0, 1, 13) for M in (1, 3, 4) for dt in (F32, BF16)])
# eat_dw_conv_fwd_dy_m, eval epilogue: dymn10 at B = 256 (3x3: slide kernel, 5x5: tile kernel), dymn20 layers 12-14 at
# B = 128, M = 1..4 on dymn10 layer 4
DW_EVAL = ([("dymn10", B_BENCH, l, 2) for l in _distinct(D10, _dw_key)]
           + [("dymn20", B_STEP, l, 2) for l in _distinct(D20[12:], _dw_key)]
           + [("dymn10", B_BENCH, D10[4], M) for M in (1, 3, 4)])
DW_TRAIN = [("dymn10", B_BENCH, D10[i]) for i in (1, 3, 4, 13)]           # 3x3 s2, 5x5 s2 / s1, C = 960
CTX = _distinct(D10, lambda l: (l["Fi"], l["Ti"], l["cin"]))              # ContextGen inputs
# eat_seq_pool: (Ltot, row0, L, H, stride) of the step, frequency and time halves of every layer's joint sequence
SEQ = sorted({(l["Fi"] + l["Ti"], r0, n, l["H"], l["s"]) for l in D10 for r0, n in ((0, l["Fi"]), (l["Fi"], l["Ti"]))})
ATT = sorted({(l["H"], l["cexp"], l["k"]) for l in D10 + D20})            # (H, C, ksize) of the attention / mix
WMIX_N = sorted({max(l["cexp"] * l["cout"] for l in D10), max(l["cexp"] * l["cout"] for l in D20),
                 max(l["cexp"] * l["k"] ** 2 for l in D10)})
# the 1x1 DynamicConvs of dymn10 at 32,000 and 8,000 rows per sample: (name, rows per sample, N, K)
PW_DYN = [(f"l{l['i']}_{w}", rps, n, kk) for l in D10
          for w, rps, n, kk in (("exp", l["Fi"] * l["Ti"], l["cexp"], l["cin"]), ("proj", l["Fo"] * l["To"], l["cout"], l["cexp"]))
          if rps in (32000, 8000) and not (w == "exp" and l["cexp"] == l["cin"])]


def _ids(cases):
    return [f"{c[0]}_B{c[1]}_l{c[2]['i']}_M{c[3]}" + ("" if len(c) == 4 else ("_bf16" if c[4] else "_f32")) for c in cases]


# ------------------------------------------------------------------------------------------------ the launch regime
def _ew_grid(B, nvec):
    """grid.x of dy_act_fwd_launch (dymn_kernels.cu:453) and eat_ctx_pool_bwd (dymn_kernels.cu:660): min(132 * 8 / B + 1,
    vectors / 256) CTAs per sample, 256 threads, one 4-channel vector per thread and trip"""
    return max(1, min(SMS * 8 // max(B, 1) + 1, _cdiv(nvec, 256)))


def _ew_trips(B, F, T, C):
    nvec = F * T * (C // 4)
    return _cdiv(nvec, _ew_grid(B, nvec) * 256)


def test_cases_reach_the_steady_state():
    # element-wise DyReLU-B forward (output shapes) and ContextGen backward (input shapes): grid-stride trips per thread
    fwd = {l["i"]: _ew_trips(B_BENCH, *_act_shape(l)) for l in D10}
    bwd = {l["i"]: _ew_trips(B_BENCH, l["Fi"], l["Ti"], l["cin"]) for l in CTX}
    report(f"[plan] dymn10 B={B_BENCH}: dy_act_fwd trips per thread by layer {fwd}; ctx_pool_bwd {bwd}")
    assert _ew_grid(B_BENCH, 64 * 500 * 4) == 5 and fwd[0] >= 100 and fwd[1] >= 100 and max(bwd.values()) >= 100
    # dy_act_bwd (dymn_kernels.cu:465): grid (C / 32 x To / 32, B), each thread walks Fo rows; dcoef of a (b, c) sums
    # Fo * To pixels
    assert max(l["Fo"] * l["To"] for l in D10) == 32000 and max(l["Fo"] for l in D10) == 64
    # slide kernel, eval with the per-sample DyReLU-B epilogue (kind 0, per_sample = 1)
    slide = []
    for t, B, l, M in _distinct(DW_EVAL, lambda c: (c[0], c[1], c[2]["i"])):
        if l["k"] == 3:
            for dt in (F32, BF16):
                pl = _dw_plan(0, dt, B, l["Fi"], l["Ti"], l["cexp"], 3, l["s"], per_sample=1)
                slide.append(pl["per_slot"])
                report(f"[plan] dw slide eval {t} l{l['i']} B={B} {'bf16' if dt else 'f32'}: {pl['per_slot']:.1f} units "
                       f"per thread slot, {pl['groups']} CTA groups, segments of {pl['seg']} rows of {pl['rows']}")
    assert max(slide) >= 4
    # tile kernel (kind 4), every 5x5 eval layer: each CTA walks several tiles with one set of DyReLU-B coefficients
    for t, B, l, M in _distinct(DW_EVAL, lambda c: (c[0], c[1], c[2]["i"])):
        if l["k"] == 5:
            pl = _dw_plan(4, F32, B, l["Fi"], l["Ti"], l["cexp"], 5, l["s"])
            per_cta = _cdiv(pl["tiles"], pl["groups"])
            report(f"[plan] dw tile eval {t} l{l['i']} B={B}: {pl['chunks']} channel chunks, {pl['tiles']} tiles, "
                   f"{pl['groups']} CTAs per chunk and sample, {per_cta} tiles per CTA")
            assert per_cta >= 2 or pl["tiles"] == 1, (t, l, pl)        # 4 x 32 at stride 1 is one tile
            if t == "dymn20":
                assert pl["chunks"] >= 40, (t, l, pl)
    l3 = _dw_plan(4, F32, B_BENCH, D10[3]["Fi"], D10[3]["Ti"], D10[3]["cexp"], 5, 2)     # block 3: one CTA, 32 tiles
    assert (l3["tiles"], l3["groups"]) == (32, 1), l3
    # dyn_wgrad_mix (dymn_kernels.cu:377, 390): B / 4 four-sample trips, then B % 4 single samples, one fp32 chain per
    # dW entry; dyconv_att_bwd (dymn_kernels.cu:316, 319): one fp32 atomic per sample into each dWr / dbr entry
    assert (B_BENCH // 4, B_BENCH % 4) == (64, 0) and (255 // 4, 255 % 4) == (63, 3)
    assert max(WMIX_N) == 614400 and max(h for h, _, _ in ATT) == 256
    # the 1x1 DynamicConv at 32,000 rows per sample: hundreds of M tiles per CTA
    pls = {n: tma_plan(B_STEP * rps, N, K, rps) for n, rps, N, K in PW_DYN}
    for n, pl in pls.items():
        report(f"[plan] pw_tma_dyn {n} B={B_STEP}: {pl['m_tiles']} M tiles on {pl['grid']} CTAs, up to {pl['per_cta']}")
    assert {rps for _, rps, _, _ in PW_DYN} == {32000, 8000} and max(pl["per_cta"] for pl in pls.values()) >= 100


# ------------------------------------------------------------------------------------------------ checks
def _elem(got, ref, rel, floor, what):
    """per-output: |got - ref| <= rel |ref| + floor; returns the worst error / bound"""
    err = (got.double() - ref).abs()
    bound = rel * ref.abs() + floor + 1e-300
    worst = (err / bound).max().item()
    assert worst <= 1.0, f"{what}: worst error / bound {worst:.3f}"
    return worst


def _sum(got, ref, mag, what, ulps=SUM_ULPS):
    """long sum: |got - ref| <= ulps * 2^-24 * sum |terms|; returns the worst error / bound"""
    worst = ((got.double() - ref).abs() / (ulps * U * mag + 1e-300)).max().item()
    assert worst <= 1.0, f"{what}: worst error / bound {worst:.3f} (bound {ulps} x 2^-24 sum |terms|)"
    return worst


def _peak(what):
    peak = torch.cuda.max_memory_allocated() / GIB
    assert peak < 8, f"{what}: peak device memory {peak:.2f} GiB"
    return peak


# ------------------------------------------------------------------------------------------------ DyReLU-B x CoordAtt
# p = max_m (u a_m + b_m) * ca_f * ca_t, u = z * scale + shift, (a, b) = (2 theta - 1) * lam + init (dy_block.py:157-201)
def _buffers(M, device="cuda"):
    """DyReLU-B's lambdas / init_v for M pieces (dy_block.py:149-152)"""
    return (torch.tensor([1.0] * M + [0.5] * M, device=device),
            torch.tensor([1.0] + [0.0] * (2 * M - 1), device=device))


def _coef(theta, lam, init):
    """-> coefficients [B, C, 2M] and the magnitude of their terms |2 theta - 1| lam + |init| (a slope of piece 0 with
    theta near 0 cancels in fp32, so its error is relative to that, not to its value)"""
    t = 2 * theta.double() - 1
    return t * lam.double() + init.double(), t.abs() * lam.double() + init.double().abs()


def _dy_ref(z, scale, shift, theta, lam, init, ca_f, ca_t, dp, M, tie_high=False):
    """fp64 forward and gradients of DyReLU-B x CoordAtt (closed form of autograd of the expression above: each pixel's
    gradient goes to the piece that attains the max, the lowest on a tie; tie_high: the highest), and the magnitudes of
    the terms of each result"""
    co, tm = _coef(theta, lam, init)
    u = z.double() * scale.double() + shift.double()
    a, b = co[:, None, None, :, :M], co[:, None, None, :, M:]
    lines = u.unsqueeze(-1) * a + b
    idx = (M - 1 - lines.flip(-1).argmax(-1)) if tie_high else lines.argmax(-1)
    sel = Fn.one_hot(idx, M).double()
    del lines
    r = ((u.unsqueeze(-1) * a + b) * sel).sum(-1)
    ua = u.abs()
    rmag = (ua.unsqueeze(-1) * tm[:, None, None, :, :M] + tm[:, None, None, :, M:]).amax(-1)
    slope, smag = (a * sel).sum(-1), (tm[:, None, None, :, :M] * sel).sum(-1)
    cf, ct = ca_f.double()[:, :, None, :], ca_t.double()[:, None, :, :]
    q = cf * ct
    g = dp.double()
    dr = g * q
    ga = g.abs()
    sd = dr.unsqueeze(-1) * sel
    return dict(out=r * q, m_out=rmag * q, du=dr * slope, m_du=dr.abs() * smag,
                dcaf=(g * r * ct).sum(2), m_dcaf=(ga * rmag * ct).sum(2),
                dcat=(g * r * cf).sum(1), m_dcat=(ga * rmag * cf).sum(1),
                dcoef=torch.cat([(sd * u.unsqueeze(-1)).sum((1, 2)), sd.sum((1, 2))], -1),
                m_dcoef=torch.cat([(sd.abs() * ua.unsqueeze(-1)).sum((1, 2)), sd.abs().sum((1, 2))], -1))


def _away_from_kinks(z, scale, shift, theta, lam, init, M, dtype, margin=1e-3):
    """moves every pixel whose two largest pieces lie within margin of each other (there fp32 and fp64 may pick
    different pieces and the gradient jumps), in place, slice by slice.  Where two pieces of a channel are nearly the
    same line no shift of the pixel helps: after three tries that channel's theta moves (to another value in (0, 1))"""
    if M == 1:
        return
    for b0 in range(0, z.shape[0], CHUNK):
        sl = slice(b0, b0 + CHUNK)
        for it in range(12):
            co, _ = _coef(theta[sl], lam, init)
            u = z[sl].double() * scale.double() + shift.double()
            top = (u.unsqueeze(-1) * co[:, None, None, :, :M] + co[:, None, None, :, M:]).topk(2, -1)[0]
            near = (top[..., 0] - top[..., 1]) < margin
            if not bool(near.any()):
                break
            z[sl] = torch.where(near, (z[sl].float() + 0.37).to(DT[dtype]), z[sl])
            if it >= 3:
                chan = near.any(2).any(1)                                                    # [b, C]
                theta[sl] = torch.where(chan[..., None], torch.remainder(theta[sl] + 0.29, 1.0), theta[sl])
        else:
            raise AssertionError("could not move the inputs away from the kinks")


def _dy_params(B, Fo, To, C, M, g):
    """BatchNorm affine, theta, DyReLU-B buffers and the CoordAtt gates (sigmoid outputs)"""
    d = dict(scale=torch.rand(C, device="cuda", generator=g) + 0.5, shift=torch.randn(C, device="cuda", generator=g) * 0.3,
             theta=torch.sigmoid(torch.randn(B, C, 2 * M, device="cuda", generator=g)),
             ca_f=torch.sigmoid(torch.randn(B, Fo, C, device="cuda", generator=g)),
             ca_t=torch.sigmoid(torch.randn(B, To, C, device="cuda", generator=g)))
    d["lam"], d["init"] = _buffers(M)
    return d


def _dy_inputs(B, Fo, To, C, M, dtype, g, ties=False):
    d = _dy_params(B, Fo, To, C, M, g)
    d["z"] = torch.randn(B, Fo, To, C, device="cuda", generator=g).to(DT[dtype])
    d["dp"] = torch.randn(B, Fo, To, C, device="cuda", generator=g).to(DT[dtype])
    if ties:
        # pieces (a, b) = (1, 0), (0.5, 0.25), (0.5, 0.25), (1, -0.5) in every channel, u in [-1.5, -0.5): pieces 1 and 2
        # tie at the max, 0.5 above the others; theta = 0.5, 0.75, 0.75, 1 | 0.5, 0.75, 0.75, 0 is exact in fp32
        assert M == 4
        d["theta"] = torch.tensor([0.5, 0.75, 0.75, 1.0, 0.5, 0.75, 0.75, 0.0], device="cuda").expand(B, C, 8).contiguous()
        d["scale"], d["shift"] = torch.ones(C, device="cuda"), torch.zeros(C, device="cuda")
        d["z"] = (-0.5 - torch.rand(B, Fo, To, C, device="cuda", generator=g)).to(DT[dtype])
    else:
        _away_from_kinks(d["z"], d["scale"], d["shift"], d["theta"], d["lam"], d["init"], M, dtype)
    return d


def _check_dy_act(tag, B, l, M, dtype, seed, ties=False):
    Fo, To, C = _act_shape(l)
    L = lib()
    torch.cuda.reset_peak_memory_stats()
    g = _gen(seed)
    d = _dy_inputs(B, Fo, To, C, M, dtype, g, ties)
    P = [d[n].data_ptr() for n in ("scale", "shift", "theta", "lam", "init", "ca_f", "ca_t")]
    out = torch.full_like(d["z"], float("nan"))
    L.dy_act_fwd_m(d["z"].data_ptr(), out.data_ptr(), dtype, *P, M, B, Fo, To, C, _st())
    # dcaf / dcoef accumulate onto nonzero contents, dcat / du are overwritten (prefilled with NaN)
    dcaf0 = torch.randn(B, Fo, C, device="cuda", generator=g)
    dcoef0 = torch.randn(B, C, 2 * M, device="cuda", generator=g)
    dcaf, dcoef = dcaf0.clone(), dcoef0.clone()
    dcat = torch.full((B, To, C), float("nan"), device="cuda")
    du = torch.full_like(d["z"], float("nan"))
    L.dy_act_bwd_m(d["dp"].data_ptr(), d["z"].data_ptr(), du.data_ptr(), dtype, *P, dcaf.data_ptr(), dcat.data_ptr(),
                   dcoef.data_ptr(), M, B, Fo, To, C, _st())
    rel = 1e-6 if dtype == F32 else BF16_REL
    w = dict(fwd=0.0, du=0.0, dcaf=0.0, dcat=0.0, dcoef=0.0)
    for b0 in range(0, B, CHUNK // 2):                    # M = 4 at 64 x 500: the per-piece tensors of 16 samples are 0.5 GB
        sl = slice(b0, b0 + CHUNK // 2)
        R = _dy_ref(*(d[n][sl] if d[n].shape[0] == B and d[n].dim() > 1 else d[n]
                      for n in ("z", "scale", "shift", "theta", "lam", "init", "ca_f", "ca_t", "dp")), M)
        w["fwd"] = max(w["fwd"], _elem(out[sl], R["out"], rel, 1e-6 * R["m_out"], "dy_act_fwd_m"))
        w["du"] = max(w["du"], _elem(du[sl], R["du"], rel, 1e-6 * R["m_du"], "dy_act_bwd_m du"))
        w["dcaf"] = max(w["dcaf"], _sum(dcaf[sl], dcaf0[sl].double() + R["dcaf"], dcaf0[sl].double().abs() + R["m_dcaf"],
                                        "dcaf"))
        w["dcat"] = max(w["dcat"], _sum(dcat[sl], R["dcat"], R["m_dcat"], "dcat"))
        w["dcoef"] = max(w["dcoef"], _sum(dcoef[sl], dcoef0[sl].double() + R["dcoef"],
                                          dcoef0[sl].double().abs() + R["m_dcoef"], "dcoef"))
        del R
    peak = _peak("dy_act")
    report(f"[kernel] dy_act_m {tag} l{l['i']} B={B} {Fo}x{To}x{C} M={M}{' ties' if ties else ''} "
           f"{'bf16' if dtype else 'f32'}: worst error/bound " + " ".join(f"{k} {v:.3f}" for k, v in w.items())
           + f"; peak {peak:.2f} GiB")


@pytest.mark.gpu
@pytest.mark.parametrize("case", ACT_CASES, ids=_ids(ACT_CASES))
def test_dy_act_at_the_bench_batch(case):
    tag, B, l, M, dtype = case
    _check_dy_act(tag, B, l, M, dtype, seed=l["i"] * 10 + M + 100 * dtype)


@pytest.mark.gpu
def test_dy_act_ties_go_to_the_lowest_piece_at_the_bench_batch():
    """M = 4 with pieces 1 and 2 identical at every pixel of dymn10 layer 13 at B = 256: all of dcoef goes to piece 1"""
    _check_dy_act("dymn10", B_BENCH, D10[13], 4, F32, seed=13, ties=True)


@pytest.mark.gpu
def test_coef_and_sigmoid_backward_at_the_step_n():
    """eat_dyrelu_coef_bwd_m (n = B C 2M) and eat_sigmoid_bwd (the CoordAtt gates, n = B Fo C and B To C) at every n of
    the dymn10 step at B = 128: a product of five / three factors per element, 1e-6 relative"""
    L = lib()
    g = _gen(1)
    coef_n = sorted({(B_STEP * l["cexp"] * 2 * M, M) for l in D10 for M in (1, 2, 3, 4)})
    sig_n = sorted({B_STEP * l[d] * l["cexp"] for l in D10 for d in ("Fo", "To")})
    w = [0.0, 0.0]
    for n, M in coef_n:
        lam, _ = _buffers(M)
        dc = torch.randn(n, device="cuda", generator=g)
        s = torch.sigmoid(torch.randn(n, device="cuda", generator=g))
        out = torch.full_like(s, float("nan"))
        L.dyrelu_coef_bwd_m(dc.data_ptr(), s.data_ptr(), lam.data_ptr(), out.data_ptr(), n, M, _st())
        sd = s.double()
        ref = dc.double() * lam.double().repeat(n // (2 * M)) * 2 * sd * (1 - sd)
        w[0] = max(w[0], _elem(out, ref, 1e-6, 0.0, f"dyrelu_coef_bwd_m n={n} M={M}"))
    for n in sig_n:
        dc = torch.randn(n, device="cuda", generator=g)
        s = torch.sigmoid(torch.randn(n, device="cuda", generator=g))
        out = torch.full_like(s, float("nan"))
        L.sigmoid_bwd(dc.data_ptr(), s.data_ptr(), out.data_ptr(), n, _st())
        w[1] = max(w[1], _elem(out, dc.double() * s.double() * (1 - s.double()), 1e-6, 0.0, f"sigmoid_bwd n={n}"))
    report(f"[kernel] dyrelu_coef_bwd_m n up to {max(coef_n)[0]}: worst error/bound {w[0]:.3f}; sigmoid_bwd n up to "
           f"{max(sig_n)}: {w[1]:.3f}")


# ------------------------------------------------------------------------------------------------ depthwise + epilogue
def _tables(B, C, k, g, pad=8, mean=0.0, spread=1.0):
    """per-sample tap-major tables [B, k*k, C] = sum_j att[b, j] W_j (a softmax over four banks of spread * randn / k +
    mean, dy_block.py:111-117) at a padded stride (NaN in the gaps): -> (buffer, stride, tables)"""
    kk = k * k
    W = torch.randn(4, kk, C, device="cuda", generator=g) * (spread / k) + mean
    att = torch.softmax(torch.randn(B, 4, device="cuda", generator=g), 1)
    w = torch.einsum("bj,jtc->btc", att, W)
    bstride = kk * C + pad
    buf = torch.full((B * bstride + 256,), float("nan"), device="cuda")
    buf[:B * bstride].view(B, bstride)[:, :kk * C] = w.reshape(B, kk * C)
    return buf, bstride, w


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [F32, BF16], ids=["f32", "bf16"])
@pytest.mark.parametrize("case", DW_EVAL, ids=_ids(DW_EVAL))
def test_dw_conv_dy_eval_at_the_bench_batch(case, dtype):
    """eat_dw_conv_fwd_dy_m with the eval epilogue (BN affine + DyReLU-B + CoordAtt): output prefilled with NaN, so a
    tile or unit the walk never stores fails"""
    tag, B, l, M = case
    Fi, Ti, Fo, To, C, k, s = l["Fi"], l["Ti"], l["Fo"], l["To"], l["cexp"], l["k"], l["s"]
    torch.cuda.reset_peak_memory_stats()
    g = _gen(l["i"] * 7 + M + B + dtype)
    x = torch.randn(B, Fi, Ti, C, device="cuda", generator=g).to(DT[dtype])
    buf, bstride, w = _tables(B, C, k, g)
    d = _dy_params(B, Fo, To, C, M, g)
    out = torch.full((B, Fo, To, C), float("nan"), device="cuda", dtype=DT[dtype])
    lib().dw_conv_fwd_dy_m(x.data_ptr(), buf.data_ptr(), bstride, out.data_ptr(), dtype, B, Fi, Ti, C, k, s, 0, 0, 0,
                           d["scale"].data_ptr(), d["shift"].data_ptr(), d["theta"].data_ptr(), d["lam"].data_ptr(),
                           d["init"].data_ptr(), d["ca_f"].data_ptr(), d["ca_t"].data_ptr(), M, 0, 0, _st())
    rel = 1e-6 if dtype == F32 else BF16_REL
    worst = 0.0
    for b0 in range(0, B, CHUNK):
        sl = slice(b0, b0 + CHUNK)
        xd, wd = x[sl].double(), w[sl].double()
        conv, cmag = du.conv_ps(xd, wd, k, s), du.conv_ps(xd.abs(), wd.abs(), k, s)
        del xd
        co, tm = _coef(d["theta"][sl], d["lam"], d["init"])
        u = conv * d["scale"].double() + d["shift"].double()
        umag = cmag * d["scale"].double() + d["shift"].double().abs()
        lines = u.unsqueeze(-1) * co[:, None, None, :, :M] + co[:, None, None, :, M:]
        q = d["ca_f"][sl].double()[:, :, None, :] * d["ca_t"][sl].double()[:, None, :, :]
        ref = lines.max(-1)[0] * q          # continuous in u: no kink margin needed for the forward alone
        del lines, conv
        mag = (umag.unsqueeze(-1) * tm[:, None, None, :, :M] + tm[:, None, None, :, M:]).amax(-1) * q
        # k*k fp32 products, then the epilogue: 1e-5 of the magnitude of the terms; bf16 adds one output rounding
        worst = max(worst, _elem(out[sl], ref, rel, 1e-5 * mag, f"dw_conv_fwd_dy_m eval {tag} l{l['i']}"))
        del ref, mag, cmag, umag, u, q
    peak = _peak("dw eval")
    report(f"[kernel] dw_conv_fwd_dy_m eval {tag} l{l['i']} B={B} {Fi}x{Ti}x{C} k{k} s{s} M={M} "
           f"{'bf16' if dtype else 'f32'}: worst error/bound {worst:.3f}; "
           f"peak {peak:.2f} GiB")


@pytest.mark.gpu
@pytest.mark.parametrize("case", DW_TRAIN, ids=[f"{t}_B{B}_l{l['i']}" for t, B, l in DW_TRAIN])
def test_dw_conv_dy_training_at_the_bench_batch(case):
    """eat_dw_conv_fwd_dy_m's training form: the expand BatchNorm + activation on load, per-sample tables at a padded
    stride, raw output and fp64 statistics.  Input 4 + 0.25 randn and tables mixed from banks whose taps share a mean of
    1/k against a spread of 0.1/k, so the output's mean is several times its std in every channel (E[x^2] - E[x]^2
    cancels).  The zero padding at the borders is what spreads the output: mean/std 15 at 32 x 250, 5.5 at 4 x 32 (5x5,
    every row within two of an edge); asserted, no channel below 4"""
    tag, B, l = case
    Fi, Ti, Fo, To, C, k, s = l["Fi"], l["Ti"], l["Fo"], l["To"], l["cexp"], l["k"], l["s"]
    act = RELU if l["i"] < 6 else HS
    torch.cuda.reset_peak_memory_stats()
    g = _gen(500 + l["i"])
    x = dc((B, Fi, Ti, C), g)
    buf, bstride, w = _tables(B, C, k, g, mean=1.0 / k, spread=0.1)
    isc = torch.rand(C, device="cuda", generator=g) + 0.5
    ish = torch.rand(C, device="cuda", generator=g) - 0.5
    out = torch.full((B, Fo, To, C), float("nan"), device="cuda")
    stats = torch.zeros(2, C, device="cuda", dtype=torch.float64)
    lib().dw_conv_fwd_dy_m(x.data_ptr(), buf.data_ptr(), bstride, out.data_ptr(), F32, B, Fi, Ti, C, k, s, isc.data_ptr(),
                           ish.data_ptr(), act, 0, 0, 0, 0, 0, 0, 0, 2, stats[0].data_ptr(), stats[1].data_ptr(), _st())
    ref = torch.zeros(2, C, device="cuda", dtype=torch.float64)
    mag = torch.zeros_like(ref)
    worst = 0.0
    for b0 in range(0, B, CHUNK):
        sl = slice(b0, b0 + CHUNK)
        a = x[sl].double() * isc.double() + ish.double()
        xf = torch.relu(a) if act == RELU else Fn.hardswish(a)
        del a
        wd = w[sl].double()
        raw, rmag = du.conv_ps(xf, wd, k, s), du.conv_ps(xf.abs(), wd.abs(), k, s)
        del xf
        worst = max(worst, _elem(out[sl], raw, 1e-6, 1e-5 * rmag, "dw_conv_fwd_dy_m training"))
        ref += torch.stack([raw.sum((0, 1, 2)), (raw * raw).sum((0, 1, 2))])
        mag += torch.stack([rmag.sum((0, 1, 2)), (rmag * rmag).sum((0, 1, 2))])
        del raw, rmag
    del x
    w_s = _sum(stats[0], ref[0], mag[0], "stat_sum")
    w_q = _sum(stats[1], ref[1], mag[1], "stat_sq")
    report(f"[kernel] dw_conv_fwd_dy_m training {tag} l{l['i']} B={B} {Fi}x{Ti}x{C} k{k} s{s}: worst error/bound "
           f"output {worst:.3f}, stat_sum {w_s:.3f}, stat_sq {w_q:.3f}")
    n = B * Fo * To
    mstd = (ref[0] / n).abs() / (ref[1] / n - (ref[0] / n) ** 2).clamp_min(1e-30).sqrt()
    report(f"[kernel] dw_conv_fwd_dy_m training {tag} l{l['i']}: output mean/std per channel min {mstd.min().item():.1f}, "
           f"median {mstd.median().item():.1f}")
    assert mstd.min().item() >= 4, (mstd.min().item(), mstd.median().item())
    bn_variance_check(out, stats, ref, n, C, EPS, f"dw_conv_fwd_dy_m training {tag} l{l['i']}")
    report(f"[kernel] dw_conv_fwd_dy_m training {tag} l{l['i']}: peak {_peak('dw training'):.2f} GiB")


# ------------------------------------------------------------------------------------------------ ContextGen pooling
def _ctx_ref(x, tv=None):
    """[mean over t < T_b | mean over f, 0 for t >= T_b] of x [B, F, T, C] and the same of |x|"""
    B, F, T, C = x.shape
    xd = x.double()
    if tv is None:
        return (torch.cat([xd.mean(2), xd.mean(1)], 1), torch.cat([xd.abs().mean(2), xd.abs().mean(1)], 1))
    m = (torch.arange(T, device=x.device)[None, :] < tv[:, None]).double()               # [B, T]
    xm = xd * m[:, None, :, None]
    n = tv.double()[:, None, None]
    return (torch.cat([xm.sum(2) / n, xm.mean(1)], 1), torch.cat([xm.abs().sum(2) / n, xm.abs().mean(1)], 1))


@pytest.mark.gpu
@pytest.mark.parametrize("l", CTX, ids=[f"l{l['i']}_{l['Fi']}x{l['Ti']}x{l['cin']}" for l in CTX])
def test_ctx_pool_at_the_bench_batch(l):
    """eat_ctx_pool, eat_ctx_pool_len (per-clip lengths, including 1 and T) and eat_ctx_pool_bwd (added onto dx) at
    every ContextGen input shape of dymn10, B = 256.  The means: a chain of T (F) fp32 adds and one scaling each,
    SUM_ULPS * 2^-24 * the mean of |terms|; the backward: three terms per element, 1e-6 of their magnitude"""
    B, F, T, C = B_BENCH, l["Fi"], l["Ti"], l["cin"]
    L = lib()
    torch.cuda.reset_peak_memory_stats()
    g = _gen(F + T + C)
    x = torch.randn(B, F, T, C, device="cuda", generator=g)
    tv = torch.randint(1, T + 1, (B,), device="cuda", generator=g, dtype=torch.int32)
    tv[0], tv[1], tv[2] = 1, T, T - 1
    out = torch.full((B, F + T, C), float("nan"), device="cuda")
    out_len = torch.full((B, F + T, C), float("nan"), device="cuda")
    L.ctx_pool(x.data_ptr(), F32, out.data_ptr(), B, F, T, C, _st())
    L.ctx_pool_len(x.data_ptr(), F32, out_len.data_ptr(), B, F, T, C, tv.data_ptr(), _st())
    dg = torch.randn(B, F + T, C, device="cuda", generator=g)
    dx0 = torch.randn(B, F, T, C, device="cuda", generator=g)
    dx = dx0.clone()
    L.ctx_pool_bwd(dg.data_ptr(), dx.data_ptr(), F32, B, F, T, C, _st())
    w = [0.0, 0.0, 0.0]
    for b0 in range(0, B, CHUNK):
        sl = slice(b0, b0 + CHUNK)
        ref, mag = _ctx_ref(x[sl])
        w[0] = max(w[0], _sum(out[sl], ref, mag, "ctx_pool"))
        ref, mag = _ctx_ref(x[sl], tv[sl])
        w[1] = max(w[1], _sum(out_len[sl], ref, mag, "ctx_pool_len"))
        beyond = torch.arange(T, device="cuda")[None, :] >= tv[sl, None]
        assert bool((out_len[sl, F:][beyond] == 0).all()), "ctx_pool_len: time positions past the clip are not 0"
        gd, d0 = dg[sl].double(), dx0[sl].double()
        ref = d0 + gd[:, :F, None, :] / T + gd[:, None, F:, :] / F
        mag = d0.abs() + gd[:, :F, None, :].abs() / T + gd[:, None, F:, :].abs() / F
        w[2] = max(w[2], _elem(dx[sl], ref, 1e-6, 1e-6 * mag, "ctx_pool_bwd"))
        del ref, mag, gd, d0
    report(f"[kernel] ctx_pool dymn10 l{l['i']} B={B} {F}x{T}x{C}: worst error/bound fwd {w[0]:.3f} len {w[1]:.3f} "
           f"bwd {w[2]:.3f}; peak {_peak('ctx_pool'):.2f} GiB")


# ------------------------------------------------------------------------------------------------ sequence pooling
def _pool_rows(v, s):
    """AvgPool(3, s, pad 1, count_include_pad) along dim 1 of [B, L, H], or the rows themselves for s = 1"""
    if s == 1:
        return v
    Lo = (v.shape[1] - 1) // s + 1
    vp = Fn.pad(v, (0, 0, 1, 1))
    return sum(vp[:, j:j + s * (Lo - 1) + 1:s] for j in range(3)) / 3


def _pool_rows_t(dout, L_, s):
    """the transpose of _pool_rows: [B, Lo, H] -> [B, L, H]"""
    if s == 1:
        return dout
    B, Lo, H = dout.shape
    dp = torch.zeros(B, L_ + 2, H, dtype=dout.dtype, device=dout.device)
    for j in range(3):
        dp[:, j:j + s * (Lo - 1) + 1:s] += dout / 3
    return dp[:, 1:L_ + 1]


@pytest.mark.gpu
def test_seq_pool_at_the_step_shapes():
    """eat_seq_pool (with and without the joint BatchNorm + Hardswish on load) and eat_seq_pool_bwd at every
    (Ltot, row0, L, H, stride) of the dymn10 step at B = 128: at most three terms per output, 1e-6 of their magnitude
    (pre-activation magnitudes with the affine); rows outside the window keep their contents"""
    L = lib()
    B = B_STEP
    w = [0.0, 0.0]
    for Ltot, row0, L_, H, s in SEQ:
        g = _gen(Ltot + row0 + H + s)
        x = torch.randn(B, Ltot, H, device="cuda", generator=g)
        sc = torch.rand(H, device="cuda", generator=g) + 0.5
        sh = torch.randn(H, device="cuda", generator=g) * 0.3
        Lo = (L_ - 1) // s + 1
        rows = x.double()[:, row0:row0 + L_]
        for aff in (False, True):
            out = torch.full((B, Lo, H), float("nan"), device="cuda")
            L.seq_pool(x.data_ptr(), out.data_ptr(), B, Ltot, row0, L_, H, s, sc.data_ptr() if aff else 0,
                       sh.data_ptr() if aff else 0, HS if aff else 0, _st())
            v, vmag = rows, rows.abs()
            if aff:
                v = Fn.hardswish(rows * sc.double() + sh.double())
                vmag = 2 * ((rows * sc.double()).abs() + sh.double().abs())    # hardswish slope <= 1.5
            w[0] = max(w[0], _elem(out, _pool_rows(v, s), 1e-6, 1e-6 * _pool_rows(vmag, s),
                                   f"seq_pool {(Ltot, row0, L_, H, s)} aff={aff}"))
        dout = torch.randn(B, Lo, H, device="cuda", generator=g)
        dsrc = torch.full((B, Ltot, H), 12345.0, device="cuda")
        L.seq_pool_bwd(dout.data_ptr(), dsrc.data_ptr(), B, Ltot, row0, L_, H, s, _st())
        keep = torch.ones(Ltot, dtype=torch.bool, device="cuda")
        keep[row0:row0 + L_] = False
        assert bool((dsrc[:, keep] == 12345.0).all()), "seq_pool_bwd wrote outside rows [row0, row0 + L)"
        w[1] = max(w[1], _elem(dsrc[:, row0:row0 + L_], _pool_rows_t(dout.double(), L_, s), 1e-6,
                               1e-6 * _pool_rows_t(dout.double().abs(), L_, s), f"seq_pool_bwd {(Ltot, row0, L_, H, s)}"))
    report(f"[kernel] seq_pool B={B}, {len(SEQ)} windows, Ltot up to {max(c[0] for c in SEQ)}, L up to "
           f"{max(c[2] for c in SEQ)}: worst error/bound fwd {w[0]:.3f} bwd {w[1]:.3f}")


# ------------------------------------------------------------------------------------------------ DynamicConv attention
@pytest.mark.gpu
@pytest.mark.parametrize("temp", [30.0, 1.0], ids=["T30", "T1"])
def test_dyconv_attention_and_mix_at_the_bench_batch(temp):
    """eat_dyconv_att / eat_dyconv_att_bwd (256 fp32 atomics into every dWr / dbr entry) and eat_dyconv_mix_dw at
    B = 256, k = 4, for every (H, C) of dymn10 and dymn20 (H 32-256, C up to 1920)"""
    L = lib()
    B, nk = B_BENCH, 4
    w = dict(att=0.0, dWr=0.0, dbr=0.0, dh_c=0.0, mix=0.0)
    for H, C, ks in ATT:
        g = _gen(H * 10 + C + int(temp))
        hc = Fn.hardswish(torch.randn(B, H, device="cuda", generator=g))
        wr = torch.randn(nk, H, device="cuda", generator=g) / H ** 0.5 * 4
        br = torch.randn(nk, device="cuda", generator=g)
        att = torch.full((B, nk), float("nan"), device="cuda")
        L.dyconv_att(hc.data_ptr(), wr.data_ptr(), br.data_ptr(), temp, att.data_ptr(), B, H, nk, _st())
        hd, wd, bd = hc.double(), wr.double(), br.double()
        ref = torch.softmax((hd @ wd.t() + bd) / temp, -1)
        # each logit is an fp32 dot product over H: a few ulp of sum |w h|, which exp turns into a relative error of att
        lmag = (hd.abs() @ wd.abs().t() + bd.abs()) / temp
        w["att"] = max(w["att"], _elem(att, ref, 1e-6, 1e-5 * ref * lmag.amax(1, keepdim=True), f"dyconv_att H{H}"))
        datt = torch.randn(B, nk, device="cuda", generator=g)
        dwr0, dbr0, dhc0 = (torch.randn(*sh, device="cuda", generator=g) for sh in ((nk, H), (nk,), (B, H)))
        dwr, dbr, dhc = dwr0.clone(), dbr0.clone(), dhc0.clone()
        a32 = ref.float()
        L.dyconv_att_bwd(datt.data_ptr(), a32.data_ptr(), temp, hc.data_ptr(), wr.data_ptr(), dwr.data_ptr(),
                         dbr.data_ptr(), dhc.data_ptr(), B, H, nk, _st())
        a, dd = a32.double(), datt.double()
        dl = a * (dd - (a * dd).sum(1, keepdim=True)) / temp
        dl_mag = a * (dd.abs() + (a * dd.abs()).sum(1, keepdim=True)) / temp
        w["dWr"] = max(w["dWr"], _sum(dwr, dwr0.double() + dl.t() @ hd, dl_mag.t() @ hd.abs() + dwr0.double().abs(),
                                      f"dWr H{H}"))
        w["dbr"] = max(w["dbr"], _sum(dbr, dbr0.double() + dl.sum(0), dl_mag.sum(0) + dbr0.double().abs(), f"dbr H{H}"))
        w["dh_c"] = max(w["dh_c"], _sum(dhc, dhc0.double() + dl @ wd, dl_mag @ wd.abs() + dhc0.double().abs(),
                                        f"dh_c H{H}"))
        Wb = torch.randn(nk, C, ks * ks, device="cuda", generator=g)
        wt = torch.full((B, ks * ks, C), float("nan"), device="cuda")
        L.dyconv_mix_dw(Wb.data_ptr(), a32.data_ptr(), wt.data_ptr(), B, C, ks, nk, _st())
        ref = torch.einsum("bj,jct->btc", a, Wb.double())
        mag = torch.einsum("bj,jct->btc", a, Wb.double().abs())
        w["mix"] = max(w["mix"], _elem(wt, ref, 0.0, 1e-6 * mag, f"dyconv_mix_dw C{C} k{ks}"))   # four fp32 products
    report(f"[kernel] dyconv_att B={B} T={temp:g}, {len(ATT)} (H, C) pairs: worst error/bound "
           + " ".join(f"{k} {v:.3f}" for k, v in w.items()))


# ------------------------------------------------------------------------------------------------ DynamicConv bank grads
# dW[k] += sum_b att[b, k] S[b];  datt[b, k] = <S[b], W[k]>
@pytest.mark.gpu
@pytest.mark.parametrize("B", [B_STEP, B_BENCH, 255])
def test_dyn_wgrad_mix_at_the_bench_batch(B):
    """B = 128, 256: four-sample trips only; 255: 63 trips and a tail of three.  n up to dymn20's 1920 x 320"""
    L = lib()
    torch.cuda.reset_peak_memory_stats()
    nk = 4
    w = [0.0, 0.0]
    for n in WMIX_N:
        g = _gen(B + n)
        S = torch.randn(B, n, device="cuda", generator=g)
        att = torch.softmax(torch.randn(B, nk, device="cuda", generator=g) * 2, 1)
        W = torch.randn(nk, n, device="cuda", generator=g)
        dW0 = torch.randn(nk, n, device="cuda", generator=g)
        dW = dW0.clone()
        datt = torch.full((B, nk), float("nan"), device="cuda")
        L.dyn_wgrad_mix(S.data_ptr(), att.data_ptr(), W.data_ptr(), dW.data_ptr(), datt.data_ptr(), B, n, nk, _st())
        ad = att.double()
        rd = torch.zeros(B, nk, device="cuda", dtype=torch.float64)
        rm = torch.zeros_like(rd)
        for c0, c1 in chunks(n, B, 1 << 24):
            s = S[:, c0:c1].double()
            wd = W[:, c0:c1].double()
            ref = dW0[:, c0:c1].double() + ad.t() @ s
            mag = dW0[:, c0:c1].double().abs() + ad.t() @ s.abs()
            # dW: each entry is one fp32 fma chain over the B samples in sample order, then one add onto the prefill:
            # that order guarantees (B + 1) * 2^-24 * sum |terms| and no less, so the bound is the chain's length
            w[0] = max(w[0], _sum(dW[:, c0:c1], ref, mag, f"dW n{n}", ulps=B + 1))
            rd += s @ wd.t()
            rm += s.abs() @ wd.abs().t()
            del s, wd, ref, mag
        w[1] = max(w[1], _sum(datt, rd, rm, f"datt n{n}"))
        del S, W, dW, dW0
    report(f"[kernel] dyn_wgrad_mix B={B} n up to {max(WMIX_N)}: worst error/bound dW {w[0]:.3f} (bound {B + 1} x 2^-24 "
           f"sum|terms|), datt {w[1]:.3f}; peak {_peak('dyn_wgrad_mix'):.2f} GiB")


# ------------------------------------------------------------------------------------------------ 1x1 DynamicConv
@pytest.mark.gpu
@pytest.mark.parametrize("case", PW_DYN, ids=[c[0] for c in PW_DYN])
def test_pw_dyn_statistics_and_per_sample_wgrad(case):
    """dymn10's 1x1 DynamicConvs at 32,000 / 8,000 rows per sample, B = 128: eat_pw_tma_dyn_fwd's output per sample
    against fp64 (2e-4 of the sample's largest output), its statistics against fp64 sums of its own output (prefilled with NaN) and the variance eat_bn_finalize derives from them (mean/std
    4-24 per column), as test_gpu_zz_pw_steady.py; eat_pw_tc_wgrad_persample on positive operands within
    (1e-4 + SUM_ULPS * 2^-24) * sum |terms| (the bf16x3 products and one flush window, test_gpu_zz_pw_steady.py)"""
    name, rps, N, K = case
    L = lib()
    B = B_STEP
    M = B * rps
    torch.cuda.reset_peak_memory_stats()
    g = _gen(rps + N + K)
    A, W, att = fwd_operands(M, N, K, rps, g)
    C = torch.full((M, N), float("nan"), device="cuda")
    stats = torch.zeros(2, N, device="cuda", dtype=torch.float64)
    ws = torch.empty(B * N * ((K + 31) // 32) * 128, device="cuda", dtype=torch.uint8)
    L.pw_tma_dyn_fwd(A.data_ptr(), W.data_ptr(), att.data_ptr(), W.shape[0], 0, C.data_ptr(), M, N, K, rps, 0, 0, 0, 0,
                     stats[0].data_ptr(), stats[1].data_ptr(), ws.data_ptr(), ws.numel(), _st())
    del ws
    ref = torch.zeros(2, N, device="cuda", dtype=torch.float64)
    mag = torch.zeros(N, device="cuda", dtype=torch.float64)
    for m0, m1 in chunks(M, N):
        c = C[m0:m1].double()
        ref += torch.stack([c.sum(0), (c * c).sum(0)])
        mag += c.abs().sum(0)
        del c
    u_s, u_q = ulps(stats[0], ref[0], mag), ulps(stats[1], ref[1], ref[1])
    bn_variance_check(C, stats, ref, M, N, EPS, f"pw_tma_dyn fwd stats dymn10 {name}")
    assert u_s <= SUM_ULPS and u_q <= SUM_ULPS, (u_s, u_q)
    # the output itself, sample by sample against A_b . (sum_j att[b, j] W_j)^T in fp64: a tile that mixes in another
    # sample's kernel agrees with its own statistics but not with this; bf16x3 products, 2e-4 of the sample's largest
    # output (test_gpu_gemm.py)
    Wd, ad = W.double(), att.double()
    w_c = 0.0
    for b in range(B):
        want = A[b * rps:(b + 1) * rps].double() @ torch.einsum("j,jnk->nk", ad[b], Wd).t()
        w_c = max(w_c, ((C[b * rps:(b + 1) * rps].double() - want).abs().max() / (2e-4 * want.abs().max())).item())
        assert w_c <= 1.0, f"pw_tma_dyn_fwd output, sample {b}: worst error / bound {w_c:.3f}"
    del A, C
    G, X = dc((M, N), g), dc((M, K), g)
    S = torch.zeros(B, N, K, device="cuda")
    L.pw_tc_wgrad_persample(G.data_ptr(), X.data_ptr(), F32, S.data_ptr(), M, N, K, rps, _st())
    rS, mS = wgrad_ref(G, X, None, 0, None, rps, True)
    u_w = check_prod(S, rS, mS, f"S {name}")
    report(f"[kernel] pw dyn dymn10 {name} B={B} rows/sample {rps} N {N} K {K}: worst error/bound output {w_c:.3f}, "
           f"stat_sum {u_s / SUM_ULPS:.3f} stat_sq {u_q / SUM_ULPS:.3f}, per-sample S {u_w / (C_PROD / U + SUM_ULPS):.3f}; "
           f"peak {_peak('pw dyn'):.2f} GiB")


# ------------------------------------------------------------------------------------------------ whole network
# Among 256 clips of this synthetic state some amplify rounding ~100x more than the five of the B = 5 tests: there plain
# fp32 torch (TF32 off) is itself outside the B = 5 bounds (measured on an H100: eval logits 4.8e-4 on one clip against
# 1e-4; the B = 128 step's logits 3.6e-4 against 5e-5 and gradients up to 2.6e-2 against 1e-2, where fp32 torch on the
# CPU and the engine's exact route land within 1.2x of each other, median over tensors).  So every whole-network bound
# below is the B = 5 bound plus K times plain fp32's own error on the same clip, sample or tensor, the larger of fp32
# torch on the GPU and on the CPU (two summation orders: on a single tensor one can be 50x luckier than the other).  K = 4
# for the exact-fp32 route (the same arithmetic in another order: measured up to 3.6x one fp32 run on a tensor), K = 2^8
# for the tensor-core routes (their bf16x3 products carry 2^-16 relative error, 2^8 times fp32's unit roundoff, and a
# clip that amplifies fp32 rounding amplifies that as much: measured up to 100x fp32's error on one clip, 20-35x
# typically).  No bound is let past dymn_util.CAP_REL (0.5 relative L2) or CAP_LOGITS (3e-2 on a logit), so none can
# pass a zeroed or unrelated gradient; the tensors that reach the cap are reported by name, and
# test_dymn10_step_b128_bounds_see_sample_index_defects shows that the bounds actually applied see a sample-indexing slip.
K_ROUTE = {"simt": 4.0, "auto": 256.0, "auto_tma": 256.0, "auto_reg": 256.0}


@pytest.mark.gpu
def test_dymn10_eval_b256_10s_matches_fp64_oracle():
    """dymn10 eval at B = 256 x 1000 frames from the golden state with its BatchNorm buffers calibrated on the batch
    (one training-mode oracle pass with momentum 1, fp32 on the GPU: it only defines the state every side runs).  Per
    clip, logits against the fp64 oracle (GPU, chunks of 16, no grad): exact-fp32 route 1e-4 (the B = 5 eval bound),
    default route 5e-4 (the B = 5 step's tensor-core logits bound), each plus K x plain fp32's error on the clip, capped
    at CAP_LOGITS.  Four of the clips again at B = 4 through the same route and library agree with the B = 256 run to
    1e-5 of the clip's largest logit plus 4 x plain fp32's error on it: the two runs differ only in the order of fp32
    sums (the 1x1 GEMMs' tiles never straddle samples), so the exact route's K applies to both routes"""
    tag, B, frames = "dymn10", B_BENCH, 1000
    temp = du.temperature(tag)
    spec, _ = du.train_inputs(B, frames)
    model = build_model(tag)
    sd32 = {k: v.cuda() for k, v in model.state_dict().items()}
    cal = du.calibrate(sd32, spec.cuda(), 1.0, temp)
    sd32.update(cal)
    sd64 = {k: (v.double() if v.is_floating_point() else v) for k, v in sd32.items()}

    def oracle(sd, dtype, device="cuda"):
        sd = {k: v.to(device) for k, v in sd.items()}
        with torch.no_grad(), du.exact_fp32():
            return torch.cat([no.dymn_forward(sd, spec[b0:b0 + 16].to(dtype).to(device), width_mult=1.0,
                                              temperature=temp)[0] for b0 in range(0, B, 16)]).double().cpu()
    ref = oracle(sd64, torch.float64)
    e32 = torch.maximum((oracle(sd32, torch.float32) - ref).abs().amax(1),
                        (oracle(sd32, torch.float32, "cpu") - ref).abs().amax(1))
    del sd32, sd64
    torch.cuda.empty_cache()
    with torch.no_grad():
        for k, v in model.state_dict().items():
            if k in cal:
                v.copy_(cal[k])
    model = model.cuda().eval()
    pick = [0, 1, 128, 255]
    for gemm, bound in (("simt", 1e-4), ("auto", 5e-4)):
        model.engine().gemm_impl = gemm
        with torch.no_grad():
            logits = model(spec.cuda())[0].double().cpu()
            small = model(spec[pick].cuda())[0].double().cpu()
        err = (logits - ref).abs().amax(1)
        eff = (bound + K_ROUTE[gemm] * e32).clamp(max=du.CAP_LOGITS)
        capped = (eff == du.CAP_LOGITS).nonzero().flatten().tolist()
        ratio = err / eff
        ind = (small - logits[pick]).abs().amax(1) / (1e-5 * logits[pick].abs().amax(1) + K_ROUTE["simt"] * e32[pick])
        c = ratio.argmax().item()
        report(f"[parity] {tag} B={B} x {frames} frames eval gemm={gemm}: logit max-abs err {err.max().item():.2e} "
               f"(plain fp32 {e32.max().item():.2e}, median {err.median().item():.2e} / {e32.median().item():.2e}; "
               f"logits up to {ref.abs().max().item():.2e}); worst error/bound {ratio.max().item():.3f} (clip {c}: "
               f"{err[c].item():.2e}, plain fp32 {e32[c].item():.2e}); clips at the {du.CAP_LOGITS} cap {capped}; "
               f"B=4 vs B=256 worst error/bound {ind.max().item():.3f}")
        assert ratio.max().item() <= 1.0, (gemm, c, err[c].item(), e32[c].item())
        assert ind.max().item() <= 1.0, (gemm, ind)


_STEP = {}


def _step_refs():
    """the fp64 oracle step of dymn10 at B = 128 x 101 frames (GPU) and the two plain fp32 steps (GPU, CPU), cached"""
    if "dymn10" not in _STEP:
        tag = "dymn10"
        temp = du.temperature(tag)
        inputs = du.train_inputs(B_STEP, 101)
        ref = du.oracle_step(tag, temp, *inputs, device="cuda", with_eval=False)
        with du.exact_fp32():
            f32 = [du.oracle_step(tag, temp, *inputs, device=dev, with_eval=False, dtype=torch.float32)
                   for dev in ("cuda", "cpu")]
        _STEP[tag] = inputs, ref, f32
        torch.cuda.empty_cache()
    return _STEP["dymn10"]


@pytest.mark.gpu
@pytest.mark.parametrize("route", list(du.TRAIN_ROUTES))
def test_dymn10_train_step_b128_matches_fp64_oracle(route):
    """one dymn10 training step at B = 128 x 101 frames, dropout off, against autograd through the fp64 oracle on the GPU:
    loss, logits per sample, every BatchNorm running statistic and every gradient tensor, with the bounds of the B = 5
    test (test_gpu_zz_dymn_kernels.py) plus K x plain fp32's error on the same quantity, capped"""
    inputs, ref, f32 = _step_refs()
    gemm, min_rps = du.TRAIN_ROUTES[route]
    model, loss, logits = du.engine_step("dymn10", "fp32", gemm, *inputs, dyn_tma_min_rps=min_rps)
    du.check_train_step(f"dymn10 B={B_STEP} x 101 frames train", route, model, loss, logits, ref, fp32=f32,
                        k=K_ROUTE[route])


def _rolled_h_c(fn):
    """fn(x, h_c, sd, pfx, ...) called with the context of sample b + 1"""
    return lambda x, h_c, *a: fn(x, h_c.roll(-1, 0), *a)


@pytest.mark.gpu
@pytest.mark.parametrize("defect", ["theta", "attention"])
def test_dymn10_step_b128_bounds_see_sample_index_defects(defect, monkeypatch):
    """the fp64 oracle with DyReLU-B's theta (or every DynamicConv's attention) computed from sample b + 1's context, at
    the step's B = 128 x 101 frames: a kernel with that slip would sit where this oracle does, and it lands >= 20x outside
    the bounds test_dymn10_train_step_b128_matches_fp64_oracle applies on every route (the largest of relative L2 / bound
    over the gradient tensors and |logit error| / bound over the samples)"""
    inputs, ref, f32 = _step_refs()
    monkeypatch.setattr(no, "_dyrelu_b" if defect == "theta" else "_dyconv",
                        _rolled_h_c(no._dyrelu_b if defect == "theta" else no._dyconv))
    bad = du.oracle_step("dymn10", du.temperature("dymn10"), *inputs, device="cuda", with_eval=False)
    margins = {route: du.defect_margin(du.step_bounds(route, ref, f32, K_ROUTE[route]), bad["grads"], bad["logits"], ref)
               for route in du.TRAIN_ROUTES}
    report(f"[defect] dymn10 B={B_STEP} step, {defect} of sample b + 1: " +
           ", ".join(f"{r} bound x{m:.0f} ({w}; gradient tensors alone x{mg:.1f})" for r, (m, w, mg) in margins.items()))
    for r, (m, w, _) in margins.items():
        assert m >= 20, f"{defect}: the {r} bounds are only {m:.1f}x below the defect ({w})"


# ------------------------------------------------------------------------------------------------ the bounds see defects
# No GPU: each defect is planted in an fp64 reference of a regime case at a size a CPU runs in seconds, and its distance
# from the clean result, over the bound the GPU test applies, must be >= 20.
def _cpu_dy(B, Fo, To, C, M, seed, ties=False):
    g = _gen(seed, "cpu")
    lam, init = _buffers(M, "cpu")
    d = dict(z=torch.randn(B, Fo, To, C, generator=g), scale=torch.rand(C, generator=g) + 0.5,
             shift=torch.randn(C, generator=g) * 0.3, theta=torch.sigmoid(torch.randn(B, C, 2 * M, generator=g)),
             lam=lam, init=init, ca_f=torch.sigmoid(torch.randn(B, Fo, C, generator=g)),
             ca_t=torch.sigmoid(torch.randn(B, To, C, generator=g)), dp=torch.randn(B, Fo, To, C, generator=g))
    if ties:
        d["theta"] = torch.tensor([0.5, 0.75, 0.75, 1.0, 0.5, 0.75, 0.75, 0.0]).expand(B, C, 8).contiguous()
        d["scale"], d["shift"] = torch.ones(C), torch.zeros(C)
        d["z"] = -0.5 - torch.rand(B, Fo, To, C, generator=g)
    return d


def _args(d):
    return [d[n] for n in ("z", "scale", "shift", "theta", "lam", "init", "ca_f", "ca_t", "dp")]


def _ratio_elem(bad, ref, mag, rel, c):
    return ((bad - ref).abs() / (rel * ref.abs() + c * mag + 1e-300)).max().item()


def _ratio_sum(bad, ref, mag, ulps=SUM_ULPS):
    return ((bad - ref).abs() / (ulps * U * mag + 1e-300)).max().item()


def test_bounds_see_planted_defects():
    r = {}
    # theta / ca_t of sample b + 1 in the forward: dymn10 layer 1's output shape
    l = D10[1]
    d = _cpu_dy(3, *_act_shape(l), 2, 1)
    R = _dy_ref(*_args(d), 2)
    nxt = lambda t: t.roll(-1, 0)
    for what in ("theta", "ca_t"):
        bad = _dy_ref(*_args({**d, what: nxt(d[what])}), 2)
        r[f"fwd {what} of sample b + 1"] = _ratio_elem(bad["out"], R["out"], R["m_out"], 1e-6, 1e-6)
    # one 32-column block missing from dcoef (a CTA of dy_act_bwd_m dropped): layer 0, 64 x 500 x 16, the last block
    l = D10[0]
    d = _cpu_dy(2, *_act_shape(l), 2, 2)
    R = _dy_ref(*_args(d), 2)
    dp = d["dp"].clone()
    dp[:, :, 480:512] = 0
    bad = _dy_ref(*_args({**d, "dp": dp}), 2)
    dc0 = torch.randn(R["dcoef"].shape, generator=_gen(3, "cpu"), dtype=torch.float64)
    r["dcoef without one 32-column block"] = _ratio_sum(bad["dcoef"], R["dcoef"], R["m_dcoef"] + dc0.abs())
    # a tie given to the highest piece: M = 4, pieces 1 and 2 identical
    d = _cpu_dy(2, 4, 32, 64, 4, 4, ties=True)
    R = _dy_ref(*_args(d), 4)
    bad = _dy_ref(*_args(d), 4, tie_high=True)
    dc0 = torch.randn(R["dcoef"].shape, generator=_gen(5, "cpu"), dtype=torch.float64)
    r["dcoef with ties to the highest piece"] = _ratio_sum(bad["dcoef"], R["dcoef"], R["m_dcoef"] + dc0.abs())
    # dyn_wgrad_mix without its last four-sample trip, B = 256
    g = _gen(6, "cpu")
    B, n = B_BENCH, 4096
    S = torch.randn(B, n, generator=g, dtype=torch.float64)
    att = torch.softmax(torch.randn(B, 4, generator=g, dtype=torch.float64) * 2, 1)
    dW0 = torch.randn(4, n, generator=g, dtype=torch.float64)
    ref, mag = dW0 + att.t() @ S, dW0.abs() + att.t() @ S.abs()
    r["dW without the last four-sample trip"] = _ratio_sum(dW0 + att[:-4].t() @ S[:-4], ref, mag, ulps=B + 1)
    # the tile walk stopping one tile early: dymn10 layer 4 (16 x 125, C = 120, 5x5), the last tile's outputs unwritten
    l = D10[4]
    pl = _dw_plan(4, F32, 2, l["Fi"], l["Ti"], l["cexp"], 5, 1)
    assert pl["tiles"] == _cdiv(l["Fo"], 8) * _cdiv(l["To"], 32)
    g = _gen(7, "cpu")
    x = torch.randn(2, l["Fi"], l["Ti"], l["cexp"], generator=g, dtype=torch.float64)
    w = torch.randn(2, 25, l["cexp"], generator=g, dtype=torch.float64) / 5
    conv, cmag = du.conv_ps(x, w, 5, 1), du.conv_ps(x.abs(), w.abs(), 5, 1)
    bad = conv.clone()
    bad[:, 8:16, 96:128] = 0
    r["tile walk one tile short"] = _ratio_elem(bad, conv, cmag, 1e-6, 1e-5)
    report("[defect] dymn steady: " + ", ".join(f"{k} {v:.0f}x" for k, v in r.items()))
    for k, v in r.items():
        assert v >= 20, f"{k}: the bound is only {v:.1f}x below the defect"
