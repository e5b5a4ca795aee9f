"""MN's dilated tail on the GPU: the dilated depthwise entry points one by one against float64 F.conv2d(dilation=2) and
its autograd, eval parity with the reference's goldens, the training step against the fp64 oracle of
tests/dilated_util.py (with a planted defect that must land outside the bounds), the trainers and the attention head."""
import contextlib
import io

import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

from efficientat_b200._lib import lib
from tests import dilated_util as du
from tests.test_gpu_zz_mn_kernels import BOUNDS, KNEE_MARGIN, _buffer_error, _check_step, _set_route
from tests.util import fmap_digest, golden, topk_match

F32, BF16 = 0, 1
NONE, RELU, HS = 0, 1, 2
DT = {F32: torch.float32, BF16: torch.bfloat16}
EPS = 1e-3


def _st():
    return torch.cuda.current_stream().cuda_stream


def _p(t):
    return 0 if t is None else t.data_ptr()


def _act(x, act):
    return Fn.relu(x) if act == RELU else Fn.hardswish(x) if act == HS else x


def _nchw(t):
    return t.permute(0, 3, 1, 2)


def _conv(x, w, k):          # x [B, C, F, T] fp64, w [C, 1, k, k]
    return Fn.conv2d(x, w, None, 1, (k - 1) // 2 * 2, 2, x.shape[1])


# (B, F, T, C): every B in {1, 5, 37}, odd and even F and T, F = 1 and T = 1 (empty sub-grids), the mn10 10 s tail
# (8 x 63) and 2 s tail (8 x 13), C in {64, 480, 672, 960} and 1048 (fp32: 262 vectors in 3 chunks of 88, 88, 86; bf16:
# 131 vectors in 2 chunks of 66 and 65)
SHAPES = [(1, 8, 13, 64), (5, 8, 63, 672), (37, 1, 9, 480), (5, 9, 5, 960), (1, 1, 1, 64), (37, 7, 32, 64),
          (5, 2, 3, 1048), (1, 8, 63, 960), (5, 3, 1, 672)]
MODES = ["train_fwd", "eval", "dgrad", "wgrad"]


def _data(B, F, T, C, k, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, F, T, C, device="cuda", generator=g).to(DT[dtype])
    w = torch.randn(C, 1, k, k, device="cuda", generator=g) / k
    sc = 0.5 + torch.rand(2, C, device="cuda", generator=g)
    sc[1] -= 1.0
    return g, x, w, sc


def _repack(w, C, k):
    wt = torch.empty(k * k, C, device="cuda")
    lib().dw_repack(w.data_ptr(), wt.data_ptr(), C, k, _st())
    return wt


def _bound(ref, dtype, fp32_out=False):
    mag = max(ref.abs().max().item(), 1e-30)
    return mag * (2e-5 if dtype == F32 or fp32_out else 8e-3)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("k", [3, 5])
@pytest.mark.parametrize("dtype", [F32, BF16], ids=["f32", "bf16"])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "B{}_F{}_T{}_C{}".format(*s))
def test_dilated_dw_matches_fp64(shape, dtype, k, mode):
    B, F, T, C = shape
    g, x, w, sc = _data(B, F, T, C, k, dtype, seed=1000 * SHAPES.index(shape) + 100 * dtype + 10 * k + MODES.index(mode))
    wt = _repack(w, C, k)
    xd, wd = _nchw(x).double(), w.double()
    L = lib()
    if mode == "train_fwd":          # BatchNorm + activation of the expand output on load, raw output, fp64 statistics
        for act in (RELU, HS):
            out = torch.empty_like(x)
            stats = torch.zeros(2, C, device="cuda", dtype=torch.float64)
            L.dw_conv_fwd_dil(x.data_ptr(), wt.data_ptr(), out.data_ptr(), dtype, B, F, T, C, k, 1, 2, sc[0].data_ptr(),
                              sc[1].data_ptr(), act, 0, 0, 0, 0, stats[0].data_ptr(), stats[1].data_ptr(), _st())
            xin = _act(xd * sc[0].double().view(1, -1, 1, 1) + sc[1].double().view(1, -1, 1, 1), act)
            ref = _conv(xin, wd, k)
            got = _nchw(out).double()
            assert (got - ref).abs().max().item() <= _bound(ref, dtype), act
            # the statistics are of the kernel's own (unrounded) outputs: compare against the reference's, scaled
            s1, s2 = ref.sum((0, 2, 3)), (ref * ref).sum((0, 2, 3))
            tol = 2e-5 if dtype == F32 else 8e-3
            assert (stats[0] - s1).abs().max().item() <= tol * (ref.abs().sum((0, 2, 3)).max().item() + 1e-30)
            assert (stats[1] - s2).abs().max().item() <= tol * (s2.max().item() + 1e-30)
    elif mode == "eval":             # folded BatchNorm + activation epilogue, SE squeeze sums into pool
        for act in (RELU, HS):
            out = torch.empty_like(x)
            pool = torch.zeros(B, C, device="cuda")
            L.dw_conv_fwd_dil(x.data_ptr(), wt.data_ptr(), out.data_ptr(), dtype, B, F, T, C, k, 1, 2, 0, 0, 0,
                              sc[0].data_ptr(), sc[1].data_ptr(), act, pool.data_ptr(), 0, 0, _st())
            ref = _act(_conv(xd, wd, k) * sc[0].double().view(1, -1, 1, 1) + sc[1].double().view(1, -1, 1, 1), act)
            assert (_nchw(out).double() - ref).abs().max().item() <= _bound(ref, dtype), act
            pref = ref.sum((2, 3))
            tol = 2e-5 if dtype == F32 else 8e-3
            assert (pool.double() - pref).abs().max().item() <= tol * (ref.abs().sum((2, 3)).max().item() + 1e-30)
    elif mode == "dgrad":            # mirrored taps, with and without the residual-gradient add
        dz = torch.randn(B, F, T, C, device="cuda", generator=g).to(DT[dtype])
        res = torch.randn(B, F, T, C, device="cuda", generator=g).to(DT[dtype])
        xr = xd.clone().requires_grad_(True)
        _conv(xr, wd, k).backward(_nchw(dz).double())
        for r in (None, res):
            din = torch.empty_like(x)
            L.dw_conv_dgrad_dil(dz.data_ptr(), wt.data_ptr(), _p(r), din.data_ptr(), dtype, B, F, T, C, k, 1, 2, _st())
            ref = xr.grad + (0 if r is None else _nchw(r).double())
            assert (_nchw(din).double() - ref).abs().max().item() <= _bound(ref, dtype)
    else:                            # weight gradient, with and without the input transform on load
        dz = torch.randn(B, F, T, C, device="cuda", generator=g).to(DT[dtype])
        for act in (None, RELU, HS):
            dw = torch.zeros(C, 1, k, k, device="cuda")
            L.dw_conv_wgrad_dil(dz.data_ptr(), x.data_ptr(), 0 if act is None else sc[0].data_ptr(),
                                0 if act is None else sc[1].data_ptr(), act or 0, dw.data_ptr(), dtype, B, F, T, C, k, 1, 2,
                                _st())
            xin = xd if act is None else _act(xd * sc[0].double().view(1, -1, 1, 1) + sc[1].double().view(1, -1, 1, 1), act)
            wr = wd.clone().requires_grad_(True)
            _conv(xin, wr, k).backward(_nchw(dz).double())
            ref = wr.grad
            # fp32 sums of B*F*T products per tap: bounded by the sum of the products' magnitudes
            wa = wd.abs().requires_grad_(True)
            _conv(xin.abs(), wa, k).backward(_nchw(dz).double().abs())
            assert (dw.double() - ref).abs().max().item() <= 1e-5 * wa.grad.max().item() + 1e-30


# ------------------------------------------------------------------------------------------ eval parity with the goldens
@pytest.mark.gpu
@pytest.mark.parametrize("gemm", ["simt", "auto"])
@pytest.mark.parametrize("tag", list(du.CASES))
def test_eval_matches_reference_vectors(tag, gemm):
    g = golden(tag)
    model = du.build_model(tag).cuda().eval()
    model.engine().gemm_impl = gemm
    spec, _ = du.net_inputs(tag)
    with torch.no_grad():
        logits, feat = model(spec.cuda())
        _, fmaps = model._forward_impl(spec.cuda(), return_fmaps=True)
    logits, feat = logits.cpu().numpy(), feat.cpu().numpy()
    assert list(fmaps[-1].shape) == list(g["last_shape"])
    assert np.abs(logits - g["eval_logits"]).max() <= 1e-3
    assert np.abs(feat - g["eval_feat"]).max() <= 1e-3
    assert topk_match(logits, g["eval_logits"], 10, tie_tol=1e-5)
    d = fmap_digest([f.float().cpu() for f in fmaps])
    assert np.abs(d - g["eval_fmaps"]).max() < 1e-3 * max(1.0, np.abs(g["eval_fmaps"]).max())


# ------------------------------------------------------------------------------------------ training step
TAG, B_STEP, FRAMES = "mn04_dilated", 5, 201
SEED = 23            # every Hardswish pre-activation of the oracle step lies >= KNEE_MARGIN from a knee (asserted below)
_ORACLE = {}


def _inputs(B=B_STEP, frames=FRAMES):
    from efficientat_b200.synth import synth_labels, synth_waveform
    spec = synth_waveform(B, 128 * frames, seed=SEED, std=0.7).view(B, 1, 128, frames)
    return spec, synth_labels(B, 527, seed=5)


def _knee_distance(sd, spec, width):
    """smallest distance of a Hardswish pre-activation of the oracle's training forward from a knee, relative to the
    magnitude of its terms (|z scale| + |shift|), as tests/test_gpu_zz_mn_kernels.py measures it"""
    from oracle import net_oracle as no
    ob, oa = no._bn, no._act
    last, worst = {}, [float("inf"), None]

    def bn(x, sd_, pfx, training):
        out = ob(x, sd_, pfx, training)
        last.update(z=x, out=out, pfx=pfx)
        return out

    def act(x, kind):
        if kind == "HS" and last.get("out") is x:
            z, pfx = last["z"], last["pfx"]
            mean = z.mean((0, 2, 3), keepdim=True)
            s = sd[pfx + ".weight"].view(1, -1, 1, 1) / torch.sqrt(z.var((0, 2, 3), unbiased=False, keepdim=True) + EPS)
            sh = sd[pfx + ".bias"].view(1, -1, 1, 1) - mean * s
            u = z * s + sh
            r = (torch.minimum((u - 3).abs(), (u + 3).abs()) / ((z * s).abs() + sh.abs())).min().item()
            if r < worst[0]:
                worst[:] = [r, pfx]
        return oa(x, kind)
    no._bn, no._act = bn, act
    try:
        with torch.no_grad():
            du.mn_forward({k: v.clone() for k, v in sd.items()}, spec.double(), width_mult=width, dilated=True,
                          training=True)
    finally:
        no._bn, no._act = ob, oa
    return worst


def _oracle_step(undilated_blocks=()):
    key = tuple(undilated_blocks)
    if key in _ORACLE:
        return _ORACLE[key]
    width = du.CASES[TAG][0]
    model = du.build_model(TAG)
    params = [k for k, _ in model.named_parameters()]
    sd = {k: (v.double() if v.is_floating_point() else v).clone() for k, v in model.state_dict().items()}
    spec, y = _inputs()
    if not key:
        r, where = _knee_distance(sd, spec, width)
        assert r >= KNEE_MARGIN, f"a Hardswish pre-activation of {where} lies {r:.1e} from a knee"
    for k in params:
        sd[k].requires_grad_(True)
    logits, _ = du.mn_forward(sd, spec.double(), width_mult=width, dilated=True, training=True,
                              undilated_blocks=undilated_blocks)
    loss = Fn.binary_cross_entropy_with_logits(logits, y.double())
    loss.backward()
    _ORACLE[key] = dict(loss=loss.item(), logits=logits.detach(), grads={k: sd[k].grad.detach() for k in params},
                        buffers={k: v.detach().clone() for k, v in sd.items() if k not in params})
    return _ORACLE[key]


def _engine_step(route):
    model = du.build_model(TAG).cuda().train()
    _set_route(model.engine(), route)
    model.classifier[4].p = 0.0
    spec, y = _inputs()
    logits, _ = model(spec.cuda())
    loss = Fn.binary_cross_entropy_with_logits(logits, y.cuda())
    loss.backward()
    grads = {n: p.grad.detach().double().cpu() for n, p in model.named_parameters()}
    return model, loss.item(), logits.detach().double().cpu(), grads


@pytest.mark.gpu
@pytest.mark.parametrize("route", ["exact", "auto"])
def test_train_step_matches_fp64_oracle(route):
    """mn04 dilated, B = 5, 201 frames (8 x 13 in the tail), dropout off: loss, logits, every gradient and every BatchNorm
    buffer against autograd through the fp64 oracle, with the bounds of tests/test_gpu_zz_mn_kernels.py"""
    ref = _oracle_step()
    model, loss, logits, grads = _engine_step(route)
    _check_step(f"{TAG} B={B_STEP} train route={route}", BOUNDS["exact" if route == "exact" else "auto"], loss, logits,
                grads, ref, _buffer_error(model, ref))


@pytest.mark.gpu
@pytest.mark.parametrize("route", ["exact", "auto"])
def test_planted_undilated_block_is_caught(route):
    """an oracle that runs block 13 (the first dilated block) undilated and at stride 2 lands outside the bounds"""
    model, loss, logits, grads = _engine_step(route)
    wrong = _oracle_step(undilated_blocks=(13,))
    with pytest.raises(AssertionError):
        _check_step(f"{TAG} planted defect route={route}", BOUNDS["exact" if route == "exact" else "auto"], loss, logits,
                    grads, wrong)


# ------------------------------------------------------------------------------------------ trainers and the MHA head
def _trainer(cls, graph, **kw):
    from efficientat_b200.models.preprocess import AugmentMelSTFT
    model = du.build_model(TAG).cuda()
    with contextlib.redirect_stdout(io.StringIO()):
        mel = AugmentMelSTFT(freqm=0, timem=0).cuda()
    model.classifier[4].p = 0.0
    return model, cls(model, mel, cuda_graph=graph, **kw)


@pytest.mark.gpu
def test_audioset_trainer_graph_equals_eager():
    from efficientat_b200.synth import synth_labels, synth_waveform
    from efficientat_b200.train import AudioSetTrainer
    B = 5
    wave = synth_waveform(B, 64000, seed=31).cuda()
    y = synth_labels(B, 527, seed=32).cuda()
    teacher = synth_labels(B, 527, seed=33).cuda()
    perm, lam = torch.tensor([1, 2, 3, 4, 0]), torch.full((B,), 0.7)
    losses, deltas = [], []
    for graph in (False, True):
        model, tr = _trainer(AudioSetTrainer, graph, lr=4e-4, kd_lambda=0.1, mixup_alpha=0.3)
        start = tr.flat_p.detach().clone()
        losses.append([tr.step(wave, y, teacher, perm=perm, lam=lam).sum().item() for _ in range(2)])  # 2nd: a replay
        deltas.append(tr.flat_p.detach() - start)
    # the first loss is computed before any update: the same up to fp32 summation order.  Adam's first steps move each
    # parameter by about lr * sign(gradient), so noise-level gradients (atomic summation order) flip whole steps: the
    # total update is compared in relative L2, as the fine-tuning trainer tests do
    assert abs(losses[0][0] - losses[1][0]) <= 1e-6 * abs(losses[0][0])
    assert abs(losses[0][1] - losses[1][1]) <= 1e-4 * abs(losses[0][1])
    assert ((deltas[0] - deltas[1]).norm() / deltas[0].norm()).item() <= 5e-2


@pytest.mark.gpu
@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
def test_finetune_trainer_ce_step(graph):
    from efficientat_b200.finetune import FineTuneTrainer
    from efficientat_b200.synth import synth_waveform
    B = 5
    wave = synth_waveform(B, 64000, seed=41).cuda()
    y = torch.tensor([3, 1, 526, 0, 3], device="cuda")
    model, tr = _trainer(FineTuneTrainer, graph, loss="ce", lr=4e-4, mixup_alpha=0.0)
    before = tr.flat_p.detach().clone()
    losses = [tr.step(wave, y).item() for _ in range(2)]
    assert all(np.isfinite(losses)) and losses[1] < losses[0]
    assert (tr.flat_p - before).abs().max().item() > 0


def _mha_model(precision="fp32"):
    from efficientat_b200.models.mn.model import get_model
    from efficientat_b200.synth import set_bn_stats
    from tests.mha_util import HEAD, mha_state_
    torch.manual_seed(0)
    with contextlib.redirect_stdout(io.StringIO()):
        m = get_model(width_mult=0.4, dilated=True, head_type=HEAD, multihead_attention_heads=4, precision=precision,
                      verbose=False)
    mha_state_(m, 4)
    g = golden(TAG)
    return set_bn_stats(m, g["cal_rm"], g["cal_rv"])


def _mha_oracle(sd, spec, training):
    from tests.mha_util import mha_head
    C = sd["classifier.subspace_proj.weight"].shape[1]
    z = torch.zeros((), dtype=torch.float64)
    sd2 = dict(sd)
    sd2.update({"classifier.2.weight": z.expand(1, C), "classifier.2.bias": z.expand(1),
                "classifier.5.weight": z.expand(1, 1), "classifier.5.bias": z.expand(1)})
    _, _, fmaps = du.mn_forward(sd2, spec.double(), width_mult=0.4, dilated=True, training=training, return_fmaps=True)
    return mha_head(fmaps[-1], sd["classifier.subspace_proj.weight"], sd["classifier.subspace_proj.bias"],
                    sd["classifier.head_weight"], 4, 527)


@pytest.mark.gpu
def test_mha_head_on_dilated_model_eval_and_train():
    """the attention head over the dilated tail's 13 time steps (2 s clips): eval logits, and one training step (exact
    route) for loss, logits and every gradient against fp64 autograd"""
    spec, y = _inputs()
    model = _mha_model().cuda().eval()
    sd = {k: (v.double() if v.is_floating_point() else v).clone() for k, v in _mha_model().state_dict().items()}
    with torch.no_grad():
        got, _ = model(spec.cuda())
        ref = _mha_oracle(sd, spec, False)
    assert (got.double().cpu() - ref).abs().max().item() <= 1e-3
    model.train()
    _set_route(model.engine(), "exact")
    logits, _ = model(spec.cuda())
    loss = Fn.binary_cross_entropy_with_logits(logits, y.cuda())
    loss.backward()
    params = [k for k, _ in model.named_parameters()]
    for k in params:
        sd[k].requires_grad_(True)
    rlog = _mha_oracle(sd, spec, True)
    rloss = Fn.binary_cross_entropy_with_logits(rlog, y.double())
    rloss.backward()
    assert abs(loss.item() - rloss.item()) <= 2e-7 * max(1.0, rloss.item())
    assert (logits.detach().double().cpu() - rlog.detach()).abs().max().item() <= 5e-6
    gp = dict(model.named_parameters())
    bad = []
    for k in params:
        r, gg = sd[k].grad, gp[k].grad.double().cpu()
        if r.norm().item() > 1e-9 and (gg - r).norm().item() > BOUNDS["exact"]["rel"] * r.norm().item():
            bad.append(f"{k}: {(gg - r).norm().item() / r.norm().item():.2e}")
    assert not bad, "\n".join(bad)
