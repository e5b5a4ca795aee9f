"""Gradients through the embedding and the feature maps, on the GPU.

- eat_fmap_grad_nhwc against torch: NCHW, channels-last, stride 0 on F, on T and on C, sliced views with an offset;
  fp32 and bf16 on each side; accumulate and overwrite; B in {1, 5, 37}, odd F and T down to 1, C in {8, 24, 960}.
  An fp32 result is bit-identical to torch's add, a bf16 one within 1 ulp.
- Whole networks in train(), B = 5, 2 s clips, on the simt and auto routes: mn04 (mlp head, attention head, dilated)
  and dymn04 with dyrelu_k 2 and 3, the losses of tests/fmap_grad_util.py (bce + <r, features>, bce + the 17 maps'
  terms): every parameter gradient and the spectrogram's against autograd through the fp64 oracle, with the bounds of
  the input-gradient tests (tests/test_gpu_zz_input_grad.py) for MN and bounds set by DyReLU-B's run-to-run piece
  changes for DyMN; bf16 storage with its bounds.  A planted defect (the
  oracle without block 7's term) lands outside them.
- Other loss shapes: the embedding alone (the classifier's .grad stays None), one middle block's map, a per-frame head
  on the last map's frequency mean; eval() with an input that requires grad and an embedding-distance loss.
- Safety and no regression: an in-place edit of a returned map raises; the launch lists of a plain training step, an
  eval forward and both trainers (eager and CUDA-graph captured) are the same before and after the feature ran and
  contain no eat_fmap_grad_nhwc, and their logits and features agree up to the reordering of the batch statistics'
  atomics; the maps' forward gives the same logits, and the last map's global mean is the features."""
import contextlib
import io
import zlib

import pytest
import torch
import torch.nn.functional as Fn

from efficientat_b200._lib import lib
from tests import fmap_grad_util as fu
from tests.util import golden, report

pytestmark = pytest.mark.gpu

# ------------------------------------------------------------------------------------------------ eat_fmap_grad_nhwc
DT = {"fp32": torch.float32, "bf16": torch.bfloat16}
CODE = {torch.float32: 0, torch.bfloat16: 1}
SHAPES = [(1, 1), (7, 1), (1, 9), (5, 33), (17, 3), (64, 63)]


def _src(layout, B, C, F, T, dtype, g):
    r = lambda *s: torch.randn(*s, generator=g).to(dtype).cuda()     # noqa: E731
    if layout == "nchw":
        return r(B, C, F, T)
    if layout == "channels_last":
        return r(B, F, T, C).permute(0, 3, 1, 2)
    if layout == "f0":                              # the gradient of a frequency mean
        return r(B, C, 1, T).expand(B, C, F, T)
    if layout == "t0":
        return r(B, C, F, 1).expand(B, C, F, T)
    if layout == "c0":
        return r(B, 1, F, T).expand(B, C, F, T)
    if layout == "slice_nchw":
        return r(B + 1, C + 8, F + 2, T + 3)[1:, 8:, 2:, 3:]
    if layout == "slice_cl":                        # channels fastest, at an offset that is not 16-byte aligned
        return r(B, F + 1, T, C + 3)[:, 1:, :, 3:].permute(0, 3, 1, 2)
    raise ValueError(layout)


def _fmap_grad(src, dst, acc):
    B, F, T, C = dst.shape
    lib().fmap_grad_nhwc(src.data_ptr(), CODE[src.dtype], *src.stride(), dst.data_ptr(), CODE[dst.dtype], B, C, F, T,
                         int(acc), torch.cuda.current_stream().cuda_stream)


@pytest.mark.parametrize("B", [1, 5, 37])
@pytest.mark.parametrize("C", [8, 24, 960])
@pytest.mark.parametrize("dst_dt", ["fp32", "bf16"])
@pytest.mark.parametrize("src_dt", ["fp32", "bf16"])
@pytest.mark.parametrize("layout", ["nchw", "channels_last", "f0", "t0", "c0", "slice_nchw", "slice_cl"])
def test_fmap_grad_kernel_matches_torch(layout, src_dt, dst_dt, C, B):
    g = torch.Generator().manual_seed(zlib.crc32(f"{layout} {src_dt} {dst_dt} {C} {B}".encode()))
    for F, T in SHAPES:
        if B * C * F * T > (1 << 24):
            continue
        src = _src(layout, B, C, F, T, DT[src_dt], g)
        base = torch.randn(B, F, T, C, generator=g).to(DT[dst_dt]).cuda()
        for acc in (False, True):
            dst = base.clone()
            _fmap_grad(src, dst, acc)
            want = src.permute(0, 2, 3, 1).float()
            if acc:
                want = base.float() + want
            want = want.to(DT[dst_dt])
            if dst_dt == "fp32":
                assert torch.equal(dst, want), f"{layout} {src_dt}->{dst_dt} acc {acc} B {B} C {C} F {F} T {T}"
            else:
                # 1 ulp of bf16 at the expected value
                ulp = torch.ldexp(torch.ones_like(want.float()), torch.frexp(want.float())[1] - 8)
                err = (dst.float() - want.float()).abs()
                assert bool((err <= ulp).all()), f"{layout} {src_dt}->{dst_dt} acc {acc} B {B} C {C} F {F} T {T}"


# ------------------------------------------------------------------------------------------------ whole networks
B_NET = 5
# the bounds of the training-step input-gradient tests (tests/test_gpu_zz_input_grad.py): rel L2 of the spectrogram
# gradient, of all parameter gradients together, and per parameter tensor (plus 1e-2 of the whole gradient's norm)
BOUNDS = {"simt": (1e-4, 1e-4, 2e-4), "auto": (3e-2, 3e-2, 6e-2)}
# DyMN at B = 5: where two DyReLU-B pieces nearly tie, fp32 rounding moves a pixel from one piece to the other, and the
# order of the batch statistics' atomics changes that rounding from run to run, so the simt route's error jumps between
# runs of the same code.  Measured over three runs (dymn04, dyrelu_k 2 and 3, both losses): 1.1e-5 to 3.5e-3 for the
# spectrogram, up to 3.3e-3 for all parameters, 4.4e-3 for one tensor, cos >= 0.999994.  The planted defect below lands
# at 6.2e-2 to 9.8e-2, cos 0.9974.  On the auto route: the eval-mode auto bounds of the input-gradient tests (measured
# at most 2.4e-2, cos 0.99970)
DYMN_BOUNDS = {"simt": (2e-2, 2e-2, 3e-2), "auto": (8e-2, 8e-2, 0.2)}
DYMN_SIMT_COS = 0.9995
COS_MIN = 0.998
BF16_REL, BF16_COS = 1.0, 0.5
_ORACLE = {}


def _inputs():
    spec, y = fu.net_inputs(batch=B_NET)
    return spec, y


def _model(tag, precision="fp32"):
    with contextlib.redirect_stdout(io.StringIO()):
        model = fu.build_model(tag, golden("fmap_grad"), precision=precision).cuda().train()
    for m in model.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    return model


def _forward(model, tag, x, kind):
    """-> (logits, features or None, maps or None) through the reference's public calls"""
    if kind == "fmaps":
        if fu.CASES[tag][0] == "mn":
            logits, fmaps = model._forward_impl(x, return_fmaps=True)
        else:
            logits, fmaps = model(x, return_fmaps=True)
        return logits, None, fmaps
    logits, feat = model(x)
    return logits, feat, None


def _oracle(tag, kind, skip=()):
    key = (tag, kind, skip)
    if key not in _ORACLE:
        model = fu.build_model(tag, golden("fmap_grad"))
        spec, y = _inputs()
        _, dx, grads = fu.oracle_grads(tag, model, kind, spec, y, skip=skip, device="cuda")
        _ORACLE[key] = dx, grads
    return _ORACLE[key]


def _engine_grads(tag, kind, route, precision="fp32"):
    model = _model(tag, precision)
    model.engine().gemm_impl = "simt" if route == "simt" else "auto"
    spec, y = _inputs()
    x = spec.cuda().requires_grad_(True)
    logits, feat, fmaps = _forward(model, tag, x, kind)
    if kind == "fmaps":
        assert len(fmaps) == 17
        r, R = fu.probes((B_NET, fmaps[-1].shape[1]), [m.shape for m in fmaps], torch.float32)
    else:
        r, R = fu.probes(feat.shape, [], torch.float32)
    fu.loss(kind, logits, feat, fmaps, y.cuda(), r.cuda(), [t.cuda() for t in R]).backward()
    return x.grad.double().cpu(), {n: p.grad.double().cpu() for n, p in model.named_parameters()}


def _rel(a, b):
    return ((a - b).norm() / b.norm()).item(), Fn.cosine_similarity(a.flatten(), b.flatten(), dim=0).item()


def _check(what, tag, route, precision, dx, grads, ref):
    rdx, rgrads = ref
    ex, cx = _rel(dx, rdx)
    names = sorted(rgrads)
    g_all = torch.cat([grads[n].flatten() for n in names])
    r_all = torch.cat([rgrads[n].flatten() for n in names])
    ea, ca = _rel(g_all, r_all)
    floor = 1e-2 * r_all.norm().item()
    worst = max(((grads[n] - rgrads[n]).norm().item() / (rgrads[n].norm().item() + floor), n) for n in names)
    report(f"fmap grad {what} {tag} {route} {precision}: dx rel {ex:.2e} cos {cx:.8f}; params rel {ea:.2e} cos {ca:.8f};"
           f" worst tensor {worst[0]:.2e} ({worst[1]})")
    if precision == "bf16":
        assert ex < BF16_REL and cx > BF16_COS, f"spectrogram gradient rel {ex:.2e} cos {cx:.6f}"
        assert bool(torch.isfinite(g_all).all())
        return
    if tag.startswith("dymn"):
        (bx, ball, bt), cmin = DYMN_BOUNDS[route], DYMN_SIMT_COS if route == "simt" else COS_MIN
    else:
        (bx, ball, bt), cmin = BOUNDS[route], COS_MIN
    assert ex < bx and cx > cmin, f"spectrogram gradient rel {ex:.2e} cos {cx:.6f}"
    assert ea < ball and ca > cmin, f"parameter gradients rel {ea:.2e} cos {ca:.6f}"
    assert worst[0] < bt, f"{worst[1]}: rel {worst[0]:.2e}"


@pytest.mark.parametrize("route", ["simt", "auto"])
@pytest.mark.parametrize("kind", fu.LOSSES)
@pytest.mark.parametrize("tag", list(fu.CASES))
def test_embedding_and_fmap_gradients_match_fp64(tag, kind, route):
    dx, grads = _engine_grads(tag, kind, route)
    _check(kind, tag, route, "fp32", dx, grads, _oracle(tag, kind))


@pytest.mark.parametrize("kind", fu.LOSSES)
@pytest.mark.parametrize("tag", ["mn04_mha", "dymn04_k2"])
def test_bf16_storage(tag, kind):
    dx, grads = _engine_grads(tag, kind, "auto", precision="bf16")
    _check(kind, tag, "auto", "bf16", dx, grads, _oracle(tag, kind))


@pytest.mark.parametrize("tag", ["mn04", "dymn04_k2"])
def test_planted_dropped_block7_map_is_caught(tag):
    dx, grads = _engine_grads(tag, "fmaps", "simt")
    with pytest.raises(AssertionError):
        _check("fmaps planted", tag, "simt", "fp32", dx, grads, _oracle(tag, "fmaps", skip=(7,)))


# ------------------------------------------------------------------------------------------------ loss shapes
def _custom(tag, loss_fn, route="simt", mode="train"):
    """engine vs fp64 oracle for loss_fn(logits, feat, fmaps) (fmaps requested in train())"""
    model = _model(tag)
    model.engine().gemm_impl = route
    model.train(mode == "train")
    spec, y = _inputs()
    x = spec.cuda().requires_grad_(True)
    if mode == "train":
        logits, feat, fmaps = _forward(model, tag, x, "fmaps")
    else:
        logits, feat = model(x)
        fmaps = None
    loss_fn(logits, feat, fmaps).backward()
    grads = {n: (p.grad.double().cpu() if p.grad is not None else None) for n, p in model.named_parameters()}
    ref_model = fu.build_model(tag, golden("fmap_grad"))
    _, rdx, rgrads = fu.oracle_grads(tag, ref_model, None, spec, y, training=mode == "train", device="cuda",
                                     loss_fn=loss_fn)
    return model, x.grad.double().cpu(), grads, rdx, rgrads


def test_embedding_alone_leaves_the_classifier_out():
    model = _model("mn04")
    spec, _ = _inputs()
    logits, feat = model(spec.cuda())
    assert feat.grad_fn is not None
    r, _ = fu.probes(feat.shape, [], torch.float32)
    (feat * r.cuda()).sum().backward()
    assert all(p.grad is None for p in model.classifier.parameters())
    assert all(p.grad is not None for n, p in model.named_parameters() if not n.startswith("classifier"))
    ref = fu.oracle_grads("mn04", fu.build_model("mn04", golden("fmap_grad")), None, spec, None, device="cuda",
                          loss_fn=lambda lo, fe, m: (fe * r.double().cuda()).sum())[2]
    names = [n for n in ref if not n.startswith("classifier")]
    got = torch.cat([model.get_parameter(n).grad.double().cpu().flatten() for n in names])
    want = torch.cat([ref[n].flatten() for n in names])
    e, c = _rel(got, want)
    report(f"fmap grad embedding alone mn04 simt: params rel {e:.2e} cos {c:.8f}")
    assert e < 3e-2 and c > COS_MIN        # auto route by default


@pytest.mark.parametrize("tag", ["mn04", "dymn04_k2"])
def test_single_middle_map_and_per_frame_head(tag):
    g = torch.Generator().manual_seed(77)
    W = None

    def middle(lo, fe, m):
        return (m[7] * m[7]).mean()

    def per_frame(lo, fe, m):
        nonlocal W
        fr = m[-1].mean(2).transpose(1, 2)                  # [B, T, C]: frequency mean, one vector per frame
        if W is None:
            W = torch.randn(10, fr.shape[-1], generator=g) * 0.1
        return Fn.binary_cross_entropy_with_logits(fr @ W.to(fr).T, torch.full(fr.shape[:2] + (10,), 0.3).to(fr))

    for name, fn in (("block 7 map", middle), ("per-frame head", per_frame)):
        _, dx, grads, rdx, rgrads = _custom(tag, fn)
        reached = {n for n, v in rgrads.items() if v is not None}
        grads = {n: grads[n] if grads[n] is not None else torch.zeros_like(rgrads[n]) for n in reached}
        rgrads = {n: rgrads[n] for n in reached}
        if name == "per-frame head":
            # the frequency mean's gradient is constant along F, and the last BatchNorm's backward subtracts its
            # per-channel mean: a cancellation that amplifies fp32 rounding.  Measured on the simt route: mn04 2.7e-3,
            # 2.0e-3, 3.6e-3 (cos 0.999996); dymn04 9.2e-4, 8.1e-4, 1.9e-3
            e, c = _rel(dx, rdx)
            ea, ca = _rel(torch.cat([grads[n].flatten() for n in sorted(reached)]),
                          torch.cat([rgrads[n].flatten() for n in sorted(reached)]))
            report(f"fmap grad {name} {tag} simt fp32: dx rel {e:.2e} cos {c:.8f}; params rel {ea:.2e} cos {ca:.8f}")
            assert e < 1e-2 and ea < 1e-2 and min(c, ca) > 0.9999
            continue
        _check(name, tag, "simt", "fp32", dx, grads, (rdx, rgrads))


def test_eval_embedding_distance_with_input_grad():
    """a frozen tagger in eval(): distance of the embedding to a target embedding, gradient to the spectrogram"""
    model = _model("mn04").eval()
    model.engine().gemm_impl = "simt"
    for p in model.parameters():
        p.requires_grad_(False)
    spec, _ = _inputs()
    target = torch.randn(B_NET, model.classifier[2].in_features, generator=torch.Generator().manual_seed(8)) * 0.1
    x = spec.cuda().requires_grad_(True)
    _, feat = model(x)
    assert feat.grad_fn is not None
    ((feat - target.cuda()) ** 2).sum().backward()
    _, rdx, _ = fu.oracle_grads("mn04", fu.build_model("mn04", golden("fmap_grad")), None, spec, None, training=False,
                                device="cuda", loss_fn=lambda lo, fe, m: ((fe - target.double().cuda()) ** 2).sum())
    e, c = _rel(x.grad.double().cpu(), rdx)
    report(f"fmap grad eval embedding distance mn04 simt: dx rel {e:.2e} cos {c:.8f}")
    # the buffers are calibrated on another batch, so the eval net amplifies its input's rounding: the bound of the
    # waveform-to-frozen-mn04 test in tests/test_gpu_zz_input_grad.py
    assert e < 3e-2 and c > 0.9995
    assert all(p.grad is None for p in model.parameters())


# ------------------------------------------------------------------------------------------------ safety, no regression
def test_in_place_edit_of_a_returned_map_raises():
    model = _model("mn04")
    logits, fmaps = model._forward_impl(_inputs()[0].cuda(), return_fmaps=True)
    with pytest.raises(RuntimeError):
        fmaps[5].mul_(2.0)
        (logits.sum() + fmaps[5].sum()).backward()


class _Recorder:
    """records the names of the C-ABI entry points called while active"""

    def __init__(self):
        self.L, self.calls, self.saved = lib(), [], {}

    def __enter__(self):
        for name in self.L.protos:
            short = name[4:]
            fn = getattr(self.L, short)
            self.saved[short] = fn

            def wrap(*a, _fn=fn, _n=short):
                self.calls.append(_n)
                return _fn(*a)
            setattr(self.L, short, wrap)
        return self

    def __exit__(self, *exc):
        for short, fn in self.saved.items():
            setattr(self.L, short, fn)


def _plain_runs(model, spec):
    """a training step, an eval forward and the trainers' steps (eager, CUDA graph) -> (launch lists, outputs)"""
    from efficientat_b200.models.preprocess import AugmentMelSTFT
    from efficientat_b200.synth import synth_labels, synth_waveform
    from efficientat_b200.train import AudioSetTrainer
    runs, outs = {}, {}
    with _Recorder() as rec:
        model.train()
        logits, feat = model(spec)
        (logits * 1.0).sum().backward()
        torch.cuda.synchronize()
    runs["train"], outs["train"] = rec.calls, (logits.detach().clone(), feat.detach().clone())
    model.zero_grad(set_to_none=True)
    with _Recorder() as rec:
        model.eval()
        with torch.no_grad():
            logits, feat = model(spec)
        torch.cuda.synchronize()
    runs["eval"], outs["eval"] = rec.calls, (logits.clone(), feat.clone())
    model.train()
    for graph in (False, True):
        with contextlib.redirect_stdout(io.StringIO()):
            mel = AugmentMelSTFT(freqm=0, timem=0, fmin_aug_range=1, fmax_aug_range=1).cuda()
        tr = AudioSetTrainer(model, mel, lr=0.0, mixup_alpha=0.3, cuda_graph=graph)
        wave = synth_waveform(4, 32000, seed=3).cuda()
        y = synth_labels(4, 527, seed=4).cuda()
        with _Recorder() as rec:
            tr.step(wave, y, perm=torch.arange(4), lam=torch.ones(4))
            torch.cuda.synchronize()
        runs["trainer_graph" if graph else "trainer"] = rec.calls
        tr.close()
    model.zero_grad(set_to_none=True)
    return runs, outs


@pytest.mark.parametrize("tag", ["mn04", "dymn04_k2"])
def test_launches_and_values_without_the_new_outputs_are_unchanged(tag):
    model = _model(tag)
    spec = _inputs()[0].cuda()
    state = {k: v.clone() for k, v in model.state_dict().items()}
    _plain_runs(model, spec)                        # host-only launch-plan queries are asked once per shape
    model.load_state_dict(state)
    before, out_b = _plain_runs(model, spec)
    for k, calls in before.items():
        assert "fmap_grad_nhwc" not in calls and calls, k
    # the feature: maps and embedding with a loss on them
    model.load_state_dict(state)
    model.train()
    logits, fmaps = _forward(model, tag, spec, "fmaps")[::2]
    (logits.sum() + sum(m.float().mean() for m in fmaps)).backward()
    logits, feat = model(spec)
    (feat.sum() + logits.sum()).backward()
    model.zero_grad(set_to_none=True)
    model.load_state_dict(state)
    after, out_a = _plain_runs(model, spec)
    assert after == before
    # the same launches on the same state; the atomics of the batch statistics and of DyMN's per-sample reductions may
    # reorder between two runs: measured at most 7.5e-6 (mn04) and 4.6e-5 (dymn04) of max(1, |output|)
    for k in out_b:
        for a, b in zip(out_a[k], out_b[k]):
            d = (a - b).abs().max().item() / max(1.0, b.abs().max().item())
            report(f"fmap grad no-regression {tag} {k}: max diff {d:.2e}")
            assert d <= 2e-4, k
    # the maps' forward gives the same logits, and the last map's global mean is the features
    model.load_state_dict(state)
    model.train()
    logits, _, fmaps = _forward(model, tag, spec, "fmaps")
    ref_logits, ref_feat = out_b["train"]
    assert (logits.detach() - ref_logits).abs().max().item() <= 2e-4 * max(1.0, ref_logits.abs().max().item())
    feat = fmaps[-1].detach().float().mean((2, 3))
    assert (feat - ref_feat).abs().max().item() <= 2e-4 * max(1.0, ref_feat.abs().max().item())
