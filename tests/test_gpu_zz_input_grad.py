"""Gradients with respect to the input spectrogram, on the GPU, against float64 autograd.

- eat_stem_dgrad alone: stride 1 and 2, F and T down to 1, several channel counts, fp32 and bf16, B in {1, 5, 37}.
- Whole networks (mn04, mn04 with the attention head, mn04 dilated, dymn04, dymn04 with dyrelu_k=3), B = 2, 201 frames,
  a fixed random cotangent on the logits, in eval() (BatchNorm on running statistics) and train() (batch statistics),
  on the exact-fp32 (simt) and tensor-core (auto) GEMM routes: the spectrogram gradient and every parameter gradient
  (BatchNorm gamma and beta included) against autograd through the fp64 oracle.  A planted defect, the eval backward
  with batch-statistics coefficients in place of c1 = c2 = 0, must fall outside the same bounds.
- Nothing else changes: the launch sequence of an eval forward and of a training step whose input does not require
  grad, their lack of a graph, the running buffers, and no weight-gradient launch when every parameter is frozen.
Every bound is a relative L2 error plus a cosine; the worst case measured on an H100 is noted beside each."""
import contextlib
import io
import types

import pytest
import torch
import torch.nn.functional as Fn

from efficientat_b200._lib import lib
from oracle import net_oracle as no
from tests import dilated_util as du
from tests import dyrelu_util as dyu
from tests import mha_util as mu
from tests.util import build_model, golden, report

pytestmark = pytest.mark.gpu

# ------------------------------------------------------------------------------------------------ eat_stem_dgrad
HS = 2


def _act_bwd64(v):
    return torch.where(v <= -3, torch.zeros_like(v), torch.where(v < 3, (2 * v + 3) / 6, torch.ones_like(v)))


STEM_SHAPES = [(1, 1), (1, 7), (5, 1), (7, 9), (16, 33)]


@pytest.mark.parametrize("B", [1, 5, 37])
@pytest.mark.parametrize("C", [8, 16, 64])
@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
@pytest.mark.parametrize("stride", [1, 2])
def test_stem_dgrad_matches_fp64(stride, dtype, C, B):
    g = torch.Generator().manual_seed(1000 * stride + 10 * C + B)
    td = torch.float32 if dtype == "fp32" else torch.bfloat16
    for F, T in STEM_SHAPES + ([(64, 501)] if B == 1 else []):
        Fo, To = (F - 1) // stride + 1, (T - 1) // stride + 1
        dy = torch.randn(B, Fo, To, C, generator=g).to(td)
        z = (torch.randn(B, Fo, To, C, generator=g) * 2).to(td)
        scale, shift = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g)
        # Hardswish' jumps at +-3: pre-activations within 1e-3 of a knee go to 0, where fp32 and fp64 agree on the side
        knee = ((z.double() * scale.double() + shift.double()).abs() - 3).abs() < 1e-3
        z = torch.where(knee, (-shift / scale).expand_as(z).to(td), z)
        mean, invstd = torch.randn(C, generator=g) * 0.1, torch.rand(C, generator=g) + 0.5
        c1, c2 = torch.randn(C, generator=g) * 0.1, torch.randn(C, generator=g) * 0.1
        w = torch.randn(C, 1, 3, 3, generator=g)
        dev = [t.cuda().contiguous() for t in (dy, z, scale, shift, mean, invstd, c1, c2, w)]
        dx = torch.full((B, F, T), float("nan"), device="cuda")
        lib().stem_dgrad(dev[0].data_ptr(), 0 if dtype == "fp32" else 1, dev[1].data_ptr(), *[t.data_ptr() for t in dev[2:6]],
                         HS, dev[6].data_ptr(), dev[7].data_ptr(), dev[8].data_ptr(), dx.data_ptr(), B, F, T, C, stride,
                         torch.cuda.current_stream().cuda_stream)
        # fp64: dz = scale * (dy * act'(z*scale+shift) - c1 - xhat*c2), then autograd of the conv
        z64, dy64 = z.double(), dy.double()
        v = z64 * scale.double() + shift.double()
        xhat = (z64 - mean.double()) * invstd.double()
        dz = scale.double() * (dy64 * _act_bwd64(v) - c1.double() - xhat * c2.double())
        x64 = torch.zeros(B, 1, F, T, dtype=torch.float64, requires_grad=True)
        Fn.conv2d(x64, w.double(), None, stride, 1).backward(dz.permute(0, 3, 1, 2))
        ref = x64.grad[:, 0]
        err = ((dx.double().cpu() - ref).norm() / ref.norm()).item()
        # fp32 sums of at most 9*C products with an fp32 BatchNorm apply: measured worst 7.1e-8
        assert err < 1e-6, f"stride {stride} {dtype} C {C} B {B} F {F} T {T}: rel {err:.2e}"
        again = torch.empty_like(dx)
        lib().stem_dgrad(dev[0].data_ptr(), 0 if dtype == "fp32" else 1, dev[1].data_ptr(), *[t.data_ptr() for t in dev[2:6]],
                         HS, dev[6].data_ptr(), dev[7].data_ptr(), dev[8].data_ptr(), again.data_ptr(), B, F, T, C, stride,
                         torch.cuda.current_stream().cuda_stream)
        assert torch.equal(again, dx)


# ------------------------------------------------------------------------------------------------ whole networks
def _mha_oracle(sd, x, training):
    return mu.mn_mha_forward(sd, x, 0.4, 4, 527, training=training)[0]


def _temp(model):
    """the DynamicConv temperature the module holds (the oracle's default is 1)"""
    return float(model.layers[0].depth_conv.temperature)


# name -> (build the CPU model with calibrated BatchNorm buffers, fp64 oracle (model, sd, x, training) -> logits)
NETS = {
    "mn04": (lambda p: build_model("mn04", precision=p), lambda m, sd, x, tr: no.mn_forward(sd, x, 0.4, training=tr)[0]),
    "mn04_mha": (lambda p: mu.build_mha_model("mn04_h4", golden("mn_mha"), precision=p),
                 lambda m, sd, x, tr: _mha_oracle(sd, x, tr)),
    "mn04_dilated": (lambda p: du.build_model("mn04_dilated", precision=p),
                     lambda m, sd, x, tr: du.mn_forward(sd, x, 0.4, dilated=True, training=tr)[0]),
    "dymn04": (lambda p: build_model("dymn04", precision=p),
               lambda m, sd, x, tr: no.dymn_forward(sd, x, 0.4, training=tr, temperature=_temp(m))[0]),
    "dymn04_k3": (lambda p: dyu.build_model(3, precision=p),
                  lambda m, sd, x, tr: dyu.dymn_forward(sd, x, 3, training=tr, temperature=_temp(m))[0]),
}
# 2 s (101 frames) or 4 s (201 frames), as the nets' golden files.  The eval nets get BatchNorm buffers calibrated on
# this very input (the batch statistics of an fp64 training forward): with the synthetic weights and other buffers an
# eval network amplifies its input's gradient by up to 1e12 (dymn04: logits of 1e8), far beyond what fp32 can follow.
B_NET = 2
FRAMES = {"mn04": 101, "mn04_mha": 101, "mn04_dilated": 201, "dymn04": 101, "dymn04_k3": 201}
_CAL = {}


def _build(net, precision):
    model = NETS[net][0](precision)
    if net not in _CAL:
        sd = {k: (v.double() if v.is_floating_point() else v).clone() for k, v in model.state_dict().items()}
        stats, orig = {}, no._bn

        def bn(x, sd_, pfx, training):
            flat = x.transpose(0, 1).reshape(x.shape[1], -1)
            stats[pfx] = (flat.mean(1), flat.var(1, unbiased=False))
            return orig(x, sd_, pfx, True)
        no._bn = bn
        try:
            with torch.no_grad():
                NETS[net][1](model, sd, _inputs(527, FRAMES[net])[0].double(), True)
        finally:
            no._bn = orig
        _CAL[net] = stats
    bufs = dict(model.named_buffers())
    for pfx, (m, v) in _CAL[net].items():
        bufs[pfx + ".running_mean"].copy_(m.float())
        bufs[pfx + ".running_var"].copy_(v.float())
    return model


def _inputs(K, frames=101):
    from efficientat_b200.synth import synth_waveform
    spec = synth_waveform(B_NET, 128 * frames, seed=21, std=0.7).view(B_NET, 1, 128, frames)
    cot = torch.randn(B_NET, K, generator=torch.Generator().manual_seed(3))
    return spec, cot


_ORACLE = {}


def _oracle(net, mode):
    key = (net, mode)
    if key not in _ORACLE:
        model = _build(net, "fp32")
        names = [k for k, _ in model.named_parameters()]
        sd = {k: (v.double() if v.is_floating_point() else v).cuda() for k, v in model.state_dict().items()}
        for k in names:
            sd[k].requires_grad_(True)
        spec, cot = _inputs(527, FRAMES[net])
        x = spec.double().cuda().requires_grad_(True)
        logits = NETS[net][1](model, sd, x, mode == "train")
        (logits * cot.double().cuda()).sum().backward()
        _ORACLE[key] = dict(dx=x.grad.cpu(), logits=logits.detach().cpu(), grads={k: sd[k].grad.cpu() for k in names},
                            cot=cot, spec=spec)
    return _ORACLE[key]


def _engine(net, mode, route, precision="fp32", planted=False):
    with contextlib.redirect_stdout(io.StringIO()):
        model = _build(net, precision).cuda()
    model.train(mode == "train")
    for m in model.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    eng = model.engine()
    eng.gemm_impl = "simt" if route == "simt" else "auto"
    if planted:
        # the eval backward with the batch-statistics coefficients c1 = s1/count, c2 = s2/count instead of zero
        orig = type(eng)._bn_bwd_coef

        def batch_coef(self, *a):
            frozen, self._bn_frozen = self._bn_frozen, False
            try:
                return orig(self, *a)
            finally:
                self._bn_frozen = frozen
        eng._bn_bwd_coef = types.MethodType(batch_coef, eng)
    ref = _oracle(net, mode)
    x = ref["spec"].cuda().requires_grad_(True)
    logits, _ = model(x)
    (logits * ref["cot"].cuda()).sum().backward()
    grads = {n: p.grad.double().cpu() for n, p in model.named_parameters()}
    return model, logits.detach().double().cpu(), x.grad.double().cpu(), grads


def _rel(a, b):
    return ((a - b).norm() / b.norm()).item(), Fn.cosine_similarity(a.flatten(), b.flatten(), dim=0).item()


# (mode, route) -> rel L2 bound of the spectrogram gradient, of all parameter gradients together, and per parameter
# tensor (plus 1e-2 of the whole gradient's norm as a floor), fp32 storage.  Worst measured on an H100 (mn04, attention
# head, dilated, dymn04) in the comments
BOUNDS = {("eval", "simt"): (1e-4, 1e-4, 3e-4),      # 2.7e-5, 2.8e-5, 5.4e-5
          ("eval", "auto"): (8e-2, 8e-2, 0.2),       # 3.2e-2, 3.9e-2, 8.0e-2 (dymn04; MN <= 3.2e-3)
          ("train", "simt"): (1e-4, 1e-4, 2e-4),     # 1.6e-5, 1.6e-5, 3.7e-5
          ("train", "auto"): (3e-2, 3e-2, 6e-2)}     # 1.6e-2, 1.6e-2, 2.3e-2
COS_MIN = 0.998                                      # 0.99928 (dymn04 eval auto, parameters)
# dymn04 with three DyReLU-B pieces: where pieces lie close together, fp32 rounding moves pixels from one piece to another
# (see tests/test_gpu_zz_dyrelu_k.py), on every route: measured 5.9e-2, 0.105, 0.141, cos 0.9958 (eval simt).  The
# planted defect lands at 0.85 (mn04) and 0.92 (dymn04) relative, cos 0.57 and 0.41
K3_BOUNDS, K3_COS = (0.15, 0.25, 0.4), 0.99
# bf16 storage rounds every activation to 2^-8, and activations near a ReLU / Hardswish knee or a DyReLU-B tie take the
# other side: the spectrogram gradient is held to a band (measured rel 0.81, cos 0.645: dymn04 eval), every gradient to
# being finite, as tests/test_gpu_zz_dyrelu_k.py holds bf16 parameter gradients
BF16_REL, BF16_COS = 1.0, 0.5


def _check(net, mode, route, precision, dx, grads):
    ref = _oracle(net, mode)
    ex, cx = _rel(dx, ref["dx"])
    names = sorted(ref["grads"])
    g_all = torch.cat([grads[n].flatten() for n in names])
    r_all = torch.cat([ref["grads"][n].flatten() for n in names])
    ea, ca = _rel(g_all, r_all)
    floor = 1e-2 * r_all.norm().item()
    worst = max((((grads[n] - ref["grads"][n]).norm().item()) / (ref["grads"][n].norm().item() + floor), n) for n in names)
    report(f"input grad {net} {mode} {route} {precision}: dx rel {ex:.2e} cos {cx:.8f}; params rel {ea:.2e} cos {ca:.8f};"
           f" worst tensor {worst[0]:.2e} ({worst[1]})")
    if precision == "bf16":
        assert ex < BF16_REL and cx > BF16_COS, f"spectrogram gradient rel {ex:.2e} cos {cx:.6f}"
        assert bool(torch.isfinite(g_all).all())
        return
    (bx, ball, bt), cmin = (K3_BOUNDS, K3_COS) if net == "dymn04_k3" else (BOUNDS[(mode, route)], COS_MIN)
    assert ex < bx and cx > cmin, f"spectrogram gradient rel {ex:.2e} cos {cx:.6f}"
    assert ea < ball and ca > cmin, f"parameter gradients rel {ea:.2e} cos {ca:.6f}"
    assert worst[0] < bt, f"{worst[1]}: rel {worst[0]:.2e}"


@pytest.mark.parametrize("route", ["simt", "auto"])
@pytest.mark.parametrize("mode", ["eval", "train"])
@pytest.mark.parametrize("net", list(NETS))
def test_input_and_parameter_gradients_match_fp64(net, mode, route):
    model, logits, dx, grads = _engine(net, mode, route)
    _check(net, mode, route, "fp32", dx, grads)
    if mode == "eval":
        # the saving forward gives the logits of the folded eval forward
        with torch.no_grad():
            plain, _ = model(_oracle(net, mode)["spec"].cuda())
        d = (logits - plain.double().cpu()).abs().max().item() / max(1.0, plain.abs().max().item())
        report(f"saving vs folded eval forward {net} {route}: logits {d:.2e}")
        # the two forwards round differently (BatchNorm applied on load vs folded into the GEMM epilogue);
        # measured 7.3e-6 (simt) and 2.9e-4 (auto) of max(1, |logits|)
        assert d < (1e-4 if route == "simt" else 3e-3), f"eval logits differ by {d:.2e}"


@pytest.mark.parametrize("mode", ["eval", "train"])
@pytest.mark.parametrize("net", ["mn04_mha", "dymn04"])
def test_bf16_storage(net, mode):
    _, _, dx, grads = _engine(net, mode, "auto", precision="bf16")
    _check(net, mode, "auto", "bf16", dx, grads)


@pytest.mark.parametrize("net", ["mn04", "dymn04"])
def test_planted_batch_statistics_coefficients_are_caught(net):
    _, _, dx, grads = _engine(net, "eval", "simt", planted=True)
    with pytest.raises(AssertionError):
        _check(net, "eval", "simt", "fp32", dx, grads)


# ------------------------------------------------------------------------------------------------ nothing else changes
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


# launches that only produce parameter gradients; in eval the BatchNorm reduce serves only gamma and beta
WGRAD_LAUNCHES = {"gemm_simt_wgrad", "pw_tc_wgrad", "stem_wgrad", "dw_conv_wgrad", "dw_conv_wgrad_dil"}


def _plain_runs(model, spec):
    """an eval forward and a training step, input without grad -> (launches, outputs)"""
    with _Recorder() as rec:
        model.eval()
        ev, _ = model(spec)
        model.train()
        tr, _ = model(spec)
        (tr * 1.0).sum().backward()
        torch.cuda.synchronize()
    return rec.calls, ev


@pytest.mark.parametrize("net", ["mn04", "dymn04"])
def test_launches_and_graphs_without_input_grad_are_unchanged(net):
    with contextlib.redirect_stdout(io.StringIO()):
        model = NETS[net][0]("fp32").cuda()
    for m in model.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    spec = _inputs(527)[0].cuda()
    _plain_runs(model, spec)                    # host-only launch-plan queries are asked once per shape
    before, ev = _plain_runs(model, spec)
    assert ev.grad_fn is None
    # exercise the feature, then the same calls again
    model.eval()
    x = spec.clone().requires_grad_(True)
    out, _ = model(x)
    out.sum().backward()
    model.zero_grad(set_to_none=True)
    after, ev = _plain_runs(model, spec)
    assert after == before
    assert ev.grad_fn is None
    for p in model.parameters():
        p.requires_grad_(False)
    model.train()
    out, _ = model(spec)
    assert out.grad_fn is None


@pytest.mark.parametrize("mode", ["eval", "train"])
@pytest.mark.parametrize("net", ["mn04", "mn04_mha", "dymn04"])
def test_frozen_loss_runs_no_weight_gradient(net, mode):
    with contextlib.redirect_stdout(io.StringIO()):
        model = NETS[net][0]("fp32").cuda()
    model.train(mode == "train")
    for p in model.parameters():
        p.requires_grad_(False)
    bufs = {k: v.clone() for k, v in model.state_dict().items() if not k.endswith(("weight", "bias"))}
    x = _inputs(527)[0].cuda().requires_grad_(True)
    out, _ = model(x)
    with _Recorder() as rec:
        out.sum().backward()
        torch.cuda.synchronize()
    wg = WGRAD_LAUNCHES - ({"dw_conv_wgrad"} if net.startswith("dymn") else set())   # DyMN: the attention gradient
    if mode == "eval":
        wg = wg | {"bn_bwd_reduce"}
    assert not wg & set(rec.calls), sorted(wg & set(rec.calls))
    assert "stem_dgrad" in rec.calls
    assert all(p.grad is None for p in model.parameters())
    assert x.grad is not None and torch.isfinite(x.grad).all()
    if mode == "eval":
        for k, v in model.state_dict().items():
            if k in bufs:
                assert torch.equal(v, bufs[k]), f"{k} changed in eval"


def test_unsupported_requests_raise():
    with contextlib.redirect_stdout(io.StringIO()):
        model = NETS["mn04"][0]("fp32").cuda().eval()
    x = _inputs(527)[0].cuda().requires_grad_(True)
    with pytest.raises(NotImplementedError, match="return_fmaps"):
        model.engine().forward(x, return_fmaps=True)
    out, _ = model(x)
    with pytest.raises(NotImplementedError, match="double backward"):
        torch.autograd.grad(out.sum(), x, create_graph=True)


# ------------------------------------------------------------------------------------------------ eat_mel_bwd
def _mel_module(n_fft, hop, n_mels, train=False):
    from efficientat_b200.models.preprocess import AugmentMelSTFT
    with contextlib.redirect_stdout(io.StringIO()):
        m = AugmentMelSTFT(n_mels=n_mels, win_length=min(800, n_fft), hopsize=hop, n_fft=n_fft,
                           freqm=20 if train else 0, timem=30 if train else 0)
    return m.cuda().train(train)


def _dense(saved, n_fft, n_mels):
    start, length, taps, _ = saved["fb"]
    fb = torch.zeros(n_mels, n_fft // 2 + 1, dtype=torch.float64)
    for m, (s, n) in enumerate(zip(start.tolist(), length.tolist())):
        fb[m, s:s + n] = taps[:n, m].double().cpu()
    return fb


def _mel64(x, fb, window, hop, n_fft, masks):
    """the log-mel chain in float64 with the given dense filterbank and SpecAugment bands (as oracle/mel_oracle.py)"""
    p = x[:, 1:] - 0.97 * x[:, :-1]
    L, half = p.shape[1], n_fft // 2
    idx = torch.arange(-half, L + half).abs()
    idx = torch.where(idx >= L, 2 * (L - 1) - idx, idx)
    frames = p[:, idx].unfold(1, n_fft, hop)[:, :1 + L // hop]
    w = torch.zeros(n_fft, dtype=torch.float64)
    lp = (n_fft - window.numel()) // 2
    w[lp:lp + window.numel()] = window.double()
    spec = torch.fft.rfft(frames * w, dim=-1)
    mel = torch.matmul(fb, (spec.real ** 2 + spec.imag ** 2).transpose(1, 2))
    out = ((mel + 1e-5).log() + 4.5) / 5.0
    if masks is not None:
        fs, fe, ts, te = (t.long().cpu() for t in masks)
        f = torch.arange(out.shape[1]).view(1, -1, 1)
        t = torch.arange(out.shape[2]).view(1, 1, -1)
        hit = ((f >= fs.view(-1, 1, 1)) & (f < fe.view(-1, 1, 1))) | ((t >= ts.view(-1, 1, 1)) & (t < te.view(-1, 1, 1)))
        out = torch.where(hit, torch.full_like(out, 0.9), out)
    return out


def _mel_case(n_fft, hop, n_mels, N, B=3, train=False, seed=0):
    from efficientat_b200.synth import synth_waveform
    torch.manual_seed(seed)
    mel = _mel_module(n_fft, hop, n_mels, train)
    wave = synth_waveform(B, N, seed=seed + 11, std=0.3)
    x = wave.cuda().requires_grad_(True)
    out = mel(x)
    saved = out.grad_fn.saved
    cot = torch.randn(out.shape, generator=torch.Generator().manual_seed(seed + 5))
    out.backward(cot.cuda())
    x64 = wave.double().requires_grad_(True)
    ref = _mel64(x64, _dense(saved, n_fft, n_mels), mel.window.cpu(), hop, n_fft, saved.get("masks"))
    assert (out.detach().double().cpu() - ref.detach()).abs().max().item() < 1e-3
    ref.backward(cot.double())
    return mel, x, saved, cot, x.grad.double().cpu(), x64.grad


MEL_BOUND = 3e-4            # rel L2 of dwave against fp64; measured worst 7.2e-5 (n_fft 256, hop 160, 128 mels)


@pytest.mark.parametrize("n_mels", [128, 64])
@pytest.mark.parametrize("hop", [320, 160])
@pytest.mark.parametrize("n_fft", [256, 512, 1024, 2048, 4096])
def test_mel_bwd_matches_fp64(n_fft, hop, n_mels):
    _, _, _, _, got, ref = _mel_case(n_fft, hop, n_mels, N=8000 + 77)
    err, cos = _rel(got, ref)
    report(f"mel bwd n_fft {n_fft} hop {hop} n_mels {n_mels}: rel {err:.2e} cos {cos:.10f}")
    assert err < MEL_BOUND and cos > 1 - 1e-8


@pytest.mark.parametrize("n_fft", [256, 1024, 4096])
def test_mel_bwd_short_clips_masks_jitter_and_repeatability(n_fft):
    # shorter than one hop (one frame); the last frame reaching into the reflect padding; training mode with masks and
    # a jittered filterbank
    for N, train in ((n_fft // 2 + 2 + 10, False), (3 * 320 + n_fft // 2 + 5, False), (16000 + 3, True)):
        mel, x, saved, cot, got, ref = _mel_case(n_fft, 320, 128, N=N, train=train, seed=N)
        err, cos = _rel(got, ref)
        report(f"mel bwd n_fft {n_fft} N {N} train {train}: rel {err:.2e} cos {cos:.10f}")
        assert err < MEL_BOUND and cos > 1 - 1e-8
        again = mel._backward(x.detach(), cot.cuda(), saved)
        assert torch.equal(again.double().cpu(), got)


def test_waveform_to_frozen_mn04_matches_fp64():
    """waveform -> AugmentMelSTFT -> frozen mn04 in eval() -> loss: the waveform's gradient against the fp64 chain"""
    from efficientat_b200.synth import synth_waveform
    from oracle import mel_oracle
    with contextlib.redirect_stdout(io.StringIO()):
        model = build_model("mn04").cuda().eval()
    for p in model.parameters():
        p.requires_grad_(False)
    mel = _mel_module(1024, 320, 128)
    wave = synth_waveform(2, 32000, seed=5)
    cot = torch.randn(2, 527, generator=torch.Generator().manual_seed(9))
    x = wave.cuda().requires_grad_(True)
    logits, _ = model(mel(x).unsqueeze(1))
    (logits * cot.cuda()).sum().backward()
    sd = {k: (v.double() if v.is_floating_point() else v).cpu() for k, v in model.state_dict().items()}
    x64 = wave.double().requires_grad_(True)
    spec = mel_oracle.mel_forward(x64, fmax=mel.fmax, dtype=torch.float64)
    ref_logits = no.mn_forward(sd, spec.unsqueeze(1), 0.4)[0]
    (ref_logits * cot.double()).sum().backward()
    err, cos = _rel(x.grad.double().cpu(), x64.grad)
    report(f"waveform -> mn04 eval: dwave rel {err:.2e} cos {cos:.8f}")
    # mn04's buffers are calibrated on another input, so this eval net amplifies the input's rounding: measured 1.1e-2,
    # cos 0.99994
    assert err < 3e-2 and cos > 0.9995
    assert all(p.grad is None for p in model.parameters())
