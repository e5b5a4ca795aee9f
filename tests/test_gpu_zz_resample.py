"""Resample on the GPU (csrc/resample.cu, efficientat_b200/resample.py).

- Both kernels against scipy.signal.resample_poly in fp64 (forward) and fp64 autograd of the restatement in
  tests/resample_util.py (adjoint), at B in {1, 5, 37} and odd N from one sample to 30 s, for 8 to 96 kHz to and from
  32 kHz, and two pairs at the rate limit whose table is staged in slices.  Bound: 2e-6 of the largest |y| of the fp64
  result; the worst ratio of each pair is reported.
- Per-clip lengths on a NaN-padded batch against scipy on each truncated clip, zeros past each clip's outputs.
- Two planted defects must fail the same bound: the filter without its gain `up`, and a one-sample alignment slip.
- 44.1 kHz waveforms -> Resample -> AugmentMelSTFT -> mn04 eval logits against the fp64 oracle fed scipy's resampling,
  with and without lengths; the waveform's gradient through a frozen mn04 (eval) and dymn04 (batch statistics).
- The tagger with sr=44100 against the tagger fed scipy's resampling, and its launches without sr unchanged.
Inputs are seeded chirps plus noise."""
import contextlib
import io

import numpy as np
import pytest
import scipy.signal as ss
import torch
import torch.nn.functional as Fn

from efficientat_b200._lib import lib
from efficientat_b200.resample import Resample
from oracle import mel_oracle
from oracle import net_oracle as no
from tests.resample_util import resample_adjoint
from tests.util import build_model, report

pytestmark = pytest.mark.gpu

NATIVE = (8000, 11025, 16000, 22050, 24000, 44100, 48000, 88200, 96000)
PAIRS = [(r, 32000) for r in NATIVE] + [(32000, r) for r in NATIVE]
LIMIT = [(2048, 1), (2047, 2)]              # 40961 / 20471 taps per output: the table goes through shared memory in slices
BOUND = 2e-6                                # of max |y64|; scipy's own fp32 path is 1.0e-6 off at 44.1 -> 32 kHz


def _signal(B, N, sr, seed):
    g = np.random.default_rng(seed)
    t = np.arange(N) / sr
    f0 = g.uniform(50, 500, (B, 1))
    chirp = np.sin(2 * np.pi * (f0 + 0.45 * sr / 2 * t / max(t[-1], 1e-9) / 2) * t)
    return (0.5 * chirp + 0.2 * g.standard_normal((B, N))).astype(np.float32)


def _ratio(got, ref):
    return float(np.abs(got.astype(np.float64) - ref).max() / max(np.abs(ref).max(), 1e-30))


def _cases(orig):
    """(B, N): odd N from one sample to 30 s"""
    return [(1, 1), (5, 3), (37, 7), (5, 1001), (37, orig // 7 * 2 + 1), (5, orig * 2 + 1), (1, orig * 30 + 1)]


@pytest.mark.parametrize("orig,new", PAIRS + LIMIT)
def test_forward_and_adjoint_match_fp64(orig, new):
    rs = Resample(orig, new).cuda()
    worst_f = worst_b = 0.0
    limit = (orig, new) in LIMIT
    for B, N in _cases(orig) if not limit else [(1, 1), (5, 3), (37, 4097), (5, 100001)]:
        x = _signal(B, N, orig, seed=B * 7 + N)
        y = rs(torch.from_numpy(x).cuda()).cpu().numpy()
        ref = ss.resample_poly(x.astype(np.float64), rs.up, rs.down, axis=1)
        assert y.shape == ref.shape
        # at the limit pairs an output is a sum of 20 000 to 40 000 products that nearly cancel: held to the input's scale
        worst_f = max(worst_f, _ratio(y, ref) * (np.abs(ref).max() / np.abs(x).max() if limit else 1.0))
        # adjoint: a seeded cotangent through the kernel's backward against the fp64 restatement (up to 2 s)
        if N <= 2 * orig + 1:
            g = torch.randn(ref.shape, generator=torch.Generator().manual_seed(N), dtype=torch.float64)
            xg = torch.from_numpy(x).cuda().requires_grad_(True)
            rs(xg).backward(g.float().cuda())
            want = resample_adjoint(g, N, orig, new).numpy()
            worst_b = max(worst_b, _ratio(xg.grad.cpu().numpy(), want))
    report(f"resample {orig} -> {new} (up {rs.up}, down {rs.down}): worst forward {worst_f:.2e}, adjoint {worst_b:.2e} "
           f"of max |y64|")
    assert worst_f <= BOUND and worst_b <= BOUND


@pytest.mark.parametrize("orig", [44100, 48000, 22050, 16000, 32000])
def test_lengths_on_nan_padded_batch(orig):
    rs = Resample(orig).cuda()
    N = orig * 2 + 1
    lengths = [N, 1, 2, 333, orig + 7, N - 1, 441]
    x = _signal(len(lengths), N, orig, seed=3)
    for b, n in enumerate(lengths):
        x[b, n:] = np.nan
    y = rs(torch.from_numpy(x).cuda(), lengths).cpu().numpy()
    counts = rs.num_samples(lengths)
    assert y.shape == (len(lengths), -(-N * rs.up // rs.down))
    worst = 0.0
    for b, (n, c) in enumerate(zip(lengths, counts)):
        ref = ss.resample_poly(x[b, :n].astype(np.float64), rs.up, rs.down)
        assert len(ref) == c
        worst = max(worst, _ratio(y[b, :c], ref))
        assert np.all(y[b, c:] == 0.0)
    report(f"resample {orig} -> 32000 with lengths: worst {worst:.2e}")
    assert worst <= BOUND and np.isfinite(y).all()


def test_planted_defects_fail_the_bound():
    rs = Resample(44100).cuda()
    x = _signal(5, 44100 + 1, 44100, seed=9)
    ref = ss.resample_poly(x.astype(np.float64), rs.up, rs.down, axis=1)
    xd = torch.from_numpy(x).cuda()
    assert _ratio(rs(xd).cpu().numpy(), ref) <= BOUND

    def run(table, offset):
        y = torch.empty(5, ref.shape[1], device="cuda")
        lib().resample_poly_fwd(xd.data_ptr(), 5, x.shape[1], 0, rs.up, rs.down, table.data_ptr(), rs.taps, offset,
                                y.data_ptr(), y.shape[1], torch.cuda.current_stream().cuda_stream)
        return y.cpu().numpy()
    no_gain = _ratio(run((rs._table / rs.up).contiguous(), rs.half_len), ref)
    slip = _ratio(run(rs._table, rs.half_len + rs.up), ref)                 # reads one input sample later
    report(f"resample planted defects: no gain {no_gain:.2e}, one-sample slip {slip:.2e}")
    assert no_gain > 100 * BOUND and slip > 100 * BOUND


def test_identity_and_repeatability():
    x = torch.from_numpy(_signal(3, 1001, 32000, seed=1)).cuda()
    rs = Resample(32000)
    with _Recorder() as rec:
        y = rs(x)
        y2 = rs(x, [1001, 5, 1])
    assert rec.calls == [] and torch.equal(y, x) and y.data_ptr() != x.data_ptr()
    assert torch.equal(y2[0], x[0]) and torch.equal(y2[1, :5], x[1, :5]) and not y2[1, 5:].any() and not y2[2, 1:].any()
    rs = Resample(44100).cuda()
    a, b = rs(x), rs(x)
    assert torch.equal(a, b) and rs(x[:0]).shape == (0, 727)
    with pytest.raises(NotImplementedError, match="double backward"):
        xg = x.clone().requires_grad_(True)
        torch.autograd.grad(rs(xg).sum(), xg, create_graph=True)


# ------------------------------------------------------------------------------------------------ composition
def _mel():
    from efficientat_b200.models.preprocess import AugmentMelSTFT
    with contextlib.redirect_stdout(io.StringIO()):
        return AugmentMelSTFT(freqm=0, timem=0).cuda().eval()


def _mn04():
    with contextlib.redirect_stdout(io.StringIO()):
        model = build_model("mn04").cuda().eval()
    model.engine().gemm_impl = "simt"           # the exact-fp32 GEMMs, so that the bound speaks of the resampler
    return model


def _sd(model):
    return {k: (v.double() if v.is_floating_point() else v).cpu() for k, v in model.state_dict().items()}


def _oracle_logits(sd, x64, fmax):
    spec = mel_oracle.mel_forward(x64, fmax=fmax, dtype=torch.float64)
    return no.mn_forward(sd, spec.unsqueeze(1), 0.4)[0]


LOGIT_BOUND = 1e-3          # max |logit error| over max(1, max |logit|)


def test_resample_mel_mn04_eval_matches_fp64():
    rs, mel, model = Resample(44100).cuda(), _mel(), _mn04()
    N = 88200 + 37
    x = _signal(3, N, 44100, seed=4)
    with torch.no_grad():
        logits = model(mel(rs(torch.from_numpy(x).cuda())).unsqueeze(1))[0].double().cpu()
    x64 = torch.from_numpy(ss.resample_poly(x.astype(np.float64), 320, 441, axis=1))
    ref = _oracle_logits(_sd(model), x64, mel.fmax)
    err = ((logits - ref).abs().max() / ref.abs().max().clamp_min(1)).item()
    report(f"44.1 kHz -> Resample -> mel -> mn04 eval: logits {err:.2e}")
    assert err < LOGIT_BOUND

    # clips of different lengths in one batch: each row against the oracle on its own clip
    lengths = [N, 44100 + 5, 30001, 12345]
    xl = _signal(len(lengths), N, 44100, seed=5)
    for b, n in enumerate(lengths):
        xl[b, n:] = np.nan
    n_out = rs.num_samples(lengths)
    with torch.no_grad():
        y = rs(torch.from_numpy(xl).cuda(), lengths)
        got = model(mel(y, n_out).unsqueeze(1), mel.num_frames(n_out))[0].double().cpu()
    sd, worst = _sd(model), 0.0
    for b, n in enumerate(lengths):
        r = _oracle_logits(sd, torch.from_numpy(ss.resample_poly(xl[b:b + 1, :n].astype(np.float64), 320, 441, axis=1)),
                           mel.fmax)
        worst = max(worst, ((got[b] - r[0]).abs().max() / r.abs().max().clamp_min(1)).item())
    report(f"44.1 kHz with lengths -> mn04 eval: worst logits {worst:.2e}")
    assert worst < LOGIT_BOUND and torch.isfinite(got).all()


def _rel(a, b):
    return ((a - b).norm() / b.norm()).item(), Fn.cosine_similarity(a.flatten(), b.flatten(), dim=0).item()


@pytest.mark.parametrize("net", ["mn04", "dymn04"])
def test_waveform_gradient_at_native_rate_matches_fp64(net):
    """44.1 kHz waveform -> Resample -> mel -> frozen net -> loss: x.grad at 44.1 kHz against fp64 autograd of the
    restated resampler, the mel oracle and the net oracle.  mn04 in eval(); dymn04 on batch statistics (train())."""
    from tests.resample_util import resample as resample64
    rs, mel = Resample(44100).cuda(), _mel()
    with contextlib.redirect_stdout(io.StringIO()):
        model = build_model(net).cuda()
    model.engine().gemm_impl = "simt"
    training = net == "dymn04"
    model.train(training)
    for m in model.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    for p in model.parameters():
        p.requires_grad_(False)
    wave = torch.from_numpy(_signal(2, 44100 + 3, 44100, seed=6))
    cot = torch.randn(2, 527, generator=torch.Generator().manual_seed(9))
    x = wave.cuda().requires_grad_(True)
    logits, _ = model(mel(rs(x)).unsqueeze(1))
    (logits * cot.cuda()).sum().backward()
    sd = _sd(model)
    x64 = wave.double().requires_grad_(True)
    spec = mel_oracle.mel_forward(resample64(x64, 44100, 32000), fmax=mel.fmax, dtype=torch.float64).unsqueeze(1)
    if net == "mn04":
        ref_logits = no.mn_forward(sd, spec, 0.4)[0]
    else:
        ref_logits = no.dymn_forward(sd, spec, 0.4, training=True,
                                     temperature=float(model.layers[0].depth_conv.temperature))[0]
    (ref_logits * cot.double()).sum().backward()
    err, cos = _rel(x.grad.double().cpu(), x64.grad)
    report(f"44.1 kHz waveform -> Resample -> mel -> {net}: dwave rel {err:.2e} cos {cos:.8f}")
    # the resampler alone is within 4e-7 of fp64 (test_forward_and_adjoint_match_fp64); the rest is the nets: mn04's eval
    # buffers are calibrated on another input, dymn04's batch statistics come from two clips, and both amplify the
    # input's rounding.  Measured on an H100: mn04 7.9e-3 (cos 0.99997), dymn04 1.1e-2 (cos 0.99994); the same chain at
    # 32 kHz without the resampler is held to 3e-2 in test_gpu_zz_input_grad.py
    assert err < 3e-2 and cos > 0.9995
    assert all(p.grad is None for p in model.parameters())


# ------------------------------------------------------------------------------------------------ tagger
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


def _tagger():
    """an EATagger over the synthetic mn04 (the released checkpoints are not needed to test the resampling)"""
    from efficientat_b200.windowed import EATagger
    t = EATagger.__new__(EATagger)
    t.device = torch.device("cuda", torch.cuda.current_device())
    t.sample_rate, t.window_size, t.hop_size, t.n_mels, t.max_batch = 32000, 800, 320, 128, 256
    t.model, t.mel = _mn04(), _mel()
    t.labels = [str(i) for i in range(527)]
    t._resamplers = {}
    return t


def test_tagger_resamples_on_the_device():
    tagger = _tagger()
    wave = _signal(1, 44100 * 7 + 11, 44100, seed=8)[0]
    ref32 = ss.resample_poly(wave.astype(np.float64), 320, 441).astype(np.float32)
    tagger.window_probabilities(ref32, 2.0, 1.0)                 # host-only launch-plan queries are asked once per shape
    with _Recorder() as rec:
        before = tagger.window_probabilities(ref32, 2.0, 1.0)
    torch.cuda.synchronize()
    got = tagger.tag_waveform(wave, 2.0, 1.0, sr=44100)
    want = tagger.tag_waveform(ref32, 2.0, 1.0)
    p_got, starts, win = tagger.window_probabilities(wave, 2.0, 1.0, sr=44100)
    p_want = before[0]
    assert (starts, win) == (before[1], before[2]) and len(got) == len(want) == len(starts)
    worst = (p_got - p_want).abs().max().item()
    report(f"tagger sr=44100 against scipy-resampled input: {len(starts)} windows, worst probability {worst:.2e}")
    assert worst < 1e-4
    for a, b in zip(got, want):
        assert (a["start"], a["end"]) == (b["start"], b["end"])
        for ta, tb in zip(a["tags"], b["tags"]):
            assert abs(ta["probability"] - tb["probability"]) < 1e-4
    # the default path launches exactly what it launched before sr was used, and no resampler
    with _Recorder() as rec2:
        tagger.window_probabilities(ref32, 2.0, 1.0)
        tagger.window_probabilities(ref32, 2.0, 1.0, sr=32000)
    assert rec2.calls == rec.calls + rec.calls and not any(c.startswith("resample") for c in rec.calls)
    with _Recorder() as rec3:
        tagger.window_probabilities(wave, 2.0, 1.0, sr=44100)
    assert rec3.calls == ["resample_poly_fwd"] + rec.calls
