"""Clips of different lengths in one eval batch (`lengths`), on the GPU.

- The new entry points against torch / fp64: eat_mel_fwd_len against per-clip eat_mel_fwd and the mel oracle;
  eat_time_pad_zero writes the padding only (sentinels in the valid region survive), fp32 and bf16, odd C, T_b = T and
  T_b = 1; eat_mean_len and eat_ctx_pool_len against fp64 torch; eat_att_pool_fwd_len against torch on the truncated
  frames.
- The six clips of tests/golden/packed.npz (0.05 s to 2.71 s), zero-padded into one batch with `lengths`, against the
  unmodified reference run on each clip alone in fp64: mn04 (mlp, attention head, dilated), dymn04 (dyrelu_k 2 and 3,
  replace_se), fp32 on the simt and auto routes within the project's 1e-3 parity bound, and bf16.
- Whole nets at B = 7 (lengths unsorted, one duplicated, one equal to T, one of 1 frame): mn04 (mlp, attention head,
  dilated), dymn04 (dyrelu_k 2 and 3, replace_se), mn10 and dymn10, against the package's own B = 1 call on each
  truncated clip, on the simt and auto routes and in bf16.
- NaN and +-1e4 past every length give bit-identical outputs (mel and nets).  Planted defects fail the per-clip
  comparison: no lengths on the padded batch, one clip's length minus one, the pools counting the padded positions.
- All lengths equal to T agree with the call without lengths; the launch lists and outputs without lengths are the
  same before and after a call with lengths; a list of waveforms through mel(x, lengths) and
  model(spec, mel.num_frames(lengths)) equals per-clip inference."""
import contextlib
import io

import pytest
import torch

from efficientat_b200._lib import lib
from tests import fmap_grad_util as fu
from tests import packed_util as pu
from tests.test_gpu_zz_fmap_grad import _plain_runs, _Recorder
from tests.util import build_model, golden, report

pytestmark = pytest.mark.gpu

DT = {"fp32": torch.float32, "bf16": torch.bfloat16}
CODE = {torch.float32: 0, torch.bfloat16: 1}
NEW_ENTRIES = {"mel_fwd_len", "time_pad_zero", "mean_len", "ctx_pool_len", "att_pool_fwd_len"}


def _st():
    return torch.cuda.current_stream().cuda_stream


def _mel(**kw):
    from efficientat_b200.models.preprocess import AugmentMelSTFT
    with contextlib.redirect_stdout(io.StringIO()):
        return AugmentMelSTFT(freqm=0, timem=0, **kw).cuda().eval()


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("n_fft", [1024, 2048])
def test_mel_len_matches_per_clip(n_fft):
    from oracle import mel_oracle
    from efficientat_b200.synth import synth_waveform
    mel = _mel(n_fft=n_fft)
    N = 64000
    lengths = [N, n_fft // 2 + 2, 20001, 31999, 320, 9600, 20001]
    lengths[4] = max(lengths[4], n_fft // 2 + 2)
    x = synth_waveform(len(lengths), N, seed=11).cuda()
    out = mel(x, lengths)
    assert out.shape == (len(lengths), 128, 1 + (N - 1) // 320)
    frames = mel.num_frames(lengths)
    for b, n in enumerate(lengths):
        one = mel(x[b:b + 1, :n])[0]
        assert one.shape[1] == frames[b]
        d = (out[b, :, :frames[b]] - one).abs().max().item()
        assert d <= 1e-6, (b, n, d)
        assert torch.all(out[b, :, frames[b]:] == 0.0)
        ref = mel_oracle.mel_forward(x[b:b + 1, :n].cpu(), n_fft=n_fft)[0]
        assert (out[b, :, :frames[b]].cpu() - ref).abs().max().item() < 1e-4
    # samples past each length are never read
    for fill in (float("nan"), 1e4, -1e4):
        y = x.clone()
        for b, n in enumerate(lengths):
            y[b, n:] = fill
        assert torch.equal(mel(y, lengths), out)


@pytest.mark.parametrize("dt", ["fp32", "bf16"])
@pytest.mark.parametrize("C", [1, 3, 37, 96])
def test_time_pad_zero_writes_the_padding_only(dt, C):
    B, F, T = 5, 7, 23
    tv = [T, 1, 11, T - 1, 2]
    g = torch.Generator().manual_seed(C)
    x = (torch.randn(B, F, T, C, generator=g) + 5.0).to(DT[dt]).cuda()       # no zero in the valid region
    y = x.clone()
    t_valid = torch.tensor(tv, dtype=torch.int32).cuda()
    lib().time_pad_zero(y.data_ptr(), CODE[DT[dt]], B, F, T, C, t_valid.data_ptr(), _st())
    for b, t in enumerate(tv):
        assert torch.equal(y[b, :, :t], x[b, :, :t])
        assert torch.all(y[b, :, t:] == 0)


@pytest.mark.parametrize("dt", ["fp32", "bf16"])
@pytest.mark.parametrize("shape", [(3, 1, 40, 5), (4, 7, 23, 37), (2, 4, 300, 960)])
def test_mean_len_matches_fp64(dt, shape):
    B, F, T, C = shape
    tv = ([T, 1, max(1, T // 2), T - 1] * 2)[:B]
    g = torch.Generator().manual_seed(T * C)
    x = torch.randn(B, F, T, C, generator=g).to(DT[dt]).cuda()
    x_pad = x.clone()
    for b, t in enumerate(tv):
        x_pad[b, :, t:] = float("nan")                      # never read
    out = torch.empty(B, C, device="cuda")
    t_valid = torch.tensor(tv, dtype=torch.int32).cuda()
    lib().mean_len(x_pad.data_ptr(), CODE[DT[dt]], out.data_ptr(), B, F, T, C, t_valid.data_ptr(), _st())
    for b, t in enumerate(tv):
        ref = x[b, :, :t].double().mean((0, 1))
        assert (out[b].double() - ref.cuda()).abs().max().item() <= 1e-5 * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize("dt", ["fp32", "bf16"])
def test_ctx_pool_len_matches_fp64(dt):
    B, F, T, C = 4, 9, 31, 24
    tv = [T, 1, 12, 30]
    g = torch.Generator().manual_seed(3)
    x = torch.randn(B, F, T, C, generator=g).to(DT[dt]).cuda()
    x_pad = x.clone()
    for b, t in enumerate(tv):
        x_pad[b, :, t:] = float("nan")
    out = torch.empty(B, F + T, C, device="cuda")
    t_valid = torch.tensor(tv, dtype=torch.int32).cuda()
    lib().ctx_pool_len(x_pad.data_ptr(), CODE[DT[dt]], out.data_ptr(), B, F, T, C, t_valid.data_ptr(), _st())
    for b, t in enumerate(tv):
        xb = x[b, :, :t].double()
        assert (out[b, :F].double() - xb.mean(1)).abs().max().item() <= 1e-5
        assert (out[b, F:F + t].double() - xb.mean(0)).abs().max().item() <= 1e-5
        assert torch.all(out[b, F + t:] == 0)


def test_att_pool_fwd_len_matches_torch():
    from tests import mha_util as mu
    B, T, H, K = 5, 17, 4, 11
    tv = [T, 1, 9, 16, 9]
    g = torch.Generator().manual_seed(5)
    P = torch.randn(B, T, 2 * H * K, generator=g).cuda()
    hw = torch.rand(H, generator=g).cuda()
    P_pad = P.clone()
    for b, t in enumerate(tv):
        P_pad[b, t:] = float("nan")
    out = torch.empty(B, K, device="cuda")
    t_valid = torch.tensor(tv, dtype=torch.int32).cuda()
    lib().att_pool_fwd_len(P_pad.data_ptr(), hw.data_ptr(), mu.EPS, out.data_ptr(), B, T, H, K, t_valid.data_ptr(), _st())
    for b, t in enumerate(tv):
        Pb = P[b, :t].double()
        a = torch.sigmoid(Pb[:, :H * K]).clamp(mu.EPS, 1 - mu.EPS).view(t, H, K)
        v = Pb[:, H * K:].view(t, H, K)
        ref = ((a * v).sum(0) / a.sum(0) * hw.double()[:, None]).sum(0)
        assert (out[b].double() - ref).abs().max().item() <= 1e-5
        # and the fixed-length kernel on the truncated frames
        one = torch.empty(1, K, device="cuda")
        lib().att_pool_fwd(P[b:b + 1, :t].contiguous().data_ptr(), hw.data_ptr(), mu.EPS, one.data_ptr(), 0, 0, 1, t, H,
                           K, _st())
        assert (out[b] - one[0]).abs().max().item() <= 1e-6


# ------------------------------------------------------------------------------------------------ nets
NETS = ["mn04", "mn04_mha", "mn04_dilated", "dymn04_k2", "dymn04_k3", "dymn04_replace_se", "mn10", "dymn10"]
T_NET = 200                                     # 2 s clips
LENGTHS = [113, T_NET, 57, 1, 113, 171, 9]      # unsorted, one duplicated, one equal to T, one of 1 frame


# DyMN nets keep synth_state_'s BatchNorm buffers: with the buffers calibrated for the training goldens their eval
# logits reach 1e7 - 1e11 on these clips, and a change of summation order in one pool moves them by 1e-3 relative
DYMN = {"dymn04_k2": dict(width_mult=0.4, dyrelu_k=2), "dymn04_k3": dict(width_mult=0.4, dyrelu_k=3),
        "dymn04_replace_se": dict(width_mult=0.4, use_dy_blocks="replace_se"), "dymn10": dict(width_mult=1.0)}


def _net(tag, precision="fp32"):
    if tag in DYMN:
        from efficientat_b200.models.dymn.model import get_model
        from efficientat_b200.synth import synth_state_
        torch.manual_seed(0)
        with contextlib.redirect_stdout(io.StringIO()):
            m = get_model(precision=precision, verbose=False, **DYMN[tag])
        synth_state_(m, seed=7)
    elif tag in fu.CASES:
        m = fu.build_model(tag, golden("fmap_grad"), precision=precision)
    else:
        m = build_model(tag, precision=precision)
    return m.cuda().eval()


def _spec(B=len(LENGTHS), T=T_NET, seed=21):
    from efficientat_b200.synth import synth_waveform
    return synth_waveform(B, 128 * T, seed=seed, std=0.7).view(B, 1, 128, T).cuda()


def _per_clip(model, x, lengths):
    outs = [model(x[b:b + 1, :, :, :n]) for b, n in enumerate(lengths)]
    return torch.cat([o[0] for o in outs]), torch.cat([o[1] for o in outs])


def _diffs(logits, feat, ref_logits, ref_feat):
    dl = (logits - ref_logits).abs().max().item()
    df = ((feat - ref_feat).norm(dim=1) / ref_feat.norm(dim=1).clamp_min(1e-12)).max().item()
    return dl, df


@pytest.mark.parametrize("route", ["simt", "auto"])
@pytest.mark.parametrize("tag", NETS)
def test_net_matches_per_clip_fp32(tag, route):
    model = _net(tag)
    model.engine().gemm_impl = route
    x = _spec()
    with torch.no_grad():
        logits, feat = model._forward_impl(x, lengths=LENGTHS)
        ref_logits, ref_feat = _per_clip(model, x, LENGTHS)
    dl, df = _diffs(logits, feat, ref_logits, ref_feat)
    report(f"packed {tag} {route}: logits max-abs {dl:.2e}, features rel {df:.2e}")
    assert dl <= 1e-4 and df <= 1e-4
    k = min(10, logits.shape[1])
    assert torch.equal(logits.topk(k, dim=1).indices, ref_logits.topk(k, dim=1).indices)


@pytest.mark.parametrize("precision", ["simt", "auto", "bf16"])
@pytest.mark.parametrize("tag", list(pu.NETS))
def test_net_matches_reference_goldens(tag, precision):
    """the six golden clips zero-padded into one batch with `lengths`, against the unmodified reference run on each clip
    alone in fp64 (tests/golden/make_golden_packed.py)"""
    g = golden("packed")
    model = pu.build_model(tag, precision="bf16" if precision == "bf16" else "fp32").cuda().eval()
    if precision != "bf16":
        model.engine().gemm_impl = precision
    x = pu.padded_batch(pu.clip_specs()).cuda()
    with torch.no_grad():
        logits, feat = model._forward_impl(x, lengths=pu.clip_frames())
    ref_l = torch.from_numpy(g[tag + "__logits"]).cuda()
    ref_f = torch.from_numpy(g[tag + "__features"]).cuda()
    dl = (logits.double() - ref_l).abs().max().item()
    df = ((feat.double() - ref_f).norm(dim=1) / ref_f.norm(dim=1)).max().item()
    report(f"packed golden {tag} {precision}: logits max-abs {dl:.2e}, features rel {df:.2e}")
    if precision == "bf16":
        # bf16 storage rounds every stored activation, and on these short clips (tails of 1 frame) that alone moves mn04's
        # features by 6e-2: the bound is the package's own bf16 error on each clip run alone, so `lengths` adds none
        with torch.no_grad():
            one = [model(s.cuda()) for s in pu.clip_specs()]
        el1 = (torch.cat([o[0] for o in one]).double() - ref_l).abs().max().item()
        ef1 = ((torch.cat([o[1] for o in one]).double() - ref_f).norm(dim=1) / ref_f.norm(dim=1)).max().item()
        report(f"packed golden {tag} bf16 clip by clip: logits max-abs {el1:.2e}, features rel {ef1:.2e}")
        assert dl <= 1.25 * el1 + 1e-2 and df <= 1.25 * ef1 + 1e-2
    else:
        assert dl <= 1e-3 and df <= 1e-3                                             # the project's parity bound
    k = min(10, logits.shape[1])
    if precision != "bf16":
        assert torch.equal(logits.topk(k, dim=1).indices, ref_l.topk(k, dim=1).indices)


@pytest.mark.parametrize("tag", NETS)
def test_net_matches_per_clip_bf16(tag):
    model = _net(tag, precision="bf16")
    x = _spec()
    with torch.no_grad():
        logits, feat = model._forward_impl(x, lengths=LENGTHS)
        ref_logits, ref_feat = _per_clip(model, x, LENGTHS)
    dl, df = _diffs(logits, feat, ref_logits, ref_feat)
    scale = max(1.0, ref_logits.abs().max().item())
    report(f"packed {tag} bf16: logits max-abs {dl:.2e} (scale {scale:.2f}), features rel {df:.2e}")
    # bf16 storage: the bound of the bf16 eval tests (tests/test_gpu_mn.py)
    assert dl <= 6e-2 * scale and df <= 6e-2


@pytest.mark.parametrize("tag", ["mn04", "mn04_mha", "dymn04_k2"])
def test_net_ignores_the_padding(tag):
    model = _net(tag)
    x = _spec()
    with torch.no_grad():
        base = model._forward_impl(x, lengths=LENGTHS)
        for fill in (float("nan"), 1e4, -1e4):
            y = x.clone()
            for b, n in enumerate(LENGTHS):
                y[b, :, :, n:] = fill
            out = model._forward_impl(y, lengths=LENGTHS)
            assert torch.equal(out[0], base[0]) and torch.equal(out[1], base[1]), fill
    # the caller's tensor is not written
    y0 = y.clone()
    with torch.no_grad():
        model._forward_impl(y, lengths=LENGTHS)
    assert torch.equal(y.nan_to_num(), y0.nan_to_num())


@pytest.mark.parametrize("tag", ["mn04", "mn04_mha", "dymn04_k2"])
def test_planted_defects_fail_the_per_clip_comparison(tag):
    model = _net(tag)
    x = _spec()
    with torch.no_grad():
        ref_logits, _ = _per_clip(model, x, LENGTHS)
        no_lengths = model._forward_impl(x)[0]
        short = list(LENGTHS)
        short[0] -= 1
        one_short = model._forward_impl(x, lengths=short)[0]
        # the pools count all T positions, as the depthwise epilogue's fused squeeze would
        L = lib()
        real = L.mean_len
        calls = []                                  # keeps the planted tables alive until the forward has run

        def full_t(xp, dt, out, B, F, T, C, t_valid, st):
            full = torch.full((B,), T, dtype=torch.int32, device="cuda")
            calls.append(full)
            return real(xp, dt, out, B, F, T, C, full.data_ptr(), st)
        L.mean_len = full_t
        try:
            pooled_padding = model._forward_impl(x, lengths=LENGTHS)[0]
        finally:
            L.mean_len = real
    assert calls
    for name, bad in (("no lengths", no_lengths), ("one clip one frame short", one_short),
                      ("pools count the padding", pooled_padding)):
        d = (bad - ref_logits).abs().max().item()
        report(f"packed planted defect {tag} {name}: logits max-abs {d:.2e}")
        assert d > 1e-4, name                       # the fp32 per-clip bound of test_net_matches_per_clip_fp32


@pytest.mark.parametrize("tag", ["mn04", "mn04_mha", "dymn04_k3"])
def test_full_lengths_equal_the_plain_call(tag):
    model = _net(tag)
    x = _spec()
    with torch.no_grad():
        a = model._forward_impl(x, lengths=[T_NET] * x.shape[0])
        b = model._forward_impl(x)
    # the plain call's squeeze-excitation pool sums in the depthwise epilogue, in another order than eat_mean_len:
    # measured up to 1.1e-5 of max(1, |logits|) (mn04_mha, auto route)
    for u, v in zip(a, b):
        d = (u - v).abs().max().item() / max(1.0, v.abs().max().item())
        report(f"packed full lengths {tag}: max diff {d:.2e}")
        assert d <= 3e-5


@pytest.mark.parametrize("tag", ["mn04", "dymn04_k2"])
def test_launches_and_values_without_lengths_are_unchanged(tag):
    model = fu.build_model(tag, golden("fmap_grad")).cuda()
    spec = fu.net_inputs()[0].cuda()
    state = {k: v.clone() for k, v in model.state_dict().items()}
    _plain_runs(model, spec)
    model.load_state_dict(state)
    torch.manual_seed(3)                            # the same dropout masks in both plain runs
    before, out_b = _plain_runs(model, spec)
    for k, calls in before.items():
        assert calls and not NEW_ENTRIES & set(calls), k
    model.load_state_dict(state)
    model.eval()
    with _Recorder() as rec, torch.no_grad():
        model._forward_impl(_spec(B=3), lengths=[50, 200, 1])
    assert NEW_ENTRIES & set(rec.calls)
    model.load_state_dict(state)
    torch.manual_seed(3)
    after, out_a = _plain_runs(model, spec)
    assert after == before
    # That the outputs without lengths are bit-identical to the parent's rests on the code and the machine code: the
    # path without lengths runs the same launches (checked above), and every pre-existing kernel compiles to the same
    # SASS as before (scripts/sass_diff.py).  Two runs of this build agree up to the reordering of atomics: the eval
    # forward runs after a training step whose batch statistics' atomics may reorder between runs and move the running
    # statistics (see test_gpu_zz_fmap_grad.py)
    for k in out_b:
        for a, b in zip(out_a[k], out_b[k]):
            assert (a - b).abs().max().item() <= 2e-4 * max(1.0, b.abs().max().item()), k


@pytest.mark.parametrize("tag", ["mn04", "dymn04_k2"])
def test_end_to_end_list_of_waveforms(tag):
    from efficientat_b200.synth import synth_waveform
    mel = _mel()
    model = _net(tag)
    secs = [0.9, 2.71, 0.05, 1.3, 2.0, 0.37]
    waves = [synth_waveform(1, int(s * 32000), seed=40 + i)[0] for i, s in enumerate(secs)]
    lengths = [w.numel() for w in waves]
    x = torch.zeros(len(waves), max(lengths))
    for b, w in enumerate(waves):
        x[b, :w.numel()] = w
    with torch.no_grad():
        spec = mel(x.cuda(), lengths)
        logits, feat = model(spec.unsqueeze(1), lengths=mel.num_frames(lengths))
        for b, w in enumerate(waves):
            ref_logits, ref_feat = model(mel(w.view(1, -1).cuda()).unsqueeze(1))
            assert (logits[b] - ref_logits[0]).abs().max().item() <= 1e-4, b
            assert (feat[b] - ref_feat[0]).norm().item() <= 1e-4 * ref_feat.norm().item(), b


# ------------------------------------------------------------------------------------------------ arguments
def test_argument_checks_on_the_device():
    mel = _mel()
    x = torch.zeros(3, 32000, device="cuda")
    for bad in ([32000, 32000], [32000] * 4, [32000, 100, 32000], [32000, 32001, 32000], [32000, 1.5, 32000],
                torch.tensor([32000.0] * 3)):
        with pytest.raises(ValueError):
            mel(x, bad)
    mel.train()
    with pytest.raises(NotImplementedError, match="lengths"):
        mel(x, [32000] * 3)
    mel.eval()
    with pytest.raises(NotImplementedError, match="lengths"):
        mel(x.clone().requires_grad_(True), [32000] * 3)
    model = _net("mn04")
    spec = _spec(B=3, T=50)
    for bad in ([50, 50], [50, 0, 50], [50, 51, 50], [50, 2.0, 50]):
        with pytest.raises(ValueError):
            model._forward_impl(spec, lengths=bad)
    with pytest.raises(NotImplementedError, match="lengths"):
        model._forward_impl(spec, return_fmaps=True, lengths=[50] * 3)
    with pytest.raises(NotImplementedError, match="lengths"):
        model._forward_impl(spec.clone().requires_grad_(True), lengths=[50] * 3)
    model.train()
    with pytest.raises(NotImplementedError, match="lengths"):
        model._forward_impl(spec, lengths=[50] * 3)
