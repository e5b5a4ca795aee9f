"""Gradients with respect to the input spectrogram, the parts that need no GPU: eat_stem_dgrad is exported and rejects
bad arguments on the host before any launch, and the autograd glue routes each call.  The numerics are in
tests/test_gpu_zz_input_grad.py."""
import ctypes
import subprocess

import pytest

from efficientat_b200 import _lib
from efficientat_b200._lib import EatError, lib

FAKE = 4096                 # never dereferenced: validation comes first


def _dgrad(dtype=0, C=16, stride=2, act=2, B=2, F=8, T=9, dy=FAKE, z=FAKE):
    lib().stem_dgrad(dy, dtype, z, FAKE, FAKE, FAKE, FAKE, act, FAKE, FAKE, FAKE, FAKE, B, F, T, C, stride, 0)


def test_stem_dgrad_is_exported():
    assert hasattr(ctypes.CDLL(_lib.LIB_PATH), "eat_stem_dgrad")
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True).stdout
    assert " T eat_stem_dgrad" in out


@pytest.mark.parametrize("kw, msg", [
    (dict(dtype=2), "dtype"),
    (dict(C=10), "channel count"),                  # fp32 vectors of 4
    (dict(C=12, dtype=1), "channel count"),         # bf16 vectors of 8
    (dict(C=4 * 257), "channel count"),             # more than 256 vectors, as eat_stem_fwd
    (dict(C=0), "channel count"),
    (dict(stride=3), "stride"),
    (dict(act=3), "act"),
    (dict(F=0), "sizes"),
    (dict(T=0), "sizes"),
    (dict(B=-1), "sizes"),
    (dict(z=0), "required"),
    (dict(dy=0), "required"),
])
def test_stem_dgrad_rejects_bad_arguments_before_any_launch(kw, msg):
    with pytest.raises(EatError, match=msg):
        _dgrad(**kw)


def test_stem_dgrad_empty_batch_is_a_no_op():
    _dgrad(B=0)
    _dgrad(B=0, z=0, dy=0)
    _dgrad(B=0, C=1024, stride=1)
    _dgrad(B=0, C=2048, dtype=1)
    with pytest.raises(EatError):
        _dgrad(B=0, stride=3)                       # the checks still come first


def test_eval_with_input_grad_takes_the_frozen_route(monkeypatch):
    """engine._dispatch: eval + input requiring grad -> the saving forward on running statistics; eval without it -> the
    folded forward; return_fmaps with an input that requires grad raises (host logic, the forwards stubbed out)"""
    import torch
    from efficientat_b200 import autograd
    from efficientat_b200.engine import MNEngine

    calls = []

    class Eng(MNEngine):
        def __init__(self, training):
            self.model = torch.nn.Linear(1, 1)
            self.model.train(training)

        def _forward_eval(self, x, return_fmaps=False):
            calls.append(("eval", x.requires_grad))
            return x.sum(), None, None

    monkeypatch.setattr(autograd, "mn_eval_grad_forward", lambda e, x: (calls.append(("eval_grad",)), (x, None))[1])
    monkeypatch.setattr(autograd, "mn_train_forward", lambda e, x, ng: (calls.append(("train", ng)), (x, None))[1])
    monkeypatch.setattr(torch.cuda, "device", lambda d: __import__("contextlib").nullcontext())
    x = torch.zeros(1, 1, 2, 2)
    Eng(False)._dispatch(x, False)
    Eng(False)._dispatch(x.clone().requires_grad_(), False)
    with torch.no_grad():
        Eng(False)._dispatch(x.clone().requires_grad_(), False)
    with pytest.raises(NotImplementedError, match="return_fmaps"):
        Eng(False)._dispatch(x.clone().requires_grad_(), True)
    e = Eng(True)
    for p in e.model.parameters():
        p.requires_grad_(False)
    e._dispatch(x, False)
    e._dispatch(x.clone().requires_grad_(), False)
    assert calls == [("eval", False), ("eval_grad",), ("eval", False), ("train", False), ("train", True)]


def _mel_bwd(B=2, N=8000, win=800, hop=320, n_fft=1024, n_mels=128, masks=(0, 0, 0, 0), work_floats=1 << 40, ptr=FAKE):
    lib().mel_bwd(ptr, FAKE, B, N, FAKE, win, hop, n_fft, FAKE, FAKE, FAKE, FAKE, 10, n_mels, 0.97, *masks, FAKE,
                  work_floats, FAKE, 0)


def test_mel_bwd_is_exported():
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True).stdout
    assert " T eat_mel_bwd" in out and " T eat_mel_bwd_workspace" in out


@pytest.mark.parametrize("kw, msg", [
    (dict(n_fft=768), "n_fft"),
    (dict(n_fft=8192), "n_fft"),
    (dict(win=1025), "geometry"),
    (dict(hop=0), "geometry"),
    (dict(n_mels=513), "geometry"),
    (dict(B=-1), "geometry"),
    (dict(N=513), "too short"),                     # N - 1 must exceed n_fft / 2
    (dict(masks=(FAKE, FAKE, 0, FAKE)), "mask"),
    (dict(ptr=0), "required"),
    (dict(work_floats=100), "work"),
    (dict(hop=1 << 20), "hop too large"),
])
def test_mel_bwd_rejects_bad_arguments_before_any_launch(kw, msg):
    with pytest.raises(EatError, match=msg):
        _mel_bwd(**kw)


def test_mel_bwd_workspace_and_empty_batch():
    n = ctypes.c_longlong()
    lib().mel_bwd_workspace(3, 320000, 320, 1024, ctypes.addressof(n))
    T, F = 1 + 319999 // 320, 16
    assert n.value == 3 * ((T + F - 1) // F) * ((F - 1) * 320 + 1024)
    lib().mel_bwd_workspace(2, 8000, 160, 4096, ctypes.addressof(n))
    assert n.value == 2 * ((1 + 7999 // 160 + 7) // 8) * (7 * 160 + 4096)       # 8 frames per CTA at n_fft 4096
    with pytest.raises(EatError, match="n_fft"):
        lib().mel_bwd_workspace(2, 8000, 160, 300, ctypes.addressof(n))
    _mel_bwd(B=0, work_floats=0, ptr=0)


@pytest.mark.parametrize("tag", ["mn04", "mn04_mha", "dymn04"])
def test_fp64_oracle_matches_reference_input_gradients(tag):
    """autograd through the fp64 oracle (oracle/net_oracle.py, oracle/mel_oracle.py, tests/mha_util.py) against the
    unmodified reference's input gradients (tests/golden/make_golden_input_grad.py): the spectrogram's in eval() and
    train(), the waveform's through the mel front end in eval()"""
    import contextlib
    import io

    import numpy as np
    import torch
    from efficientat_b200.synth import set_bn_stats, synth_state_, synth_waveform
    from oracle import mel_oracle
    from oracle import net_oracle as no
    from tests import mha_util as mu
    from tests.input_grad_util import WAVE_SAMPLES, cotangent, digest, spec_input
    from tests.util import golden

    g = golden("input_grad")
    torch.manual_seed(0)
    with contextlib.redirect_stdout(io.StringIO()):
        if tag == "mn04_mha":
            model = mu.build_mha_model("mn04_h4")
        elif tag == "mn04":
            from efficientat_b200.models.mn.model import get_model
            model = synth_state_(get_model(width_mult=0.4, verbose=False), seed=7)
        else:
            from efficientat_b200.models.dymn.model import get_model
            model = synth_state_(get_model(width_mult=0.4, verbose=False), seed=7)
    set_bn_stats(model, g[tag + "__cal_rm"], g[tag + "__cal_rv"])
    names = [k for k, _ in model.named_parameters()]

    def net(x, training):
        sd = {k: (v.double() if v.is_floating_point() else v).clone() for k, v in model.state_dict().items()}
        for k in names:
            sd[k].requires_grad_(True)
        if tag == "mn04":
            return no.mn_forward(sd, x, 0.4, training=training)[0]
        if tag == "mn04_mha":
            return mu.mn_mha_forward(sd, x, 0.4, 4, 527, training=training)[0]
        return no.dymn_forward(sd, x, 0.4, training=training, temperature=float(model.layers[0].depth_conv.temperature))[0]

    cot = cotangent()
    got = {}
    for mode in ("eval", "train"):
        x = spec_input().double().requires_grad_(True)
        (net(x, mode == "train") * cot).sum().backward()
        got["dspec_" + mode] = digest(x.grad)
    if tag != "dymn04":
        # the net's buffers are calibrated on the spectrogram above, not on this clip's log-mel: there dymn04 amplifies
        # the waveform's gradient to a norm of 4e19 and the two fp64 chains part (0.1 relative), so only MN is compared
        w = synth_waveform(2, WAVE_SAMPLES, seed=5).double().requires_grad_(True)
        (net(mel_oracle.mel_forward(w, dtype=torch.float64).unsqueeze(1), False) * cot).sum().backward()
        got["dwave_eval"] = digest(w.grad)
    for k, v in got.items():
        ref = g[f"{tag}__{k}"]
        err = np.linalg.norm(v - ref) / np.linalg.norm(ref)
        # spectrogram gradients: fp64 rounding.  Waveform: the reference's torch.stft chain and the oracle's framing +
        # rfft agree to 1.4e-5 (mn04) and 5.4e-6 (attention head)
        assert err < (1e-4 if k == "dwave_eval" else 1e-9), f"{tag} {k}: rel {err:.2e}"
