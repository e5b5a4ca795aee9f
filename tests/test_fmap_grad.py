"""Gradients through the embedding and the feature maps, the parts that need no GPU: the fp64 oracle against the
unmodified reference's gradients (tests/golden/make_golden_fmap_grad.py), the routing of train() with return_fmaps and
of each unused output through the autograd glue, and the host-side argument checks of eat_fmap_grad_nhwc.  The kernel
and the engine's numerics are in tests/test_gpu_zz_fmap_grad.py."""
import contextlib
import subprocess

import numpy as np
import pytest
import torch

from efficientat_b200 import _lib
from efficientat_b200._lib import EatError, lib
from tests import fmap_grad_util as fu
from tests.input_grad_util import digest
from tests.util import golden

FAKE = 4096                 # never dereferenced: validation comes first


# ------------------------------------------------------------------------------------------------ oracle vs reference
@pytest.mark.parametrize("kind", fu.LOSSES)
@pytest.mark.parametrize("tag", list(fu.CASES))
def test_fp64_oracle_matches_reference_gradients(tag, kind):
    g = golden("fmap_grad")
    model = fu.build_model(tag, g)
    names = [n for n, _ in model.named_parameters()]
    assert names == list(g[tag + "__names"])
    spec, y = fu.net_inputs()
    loss, dx, grads = fu.oracle_grads(tag, model, kind, spec, y)
    pfx = f"{tag}__{kind}__"
    assert abs(loss - g[pfx + "loss"]) <= 1e-10 * max(1.0, abs(g[pfx + "loss"]))
    norms, samples = fu.grad_digest(grads, names)
    # fp64 on both sides: the oracle and the reference agree to rounding
    ref_norm = g[pfx + "grad_norm"]
    # a floor for the gradients that vanish analytically (the BatchNorm shift before the next BatchNorm: ~1e-14 rounding)
    floor = 1e-6 * ref_norm.max()
    assert (np.abs(norms - ref_norm) / (ref_norm + floor)).max() < 1e-8
    assert (np.abs(samples - g[pfx + "grad_samples"]) / (ref_norm + floor)[:, None]).max() < 1e-8
    ref = g[pfx + "dspec"]
    assert np.linalg.norm(digest(dx) - ref) / np.linalg.norm(ref) < 1e-9


def test_each_map_term_moves_the_reference_gradients():
    """the goldens see every map: leaving block 7's term out of the oracle's loss moves the gradients far outside the
    bounds above"""
    g = golden("fmap_grad")
    tag = "mn04"
    model = fu.build_model(tag, g)
    names = [n for n, _ in model.named_parameters()]
    spec, y = fu.net_inputs()
    _, dx, grads = fu.oracle_grads(tag, model, "fmaps", spec, y, skip=(7,))
    norms, _ = fu.grad_digest(grads, names)
    assert np.abs(norms / g[tag + "__fmaps__grad_norm"] - 1).max() > 1e-3
    ref = g[tag + "__fmaps__dspec"]
    assert np.linalg.norm(digest(dx) - ref) / np.linalg.norm(ref) > 1e-3


# ------------------------------------------------------------------------------------------------ routing
def _eng_class():
    from efficientat_b200.engine import MNEngine

    class Eng(MNEngine):
        def __init__(self, training, calls):
            self.model = torch.nn.Linear(1, 1)
            self.model.train(training)
            self.calls = calls

        def _forward_eval(self, x, return_fmaps=False):
            self.calls.append(("eval", return_fmaps))
            return x.sum(), None, [] if return_fmaps else None
    return Eng


def test_train_with_fmaps_takes_the_graph_route(monkeypatch):
    """engine._dispatch (host logic, the forwards stubbed out): train() + return_fmaps -> mn_train_forward_fmaps, with a
    graph when a parameter or the input requires grad; eval() + fmaps without an input gradient -> the folded forward;
    eval() + an input that requires grad + fmaps still raises"""
    from efficientat_b200 import autograd
    calls = []
    monkeypatch.setattr(autograd, "mn_train_forward_fmaps",
                        lambda e, x, ng: (calls.append(("train_fmaps", ng)), (x, None, ["m"]))[1])
    monkeypatch.setattr(autograd, "mn_train_forward", lambda e, x, ng: (calls.append(("train", ng)), (x, None))[1])
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())
    Eng = _eng_class()
    x = torch.zeros(1, 1, 2, 2)
    e = Eng(True, calls)
    assert e._dispatch(x, True)[2] == ["m"]
    assert e._dispatch(x, False)[2] is None
    with torch.no_grad():
        e._dispatch(x, True)
    for p in e.model.parameters():
        p.requires_grad_(False)
    e._dispatch(x, True)
    e._dispatch(x.clone().requires_grad_(), True)
    Eng(False, calls)._dispatch(x, True)
    with pytest.raises(NotImplementedError, match="return_fmaps"):
        Eng(False, calls)._dispatch(x.clone().requires_grad_(), True)
    assert calls == [("train_fmaps", True), ("train", True), ("train_fmaps", False), ("train_fmaps", False),
                     ("train_fmaps", True), ("eval", True)]


class _FakeEngine:
    """stands in for MNEngine behind the autograd Function: CPU tensors, records what _backward receives"""
    B, C, NMAP = 2, 3, 17

    def __init__(self):
        self.model = torch.nn.Module()
        self.model.trunk = torch.nn.Linear(2, 2)
        self.model.classifier = torch.nn.Linear(2, 2)
        self.calls = []

    def param_list(self):
        return list(self.model.parameters())

    def _forward_train(self, x, frozen=False, fmaps=False):
        S = {"fmaps": [torch.randn(self.B, 4, 5, self.C) for _ in range(self.NMAP)] if fmaps else None}
        return torch.randn(self.B, 7), torch.randn(self.B, self.C), S

    def _backward(self, S, dlogits, on_ready=None, input_grad=False, wanted=None, dembed=None, dfmaps=None):
        self.calls.append(dict(dlogits=dlogits is not None, dembed=dembed is not None,
                               dfmaps=None if dfmaps is None else [g is not None for g in dfmaps], input_grad=input_grad))
        G = {p: torch.ones_like(p) for p in self.param_list()}
        G["x"] = torch.ones(self.B, 1, 4, 5)
        return G


def _fake_run(loss_fn, fmaps=True, input_grad=False):
    from efficientat_b200 import autograd
    eng = _FakeEngine()
    x = torch.zeros(2, 1, 4, 5, requires_grad=input_grad)
    if fmaps:
        logits, feat, maps = autograd.mn_train_forward_fmaps(eng, x, True)
    else:
        (logits, feat), maps = autograd.mn_train_forward(eng, x, True), None
    loss_fn(logits, feat, maps).backward()
    return eng, x


def test_unused_outputs_arrive_as_none_and_skip_the_classifier():
    # the embedding alone: no logits gradient, so the classifier is not part of the graph
    eng, _ = _fake_run(lambda lo, fe, m: fe.sum(), fmaps=False)
    assert eng.calls == [dict(dlogits=False, dembed=True, dfmaps=None, input_grad=False)]
    assert eng.model.classifier.weight.grad is None and eng.model.classifier.bias.grad is None
    assert eng.model.trunk.weight.grad is not None
    # one middle map (block 7) and the logits
    eng, _ = _fake_run(lambda lo, fe, m: lo.sum() + m[7].mean())
    assert eng.calls[0]["dlogits"] and not eng.calls[0]["dembed"]
    assert eng.calls[0]["dfmaps"] == [i == 7 for i in range(17)]
    assert eng.model.classifier.weight.grad is not None
    # a per-frame head on the last map's frequency mean, with the input's gradient
    eng, x = _fake_run(lambda lo, fe, m: m[-1].mean(2).pow(2).sum(), input_grad=True)
    assert eng.calls[0] == dict(dlogits=False, dembed=False, dfmaps=[i == 16 for i in range(17)], input_grad=True)
    assert x.grad is not None
    # the logits alone: the call of a plain training step
    eng, _ = _fake_run(lambda lo, fe, m: lo.sum(), fmaps=False)
    assert eng.calls == [dict(dlogits=True, dembed=False, dfmaps=None, input_grad=False)]


def test_maps_are_views_in_the_reference_layout_and_in_place_edits_raise():
    from efficientat_b200 import autograd
    eng = _FakeEngine()
    x = torch.zeros(2, 1, 4, 5)
    _, feat, maps = autograd.mn_train_forward_fmaps(eng, x, True)
    assert len(maps) == 17 and feat.grad_fn is not None
    assert all(m.shape == (2, 3, 4, 5) and m.grad_fn is not None for m in maps)
    assert maps[3].permute(0, 2, 3, 1).is_contiguous()               # NHWC storage
    with pytest.raises(RuntimeError):
        maps[3].mul_(2)
        maps[3].sum().backward()
    # without a graph: plain tensors
    _, feat, maps = autograd.mn_train_forward_fmaps(eng, x, False)
    assert feat.grad_fn is None and all(m.grad_fn is None for m in maps)


def test_missing_map_gradient_launches_nothing(monkeypatch):
    """engine._add_fmap_grad: an unused map (gradient None) leaves the running gradient as it is, with no launch"""
    from efficientat_b200.engine import MNEngine

    class Boom:
        def __getattr__(self, name):
            raise AssertionError(f"launch {name}")
    monkeypatch.setattr("efficientat_b200.engine.lib", lambda: Boom())
    eng = MNEngine.__new__(MNEngine)
    dy = torch.zeros(1)
    assert eng._add_fmap_grad(dy, None, (1, 1, 1, 1)) is dy
    assert eng._add_fmap_grad(None, None, (1, 1, 1, 1)) is None


# ------------------------------------------------------------------------------------------------ eat_fmap_grad_nhwc
def _fg(src=FAKE, sd=0, strides=(60, 20, 5, 1), dst=FAKE, dd=0, B=2, C=3, F=4, T=5, acc=0):
    lib().fmap_grad_nhwc(src, sd, *strides, dst, dd, B, C, F, T, acc, 0)


def test_fmap_grad_is_exported():
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True).stdout
    assert " T eat_fmap_grad_nhwc" in out


@pytest.mark.parametrize("kw", [
    dict(sd=2), dict(dd=2), dict(sd=-1), dict(dd=3),
    dict(B=-1), dict(C=-1), dict(F=-2), dict(T=-1),
    dict(strides=(-60, 20, 5, 1)), dict(strides=(60, -1, 5, 1)), dict(strides=(60, 20, -5, 1)), dict(strides=(60, 20, 5, -1)),
    dict(src=0), dict(dst=0),
])
def test_fmap_grad_rejects_bad_arguments_before_any_launch(kw):
    with pytest.raises(EatError, match="fmap grad") as e:
        _fg(**kw)
    assert "code 1" in str(e.value)                 # EAT_ERR_ARG


def test_fmap_grad_empty_batch_is_a_no_op():
    _fg(B=0)
    _fg(B=0, src=0, dst=0)
    _fg(C=0, src=0, dst=0)
    _fg(B=0, sd=1, dd=1, strides=(0, 0, 0, 0))
    with pytest.raises(EatError):
        _fg(B=0, sd=2)                              # the checks still come first
    with pytest.raises(EatError):
        _fg(B=0, strides=(-1, 0, 0, 0))
