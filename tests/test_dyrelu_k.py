"""DyReLU-B with M = dyrelu_k linear pieces without a GPU: the module tree and state_dict against the reference's, the
range check, the fp64 oracle of tests/dyrelu_util.py against the reference's goldens, and the host-side argument checks
of the entry points that take M."""
import contextlib
import io
import json
import os

import numpy as np
import pytest
import torch

from efficientat_b200._lib import EatError, lib
from tests import dyrelu_util as du
from tests.util import GOLDEN, fmap_digest, golden, topk_match

torch.set_num_threads(8)


def _sd64(model):
    return {k: v.double() if v.is_floating_point() else v.clone() for k, v in model.state_dict().items()}


def _temperature(model):
    return float(model.layers[0].depth_conv.temperature)


@pytest.mark.parametrize("M", [1, 2, 3, 4])
def test_state_dict_matches_reference(M):
    model = du.build_model(M, calibrated=False)
    sd = model.state_dict()
    if M == 2:
        want = json.load(open(os.path.join(GOLDEN, "statedict_dymn04.json")))
        assert {k: list(v.shape) for k, v in sd.items()} == want
    else:
        g = golden(du.tag(M))
        assert list(sd) == [str(n) for n in g["sd_names"]]
        assert [",".join(map(str, v.shape)) for v in sd.values()] == [str(s) for s in g["sd_shapes"]]
    for blk in model.layers:
        act = blk.depth_act
        C = blk.cnf.expanded_channels
        assert act.M == M and act.coef_net[0].out_features == 2 * M * C
        assert act.lambdas.tolist() == [1.0] * M + [0.5] * M
        assert act.init_v.tolist() == [1.0] + [0.0] * (2 * M - 1)


@pytest.mark.parametrize("M", [0, 5, 8])
def test_pieces_outside_1_to_4_raise(M):
    from efficientat_b200.models.dymn.model import get_model
    with pytest.raises(NotImplementedError, match=r"1\.\.4"), contextlib.redirect_stdout(io.StringIO()):
        get_model(width_mult=0.4, dyrelu_k=M, verbose=False)


@pytest.mark.parametrize("M", du.PIECES)
def test_oracle_eval_matches_reference(M):
    g = golden(du.tag(M))
    model = du.build_model(M)
    spec, _ = du.net_inputs()
    assert np.abs(fmap_digest([spec]) - g["spec_digest"]).max() == 0
    with torch.no_grad():
        logits, feat, fmaps = du.dymn_forward(_sd64(model), spec.double(), M, temperature=_temperature(model),
                                              return_fmaps=True)
    assert np.abs(logits.numpy() - g["eval_logits"]).max() < 1e-4
    assert np.abs(feat.numpy() - g["eval_feat"]).max() < 2e-4
    d = fmap_digest(fmaps)
    assert np.abs(d - g["eval_fmaps"]).max() < 1e-3 * max(1.0, np.abs(g["eval_fmaps"]).max())
    assert topk_match(logits.numpy(), g["eval_logits"], 10, tie_tol=1e-5)


@pytest.mark.parametrize("M", du.PIECES)
def test_oracle_train_matches_reference(M):
    g = golden(du.tag(M))
    model = du.build_model(M)
    sd = _sd64(model)
    params = {k for k, _ in model.named_parameters()}
    for k in params:
        sd[k].requires_grad_(True)
    spec, y = du.net_inputs()
    logits, _ = du.dymn_forward(sd, spec.double(), M, training=True, temperature=_temperature(model))
    loss = torch.nn.functional.binary_cross_entropy_with_logits(logits, y.double())
    loss.backward()
    assert abs(loss.item() - float(g["train_loss"])) < 1e-5
    assert np.abs(logits.detach().numpy() - g["train_logits"]).max() < 1e-4
    names = [str(n) for n in g["grad_names"]]
    assert set(names) == params
    for i, n in enumerate(names):
        gn = sd[n].grad.norm().item()
        assert abs(gn - g["grad_norm"][i]) <= 2e-3 * g["grad_norm"][i] + 1e-7, n
    for i, n in enumerate(str(s) for s in g["bn_names"]):
        assert np.abs(sd[n + ".running_mean"][:4].numpy() - g["bn_rm4"][i]).max() < 1e-5, n
        assert np.abs(sd[n + ".running_var"][:4].numpy() - g["bn_rv4"][i]).max() < 1e-5, n


def test_oracle_with_one_piece_less_differs():
    """the planted defect of the GPU tests (M - 1 of M pieces) moves the oracle's output by far more than any bound"""
    for M in (3, 4):
        model = du.build_model(M)
        sd = _sd64(model)
        spec, _ = du.net_inputs()
        with torch.no_grad():
            a, _ = du.dymn_forward(sd, spec.double(), M, temperature=_temperature(model))
            b, _ = du.dymn_forward(sd, spec.double(), M, temperature=_temperature(model), pieces_used=M - 1)
        assert (a - b).abs().max() > 1e-2, M


def test_oracle_m2_is_net_oracle():
    from oracle import net_oracle
    from tests.util import build_model, net_inputs
    model = build_model("dymn04")
    sd = _sd64(model)
    spec, _ = net_inputs("dymn04")
    with torch.no_grad():
        a, _ = du.dymn_forward(sd, spec.double(), 2, temperature=_temperature(model))
        b, _ = net_oracle.dymn_forward(sd, spec.double(), width_mult=0.4, temperature=_temperature(model))
    assert torch.equal(a, b)


# argument checks of the entry points that take M happen on the host before any launch: the fake pointers below are
# never dereferenced
FAKE = 4096


def _fwd(dtype=0, B=2, F=8, T=13, C=64, k=3, stride=1, M=3, eval_=True, in_scale=0, stats=0, shift=None, lam=None):
    e = FAKE if eval_ else 0
    lib().dw_conv_fwd_dy_m(FAKE, FAKE, 0, FAKE, dtype, B, F, T, C, k, stride, in_scale, in_scale, 0, e,
                           e if shift is None else shift, e, e if lam is None else lam, e, e, e, M, stats, stats, None)


def _act_fwd(dtype=0, B=2, F=8, T=13, C=64, M=3, null=False):
    lib().dy_act_fwd_m(FAKE, FAKE, dtype, FAKE, FAKE, 0 if null else FAKE, FAKE, FAKE, FAKE, FAKE, M, B, F, T, C, None)


def _act_bwd(dtype=0, B=2, F=8, T=13, C=64, M=3, null=False):
    lib().dy_act_bwd_m(FAKE, FAKE, FAKE, dtype, FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, 0 if null else FAKE,
                       M, B, F, T, C, None)


@pytest.mark.parametrize("fn", [_fwd, _act_fwd, _act_bwd])
@pytest.mark.parametrize("kw,code,msg", [
    (dict(M=0), 3, r"1\.\.4 linear pieces \(got 0\)"), (dict(M=5), 3, r"1\.\.4 linear pieces \(got 5\)"),
    (dict(dtype=2), 1, "dtype"), (dict(B=-1), 1, "B >= 0"), (dict(F=0), 1, "To?, C >= 1"), (dict(C=66), 1, "multiple of 4")])
def test_entry_points_reject(fn, kw, code, msg):
    with pytest.raises(EatError, match=rf"code {code}\): .*{msg}"):
        fn(**kw)


@pytest.mark.parametrize("kw,code,msg", [
    (dict(k=7), 3, "k must be 3 or 5"), (dict(stride=3), 3, "stride must be 1 or 2"),
    (dict(dtype=1, C=68), 1, "multiple of 8"), (dict(shift=0), 1, "come in sets"), (dict(lam=0), 1, "come in sets"),
    (dict(in_scale=FAKE), 1, "training forward"), (dict(stats=FAKE), 1, "training forward")])
def test_dw_fwd_rejects(kw, code, msg):
    with pytest.raises(EatError, match=rf"code {code}\): .*{msg}"):
        _fwd(**kw)


@pytest.mark.parametrize("fn", [_act_fwd, _act_bwd])
def test_dy_act_rejects_null_pointers(fn):
    with pytest.raises(EatError, match=r"code 1\): .*every tensor pointer"):
        fn(null=True)


def test_coef_bwd_rejects():
    L = lib()
    with pytest.raises(EatError, match=r"code 3\): .*1\.\.4 linear pieces"):
        L.dyrelu_coef_bwd_m(FAKE, FAKE, FAKE, FAKE, 120, 5, None)
    with pytest.raises(EatError, match=r"code 1\): .*multiple of 2M = 6"):
        L.dyrelu_coef_bwd_m(FAKE, FAKE, FAKE, FAKE, 128, 3, None)
    with pytest.raises(EatError, match=r"code 1\): .*every tensor pointer"):
        L.dyrelu_coef_bwd_m(FAKE, 0, FAKE, FAKE, 120, 3, None)
    L.dyrelu_coef_bwd_m(FAKE, FAKE, FAKE, FAKE, 0, 3, None)             # n = 0: returns before any launch


@pytest.mark.parametrize("fn", [_fwd, _act_fwd, _act_bwd])
@pytest.mark.parametrize("M", [1, 2, 3, 4])
def test_empty_batch_is_noop(fn, M):
    fn(B=0, M=M)                 # returns before any launch: no device is touched


def test_training_form_accepted_without_theta():
    _fwd(B=0, eval_=False, in_scale=FAKE, stats=FAKE)
