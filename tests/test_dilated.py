"""MN's dilated tail without a GPU: the fp64 oracle of tests/dilated_util.py against the reference's goldens, the module tree
of get_model(dilated=True), and the host-side argument checks of the dilated depthwise entry points."""
import contextlib
import io

import numpy as np
import pytest
import torch

from efficientat_b200._lib import EatError, lib
from tests import dilated_util as du
from tests.util import fmap_digest, golden, topk_match

torch.set_num_threads(8)


def _model(**kw):
    from efficientat_b200.models.mn.model import get_model
    with contextlib.redirect_stdout(io.StringIO()):
        return get_model(width_mult=kw.pop("width_mult", 1.0), verbose=False, **kw)


@pytest.mark.parametrize("tag", list(du.CASES))
def test_oracle_eval_matches_reference(tag):
    g = golden(tag)
    width, _, _, rt, _ = du.CASES[tag]
    sd = {k: v.double() if v.is_floating_point() else v.clone() for k, v in du.build_model(tag).state_dict().items()}
    spec, _ = du.net_inputs(tag)
    assert np.abs(fmap_digest([spec]) - g["spec_digest"]).max() == 0
    with torch.no_grad():
        logits, feat, fmaps = du.mn_forward(sd, spec.double(), width_mult=width, reduced_tail=rt, dilated=True,
                                            return_fmaps=True)
    assert list(fmaps[-1].shape) == list(g["last_shape"])
    assert np.abs(logits.numpy() - g["eval_logits"]).max() < 1e-4
    assert np.abs(feat.numpy() - g["eval_feat"]).max() < 2e-4
    d = fmap_digest(fmaps)
    assert np.abs(d - g["eval_fmaps"]).max() < 1e-3 * max(1.0, np.abs(g["eval_fmaps"]).max())
    assert topk_match(logits.numpy(), g["eval_logits"], 10, tie_tol=1e-5)


@pytest.mark.parametrize("tag", [t for t, c in du.CASES.items() if c[4]])
def test_oracle_train_matches_reference(tag):
    g = golden(tag)
    width, _, _, rt, _ = du.CASES[tag]
    model = du.build_model(tag)
    sd = {k: v.double() if v.is_floating_point() else v.clone() for k, v in model.state_dict().items()}
    params = {k for k, _ in model.named_parameters()}
    for k in params:
        sd[k].requires_grad_(True)
    spec, y = du.net_inputs(tag)
    logits, _ = du.mn_forward(sd, spec.double(), width_mult=width, reduced_tail=rt, dilated=True, training=True)
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


def test_oracle_undilated_block_differs():
    """the planted defect of the GPU tests (block 13 undilated) changes the oracle's output by far more than any bound"""
    tag = "mn04_dilated"
    width = du.CASES[tag][0]
    sd = {k: v.double() if v.is_floating_point() else v.clone() for k, v in du.build_model(tag).state_dict().items()}
    spec, _ = du.net_inputs(tag)
    with torch.no_grad():
        a, _ = du.mn_forward(sd, spec.double(), width_mult=width, dilated=True)
        b, _ = du.mn_forward(sd, spec.double(), width_mult=width, dilated=True, undilated_blocks=(13,))
    assert (a - b).abs().max() > 1e-2


@pytest.mark.parametrize("rt", [False, True])
def test_module_tree(rt):
    from efficientat_b200.models.mn.block_types import InvertedResidual
    m = _model(width_mult=0.4, dilated=True, reduced_tail=rt)
    plain = _model(width_mult=0.4, reduced_tail=rt)
    blocks = [b for b in m.features if isinstance(b, InvertedResidual)]
    for b in blocks[:-3]:
        dw = [c for c in b.block.modules() if isinstance(c, torch.nn.Conv2d) and c.groups > 1][0]
        assert dw.dilation == (1, 1)
    for b, res in zip(blocks[-3:], (False, True, True)):
        dw = [c for c in b.block.modules() if isinstance(c, torch.nn.Conv2d) and c.groups > 1][0]
        assert dw.stride == (1, 1) and dw.dilation == (2, 2) and dw.padding == (4, 4) and dw.kernel_size == (5, 5)
        assert b.use_res_connect is res
    assert {k: v.shape for k, v in m.state_dict().items()} == {k: v.shape for k, v in plain.state_dict().items()}
    assert list(m.state_dict()) == list(plain.state_dict())


def test_engine_plan_uses_effective_stride():
    m = _model(width_mult=0.4, dilated=True)
    blks = m.engine().blocks
    assert [(b.stride, b.dil) for b in blks[-3:]] == [(1, 2), (1, 2), (1, 2)]
    assert all(b.dil == 1 for b in blks[:-3])


def test_dymn_dilated_still_raises():
    from efficientat_b200.models.dymn.model import dymn
    with pytest.raises(NotImplementedError), contextlib.redirect_stdout(io.StringIO()):
        dymn(width_mult=0.4, dilated=True)


# argument checks of the dilated entry points happen on the host before any launch: null pointers never reach a device
def _fwd(dtype=0, B=2, F=8, T=13, C=64, k=5, stride=1, dil=2, in_scale=0, scale=0, shift=0, pool=0):
    lib().dw_conv_fwd_dil(0, 0, 0, dtype, B, F, T, C, k, stride, dil, in_scale, in_scale, 0, scale, shift, 2, pool, 0, 0, None)


def _dgrad(dtype=0, B=2, F=8, T=13, C=64, k=5, stride=1, dil=2):
    lib().dw_conv_dgrad_dil(0, 0, 0, 0, dtype, B, F, T, C, k, stride, dil, None)


def _wgrad(dtype=0, B=2, F=8, T=13, C=64, k=5, stride=1, dil=2):
    lib().dw_conv_wgrad_dil(0, 0, 0, 0, 0, 0, dtype, B, F, T, C, k, stride, dil, None)


@pytest.mark.parametrize("fn", [_fwd, _dgrad, _wgrad])
@pytest.mark.parametrize("kw,msg", [
    (dict(dil=1), "dilation must be 2"), (dict(dil=3), "dilation must be 2"), (dict(stride=2), "stride 1"),
    (dict(k=7), "k must be 3 or 5"), (dict(k=1), "k must be 3 or 5"), (dict(C=66), "multiple of 4"),
    (dict(dtype=1, C=68), "multiple of 8"), (dict(dtype=2), "dtype"), (dict(F=0), "F, T, C"), (dict(B=-1), "B >= 0")])
def test_dilated_entry_points_reject(fn, kw, msg):
    with pytest.raises(EatError, match=msg):
        fn(**kw)


@pytest.mark.parametrize("fn", [_fwd, _dgrad, _wgrad])
def test_dilated_entry_points_empty_batch_is_noop(fn):
    fn(B=0)                  # returns before any launch: no device is touched


def test_dilated_fwd_rejects_mixed_modes():
    with pytest.raises(EatError, match="training forward"):
        _fwd(B=0, in_scale=1, scale=1, shift=1)
    with pytest.raises(EatError, match="pairs"):
        _fwd(B=0, scale=1)
