"""Generate tests/golden/fmap_grad.npz by running the UNMODIFIED reference: training-step gradients of losses on the
embedding (`features`) and on the 17 feature maps, for mn04, mn04 with the attention head (4 heads), mn04 with
dilated=True, and dymn04 with dyrelu_k 2 and 3.

Run where a checkout of the original project exists (read-only), named by $EAT_REFERENCE_DIR:
    EAT_REFERENCE_DIR=<checkout> python tests/golden/make_golden_fmap_grad.py
The recipe is make_golden_dilated.py's: the seeded state (synth_state_(seed=7); mha_state_ for the attention head), one
training-mode BatchNorm calibration pass on the 2 s spectrogram (B = 2) of tests/fmap_grad_util.net_inputs, dropout 0,
then model.double().  The reference returns either the features or the maps from one forward, so each net has two
training steps (tests/fmap_grad_util.loss): bce(logits) + <r, features>, and bce(logits) + sum_i <R_i, fmap_i> / numel_i,
with seeded r and R_i.  Recorded per step: the loss, every parameter gradient's norm and 4 samples, and the input
spectrogram's gradient (tests/input_grad_util.digest).  No existing golden file is touched."""
import contextlib
import io
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
REF = os.environ["EAT_REFERENCE_DIR"]
sys.path.insert(0, REPO)
from efficientat_b200.synth import bn_modules, get_bn_stats  # noqa: E402
from tests import fmap_grad_util as fu  # noqa: E402
from tests.input_grad_util import digest  # noqa: E402

os.chdir(REF)            # helpers/utils.py opens metadata/ relative to CWD
sys.path.insert(0, REF)
with contextlib.redirect_stdout(io.StringIO()):
    from models.dymn.model import get_model as ref_dymn  # noqa: E402
    from models.mn.model import get_model as ref_mn  # noqa: E402

import warnings  # noqa: E402
warnings.filterwarnings("ignore")
torch.set_num_threads(8)


def build(tag):
    kind, kw = fu.CASES[tag]
    torch.manual_seed(0)
    with contextlib.redirect_stdout(io.StringIO()):
        m = (ref_mn if kind == "mn" else ref_dymn)(width_mult=fu.WIDTH, **kw)
    return fu.state_(tag, m)


def run(tag, res):
    model = build(tag)
    spec, y = fu.net_inputs()
    model.train()
    for _, m in bn_modules(model):
        m.momentum = 1.0
    with torch.no_grad():
        model(spec)
    for _, m in bn_modules(model):
        m.momentum = 0.01
        m.num_batches_tracked.zero_()
    cal_rm, cal_rv = get_bn_stats(model)
    res[tag + "__cal_rm"], res[tag + "__cal_rv"] = cal_rm.numpy(), cal_rv.numpy()
    for m in model.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    model.double()
    names = [n for n, _ in model.named_parameters()]
    res[tag + "__names"] = np.array(names)
    for kind in fu.LOSSES:
        model.zero_grad(set_to_none=True)
        x = spec.double().requires_grad_(True)
        if kind == "embed":
            logits, feat = model(x)
            fmaps = []
        elif fu.CASES[tag][0] == "mn":
            logits, fmaps = model._forward_impl(x, return_fmaps=True)
            feat = None
        else:
            logits, fmaps = model(x, return_fmaps=True)
            feat = None
        assert len(fmaps) in (0, 17)
        r, R = fu.probes((fu.BATCH, model_feat_dim(fmaps, feat)), [m.shape for m in fmaps])
        loss = fu.loss(kind, logits, feat, fmaps, y, r, R)
        loss.backward()
        norms, samples = fu.grad_digest({n: p.grad for n, p in model.named_parameters()}, names)
        res[f"{tag}__{kind}__loss"] = np.float64(loss.item())
        res[f"{tag}__{kind}__grad_norm"] = norms
        res[f"{tag}__{kind}__grad_samples"] = samples
        res[f"{tag}__{kind}__dspec"] = digest(x.grad)
        print(f"{tag} {kind}: loss {loss.item():.6f}, |dspec| {res[f'{tag}__{kind}__dspec'][0]:.6g}")


def model_feat_dim(fmaps, feat):
    return feat.shape[1] if feat is not None else fmaps[-1].shape[1]


if __name__ == "__main__":
    out = os.path.join(HERE, "fmap_grad.npz")
    assert not os.path.exists(out), f"{out} exists; this script only writes new files"
    res = {}
    for tag in fu.CASES:
        run(tag, res)
    np.savez_compressed(out, **res)
