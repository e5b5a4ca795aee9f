"""Generate tests/golden/mn04_dilated.npz, mn04_dilated_rt.npz and mn10_dilated_10s.npz by running the UNMODIFIED
reference MN with get_model(dilated=True) (and reduced_tail=True for the _rt file).

Run where a checkout of the original project exists (read-only), named by $EAT_REFERENCE_DIR:
    EAT_REFERENCE_DIR=<checkout> python tests/golden/make_golden_dilated.py
The recipe is make_golden.py's run_net: synth_state_(seed=7), one training-mode BatchNorm calibration pass, eval logits,
features and feature-map digests, then one training step with BCE and dropout off (loss, logits, per-parameter gradient
norms and samples, BatchNorm running statistics).  mn10_dilated_10s.npz (the benchmark's 10 s shape) holds the eval part
only.  The state_dict of a dilated model equals the undilated one, so no statedict_*.json is written, and no existing
golden file is touched.
"""
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
from efficientat_b200.synth import bn_modules, get_bn_stats, synth_labels, synth_state_, synth_waveform  # noqa: E402
from tests.util import fmap_digest  # noqa: E402

os.chdir(REF)            # helpers/utils.py opens metadata/ relative to CWD
sys.path.insert(0, REF)
with contextlib.redirect_stdout(io.StringIO()):
    from models.mn.model import get_model as ref_mn  # noqa: E402

import warnings  # noqa: E402
warnings.filterwarnings("ignore")
torch.set_num_threads(8)

# tag: (width, samples, batch, reduced_tail, training step)
CASES = {"mn04_dilated": (0.4, 64000, 2, False, True),
         "mn04_dilated_rt": (0.4, 64000, 2, True, True),
         "mn10_dilated_10s": (1.0, 320000, 2, False, False)}


def run(tag):
    width, n_samples, batch, reduced_tail, train = CASES[tag]
    out = os.path.join(HERE, f"{tag}.npz")
    assert not os.path.exists(out), f"{out} exists; this script only writes new files"
    torch.manual_seed(0)
    with contextlib.redirect_stdout(io.StringIO()):
        model = ref_mn(width_mult=width, dilated=True, reduced_tail=reduced_tail)
    synth_state_(model, seed=7)
    frames = 1 + (n_samples - 1) // 320
    spec = synth_waveform(batch, 128 * frames, seed=21, std=0.7).view(batch, 1, 128, frames)
    model.train()
    for _, m in bn_modules(model):
        m.momentum = 1.0
    with torch.no_grad():
        model(spec)
    for _, m in bn_modules(model):
        m.momentum = 0.01
        m.num_batches_tracked.zero_()
    cal_rm, cal_rv = get_bn_stats(model)
    res = {"spec_digest": fmap_digest([spec]), "cal_rm": cal_rm.numpy(), "cal_rv": cal_rv.numpy()}
    model.eval()
    with torch.no_grad():
        logits, feat = model(spec)
        _, fmaps = model._forward_impl(spec, return_fmaps=True)
    res.update(eval_logits=logits.numpy(), eval_feat=feat.numpy(), eval_fmaps=fmap_digest(fmaps),
               last_shape=np.array(fmaps[-1].shape))
    if train:
        model.train()
        for m in model.modules():
            if isinstance(m, torch.nn.Dropout):
                m.p = 0.0
        y = synth_labels(batch, 527, seed=5)
        logits_t, _ = model(spec)
        loss = torch.nn.functional.binary_cross_entropy_with_logits(logits_t, y)
        loss.backward()
        names, gnorm, gsamp = [], [], []
        for n, p in model.named_parameters():
            names.append(n)
            g = p.grad.flatten()
            gnorm.append(g.double().norm().item())
            gsamp.append(g[torch.linspace(0, g.numel() - 1, 4).long()].numpy())
        bn_names, bn_rm, bn_rv = [], [], []
        for n, m in model.named_modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                bn_names.append(n)
                bn_rm.append(m.running_mean[:4].numpy().copy())
                bn_rv.append(m.running_var[:4].numpy().copy())
        res.update(train_logits=logits_t.detach().numpy(), train_loss=np.float64(loss.item()),
                   grad_names=np.array(names), grad_norm=np.array(gnorm), grad_samples=np.stack(gsamp),
                   bn_names=np.array(bn_names), bn_rm4=np.stack(bn_rm), bn_rv4=np.stack(bn_rv))
    np.savez_compressed(out, **res)
    print(tag, "last conv", tuple(fmaps[-1].shape), "eval logits absmax", logits.abs().max().item())


if __name__ == "__main__":
    for t in (sys.argv[1:] or list(CASES)):
        run(t)
