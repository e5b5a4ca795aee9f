"""Generate tests/golden/dymn04_dyrelu_k{1,3,4}.npz by running the UNMODIFIED reference DyMN with
get_model(width_mult=0.4, dyrelu_k=M) for M = 1, 3 and 4 linear pieces in DyReLU-B.

Run where a checkout of the original project exists (read-only), named by $EAT_REFERENCE_DIR:
    EAT_REFERENCE_DIR=<checkout> python tests/golden/make_golden_dyrelu_k.py
The recipe is make_golden.py's run_net at 2 s (B = 2): synth_state_(seed=7), one training-mode BatchNorm calibration
pass, eval logits, embeddings and per-block feature-map digests, then one training step with BCE and dropout off (loss,
logits, per-parameter gradient norms and samples, BatchNorm running statistics).  Each file also records the
state_dict's keys and shapes, which differ from M = 2 only in coef_net and the [2M] DyReLU buffers.  No existing
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
    from models.dymn.model import get_model as ref_dymn  # noqa: E402

import warnings  # noqa: E402
warnings.filterwarnings("ignore")
torch.set_num_threads(8)

WIDTH, SAMPLES, BATCH = 0.4, 64000, 2
PIECES = (1, 3, 4)


def run(M):
    out = os.path.join(HERE, f"dymn04_dyrelu_k{M}.npz")
    assert not os.path.exists(out), f"{out} exists; this script only writes new files"
    torch.manual_seed(0)
    with contextlib.redirect_stdout(io.StringIO()):
        model = ref_dymn(width_mult=WIDTH, dyrelu_k=M)
    synth_state_(model, seed=7)
    sd = model.state_dict()
    frames = 1 + (SAMPLES - 1) // 320
    spec = synth_waveform(BATCH, 128 * frames, seed=21, std=0.7).view(BATCH, 1, 128, frames)
    model.train()
    for _, m in bn_modules(model):
        m.momentum = 1.0
    with torch.no_grad():
        model(spec)
    for _, m in bn_modules(model):
        m.momentum = 0.01
        m.num_batches_tracked.zero_()
    cal_rm, cal_rv = get_bn_stats(model)
    res = {"spec_digest": fmap_digest([spec]), "cal_rm": cal_rm.numpy(), "cal_rv": cal_rv.numpy(),
           "sd_names": np.array(list(sd)), "sd_shapes": np.array([",".join(map(str, v.shape)) for v in sd.values()])}
    model.eval()
    with torch.no_grad():
        logits, feat = model(spec)
        _, fmaps = model(spec, return_fmaps=True)
    res.update(eval_logits=logits.numpy(), eval_feat=feat.numpy(), eval_fmaps=fmap_digest(fmaps))
    model.train()
    for m in model.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    y = synth_labels(BATCH, 527, seed=5)
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
    print(f"dymn04 dyrelu_k={M}: eval logits absmax {logits.abs().max().item():.4g}, train loss {loss.item():.6f}")


if __name__ == "__main__":
    for M in (int(a) for a in sys.argv[1:]) if len(sys.argv) > 1 else PIECES:
        run(M)
