"""Test helpers for gradients through the embedding and the feature maps: the nets, inputs and probes of
tests/golden/make_golden_fmap_grad.py, and an fp64 oracle of its two losses built on oracle/net_oracle.py,
tests/dilated_util.py, tests/dyrelu_util.py and tests/mha_util.py.

The reference returns either `features` or the feature maps from one forward, never both, so every net has two losses:
  "embed":  bce(logits, y) + <r, features>
  "fmaps":  bce(logits, y) + sum_i <R_i, fmap_i> / numel(fmap_i)     (17 maps: stem, 15 blocks, last conv)
with r and R_i seeded standard normal tensors."""
import contextlib
import io

import numpy as np
import torch
import torch.nn.functional as F

from efficientat_b200.synth import set_bn_stats, synth_labels, synth_state_, synth_waveform
from oracle import net_oracle as no
from tests import dilated_util as du
from tests import dyrelu_util as dyu
from tests import mha_util as mu

WIDTH, SAMPLES, BATCH, HEADS, CLASSES = 0.4, 64000, 2, 4, 527        # 2 s clips at 32 kHz
# tag -> get_model keyword arguments of the reference and of this package (same factory signature)
CASES = {"mn04": ("mn", {}),
         "mn04_mha": ("mn", dict(head_type=mu.HEAD, multihead_attention_heads=HEADS, num_classes=CLASSES)),
         "mn04_dilated": ("mn", dict(dilated=True)),
         "dymn04_k2": ("dymn", dict(dyrelu_k=2)),
         "dymn04_k3": ("dymn", dict(dyrelu_k=3))}
LOSSES = ("embed", "fmaps")


def state_(tag, model):
    """the seeded state every side starts from (make_golden.py's synth_state_, mha_state_ for the attention head)"""
    if tag == "mn04_mha":
        return mu.mha_state_(model, HEADS)
    return synth_state_(model, seed=7)


def build_model(tag, golden=None, precision="fp32"):
    """this package's model (CPU) with the golden file's calibrated BatchNorm buffers when given"""
    kind, kw = CASES[tag]
    if kind == "mn":
        from efficientat_b200.models.mn.model import get_model
    else:
        from efficientat_b200.models.dymn.model import get_model
    torch.manual_seed(0)
    with contextlib.redirect_stdout(io.StringIO()):
        m = get_model(width_mult=WIDTH, precision=precision, verbose=False, **kw)
    state_(tag, m)
    if golden is not None:
        set_bn_stats(m, golden[tag + "__cal_rm"], golden[tag + "__cal_rv"])
    return m


def net_inputs(batch=BATCH, samples=SAMPLES):
    """-> (spec [B, 1, 128, T] fp32, labels [B, 527])"""
    frames = 1 + (samples - 1) // 320
    return (synth_waveform(batch, 128 * frames, seed=21, std=0.7).view(batch, 1, 128, frames),
            synth_labels(batch, CLASSES, seed=5))


def probes(feat_shape, fmap_shapes, dtype=torch.float64):
    """-> (r like the features, [R_i like each map]), seeded standard normal"""
    g = torch.Generator().manual_seed(31)
    r = torch.randn(*feat_shape, generator=g, dtype=torch.float64)
    R = [torch.randn(*s, generator=torch.Generator().manual_seed(100 + i), dtype=torch.float64)
         for i, s in enumerate(fmap_shapes)]
    return r.to(dtype), [t.to(dtype) for t in R]


def loss(kind, logits, feat, fmaps, y, r, R, skip=()):
    """the two losses of the module docstring; skip: map indices whose term is left out (a planted defect)"""
    out = F.binary_cross_entropy_with_logits(logits, y.to(logits.dtype))
    if kind == "embed":
        return out + (r.to(feat) * feat).sum()
    for i, (Ri, m) in enumerate(zip(R, fmaps)):
        if i not in skip:
            out = out + (Ri.to(m) * m).sum() / m.numel()
    return out


def temperature(model):
    """the DynamicConv temperature the module holds (the oracle's default is 1)"""
    return float(model.layers[0].depth_conv.temperature) if hasattr(model, "layers") else 1.0


def oracle_forward(tag, sd, x, training, temp=1.0):
    """fp64 (or fp32) functional net -> (logits, features, [17 maps])"""
    if tag == "mn04":
        return no.mn_forward(sd, x, WIDTH, training=training, return_fmaps=True)
    if tag == "mn04_mha":
        return mu.mn_mha_forward(sd, x, WIDTH, HEADS, CLASSES, training=training, return_fmaps=True)
    if tag == "mn04_dilated":
        return du.mn_forward(sd, x, WIDTH, dilated=True, training=training, return_fmaps=True)
    M = CASES[tag][1]["dyrelu_k"]
    return dyu.dymn_forward(sd, x, M, WIDTH, training=training, temperature=temp, return_fmaps=True)


def oracle_grads(tag, model, kind, x, y, training=True, skip=(), device="cpu", loss_fn=None):
    """autograd of a loss through the fp64 oracle on the model's state -> (loss, dx, {parameter name: gradient}).
    loss_fn(logits, feat, fmaps) replaces the two standard losses when given."""
    names = [k for k, _ in model.named_parameters()]
    sd = {k: (v.double() if v.is_floating_point() else v).clone().to(device) for k, v in model.state_dict().items()}
    for k in names:
        sd[k].requires_grad_(True)
    x = x.double().to(device).requires_grad_(True)
    logits, feat, fmaps = oracle_forward(tag, sd, x, training, temperature(model))
    if loss_fn is not None:
        lv = loss_fn(logits, feat, fmaps)
    else:
        r, R = probes(feat.shape, [m.shape for m in fmaps])
        lv = loss(kind, logits, feat, fmaps, y.to(device), r.to(device), [t.to(device) for t in R], skip)
    lv.backward()
    return lv.item(), x.grad.cpu(), {k: sd[k].grad.cpu() if sd[k].grad is not None else None for k in names}


def grad_digest(grads, names):
    """-> (norms [P], samples [P, 4]) of the named gradients, float64"""
    norms, samples = [], []
    for n in names:
        g = grads[n].detach().double().flatten()
        norms.append(g.norm().item())
        samples.append(g[torch.linspace(0, g.numel() - 1, 4).long()].numpy())
    return np.array(norms), np.stack(samples)
