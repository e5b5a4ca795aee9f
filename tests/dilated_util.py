"""Test helpers for MN's dilated tail: the models and inputs of tests/golden/make_golden_dilated.py, and an fp64/fp32
oracle of get_model(reduced_tail=..., dilated=...): the functional MN of oracle/net_oracle.py with the reference's tail
options (models/mn/model.py:237-268, models/mn/block_types.py:132,150-160).

- reduced_tail halves the channels of the last three rows and of the classifier's hidden layer.
- dilated gives the depthwise convs of the last three rows dilation 2, padding 2 * (k-1)/2 and stride 1; the residual
  connection still follows the row's nominal stride.
Built from net_oracle's helpers, so the undilated, full-tail case is net_oracle.mn_forward."""
import contextlib
import io

import torch
import torch.nn.functional as F

from efficientat_b200.synth import set_bn_stats, synth_labels, synth_state_, synth_waveform
from oracle import net_oracle as no
from tests.util import golden

N_TAIL = 3
# tag: (width, samples, batch, reduced_tail, has a training step) -- as tests/golden/make_golden_dilated.py
CASES = {"mn04_dilated": (0.4, 64000, 2, False, True),
         "mn04_dilated_rt": (0.4, 64000, 2, True, True),
         "mn10_dilated_10s": (1.0, 320000, 2, False, False)}


def build_model(tag, precision="fp32", head_type="mlp"):
    """the golden's model with its calibrated BatchNorm buffers (CPU)"""
    from efficientat_b200.models.mn.model import get_model
    width, _, _, rt, _ = CASES[tag]
    torch.manual_seed(0)
    with contextlib.redirect_stdout(io.StringIO()):
        m = get_model(width_mult=width, dilated=True, reduced_tail=rt, precision=precision, head_type=head_type,
                      verbose=False)
    synth_state_(m, seed=7)
    g = golden(tag)
    return set_bn_stats(m, g["cal_rm"], g["cal_rv"])


def net_inputs(tag):
    """-> (spec [B,1,128,T] fp32 CPU, labels [B,527]) as tests/golden/make_golden_dilated.py builds them"""
    _, n, b, _, _ = CASES[tag]
    frames = 1 + (n - 1) // 320
    return synth_waveform(b, 128 * frames, seed=21, std=0.7).view(b, 1, 128, frames), synth_labels(b, 527, seed=5)


def block_table(width_mult=1.0, strides=(2, 2, 2, 2), reduced_tail=False, dilated=False):
    rows = no.block_table(width_mult, strides)
    div = 2 if reduced_tail else 1
    first_tail = len(rows) - N_TAIL
    for i, (r, raw) in enumerate(zip(rows, no._ROWS)):
        r["dil"] = 1
        if i < first_tail:
            continue
        cin, _, cexp, cout = raw[:4]
        if i > first_tail:
            cin = cin // div
        r.update(cin=no.make_divisible(cin * width_mult), cexp=no.make_divisible(cexp // (div if i > first_tail else 1)
                                                                                  * width_mult),
                 cout=no.make_divisible(cout // div * width_mult), dil=2 if dilated else 1)
    return rows


def mn_forward(sd, x, width_mult=1.0, strides=(2, 2, 2, 2), reduced_tail=False, dilated=False, training=False,
               dropout_mask=None, return_fmaps=False, undilated_blocks=()):
    """as net_oracle.mn_forward.  undilated_blocks: 1-based block indices whose depthwise conv runs undilated (at the
    row's nominal stride) although dilated is set -- a deliberately wrong network for the tests' planted defects."""
    rows = block_table(width_mult, strides, reduced_tail, dilated)
    fmaps = []
    x = no._cna(x, sd, "features.0", 3, 2, 1, "HS", training)
    fmaps.append(x)
    for i, r in enumerate(rows, start=1):
        inp = x
        j = 0
        pfx = f"features.{i}.block"
        if r["cexp"] != r["cin"]:
            x = no._cna(x, sd, f"{pfx}.{j}", 1, 1, 1, r["act"], training)
            j += 1
        d = 1 if i in undilated_blocks else r["dil"]
        k = r["k"]
        x = F.conv2d(x, sd[f"{pfx}.{j}.0.weight"], None, 1 if d > 1 else r["stride"], (k - 1) // 2 * d, d, r["cexp"])
        x = no._act(no._bn(x, sd, f"{pfx}.{j}.1", training), r["act"])
        j += 1
        if r["se"]:
            x = no._se(x, sd, f"{pfx}.{j}.conc_se_layers.0")
            j += 1
        x = no._cna(x, sd, f"{pfx}.{j}", 1, 1, 1, None, training)
        if r["stride"] == 1 and r["cin"] == r["cout"]:
            x = x + inp
        fmaps.append(x)
    x = no._cna(x, sd, f"features.{len(rows) + 1}", 1, 1, 1, "HS", training)
    fmaps.append(x)
    logits, feat = no._head(x, sd, training, dropout_mask)
    if return_fmaps:
        return logits, feat, fmaps
    return logits, feat
