"""Test helpers for DyReLU-B with M = dyrelu_k linear pieces: the models and inputs of
tests/golden/make_golden_dyrelu_k.py, and an fp64 oracle of DyMN with M pieces built from oracle/net_oracle.py's
helpers (reference models/dymn/dy_block.py:142-188, 390-409).

DyReLU-B: theta = 2 sigmoid(coef_net(h_c)) - 1 viewed as [B, C, 2M] (channel-major), coef = theta * lambdas + init_v,
out = max_m (coef[m] x + coef[M + m]).  pieces_used < M is a deliberately wrong network for the tests' planted defects:
only the first pieces_used pieces enter the max."""
import contextlib
import io

import torch
import torch.nn.functional as F

from efficientat_b200.synth import set_bn_stats, synth_labels, synth_state_, synth_waveform
from oracle import net_oracle as no
from tests.util import golden

WIDTH, SAMPLES, BATCH = 0.4, 64000, 2
PIECES = (1, 3, 4)


def tag(M):
    return f"dymn04_dyrelu_k{M}"


def build_model(M, precision="fp32", calibrated=True):
    """the golden's model (CPU); with the calibrated BatchNorm buffers of its golden file"""
    from efficientat_b200.models.dymn.model import get_model
    torch.manual_seed(0)
    with contextlib.redirect_stdout(io.StringIO()):
        m = get_model(width_mult=WIDTH, dyrelu_k=M, precision=precision, verbose=False)
    synth_state_(m, seed=7)
    if calibrated:
        g = golden(tag(M))
        set_bn_stats(m, g["cal_rm"], g["cal_rv"])
    return m


def net_inputs(batch=BATCH, samples=SAMPLES):
    """-> (spec [B,1,128,T] fp32 CPU, labels [B,527]) as tests/golden/make_golden_dyrelu_k.py builds them"""
    frames = 1 + (samples - 1) // 320
    return (synth_waveform(batch, 128 * frames, seed=21, std=0.7).view(batch, 1, 128, frames),
            synth_labels(batch, 527, seed=5))


def dyrelu_b(x, h_c, sd, pfx, M, pieces_used=None):
    """dy_block.py:157-188 for M pieces; x [B, C, F, T]"""
    b, c = x.shape[:2]
    theta = 2 * torch.sigmoid(F.linear(h_c, sd[pfx + ".coef_net.0.weight"], sd[pfx + ".coef_net.0.bias"])) - 1
    co = theta.view(b, c, 1, 1, 2 * M) * sd[pfx + ".lambdas"] + sd[pfx + ".init_v"]
    n = M if pieces_used is None else pieces_used
    mapped = x.unsqueeze(-1) * co[..., :n] + co[..., M:M + n]
    if n == 2:
        return torch.maximum(mapped[..., 0], mapped[..., 1])
    return mapped.max(-1)[0]


def dymn_forward(sd, x, M, width_mult=WIDTH, training=False, temperature=1.0, return_fmaps=False, pieces_used=None):
    """net_oracle.dymn_forward with M DyReLU-B pieces (M = 2 is that function)"""
    rows = no.block_table(width_mult)
    fmaps = []
    x = no._cna(x, sd, "in_c", 3, 2, 1, "HS", training)
    fmaps.append(x)
    for i, r in enumerate(rows):
        inp = x
        p = f"layers.{i}"
        h_c, g_cf, g_ct = no._context_gen(x, sd, p + ".context_gen", r["stride"], training)
        if r["cexp"] != r["cin"]:
            x = no._dyconv(x, h_c, sd, p + ".exp_conv", r["cexp"], r["cin"], 1, 1, 1, temperature)
            x = no._act(no._bn(x, sd, p + ".exp_norm", training), r["act"])
        x = no._dyconv(x, h_c, sd, p + ".depth_conv", r["cexp"], 1, r["k"], r["stride"], r["cexp"], temperature)
        x = no._bn(x, sd, p + ".depth_norm", training)
        x = dyrelu_b(x, h_c, sd, p + ".depth_act", M, pieces_used)
        x = x * torch.sigmoid(g_cf) * torch.sigmoid(g_ct)
        x = no._dyconv(x, h_c, sd, p + ".proj_conv", r["cout"], r["cexp"], 1, 1, 1, temperature)
        x = no._bn(x, sd, p + ".proj_norm", training)
        if r["stride"] == 1 and r["cin"] == r["cout"]:
            x = x + inp
        fmaps.append(x)
    x = no._cna(x, sd, "out_c", 1, 1, 1, "HS", training)
    fmaps.append(x)
    logits, feat = no._head(x, sd, training)
    if return_fmaps:
        return logits, feat, fmaps
    return logits, feat
