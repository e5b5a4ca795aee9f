"""Multi-head attention pooling head (MN head_type='multihead_attention_pooling'): the golden cases, the model state
recipe shared by tests/golden/make_golden_mha.py and the tests, and an fp64 restatement of the head on top of the MN
oracle (oracle/net_oracle.py).

Head (reference models/mn/attention_pooling.py:40-56), x = output of the last 1x1 conv + BN + Hardswish [B, C, F, T]:
    m = mean_f x -> [B, T, C];  P = m W^T + b -> [B, T, 2, H, K];  a = clamp(sigmoid(P_att), eps, 1 - eps)
    out[b, k] = sum_h hw[h] sum_t a v / sum_t a
"""
import contextlib
import io

import numpy as np
import torch
import torch.nn.functional as F

from efficientat_b200.synth import set_bn_stats, synth_labels, synth_state_, synth_waveform

HEAD = "multihead_attention_pooling"
EPS = 1e-7

# case -> (width_mult, waveform samples (32 kHz, 320 hop), batch, heads, classes)
CASES = {
    "mn04_h4": (0.4, 32000, 2, 4, 527),
    "mn10_10s_h4": (1.0, 320000, 2, 4, 527),
    "mn04_h3_k50": (0.4, 32000, 2, 3, 50),      # N = 2 * 3 * 50 = 300 is not a multiple of 8: CUDA-core GEMM route
    "mn04_h1": (0.4, 32000, 2, 1, 527),
}


# ex_audioset.py --train with this head: the arguments of the mlp script golden (tests/refscripts.py) without
# --pretrained, which the reference cannot do for this head (mn/model.py:287-302), so both sides start from the
# seeded default initialisation of the same width
def script_args():
    from tests import refscripts as R
    args = [a for a in R.SCRIPT_ARGS if a != "--pretrained"]
    return args + ["--model_width", "0.4", "--head_type", HEAD]


def head_weight_values(H):
    """distinct per-head mixing weights (synth_state_ leaves raw Parameters at the reference's 1/H, which would make a
    wrong head index invisible)"""
    return torch.tensor([0.9 - 0.55 * h + 0.1 * h * h for h in range(H)], dtype=torch.float32)


ATT_GAIN = 4.0


def mha_state_(model, H):
    """synth_state_ (seeded BatchNorm / conv / Linear state, as tests/golden/make_golden.py) + distinct head weights +
    the attention rows of the projection scaled by ATT_GAIN: with synth_state_'s N(0, 1/fan_in) alone, the attention
    logits of the 1 s clips (7 frames at the head) vary so little over t that the normalised attention is nearly
    uniform, and a check of the attention path would be blind"""
    synth_state_(model, seed=7)
    head = model.classifier
    with torch.no_grad():
        head.head_weight.copy_(head_weight_values(H).view(1, H, 1))
        head.subspace_proj.weight[:H * head.out_dim].mul_(ATT_GAIN)
    return model


def case_inputs(case):
    """-> (spec [B, 1, 128, frames] fp32 CPU, labels [B, K]) as make_golden.py builds them for the mlp nets"""
    _, n, b, _, k = CASES[case]
    frames = 1 + (n - 1) // 320
    spec = synth_waveform(b, 128 * frames, seed=21, std=0.7).view(b, 1, 128, frames)
    return spec, synth_labels(b, k, seed=5)


def build_mha_model(case, golden=None, precision="fp32"):
    """this package's model for a golden case, with the golden file's calibrated BatchNorm buffers when given"""
    from efficientat_b200.models.mn.model import get_model
    width, _, _, H, K = CASES[case]
    torch.manual_seed(0)
    with contextlib.redirect_stdout(io.StringIO()):
        m = get_model(width_mult=width, num_classes=K, head_type=HEAD, multihead_attention_heads=H, precision=precision,
                      verbose=False)
    mha_state_(m, H)
    if golden is not None:
        set_bn_stats(m, golden[case + "__cal_rm"], golden[case + "__cal_rv"])
    return m


def mha_head(x, weight, bias, hw, H, K, eps=EPS):
    """the reference head's expression on x [B, C, F, T] (any dtype) -> out [B, K]"""
    m = x.mean(2).transpose(1, 2)                                     # [B, T, C]
    b, n, _ = m.shape
    p = F.linear(m, weight, bias).reshape(b, n, 2, H, K).permute(2, 0, 3, 1, 4)
    att, val = p[0], p[1]
    att = torch.clamp(torch.sigmoid(att), eps, 1. - eps)
    att = att / att.sum(2, keepdim=True)
    return ((att * val).sum(2) * hw.reshape(1, H, 1)).sum(1)


def attention_weights(x, weight, bias, H, K, eps=EPS):
    """normalised attention [B, H, T, K] of the head on x [B, C, F, T]"""
    m = x.mean(2).transpose(1, 2)
    b, n, _ = m.shape
    att = F.linear(m, weight, bias).reshape(b, n, 2, H, K).permute(2, 0, 3, 1, 4)[0]
    att = torch.clamp(torch.sigmoid(att), eps, 1. - eps)
    return att / att.sum(2, keepdim=True)


def mn_mha_forward(sd, x, width_mult, H, K, training=False, return_fmaps=False):
    """MN with this head on the oracle: the oracle's trunk (net_oracle.mn_forward, whose mlp head is fed placeholder
    weights and discarded) + mha_head.  -> (logits, features[, fmaps])"""
    from oracle import net_oracle
    C = sd["classifier.subspace_proj.weight"].shape[1]
    z = torch.zeros((), dtype=x.dtype, device=x.device)
    sd2 = dict(sd)
    sd2.update({"classifier.2.weight": z.expand(1, C), "classifier.2.bias": z.expand(1),
                "classifier.5.weight": z.expand(1, 1), "classifier.5.bias": z.expand(1)})
    _, feat, fmaps = net_oracle.mn_forward(sd2, x, width_mult=width_mult, training=training, return_fmaps=True)
    out = mha_head(fmaps[-1], sd["classifier.subspace_proj.weight"], sd["classifier.subspace_proj.bias"],
                   sd["classifier.head_weight"], H, K)
    return (out, feat, fmaps) if return_fmaps else (out, feat)


def att_far_from_uniform(att, ratio=1.5):
    """fraction of (b, h, k) whose normalised attention over t has max / min >= ratio"""
    r = att.amax(2) / att.amin(2)
    return float((r >= ratio).double().mean())


def digest(t):
    """4 strided samples"""
    f = t.detach().flatten()
    return f[torch.linspace(0, f.numel() - 1, 4).long()]


def np_(t):
    return np.asarray(t.detach().cpu().numpy())
