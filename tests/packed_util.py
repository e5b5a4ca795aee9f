"""Test helpers for clips of different lengths in one eval batch: the nets, clips and state of
tests/golden/make_golden_packed.py, shared by the generator, tests/test_packed.py and tests/test_gpu_zz_packed.py."""
import contextlib
import io

import numpy as np
import torch

from efficientat_b200.synth import set_bn_stats, synth_state_, synth_waveform
from tests import fmap_grad_util as fu

WIDTH = fu.WIDTH
SECONDS = (0.05, 0.37, 0.9, 1.3, 2.0, 2.71)              # 5 to 272 frames; the 0.05 s clip reaches 1 frame in the tail
# tag -> (kind, get_model keyword arguments of the reference and of this package)
NETS = {"mn04": fu.CASES["mn04"], "mn04_mha": fu.CASES["mn04_mha"], "mn04_dilated": fu.CASES["mn04_dilated"],
        "dymn04_k2": fu.CASES["dymn04_k2"], "dymn04_k3": fu.CASES["dymn04_k3"],
        "dymn04_replace_se": ("dymn", dict(use_dy_blocks="replace_se"))}
ORACLE = ("mn04", "mn04_mha", "mn04_dilated", "dymn04_k2", "dymn04_k3")     # nets with an fp64 functional oracle


def _fmap_golden():
    return np.load(fu.__file__.replace("fmap_grad_util.py", "golden/fmap_grad.npz"), allow_pickle=False)


def state_(tag, model):
    """the seeded state; the MN nets take the BatchNorm buffers calibrated for tests/golden/fmap_grad.npz, the DyMN nets
    keep synth_state_'s (calibrated ones drive DyMN's eval logits to 1e7 and beyond on short clips)"""
    if NETS[tag][0] == "mn":
        fu.state_(tag, model)
        g = _fmap_golden()
        return set_bn_stats(model, g[tag + "__cal_rm"], g[tag + "__cal_rv"])
    return synth_state_(model, seed=7)


def build_model(tag, precision="fp32"):
    """this package's model (CPU) in the golden's state"""
    kind, kw = NETS[tag]
    if kind == "mn":
        from efficientat_b200.models.mn.model import get_model
    else:
        from efficientat_b200.models.dymn.model import get_model
    torch.manual_seed(0)
    with contextlib.redirect_stdout(io.StringIO()):
        m = get_model(width_mult=WIDTH, precision=precision, verbose=False, **kw)
    return state_(tag, m)


def clip_frames():
    return [1 + (round(s * 32000) - 1) // 320 for s in SECONDS]


def clip_specs():
    """-> six [1, 1, 128, T_b] fp32 spectrograms (seeded)"""
    return [synth_waveform(1, 128 * t, seed=60 + i, std=0.7).view(1, 1, 128, t) for i, t in enumerate(clip_frames())]


def padded_batch(specs):
    """the clips zero-padded to the longest: [B, 1, 128, T_max]"""
    T = max(s.shape[-1] for s in specs)
    x = torch.zeros(len(specs), 1, 128, T, dtype=specs[0].dtype)
    for b, s in enumerate(specs):
        x[b, :, :, :s.shape[-1]] = s[0]
    return x


def oracle_forward(tag, model, x):
    """fp64 functional net in eval on the model's state -> (logits, features, [17 maps])"""
    sd = {k: (v.double() if v.is_floating_point() else v) for k, v in model.state_dict().items()}
    with torch.no_grad():
        return fu.oracle_forward(tag, sd, x.double(), False, fu.temperature(model))
