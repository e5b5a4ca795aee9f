"""Host-side helpers the reference scripts import from helpers/utils.py (NAME_TO_WIDTH :1-32, label table :35-46, LR
schedule :56-84, mixup :90-95, mixstyle :101-121).  Re-implemented with the same semantics and the same host RNG draws;
mixstyle's arithmetic runs on the device (eat_mixstyle)."""
import csv
import os

import numpy as np
import torch


def load_labels(path="metadata/class_labels_indices.csv"):
    """-> (display names, ids) of the AudioSet classes from the reference's metadata file (helpers/utils.py:38-46 reads
    it relative to the CWD at import time); two empty lists when the file is not there."""
    if not os.path.exists(path):
        return [], []
    with open(path, "r") as f:
        lines = list(csv.reader(f, delimiter=","))
    return [l[2] for l in lines[1:]], [l[1] for l in lines[1:]]

_MN_WIDTH = {"mn01": 0.1, "mn02": 0.2, "mn04": 0.4, "mn05": 0.5, "mn06": 0.6, "mn08": 0.8, "mn10": 1.0, "mn12": 1.2,
             "mn14": 1.4, "mn16": 1.6, "mn20": 2.0, "mn30": 3.0, "mn40": 4.0}
_DYMN_WIDTH = {"dymn04": 0.4, "dymn10": 1.0, "dymn20": 2.0}


def NAME_TO_WIDTH(name):
    """'mn10_as' -> 1.0, 'dymn20_as(2)' -> 2.0; unknown names fall back to 1.0 like the reference."""
    try:
        return _DYMN_WIDTH[name[:6]] if name.startswith("dymn") else _MN_WIDTH[name[:4]]
    except (KeyError, TypeError, AttributeError):
        return 1.0


def exp_rampup(rampup_length):
    def wrapper(epoch):
        if epoch < rampup_length:
            phase = 1.0 - float(np.clip(epoch, 0.5, rampup_length)) / rampup_length
            return float(np.exp(-5.0 * phase * phase))
        return 1.0
    return wrapper


def linear_rampdown(rampdown_length, start=0, last_value=0):
    def wrapper(epoch):
        if epoch <= start:
            return 1.0
        if epoch - start < rampdown_length:
            return last_value + (1.0 - last_value) * (rampdown_length - epoch + start) / rampdown_length
        return last_value
    return wrapper


def exp_warmup_linear_down(warmup, rampdown_length, start_rampdown, last_value):
    up, down = exp_rampup(warmup), linear_rampdown(rampdown_length, start_rampdown, last_value)
    return lambda epoch: up(epoch) * down(epoch)


def mixup(size, alpha):
    """Same RNG consumption as the reference: torch.randperm (global CPU generator) then numpy beta."""
    rn_indices = torch.randperm(size)
    lambd = np.random.beta(alpha, alpha, size).astype(np.float32)
    lambd = np.maximum(lambd, 1.0 - lambd)
    return rn_indices, torch.from_numpy(lambd)


def mixstyle(x, p=0.4, alpha=0.4, eps=1e-6, mix_labels=False):
    """Frequency-wise MixStyle (helpers/utils.py:101-121) on a [B, 1, F, T] fp32 CUDA spectrogram, by `eat_mixstyle`.

    Same host RNG draws in the same order as the reference: `np.random.rand()` for the skip test (x comes back
    unchanged with probability 1 - p), then `Beta(alpha, alpha).sample((B, 1, 1, 1))` and `torch.randperm(B)` on the
    CPU generators.  mix_labels=True also returns (perm, lambda) on x's device, as the reference does.  The statistics
    are not differentiated through (the reference detaches them) and gradients w.r.t. x are not implemented."""
    from torch.distributions.beta import Beta

    from .._lib import lib
    if np.random.rand() > p:
        return x
    if not x.is_cuda:
        raise RuntimeError("mixstyle: x must be a CUDA tensor (the product path has no CPU fallback)")
    if x.requires_grad:
        raise NotImplementedError("mixstyle: gradients w.r.t. the input spectrogram are not implemented")
    if x.dim() != 4 or x.shape[1] != 1 or x.dtype != torch.float32:
        raise ValueError(f"mixstyle: expects a [B, 1, F, T] fp32 spectrogram, got {x.dtype} {tuple(x.shape)}")
    B, _, F, T = x.shape
    lmda = Beta(alpha, alpha).sample((B, 1, 1, 1))
    perm = torch.randperm(B)
    x = x.contiguous()
    out = torch.empty_like(x)
    stats = torch.empty(2 * B * F, device=x.device, dtype=torch.float32)
    with torch.cuda.device(x.device):
        perm_d = perm.to(device=x.device, dtype=torch.int32)
        lam_d = lmda.to(device=x.device, dtype=torch.float32).reshape(B)
        lib().mixstyle(x.data_ptr(), perm_d.data_ptr(), lam_d.data_ptr(), float(eps), stats.data_ptr(), out.data_ptr(),
                       B, F, T, torch.cuda.current_stream().cuda_stream)
    if mix_labels:
        return out, perm.to(x.device), lmda.to(x.device)
    return out
