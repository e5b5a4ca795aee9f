"""Resampling on the device with scipy.signal.resample_poly's semantics: the `librosa.core.load(path, sr=32000)` step of
the reference's inference.py:45, windowed_inference.py:89 and datasets/esc50.py:115, for which
scripts/run_reference_script.py substitutes `resample_poly(x, sr // g, rate // g)`.

    rs = Resample(44100).cuda()        # 44.1 kHz -> 32 kHz
    y = rs(x)                          # x [B, N] fp32 CUDA -> y [B, ceil(N * 320 / 441)]
    spec = mel(y)

The filter is designed here in numpy (no scipy dependency) and both passes are one launch each of csrc/resample.cu:
eat_resample_poly_fwd, and for a waveform that requires grad eat_resample_poly_bwd, the exact adjoint.
"""
import math

import numpy as np
import torch
import torch.nn as nn

from ._lib import check_module_tensors, lib
from .packed import as_int_list, check_lengths

MAX_RATE = 2048      # EAT_RESAMPLE_MAX_RATE: up and down after the gcd reduction


def rates(orig_sr, new_sr):
    """-> (up, down): new_sr / orig_sr reduced by their gcd, as resample_poly reduces them."""
    for name, v in (("orig_sr", orig_sr), ("new_sr", new_sr)):
        if isinstance(v, bool) or int(v) != v or v < 1:
            raise ValueError(f"{name} must be a positive integer, got {v!r}")
    orig_sr, new_sr = int(orig_sr), int(new_sr)
    g = math.gcd(orig_sr, new_sr)
    return new_sr // g, orig_sr // g


def design_filter(up, down):
    """-> (h, half_len): resample_poly's default filter, firwin(2 half_len + 1, 1 / max(up, down),
    window=('kaiser', 5.0)) * up with half_len = 10 max(up, down), in fp64."""
    max_rate = max(up, down)
    fc = 1.0 / max_rate
    half_len = 10 * max_rate
    n = 2 * half_len + 1
    m = np.arange(n, dtype=np.float64) - half_len
    h = fc * np.sinc(fc * m) * np.kaiser(n, 5.0)
    h /= h.sum()                               # firwin(scale=True): unit gain at DC
    return h * up, half_len


def alignment(n_in, up, down, half_len):
    """-> (n_pre_pad, n_pre_remove, n_out): resample_poly's constants.  Output m of resample_poly is sample
    m + n_pre_remove of upfirdn over the filter with n_pre_pad zeros in front, i.e. sum_i x[i] h[m down - i up + half_len]:
    (m + n_pre_remove) down - n_pre_pad = m down + half_len, since half_len + n_pre_pad is a multiple of down."""
    n_pre_pad = down - half_len % down
    n_pre_remove = (half_len + n_pre_pad) // down
    return n_pre_pad, n_pre_remove, -(-n_in * up // down)


def polyphase_table(h, up, down, offset):
    """-> table [taps, up] (fp64): table[k, r] = h[p + (taps - 1 - k) up], p = (r down + offset) mod up, 0 past the
    filter's end, so that out[m] = sum_k table[k, m mod up] in[(m down + offset) // up - (taps - 1) + k]."""
    taps = -(-len(h) // up)
    p = (np.arange(up) * down + offset) % up
    idx = p[None, :] + (taps - 1 - np.arange(taps))[:, None] * up
    return np.concatenate([h, np.zeros(up, dtype=h.dtype)])[idx]     # idx < taps up <= len(h) + up - 1


class Resample(nn.Module):
    """Rows of x [B, N] at `orig_sr` -> [B, ceil(N up / down)] at `new_sr`, each row what
    scipy.signal.resample_poly(row, up, down) computes with its defaults (up / down = new_sr / orig_sr reduced).

    Accepts every pair with max(up, down) <= 2048 after the reduction (8, 11.025, 16, 22.05, 24, 44.1, 48, 88.2 and
    96 kHz to and from 32 kHz among them); other pairs raise NotImplementedError.  orig_sr == new_sr launches nothing
    and returns a copy.  The polyphase tables are fp32 buffers of the module (not persistent: they follow from the rates)."""

    def __init__(self, orig_sr, new_sr=32000):
        super().__init__()
        self.orig_sr, self.new_sr = int(orig_sr), int(new_sr)
        self.up, self.down = rates(orig_sr, new_sr)
        if max(self.up, self.down) > MAX_RATE:
            raise NotImplementedError(
                f"Resample({orig_sr}, {new_sr}): up / down = {self.up} / {self.down} after the gcd reduction; the kernels "
                f"take max(up, down) <= {MAX_RATE}")
        self.identity = self.up == self.down
        h, self.half_len = design_filter(self.up, self.down)
        fwd = polyphase_table(h, self.up, self.down, self.half_len)
        adj = polyphase_table(h[::-1].copy(), self.down, self.up, self.half_len)
        self.taps, self.taps_adj = fwd.shape[0], adj.shape[0]
        self.register_buffer("_table", torch.from_numpy(fwd).float().contiguous(), persistent=False)
        self.register_buffer("_table_adj", torch.from_numpy(adj).float().contiguous(), persistent=False)

    def extra_repr(self):
        return f"orig_sr={self.orig_sr}, new_sr={self.new_sr}, up={self.up}, down={self.down}"

    def num_samples(self, lengths):
        """each clip's output count for input sample counts `lengths`: ceil(n up / down), the `lengths` the mel takes"""
        return [-(-n * self.up // self.down) for n in as_int_list(lengths)]

    def forward(self, x, lengths=None):
        """x [B, N] -> [B, ceil(N up / down)].

        lengths: each clip's sample count, a sequence of ints or a CPU integer tensor of length B, each in [1, N].  Row
        b's first num_samples(lengths)[b] outputs then equal the resampling of x[b, :lengths[b]] alone and later outputs
        are 0.0; samples at or past lengths[b] are never read.  Not supported for an x that requires grad."""
        if x.dim() != 2 or x.shape[1] < 1:
            raise ValueError(f"expected waveform of shape [B, N] with N >= 1, got {tuple(x.shape)}")
        if lengths is not None:
            if x.requires_grad:
                raise NotImplementedError("lengths: per-clip lengths are not supported for a waveform that requires grad")
            lengths = check_lengths(lengths, x.shape[0], 1, x.shape[1])
        if not x.is_cuda:
            raise RuntimeError("efficientat_b200.Resample runs on CUDA (sm_90a) only; got a CPU tensor")
        if self.identity:
            y = x.float().clone()
            if lengths is not None:
                keep = torch.arange(x.shape[1], device=x.device)[None, :] < torch.tensor(lengths, device=x.device)[:, None]
                y = torch.where(keep, y, torch.zeros((), device=x.device))
            return y
        check_module_tensors(self, x.device, "Resample")
        with torch.cuda.device(x.device):
            if lengths is not None:
                return self._forward(x.float().contiguous(), torch.tensor(lengths, dtype=torch.int32).to(x.device))
            if torch.is_grad_enabled() and x.requires_grad:
                return _ResampleFn.apply(self, x)
            return self._forward(x.float().contiguous())

    def _forward(self, x, n_valid=None):
        b, n = x.shape
        y = torch.empty(b, -(-n * self.up // self.down), device=x.device, dtype=torch.float32)
        lib().resample_poly_fwd(x.data_ptr(), b, n, n_valid.data_ptr() if n_valid is not None else 0, self.up, self.down,
                                self._table.data_ptr(), self.taps, self.half_len, y.data_ptr(), y.shape[1],
                                torch.cuda.current_stream().cuda_stream)
        return y

    def _backward(self, dy, n):
        b = dy.shape[0]
        dx = torch.empty(b, n, device=dy.device, dtype=torch.float32)
        lib().resample_poly_bwd(dy.data_ptr(), b, n, self.up, self.down, self._table_adj.data_ptr(), self.taps_adj,
                                self.half_len, dx.data_ptr(), dy.shape[1], torch.cuda.current_stream().cuda_stream)
        return dx


class _ResampleFn(torch.autograd.Function):
    """waveform -> resampled waveform, with the waveform's gradient from eat_resample_poly_bwd (the exact adjoint)"""

    @staticmethod
    def forward(ctx, module, x):
        ctx.module, ctx.n, ctx.dtype = module, x.shape[1], x.dtype
        return module._forward(x.detach().float().contiguous())

    @staticmethod
    def backward(ctx, dy):
        if torch.is_grad_enabled():
            raise NotImplementedError("double backward (create_graph=True) through Resample is not implemented")
        with torch.cuda.device(dy.device):
            dx = ctx.module._backward(dy.float().contiguous(), ctx.n)
        return None, dx.to(ctx.dtype)
