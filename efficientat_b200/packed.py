"""Clips of different lengths in one eval batch: the host side of `lengths` (argument checks, per-stage length table).

A batch holds clip b in its first lengths[b] samples (waveform) or frames (spectrogram); the rest is padding.  Every
stage's valid time size follows from the clip's own by the conv size rule the tensors are sized with, so the device
kernels (csrc/packed.cu) only need one int32 table of them per call."""
import numbers

import torch


def as_int_list(lengths, name="lengths"):
    """A sequence of ints or a CPU integer tensor of one dimension -> list of ints; ValueError otherwise."""
    if isinstance(lengths, torch.Tensor):
        if lengths.device.type != "cpu":
            raise ValueError(f"{name} must be a CPU tensor or a sequence of ints, got a tensor on {lengths.device}")
        if lengths.dim() != 1 or lengths.dtype.is_floating_point or lengths.dtype.is_complex or lengths.dtype == torch.bool:
            raise ValueError(f"{name} must be a 1-D integer tensor, got {lengths.dtype} of shape {tuple(lengths.shape)}")
        return [int(v) for v in lengths.tolist()]
    try:
        vals = list(lengths)
    except TypeError:
        raise ValueError(f"{name} must be a sequence of ints or a CPU integer tensor, got {type(lengths).__name__}") from None
    for v in vals:
        if isinstance(v, bool) or not isinstance(v, numbers.Integral):
            raise ValueError(f"{name} must hold integers, got {v!r}")
    return [int(v) for v in vals]


def check_lengths(lengths, count, lo, hi, name="lengths"):
    """-> list of `count` ints, each in [lo, hi]; ValueError otherwise (before any launch)."""
    vals = as_int_list(lengths, name)
    if len(vals) != count:
        raise ValueError(f"{name} has {len(vals)} entries for a batch of {count}")
    bad = [v for v in vals if not lo <= v <= hi]
    if bad:
        raise ValueError(f"{name} must lie in [{lo}, {hi}], got {bad[0]}")
    return vals


def stage_sizes(engine, F, T, lengths):
    """[(F_s, T_s, [t_s for each clip])] for the network input (s = 0), the stem (s = 1) and every block's output, by the
    same _conv_out that sizes the engine's tensors (reference mn/utils.py:24-26, cnn_out_size)."""
    from .engine import _conv_out
    s0 = engine.stem[0].stride[0]
    out = [(F, T, list(lengths))]
    out.append((_conv_out(F, 3, s0), _conv_out(T, 3, s0), [_conv_out(t, 3, s0) for t in lengths]))
    for blk in engine.blocks:
        Fi, Ti, ti = out[-1]
        k, s, d = blk.k, blk.stride, blk.dil
        out.append((_conv_out(Fi, k, s, d), _conv_out(Ti, k, s, d), [_conv_out(t, k, s, d) for t in ti]))
    return out


class StageLengths:
    """Per-stage valid lengths of one call, on the host and as one int32 device table:
    rows 0 .. S-1: t_s of each clip at stage s (stage_sizes' order);
    rows S .. 2S-1: F_s + t_s, the valid rows of ContextGen's [F | T] sequence for a block whose input is stage s."""

    def __init__(self, engine, F, T, lengths, device):
        self.sizes = stage_sizes(engine, F, T, lengths)
        rows = [t for _, _, t in self.sizes] + [[Fs + v for v in t] for Fs, _, t in self.sizes]
        self.table = torch.tensor(rows, dtype=torch.int32).to(device)
        self.n = len(self.sizes)

    def ptr(self, s):
        """device pointer of stage s's row of valid time steps"""
        return self.table[s].data_ptr()

    def seq_ptr(self, s):
        """device pointer of stage s's row of valid ContextGen sequence rows (F_s + t_s)"""
        return self.table[self.n + s].data_ptr()

    def padded(self, s):
        """whether some clip is shorter than the batch at stage s"""
        _, Ts, t = self.sizes[s]
        return any(v < Ts for v in t)
