"""fp64 restatement of csrc/resample.cu's index math, as an explicit gather: autograd of `gather` is the adjoint.

    out[m] = sum_k table[k, m mod U] in[(m D + offset) // U - (taps - 1) + k],   in = 0 outside [0, len)
"""
import torch

from efficientat_b200.resample import design_filter, polyphase_table, rates


def gather(x, table, U, D, offset, n_out, lengths=None):
    """x [B, N] (any float dtype, differentiable) -> out [B, n_out]; row b reads x[b, :lengths[b]] and its outputs at or
    past ceil(lengths[b] U / D) are 0 (lengths=None: every row is whole, and all n_out outputs are computed)."""
    B, N = x.shape
    table = torch.as_tensor(table, dtype=x.dtype, device=x.device)
    taps = table.shape[0]
    m = torch.arange(n_out, device=x.device)
    i = (m[:, None] * D + offset) // U - (taps - 1) + torch.arange(taps, device=x.device)[None, :]      # [n_out, taps]
    w = table[:, m % U].t()                                                                          # [n_out, taps]
    lens = torch.full((B,), N, device=x.device) if lengths is None else torch.as_tensor(lengths, device=x.device)
    inside = (i[None] >= 0) & (i[None] < lens[:, None, None])                                        # [B, n_out, taps]
    xi = x[:, i.clamp(0, N - 1)]                                                                      # [B, n_out, taps]
    out = (torch.where(inside, xi, torch.zeros((), dtype=x.dtype, device=x.device)) * w).sum(-1)
    if lengths is not None:
        n_valid = -(-lens * U // D)
        out = torch.where(m[None, :] < n_valid[:, None], out, torch.zeros((), dtype=x.dtype, device=x.device))
    return out


def tables(orig_sr, new_sr):
    """-> (up, down, half_len, forward table, adjoint table) in fp64, as Resample builds them"""
    up, down = rates(orig_sr, new_sr)
    h, hl = design_filter(up, down)
    return up, down, hl, polyphase_table(h, up, down, hl), polyphase_table(h[::-1].copy(), down, up, hl)


def resample(x, orig_sr, new_sr, lengths=None):
    """the forward restated: x [B, N] -> [B, ceil(N up / down)]"""
    up, down, hl, fwd, _ = tables(orig_sr, new_sr)
    return gather(x, fwd, up, down, hl, -(-x.shape[1] * up // down), lengths)


def resample_adjoint(g, n_in, orig_sr, new_sr):
    """the adjoint restated over its own table: g [B, n_out] -> [B, n_in]"""
    up, down, hl, _, adj = tables(orig_sr, new_sr)
    return gather(g, adj, down, up, hl, n_in)
