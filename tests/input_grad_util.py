"""Test helpers for gradients with respect to the input: the inputs, cotangent and digest of
tests/golden/make_golden_input_grad.py."""
import torch

from efficientat_b200.synth import synth_waveform

BATCH, FRAMES, WAVE_SAMPLES = 2, 101, 32000        # 2 s clips


def spec_input():
    """[B, 1, 128, 101] fp32, as tests/util.net_inputs('mn04')"""
    return synth_waveform(BATCH, 128 * FRAMES, seed=21, std=0.7).view(BATCH, 1, 128, FRAMES)


def cotangent():
    return torch.randn(BATCH, 527, generator=torch.Generator().manual_seed(3), dtype=torch.float64)


def digest(g):
    """float64 [1 + 64 + 4]: the norm, 64 strided samples and the projections on four seeded random vectors"""
    f = g.detach().double().flatten()
    probes = torch.randn(4, f.numel(), generator=torch.Generator().manual_seed(17), dtype=torch.float64)
    idx = torch.linspace(0, f.numel() - 1, 64).long()
    return torch.cat([f.norm().view(1), f[idx], probes @ f]).numpy()
