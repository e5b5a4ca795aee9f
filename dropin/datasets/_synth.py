"""Deterministic synthetic clips shared by the downstream-task stand-ins (esc50, dcase20, fsd50k, openmic).

Clip i of a split is N(0, 0.1^2) noise from a generator seeded by (dataset, split, i) plus a tone whose pitch follows
its first label, so that a clip depends neither on the batch size nor on the order of access, and a model can learn
something from it.  Sizes come from the environment, as for the synthetic AudioSet (datasets/audioset.py):
    EAT_SYNTH_CLIP_SECONDS (the dataset's clip length)   EAT_SYNTH_TRAIN_CLIPS   EAT_SYNTH_TEST_CLIPS
"""
import os
import zlib

import numpy as np
import torch
from torch.utils.data import Dataset as TorchDataset


def env_int(name, default):
    return int(os.environ.get(name, default))


def clip_seconds(default):
    return float(os.environ.get("EAT_SYNTH_CLIP_SECONDS", default))


def seed(tag, i):
    return (zlib.crc32(f"{tag}{i}".encode()) ^ 0x5EA7) & 0x7FFFFFFF


def clip(tag, i, n_samples, label, resample_rate=32000):
    g = torch.Generator()
    g.manual_seed(seed(tag + "x", i))
    x = torch.empty(n_samples, dtype=torch.float32).normal_(0.0, 0.1, generator=g)
    t = torch.arange(n_samples, dtype=torch.float32) / float(resample_rate)
    f0 = 110.0 + 40.0 * label
    x += 0.05 * torch.sin(2 * np.pi * f0 * t) + 0.02 * torch.sin(2 * np.pi * (2.5 * f0 + 31.0) * t)
    return x.numpy()


def no_augment(name, roll, wavmix):
    if roll or wavmix:
        raise NotImplementedError(f"the synthetic {name} stand-in has no roll / waveform-mixing augmentation "
                                  "(pass --no_roll --no_wavmix)")


class SyntheticClips(TorchDataset):
    """item = (waveform [1, N] float32, file name, target) + `extra(i)`; `label(i)` is the class that sets the tone,
    `target(i)` what the item carries; `seconds(i)` the clip length (variable-length evaluation)"""

    def __init__(self, tag, n, label, target, seconds, resample_rate=32000, gain_augment=0, extra=None):
        self.tag, self.n, self.label, self.target, self.seconds = tag, n, label, target, seconds
        self.resample_rate, self.gain_augment, self.extra = resample_rate, gain_augment, extra

    def __len__(self):
        return self.n

    def __getitem__(self, index):
        n_samples = int(round(self.seconds(index) * self.resample_rate))
        x = clip(self.tag, index, n_samples, self.label(index), self.resample_rate)
        if self.gain_augment:                                   # the reference's pydub_augment draw
            gain = torch.randint(self.gain_augment * 2, (1,)).item() - self.gain_augment
            x = x * (10 ** (gain / 20))
        item = (x.reshape(1, -1), f"{self.tag}_{index:06d}.wav", self.target(index))
        return item + tuple(self.extra(index)) if self.extra is not None else item
