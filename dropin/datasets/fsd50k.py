"""Synthetic stand-in for the reference's `datasets/fsd50k.py` (HDF5 files of mp3 bytes, decoded with PyAV).
Entry points of ex_fsd50k.py: get_training_set(roll, wavmix, gain_augment, resample_rate), get_valid_set(resample_rate,
variable_eval) and get_eval_set(resample_rate, variable_eval); item = (waveform [1, N] float32, file name, multi-hot
target [200] float32).  Every class has positive and negative clips in any split of 5 or more clips (the scripts'
ROC needs both).  variable_eval: clips of different lengths (between 0.5x and 1x the clip length; the scripts then
evaluate with batch size 1).  10 s clips by default (EAT_SYNTH_CLIP_SECONDS)."""
import numpy as np

from ._synth import SyntheticClips, clip_seconds, env_int, no_augment

NUM_CLASSES = 200


def _target(i):
    y = np.zeros(NUM_CLASSES, dtype=np.float32)
    y[(np.arange(NUM_CLASSES) + i) % 5 == 0] = 1.0
    return y


def _dataset(split, n, resample_rate, gain_augment=0, variable=False):
    secs = clip_seconds(10)
    length = (lambda i: secs * (0.5 + 0.5 * ((i * 7) % 11) / 10.0)) if variable else (lambda i: secs)
    return SyntheticClips(f"fsd50k_{split}", n, lambda i: i % 5, _target, length, resample_rate, gain_augment)


def get_training_set(roll=False, wavmix=False, gain_augment=0, resample_rate=32000):
    no_augment("FSD50K", roll, wavmix)
    return _dataset("train", env_int("EAT_SYNTH_TRAIN_CLIPS", 1000), resample_rate, gain_augment)


def get_valid_set(resample_rate=32000, variable_eval=None):
    return _dataset("valid", env_int("EAT_SYNTH_TEST_CLIPS", 200), resample_rate, variable=bool(variable_eval))


def get_eval_set(resample_rate=32000, variable_eval=None):
    return _dataset("eval", env_int("EAT_SYNTH_TEST_CLIPS", 200), resample_rate, variable=bool(variable_eval))
