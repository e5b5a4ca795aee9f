"""Synthetic stand-in for the reference's `datasets/esc50.py` (the real one reads the ESC-50 wav files with librosa).
Entry points of ex_esc50.py: get_training_set(resample_rate, roll, wavmix, gain_augment, fold) and
get_test_set(resample_rate, fold); item = (waveform [1, N] float32, file name, one-hot target [50] float32).
5 s clips by default (EAT_SYNTH_CLIP_SECONDS); the fold selects a disjoint clip range."""
import numpy as np

from ._synth import SyntheticClips, clip_seconds, env_int, no_augment

NUM_CLASSES = 50


def _one_hot(c):
    y = np.zeros(NUM_CLASSES, dtype=np.float32)
    y[c] = 1.0
    return y


def _dataset(split, n, fold, resample_rate, gain_augment=0):
    secs = clip_seconds(5)
    return SyntheticClips(f"esc50_f{fold}_{split}", n, lambda i: i % NUM_CLASSES,
                          lambda i: _one_hot(i % NUM_CLASSES), lambda i: secs, resample_rate, gain_augment)


def get_training_set(resample_rate=32000, roll=False, wavmix=False, gain_augment=0, fold=1):
    no_augment("ESC-50", roll, wavmix)
    return _dataset("train", env_int("EAT_SYNTH_TRAIN_CLIPS", 1600), fold, resample_rate, gain_augment)


def get_test_set(resample_rate=32000, fold=1):
    return _dataset("test", env_int("EAT_SYNTH_TEST_CLIPS", 400), fold, resample_rate)
