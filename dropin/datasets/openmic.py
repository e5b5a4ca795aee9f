"""Synthetic stand-in for the reference's `datasets/openmic.py` (HDF5 files of mp3 bytes, decoded with PyAV).
Entry points of ex_openmic.py: get_training_set(roll, wavmix, gain_augment, resample_rate) and
get_test_set(resample_rate); item = (waveform [1, N] float32, file name, target [40] float32) with target[:20] the
instrument scores in [0, 1] and target[20:] the 0/1 mask of the observed ones.  Every instrument is observed both
present and absent in any split of 6 or more clips.  10 s clips by default (EAT_SYNTH_CLIP_SECONDS)."""
import numpy as np

from ._synth import SyntheticClips, clip_seconds, env_int, no_augment

NUM_CLASSES = 20


def _target(i):
    c = np.arange(NUM_CLASSES)
    y = np.zeros(2 * NUM_CLASSES, dtype=np.float32)
    y[:NUM_CLASSES] = np.where((c + i) % 3 == 0, 0.9, 0.1)            # scores either side of the 0.5 threshold
    y[NUM_CLASSES:] = ((c + 2 * i) % 7 != 0).astype(np.float32)       # about one label in seven unobserved
    return y


def _dataset(split, n, resample_rate, gain_augment=0):
    secs = clip_seconds(10)
    return SyntheticClips(f"openmic_{split}", n, lambda i: i % 3, _target, lambda i: secs, resample_rate, gain_augment)


def get_training_set(roll=False, wavmix=False, gain_augment=0, resample_rate=32000):
    no_augment("OpenMIC", roll, wavmix)
    return _dataset("train", env_int("EAT_SYNTH_TRAIN_CLIPS", 1000), resample_rate, gain_augment)


def get_test_set(resample_rate=32000):
    return _dataset("test", env_int("EAT_SYNTH_TEST_CLIPS", 250), resample_rate)
