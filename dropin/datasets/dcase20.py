"""Synthetic stand-in for the reference's `datasets/dcase20.py` (TAU Urban Acoustic Scenes 2020 Mobile, read with
librosa and optionally cached).  Entry points of ex_dcase20.py: get_training_set(cache_path, resample_rate, roll,
gain_augment, wavmix) and get_test_set(cache_path, resample_rate); item = (waveform [1, N] float32, file name,
scene index int, recording device str, city str, index int).  `cache_path` is accepted and unused.  10 s clips by
default (EAT_SYNTH_CLIP_SECONDS)."""
from ._synth import SyntheticClips, clip_seconds, env_int, no_augment

NUM_CLASSES = 10
DEVICES = ("a", "b", "c", "s1", "s2", "s3")
CITIES = ("barcelona", "helsinki", "lisbon", "london", "lyon", "milan", "paris", "prague", "stockholm", "vienna")


def _dataset(split, n, resample_rate, gain_augment=0):
    secs = clip_seconds(10)
    return SyntheticClips(f"dcase20_{split}", n, lambda i: i % NUM_CLASSES, lambda i: i % NUM_CLASSES, lambda i: secs,
                          resample_rate, gain_augment,
                          extra=lambda i: (DEVICES[i % len(DEVICES)], CITIES[(i // 3) % len(CITIES)], i))


def get_training_set(cache_path=None, resample_rate=32000, roll=False, gain_augment=False, wavmix=False):
    no_augment("DCASE20", roll, wavmix)
    return _dataset("train", env_int("EAT_SYNTH_TRAIN_CLIPS", 1400), resample_rate, int(gain_augment))


def get_test_set(cache_path=None, resample_rate=32000):
    return _dataset("test", env_int("EAT_SYNTH_TEST_CLIPS", 300), resample_rate)
