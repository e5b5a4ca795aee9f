"""Shared by tests/golden/make_golden_wave_aug.py, tests/test_wave_aug.py and tests/test_gpu_zz_wave_aug.py: the golden
cases of the waveform augmentation and an fp64 restatement of the reference's semantics (augment.py's docstring)."""
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "wave_aug.npz")
SEED = 1234
S, N = 6, 1001                     # N odd; roll shifts reach +-4000, so most exceed N
SOURCE_KINDS = ("esc50", "fsd50k", "openmic", "dcase20", "audioset")
NUM_CLASSES = {"esc50": 50, "fsd50k": 200, "openmic": 40, "dcase20": 10, "audioset": 527}

# name -> (kind, gain_augment, roll, wavmix, rate)
CASES = {
    "esc50": ("esc50", 12, True, True, 0.5),
    "esc50_g0": ("esc50", 0, True, True, 0.5),
    "esc50_rate1_noroll": ("esc50", 4, False, True, 1.0),
    "esc50_rate0": ("esc50", 12, True, True, 0.0),
    "fsd50k": ("fsd50k", 12, True, True, 0.5),
    "openmic": ("openmic", 12, True, True, 0.5),
    "openmic_rate1": ("openmic", 12, True, True, 1.0),
    "dcase20": ("dcase20", 12, True, True, 0.5),
    "dcase20_nomix": ("dcase20", 12, True, False, 0.5),
    "audioset": ("audioset", 12, True, True, 0.5),
    "audioset_gain": ("audioset", 4, False, False, 0.5),
}


def indices():
    return np.array([0, 3, 5, 3, 1, 2, 4, 0], dtype=np.int64)


def make_sources(kind):
    """-> (waves [S, N] float32 with a per-clip DC offset, targets as the base dataset returns them)"""
    rng = np.random.default_rng(SOURCE_KINDS.index(kind) + 11)
    waves = (0.1 * rng.standard_normal((S, N)) + rng.uniform(-0.05, 0.05, (S, 1))).astype(np.float32)
    C = NUM_CLASSES[kind]
    if kind == "dcase20":
        return waves, rng.integers(0, C, S).astype(np.int64)
    if kind == "esc50":
        t = np.zeros((S, C))
        t[np.arange(S), rng.integers(0, C, S)] = 1
        return waves, t
    if kind == "openmic":
        scores = rng.uniform(0, 1, (S, C // 2))
        mask = (rng.uniform(0, 1, (S, C // 2)) < 0.4).astype(np.float64)
        return waves, np.concatenate([scores, mask], axis=1).astype(np.float32)
    return waves, (rng.uniform(0, 1, (S, C)) < 0.05).astype(np.float32)


def load_case(g, name):
    """-> (kind, gain, roll, wavmix, rate, sources, labels, draws dict of numpy arrays, wave, y) of one golden case"""
    kind, G, roll, wavmix, rate = CASES[name]
    d = {k: g[f"{name}__{k}"] for k in ("idx1", "idx2", "shift1", "shift2", "gain1", "gain2", "lam")}
    return (kind, G, roll, wavmix, rate, g[kind + "__source"], g[kind + "__labels"], d, g[name + "__wave"],
            g[name + "__y"])


def restate(kind, wavmix, src, labels, d):
    """fp64 statement of the reference's augmentation of one batch: (waves [B, N], labels) from the draws `d`"""
    src = np.asarray(src, dtype=np.float64)
    xs, ys = [], []
    for b in range(len(d["idx1"])):
        p, q = int(d["idx1"][b]), int(d["idx2"][b])
        x1 = 10.0 ** (float(d["gain1"][b]) / 20.0) * np.roll(src[p], int(d["shift1"][b]))
        y1 = np.asarray(labels[p], dtype=np.float64)
        if kind == "dcase20":
            y1 = np.eye(NUM_CLASSES[kind])[int(labels[p])] if wavmix else np.array([float(labels[p])])
        if q < 0:
            xs.append(x1)
            ys.append(y1)
            continue
        l = float(d["lam"][b])
        x2 = 10.0 ** (float(d["gain2"][b]) / 20.0) * np.roll(src[q], int(d["shift2"][b]))
        x = l * (x1 - x1.mean()) + (1 - l) * (x2 - x2.mean())
        xs.append(x - x.mean())
        y2 = np.eye(NUM_CLASSES[kind])[int(labels[q])] if kind == "dcase20" else np.asarray(labels[q], dtype=np.float64)
        if kind == "openmic":
            H = len(y1) // 2
            m1, m2 = (y1[H:] > 0.5).astype(np.float64), (y2[H:] > 0.5).astype(np.float64)
            ys.append(np.concatenate([l * y1[:H] * m1 + (1 - l) * y2[:H] * m2, np.maximum(m1, m2)]))
        else:
            ys.append(l * y1 + (1 - l) * y2)
    return np.stack(xs), np.stack(ys)
