"""Generate tests/golden/wave_aug.npz by running the UNMODIFIED reference's waveform augmentation: `PreprocessDataset`,
`get_roll_func` and `get_gain_augment_func` (datasets/helpers/audiodatasets.py) and, from each dataset module,
`MixupDataset`, `pydub_augment`, `pad_or_truncate` (and DCASE20's `SimpleSelectionDataset`, AudioSet's
`AddIndexDataset`), wrapped as each module's `get_training_set` wraps them.

Run where a checkout of the original project exists (read-only), named by $EAT_REFERENCE_DIR:
    EAT_REFERENCE_DIR=<checkout> python tests/golden/make_golden_wave_aug.py

The dataset modules cannot be imported here (their import asserts a configured `dataset_dir` and needs the audio
decoders), so the definitions above are taken from their source text as they stand and executed on their own.  The
base dataset, which decodes audio in the reference, is an in-memory stand-in per kind that returns what the decoder
path returns: a fixed-length float32 clip (gain applied before `pad_or_truncate` as in the reference's
`__getitem__`), its name and its target.  Clips: S = 6, N = 1001 samples (odd; most roll shifts exceed N), with a
per-clip DC offset so that the re-centering of the mixing matters.

Recorded per case (tests/wave_aug_util.CASES): the sources and labels, the batch's indices, the draws as the
reference made them (recorded by wrapping torch.rand / torch.randint / np.random.random_integers / np.random.beta
while the reference code runs), the augmented waveforms and labels, and the next torch.rand / np.random.rand values
after the batch (so that a re-implementation must consume exactly as many draws)."""
import ast
import importlib.util
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
REF = os.environ["EAT_REFERENCE_DIR"]
sys.path.insert(0, REPO)
from tests import wave_aug_util as wu  # noqa: E402

spec = importlib.util.spec_from_file_location("ref_audiodatasets", os.path.join(REF, "datasets", "helpers", "audiodatasets.py"))
AD = importlib.util.module_from_spec(spec)
spec.loader.exec_module(AD)


def ref_defs(module, names):
    """the named top-level definitions of datasets/<module>.py, executed from their unmodified source text"""
    src = open(os.path.join(REF, "datasets", module + ".py")).read()
    tree = ast.parse(src)
    ns = {"torch": torch, "np": np, "TorchDataset": torch.utils.data.Dataset}
    for node in tree.body:
        if isinstance(node, (ast.ClassDef, ast.FunctionDef)) and node.name in names:
            exec(compile(ast.Module([node], []), f"{module}.py", "exec"), ns)
    missing = [n for n in names if n not in ns]
    assert not missing, missing
    return ns


class Base(torch.utils.data.Dataset):
    """in-memory stand-in for the decoding dataset of esc50 / fsd50k / openmic / audioset"""

    def __init__(self, defs, waves, targets, gain_augment):
        self.defs, self.waves, self.targets, self.gain_augment = defs, waves, targets, gain_augment

    def __len__(self):
        return len(self.waves)

    def __getitem__(self, index):
        waveform = self.waves[index].copy()
        waveform = self.defs["pydub_augment"](waveform, self.gain_augment)
        waveform = self.defs["pad_or_truncate"](waveform, self.waves.shape[1])
        return waveform.reshape(1, -1), f"clip{index}", self.targets[index].copy()


class DcaseBase(torch.utils.data.Dataset):
    """in-memory stand-in for dcase20.BasicDCASE20Dataset: (sig [1, N], file, label, device, city)"""

    def __init__(self, waves, labels):
        self.waves, self.labels = waves, torch.from_numpy(labels)

    def __len__(self):
        return len(self.waves)

    def __getitem__(self, index):
        return torch.from_numpy(self.waves[index][np.newaxis].copy()), f"clip{index}", self.labels[index], 0, 0


def training_set(kind, waves, targets, G, roll, wavmix, rate):
    """each module's get_training_set, over the stand-in base"""
    if kind == "dcase20":
        d = ref_defs("dcase20", ["SimpleSelectionDataset", "MixupDataset"])
        ds = d["SimpleSelectionDataset"](DcaseBase(waves, targets), list(range(len(waves))))
        if roll:
            ds = AD.PreprocessDataset(ds, AD.get_roll_func())
        if G:
            ds = AD.PreprocessDataset(ds, AD.get_gain_augment_func(G))
        if wavmix:
            ds = d["MixupDataset"](ds, rate=rate)
        return ds
    names = ["MixupDataset", "pydub_augment", "pad_or_truncate"] + (["AddIndexDataset"] if kind == "audioset" else [])
    d = ref_defs(kind, names)
    ds = Base(d, waves, targets, G)
    if roll:
        ds = AD.PreprocessDataset(ds, AD.get_roll_func())
    if wavmix:
        ds = d["MixupDataset"](ds, rate=rate)
    if kind == "audioset":
        ds = d["AddIndexDataset"](ds)
    return ds


class Recorder:
    """records the global-generator draws the reference code makes, in order"""

    def __init__(self):
        self.log = []
        self.orig = (torch.rand, torch.randint, np.random.random_integers, np.random.beta)

    def __enter__(self):
        rand, randint, rint, beta = self.orig
        log = self.log

        def w_rand(*a, **k):
            v = rand(*a, **k)
            log.append(("rand", float(v)))
            return v

        def w_randint(high, size, **k):
            v = randint(high, size, **k)
            log.append(("randint", int(high), int(v)))
            return v

        def w_rint(lo, hi, *a):
            v = rint(lo, hi, *a)
            log.append(("shift", int(v)))
            return v

        def w_beta(a, b, *r):
            v = beta(a, b, *r)
            log.append(("beta", float(v)))
            return v
        torch.rand, torch.randint, np.random.random_integers, np.random.beta = w_rand, w_randint, w_rint, w_beta
        return self

    def __exit__(self, *exc):
        torch.rand, torch.randint, np.random.random_integers, np.random.beta = self.orig


def decode(log, G, S):
    """one item's draw log -> (idx2, gain1, shift1, gain2, shift2, lam); gains in dB (2G differs from S in every case)"""
    assert 2 * G != S
    idx2, gains, shifts, lam = -1, [], [], 1.0
    for e in log:
        if e[0] == "randint" and e[1] == 2 * G:
            gains.append(e[2] - G)
        elif e[0] == "randint" and e[1] == S:
            idx2 = e[2]
        elif e[0] == "shift":
            shifts.append(e[1])
        elif e[0] == "beta":
            lam = max(e[1], 1. - e[1])
    gains += [0] * (2 - len(gains))
    shifts += [0] * (2 - len(shifts))
    return idx2, gains[0], shifts[0], gains[1], shifts[1], lam


def run(name, case, res):
    kind, G, roll, wavmix, rate = case
    waves, targets = wu.make_sources(kind)
    ds = training_set(kind, waves, targets, G, roll, wavmix, rate)
    idx = wu.indices()
    torch.manual_seed(wu.SEED)
    np.random.seed(wu.SEED)
    xs, ys, draws = [], [], []
    for i in idx:
        with Recorder() as r:
            item = ds[int(i)]
        x, y = item[0], item[2]
        xs.append(np.asarray(x, dtype=np.float64).reshape(-1))
        ys.append(np.asarray(y, dtype=np.float64).reshape(-1) if not np.isscalar(y) and np.ndim(y) else
                  np.array([float(y)]))
        if kind == "audioset":
            assert item[3] == i               # the primary index for the teacher lookup
        draws.append(decode(r.log, G, len(waves)))
    d = np.array(draws, dtype=np.float64)
    res[name + "__idx1"] = idx
    res[name + "__idx2"] = d[:, 0].astype(np.int64)
    res[name + "__gain1"], res[name + "__shift1"] = d[:, 1].astype(np.int64), d[:, 2].astype(np.int64)
    res[name + "__gain2"], res[name + "__shift2"] = d[:, 3].astype(np.int64), d[:, 4].astype(np.int64)
    res[name + "__lam"] = d[:, 5]
    res[name + "__wave"] = np.stack(xs).astype(np.float32)
    res[name + "__y"] = np.stack(ys).astype(np.float32)
    res[name + "__next"] = np.array([torch.rand(1).item(), np.random.rand()])
    print(f"{name}: mixed {int((d[:, 0] >= 0).sum())}/{len(idx)}, shifts {d[:, 2].astype(int).tolist()}, "
          f"gains {d[:, 1].astype(int).tolist()}")


if __name__ == "__main__":
    out = os.path.join(HERE, "wave_aug.npz")
    assert not os.path.exists(out), f"{out} exists; this script only writes new files"
    res = {}
    for kind in wu.SOURCE_KINDS:
        waves, targets = wu.make_sources(kind)
        res[kind + "__source"] = waves
        res[kind + "__labels"] = targets
    for name, case in wu.CASES.items():
        run(name, case, res)
    np.savez_compressed(out, **res)
