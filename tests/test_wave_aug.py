"""Waveform augmentation (efficientat_b200/augment.py, csrc/wave_aug.cu) without a GPU:
- `WaveAugment.draw` makes the draws the reference's wrapped datasets make (tests/golden/wave_aug.npz, recorded from the
  unmodified reference), for every dataset kind, with and without gain, roll and mixing, at rates 0, 0.5 and 1, and
  leaves the global generators where the reference leaves them;
- the fp64 restatement (tests/wave_aug_util.restate) applied to those draws reproduces the reference's waveforms and
  labels, so the GPU tests can measure the kernels against it;
- every new C entry point rejects bad arguments before any launch, and B = 0 is a no-op;
- WaveAugment rejects bad options, stores and draws on the host."""
import numpy as np
import pytest
import torch

from efficientat_b200._lib import EatError, lib
from efficientat_b200.augment import KINDS, LABEL_ONEHOT, LABEL_OPENMIC, LABEL_PLAIN, WaveAugment
from tests import wave_aug_util as wu


@pytest.fixture(scope="module")
def g():
    return np.load(wu.GOLDEN)


def _aug(name):
    kind, G, roll, wavmix, rate = wu.CASES[name]
    return WaveAugment(kind, gain_augment=G, roll=roll, wavmix=wavmix, rate=rate)


@pytest.mark.parametrize("name", list(wu.CASES))
def test_draw_matches_reference_draws(g, name):
    kind, *_, d, _, _ = wu.load_case(g, name)
    torch.manual_seed(wu.SEED)
    np.random.seed(wu.SEED)
    got = _aug(name).draw(wu.indices(), wu.S)
    for k, v in d.items():
        np.testing.assert_array_equal(got[k].numpy(), v, err_msg=f"{name}: {k}")
    # the generators are left exactly where the reference leaves them
    np.testing.assert_array_equal([torch.rand(1).item(), np.random.rand()], g[name + "__next"])


def test_golden_cases_cover_the_edges(g):
    assert not g["esc50_g0__gain1"].any() and not g["esc50_rate1_noroll__shift1"].any()
    assert (g["esc50_rate0__idx2"] == -1).all() and (g["esc50_rate1_noroll__idx2"] >= 0).all()
    shifts = np.concatenate([g[n + "__shift1"] for n in wu.CASES])
    assert (np.abs(shifts) > wu.N).any() and (np.abs(shifts[shifts != 0]) < wu.N).any()
    assert set(KINDS) == {c[0] for c in wu.CASES.values()}


@pytest.mark.parametrize("name", list(wu.CASES))
def test_restatement_matches_reference_outputs(g, name):
    kind, G, roll, wavmix, rate, src, labels, d, wave, y = wu.load_case(g, name)
    x, yy = wu.restate(kind, wavmix, src, labels, d)
    scale = np.abs(wave).max()
    assert np.abs(x - wave).max() <= 2e-6 * scale, name
    np.testing.assert_allclose(yy, y, rtol=0, atol=1e-6, err_msg=name)


def test_restatement_is_not_trivially_close():
    """planted defects in the restatement would be caught: no re-centering, the roll sign flipped"""
    g = np.load(wu.GOLDEN)
    kind, G, roll, wavmix, rate, src, labels, d, wave, y = wu.load_case(g, "esc50")
    flipped = dict(d, shift1=-d["shift1"])
    x, _ = wu.restate(kind, wavmix, src, labels, flipped)
    assert np.abs(x - wave).max() > 1e-2
    mixed = d["idx2"] >= 0
    assert np.abs(wave[mixed].mean(axis=1)).max() < 1e-6 < np.abs(np.asarray(src).mean(axis=1)).min()


def test_entry_points_reject_bad_arguments_before_any_launch():
    L = lib()
    p = 16                                  # a non-null pointer that is never dereferenced: the checks come first
    with pytest.raises(EatError):
        L.clip_sum(p, -1, 8, p, None)
    with pytest.raises(EatError):
        L.clip_sum(p, 2, 0, p, None)
    with pytest.raises(EatError):
        L.clip_sum(0, 2, 8, p, None)
    with pytest.raises(EatError):
        L.clip_sum(p, 2, 8, 0, None)
    L.clip_sum(0, 0, 8, 0, None)            # S = 0: no-op

    def aug(src=p, sums=p, S=4, N=8, i1=p, i2=p, s1=p, s2=p, g1=p, g2=p, lam=p, out=p, B=2):
        L.wave_aug(src, sums, S, N, i1, i2, s1, s2, g1, g2, lam, out, B, None)
    for kw in ({"B": -1}, {"B": 65536}, {"S": 0}, {"N": 0}, {"N": (1 << 30) + 1}, {"src": 0}, {"i1": 0}, {"i2": 0},
               {"s1": 0}, {"s2": 0}, {"g1": 0}, {"g2": 0}, {"lam": 0}, {"out": 0}):
        with pytest.raises(EatError):
            aug(**kw)
    aug(src=0, sums=0, i1=0, i2=0, s1=0, s2=0, g1=0, g2=0, lam=0, out=0, B=0)           # B = 0: no-op

    def mix(rule=LABEL_PLAIN, yp=p, yi=0, S=4, C=6, i1=p, i2=p, lam=p, B=2, out=p):
        L.label_mix(rule, yp, yi, S, C, i1, i2, lam, B, out, None)
    for kw in ({"rule": 3}, {"rule": -1}, {"B": -1}, {"S": 0}, {"C": 0}, {"rule": LABEL_OPENMIC, "C": 5},
               {"yp": 0}, {"yi": p}, {"rule": LABEL_ONEHOT}, {"rule": LABEL_ONEHOT, "yp": 0, "yi": 0},
               {"i1": 0}, {"i2": 0}, {"lam": 0}, {"out": 0}):
        with pytest.raises(EatError):
            mix(**kw)
    mix(i1=0, i2=0, lam=0, out=0, B=0)                                                  # B = 0: no-op


def test_wave_augment_rejects_bad_options():
    for kw in ({"kind": "esc"}, {"kind": "esc50", "gain_augment": -1}, {"kind": "esc50", "gain_augment": 1.5},
               {"kind": "esc50", "shift_range": -3}, {"kind": "esc50", "beta": 0},
               {"kind": "esc50", "labels": torch.zeros(2, 3)}):
        with pytest.raises(ValueError):
            WaveAugment(**kw)
    with pytest.raises(ValueError):                        # a store must be an fp32 CUDA tensor
        WaveAugment("esc50", source=torch.zeros(2, 8), labels=torch.zeros(2, 3))


def test_check_draws():
    a = WaveAugment("esc50", gain_augment=12, roll=True, wavmix=True)
    torch.manual_seed(0)
    np.random.seed(0)
    d = a.draw([0, 1, 2], 3)
    a.check_draws(d, 3, 3)
    bad = [dict(d, idx1=torch.tensor([0, 1, 3])), dict(d, idx1=torch.tensor([-1, 1, 2])),
           dict(d, idx2=torch.tensor([-2, 0, 0])), dict(d, idx2=torch.tensor([0, 0, 3])),
           dict(d, shift1=torch.tensor([4001, 0, 0])), dict(d, shift2=torch.tensor([0, -4001, 0])),
           dict(d, lam=torch.tensor([1.5, 1.0, 1.0])), dict(d, gain1=torch.tensor([0, 0, 500])),
           dict(d, lam=torch.ones(2, dtype=torch.float64)), {k: v for k, v in d.items() if k != "gain2"}]
    for b in bad:
        with pytest.raises(ValueError):
            a.check_draws(b, 3, 3)


def test_no_draws_without_augmentation():
    torch.manual_seed(5)
    np.random.seed(5)
    first = (torch.rand(1).item(), np.random.rand())
    torch.manual_seed(5)
    np.random.seed(5)
    d = WaveAugment("openmic").draw(range(4), 4)
    assert (d["idx2"] == -1).all() and not d["gain1"].any() and not d["shift1"].any()
    assert (torch.rand(1).item(), np.random.rand()) == first
