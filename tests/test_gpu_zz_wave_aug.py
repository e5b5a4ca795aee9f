"""Waveform augmentation on the device (csrc/wave_aug.cu through efficientat_b200/augment.py) against the fp64
restatement of the reference (tests/wave_aug_util.restate, itself pinned to the reference by tests/test_wave_aug.py):
- every golden case, from the resident store and from the batch, waveforms and labels under the three label rules;
- edge draws: shifts 0, +-4000 and beyond N, odd N, B = 1, a partner equal to the item itself, gains of +-12 dB,
  mixed and unmixed rows;
- planted defects (the roll sign flipped, the re-centering dropped) that must fail;
- the trainers' step with `augment` (FineTuneTrainer with DCASE20's soft targets and OpenMIC's masked BCE, eager and
  graph; AudioSetTrainer with a teacher) against the same trainer without `augment` fed the restated batch;
- with `augment=None` the trainers launch exactly the entry points they launched before."""
import contextlib
import io

import numpy as np
import pytest
import torch

from efficientat_b200._lib import lib
from efficientat_b200.augment import WaveAugment
from tests import wave_aug_util as wu
from tests.test_gpu_zz_fmap_grad import _plain_runs, _Recorder
from tests.util import golden, report

pytestmark = pytest.mark.gpu

NEW_ENTRIES = {"clip_sum", "wave_aug", "label_mix"}


def _g():
    return np.load(wu.GOLDEN)


def _check(name, got_x, got_y, ref_x, ref_y):
    ex = np.abs(got_x.double().cpu().numpy() - ref_x).max() / np.abs(ref_x).max()
    ey = np.abs(got_y.double().cpu().numpy().reshape(ref_y.shape) - ref_y).max()
    report(f"wave_aug {name}: waveform max rel err {ex:.2e}, labels max abs err {ey:.2e}")
    assert ex <= 1e-6 and ey <= 1e-6, (name, ex, ey)


@pytest.mark.parametrize("name", list(wu.CASES))
def test_store_matches_restatement(name):
    kind, G, roll, wavmix, rate, src, labels, d, wave, y = wu.load_case(_g(), name)
    a = WaveAugment(kind, gain_augment=G, roll=roll, wavmix=wavmix, rate=rate,
                    source=torch.from_numpy(src).cuda(), labels=torch.from_numpy(labels).cuda())
    x_out, y_out = a(torch.from_numpy(d["idx1"]), None, {k: torch.from_numpy(v) for k, v in d.items()})
    ref_x, ref_y = wu.restate(kind, wavmix, src, labels, d)
    _check(name + " store", x_out, y_out, ref_x, ref_y)
    _check(name + " store vs reference", x_out, y_out, wave.astype(np.float64), y.astype(np.float64))


@pytest.mark.parametrize("name", list(wu.CASES))
def test_batch_matches_restatement(name):
    kind, G, roll, wavmix, rate, src, labels, _, _, _ = wu.load_case(_g(), name)
    idx = wu.indices()
    wave, yb = src[idx], labels[idx]
    a = WaveAugment(kind, gain_augment=G, roll=roll, wavmix=wavmix, rate=rate)
    torch.manual_seed(5)
    np.random.seed(5)
    d = a.draw(range(len(idx)), len(idx))
    x_out, y_out = a(torch.from_numpy(wave).cuda(), torch.from_numpy(yb).cuda(), d)
    ref_x, ref_y = wu.restate(kind, wavmix, wave, yb, {k: v.numpy() for k, v in d.items()})
    _check(name + " batch", x_out, y_out, ref_x, ref_y)


def _edge_draws():
    # shifts 0, +-4000, beyond N (1001) both ways, small; a self-partner (row 2); gains +-12 dB; mixed and unmixed rows
    return {"idx1": torch.tensor([0, 1, 2, 3, 4, 5, 0]), "idx2": torch.tensor([-1, 4, 2, -1, 0, 5, 3]),
            "shift1": torch.tensor([0, 4000, -4000, 1500, -2999, 1, 0]),
            "shift2": torch.tensor([0, -4000, 4000, 0, 7, -1001, 1001]),
            "gain1": torch.tensor([12, -12, 0, -12, 12, 3, 0]), "gain2": torch.tensor([0, 12, -12, 0, -12, 0, 12]),
            "lam": torch.tensor([1.0, 0.5, 0.73, 1.0, 0.999, 0.5, 0.61], dtype=torch.float64)}


@pytest.mark.parametrize("kind", ["esc50", "dcase20", "openmic"])
def test_edge_draws(kind):
    g = _g()
    src, labels = g[kind + "__source"], g[kind + "__labels"]
    a = WaveAugment(kind, gain_augment=12, roll=True, wavmix=True,
                    source=torch.from_numpy(src).cuda(), labels=torch.from_numpy(labels).cuda())
    d = _edge_draws()
    x_out, y_out = a(d["idx1"], None, d)
    _check(f"edge {kind}", x_out, y_out, *wu.restate(kind, True, src, labels, {k: v.numpy() for k, v in d.items()}))
    for b in range(len(d["idx1"])):                      # B = 1, each row alone
        db = {k: v[b:b + 1] for k, v in d.items()}
        x1, y1 = a(db["idx1"], None, db)
        assert torch.equal(x1[0], x_out[b]) and torch.equal(y1[0], y_out[b]), b


def test_planted_defects_fail():
    g = _g()
    kind, G, roll, wavmix, rate, src, labels, d, _, _ = wu.load_case(g, "esc50")
    a = WaveAugment(kind, gain_augment=G, roll=True, wavmix=True, source=torch.from_numpy(src).cuda(),
                    labels=torch.from_numpy(labels).cuda())
    ref_x, _ = wu.restate(kind, wavmix, src, labels, d)
    dt = {k: torch.from_numpy(v) for k, v in d.items()}
    flipped, _ = a(dt["idx1"], None, dict(dt, shift1=-dt["shift1"], shift2=-dt["shift2"]))
    good_sums = a.sums
    a.sums = torch.zeros_like(good_sums)                 # the means never removed
    uncentred, _ = a(dt["idx1"], None, dt)
    a.sums = good_sums
    for what, bad in (("roll sign flipped", flipped), ("re-centering dropped", uncentred)):
        e = np.abs(bad.double().cpu().numpy() - ref_x).max() / np.abs(ref_x).max()
        report(f"wave_aug planted defect {what}: max rel err {e:.2e}")
        assert e > 1e-3, what


def _net(num_classes):
    from efficientat_b200.models.mn.model import get_model
    from efficientat_b200.synth import set_bn_stats, synth_state_
    torch.manual_seed(0)
    with contextlib.redirect_stdout(io.StringIO()):
        m = get_model(width_mult=0.4, num_classes=num_classes, verbose=False)
    synth_state_(m, seed=7)
    gm = golden("mn04")
    m = set_bn_stats(m, gm["cal_rm"], gm["cal_rv"]).cuda()
    for mod in m.modules():
        if isinstance(mod, torch.nn.Dropout):
            mod.p = 0.0
    return m


def _mel():
    from efficientat_b200.models.preprocess import AugmentMelSTFT
    with contextlib.redirect_stdout(io.StringIO()):
        return AugmentMelSTFT(freqm=0, timem=0).cuda()


def _store(kind, S=6, N=32000):
    rng = np.random.default_rng(3)
    src = (0.1 * rng.standard_normal((S, N)) + rng.uniform(-0.05, 0.05, (S, 1))).astype(np.float32)
    if kind == "dcase20":
        labels = rng.integers(0, 10, S).astype(np.int64)
    else:
        labels = np.concatenate([rng.uniform(0, 1, (S, 20)), (rng.uniform(0, 1, (S, 20)) < 0.5)], 1).astype(np.float32)
    return src, labels


def _compare(tag, p0, params_a, params_b, losses_a, losses_b):
    """losses and Adam updates of the two runs; the bounds are those of tests/test_gpu_finetune_trainer.py, whose
    comparison also feeds the same step two batches that differ by fp32 rounding"""
    err = max(abs(x - y) / abs(y) for x, y in zip(losses_a, losses_b))
    num = sum((p - q).norm().item() ** 2 for p, q in zip(params_a, params_b)) ** 0.5
    den = sum((q - o).norm().item() ** 2 for q, o in zip(params_b, p0)) ** 0.5
    report(f"wave_aug trainer {tag}: loss rel err {err:.2e}, update rel diff {num / den:.2e}")
    assert err <= 2e-4 and num / den <= 5e-2, (tag, err, num / den)


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("kind,loss", [("dcase20", "ce"), ("openmic", "bce_masked")])
def test_finetune_step_with_store(kind, loss, graph):
    from efficientat_b200.finetune import FineTuneTrainer
    src, labels = _store(kind)
    C = 10 if kind == "dcase20" else 20
    idx = [torch.tensor([0, 4, 2, 5]), torch.tensor([1, 1, 3, 0]), torch.tensor([5, 2, 0, 3])]
    aug = WaveAugment(kind, gain_augment=12, roll=True, wavmix=True, source=torch.from_numpy(src).cuda(),
                      labels=torch.from_numpy(labels).cuda())
    torch.manual_seed(11)
    np.random.seed(12)
    draws = [aug.draw(i, len(src)) for i in idx]
    assert any((d["idx2"] >= 0).any() for d in draws) and any((d["idx2"] < 0).any() for d in draws)
    mix = [(torch.randperm(4, generator=torch.Generator().manual_seed(20 + k)),
            torch.rand(4, generator=torch.Generator().manual_seed(30 + k)) * 0.5 + 0.5) for k in range(3)]
    runs = {}
    for with_aug in (True, False):
        model = _net(C)
        p0 = [p.detach().clone() for p in model.parameters()]
        tr = FineTuneTrainer(model, _mel(), loss=loss, lr=4e-4, cuda_graph=graph, augment=aug if with_aug else None)
        losses = []
        for i, d, (rn, lam) in zip(idx, draws, mix):
            if with_aug:
                out = tr.step(i, None, perm=rn, lam=lam, draws=d)
            else:
                x, y = wu.restate(kind, True, src, labels, {k: v.numpy() for k, v in d.items()})
                out = tr.step(torch.from_numpy(x).float().cuda(), torch.from_numpy(y).float().cuda(), perm=rn, lam=lam)
            losses.append(out.item())
        runs[with_aug] = ([p.detach().clone() for p in model.parameters()], losses)
    _compare(f"{kind} {loss} graph={graph}", p0, runs[True][0], runs[False][0], runs[True][1], runs[False][1])


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
def test_audioset_step_with_batch_source_and_teacher(graph):
    from efficientat_b200.synth import synth_labels, synth_waveform
    from efficientat_b200.train import AudioSetTrainer
    B = 4
    wave = synth_waveform(B, 32000, seed=5).cuda()
    y = synth_labels(B, 527, seed=6).cuda()
    teacher = torch.sigmoid(torch.randn(B, 527, generator=torch.Generator().manual_seed(7))).cuda()
    known = torch.tensor([1.0, 0.0, 1.0, 1.0]).cuda()
    aug = WaveAugment("audioset", gain_augment=12, roll=True, wavmix=True, rate=0.75)
    torch.manual_seed(3)
    np.random.seed(4)
    draws = [aug.draw(range(B), B) for _ in range(2)]
    mix = [(torch.randperm(B, generator=torch.Generator().manual_seed(20 + k)),
            torch.rand(B, generator=torch.Generator().manual_seed(30 + k)) * 0.5 + 0.5) for k in range(2)]
    runs = {}
    for with_aug in (True, False):
        model = _net(527)
        p0 = [p.detach().clone() for p in model.parameters()]
        tr = AudioSetTrainer(model, _mel(), lr=4e-4, kd_lambda=0.1, cuda_graph=graph, augment=aug if with_aug else None)
        losses = []
        for d, (rn, lam) in zip(draws, mix):
            if with_aug:
                out = tr.step(wave, y, teacher, perm=rn, lam=lam, teacher_known=known, draws=d)
            else:
                x, yy = wu.restate("audioset", True, wave.cpu().numpy(), y.cpu().numpy(), {k: v.numpy() for k, v in d.items()})
                out = tr.step(torch.from_numpy(x).float().cuda(), torch.from_numpy(yy).float().cuda(), teacher, perm=rn,
                              lam=lam, teacher_known=known)
            losses.append(out.sum().item())
        runs[with_aug] = ([p.detach().clone() for p in model.parameters()], losses)
    _compare(f"audioset teacher graph={graph}", p0, runs[True][0], runs[False][0], runs[True][1], runs[False][1])


def test_store_step_draws_on_its_own():
    """without `draws` the step draws from the global generators as WaveAugment.draw does"""
    from efficientat_b200.finetune import FineTuneTrainer
    src, labels = _store("dcase20")
    aug = WaveAugment("dcase20", gain_augment=12, roll=True, wavmix=True, source=torch.from_numpy(src).cuda(),
                      labels=torch.from_numpy(labels).cuda())
    idx = torch.tensor([0, 4, 2, 5])
    outs = []
    for explicit in (False, True):
        tr = FineTuneTrainer(_net(10), _mel(), loss="ce", lr=4e-4, mixup_alpha=0.0, augment=aug)
        torch.manual_seed(9)
        np.random.seed(9)
        outs.append(tr.step(idx, None, draws=aug.draw(idx, len(src)) if explicit else None).item())
        outs.append((torch.rand(1).item(), np.random.rand()))         # the generators after the step
    # the step's batch statistics sum with atomics, so the two losses agree to fp32 rounding, not bit for bit
    assert abs(outs[0] - outs[2]) <= 1e-5 * abs(outs[2]), outs
    assert outs[1] == outs[3], outs


def test_augment_none_launches_are_unchanged():
    from tests import fmap_grad_util as fu
    model = fu.build_model("mn04", golden("fmap_grad")).cuda()
    spec = fu.net_inputs()[0].cuda()
    state = {k: v.clone() for k, v in model.state_dict().items()}
    _plain_runs(model, spec)                        # one-time launches (weight repacking) happen here
    model.load_state_dict(state)
    torch.manual_seed(3)
    before, out_b = _plain_runs(model, spec)
    for k, calls in before.items():
        assert calls and not NEW_ENTRIES & set(calls), k
    model.load_state_dict(state)
    src, labels = _store("openmic", N=8000)
    aug = WaveAugment("openmic", gain_augment=12, roll=True, wavmix=True, rate=1.0,
                      source=torch.from_numpy(src).cuda(), labels=torch.from_numpy(labels).cuda())
    with _Recorder() as rec:
        aug(torch.tensor([0, 1]), None)
    assert NEW_ENTRIES - {"clip_sum"} <= set(rec.calls)
    model.load_state_dict(state)
    torch.manual_seed(3)
    after, out_a = _plain_runs(model, spec)
    assert after == before
    for k in out_b:
        for a, b in zip(out_a[k], out_b[k]):
            assert (a - b).abs().max().item() <= 2e-4 * max(1.0, b.abs().max().item()), k
