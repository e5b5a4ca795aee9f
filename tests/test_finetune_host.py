"""Host-side checks of the fine-tuning surface (no GPU): the import paths ex_dcase20.py and the other downstream
scripts use, the synthetic downstream datasets, argument validation of eat_ce_loss / eat_bce_masked_loss /
eat_mixstyle (it runs before any device call, so fake pointers are safe), and the closed-form gradients the two loss
kernels implement, restated in float64 and checked against autograd of the scripts' loss expressions."""
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

from efficientat_b200._lib import EatError, lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref")
FAKE = 256                              # a non-null address that is never dereferenced


def _run(code):
    env = dict(os.environ, PYTHONPATH=os.path.join(ROOT, "dropin") + os.pathsep + ROOT)
    return subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, cwd=ROOT)


def test_mixstyle_resolves_through_dropin():
    r = _run("import os\n"
             "from helpers.utils import mixstyle, mixup\n"
             "assert mixstyle.__module__ == 'efficientat_b200.helpers.utils', mixstyle.__module__\n"
             "import datasets.esc50, datasets.dcase20, datasets.fsd50k, datasets.openmic\n"
             "for m in (datasets.esc50, datasets.dcase20, datasets.fsd50k, datasets.openmic):\n"
             "    assert os.sep + 'dropin' + os.sep in m.__file__, m.__file__\n"
             "print('ok')\n")
    assert r.returncode == 0 and "ok" in r.stdout, r.stderr[-2000:]


def test_mixstyle_refuses_host_tensors():
    from efficientat_b200.helpers.utils import mixstyle
    x = torch.zeros(2, 1, 4, 8)
    with pytest.raises(RuntimeError, match="CUDA"):
        mixstyle(x, p=1.0)


@pytest.mark.skipif(not os.path.isfile(os.path.join(REF, "ex_dcase20.py")), reason="needs oracle/_ref (build())")
@pytest.mark.parametrize("side", ["ours", "reference"])
def test_downstream_scripts_import_under_the_launcher(side):
    """`--help` exits after the module-level imports: ex_dcase20.py's `from helpers.utils import ... mixstyle` and
    `from datasets.dcase20 import ...` resolve (the synthetic stand-in on both sides; the GPU script tests run all four)"""
    for script in ("ex_dcase20.py",):
        r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "run_reference_script.py"), "--side", side,
                            "--ref-root", REF, script, "--", "--help"], capture_output=True, text=True, cwd=REF,
                           env=dict(os.environ, WANDB_MODE="disabled"))
        assert r.returncode == 0 and "usage" in r.stdout, (script, r.stderr[-3000:])


def test_synthetic_downstream_datasets_have_the_script_layouts():
    """item layouts of the four stand-ins as the scripts unpack them; run in a subprocess so that `datasets` (which
    site-packages may also provide) is imported from dropin/ and does not leak into this process"""
    code = """
import numpy as np, torch
import datasets.esc50 as esc, datasets.dcase20 as dc, datasets.fsd50k as fsd, datasets.openmic as om
x, f, y = esc.get_training_set(resample_rate=32000, roll=False, wavmix=False, fold=1)[3]
assert x.shape == (1, 8000) and x.dtype == np.float32 and y.shape == (50,) and y.sum() == 1.0
x, f, y, d, c, i = dc.get_training_set(None, 32000, roll=False, gain_augment=False, wavmix=False)[7]
assert isinstance(y, int) and 0 <= y < 10 and isinstance(d, str) and isinstance(c, str) and i == 7
assert len(dc.get_test_set(cache_path="/nonexistent")) == 10
ys = torch.stack([torch.as_tensor(fsd.get_valid_set()[i][2]) for i in range(10)])
assert ys.shape == (10, 200) and (ys.sum(0) > 0).all() and (ys.sum(0) < 10).all()
assert len({fsd.get_valid_set(variable_eval=True)[i][0].shape[1] for i in range(10)}) > 1
x, f, y = om.get_test_set()[0]
assert y.shape == (40,) and set(y[20:].tolist()) <= {0.0, 1.0}
assert (esc.get_test_set()[2][0] == esc.get_test_set()[2][0]).all()          # deterministic clips
try:
    esc.get_training_set(roll=True)
    raise SystemExit("roll accepted")
except NotImplementedError:
    pass
print("ok")
"""
    env = dict(os.environ, PYTHONPATH=os.path.join(ROOT, "dropin") + os.pathsep + ROOT, EAT_SYNTH_CLIP_SECONDS="0.25",
               EAT_SYNTH_TRAIN_CLIPS="12", EAT_SYNTH_TEST_CLIPS="10")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, cwd=ROOT)
    assert r.returncode == 0 and "ok" in r.stdout, r.stderr[-2000:]


def _fails(name, *args):
    with pytest.raises(EatError) as e:
        getattr(lib(), name)(*args)
    return str(e.value)


def test_argument_validation_runs_before_any_launch():
    # eat_ce_loss(logits, y_index, y_prob, perm, lam, B, C, dlogits, loss_acc, stream)
    assert "exactly one" in _fails("ce_loss", FAKE, 0, 0, 0, 0, 4, 10, FAKE, FAKE, 0)
    assert "exactly one" in _fails("ce_loss", FAKE, FAKE, FAKE, 0, 0, 4, 10, FAKE, FAKE, 0)
    assert "C >= 1" in _fails("ce_loss", FAKE, FAKE, 0, 0, 0, 4, 0, FAKE, FAKE, 0)
    assert "go together" in _fails("ce_loss", FAKE, FAKE, 0, FAKE, 0, 4, 10, FAKE, FAKE, 0)
    assert "required" in _fails("ce_loss", 0, FAKE, 0, 0, 0, 4, 10, FAKE, FAKE, 0)
    lib().ce_loss(FAKE, FAKE, 0, 0, 0, 0, 10, FAKE, FAKE, 0)                  # B == 0: nothing to do
    # eat_bce_masked_loss(logits, y, y_stride, mask, mask_stride, perm, lam, B, C, dlogits, loss_acc, stream)
    assert "stride" in _fails("bce_masked_loss", FAKE, FAKE, 19, FAKE, 40, 0, 0, 4, 20, FAKE, FAKE, 0)
    assert "stride" in _fails("bce_masked_loss", FAKE, FAKE, 40, FAKE, 10, 0, 0, 4, 20, FAKE, FAKE, 0)
    assert "go together" in _fails("bce_masked_loss", FAKE, FAKE, 40, FAKE, 40, 0, FAKE, 4, 20, FAKE, FAKE, 0)
    assert "required" in _fails("bce_masked_loss", FAKE, FAKE, 40, 0, 40, 0, 0, 4, 20, FAKE, FAKE, 0)
    lib().bce_masked_loss(FAKE, FAKE, 40, FAKE, 40, 0, 0, 0, 20, FAKE, FAKE, 0)
    # eat_mixstyle(x, perm, lam, eps, stats, out, B, F, T, stream)
    assert "T >= 2" in _fails("mixstyle", FAKE, FAKE, FAKE, 1e-6, FAKE, 2 * FAKE, 4, 128, 1, 0)
    assert "F >= 1" in _fails("mixstyle", FAKE, FAKE, FAKE, 1e-6, FAKE, 2 * FAKE, 4, 0, 10, 0)
    assert "eps" in _fails("mixstyle", FAKE, FAKE, FAKE, -1.0, FAKE, 2 * FAKE, 4, 128, 10, 0)
    assert "alias" in _fails("mixstyle", FAKE, FAKE, FAKE, 1e-6, FAKE, FAKE, 4, 128, 10, 0)
    assert "required" in _fails("mixstyle", FAKE, 0, FAKE, 1e-6, FAKE, 2 * FAKE, 4, 128, 10, 0)
    lib().mixstyle(FAKE, FAKE, FAKE, 1e-6, FAKE, 2 * FAKE, 0, 128, 10, 0)


@pytest.mark.parametrize("index", [True, False])
def test_soft_ce_gradient_closed_form(index):
    """eat_ce_loss's dz = (S softmax(z) - y_mix) / B, S = sum_c y_mix, against autograd of ex_esc50.py:103-118"""
    g = torch.Generator().manual_seed(1)
    B, C = 7, 13
    z = (torch.randn(B, C, generator=g, dtype=torch.float64) * 3).requires_grad_(True)
    y = torch.randint(0, C, (B,), generator=g) if index else torch.rand(B, C, generator=g, dtype=torch.float64)
    rn, lam = torch.randperm(B, generator=g), torch.rand(B, generator=g, dtype=torch.float64)
    loss = (F.cross_entropy(z, y, reduction="none") * lam + F.cross_entropy(z, y[rn], reduction="none") * (1. - lam)).mean()
    loss.backward()
    t = F.one_hot(y, C).double() if index else y
    y_mix = t * lam[:, None] + t[rn] * (1. - lam[:, None])
    S = y_mix.sum(1, keepdim=True)
    lse = torch.logsumexp(z.detach(), dim=1, keepdim=True)
    assert torch.allclose((y_mix * (lse - z.detach())).sum(1).mean(), loss.detach(), rtol=1e-12)
    dz = (S * torch.softmax(z.detach(), dim=1) - y_mix) / B
    assert (dz - z.grad).abs().max().item() <= 1e-14


def test_masked_bce_gradient_closed_form():
    """eat_bce_masked_loss's dz = mask * (sigmoid(z) - y_mix) / (B C), targets binarised before the blend, against
    autograd of ex_openmic.py:101-121"""
    g = torch.Generator().manual_seed(2)
    B, C = 6, 20
    z = (torch.randn(B, C, generator=g, dtype=torch.float64) * 3).requires_grad_(True)
    batch = torch.rand(B, 2 * C, generator=g, dtype=torch.float64)
    batch[:, C:] = (batch[:, C:] > 0.3).double()
    rn, lam = torch.randperm(B, generator=g), torch.rand(B, generator=g, dtype=torch.float64)
    y_mask, y = batch[:, C:], (batch[:, :C] > 0.5).double()
    y_mix = y * lam[:, None] + y[rn] * (1. - lam[:, None])
    loss = (y_mask * F.binary_cross_entropy_with_logits(z, y_mix, reduction="none")).mean()
    loss.backward()
    dz = y_mask * (torch.sigmoid(z.detach()) - y_mix) / (B * C)
    assert (dz - z.grad).abs().max().item() <= 1e-15
