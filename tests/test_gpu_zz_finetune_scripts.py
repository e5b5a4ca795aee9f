"""The reference's four downstream scripts (ex_esc50.py, ex_dcase20.py, ex_fsd50k.py, ex_openmic.py), unchanged, running
on this package through scripts/run_reference_script.py --side ours --cuda: `helpers.utils` (mixup, mixstyle) and the
models resolve to this repository, `datasets.<task>` to the synthetic stand-ins under dropin/datasets.  mn04_as is
loaded from its release file with a different class count, so the "Dropping last layer" branch runs.  What each script
logs per epoch and the checkpoint it saves are compared with tests/golden/script_<task>.json, produced by the same
launcher with --side reference on CPU (tests/golden/make_golden_finetune.py).  Skipped without oracle/_ref."""
import json
import os
import re

import pytest
import torch

from tests import finetune_scripts as FS
from tests import refscripts as R
from tests.util import GOLDEN, report

pytestmark = pytest.mark.gpu

needs_ref = pytest.mark.skipif(R.ref_root() is None, reason="oracle/_ref (mirror of the reference checkout) not present")


@needs_ref
@pytest.mark.parametrize("run", list(FS.RUNS))
def test_downstream_script_runs_unchanged_and_matches_reference_run(run, tmp_path):
    """Per epoch: train loss to 2e-4 (the later steps depend on Adam updates), validation loss to 2e-3, mAP to 2e-3 and
    ROC to 5e-3 (as tests/test_gpu_refscripts.py), learning rate exactly; accuracy over the 20 validation clips to one
    clip (an arg-max between two near-equal logits may fall either way).  Checkpoint: every tensor's norm to 2e-3 of
    the reference run's, 5 % for the BatchNorm biases whose gradient is analytically zero (they random-walk by +-lr per
    Adam step in either implementation) and for the new classifier's bias (it starts at zero, so it consists only of
    its Adam updates)."""
    with open(os.path.join(GOLDEN, f"script_{FS.TASK[run]}.json")) as f:
        g = json.load(f)[run]
    wd = str(tmp_path)
    env = R.make_workdir(wd, checkpoints=("mn04_as",), env=FS.ENV)
    log, ck = os.path.join(wd, "log.json"), os.path.join(wd, "final.pt")
    r = R.run_script(wd, "ours", g["script"], g["args"] + ["--cuda"], env, log_json=log, keep_checkpoint=ck)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    assert "Dropping last layer" in r.stdout or "Dropping last layer" in r.stderr
    epochs = R.read_log(log)
    assert len(epochs) == len(g["epochs"]) == 2
    rep = []
    for e, (got, want) in enumerate(zip(epochs, g["epochs"])):
        assert set(got) == set(want), (got, want)
        rep.append({k: (round(got[k], 6), round(want[k], 6)) for k in want})
        assert abs(got["train_loss"] - want["train_loss"]) <= 2e-4, (e, got, want)
        assert abs(got["val_loss"] - want["val_loss"]) <= 2e-3, (e, got, want)
        if "accuracy" in want:
            assert abs(got["accuracy"] - want["accuracy"]) <= 1.0 / 20 + 1e-9, (e, got, want)
        if "learning_rate" in want:
            assert abs(got["learning_rate"] - want["learning_rate"]) <= 1e-12
        if "mAP" in want:
            assert abs(got["mAP"] - want["mAP"]) <= 2e-3 and abs(got["ROC"] - want["ROC"]) <= 5e-3, (e, got, want)
    report(f"[parity] {g['script']} {run} epochs (ours, reference): " + json.dumps(rep))
    sd = torch.load(ck, map_location="cpu")
    assert list(sd.keys()) == list(g["final_state"].keys())
    worst = (0.0, None)
    for k, want in g["final_state"].items():
        if "int" in want:
            assert int(sd[k]) == want["int"], k
            continue
        n = sd[k].double().norm().item()
        rel = abs(n - want["norm"]) / max(want["norm"], 1e-9)
        tol = 5e-2 if re.search(r"block\.\d\.1\.bias$", k) or k == "classifier.5.bias" else 2e-3
        assert rel <= tol, (k, n, want["norm"])
        if rel > worst[0] and tol < 1e-2:
            worst = (rel, k)
    report(f"[parity] {g['script']} {run} final checkpoint: worst tensor-norm rel err {worst[0]:.2e} ({worst[1]})")
