"""Goldens of the four downstream scripts run unchanged with the reference's own modules on CPU
(scripts/run_reference_script.py --side reference): tests/golden/script_{esc50,dcase20,fsd50k,openmic}.json with every
logged record (loss, accuracy / mAP / ROC, validation loss, learning rate) and a digest of the saved checkpoint.
tests/test_gpu_zz_finetune_scripts.py runs the same scripts with `--side ours --cuda`.

    python tests/golden/make_golden_finetune.py          (needs oracle/_ref, i.e. a reference checkout at build time)
"""
import json
import os
import sys
import tempfile

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REPO)

from tests import finetune_scripts as FS          # noqa: E402
from tests import refscripts as R                  # noqa: E402


def state_digest(sd):
    """per-tensor L2 norm + 4 strided samples of a state_dict, as tests/golden/make_golden.py records it"""
    out = {}
    for k, v in sd.items():
        if not torch.is_floating_point(v):
            out[k] = {"int": int(v)}
            continue
        f = v.detach().flatten().double()
        idx = torch.linspace(0, f.numel() - 1, 4).long()
        out[k] = {"norm": f.norm().item(), "samples": [float(x) for x in f[idx]]}
    return out


def main():
    assert R.ref_root() is not None, "oracle/_ref is missing: run `python oracle/make_ref.py`"
    out = {}
    for name, (script, extra) in FS.RUNS.items():
        with tempfile.TemporaryDirectory() as wd:
            env = R.make_workdir(wd, checkpoints=("mn04_as",), env=FS.ENV)
            log, ck = os.path.join(wd, "log.json"), os.path.join(wd, "final.pt")
            args = FS.COMMON + extra
            r = R.run_script(wd, "reference", script, args, env, log_json=log, keep_checkpoint=ck)
            assert r.returncode == 0, r.stderr[-3000:]
            sd = torch.load(ck, map_location="cpu")
            out.setdefault(FS.TASK[name], {})[name] = {"script": script, "args": args, "env": FS.ENV,
                                                       "epochs": R.read_log(log), "final_state": state_digest(sd)}
            print(name, [{k: round(v, 5) for k, v in e.items()} for e in out[FS.TASK[name]][name]["epochs"]], flush=True)
    for task, runs in out.items():
        with open(os.path.join(HERE, f"script_{task}.json"), "w") as fh:
            json.dump(runs, fh, indent=0)


if __name__ == "__main__":
    main()
