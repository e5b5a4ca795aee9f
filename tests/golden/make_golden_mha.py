"""Generate tests/golden/mn_mha.npz and statedict_mn04_mha.json by running the UNMODIFIED reference MN with
head_type='multihead_attention_pooling' (models/mn/attention_pooling.py).

Run where a checkout of the original project exists (read-only), named by $EAT_REFERENCE_DIR:
    EAT_REFERENCE_DIR=<checkout> python tests/golden/make_golden_mha.py
The tests only read the files.  The model state follows the calibrated-state recipe of make_golden.py (run_net):
synth_state_, one training-mode BatchNorm calibration pass, eval outputs, then one training step with BCE; on top of it
the head weights get distinct values per head (tests/mha_util.mha_state_).  Per case (tests/mha_util.CASES) the file
holds, under "<case>__<name>": the calibrated BatchNorm buffers, eval logits / features / feature-map digests, the
training step's logits, loss, per-parameter gradient norms and samples and BatchNorm running statistics, and the
fraction of (b, h, k) whose normalised attention over t has max / min >= 1.5 (eval and training), which the tests
require to be large: an attention that is uniform over t would hide errors in the attention path.
"""
import contextlib
import io
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
REF = os.environ["EAT_REFERENCE_DIR"]
sys.path.insert(0, REPO)
from efficientat_b200.synth import bn_modules, get_bn_stats  # noqa: E402
from tests.mha_util import CASES, HEAD, att_far_from_uniform, attention_weights, case_inputs, mha_state_  # noqa: E402
from tests.util import fmap_digest  # noqa: E402

os.chdir(REF)            # helpers/utils.py opens metadata/ relative to CWD
sys.path.insert(0, REF)
with contextlib.redirect_stdout(io.StringIO()):
    from models.mn.model import get_model as ref_mn  # noqa: E402

import warnings  # noqa: E402
warnings.filterwarnings("ignore")
torch.set_num_threads(8)


def run_case(case, res):
    width, _, batch, H, K = CASES[case]
    torch.manual_seed(0)
    with contextlib.redirect_stdout(io.StringIO()):
        model = ref_mn(width_mult=width, num_classes=K, head_type=HEAD, multihead_attention_heads=H)
    mha_state_(model, H)
    spec, y = case_inputs(case)
    head_in = []
    model.classifier.register_forward_hook(lambda mod, inp, out: head_in.append(inp[0].detach()))
    model.train()
    for _, m in bn_modules(model):
        m.momentum = 1.0
    with torch.no_grad():
        model(spec)
    for _, m in bn_modules(model):
        m.momentum = 0.01
        m.num_batches_tracked.zero_()
    cal_rm, cal_rv = get_bn_stats(model)
    r = {"cal_rm": cal_rm.numpy(), "cal_rv": cal_rv.numpy(),
         "head_weight": model.classifier.head_weight.detach().numpy().copy()}
    proj = model.classifier.subspace_proj
    if case == "mn04_h4":
        with open(os.path.join(HERE, "statedict_mn04_mha.json"), "w") as fh:     # on-disk checkpoint contract
            json.dump({k: list(v.shape) for k, v in model.state_dict().items()}, fh, indent=0)
    # ---- eval
    model.eval()
    head_in.clear()
    with torch.no_grad():
        logits, feat = model(spec)
        _, fmaps = model._forward_impl(spec, return_fmaps=True)
    att = attention_weights(head_in[0], proj.weight, proj.bias, H, K)
    r.update(eval_logits=logits.numpy(), eval_feat=feat.numpy(), eval_fmaps=fmap_digest(fmaps),
             eval_att_far=np.float64(att_far_from_uniform(att)))
    # ---- one training step (batch-statistics BatchNorm; the head has no dropout, the trunk none either)
    model.train()
    head_in.clear()
    logits_t, _ = model(spec)
    with torch.no_grad():
        att_t = attention_weights(head_in[0], proj.weight, proj.bias, H, K)
    loss = torch.nn.functional.binary_cross_entropy_with_logits(logits_t, y)
    loss.backward()
    names, gnorm, gsamp = [], [], []
    for n, p in model.named_parameters():
        names.append(n)
        g = p.grad.flatten()
        gnorm.append(g.double().norm().item())
        gsamp.append(g[torch.linspace(0, g.numel() - 1, 4).long()].numpy())
    bn_names, bn_rm, bn_rv = [], [], []
    for n, m in model.named_modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            bn_names.append(n)
            bn_rm.append(m.running_mean[:4].numpy().copy())
            bn_rv.append(m.running_var[:4].numpy().copy())
    r.update(train_logits=logits_t.detach().numpy(), train_loss=np.float64(loss.item()), grad_names=np.array(names),
             grad_norm=np.array(gnorm), grad_samples=np.stack(gsamp), bn_names=np.array(bn_names),
             bn_rm4=np.stack(bn_rm), bn_rv4=np.stack(bn_rv), train_att_far=np.float64(att_far_from_uniform(att_t)))
    res.update({f"{case}__{k}": v for k, v in r.items()})
    print(case, "eval logits absmax", logits.abs().max().item(), "train loss", loss.item(),
          "attention far from uniform (eval, train)", r["eval_att_far"], r["train_att_far"])


def nets():
    res = {}
    for case in CASES:
        run_case(case, res)
    np.savez_compressed(os.path.join(HERE, "mn_mha.npz"), **res)


def script():
    """ex_audioset.py --train with this head, unchanged, on the reference's own modules (CPU), as make_golden.py's
    golden_script does for the mlp head -> script_mn04_mha.json (tests/test_gpu_zz_mha_head.py runs it with --side ours)"""
    import tempfile
    from tests import refscripts as R
    from tests.mha_util import script_args
    from make_golden import state_digest      # this directory is on sys.path: the script's own
    os.chdir(REPO)
    with tempfile.TemporaryDirectory() as wd:
        env = R.make_workdir(wd, checkpoints=())
        log, ck = os.path.join(wd, "log.json"), os.path.join(wd, "final.pt")
        r = R.run_script(wd, "reference", "ex_audioset.py", script_args(), env, log_json=log, keep_checkpoint=ck)
        assert r.returncode == 0, r.stderr[-3000:]
        sd = torch.load(ck, map_location="cpu")
        res = {"args": script_args(), "env": R.SCRIPT_ENV, "epochs": R.read_log(log), "final_state": state_digest(sd)}
    with open(os.path.join(HERE, "script_mn04_mha.json"), "w") as fh:
        json.dump(res, fh, indent=0)
    print("script: epochs", [e["train_loss"] for e in res["epochs"]])


if __name__ == "__main__":
    for job in (sys.argv[1:] or ["nets", "script"]):
        {"nets": nets, "script": script}[job]()
