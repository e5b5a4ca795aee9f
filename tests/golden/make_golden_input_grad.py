"""Generate tests/golden/input_grad.npz by running the UNMODIFIED reference on the CPU in float64: gradients with
respect to the input spectrogram of mn04, mn04 with the attention head (4 heads) and dymn04, in eval() and train(), and
with respect to the waveform through AugmentMelSTFT into the eval-mode net.

Run where a checkout of the original project exists (read-only), named by $EAT_REFERENCE_DIR:
    EAT_REFERENCE_DIR=<checkout> python tests/golden/make_golden_input_grad.py
Each net: make_golden.py's state (synth_state_(seed=7), or mha_state_ for the attention head) and its training-mode
BatchNorm calibration pass on the 2 s spectrogram (B = 2) of tests/util.net_inputs, then model.double().  A fixed random
cotangent on the logits (seed 3); dropout and masks off; the mel front end in float64 through the default dtype.
Recorded per gradient: its norm, 64 strided samples and its projections on four seeded random vectors (seed 17), in
float64.  No existing golden file is touched."""
import contextlib
import io
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
REF = os.environ["EAT_REFERENCE_DIR"]
sys.path.insert(0, REPO)
from efficientat_b200.synth import bn_modules, get_bn_stats, synth_state_, synth_waveform  # noqa: E402
from tests.input_grad_util import WAVE_SAMPLES, cotangent, digest, spec_input  # noqa: E402
from tests.mha_util import mha_state_  # noqa: E402

os.chdir(REF)            # helpers/utils.py opens metadata/ relative to CWD
sys.path.insert(0, REF)
with contextlib.redirect_stdout(io.StringIO()):
    from models.dymn.model import get_model as ref_dymn  # noqa: E402
    from models.mn.model import get_model as ref_mn  # noqa: E402
    from models.preprocess import AugmentMelSTFT as RefMel  # noqa: E402

import warnings  # noqa: E402
warnings.filterwarnings("ignore")
torch.set_num_threads(8)


def build(tag):
    torch.manual_seed(0)
    with contextlib.redirect_stdout(io.StringIO()):
        if tag == "mn04":
            m = synth_state_(ref_mn(width_mult=0.4), seed=7)
        elif tag == "mn04_mha":
            m = ref_mn(width_mult=0.4, num_classes=527, head_type="multihead_attention_pooling", multihead_attention_heads=4)
            mha_state_(m, 4)
        else:
            m = synth_state_(ref_dymn(width_mult=0.4), seed=7)
    return m


def run(tag, res):
    model = build(tag)
    spec = spec_input()
    model.train()
    for _, m in bn_modules(model):
        m.momentum = 1.0
    with torch.no_grad():
        model(spec)
    for _, m in bn_modules(model):
        m.momentum = 0.01
        m.num_batches_tracked.zero_()
    cal_rm, cal_rv = get_bn_stats(model)
    res[tag + "__cal_rm"], res[tag + "__cal_rv"] = cal_rm.numpy(), cal_rv.numpy()
    for m in model.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    model.double()
    cot = cotangent()
    # eval: spectrogram, then waveform -> AugmentMelSTFT -> net
    model.eval()
    x = spec.double().requires_grad_(True)
    (model(x)[0] * cot).sum().backward()
    res[tag + "__dspec_eval"] = digest(x.grad)
    # the reference builds its mel filterbank in the default dtype at every call (preprocess.py:52-55)
    torch.set_default_dtype(torch.float64)
    try:
        with contextlib.redirect_stdout(io.StringIO()):
            mel = RefMel(freqm=0, timem=0).eval()
        w = synth_waveform(2, WAVE_SAMPLES, seed=5).double().requires_grad_(True)
        (model(mel(w).unsqueeze(1))[0] * cot).sum().backward()
    finally:
        torch.set_default_dtype(torch.float32)
    res[tag + "__dwave_eval"] = digest(w.grad)
    # train: batch-statistics BatchNorm (updates the running buffers, so it runs last)
    model.train()
    x = spec.double().requires_grad_(True)
    (model(x)[0] * cot).sum().backward()
    res[tag + "__dspec_train"] = digest(x.grad)
    print(f"{tag}: |dspec| eval {res[tag + '__dspec_eval'][0]:.6g} train {res[tag + '__dspec_train'][0]:.6g}, "
          f"|dwave| {res[tag + '__dwave_eval'][0]:.6g}")


if __name__ == "__main__":
    out = os.path.join(HERE, "input_grad.npz")
    assert not os.path.exists(out), f"{out} exists; this script only writes new files"
    res = {}
    for tag in ("mn04", "mn04_mha", "dymn04"):
        run(tag, res)
    np.savez_compressed(out, **res)
