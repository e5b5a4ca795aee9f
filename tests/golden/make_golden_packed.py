"""Generate tests/golden/packed.npz by running the UNMODIFIED reference in eval, one clip at a time: the per-clip results
that a batch of clips of different lengths with `lengths` must reproduce.

Run where a checkout of the original project exists (read-only), named by $EAT_REFERENCE_DIR:
    EAT_REFERENCE_DIR=<checkout> python tests/golden/make_golden_packed.py
Nets (tests/packed_util.NETS): mn04 (mlp head), mn04 with the attention head (4 heads), mn04 dilated, dymn04 with
dyrelu_k 2 and 3, dymn04 with use_dy_blocks="replace_se".  State: synth_state_(seed=7) (mha_state_ for the attention
head); the MN nets take the calibrated BatchNorm buffers of tests/golden/fmap_grad.npz, the DyMN nets keep
synth_state_'s buffers (calibrated ones drive their eval logits to 1e7 and beyond on short clips).  Clips
(tests/packed_util.clip_specs): six seeded spectrograms of 0.05, 0.37, 0.9, 1.3, 2.0 and 2.71 s (5 to 272 frames).
Recorded per net, in fp64: each clip's logits and features, each clip's 17 map time sizes (stem, 15 blocks, last conv),
and the logits of the six clips zero-padded into one batch.  No existing golden file is touched."""
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
from tests import packed_util as pu  # noqa: E402

os.chdir(REF)            # helpers/utils.py opens metadata/ relative to CWD
sys.path.insert(0, REF)
with contextlib.redirect_stdout(io.StringIO()):
    from models.dymn.model import get_model as ref_dymn  # noqa: E402
    from models.mn.model import get_model as ref_mn  # noqa: E402

import warnings  # noqa: E402
warnings.filterwarnings("ignore")
torch.set_num_threads(8)


def forward(tag, model, x, fmaps):
    if pu.NETS[tag][0] == "mn":
        return model._forward_impl(x, return_fmaps=True) if fmaps else model(x)
    return model(x, return_fmaps=fmaps)


def run(tag, res):
    kind, kw = pu.NETS[tag]
    torch.manual_seed(0)
    with contextlib.redirect_stdout(io.StringIO()):
        model = (ref_mn if kind == "mn" else ref_dymn)(width_mult=pu.WIDTH, **kw)
    pu.state_(tag, model)
    model.double().eval()
    specs = pu.clip_specs()
    logits, feats, sizes = [], [], []
    with torch.no_grad():
        for s in specs:
            lo, fe = forward(tag, model, s.double(), False)
            _, maps = forward(tag, model, s.double(), True)
            assert len(maps) == 17
            logits.append(lo.reshape(-1).numpy())
            feats.append(fe.reshape(-1).numpy())
            sizes.append([m.shape[-1] for m in maps])
        padded, _ = forward(tag, model, pu.padded_batch(specs).double(), False)
    res[tag + "__logits"] = np.stack(logits)
    res[tag + "__features"] = np.stack(feats)
    res[tag + "__sizes"] = np.array(sizes, dtype=np.int64)
    res[tag + "__padded_logits"] = padded.numpy()
    d = np.abs(res[tag + "__padded_logits"] - res[tag + "__logits"]).max()
    print(f"{tag}: |logits| {np.abs(res[tag + '__logits']).max():.4g}, padded batch off by {d:.3g}, "
          f"last sizes {res[tag + '__sizes'][:, -1].tolist()}")


if __name__ == "__main__":
    out = os.path.join(HERE, "packed.npz")
    assert not os.path.exists(out), f"{out} exists; this script only writes new files"
    res = {"frames": np.array(pu.clip_frames(), dtype=np.int64)}
    for tag in pu.NETS:
        run(tag, res)
    np.savez_compressed(out, **res)
