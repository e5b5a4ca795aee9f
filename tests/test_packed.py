"""Clips of different lengths in one eval batch (`lengths`), without a GPU.

- Goldens (tests/golden/packed.npz, the unmodified reference run one clip at a time): the fp64 oracle per clip matches
  them; the six clips zero-padded into one batch give logits far from the per-clip ones, so the goldens see padding;
  the host's per-stage table equals the reference's map sizes of each clip.
- Length arithmetic: the host's per-stage table (efficientat_b200.packed.stage_sizes) equals the map sizes of the fp64
  oracle nets at every clip length, for MN, MN with strides (2, 2, 2, 1), dilated MN and DyMN.
- Argument checks: a wrong count, a value out of range, a non-integer, a tensor on the device; eval only, no input that
  requires grad, no return_fmaps.  Every new C entry point rejects bad arguments with EatError before any launch, and
  B = 0 is a no-op."""
import contextlib
import io

import numpy as np
import pytest
import torch

from efficientat_b200._lib import EatError, lib
from efficientat_b200.packed import StageLengths, as_int_list, check_lengths, stage_sizes
from efficientat_b200.synth import synth_state_
from oracle import net_oracle as no
from tests import dilated_util as du
from tests import packed_util as pu
from tests.util import golden

F_IN = 16                                    # the frequency size does not change any time size
CLIPS = list(range(1, 14)) + [31, 64, 99, 100, 101]


def _model(kind, **kw):
    if kind == "mn":
        from efficientat_b200.models.mn.model import get_model
    else:
        from efficientat_b200.models.dymn.model import get_model
    torch.manual_seed(0)
    with contextlib.redirect_stdout(io.StringIO()):
        m = get_model(width_mult=0.4, verbose=False, **kw)
    return synth_state_(m, seed=7).eval()


CASES = {
    "mn": ("mn", {}, lambda sd, x: no.mn_forward(sd, x, width_mult=0.4, return_fmaps=True)),
    "mn_s2221": ("mn", dict(strides=(2, 2, 2, 1)),
                 lambda sd, x: no.mn_forward(sd, x, width_mult=0.4, strides=(2, 2, 2, 1), return_fmaps=True)),
    "mn_dilated": ("mn", dict(dilated=True),
                   lambda sd, x: du.mn_forward(sd, x, width_mult=0.4, dilated=True, return_fmaps=True)),
    "dymn": ("dymn", {}, lambda sd, x: no.dymn_forward(sd, x, width_mult=0.4, return_fmaps=True)),
}


@pytest.mark.parametrize("case", list(CASES))
def test_stage_table_matches_the_oracle_map_sizes(case):
    kind, kw, fwd = CASES[case]
    model = _model(kind, **kw)
    sd = model.state_dict()
    sizes = stage_sizes(model.engine(), F_IN, max(CLIPS), CLIPS)
    assert len(sizes) == 2 + len(model.engine().blocks)
    for b, t in enumerate(CLIPS):
        x = torch.randn(1, 1, F_IN, t, generator=torch.Generator().manual_seed(t))
        with torch.no_grad():
            fmaps = fwd(sd, x)[2]
        # fmaps: stem, every block, last conv; sizes: the input, stem, every block
        got = [s[2][b] for s in sizes[1:]]
        want = [f.shape[-1] for f in fmaps[:len(got)]]
        assert got == want, (t, got, want)
        assert sizes[0][2][b] == t
    # the batch's own sizes are those of its longest clip
    assert [s[1] for s in sizes] == [s[2][CLIPS.index(max(CLIPS))] for s in sizes]


@pytest.mark.parametrize("tag", pu.ORACLE)
def test_fp64_oracle_per_clip_matches_reference_goldens(tag):
    g = golden("packed")
    model = pu.build_model(tag)
    for b, spec in enumerate(pu.clip_specs()):
        logits, feat, _ = pu.oracle_forward(tag, model, spec)
        ref_l, ref_f = g[tag + "__logits"][b], g[tag + "__features"][b]
        # fp64 on both sides: rounding only
        assert np.abs(logits[0].numpy() - ref_l).max() <= 1e-9 * max(1.0, np.abs(ref_l).max()), b
        assert np.abs(feat[0].numpy() - ref_f).max() <= 1e-9 * max(1.0, np.abs(ref_f).max()), b


@pytest.mark.parametrize("tag", list(pu.NETS))
def test_padded_batch_goldens_differ_from_per_clip(tag):
    g = golden("packed")
    d = np.abs(g[tag + "__padded_logits"] - g[tag + "__logits"]).max()
    # the DyMN nets keep synth_state_'s BatchNorm buffers, under which their features vary little from clip to clip
    # (the padded batch moves their logits by 4.2e-3 - 4.4e-3); the MN nets move by 0.26 - 0.76
    assert d > (1e-2 if pu.NETS[tag][0] == "mn" else 2e-3), d


@pytest.mark.parametrize("tag", list(pu.NETS))
def test_stage_table_matches_reference_map_sizes(tag):
    g = golden("packed")
    frames = pu.clip_frames()
    assert g["frames"].tolist() == frames
    sizes = stage_sizes(pu.build_model(tag).engine(), 128, max(frames), frames)
    for b in range(len(frames)):
        got = [s[2][b] for s in sizes[1:]]
        want = g[tag + "__sizes"][b].tolist()
        assert got == want[:len(got)] and want[-1] == got[-1], (b, got, want)   # the last conv keeps the last block's


def test_stage_lengths_table_rows():
    model = _model("dymn")
    lens = StageLengths(model.engine(), F_IN, 20, [20, 3, 1], torch.device("cpu"))
    S = lens.n
    assert tuple(lens.table.shape) == (2 * S, 3) and lens.table.dtype == torch.int32
    for s, (Fs, _, t) in enumerate(lens.sizes):
        assert lens.table[s].tolist() == t
        assert lens.table[S + s].tolist() == [Fs + v for v in t]
    assert lens.padded(0) and not StageLengths(model.engine(), F_IN, 20, [20, 20], torch.device("cpu")).padded(0)
    empty = StageLengths(model.engine(), F_IN, 20, [], torch.device("cpu"))      # B = 0
    assert not any(empty.padded(s) for s in range(empty.n))


def test_length_arguments():
    assert check_lengths([3, 1, 2], 3, 1, 3) == [3, 1, 2]
    assert check_lengths(torch.tensor([3, 1, 2], dtype=torch.int32), 3, 1, 3) == [3, 1, 2]
    assert check_lengths((4, 4), 2, 1, 4) == [4, 4]
    for bad in ([3, 1], [3, 1, 2, 2], [3, 0, 2], [3, 4, 2], [3, 1.0, 2], [3, True, 2], [3, "2", 2],
                torch.tensor([3.0, 1.0, 2.0]), torch.tensor([[3, 1, 2]]), 5):
        with pytest.raises(ValueError):
            check_lengths(bad, 3, 1, 3)
    assert as_int_list(torch.tensor([5, 6])) == [5, 6]


def test_model_and_mel_length_checks():
    from efficientat_b200.models.preprocess import AugmentMelSTFT
    with contextlib.redirect_stdout(io.StringIO()):
        mel = AugmentMelSTFT(freqm=0, timem=0)
    assert mel.num_frames([32000, 320, 321, 1600]) == [100, 1, 2, 5]
    for kind in ("mn", "dymn"):
        model = _model(kind)
        eng = model.engine()
        x = torch.zeros(3, 1, 128, 50)
        assert eng._check_lengths(x, False, None) is None
        assert eng._check_lengths(x, False, [50, 1, 7]) == [50, 1, 7]
        for bad in ([50, 1], [50, 0, 7], [50, 51, 7], [50, 1.5, 7]):
            with pytest.raises(ValueError):
                eng._check_lengths(x, False, bad)
        with pytest.raises(NotImplementedError, match="lengths"):
            eng._check_lengths(x, True, [50, 1, 7])
        with pytest.raises(NotImplementedError, match="lengths"):
            eng._check_lengths(x.clone().requires_grad_(True), False, [50, 1, 7])
        model.train()
        with pytest.raises(NotImplementedError, match="lengths"):
            eng._check_lengths(x, False, [50, 1, 7])


def test_entry_points_reject_bad_arguments_before_any_launch():
    L = lib()
    p = 16                                  # a non-null pointer that is never dereferenced: the checks come first
    pad = lambda *a: L.time_pad_zero(a[0], a[1], *a[2:])              # noqa: E731  (x, dtype, B, F, T, C, t_valid, st)
    ctx = lambda *a: L.ctx_pool_len(a[0], a[1], p, *a[2:])            # noqa: E731  (x, dtype, out, B, F, T, C, ...)
    mean = lambda *a: L.mean_len(a[0], a[1], p, *a[2:])               # noqa: E731
    for fn in (pad, ctx, mean):
        with pytest.raises(EatError):
            fn(p, 2, 1, 1, 1, 8, p, None)                    # dtype
        with pytest.raises(EatError):
            fn(p, 0, -1, 1, 1, 8, p, None)                   # B
        with pytest.raises(EatError):
            fn(p, 0, 1, 0, 1, 8, p, None)                    # F
        with pytest.raises(EatError):
            fn(p, 0, 1, 1, 0, 8, p, None)                    # T
        with pytest.raises(EatError):
            fn(p, 0, 1, 1, 1, 0, p, None)                    # C
        with pytest.raises(EatError):
            fn(0, 0, 1, 1, 1, 8, p, None)                    # x
        with pytest.raises(EatError):
            fn(p, 0, 1, 1, 1, 8, 0, None)                    # t_valid
    with pytest.raises(EatError):
        L.ctx_pool_len(p, 0, p, 1, 1, 1, 6, p, None)         # C not a multiple of the vector width
    with pytest.raises(EatError):
        L.ctx_pool_len(p, 0, 1, 1, 1, 8, p, 0, None)         # out
    with pytest.raises(EatError):
        L.mean_len(p, 0, 0, 1, 1, 1, 8, p, None)             # out
    with pytest.raises(EatError):
        L.att_pool_fwd_len(p, p, 1e-7, p, 1, 4, 2, 3, 0, None)            # t_valid
    with pytest.raises(EatError):
        L.att_pool_fwd_len(p, p, 0.7, p, 1, 4, 2, 3, p, None)            # eps
    with pytest.raises(EatError):
        L.att_pool_fwd_len(p, p, 1e-7, p, 1, 0, 2, 3, p, None)           # T
    mel_args = lambda B, N, n_fft, nv: (p, B, N, p, 800, 320, n_fft, p, p, p, p, 20, 128, 0.97, p, nv, None)  # noqa: E731
    with pytest.raises(EatError):
        L.mel_fwd_len(*mel_args(2, 32000, 1024, 0))                       # n_valid
    with pytest.raises(EatError):
        L.mel_fwd_len(*mel_args(2, 32000, 1000, p))                       # n_fft
    with pytest.raises(EatError):
        L.mel_fwd_len(*mel_args(2, 500, 1024, p))                         # too short for reflect padding
    # B = 0: nothing to do, nothing launched
    L.time_pad_zero(0, 0, 0, 1, 1, 8, 0, None)
    L.mean_len(0, 0, 0, 0, 1, 1, 8, 0, None)
    L.ctx_pool_len(0, 0, 0, 0, 1, 1, 8, 0, None)
    L.att_pool_fwd_len(0, 0, 1e-7, 0, 0, 4, 2, 3, 0, None)
    L.mel_fwd_len(*mel_args(0, 32000, 1024, 0))
