"""Resample (efficientat_b200/resample.py) without a GPU: the numpy filter, the alignment constants and the fp64
restatement of the kernels' index math against scipy.signal.resample_poly, the adjoint identity, and the argument checks
of the module and of both C entry points."""
import numpy as np
import pytest
import scipy.signal as ss
import torch

from efficientat_b200._lib import EatError, lib
from efficientat_b200.resample import Resample, alignment, design_filter, rates
from tests.resample_util import resample, resample_adjoint

NATIVE = (8000, 11025, 16000, 22050, 24000, 44100, 48000, 88200, 96000)
PAIRS = [(r, 32000) for r in NATIVE] + [(32000, r) for r in NATIVE]
LIMIT = [(2047, 2048), (2048, 2047), (1, 2048), (2048, 1)]                      # max(up, down) = 2048


def _signal(n, seed):
    g = np.random.default_rng(seed)
    t = np.arange(n) / 44100.0
    return np.sin(2 * np.pi * (200 + 3000 * t) * t) + 0.3 * g.standard_normal(n)


@pytest.mark.parametrize("orig,new", PAIRS + LIMIT)
def test_filter_matches_scipy_firwin(orig, new):
    up, down = rates(orig, new)
    h, hl = design_filter(up, down)
    ref = ss.firwin(2 * hl + 1, 1.0 / max(up, down), window=("kaiser", 5.0)) * up
    assert hl == 10 * max(up, down) and h.shape == ref.shape
    assert np.abs(h - ref).max() <= 1e-15 * up


def _scipy_constants(n_in, up, down):
    """the constants as scipy.signal.resample_poly (scipy/signal/_signaltools.py) computes them"""
    hl = 10 * max(up, down)
    n_out = n_in * up
    n_out = n_out // down + bool(n_out % down)
    n_pre_pad = down - hl % down
    return n_pre_pad, (hl + n_pre_pad) // down, n_out


@pytest.mark.parametrize("orig,new", [(48000, 32000), (16000, 32000), (32000, 16000), (44100, 32000), (32000, 8000)])
def test_alignment_constants_and_output_count(orig, new):
    up, down = rates(orig, new)
    _, hl = design_filter(up, down)
    for n_in in list(range(1, hl + 8)) if hl < 100 else [1, 2, 3, down - 1, down, down + 1, hl - 1, hl, hl + 1, hl + 500]:
        pre_pad, pre_remove, n_out = alignment(n_in, up, down, hl)
        assert (pre_pad, pre_remove, n_out) == _scipy_constants(n_in, up, down)
        assert pre_remove * down - pre_pad == hl                  # the kernels' offset
        assert n_out == len(ss.resample_poly(np.zeros(n_in), up, down))


@pytest.mark.parametrize("orig,new", PAIRS + [(32000, 16000), (2047, 2048), (1, 2048)])
def test_restatement_matches_resample_poly(orig, new):
    up, down = rates(orig, new)
    _, hl = design_filter(up, down)
    lens = [1, 2, 7, 333, 1001] + ([hl // up + 3] if hl // up + 3 < 4000 else [])
    for n in lens:
        x = _signal(n, seed=n)
        ref = ss.resample_poly(x, up, down)
        got = resample(torch.from_numpy(x)[None], orig, new)[0].numpy()
        assert got.shape == ref.shape
        assert np.abs(got - ref).max() <= 1e-12 * max(1.0, np.abs(ref).max()), (orig, new, n)


@pytest.mark.parametrize("orig,new", [(44100, 32000), (48000, 32000), (16000, 32000), (32000, 16000), (11025, 32000)])
def test_adjoint_identity(orig, new):
    up, down = rates(orig, new)
    g = torch.Generator().manual_seed(1)
    for n in (1, 5, 999):
        x = torch.randn(3, n, generator=g, dtype=torch.float64)
        n_out = -(-n * up // down)
        gy = torch.randn(3, n_out, generator=g, dtype=torch.float64)
        lhs = (resample(x, orig, new) * gy).sum()
        rhs = (x * resample_adjoint(gy, n, orig, new)).sum()
        assert abs(lhs - rhs) <= 1e-12 * (lhs.abs() + 1)
        # and the adjoint table is what autograd of the forward gather gives
        xg = x.clone().requires_grad_(True)
        resample(xg, orig, new).backward(gy)
        assert torch.allclose(xg.grad, resample_adjoint(gy, n, orig, new), rtol=0, atol=1e-12)


def test_num_samples_and_rates():
    rs = Resample(44100)
    assert (rs.up, rs.down, rs.half_len, rs.taps) == (320, 441, 4410, 28)
    assert rs.num_samples([1, 441, 442, 441000]) == [1, 320, 321, 320000]
    assert rs.num_samples(torch.tensor([2, 3])) == [2, 3]
    assert Resample(32000, 16000).num_samples([1, 2, 3]) == [1, 1, 2]
    assert Resample(48000).num_samples([3, 4]) == [2, 3]
    assert Resample(32000).identity and Resample(64000, 32000).num_samples([5]) == [3]
    assert not rs._table.dtype.is_complex and "_table" not in rs.state_dict()


def test_module_argument_checks():
    with pytest.raises(NotImplementedError, match="2048"):
        Resample(44101)                                            # up / down = 32000 / 44101
    with pytest.raises(NotImplementedError, match="2048"):
        Resample(32000, 2049)
    with pytest.raises(ValueError):
        Resample(0)
    with pytest.raises(ValueError):
        Resample(44100.5)
    rs = Resample(44100)
    x = torch.zeros(2, 100)
    with pytest.raises(RuntimeError, match="CUDA"):
        rs(x)
    with pytest.raises(ValueError):
        rs(torch.zeros(100))
    for bad in ([0, 5], [5, 101], [5], [1.5, 2], torch.tensor([5.0, 6.0])):
        with pytest.raises(ValueError):
            rs(x, bad)
    with pytest.raises(NotImplementedError, match="grad"):
        rs(x.requires_grad_(True), [5, 6])


def test_entry_point_argument_checks():
    """validation comes before any launch, so these calls are safe without a GPU"""
    L = lib()
    fake = 4096                                                    # never dereferenced
    n_out = -(-1000 * 320 // 441)
    for fn, rows in ((L.resample_poly_fwd, 320), (L.resample_poly_bwd, 441)):
        args = lambda **kw: dict(dict(B=2, N=1000, up=320, down=441, taps=28, off=4410, n_out=n_out), **kw)

        def call(B, N, up, down, taps, off, n_out, ptr=fake):
            if fn is L.resample_poly_fwd:
                fn(ptr, B, N, 0, up, down, fake, taps, off, fake, n_out, 0)
            else:
                fn(ptr, B, N, up, down, fake, taps, off, fake, n_out, 0)
        with pytest.raises(EatError, match="at most 2048"):
            call(**args(up=2049))
        with pytest.raises(EatError, match="at most 2048"):
            call(**args(down=2049))
        with pytest.raises(EatError, match="43008 floats"):
            call(**args(taps=43008 // rows + 1))
        with pytest.raises(EatError, match="n_out must be"):
            call(**args(n_out=n_out + 1))
        with pytest.raises(EatError, match="need B >= 0"):
            call(**args(B=-1))
        with pytest.raises(EatError, match="need B >= 0"):
            call(**args(N=0))
        with pytest.raises(EatError, match="need B >= 0"):
            call(**args(off=-1))
        with pytest.raises(EatError, match="are required"):
            call(**args(), ptr=0)
        call(**args(B=0), ptr=0)                                   # an empty batch is a no-op
    with pytest.raises(EatError, match="fit in int32"):
        L.resample_poly_fwd(fake, 1, 1 << 30, 0, 3, 1, fake, 21, 30, fake, 3 << 30 & 0x7fffffff, 0)
