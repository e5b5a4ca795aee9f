"""The C-ABI shared library loads (no GPU needed) and exports every symbol include/eat_b200.h declares."""
import ctypes
import os
import re
import subprocess

import pytest

from efficientat_b200 import _lib


def test_library_exports_every_declared_symbol():
    assert os.path.exists(_lib.LIB_PATH), "run `python -m efficientat_b200.build` first"
    protos = _lib.parse_header()
    assert len(protos) >= 12
    dll = ctypes.CDLL(_lib.LIB_PATH)
    for name in protos:
        assert hasattr(dll, name), f"{name} declared in include/eat_b200.h but not exported"
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True).stdout
    exported = set(re.findall(r" T (eat_\w+)", out))
    assert exported == set(protos), f"header/library mismatch: {exported ^ set(protos)}"


def test_abi_version_and_error_string():
    l = _lib.lib()
    assert l.abi_version() == 3
    assert isinstance(l.last_error(), bytes)


def test_no_torch_types_in_signatures():
    text = re.sub(r"/\*.*?\*/", "", open(_lib.HEADER_PATH).read(), flags=re.S)     # strip comments
    assert "at::" not in text and "torch" not in text and "Tensor" not in text


def test_product_does_not_import_oracle():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    pkg = os.path.join(root, "efficientat_b200")
    for dp, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(".py"):
                src = open(os.path.join(dp, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle", src, re.M), f"{f} imports the oracle"


def test_depthwise_launch_plan_host_logic():
    """eat_dw_plan (host only): the sliding-window kernels' launch plan covers every channel, keeps all CTAs resident,
    and at the bench batch size loses little to the rounding of units per thread."""
    import ctypes
    from efficientat_b200._lib import lib
    L = lib()
    plan = (ctypes.c_int * 6)()
    shapes = [(64, 500, 16, 3, 1), (64, 500, 64, 3, 2), (32, 250, 72, 3, 1), (32, 250, 72, 5, 2), (16, 125, 120, 5, 1),
              (16, 125, 240, 3, 2), (8, 63, 200, 3, 1), (8, 63, 672, 5, 2), (4, 32, 960, 5, 1), (1, 9, 32, 3, 1), (5, 3, 2560, 5, 2)]
    for kind in (0, 1, 2):
        for dtype in (0, 1):
            for B in (1, 8, 256):
                for per_sample in (0, 1):
                    for (F, T, C, k, s) in shapes:
                        if kind == 2 and s != 2:
                            continue
                        if kind == 1 and k == 5 and dtype == 1:
                            with pytest.raises(RuntimeError):
                                L.dw_plan(kind, dtype, B, F, T, C, k, s, per_sample, ctypes.addressof(plan))
                            continue
                        L.dw_plan(kind, dtype, B, F, T, C, k, s, per_sample, ctypes.addressof(plan))
                        chunks, cvc, seg, groups, gy, P = list(plan)
                        V = (8 if dtype else 4) if not (kind == 1 and k == 5) else 2
                        pad = (k - 1) // 2
                        Fo, To = (F + 2 * pad - k) // s + 1, (T + 2 * pad - k) // s + 1
                        rows, cols = ((F + 1) // 2, T) if kind == 2 else (Fo, To)
                        assert chunks >= 1 and cvc >= 1 and chunks * cvc >= C // V and cvc * V <= 512 and cvc <= 128
                        assert 1 <= seg <= max(rows, 1) and groups >= 1 and gy >= 1 and P in (1, 2, 4)
                        assert chunks * groups * gy <= 132 * 5 or per_sample      # one resident wave unless blockIdx.y = sample
                        if per_sample:
                            assert gy == B
                        if B == 256 and not per_sample and F >= 4 and T >= 32:
                            ppb = max(1, 128 // cvc)
                            units = -(-cols // P) * -(-rows // seg) * B
                            slots = groups * gy * ppb
                            rounds = -(-units // slots)
                            assert rounds * slots <= 1.34 * units, (kind, dtype, (F, T, C, k, s), list(plan), rounds * slots / units)
    with pytest.raises(RuntimeError):
        L.dw_plan(0, 0, 1, 8, 8, 6, 3, 1, 0, ctypes.addressof(plan))       # channels not a multiple of the vector width
    # kind 4, the 5x5 tile kernel: 32-channel chunks, FR x 32/stride tiles, about six CTAs per SM over chunks and
    # samples, never more CTAs per chunk than tiles; blockIdx.y is the sample
    for B in (1, 3, 256):
        for (F, T, C, k, s) in shapes:
            if k != 5:
                with pytest.raises(RuntimeError):
                    L.dw_plan(4, 0, B, F, T, C, k, s, 0, ctypes.addressof(plan))
                continue
            L.dw_plan(4, 0, B, F, T, C, k, s, 0, ctypes.addressof(plan))
            chunks, cc, tiles, groups, gy, FR = list(plan)
            Fo, To = (F + 4 - k) // s + 1, (T + 4 - k) // s + 1
            assert cc == 32 and chunks * 32 >= C > (chunks - 1) * 32 and gy == B and FR == (8 if s == 1 else 4)
            assert tiles == -(-Fo // FR) * -(-To // (32 // s)) and 1 <= groups <= tiles
            assert groups in (1, tiles) or chunks * groups * B <= 132 * 6
            if B == 256 and tiles > 1:
                assert groups < tiles                                     # several tiles per CTA at the bench batch


def test_argument_errors_are_reported_before_any_launch():
    """Error behaviour of the boundary (SURVEY section 8b: int status + message, the shim raises): invalid arguments are
    rejected on the host, so these calls are safe without a GPU.  Covers the entry points added for the BatchNorm-backward
    fusions; the binding turns a non-zero status into EatError carrying eat_last_error()."""
    import pytest
    from efficientat_b200._lib import EatError, lib
    L = lib()
    fake = 4096                                                   # never dereferenced: validation comes first
    with pytest.raises(EatError, match="multiple of the vector width"):
        L.se_bn_bwd_reduce(fake, fake, fake, fake, fake, 1, fake, fake, 3, 0, 2, 16, 10, 0)           # C = 10, fp32 vectors of 4
    with pytest.raises(EatError, match="multiple of the vector width"):
        L.se_bn_bwd_reduce(fake, fake, fake, fake, fake, 1, fake, fake, 3, 1, 2, 16, 12, 0)           # C = 12, bf16 vectors of 8
    with pytest.raises(EatError, match="parts and P must be positive"):
        L.se_bn_bwd_reduce(fake, fake, fake, fake, fake, 1, fake, fake, 0, 0, 2, 16, 16, 0)
    with pytest.raises(EatError, match="parts must be positive"):
        L.se_bn_bwd_combine(fake, 0, fake, fake, fake, 2, 16, fake, fake, 0)
    with pytest.raises(EatError, match="are required"):
        L.dw_conv_dgrad_bnred(fake, fake, 0, fake, 0, fake, fake, fake, fake, 1, fake, fake, 0, 2, 8, 8, 16, 3, 2, 0)   # z missing
    with pytest.raises(EatError, match="stride 2"):
        L.dw_conv_dgrad_bnred(fake, fake, 0, fake, fake, fake, fake, fake, fake, 1, fake, fake, 0, 2, 8, 8, 16, 3, 1, 0)
    with pytest.raises(EatError, match="fp32 storage"):
        L.dw_conv_dgrad_bnred(fake, fake, 0, fake, fake, fake, fake, fake, fake, 1, fake, fake, 1, 2, 8, 8, 16, 3, 2, 0)
    with pytest.raises(EatError, match="multiple of the vector width"):
        L.bn_bwd_apply(fake, 0, 0, fake, fake, fake, fake, fake, 1, fake, fake, fake, 0, 2, 16, 10, 0)
    with pytest.raises(EatError, match="multiple of the vector width"):
        L.bn_act_pool(fake, fake, fake, 1, fake, 1.0, 0, 2, 16, 10, 0)
    # empty batches are a no-op, not an error
    L.se_bn_bwd_reduce(fake, fake, fake, fake, fake, 1, fake, fake, 3, 0, 0, 16, 16, 0)
    L.se_bn_bwd_combine(fake, 3, fake, fake, fake, 0, 16, fake, fake, 0)
    L.dw_conv_dgrad_bnred(fake, fake, 0, fake, fake, fake, fake, fake, fake, 1, fake, fake, 0, 0, 8, 8, 16, 3, 2, 0)
