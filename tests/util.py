"""Shared helpers for the test-suite: model/state/input construction identical to tests/golden/make_golden.py."""
import contextlib
import io
import os

import numpy as np
import torch

from efficientat_b200.synth import set_bn_stats, synth_labels, synth_state_, synth_waveform

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
NETS = {"mn10": ("mn", 1.0, 64000, 2), "mn04": ("mn", 0.4, 32000, 2), "mn20": ("mn", 2.0, 32000, 1),
        "dymn10": ("dymn", 1.0, 64000, 2), "dymn04": ("dymn", 0.4, 32000, 2),
        # the benchmarked shape (10 s clips = 1000 frames) and the widths BASELINE.json's configs C4 / C5 name
        "mn10_10s": ("mn", 1.0, 320000, 2), "dymn20_10s": ("dymn", 2.0, 320000, 2), "dymn20": ("dymn", 2.0, 64000, 2),
        "mn40_10s": ("mn", 4.0, 320000, 1)}


# resolved once, at import: tests that change the working directory (tests/test_gpu_zz_f4.py) must keep writing to the same file
_REPORT = os.path.abspath(os.environ["EAT_TEST_REPORT"]) if os.environ.get("EAT_TEST_REPORT") else None


def report(line):
    """parity figures the tests measure: printed, and appended to $EAT_TEST_REPORT when set"""
    print(line)
    if _REPORT:
        try:
            with open(_REPORT, "a") as f:
                f.write(line + "\n")
        except OSError:
            pass                      # the report is a convenience; it must never fail a parity test


def golden(name):
    return np.load(os.path.join(GOLDEN, name + ".npz"), allow_pickle=False)


def build_model(tag, precision="fp32", seed=7):
    kind, width, _, _ = NETS[tag]
    if kind == "mn":
        from efficientat_b200.models.mn.model import get_model
    else:
        from efficientat_b200.models.dymn.model import get_model
    torch.manual_seed(0)
    m = get_model(width_mult=width, precision=precision, verbose=False)
    synth_state_(m, seed=seed)
    g = golden(tag)
    return set_bn_stats(m, g["cal_rm"], g["cal_rv"])       # calibrated BN buffers (see make_golden.py)


def net_inputs(tag):
    """-> (spec [B,1,128,T] fp32 CPU, labels [B,527]) exactly as tests/golden/make_golden.py builds them."""
    _, _, n, b = NETS[tag]
    frames = 1 + (n - 1) // 320
    spec = synth_waveform(b, 128 * frames, seed=21, std=0.7).view(b, 1, 128, frames)
    return spec, synth_labels(b, 527, seed=5)


def fmap_digest(fmaps):
    out = []
    for f in fmaps:
        flat = f.flatten()
        idx = torch.linspace(0, flat.numel() - 1, 8).long()
        out.append(torch.cat([f.mean().view(1), f.abs().max().view(1), flat[idx]]))
    return torch.stack(out).numpy()


def topk_match(got, want, k=10, tie_tol=0.0):
    """Top-k label indices must agree rank by rank; a swap is tolerated only between classes whose
    *reference* logits differ by less than tie_tol (a near-tie no finite-precision path can order)."""
    got, want = np.asarray(got), np.asarray(want)
    for b in range(want.shape[0]):
        gi, wi = np.argsort(-got[b])[:k], np.argsort(-want[b])[:k]
        for r in range(k):
            if gi[r] != wi[r] and abs(want[b, gi[r]] - want[b, wi[r]]) > tie_tol:
                return False
    return True


def bn_variance_check(out, stats, ref, n, C, eps, what, factor=2):
    """var + eps from eat_bn_finalize of the kernel's sums vs torch.var_mean (fp32) of the same output, both through an
    fp32 invstd, against fp64"""
    from efficientat_b200._lib import lib
    L = lib()
    gamma, beta = torch.ones(C, device="cuda"), torch.zeros(C, device="cuda")
    bn = torch.full((4, C), float("nan"), device="cuda")
    L.bn_finalize(stats[0].contiguous().data_ptr(), stats[1].contiguous().data_ptr(), float(n), gamma.data_ptr(),
                  beta.data_ptr(), eps, 0.01, 0, 0, 0, bn[0].data_ptr(), bn[1].data_ptr(), bn[2].data_ptr(),
                  bn[3].data_ptr(), C, torch.cuda.current_stream().cuda_stream)
    mean64 = ref[0] / n
    ve64 = ref[1] / n - mean64 * mean64 + eps
    var_t, _ = torch.var_mean(out.reshape(-1, C), dim=0, unbiased=False)
    ve_t = 1.0 / torch.rsqrt(var_t + eps).double() ** 2
    ve_k = 1.0 / bn[3].double() ** 2
    e_k = ((ve_k - ve64).abs() / ve64).max().item()
    e_t = ((ve_t - ve64).abs() / ve64).max().item()
    ratio = (mean64.abs() / (ve64 - eps).clamp_min(1e-30).sqrt()).max().item()
    report(f"[kernel] {what}: var + eps rel err kernel {e_k:.2e}, torch fp32 {e_t:.2e}, ratio {e_k / e_t:.2f} (bound {factor}; "
           f"mean/std up to {ratio:.0f})")
    assert e_k <= factor * e_t, f"{what}: variance {e_k:.3e} relative vs torch fp32 {e_t:.3e}"
