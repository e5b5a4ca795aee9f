"""CPU tests of the mel front end at every supported n_fft (256 ... 4096):

* the mixed-radix Stockham FFT of csrc/fft_core.cuh (radix-8 passes, then the radix-2/4 tail) at every complex length
  M = n_fft / 2, compiled as plain C++ and driven by a harness that emulates mel_kernel's gather / barrier / scatter
  rounds (M/8 work items of 8 values each), real-FFT split included, against numpy.fft.rfft of length n_fft;
* eat_mel_fwd's argument validation, which happens on the host before any device call, so fake pointers are safe."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZES = (256, 512, 1024, 2048, 4096)
HARNESS = r"""
#include <cstdio>
#include <cstdlib>
#include <cmath>
#include <vector>
#include "fft_core.cuh"
int main(int argc, char** argv) {
  const int M = atoi(argv[1]), G = M / 8;
  int log2m = 0;
  while ((1 << log2m) < M) ++log2m;
  std::vector<float> x(2 * M);
  for (int i = 0; i < 2 * M; ++i) if (scanf("%f", &x[i]) != 1) return 1;
  std::vector<float2> tw(2 * M), z(M);
  for (int m = 0; m < M; ++m) {
    tw[m] = make_float2((float)cos(2 * M_PI * m / M), (float)-sin(2 * M_PI * m / M));
    tw[M + m] = make_float2((float)cos(2 * M_PI * m / (2 * M)), (float)-sin(2 * M_PI * m / (2 * M)));
  }
  for (int n = 0; n < M; ++n) z[n] = make_float2(x[2 * n], x[2 * n + 1]);
  // radix-8 passes: every work item gathers, then (barrier) every work item scatters
  int Ns = 1;
  for (int pass = 0; pass < log2m / 3; ++pass, Ns *= 8) {
    std::vector<float2> out(M);
    for (int j = 0; j < G; ++j) {
      float2 v[8];
      for (int r = 0; r < 8; ++r) v[r] = z[j + G * r];
      stockham8_compute_m(v, j, Ns, M, tw.data());
      for (int r = 0; r < 8; ++r) out[stockham8_dst(j, Ns, r)] = v[r];
    }
    z = out;
  }
  // tail: in place, each thread writes back the slots it read
  if (log2m % 3) {
    for (int j = 0; j < G; ++j) {
      float2 v[8];
      for (int r = 0; r < 8; ++r) v[r] = z[j + G * r];
      if (log2m % 3 == 1) stockham2_tail(v, j, M, tw.data());
      else stockham4_tail(v, j, M, tw.data());
      for (int r = 0; r < 8; ++r) z[j + G * r] = v[r];
    }
  }
  for (int k = 0; k <= M; ++k) {
    float2 X = (k < M) ? rfft_split(z[k], z[(M - k) & (M - 1)], tw[M + k]) : make_float2(z[0].x - z[0].y, 0.f);
    printf("%.9g %.9g\n", X.x, X.y);
  }
  return 0;
}
"""


@pytest.fixture(scope="module")
def harness():
    with tempfile.TemporaryDirectory() as d:
        src = os.path.join(d, "h.cpp")
        with open(src, "w") as fh:
            fh.write(HARNESS)
        exe = os.path.join(d, "h")
        subprocess.run(["g++", "-O2", "-x", "c++", "-I", os.path.join(ROOT, "efficientat_b200", "csrc"), src, "-o", exe],
                       check=True)
        yield exe


@pytest.mark.parametrize("n_fft", SIZES)
def test_mixed_radix_stockham_rfft_matches_numpy(harness, n_fft):
    rng = np.random.default_rng(n_fft)
    for trial in range(3):
        x = rng.standard_normal(n_fft).astype(np.float32)
        if trial == 2:
            x[: n_fft // 3] = 0.0                # a window-like zero run: exercises every twiddle on sparse input
        out = subprocess.run([harness, str(n_fft // 2)], input=" ".join(f"{v:.9g}" for v in x), capture_output=True,
                             text=True, check=True).stdout
        got = np.array([[float(a) for a in line.split()] for line in out.strip().splitlines()])
        assert got.shape == (n_fft // 2 + 1, 2)
        ref = np.fft.rfft(x.astype(np.float64))
        err = np.abs(got[:, 0] + 1j * got[:, 1] - ref).max()
        # fp32 FFT round-off grows like log2(n_fft); 2e-4 of the peak is the bound test_fft_core.py uses at 1024
        assert err < 2e-4 * np.abs(ref).max(), (n_fft, trial, err)


def _mel_fwd(n_fft, win_length=None, hop=160, n_mels=64, N=32000, B=2):
    from efficientat_b200._lib import lib
    fake = 4096                                                  # never dereferenced: validation comes first
    win_length = n_fft if win_length is None else win_length
    lib().mel_fwd(fake, B, N, fake, win_length, hop, n_fft, fake, fake, fake, fake, 8, n_mels, 0.97, fake, 0)


def _code(fn):
    from efficientat_b200._lib import EatError
    with pytest.raises(EatError) as ei:
        fn()
    return str(ei.value)


@pytest.mark.parametrize("n_fft", [400, 800, 8192, 128, 1000, 0, -1024])
def test_mel_fwd_rejects_unsupported_n_fft(n_fft):
    msg = _code(lambda: _mel_fwd(n_fft, win_length=max(1, min(n_fft, 100))))
    assert "code 3" in msg and "256, 512, 1024, 2048, 4096" in msg, msg


@pytest.mark.parametrize("n_fft", SIZES)
def test_mel_fwd_geometry_errors(n_fft):
    assert "code 1" in _code(lambda: _mel_fwd(n_fft, win_length=n_fft + 1))          # window longer than the frame
    assert "code 1" in _code(lambda: _mel_fwd(n_fft, hop=0))
    assert "code 1" in _code(lambda: _mel_fwd(n_fft, n_mels=513))
    assert "code 1" in _code(lambda: _mel_fwd(n_fft, N=n_fft // 2 + 1))                # N - 1 = n_fft/2: too short
    # a hop whose signal slice cannot fit in shared memory
    msg = _code(lambda: _mel_fwd(n_fft, hop=1 << 20, N=1 << 22))
    assert "code 3" in msg and "shared-memory" in msg, msg


def test_mel_fwd_empty_batch_is_a_no_op():
    for n_fft in SIZES:
        _mel_fwd(n_fft, B=0)
