// Fused log-mel front end: pre-emphasis + reflect pad + framing + window + n_fft-point real FFT in
// shared memory + power + banded mel filterbank + log + affine.   One kernel, waveform in,
// normalised log-mel out.  Replaces reference models/preprocess.py:40-67 (eval path; the
// fmin/fmax jitter of the training path only changes the filterbank table passed in).
//
// n_fft is a power of two in [256, 4096]; mel_kernel<M> is instantiated per complex FFT length M = n_fft / 2.
// Work decomposition: grid = (ceil(T / F), B).  A CTA owns F consecutive frames of one clip: it stages its slice of the
// pre-emphasised, reflect-padded signal in shared memory once (the frames overlap by n_fft - hop samples), then its
// 256 threads, as independent groups of M/8 (group-local barriers), transform one frame per group and round: M-point
// complex FFT as floor(log8 M) radix-8 Stockham passes plus one radix-2/4 pass when log2 M is not a multiple of 3,
// 8 complex values per thread in registers.
//
//   n_fft   M     passes    threads/group  groups  F (frames/CTA)  rounds
//   256     128   8·8·2     16             16      16              1
//   512     256   8·8·4     32             8       16              2
//   1024    512   8·8·8     64             4       16              4
//   2048    1024  8·8·8·2   128            2       16              8
//   4096    2048  8·8·8·4   256            1       8               8
//
// Results are staged in shared memory as [n_mels][F] so the global store is 4·F bytes per mel row.
// Algorithmic HBM bytes: 4*N read + 4*n_mels*T written per clip (1.792 MB at 10 s / 32 kHz / hop 320 / 128 mels).
#include "common.cuh"
#include "fft_core.cuh"
#include <math.h>

#include <algorithm>
#include <cstdio>

namespace {

constexpr int kThreads = 256;
constexpr size_t kSmemCap = 227 * 1024;     // opt-in shared memory per block on sm_90

template <int M>
struct MelShape {
  static_assert(M >= 128 && M <= 2048 && (M & (M - 1)) == 0, "complex FFT length: a power of two in [128, 2048]");
  static constexpr int kNfft = 2 * M;
  static constexpr int kGroupThreads = M / 8;                     // one radix-8 work item per thread
  static constexpr int kGroups = kThreads / kGroupThreads;
  static constexpr int kFrames = M == 2048 ? 8 : 16;             // frames per CTA; 8 at n_fft 4096 keeps long hops
                                                                  // within shared memory next to the 48 KB of tables
  static constexpr int kPow = M + 4;                              // power bins 0..M, padded to 16 B
  static constexpr int kLog2 = M == 128 ? 7 : M == 256 ? 8 : M == 512 ? 9 : M == 1024 ? 10 : 11;
  static constexpr int kLog2Group = kLog2 - 3;
  static constexpr int kRadix8End = kLog2 >= 9 ? 512 : 64;        // radix-8 passes run at Ns = 1, 8 (, 64)
  static constexpr int kTail = kLog2 % 3 == 0 ? 1 : kLog2 % 3 == 1 ? 2 : 4;   // radix of the last pass, 1 = none
  static_assert(kFrames % kGroups == 0, "whole rounds");
  // bytes that do not depend on the geometry: twiddles, window, per-group FFT and power buffers
  static constexpr size_t kSmemFixed = kNfft * sizeof(float2) + kNfft * sizeof(float) +
                                       kGroups * (M * sizeof(float2) + kPow * sizeof(float));
};

struct MelParams {
  const float* wave;     // [B, N]
  const float* window;   // [win_length]
  const float2* twiddle; // [M] exp(-2 pi i m/M) followed by [M] exp(-2 pi i k/n_fft), M = n_fft / 2
  const int* fb_start;   // [n_mels] first FFT bin of each filter
  const int* fb_len;     // [n_mels] number of taps
  const float* fb_w;     // [max_len][n_mels] taps, tap-major
  float* out;            // [B, n_mels, T]
  int B, N, T, n_mels, win_length, hop, max_len;
  int seg_len;           // samples of the pre-emphasised, reflect-padded signal a CTA stages: (frames - 1) * hop + n_fft
  float preemph;         // 0.97
  float log_offset;      // 1e-5
  float out_add, out_div;   // (v + 4.5) / 5
  const int* n_valid;    // [B] each clip's sample count (eat_mel_fwd_len), or null
};

// sample s of the pre-emphasised signal p (length L = N-1) extended by reflection (torch.stft center=True);
// positions only frames beyond T would touch (double reflection) read as 0
__device__ __forceinline__ float preemph_sample(const float* __restrict__ x, int s, int L, float c) {
  int q = s < 0 ? -s : s;
  if (q >= L) q = 2 * (L - 1) - q;
  if (q < 0 || q >= L) return 0.f;
  return __ldg(x + q + 1) - c * __ldg(x + q);
}

// the groups of a CTA work on different frames: no CTA barrier.  bar.sync takes thread counts that are multiples
// of 32 and a CTA has 16 barrier ids, so groups of one warp (n_fft 512) or half a warp (n_fft 256) use __syncwarp
template <int G>
__device__ __forceinline__ void group_sync(int grp) {
  static_assert(G == 16 || G % 32 == 0, "group size");
  if constexpr (G >= 64) {
    asm volatile("bar.sync %0, %1;" ::"r"(grp + 1), "n"(G) : "memory");
  } else if constexpr (G == 32) {
    __syncwarp();
  } else {
    __syncwarp(0xffffu << (16 * (grp & 1)));
  }
}

// kLen: clip b is the first n_valid[b] samples of its row; its frames end at 1 + (n_valid[b] - 1) / hop, past which the
// output is 0, and pre-emphasis and reflection use its own last sample
template <int M, bool kLen = false>
__global__ void __launch_bounds__(kThreads) mel_kernel(MelParams p) {
  using S = MelShape<M>;
  constexpr int G = S::kGroupThreads, F = S::kFrames, NF = S::kNfft;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float2* s_tw = reinterpret_cast<float2*>(smem_raw);                 // n_fft float2
  float* s_win = reinterpret_cast<float*>(s_tw + NF);                 // n_fft floats, zero-padded window
  float2* s_fft = reinterpret_cast<float2*>(s_win + NF);              // kGroups * M float2
  float* s_pow = reinterpret_cast<float*>(s_fft + S::kGroups * M);    // kGroups * (M + 4) floats
  float* s_out = s_pow + S::kGroups * S::kPow;                        // n_mels * (F + 1) floats
  float* s_sig = s_out + p.n_mels * (F + 1);                          // seg_len floats: the CTA's slice of the signal

  const int tid = threadIdx.x;
  const int grp = tid >> S::kLog2Group;
  const int j = tid & (G - 1);
  const int b = blockIdx.y;
  const int t_base = blockIdx.x * F;
  const float* __restrict__ x = p.wave + (size_t)b * p.N;
  const int L = kLen ? p.n_valid[b] - 1 : p.N - 1;
  const int Tb = kLen ? 1 + L / p.hop : p.T;
  if constexpr (kLen) {
    if (t_base >= Tb) {                 // the whole tile lies past the clip's frames: zeros only, nothing staged or read
      for (int i = tid; i < p.n_mels * F; i += kThreads) {
        const int m = i / F, t = t_base + i % F;
        if (t < p.T) p.out[((size_t)b * p.n_mels + m) * p.T + t] = 0.f;
      }
      return;
    }
  }
  const int lp = (NF - p.win_length) / 2;

  for (int i = tid; i < NF; i += kThreads) {
    s_tw[i] = p.twiddle[i];
    int wi = i - lp;
    s_win[i] = (wi >= 0 && wi < p.win_length) ? p.window[wi] : 0.f;
  }
  // pre-emphasis + reflection once per sample (coalesced), instead of 32 scalar global loads per thread and frame:
  // neighbouring frames overlap by n_fft - hop samples
  {
    const int s0 = t_base * p.hop - M;
    for (int i = tid; i < p.seg_len; i += kThreads) s_sig[i] = preemph_sample(x, s0 + i, L, p.preemph);
  }
  __syncthreads();

  float2* zf = s_fft + grp * M;
  float* pw = s_pow + grp * S::kPow;

  for (int round = 0; round < F / S::kGroups; ++round) {
    const int fl = round * S::kGroups + grp;   // frame index inside the CTA tile
    const int t = t_base + fl;
    const bool live = t < Tb;                  // uniform within a group
    float2 v[8];
    // ---- pass 1 (Ns = 1): window the staged samples
    if (live) {
      const float* sg = s_sig + fl * p.hop;
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        const int n = j + G * r;
        v[r] = make_float2(s_win[2 * n] * sg[2 * n], s_win[2 * n + 1] * sg[2 * n + 1]);
      }
      stockham8_compute_m(v, j, 1, M, s_tw);
#pragma unroll
      for (int r = 0; r < 8; ++r) zf[stockham8_dst(j, 1, r)] = v[r];
    }
    group_sync<G>(grp);
    // ---- the other radix-8 passes (Ns = 8 (, 64)), in place with a barrier between gather and scatter
#pragma unroll
    for (int Ns = 8; Ns < S::kRadix8End; Ns *= 8) {
      if (live) {
#pragma unroll
        for (int r = 0; r < 8; ++r) v[r] = zf[j + G * r];
        stockham8_compute_m(v, j, Ns, M, s_tw);
      }
      group_sync<G>(grp);
      if (live) {
#pragma unroll
        for (int r = 0; r < 8; ++r) zf[stockham8_dst(j, Ns, r)] = v[r];
      }
      group_sync<G>(grp);
    }
    // ---- radix-2 / radix-4 tail: every thread writes back exactly the slots it read
    if constexpr (S::kTail != 1) {
      if (live) {
#pragma unroll
        for (int r = 0; r < 8; ++r) v[r] = zf[j + G * r];
        if constexpr (S::kTail == 2) stockham2_tail(v, j, M, s_tw);
        else stockham4_tail(v, j, M, s_tw);
#pragma unroll
        for (int r = 0; r < 8; ++r) zf[j + G * r] = v[r];
      }
      group_sync<G>(grp);
    }
    // ---- real-FFT split + power spectrum, bins 0..M
    if (live) {
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        int k = j + G * r;
        float2 X = rfft_split(zf[k], zf[(M - k) & (M - 1)], s_tw[M + k]);
        pw[k] = X.x * X.x + X.y * X.y;
      }
      if (j == 0) { float2 z0 = zf[0]; float nyq = z0.x - z0.y; pw[M] = nyq * nyq; }
    }
    group_sync<G>(grp);
    // ---- banded mel + log + affine into the staging tile
    if (live) {
      for (int m = j; m < p.n_mels; m += G) {
        int st = __ldg(p.fb_start + m), len = __ldg(p.fb_len + m);
        float acc = 0.f;
        for (int i = 0; i < len; ++i) acc = fmaf(__ldg(p.fb_w + (size_t)i * p.n_mels + m), pw[st + i], acc);
        s_out[m * (F + 1) + fl] = (logf(acc + p.log_offset) + p.out_add) / p.out_div;
      }
    }
    group_sync<G>(grp);                         // zf / pw are rewritten by this group's next round
  }
  __syncthreads();
  // ---- store: F consecutive frames (4·F bytes) of one mel row per F lanes, 32 / F mel rows per warp instruction
  const int lane = tid & 31, warp = tid >> 5;
  const int fo = lane & (F - 1), sub = lane / F;
  const int t = t_base + fo;
  for (int m = warp * (32 / F) + sub; m < p.n_mels; m += (kThreads / 32) * (32 / F)) {
    if constexpr (kLen) {
      if (t < p.T) p.out[((size_t)b * p.n_mels + m) * p.T + t] = t < Tb ? s_out[m * (F + 1) + fo] : 0.f;
    } else {
      if (t < p.T) p.out[((size_t)b * p.n_mels + m) * p.T + t] = s_out[m * (F + 1) + fo];
    }
  }
}


template <int M>
int mel_launch(MelParams p, cudaStream_t stream) {
  using S = MelShape<M>;
  const long long seg_len = (long long)(S::kFrames - 1) * p.hop + S::kNfft;
  const size_t smem = S::kSmemFixed + ((size_t)p.n_mels * (S::kFrames + 1) + (size_t)seg_len) * sizeof(float);
  if (smem > kSmemCap) {
    eat_set_error("eat_mel_fwd: hop too large for the shared-memory signal slice"); return EAT_ERR_UNSUPPORTED;
  }
  p.seg_len = (int)seg_len;
  dim3 grid(ceil_div(p.T, S::kFrames), p.B);
  if (p.n_valid == nullptr) {
    static unsigned long long attr_mask = 0;
    if (int rc = eat_opt_in_smem(mel_kernel<M>, kSmemCap, attr_mask)) return rc;
    mel_kernel<M><<<grid, kThreads, smem, stream>>>(p);
  } else {
    static unsigned long long attr_mask_len = 0;
    if (int rc = eat_opt_in_smem(mel_kernel<M, true>, kSmemCap, attr_mask_len)) return rc;
    mel_kernel<M, true><<<grid, kThreads, smem, stream>>>(p);
  }
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

// ---- backward: dspec [B, n_mels, T] -> dwave [B, N], the adjoint of mel_kernel (masks, affine, log, filterbank, power,
// real FFT, window, overlap-add, reflect padding, pre-emphasis).  The frame spectra are recomputed, not stored.
//
// mel_bwd_kernel<M>: the forward's tiling (F frames of one clip per CTA, groups of M/8 threads per frame).  Per frame:
// the forward FFT gives X[k], k = 0..M, and the mel energies; dmel = dspec / (5 (mel + 1e-5)) (0 where masked);
// dpow[k] = sum_m fb[m, k] dmel[m], gathered per bin over the filters that cover it (s_first / s_last), so no bin is
// written twice; dframe[i] = sum_k 2 dpow[k] Re(X[k] e^{+2 pi i k i / n_fft}) over the one-sided spectrum, which is the
// unnormalised inverse real DFT of the Hermitian spectrum Z[k] = dpow[k] X[k] (k = 1..M-1), Z[0] = 2 dpow[0] X[0],
// Z[M] = 2 dpow[M] X[M].  It runs as the same M-point complex FFT (fft_core.cuh) on conj(A + iB) with
// A[k] = Z[k] + conj(Z[M-k]), B[k] = (Z[k] - conj(Z[M-k])) e^{+2 pi i k / n_fft}: the conjugated result holds the even
// samples in its real and the odd samples in its imaginary parts.  The windowed frame gradients of a round are added
// into the CTA's slice of the padded-signal gradient in group order (one CTA barrier per round), and the slice is
// written to `work` [B][CTAs][seg_len].  mel_bwd_gather_kernel sums, for every waveform sample, the slices that overlap
// each padded position that reads it (reflect padding folded back) in a fixed order and applies the pre-emphasis'
// adjoint.  No floating-point atomics: the result is bitwise repeatable.
struct MelBwdParams {
  const float* dspec;    // [B, n_mels, T]
  const float* wave;     // [B, N]
  const float* window;
  const float2* twiddle;
  const int* fb_start;
  const int* fb_len;
  const float* fb_w;
  const int *fs, *fe, *ts, *te;   // [B] SpecAugment bands of the forward, or all null
  float* work;           // [B, ceil(T / F), seg_len]
  int B, N, T, n_mels, win_length, hop, seg_len;
  float preemph, log_offset, out_div;
};

template <int M>
__global__ void __launch_bounds__(kThreads) mel_bwd_kernel(MelBwdParams p) {
  using S = MelShape<M>;
  constexpr int G = S::kGroupThreads, F = S::kFrames, NF = S::kNfft, NG = S::kGroups;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float2* s_tw = reinterpret_cast<float2*>(smem_raw);                 // n_fft float2
  float2* s_fft = s_tw + NF;                                          // NG * M float2
  float2* s_X = s_fft + NG * M;                                       // NG * (M + 4) float2: X[k], then Z[k]
  float* s_win = reinterpret_cast<float*>(s_X + NG * (M + 4));        // n_fft floats, zero-padded window
  float* s_pow = s_win + NF;                                          // NG * (M + 4) floats: power, then dpow
  int* s_first = reinterpret_cast<int*>(s_pow + NG * S::kPow);        // M + 4: first / last filter covering bin k
  int* s_last = s_first + (M + 4);
  float* s_g = reinterpret_cast<float*>(s_last + (M + 4));            // n_mels * (F + 1): dspec tile, then dmel
  float* s_acc = s_g + p.n_mels * (F + 1);                            // seg_len: gradient of the padded signal slice

  const int tid = threadIdx.x;
  const int grp = tid >> S::kLog2Group;
  const int j = tid & (G - 1);
  const int b = blockIdx.y;
  const int t_base = blockIdx.x * F;
  const float* __restrict__ x = p.wave + (size_t)b * p.N;
  const int L = p.N - 1;
  const int lp = (NF - p.win_length) / 2;

  for (int i = tid; i < NF; i += kThreads) {
    s_tw[i] = p.twiddle[i];
    int wi = i - lp;
    s_win[i] = (wi >= 0 && wi < p.win_length) ? p.window[wi] : 0.f;
  }
  for (int k = tid; k <= M; k += kThreads) { s_first[k] = p.n_mels; s_last[k] = -1; }
  for (int i = tid; i < p.seg_len; i += kThreads) s_acc[i] = 0.f;
  for (int i = tid; i < p.n_mels * F; i += kThreads) {
    const int m = i / F, fo = i % F, t = t_base + fo;
    float g = 0.f;
    if (t < p.T) {
      const bool masked = p.fs != nullptr && ((m >= p.fs[b] && m < p.fe[b]) || (t >= p.ts[b] && t < p.te[b]));
      g = masked ? 0.f : p.dspec[((size_t)b * p.n_mels + m) * p.T + t];
    }
    s_g[m * (F + 1) + fo] = g;
  }
  __syncthreads();
  for (int m = tid; m < p.n_mels; m += kThreads) {
    const int st = __ldg(p.fb_start + m), len = __ldg(p.fb_len + m);
    for (int i = 0; i < len; ++i) { atomicMin(s_first + st + i, m); atomicMax(s_last + st + i, m); }
  }
  __syncthreads();

  float2* zf = s_fft + grp * M;
  float2* zx = s_X + grp * (M + 4);
  float* pw = s_pow + grp * S::kPow;

  for (int round = 0; round < F / NG; ++round) {
    const int fl = round * NG + grp;
    const int t = t_base + fl;
    const bool live = t < p.T;                 // uniform within a group
    float2 v[8];
    // ---- recompute the frame's spectrum: the forward's passes
    if (live) {
      const int s0 = t * p.hop - M;
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        const int n = j + G * r;
        v[r] = make_float2(s_win[2 * n] * preemph_sample(x, s0 + 2 * n, L, p.preemph),
                           s_win[2 * n + 1] * preemph_sample(x, s0 + 2 * n + 1, L, p.preemph));
      }
    }
#pragma unroll
    for (int pass = 0; pass < 2; ++pass) {
      // pass 0: forward FFT of the windowed frame; pass 1: the inverse of the spectrum gradient (v = conj(A + iB))
      if (live) {
        stockham8_compute_m(v, j, 1, M, s_tw);
#pragma unroll
        for (int r = 0; r < 8; ++r) zf[stockham8_dst(j, 1, r)] = v[r];
      }
      group_sync<G>(grp);
#pragma unroll
      for (int Ns = 8; Ns < S::kRadix8End; Ns *= 8) {
        if (live) {
#pragma unroll
          for (int r = 0; r < 8; ++r) v[r] = zf[j + G * r];
          stockham8_compute_m(v, j, Ns, M, s_tw);
        }
        group_sync<G>(grp);
        if (live) {
#pragma unroll
          for (int r = 0; r < 8; ++r) zf[stockham8_dst(j, Ns, r)] = v[r];
        }
        group_sync<G>(grp);
      }
      if constexpr (S::kTail != 1) {
        if (live) {
#pragma unroll
          for (int r = 0; r < 8; ++r) v[r] = zf[j + G * r];
          if constexpr (S::kTail == 2) stockham2_tail(v, j, M, s_tw);
          else stockham4_tail(v, j, M, s_tw);
#pragma unroll
          for (int r = 0; r < 8; ++r) zf[j + G * r] = v[r];
        }
        group_sync<G>(grp);
      }
      if (pass == 1) break;
      // ---- spectrum and power, bins 0..M
      if (live) {
#pragma unroll
        for (int r = 0; r < 8; ++r) {
          const int k = j + G * r;
          const float2 X = rfft_split(zf[k], zf[(M - k) & (M - 1)], s_tw[M + k]);
          zx[k] = X;
          pw[k] = X.x * X.x + X.y * X.y;
        }
        if (j == 0) { const float2 z0 = zf[0]; const float nyq = z0.x - z0.y; zx[M] = make_float2(nyq, 0.f); pw[M] = nyq * nyq; }
      }
      group_sync<G>(grp);
      // ---- mel energies as the forward computes them -> dmel, in place of the dspec tile
      if (live) {
        for (int m = j; m < p.n_mels; m += G) {
          const int st = __ldg(p.fb_start + m), len = __ldg(p.fb_len + m);
          float acc = 0.f;
          for (int i = 0; i < len; ++i) acc = fmaf(__ldg(p.fb_w + (size_t)i * p.n_mels + m), pw[st + i], acc);
          s_g[m * (F + 1) + fl] /= p.out_div * (acc + p.log_offset);
        }
      }
      group_sync<G>(grp);
      // ---- dpow per bin (transposed filterbank), Z[k] = dpow[k] X[k] (twice at k = 0 and M)
      if (live) {
        for (int k = j; k <= M; k += G) {
          float d = 0.f;
          for (int m = s_first[k]; m <= s_last[k]; ++m) {
            const int i = k - __ldg(p.fb_start + m);
            if (i >= 0 && i < __ldg(p.fb_len + m)) d = fmaf(__ldg(p.fb_w + (size_t)i * p.n_mels + m), s_g[m * (F + 1) + fl], d);
          }
          if (k == 0 || k == M) d *= 2.f;
          zx[k] = make_float2(zx[k].x * d, zx[k].y * d);
        }
      }
      group_sync<G>(grp);
      if (live) {
#pragma unroll
        for (int r = 0; r < 8; ++r) {
          const int k = j + G * r;
          const float2 zk = zx[k], zm = zx[M - k];
          const float2 a = make_float2(zk.x + zm.x, zk.y - zm.y);
          const float2 w = make_float2(s_tw[M + k].x, -s_tw[M + k].y);       // e^{+2 pi i k / n_fft}
          const float2 bb = cmul(make_float2(zk.x - zm.x, zk.y + zm.y), w);
          v[r] = make_float2(a.x - bb.y, -(a.y + bb.x));                     // conj(A + iB)
        }
      }
      group_sync<G>(grp);                       // zf is rewritten by the inverse's first pass
    }
    // ---- windowed frame gradient, in place: float2 n of zf becomes floats 2n, 2n+1
    if (live) {
      float* df = reinterpret_cast<float*>(zf);
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        const int n = j + G * r;
        const float2 c = zf[n];
        df[2 * n] = s_win[2 * n] * c.x;
        df[2 * n + 1] = -s_win[2 * n + 1] * c.y;
      }
    }
    __syncthreads();
    // ---- overlap-add of the round's frames into the slice, in group order
    for (int i = tid; i < p.seg_len; i += kThreads) {
      float a = s_acc[i];
#pragma unroll
      for (int g = 0; g < NG; ++g) {
        const int f2 = round * NG + g, o = i - f2 * p.hop;
        if (t_base + f2 < p.T && o >= 0 && o < NF) a += reinterpret_cast<const float*>(s_fft + g * M)[o];
      }
      s_acc[i] = a;
    }
    __syncthreads();
  }
  float* out = p.work + ((size_t)b * gridDim.x + blockIdx.x) * p.seg_len;
  for (int i = tid; i < p.seg_len; i += kThreads) out[i] = s_acc[i];
}

// dwave[b, n] = gp[n-1] - preemph * gp[n] (pre-emphasis p[q] = x[q+1] - c x[q], q < L = N-1), where gp[q] sums the
// padded-signal gradient over the positions s in [-M, (T-1) hop + M) that read p[q] (s = q, -q, 2(L-1) - q), each
// the sum of the CTA slices covering it, in slice order
__global__ void mel_bwd_gather_kernel(const float* __restrict__ work, float* __restrict__ dwave, int B, int N, int T,
                                      int hop, int M, int frames, int seg_len, int ctas, float preemph) {
  const long long n_all = (long long)B * N;
  const int L = N - 1, span = frames * hop, s_end = (T - 1) * hop + M;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < n_all; idx += (long long)gridDim.x * blockDim.x) {
    const int b = (int)(idx / N), n = (int)(idx % N);
    const float* wb = work + (size_t)b * ctas * seg_len;
    auto at = [&](int s) {                      // gradient of padded position s
      float a = 0.f;
      if (s < -M || s >= s_end) return a;
      const int u = s + M;
      const int c_hi = min(ctas - 1, u / span), c_lo = u >= seg_len ? (u - seg_len) / span + 1 : 0;
      for (int c = c_lo; c <= c_hi; ++c) a += __ldg(wb + (size_t)c * seg_len + (u - c * span));
      return a;
    };
    auto gp = [&](int q) {
      float a = at(q);
      if (q > 0) a += at(-q);
      if (q < L - 1) a += at(2 * (L - 1) - q);
      return a;
    };
    float d = 0.f;
    if (n >= 1) d = gp(n - 1);
    if (n < L) d = fmaf(-preemph, gp(n), d);
    dwave[idx] = d;
  }
}

template <int M>
size_t mel_bwd_smem(int n_mels, int seg_len) {
  using S = MelShape<M>;
  return S::kNfft * (sizeof(float2) + sizeof(float)) +
         S::kGroups * (M * sizeof(float2) + (M + 4) * sizeof(float2) + S::kPow * sizeof(float)) +
         2 * (M + 4) * sizeof(int) + ((size_t)n_mels * (S::kFrames + 1) + (size_t)seg_len) * sizeof(float);
}

template <int M>
int mel_bwd_launch(MelBwdParams p, float* dwave, long long work_floats, cudaStream_t stream) {
  using S = MelShape<M>;
  const long long seg_len = (long long)(S::kFrames - 1) * p.hop + S::kNfft;
  const size_t smem = mel_bwd_smem<M>(p.n_mels, (int)std::min(seg_len, (long long)INT32_MAX));
  if (seg_len > INT32_MAX || smem > kSmemCap) {
    eat_set_error("eat_mel_bwd: hop too large for the shared-memory signal slice"); return EAT_ERR_UNSUPPORTED;
  }
  const int ctas = ceil_div(p.T, S::kFrames);
  if (work_floats < (long long)p.B * ctas * seg_len) { eat_set_error("eat_mel_bwd: work too small"); return EAT_ERR_ARG; }
  if (p.B == 0) return EAT_OK;
  p.seg_len = (int)seg_len;
  static unsigned long long attr_mask = 0;
  if (int rc = eat_opt_in_smem(mel_bwd_kernel<M>, kSmemCap, attr_mask)) return rc;
  mel_bwd_kernel<M><<<dim3(ctas, p.B), kThreads, smem, stream>>>(p);
  EAT_CHECK_LAUNCH();
  const long long n_all = (long long)p.B * p.N;
  const int grid = (int)std::min((long long)kNumSMs * 16, (n_all + 255) / 256);
  mel_bwd_gather_kernel<<<grid, 256, 0, stream>>>(p.work, dwave, p.B, p.N, p.T, p.hop, M, S::kFrames, p.seg_len, ctas,
                                                  p.preemph);
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

// training-time SpecAugment bands (torchaudio Frequency/TimeMasking, iid per example): positions inside
// [fs,fe) x all t or all f x [ts,te) are overwritten with `fill`.
__global__ void mel_mask_kernel(float* __restrict__ spec, int B, int F, int T, const int* __restrict__ fs,
                                const int* __restrict__ fe, const int* __restrict__ ts, const int* __restrict__ te,
                                float fill) {
  const long long n = (long long)B * F * T;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    int t = (int)(i % T), f = (int)((i / T) % F), b = (int)(i / ((long long)T * F));
    if ((f >= fs[b] && f < fe[b]) || (t >= ts[b] && t < te[b])) spec[i] = fill;
  }
}

// Kaldi triangular filterbank in banded form, built on the device (training: fmin/fmax change every call,
// reference models/preprocess.py:45-55 rebuilds it on the CPU and copies it over).  One thread per mel row;
// same fp32 op order as torchaudio.compliance.kaldi.get_mel_banks(vtln_warp = 1).
__global__ void mel_filterbank_kernel(int n_mels, int n_bins /* n_fft/2 */, float bin_width, float mel_lo, float delta,
                                      int* __restrict__ fb_start, int* __restrict__ fb_len, float* __restrict__ fb_w,
                                      int cap) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= n_mels) return;
  const float left = mel_lo + (float)m * delta;
  const float center = mel_lo + ((float)m + 1.0f) * delta;
  const float right = mel_lo + ((float)m + 2.0f) * delta;
  int first = -1, last = -1;
  for (int j = 0; j < n_bins; ++j) {
    const float mel = 1127.0f * logf(1.0f + bin_width * (float)j / 700.0f);
    const float w = fmaxf(0.f, fminf((mel - left) / (center - left), (right - mel) / (right - center)));
    if (w != 0.f) { if (first < 0) first = j; last = j; }
  }
  int len = first < 0 ? 0 : last - first + 1;
  if (len > cap) len = cap;
  fb_start[m] = first < 0 ? 0 : first;
  fb_len[m] = len;
  for (int i = 0; i < len; ++i) {
    const float mel = 1127.0f * logf(1.0f + bin_width * (float)(first + i) / 700.0f);
    fb_w[(size_t)i * n_mels + m] = fmaxf(0.f, fminf((mel - left) / (center - left), (right - mel) / (right - center)));
  }
}

}  // namespace

extern "C" int eat_mel_filterbank(int n_mels, int n_fft, float sample_rate, double fmin, double fmax, int* fb_start,
                                  int* fb_len, float* fb_w, int cap, cudaStream_t stream) {
  const double nyq = 0.5 * sample_rate;
  if (fmax <= 0.0) fmax += nyq;
  if (!(0.0 <= fmin && fmin < nyq && 0.0 < fmax && fmax <= nyq && fmin < fmax) || n_mels < 1 || cap < 1) {
    eat_set_error("eat_mel_filterbank: bad fmin/fmax"); return EAT_ERR_ARG;
  }
  const double mel_lo = 1127.0 * log(1.0 + fmin / 700.0), mel_hi = 1127.0 * log(1.0 + fmax / 700.0);
  const double delta = (mel_hi - mel_lo) / (n_mels + 1);
  mel_filterbank_kernel<<<(n_mels + 63) / 64, 64, 0, stream>>>(n_mels, n_fft / 2, sample_rate / n_fft, (float)mel_lo,
                                                              (float)delta, fb_start, fb_len, fb_w, cap);
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

extern "C" int eat_mel_mask(float* spec, int B, int F, int T, const int* f_start, const int* f_end,
                            const int* t_start, const int* t_end, float fill, cudaStream_t stream) {
  if (B == 0) return EAT_OK;
  long long n = (long long)B * F * T;
  int grid = (int)((n + 255) / 256 > kNumSMs * 16 ? kNumSMs * 16 : (n + 255) / 256);
  mel_mask_kernel<<<grid, 256, 0, stream>>>(spec, B, F, T, f_start, f_end, t_start, t_end, fill);
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

namespace {
// n_valid: null for eat_mel_fwd; the per-clip sample counts for eat_mel_fwd_len
int mel_fwd_impl(const float* wave, int B, int N, const float* window, int win_length, int hop, int n_fft,
                 const float* twiddle, const int* fb_start, const int* fb_len, const float* fb_w, int max_len, int n_mels,
                 float preemph, float* out, const int* n_valid, cudaStream_t stream) {
  if (n_fft != 256 && n_fft != 512 && n_fft != 1024 && n_fft != 2048 && n_fft != 4096) {
    eat_set_error("eat_mel_fwd: n_fft must be one of 256, 512, 1024, 2048, 4096"); return EAT_ERR_UNSUPPORTED;
  }
  if (win_length > n_fft || win_length < 1 || hop < 1 || n_mels < 1 || n_mels > 512 || B < 0) {
    eat_set_error("eat_mel_fwd: bad geometry"); return EAT_ERR_ARG;
  }
  if (N - 1 <= n_fft / 2) { eat_set_error("eat_mel_fwd: waveform too short for reflect padding"); return EAT_ERR_ARG; }
  if (B == 0) return EAT_OK;
  MelParams p;
  p.wave = wave; p.window = window; p.twiddle = reinterpret_cast<const float2*>(twiddle);
  p.fb_start = fb_start; p.fb_len = fb_len; p.fb_w = fb_w; p.out = out;
  p.B = B; p.N = N; p.T = 1 + (N - 1) / hop; p.n_mels = n_mels; p.win_length = win_length; p.hop = hop;
  p.max_len = max_len; p.preemph = preemph; p.log_offset = 1e-5f; p.out_add = 4.5f; p.out_div = 5.f;
  p.n_valid = n_valid;
  switch (n_fft) {
    case 256: return mel_launch<128>(p, stream);
    case 512: return mel_launch<256>(p, stream);
    case 1024: return mel_launch<512>(p, stream);
    case 2048: return mel_launch<1024>(p, stream);
    default: return mel_launch<2048>(p, stream);
  }
}
}  // namespace

extern "C" int eat_mel_fwd(const float* wave, int B, int N, const float* window, int win_length, int hop,
                           int n_fft, const float* twiddle, const int* fb_start, const int* fb_len,
                           const float* fb_w, int max_len, int n_mels, float preemph, float* out,
                           cudaStream_t stream) {
  return mel_fwd_impl(wave, B, N, window, win_length, hop, n_fft, twiddle, fb_start, fb_len, fb_w, max_len, n_mels,
                      preemph, out, nullptr, stream);
}

extern "C" int eat_mel_fwd_len(const float* wave, int B, int N, const float* window, int win_length, int hop,
                               int n_fft, const float* twiddle, const int* fb_start, const int* fb_len,
                               const float* fb_w, int max_len, int n_mels, float preemph, float* out, const int* n_valid,
                               cudaStream_t stream) {
  if (B > 0 && n_valid == nullptr) { eat_set_error("eat_mel_fwd_len: n_valid is required"); return EAT_ERR_ARG; }
  return mel_fwd_impl(wave, B, N, window, win_length, hop, n_fft, twiddle, fb_start, fb_len, fb_w, max_len, n_mels,
                      preemph, out, n_valid, stream);
}

namespace {
int mel_geometry_check(const char* who, int B, int N, int win_length, int hop, int n_fft, int n_mels) {
  char msg[160];
  int rc = EAT_OK;
  if (n_fft != 256 && n_fft != 512 && n_fft != 1024 && n_fft != 2048 && n_fft != 4096) {
    snprintf(msg, sizeof msg, "%s: n_fft must be one of 256, 512, 1024, 2048, 4096", who); rc = EAT_ERR_UNSUPPORTED;
  } else if (win_length > n_fft || win_length < 1 || hop < 1 || n_mels < 1 || n_mels > 512 || B < 0) {
    snprintf(msg, sizeof msg, "%s: bad geometry", who); rc = EAT_ERR_ARG;
  } else if (N - 1 <= n_fft / 2) {
    snprintf(msg, sizeof msg, "%s: waveform too short for reflect padding", who); rc = EAT_ERR_ARG;
  }
  if (rc != EAT_OK) eat_set_error(msg);
  return rc;
}
int mel_frames_per_cta(int n_fft) { return n_fft == 4096 ? MelShape<2048>::kFrames : MelShape<128>::kFrames; }
}  // namespace

extern "C" int eat_mel_bwd_workspace(int B, int N, int hop, int n_fft, long long* floats) {
  if (int rc = mel_geometry_check("eat_mel_bwd_workspace", B, N, n_fft, hop, n_fft, 1)) return rc;
  if (floats == nullptr) { eat_set_error("eat_mel_bwd_workspace: floats is null"); return EAT_ERR_ARG; }
  const int F = mel_frames_per_cta(n_fft), T = 1 + (N - 1) / hop;
  *floats = (long long)B * ((T + F - 1) / F) * ((long long)(F - 1) * hop + n_fft);
  return EAT_OK;
}

extern "C" int eat_mel_bwd(const float* dspec, const float* wave, int B, int N, const float* window, int win_length, int hop,
                           int n_fft, const float* twiddle, const int* fb_start, const int* fb_len, const float* fb_w,
                           int max_len, int n_mels, float preemph, const int* f_start, const int* f_end,
                           const int* t_start, const int* t_end, float* work, long long work_floats, float* dwave,
                           cudaStream_t stream) {
  if (int rc = mel_geometry_check("eat_mel_bwd", B, N, win_length, hop, n_fft, n_mels)) return rc;
  const bool masks = f_start != nullptr || f_end != nullptr || t_start != nullptr || t_end != nullptr;
  if (masks && (f_start == nullptr || f_end == nullptr || t_start == nullptr || t_end == nullptr)) {
    eat_set_error("eat_mel_bwd: the four mask bounds are given together or not at all"); return EAT_ERR_ARG;
  }
  if (B > 0 && (dspec == nullptr || wave == nullptr || window == nullptr || twiddle == nullptr || fb_start == nullptr ||
                fb_len == nullptr || fb_w == nullptr || work == nullptr || dwave == nullptr)) {
    eat_set_error("eat_mel_bwd: dspec, wave, window, twiddle, the filterbank, work and dwave are required");
    return EAT_ERR_ARG;
  }
  (void)max_len;
  MelBwdParams p;
  p.dspec = dspec; p.wave = wave; p.window = window; p.twiddle = reinterpret_cast<const float2*>(twiddle);
  p.fb_start = fb_start; p.fb_len = fb_len; p.fb_w = fb_w;
  p.fs = f_start; p.fe = f_end; p.ts = t_start; p.te = t_end; p.work = work;
  p.B = B; p.N = N; p.T = 1 + (N - 1) / hop; p.n_mels = n_mels; p.win_length = win_length; p.hop = hop; p.seg_len = 0;
  p.preemph = preemph; p.log_offset = 1e-5f; p.out_div = 5.f;
  switch (n_fft) {
    case 256: return mel_bwd_launch<128>(p, dwave, work_floats, stream);
    case 512: return mel_bwd_launch<256>(p, dwave, work_floats, stream);
    case 1024: return mel_bwd_launch<512>(p, dwave, work_floats, stream);
    case 2048: return mel_bwd_launch<1024>(p, dwave, work_floats, stream);
    default: return mel_bwd_launch<2048>(p, dwave, work_floats, stream);
  }
}
