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

template <int M>
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
  const int L = p.N - 1;
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
    const bool live = t < p.T;                 // uniform within a group
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
    if (t < p.T) p.out[((size_t)b * p.n_mels + m) * p.T + t] = s_out[m * (F + 1) + fo];
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
  static unsigned long long attr_mask = 0;
  if (int rc = eat_opt_in_smem(mel_kernel<M>, kSmemCap, attr_mask)) return rc;
  dim3 grid(ceil_div(p.T, S::kFrames), p.B);
  mel_kernel<M><<<grid, kThreads, smem, stream>>>(p);
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

extern "C" int eat_mel_fwd(const float* wave, int B, int N, const float* window, int win_length, int hop,
                           int n_fft, const float* twiddle, const int* fb_start, const int* fb_len,
                           const float* fb_w, int max_len, int n_mels, float preemph, float* out,
                           cudaStream_t stream) {
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
  switch (n_fft) {
    case 256: return mel_launch<128>(p, stream);
    case 512: return mel_launch<256>(p, stream);
    case 1024: return mel_launch<512>(p, stream);
    case 2048: return mel_launch<1024>(p, stream);
    default: return mel_launch<2048>(p, stream);
  }
}
