// Waveform augmentation of the fine-tuning and AudioSet datasets, on the device: gain, roll and waveform mixing
// (reference datasets/helpers/audiodatasets.py:26-51, the `pydub_augment` of esc50.py:39-44 / fsd50k.py:62-67 /
// openmic.py:56-61 / audioset.py:58-63, and the `MixupDataset` of esc50.py:47-69, dcase20.py:100-118,
// fsd50k.py:70-92, openmic.py:74-95, audioset.py:66-88).  The random draws come from the host (efficientat_b200/augment.py);
// these kernels apply them.
//   eat_clip_sum   fp64 sum of each source clip: the means of the mixing.  A roll does not change a sum and a gain
//                  scales it, so mean(gain * roll(x)) = gain * sum(x) / N.
//   eat_wave_aug   out[b, n] = c1 x_p[(n - s1) mod N] + c2 x_q[(n - s2) mod N] - c0: one pass, each source sample read
//                  once per output sample, the roll's wrap-around a select on the index, not a branch.
//   eat_label_mix  the matching label blend, under the plain, one-hot (DCASE20) and OpenMIC rules.
// No atomics: every result is bitwise repeatable.
#include <math.h>

#include "common.cuh"

namespace {

constexpr int kSumThreads = 512;
constexpr int kAugThreads = 256;
constexpr int kAugUnroll = 4;      // outputs per thread and pass: four independent loads of each source in flight

__global__ void __launch_bounds__(kSumThreads) clip_sum_kernel(const float* __restrict__ x, int N, double* __restrict__ sums) {
  __shared__ double red[kSumThreads / 32];
  const float* row = x + (size_t)blockIdx.x * N;
  double acc = 0.0;
  for (int n = threadIdx.x; n < N; n += kSumThreads) acc += (double)row[n];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
#pragma unroll
    for (int w = 0; w < kSumThreads / 32; ++w) s += red[w];
    sums[blockIdx.x] = s;
  }
}

// (n - s) mod N for 0 <= n < N, with sm = s mod N in [0, N): the wrap is a select
__device__ __forceinline__ int rolled(int n, int sm, int N) {
  const int j = n - sm;
  return j < 0 ? j + N : j;
}

// grid (chunks, B).  Row b: primary p = idx1[b], partner q = idx2[b] (-1: not mixed).  Not mixed: c1 = gain1, c2 = 0,
// c0 = 0.  Mixed, with l = lam[b]: c1 = l gain1, c2 = (1 - l) gain2 and c0 = (c1 sum_p + c2 sum_q) / N, the mean of the
// blend, removed so that the row comes out centred as x - x.mean() leaves it.  An index outside its range, or a mixed
// row without sums, makes the row NaN.
__global__ void __launch_bounds__(kAugThreads) wave_aug_kernel(const float* __restrict__ src, const double* __restrict__ sums,
                                                               int S, int N, const int* __restrict__ idx1,
                                                               const int* __restrict__ idx2, const int* __restrict__ shift1,
                                                               const int* __restrict__ shift2, const float* __restrict__ gain1,
                                                               const float* __restrict__ gain2, const float* __restrict__ lam,
                                                               float* __restrict__ out) {
  const int b = blockIdx.y;
  const int p = idx1[b], q = idx2[b];
  float* o = out + (size_t)b * N;
  const int stride = gridDim.x * kAugThreads;
  int n0 = blockIdx.x * kAugThreads * kAugUnroll + threadIdx.x;
  const bool mixed = q >= 0;
  if (p < 0 || p >= S || q >= S || q < -1 || (mixed && sums == nullptr)) {
    for (int n = blockIdx.x * kAugThreads + threadIdx.x; n < N; n += stride) o[n] = __int_as_float(0x7fc00000);
    return;
  }
  const float* xp = src + (size_t)p * N;
  const int s1 = ((shift1[b] % N) + N) % N;
  if (!mixed) {
    const float c1 = gain1[b];
    for (; n0 < N; n0 += stride * kAugUnroll) {
      float v[kAugUnroll];
#pragma unroll
      for (int u = 0; u < kAugUnroll; ++u) {
        const int n = n0 + u * kAugThreads;
        v[u] = n < N ? xp[rolled(n, s1, N)] : 0.f;
      }
#pragma unroll
      for (int u = 0; u < kAugUnroll; ++u) {
        const int n = n0 + u * kAugThreads;
        if (n < N) o[n] = c1 * v[u];
      }
    }
    return;
  }
  const float* xq = src + (size_t)q * N;
  const int s2 = ((shift2[b] % N) + N) % N;
  const double l = (double)lam[b];
  const double d1 = l * (double)gain1[b], d2 = (1.0 - l) * (double)gain2[b];
  const float c1 = (float)d1, c2 = (float)d2;
  const float c0 = (float)((d1 * sums[p] + d2 * sums[q]) / (double)N);
  for (; n0 < N; n0 += stride * kAugUnroll) {
    float v[kAugUnroll], w[kAugUnroll];
#pragma unroll
    for (int u = 0; u < kAugUnroll; ++u) {
      const int n = n0 + u * kAugThreads;
      v[u] = n < N ? xp[rolled(n, s1, N)] : 0.f;
      w[u] = n < N ? xq[rolled(n, s2, N)] : 0.f;
    }
#pragma unroll
    for (int u = 0; u < kAugUnroll; ++u) {
      const int n = n0 + u * kAugThreads;
      if (n < N) o[n] = fmaf(c1, v[u], fmaf(c2, w[u], -c0));
    }
  }
}

// grid-stride over out [B, C].  Row b blends the label rows of p = idx1[b] and q = idx2[b] (-1: row p alone).
__global__ void label_mix_kernel(int rule, const float* __restrict__ yp, const int* __restrict__ yi, int S, int C,
                                 const int* __restrict__ idx1, const int* __restrict__ idx2, const float* __restrict__ lam,
                                 int B, float* __restrict__ out) {
  const long long total = (long long)B * C;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int b = (int)(i / C), c = (int)(i % C);
    const int p = idx1[b], q = idx2[b];
    if (p < 0 || p >= S || q >= S || q < -1) { out[i] = __int_as_float(0x7fc00000); continue; }
    const float l = q >= 0 ? lam[b] : 1.f;
    float v;
    if (rule == EAT_LABEL_ONEHOT) {
      const int k1 = yi[p], k2 = q >= 0 ? yi[q] : -1;
      if (k1 < 0 || k1 >= C || (q >= 0 && (k2 < 0 || k2 >= C))) v = __int_as_float(0x7fc00000);
      else v = (k1 == c ? l : 0.f) + (k2 == c ? 1.f - l : 0.f);
    } else if (q < 0) {
      v = yp[(size_t)p * C + c];
    } else if (rule == EAT_LABEL_PLAIN) {
      v = yp[(size_t)p * C + c] * l + yp[(size_t)q * C + c] * (1.f - l);
    } else {                            // OpenMIC: C = 2H, scores | mask; scores masked before the blend, masks max-ed
      const int H = C / 2;
      const int cm = c < H ? c + H : c;
      const float m1 = yp[(size_t)p * C + cm] > 0.5f ? 1.f : 0.f, m2 = yp[(size_t)q * C + cm] > 0.5f ? 1.f : 0.f;
      v = c < H ? yp[(size_t)p * C + c] * m1 * l + yp[(size_t)q * C + c] * m2 * (1.f - l) : fmaxf(m1, m2);
    }
    out[i] = v;
  }
}

}  // namespace

extern "C" {

int eat_clip_sum(const float* x, int S, int N, double* sums, cudaStream_t st) {
  if (S < 0 || N < 1) { eat_set_error("clip_sum: need S >= 0 and N >= 1"); return EAT_ERR_ARG; }
  if (S == 0) return EAT_OK;
  if (x == nullptr || sums == nullptr) { eat_set_error("clip_sum: x and sums are required"); return EAT_ERR_ARG; }
  clip_sum_kernel<<<S, kSumThreads, 0, st>>>(x, N, sums);
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

int eat_wave_aug(const float* src, const double* sums, int S, int N, const int* idx1, const int* idx2, const int* shift1,
                 const int* shift2, const float* gain1, const float* gain2, const float* lam, float* out, int B,
                 cudaStream_t st) {
  if (B < 0 || B > 65535 || S < 1 || N < 1 || N > (1 << 30)) {
    eat_set_error("wave_aug: need 0 <= B <= 65535, S >= 1 and 1 <= N <= 2^30"); return EAT_ERR_ARG;
  }
  if (B == 0) return EAT_OK;
  if (src == nullptr || idx1 == nullptr || idx2 == nullptr || shift1 == nullptr || shift2 == nullptr ||
      gain1 == nullptr || gain2 == nullptr || lam == nullptr || out == nullptr) {
    eat_set_error("wave_aug: src, idx1, idx2, shift1, shift2, gain1, gain2, lam and out are required"); return EAT_ERR_ARG;
  }
  // about four resident CTAs per SM over the whole batch; each thread then walks its row with kAugUnroll loads in flight
  const int per_row = ceil_div(N, kAugThreads * kAugUnroll);
  const int chunks = max(1, min(per_row, ceil_div(kNumSMs * 4 * 8, B)));
  wave_aug_kernel<<<dim3(chunks, B), kAugThreads, 0, st>>>(src, sums, S, N, idx1, idx2, shift1, shift2, gain1, gain2, lam, out);
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

int eat_label_mix(int rule, const float* y_prob, const int* y_index, int S, int C, const int* idx1, const int* idx2,
                  const float* lam, int B, float* out, cudaStream_t st) {
  if (rule != EAT_LABEL_PLAIN && rule != EAT_LABEL_ONEHOT && rule != EAT_LABEL_OPENMIC) {
    eat_set_error("label_mix: rule must be EAT_LABEL_PLAIN, EAT_LABEL_ONEHOT or EAT_LABEL_OPENMIC"); return EAT_ERR_ARG;
  }
  if (B < 0 || S < 1 || C < 1 || (rule == EAT_LABEL_OPENMIC && C % 2)) {
    eat_set_error("label_mix: need B >= 0, S >= 1, C >= 1 (even for EAT_LABEL_OPENMIC)"); return EAT_ERR_ARG;
  }
  if ((rule == EAT_LABEL_ONEHOT) != (y_index != nullptr) || (y_prob != nullptr) == (y_index != nullptr)) {
    eat_set_error("label_mix: EAT_LABEL_ONEHOT takes y_index only, the other rules y_prob only"); return EAT_ERR_ARG;
  }
  if (B == 0) return EAT_OK;
  if (idx1 == nullptr || idx2 == nullptr || lam == nullptr || out == nullptr) {
    eat_set_error("label_mix: idx1, idx2, lam and out are required"); return EAT_ERR_ARG;
  }
  const int grid = (int)min((long long)kNumSMs * 2, ceil_div_ll((long long)B * C, 256));
  label_mix_kernel<<<grid, 256, 0, st>>>(rule, y_prob, y_index, S, C, idx1, idx2, lam, B, out);
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

}  // extern "C"
