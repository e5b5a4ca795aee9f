// Clips of different lengths in one eval batch.  A batch [B, F, T, C] holds clip b in its first t_valid[b] time steps;
// the rest is padding.  Only the operations that mix values along time see the padding, and these kernels keep each
// clip's result equal to the one it gets alone:
//   eat_time_pad_zero  writes 0 into the padding, so that a convolution's taps past a clip's end read what its own
//                      zero padding would supply;
//   eat_mean_len       the mean over the valid region only (squeeze-excitation, global average pool, ContextGen's h_c);
//   eat_ctx_pool_len   ContextGen's pair of means (dy_block.py:236-240) with the mean over time taken over t < t_valid.
// None of them uses atomics: the sums run in a fixed order, so the results do not depend on the padding's content.
#include <cstdio>

#include "common.cuh"

namespace {

constexpr int kMeanLanes = 32;     // channels per CTA of eat_mean_len (one warp row)
constexpr int kMeanRows = 16;      // rows of the CTA, each walking its own share of the valid positions

template <typename T>
__global__ void __launch_bounds__(256) time_pad_zero_kernel(T* __restrict__ x, int F, int Tn, int C,
                                                            const int* __restrict__ t_valid) {
  const int f = blockIdx.x, b = blockIdx.y;
  const int tb = t_valid[b];
  const long long n = (long long)(Tn - tb) * C;          // the padding of one (sample, frequency) row is contiguous
  T* row = x + (((long long)b * F + f) * Tn + tb) * C;
  for (long long i = threadIdx.x; i < n; i += blockDim.x) row[i] = from_f32<T>(0.f);
}

// out[b, c] = sum over f < F, t < t_valid[b] of x[b, f, t, c], divided by F * t_valid[b]
template <typename T>
__global__ void __launch_bounds__(kMeanLanes * kMeanRows) mean_len_kernel(const T* __restrict__ x, float* __restrict__ out,
                                                                        int F, int Tn, int C,
                                                                        const int* __restrict__ t_valid) {
  __shared__ float red[kMeanRows][kMeanLanes + 1];
  const int b = blockIdx.y;
  const int c = blockIdx.x * kMeanLanes + threadIdx.x;
  const int tb = t_valid[b];
  float acc = 0.f;
  if (c < C) {
    const T* xb = x + (long long)b * F * Tn * C + c;
    for (int f = 0; f < F; ++f) {
      const T* xf = xb + (long long)f * Tn * C;
      for (int t = threadIdx.y; t < tb; t += kMeanRows) acc += to_f32<T>(xf[(long long)t * C]);
    }
  }
  red[threadIdx.y][threadIdx.x] = acc;
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
    float s = 0.f;
#pragma unroll
    for (int r = 0; r < kMeanRows; ++r) s += red[r][threadIdx.x];
    out[(long long)b * C + c] = s * (1.f / ((float)F * (float)tb));
  }
}

// rows f < F: mean over t < t_valid[b]; rows F + t: mean over f for t < t_valid[b], 0 beyond
template <typename T>
__global__ void __launch_bounds__(256) ctx_pool_len_kernel(const T* __restrict__ x, float* __restrict__ out, int F, int Tn,
                                                           int C, const int* __restrict__ t_valid) {
  constexpr int V = Vec<T>::N;
  const int cv = C / V;
  const int b = blockIdx.y;
  const int tb = t_valid[b];
  const int items = (F + Tn) * cv;
  const T* xb = x + (size_t)b * F * Tn * C;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < items; i += gridDim.x * blockDim.x) {
    const int cvi = i % cv, pos = i / cv;
    const int c0 = cvi * V;
    float acc[V];
#pragma unroll
    for (int k = 0; k < V; ++k) acc[k] = 0.f;
    if (pos < F) {
      const T* p = xb + (size_t)pos * Tn * C + c0;
      for (int t = 0; t < tb; ++t) {
        float v[V];
        Vec<T>::load(p + (size_t)t * C, v);
#pragma unroll
        for (int k = 0; k < V; ++k) acc[k] += v[k];
      }
      const float inv = 1.f / tb;
#pragma unroll
      for (int k = 0; k < V; ++k) acc[k] *= inv;
    } else if (pos - F < tb) {
      const T* p = xb + (size_t)(pos - F) * C + c0;
      for (int f = 0; f < F; ++f) {
        float v[V];
        Vec<T>::load(p + (size_t)f * Tn * C, v);
#pragma unroll
        for (int k = 0; k < V; ++k) acc[k] += v[k];
      }
      const float inv = 1.f / F;
#pragma unroll
      for (int k = 0; k < V; ++k) acc[k] *= inv;
    }
    float* o = out + ((size_t)b * (F + Tn) + pos) * C + c0;
#pragma unroll
    for (int k = 0; k < V; ++k) o[k] = acc[k];
  }
}

int len_check(const char* who, const void* x, int dtype, int B, int F, int T, int C, const int* t_valid) {
  static char msg[200];
  if (dtype != EAT_F32 && dtype != EAT_BF16) {
    snprintf(msg, sizeof msg, "%s: dtype must be EAT_F32 or EAT_BF16", who); eat_set_error(msg); return EAT_ERR_ARG;
  }
  if (B < 0 || F < 1 || T < 1 || C < 1 || B > 65535 || F > 65535) {
    snprintf(msg, sizeof msg, "%s: need 0 <= B <= 65535, 1 <= F <= 65535 and T, C >= 1", who);
    eat_set_error(msg); return EAT_ERR_ARG;
  }
  if (B > 0 && (x == nullptr || t_valid == nullptr)) {
    snprintf(msg, sizeof msg, "%s: x and t_valid are required", who); eat_set_error(msg); return EAT_ERR_ARG;
  }
  return EAT_OK;
}

}  // namespace

extern "C" {

int eat_time_pad_zero(void* x, int dtype, int B, int F, int T, int C, const int* t_valid, cudaStream_t st) {
  if (int rc = len_check("time_pad_zero", x, dtype, B, F, T, C, t_valid)) return rc;
  if (B == 0) return EAT_OK;
  const dim3 grid(F, B);
  if (dtype == EAT_BF16) time_pad_zero_kernel<__nv_bfloat16><<<grid, 256, 0, st>>>((__nv_bfloat16*)x, F, T, C, t_valid);
  else time_pad_zero_kernel<float><<<grid, 256, 0, st>>>((float*)x, F, T, C, t_valid);
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

int eat_mean_len(const void* x, int dtype, float* out, int B, int F, int T, int C, const int* t_valid, cudaStream_t st) {
  if (int rc = len_check("mean_len", x, dtype, B, F, T, C, t_valid)) return rc;
  if (B == 0) return EAT_OK;
  if (out == nullptr) { eat_set_error("mean_len: out is required"); return EAT_ERR_ARG; }
  const dim3 grid(ceil_div(C, kMeanLanes), B), block(kMeanLanes, kMeanRows);
  if (dtype == EAT_BF16) mean_len_kernel<__nv_bfloat16><<<grid, block, 0, st>>>((const __nv_bfloat16*)x, out, F, T, C, t_valid);
  else mean_len_kernel<float><<<grid, block, 0, st>>>((const float*)x, out, F, T, C, t_valid);
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

int eat_ctx_pool_len(const void* x, int dtype, float* out, int B, int F, int T, int C, const int* t_valid,
                     cudaStream_t st) {
  if (int rc = len_check("ctx_pool_len", x, dtype, B, F, T, C, t_valid)) return rc;
  const int V = dtype == EAT_BF16 ? 8 : 4;
  if (C % V != 0) { eat_set_error("ctx_pool_len: channels must be a multiple of the vector width"); return EAT_ERR_ARG; }
  if (B == 0) return EAT_OK;
  if (out == nullptr) { eat_set_error("ctx_pool_len: out is required"); return EAT_ERR_ARG; }
  const dim3 grid(ceil_div((F + T) * (C / V), 256), B);
  if (dtype == EAT_BF16) ctx_pool_len_kernel<__nv_bfloat16><<<grid, 256, 0, st>>>((const __nv_bfloat16*)x, out, F, T, C, t_valid);
  else ctx_pool_len_kernel<float><<<grid, 256, 0, st>>>((const float*)x, out, F, T, C, t_valid);
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

}  // extern "C"
