// Shared device helpers for the EfficientAT H100 kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>

#include "../../include/eat_b200.h"   // the C ABI: declarations here are checked against definitions

#define EAT_CHECK_LAUNCH()                                   \
  do {                                                       \
    cudaError_t e__ = cudaGetLastError();                    \
    if (e__ != cudaSuccess) { eat_set_error(cudaGetErrorString(e__)); return EAT_ERR_CUDA; } \
  } while (0)

void eat_set_error(const char* msg);

// streaming multiprocessors of an H100 SXM: grid caps of the grid-stride kernels (one or a few resident waves)
constexpr int kNumSMs = 132;

// cudaFuncAttributeMaxDynamicSharedMemorySize is a per-DEVICE attribute: remember it per (kernel instantiation, device)
// so that a process driving several GPUs opts every one of them in.  `mask` is a function-local static of the caller.
template <typename K>
inline int eat_opt_in_smem(K kernel, size_t bytes, unsigned long long& mask) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) { eat_set_error("cudaGetDevice failed"); return EAT_ERR_CUDA; }
  const unsigned long long bit = 1ull << (dev & 63);
  if (!(mask & bit)) {
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e != cudaSuccess) { eat_set_error(cudaGetErrorString(e)); return EAT_ERR_CUDA; }
    mask |= bit;
  }
  return EAT_OK;
}

__host__ __device__ inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
__host__ __device__ inline long long ceil_div_ll(long long a, long long b) { return (a + b - 1) / b; }

__device__ __forceinline__ float act_fwd(float v, int act) {
  if (act == EAT_ACT_RELU) return fmaxf(v, 0.f);
  if (act == EAT_ACT_HSWISH) return v * fminf(fmaxf(v + 3.f, 0.f), 6.f) * (1.f / 6.f);
  if (act == EAT_ACT_SIGMOID) return 1.f / (1.f + expf(-v));
  return v;
}
// derivative of the activation w.r.t. its input, evaluated at pre-activation v
// (hardswish' = 0 for v<=-3, 1 for v>=3, (2v+3)/6 in between, as torch 2.x's hardswish_backward -- the torch the golden
// vectors and the oracle are produced with; torch 1.13 gave -1/2 at -3 and 3/2 at 3; relu' = v>0)
__device__ __forceinline__ float act_bwd(float v, int act) {
  if (act == EAT_ACT_RELU) return v > 0.f ? 1.f : 0.f;
  if (act == EAT_ACT_HSWISH) return v <= -3.f ? 0.f : (v < 3.f ? (2.f * v + 3.f) * (1.f / 6.f) : 1.f);
  return 1.f;
}
__device__ __forceinline__ float sigmoidf_(float v) { return 1.f / (1.f + expf(-v)); }

// ---- vector load/store of V contiguous channels as fp32, for fp32 (V=4) and bf16 (V=8) storage.
template <typename T> struct Vec;
template <> struct Vec<float> {
  static constexpr int N = 4;
  __device__ __forceinline__ static void load(const float* p, float (&v)[4]) {
    float4 t = *reinterpret_cast<const float4*>(p);
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
  }
  __device__ __forceinline__ static void store(float* p, const float (&v)[4]) {
    *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
  }
};
template <> struct Vec<__nv_bfloat16> {
  static constexpr int N = 8;
  __device__ __forceinline__ static void load(const __nv_bfloat16* p, float (&v)[8]) {
    uint4 t = *reinterpret_cast<const uint4*>(p);
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&t);
#pragma unroll
    for (int i = 0; i < 4; ++i) { float2 f = __bfloat1622float2(h[i]); v[2 * i] = f.x; v[2 * i + 1] = f.y; }
  }
  __device__ __forceinline__ static void store(__nv_bfloat16* p, const float (&v)[8]) {
    uint4 t;
    __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&t);
#pragma unroll
    for (int i = 0; i < 4; ++i) h[i] = __floats2bfloat162_rn(v[2 * i], v[2 * i + 1]);
    *reinterpret_cast<uint4*>(p) = t;
  }
};

template <typename T> __device__ __forceinline__ float to_f32(T v);
template <> __device__ __forceinline__ float to_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_f32<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }
template <typename T> __device__ __forceinline__ T from_f32(float v);
template <> __device__ __forceinline__ float from_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ __nv_bfloat16 from_f32<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

// Per-channel affine + activation + per-(sample,channel) gate applied to an operand as it is loaded:
//   v' = act(v * scale[c] + shift[c]) * gate[b * C + c]
// scale == nullptr -> no affine/act;  gate == nullptr -> no gate.
struct InXform {
  const float* scale;
  const float* shift;
  const float* gate;
  int act;
  int rows_per_sample;   // F*T of the tensor the gate indexes (rows -> sample index)
};

struct DyEpi {
  const float* theta;    // [B, C, 2M] sigmoid(coef_net(h_c)) or nullptr (M = DyReLU-B pieces, 2 unless stated)
  const float* lam;      // [2M] lambdas
  const float* init;     // [2M] init_v
  const float* ca_f;     // [B, Fo, C] sigmoid(g_cf) or nullptr
  const float* ca_t;     // [B, To, C] sigmoid(g_ct)
  long long wt_bstride;  // floats between the weight tables of consecutive samples (0: shared weights)
};

// DyReLU-B with M linear pieces (dy_block.py:172-188) for one channel, the form every kernel with a DyReLU-B epilogue or
// backward holds in registers.  theta points at the channel's 2M values of sigmoid(coef_net(h_c)), channel-major
// ([B, C, 2M]); a_m = (2 theta_m - 1) lam_m + init_m is the slope of piece m and b_m = (2 theta_{M+m} - 1) lam_{M+m} +
// init_{M+m} its offset; out = max_m (a_m x + b_m).
template <int M>
struct DyCoef {
  float a[M], b[M];
  // ldg: read theta through the read-only data cache.  For even M the 2M values are read as 16-byte vectors (theta
  // 16-byte aligned); lam and init are plain loads.
  __device__ __forceinline__ void load(const float* theta, const float* lam, const float* init, bool ldg) {
    float th[2 * M];
    if constexpr (M % 2 == 0) {
#pragma unroll
      for (int q = 0; q < M / 2; ++q) {
        const float4* p = reinterpret_cast<const float4*>(theta) + q;
        const float4 t = ldg ? __ldg(p) : *p;
        th[4 * q] = t.x; th[4 * q + 1] = t.y; th[4 * q + 2] = t.z; th[4 * q + 3] = t.w;
      }
    } else {
#pragma unroll
      for (int j = 0; j < 2 * M; ++j) th[j] = ldg ? __ldg(theta + j) : theta[j];
    }
#pragma unroll
    for (int m = 0; m < M; ++m) a[m] = (2.f * th[m] - 1.f) * lam[m] + init[m];
#pragma unroll
    for (int m = 0; m < M; ++m) b[m] = (2.f * th[M + m] - 1.f) * lam[M + m] + init[M + m];
  }
  __device__ __forceinline__ void zero() {
#pragma unroll
    for (int m = 0; m < M; ++m) a[m] = b[m] = 0.f;
  }
  __device__ __forceinline__ float apply(float x) const {
    float o = fmaf(x, a[0], b[0]);
#pragma unroll
    for (int m = 1; m < M; ++m) o = fmaxf(o, fmaf(x, a[m], b[m]));
    return o;
  }
};

// sliding-window depthwise convolution (dw_slide.cu); same contract as launch_dw in conv_kernels.cu.  dyk: DyReLU-B
// pieces of the eval epilogue (1..4; only read when dy.theta is set)
int dw_slide_launch(const void* in, const float* wt, void* out, int dtype, int B, int F, int Tn, int C, int k, int stride,
                    InXform xf, const float* scale, const float* shift, int act, const void* res, int flip, float* pool,
                    double* ssum, double* ssq, cudaStream_t st, DyEpi dy, int dyk = 2);

int dw_wgrad_slide_launch(const void* dz, const void* in, InXform xf, float* dw, long long dw_bstride, int dtype, int B,
                          int F, int Tn, int C, int k, int stride, cudaStream_t st);

// launch plan of the shared-memory tile kernel dw_tile_kernel (conv_kernels.cu): 32-channel chunks, FR x TT output tiles
// per chunk, `groups` CTAs per (chunk, sample) that stride over the tiles; gridDim = (chunks * groups, B)
struct DwTilePlan { int chunks, tiles, groups, FR, TT; };
DwTilePlan dw_tile_plan(int B, int Fo, int To, int C, int stride);

// z != nullptr: BatchNorm-backward reduce of the layer behind din in the epilogue (fp32 storage; see Dg2Args in dw_slide.cu)
int dw_dgrad2_slide_launch(const void* dz, const float* wt, long long wt_bstride, const void* res, void* din, int dtype,
                           int B, int F, int Tn, int C, int k, cudaStream_t st, const void* z = nullptr,
                           const float* zscale = nullptr, const float* zshift = nullptr, const float* zmean = nullptr,
                           const float* zinvstd = nullptr, int zact = 0, double* s1 = nullptr, double* s2 = nullptr);

// CUDA-core weight gradient for narrow 1x1 convolutions (wgrad_narrow.cu); EAT_ERR_UNSUPPORTED = shape out of range
int wgrad_narrow_launch(const float* G, const float* A, float* dW, long long M, int N, int K, const float* in_scale,
                        const float* in_shift, int in_act, cudaStream_t st);

// argument checks of the entry points that take per-clip lengths t_valid [B] of a [B, F, T, C] batch (packed.cu)
int len_check(const char* who, const void* x, int dtype, int B, int F, int T, int C, const int* t_valid);

// C[M, N] = alpha * A[M, K] . W[K, N], fp32, 32 x 32 tiles (gemm_simt.cu)
int gemm_small_kn_launch(const float* A, const float* W, float* C, int M, int N, int K, float alpha, cudaStream_t st);

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
