// Gradients of the returned feature maps into the engine's NHWC storage (eat_fmap_grad_nhwc).
//
// Autograd hands the gradient of a map returned as a [B, C, F, T] view in whatever layout the loss produced: contiguous
// NCHW, channels-last, or an expanded broadcast (a frequency mean gives stride 0 on F).  The backward chain wants it
// as a contiguous [B, F, T, C] tensor of the storage dtype, added to the gradient coming from the layers above.
//   - src fastest along T or F: a shared-memory tiled transpose, 32 positions of that axis x 32 channels per tile;
//     the loads run along the source's unit-stride axis, the stores are 16 bytes along C.
//   - src fastest along C (or not varying along C): 8 channels per thread, 16-byte stores (two for fp32 dst) and,
//     when the source is contiguous and aligned along C, 16-byte loads.
//   - C not a multiple of 8 or a misaligned dst: one element per thread.
// The arithmetic is fp32: dst = (accumulate ? dst : 0) + src, one rounding to the dst dtype.
#include "common.cuh"

namespace {

constexpr int kFgThreads = 256;
constexpr int kTile = 32;          // transpose tile: kTile positions of the unit-stride axis x kTile channels

bool unaligned16(const void* p) { return ((uintptr_t)p & 15) != 0; }

// 8 consecutive elements <-> fp32, with 16-byte accesses (p 16-byte aligned)
template <typename T> __device__ __forceinline__ void load8(const T* p, float (&v)[8]);
template <> __device__ __forceinline__ void load8<float>(const float* p, float (&v)[8]) {
  const float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 4);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
template <> __device__ __forceinline__ void load8<__nv_bfloat16>(const __nv_bfloat16* p, float (&v)[8]) {
  Vec<__nv_bfloat16>::load(p, v);
}
template <typename T> __device__ __forceinline__ void store8(T* p, const float (&v)[8]);
template <> __device__ __forceinline__ void store8<float>(float* p, const float (&v)[8]) {
  *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
  *reinterpret_cast<float4*>(p + 4) = make_float4(v[4], v[5], v[6], v[7]);
}
template <> __device__ __forceinline__ void store8<__nv_bfloat16>(__nv_bfloat16* p, const float (&v)[8]) {
  Vec<__nv_bfloat16>::store(p, v);
}

// src fastest along C: thread i owns channels 8*(i % (C/8)) .. +7 of pixel i / (C/8)
template <typename TS, typename TD, bool VLOAD>
__global__ void __launch_bounds__(kFgThreads) fmap_grad_direct_kernel(
    const TS* __restrict__ src, long long sB, long long sC, long long sF, long long sT, TD* __restrict__ dst, int B,
    int C, int F, int T, int acc) {
  const int CG = C / 8;
  const long long n = (long long)B * F * T * CG;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int cg = (int)(i % CG);
    const long long pix = i / CG;
    const int t = (int)(pix % T);
    const long long bf = pix / T;
    const int f = (int)(bf % F), b = (int)(bf / F);
    const TS* s = src + b * sB + f * sF + t * sT + 8LL * cg * sC;
    float v[8];
    if (VLOAD) {
      load8(s, v);
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = to_f32(s[j * sC]);
    }
    TD* d = dst + pix * C + 8 * cg;
    if (acc) {
      float o[8];
      load8(d, o);
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = o[j] + v[j];
    }
    store8(d, v);
  }
}

// src fastest along axis u (T or F).  Outer index o = (b, w) with w the other spatial axis; the src offset of
// (b, w, u, c) is b*sB + w*sW + u*sU + c*sC, the dst offset b*dB + w*dW + u*dU + c (C % 8 == 0)
template <typename TS, typename TD>
__global__ void __launch_bounds__(kFgThreads) fmap_grad_transpose_kernel(
    const TS* __restrict__ src, long long sB, long long sW, long long sU, long long sC, TD* __restrict__ dst, long long dB,
    long long dW, long long dU, int B, int W, int U, int C, int acc) {
  constexpr int VD = sizeof(TD) == 4 ? 4 : 8;       // dst elements per 16-byte store
  __shared__ float tile[kTile][kTile + 1];          // [channel][u]
  const int tu = ceil_div(U, kTile), tc = ceil_div(C, kTile);
  const long long ntiles = (long long)B * W * tu * tc;
  const int lane = threadIdx.x % kTile, row = threadIdx.x / kTile;
  for (long long tl = blockIdx.x; tl < ntiles; tl += gridDim.x) {
    const int ic = (int)(tl % tc);
    long long r = tl / tc;
    const int iu = (int)(r % tu);
    r /= tu;
    const int w = (int)(r % W), b = (int)(r / W);
    const int u0 = iu * kTile, c0 = ic * kTile;
    const TS* s = src + b * sB + w * sW;
    const int u = u0 + lane;
#pragma unroll
    for (int cc = row; cc < kTile; cc += kFgThreads / kTile) {
      const int c = c0 + cc;
      tile[cc][lane] = (u < U && c < C) ? to_f32(s[u * sU + c * sC]) : 0.f;
    }
    __syncthreads();
    TD* d = dst + b * dB + w * dW;
    for (int k = threadIdx.x; k < kTile * (kTile / VD); k += kFgThreads) {
      const int uu = k / (kTile / VD), cq = (k % (kTile / VD)) * VD;
      if (u0 + uu < U && c0 + cq < C) {
        TD* p = d + (long long)(u0 + uu) * dU + c0 + cq;
        float v[VD];
#pragma unroll
        for (int j = 0; j < VD; ++j) v[j] = tile[cq + j][uu];
        if (acc) {
          float o[VD];
          Vec<TD>::load(p, o);
#pragma unroll
          for (int j = 0; j < VD; ++j) v[j] = o[j] + v[j];
        }
        Vec<TD>::store(p, v);
      }
    }
    __syncthreads();
  }
}

// any C, any alignment: one dst element per thread
template <typename TS, typename TD>
__global__ void __launch_bounds__(kFgThreads) fmap_grad_scalar_kernel(
    const TS* __restrict__ src, long long sB, long long sC, long long sF, long long sT, TD* __restrict__ dst, int B,
    int C, int F, int T, int acc) {
  const long long n = (long long)B * F * T * C;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const long long pix = i / C;
    const int t = (int)(pix % T);
    const long long bf = pix / T;
    const int f = (int)(bf % F), b = (int)(bf / F);
    float v = to_f32(src[b * sB + c * sC + f * sF + t * sT]);
    if (acc) v = to_f32(dst[i]) + v;
    dst[i] = from_f32<TD>(v);
  }
}

int grid_for(long long work) { return (int)min((long long)kNumSMs * 16, max(1LL, ceil_div_ll(work, kFgThreads))); }

template <typename TS, typename TD>
int launch(const void* src_, long long sB, long long sC, long long sF, long long sT, void* dst_, int B, int C, int F,
           int T, int acc, cudaStream_t st) {
  const TS* src = (const TS*)src_;
  TD* dst = (TD*)dst_;
  // the unit axis: the smallest positive stride among the axes longer than one; C wins ties, and a source that does
  // not vary along C (sC == 0) is read by the direct path, one broadcast value per pixel
  int axis = 0;                                     // 0: C, 1: F, 2: T
  long long best = -1;
  const long long strides[3] = {sC, sF, sT};
  const int sizes[3] = {C, F, T};
  for (int a = 0; a < 3; ++a)
    if (sizes[a] > 1 && strides[a] > 0 && (best < 0 || strides[a] < best)) { best = strides[a]; axis = a; }
  const bool vec = C % 8 == 0 && !unaligned16(dst);
  if (!vec) {
    fmap_grad_scalar_kernel<TS, TD><<<grid_for((long long)B * F * T * C), kFgThreads, 0, st>>>(
        src, sB, sC, sF, sT, dst, B, C, F, T, acc);
  } else if (axis == 0 || sC == 0) {
    const long long work = (long long)B * F * T * (C / 8);
    const bool vload = sC == 1 && !unaligned16(src) && sB % 8 == 0 && sF % 8 == 0 && sT % 8 == 0;
    if (vload)
      fmap_grad_direct_kernel<TS, TD, true><<<grid_for(work), kFgThreads, 0, st>>>(src, sB, sC, sF, sT, dst, B, C, F, T, acc);
    else
      fmap_grad_direct_kernel<TS, TD, false><<<grid_for(work), kFgThreads, 0, st>>>(src, sB, sC, sF, sT, dst, B, C, F, T, acc);
  } else {
    const long long dB = (long long)F * T * C;
    // axis T: o = (b, f), u = t;  axis F: o = (b, t), u = f
    const int W = axis == 2 ? F : T, U = axis == 2 ? T : F;
    const long long sW = axis == 2 ? sF : sT, sU = axis == 2 ? sT : sF;
    const long long dW = axis == 2 ? (long long)T * C : C, dU = axis == 2 ? C : (long long)T * C;
    const long long tiles = (long long)B * W * ceil_div(U, kTile) * ceil_div(C, kTile);
    const int grid = (int)min((long long)kNumSMs * 8, tiles);
    fmap_grad_transpose_kernel<TS, TD><<<grid, kFgThreads, 0, st>>>(src, sB, sW, sU, sC, dst, dB, dW, dU, B, W, U, C, acc);
  }
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

}  // namespace

extern "C" {

int eat_fmap_grad_nhwc(const void* src, int src_dtype, long long sB, long long sC, long long sF, long long sT, void* dst,
                       int dst_dtype, int B, int C, int F, int T, int accumulate, cudaStream_t st) {
  if ((src_dtype != EAT_F32 && src_dtype != EAT_BF16) || (dst_dtype != EAT_F32 && dst_dtype != EAT_BF16)) {
    eat_set_error("fmap grad: src_dtype and dst_dtype must be EAT_F32 or EAT_BF16"); return EAT_ERR_ARG;
  }
  if (B < 0 || C < 0 || F < 0 || T < 0) { eat_set_error("fmap grad: negative sizes"); return EAT_ERR_ARG; }
  if (sB < 0 || sC < 0 || sF < 0 || sT < 0) { eat_set_error("fmap grad: negative strides"); return EAT_ERR_ARG; }
  if (B == 0 || C == 0 || F == 0 || T == 0) return EAT_OK;
  if (src == nullptr || dst == nullptr) { eat_set_error("fmap grad: src and dst are required"); return EAT_ERR_ARG; }
  const int acc = accumulate != 0;
  if (src_dtype == EAT_F32)
    return dst_dtype == EAT_F32 ? launch<float, float>(src, sB, sC, sF, sT, dst, B, C, F, T, acc, st)
                                : launch<float, __nv_bfloat16>(src, sB, sC, sF, sT, dst, B, C, F, T, acc, st);
  return dst_dtype == EAT_F32 ? launch<__nv_bfloat16, float>(src, sB, sC, sF, sT, dst, B, C, F, T, acc, st)
                              : launch<__nv_bfloat16, __nv_bfloat16>(src, sB, sC, sF, sT, dst, B, C, F, T, acc, st);
}

}  // extern "C"
