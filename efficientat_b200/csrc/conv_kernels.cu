// Bandwidth-bound kernels of the MobileNetV3 path, NHWC activations ([B, F, T, C], C innermost):
//   stem 3x3 conv (Cin = 1), depthwise k x k conv, BatchNorm helpers, squeeze-excitation MLP.
// Every kernel takes an optional per-channel affine+activation on its INPUT (the BatchNorm +
// activation of the producing layer, applied on load so the normalised tensor is never written)
// and either a folded affine+activation epilogue (eval) or raw output + per-channel batch
// statistics (training).  Reference semantics: torchvision ConvNormActivation as used at
// models/mn/model.py:125-133 and models/mn/block_types.py:140-170; SqueezeExcitation
// models/mn/block_types.py:72-83.
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "common.cuh"
#include <stdlib.h>

namespace {

constexpr int kThreads = 256;
constexpr bool kPoolV2Default = true;    // eat_bn_act_pool: kernel generation used when EAT_POOL is not set (v2: 0.54 -> 0.45 ms per mn10 step)

// 4 consecutive channels <-> fp32 registers, for either storage type (16 B fp32 / 8 B bf16)
template <typename T> struct Vec4IO;
template <> struct Vec4IO<float> {
  __device__ __forceinline__ static void load(const float* p, float (&v)[4]) { Vec<float>::load(p, v); }
  __device__ __forceinline__ static void store(float* p, const float (&v)[4]) { Vec<float>::store(p, v); }
};
template <> struct Vec4IO<__nv_bfloat16> {
  __device__ __forceinline__ static void load(const __nv_bfloat16* p, float (&v)[4]) {
    uint2 t = *reinterpret_cast<const uint2*>(p);
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&t);
    float2 a = __bfloat1622float2(h[0]), b = __bfloat1622float2(h[1]);
    v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y;
  }
  __device__ __forceinline__ static void store(__nv_bfloat16* p, const float (&v)[4]) {
    uint2 t;
    __nv_bfloat162 a = __floats2bfloat162_rn(v[0], v[1]), b = __floats2bfloat162_rn(v[2], v[3]);
    t.x = *reinterpret_cast<uint32_t*>(&a); t.y = *reinterpret_cast<uint32_t*>(&b);
    *reinterpret_cast<uint2*>(p) = t;
  }
};

// ------------------------------------------------------------------------------------------
// Stem: x [B, F, T] fp32 (one input channel) -> out [B, Fo, To, C] ; 3x3, pad 1, stride s.
template <typename TO>
__global__ void __launch_bounds__(kThreads) stem_kernel(
    const float* __restrict__ x, const float* __restrict__ w /*[C,1,3,3]*/, TO* __restrict__ out,
    int B, int F, int T, int Fo, int To, int C, int stride,
    const float* __restrict__ scale, const float* __restrict__ shift, int act,
    double* __restrict__ stat_sum, double* __restrict__ stat_sq) {
  constexpr int V = Vec<TO>::N;
  extern __shared__ float smem[];
  float* s_w = smem;            // [9][C]
  for (int i = threadIdx.x; i < 9 * C; i += kThreads) { int c = i % C, tap = i / C; s_w[i] = w[c * 9 + tap]; }
  __syncthreads();
  const int cv = C / V;
  const int ppb = kThreads / cv;
  const int cvi = threadIdx.x % cv, slot = threadIdx.x / cv;
  const bool active = slot < ppb;
  const long long npix = (long long)B * Fo * To;
  double lsum[V], lsq[V];      // fp64 from the first term: in fp32, E[x^2] - E[x]^2 cancels when |mean| >> std
#pragma unroll
  for (int i = 0; i < V; ++i) { lsum[i] = 0.0; lsq[i] = 0.0; }
  if (active) {
    // 32-bit index math (the launcher guarantees npix < 2^31): three 64-bit div/mod per pixel cost more than the 9 taps
    const unsigned ppx = (unsigned)To * (unsigned)Fo;
    for (unsigned pix = blockIdx.x * ppb + slot; pix < (unsigned)npix; pix += gridDim.x * ppb) {
      const unsigned b_ = pix / ppx, rem_ = pix - b_ * ppx;
      const int fo = (int)(rem_ / (unsigned)To), to = (int)(rem_ - (rem_ / (unsigned)To) * (unsigned)To), b = (int)b_;
      float acc[V];
#pragma unroll
      for (int i = 0; i < V; ++i) acc[i] = 0.f;
#pragma unroll
      for (int ky = 0; ky < 3; ++ky) {
        int f = fo * stride - 1 + ky;
        if (f < 0 || f >= F) continue;
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) {
          int t = to * stride - 1 + kx;
          if (t < 0 || t >= T) continue;
          float xv = __ldg(x + ((size_t)b * F + f) * T + t);
          const float* wp = s_w + (ky * 3 + kx) * C + cvi * V;
#pragma unroll
          for (int i = 0; i < V; ++i) acc[i] = fmaf(xv, wp[i], acc[i]);
        }
      }
      if (scale != nullptr) {
#pragma unroll
        for (int i = 0; i < V; ++i) acc[i] = act_fwd(fmaf(acc[i], scale[cvi * V + i], shift[cvi * V + i]), act);
      } else {
#pragma unroll
        for (int i = 0; i < V; ++i) { lsum[i] += acc[i]; lsq[i] = fma((double)acc[i], (double)acc[i], lsq[i]); }
      }
      Vec<TO>::store(out + (size_t)pix * C + cvi * V, acc);
    }
  }
  if (stat_sum != nullptr) {
    // the weight table is no longer read: its space holds the CTA's fp64 sums ([2][C] doubles <= [9][C] floats)
    double* d_sum = reinterpret_cast<double*>(smem);
    __syncthreads();
    for (int i = threadIdx.x; i < 2 * C; i += kThreads) d_sum[i] = 0.0;
    __syncthreads();
    if (active) {
#pragma unroll
      for (int i = 0; i < V; ++i) { atomicAdd(&d_sum[cvi * V + i], lsum[i]); atomicAdd(&d_sum[C + cvi * V + i], lsq[i]); }
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += kThreads) {
      atomicAdd(stat_sum + c, d_sum[c]);
      atomicAdd(stat_sq + c, d_sum[C + c]);
    }
  }
}

// Row-oriented stem (fp32 output, C <= 64): a CTA walks output rows (b, fo); a thread owns one channel vector -- its nine
// weight vectors live in registers -- and every (256 / cv)-th output column of the row.  No divisions per pixel, no
// shared-memory weight reads, and U = 4 independent pixels per trip so that their 36 input loads overlap.
template <int S>
__global__ void __launch_bounds__(kThreads) stem_row_kernel(
    const float* __restrict__ x, const float* __restrict__ w /*[C,1,3,3]*/, float* __restrict__ out,
    int B, int F, int T, int Fo, int To, int C,
    const float* __restrict__ scale, const float* __restrict__ shift, int act,
    double* __restrict__ stat_sum, double* __restrict__ stat_sq) {
  constexpr int V = 4, U = 4;
  __shared__ double s_sum[2 * 64];
  for (int i = threadIdx.x; i < 2 * C; i += kThreads) s_sum[i] = 0.0;
  __syncthreads();
  const int cv = C / V;
  const int ppb = kThreads / cv;
  const int cvi = threadIdx.x % cv, slot = threadIdx.x / cv;
  const bool active = slot < ppb;
  float wr[9][V], sc[V], sh[V];
  double lsum[V], lsq[V];      // fp64 from the first term: in fp32, E[x^2] - E[x]^2 cancels when |mean| >> std
#pragma unroll
  for (int q = 0; q < 9; ++q)
#pragma unroll
    for (int i = 0; i < V; ++i) wr[q][i] = w[(cvi * V + i) * 9 + q];
#pragma unroll
  for (int i = 0; i < V; ++i) {
    sc[i] = scale != nullptr ? scale[cvi * V + i] : 1.f;
    sh[i] = scale != nullptr ? shift[cvi * V + i] : 0.f;
    lsum[i] = 0.0; lsq[i] = 0.0;
  }
  const int rows = B * Fo;
  if (active) {
    for (int row = blockIdx.x; row < rows; row += gridDim.x) {
      const int b = row / Fo, fo = row - b * Fo;
      const float* xb = x + (size_t)b * F * T;
      float* orow = out + (size_t)row * To * C + cvi * V;
      const int f0 = fo * S - 1;
      for (int to0 = slot; to0 < To; to0 += U * ppb) {
        float xv[U][9];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int to = to0 + u * ppb, t0 = to * S - 1;
#pragma unroll
          for (int ky = 0; ky < 3; ++ky) {
            const int f = f0 + ky;
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) {
              const int t = t0 + kx;
              xv[u][ky * 3 + kx] = (to < To && f >= 0 && f < F && t >= 0 && t < T) ? __ldg(xb + (size_t)f * T + t) : 0.f;
            }
          }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int to = to0 + u * ppb;
          if (to >= To) break;
          float acc[V] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
          for (int q = 0; q < 9; ++q)
#pragma unroll
            for (int i = 0; i < V; ++i) acc[i] = fmaf(xv[u][q], wr[q][i], acc[i]);
          if (scale != nullptr) {
#pragma unroll
            for (int i = 0; i < V; ++i) acc[i] = act_fwd(fmaf(acc[i], sc[i], sh[i]), act);
          } else {
#pragma unroll
            for (int i = 0; i < V; ++i) { lsum[i] += acc[i]; lsq[i] = fma((double)acc[i], (double)acc[i], lsq[i]); }
          }
          *reinterpret_cast<float4*>(orow + (size_t)to * C) = make_float4(acc[0], acc[1], acc[2], acc[3]);
        }
      }
    }
  }
  if (stat_sum != nullptr) {
    if (active) {
#pragma unroll
      for (int i = 0; i < V; ++i) { atomicAdd(&s_sum[cvi * V + i], lsum[i]); atomicAdd(&s_sum[C + cvi * V + i], lsq[i]); }
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += kThreads) {
      atomicAdd(stat_sum + c, s_sum[c]);
      atomicAdd(stat_sq + c, s_sum[C + c]);
    }
  }
}

// ------------------------------------------------------------------------------------------
// Depthwise k x k conv, pad (k-1)/2, stride S.  in [B, F, T, C] -> out [B, Fo, To, C].
// wt: repacked weights [k*k][C] (flip != 0 reads them mirrored: the stride-1 data gradient is the same convolution
// with the kernel flipped).  grid = (chunks x tile groups, B): per-(sample, channel) pooling stays inside a CTA column.
// All 3x3 cases and the 5x5 training forward run in the register sliding-window kernel (dw_slide.cu); the kernel below
// serves the 5x5 eval (squeeze-excitation pooling / DyMN epilogue) and wide 5x5 stride-1 data-gradient cases.
// MODE 0: training forward (optional input BN+act, raw output + batch statistics)
// MODE 1: eval forward (folded BN + act epilogue, SE pooling, DyMN epilogue)     MODE 2: stride-1 data gradient
// ------------------------------------------------------------------------------------------
// Shared-memory tiled depthwise convolution.  A CTA stages an input tile
// ((FR-1)*S+K rows x (TT-1)*S+K columns x 32 channels) in shared memory as fp32, applying the producing layer's
// BatchNorm + activation ONCE per element, then
// every thread computes a strip of P outputs for one 4-channel vector from shared memory (LDS.128).
// DM: DyReLU-B pieces of the MODE 1 DyMN epilogue (DyCoef, common.cuh).  The 2 DM coefficients per channel vector stay
// in registers: DM = 2 at 3 CTAs per SM, DM = 1 at 2, DM = 3, 4 at one (no spills; DESIGN.md section 4)
template <typename T, int K, int S, int MODE, int DM = 2>
__global__ void __launch_bounds__(kThreads, DM == 2 ? 3 : (DM == 1 ? 2 : 1)) dw_tile_kernel(
    const T* __restrict__ in, const float* __restrict__ wt, T* __restrict__ out,
    int F, int Tn, int Fo, int To, int C, InXform xf,
    const float* __restrict__ scale, const float* __restrict__ shift, int act, const T* __restrict__ res, int flip,
    float* __restrict__ pool, double* __restrict__ stat_sum, double* __restrict__ stat_sq, DyEpi dy) {
  constexpr bool kAff = MODE == 1, kStats = MODE == 0, kXf = MODE == 0, kRes = MODE == 2, kDy = MODE == 1, kPool = MODE == 1;
  static_assert(DM >= 1 && DM <= 4 && (DM == 2 || MODE == 1), "DyReLU-B pieces: 1..4, eval epilogue only");
  constexpr int VG = Vec<T>::N;                 // channels per 16-byte global vector
  constexpr int CC = 32;                        // channels per tile
  constexpr int CCV = CC / 4;
  constexpr int FR = (S == 1) ? 8 : 4;
  constexpr int TT = (S == 1) ? 32 : 16;
  constexpr int P = (S == 1) ? 8 : 2;
  constexpr int SPR = TT / P;
  constexpr int IR = (FR - 1) * S + K, IT = (TT - 1) * S + K;
  constexpr int NIN = (P - 1) * S + K;
  constexpr int PAD = (K - 1) / 2;
  constexpr int ITEMS = FR * SPR * CCV;
  static_assert(ITEMS % kThreads == 0 || ITEMS < kThreads || true, "");
  extern __shared__ __align__(16) float smem[];
  float* s_in = smem;                           // [IR*IT][CC]
  float* s_w = s_in + IR * IT * CC;             // [K*K][CC]
  float* s_sum = s_w + K * K * CC;              // [CC]
  float* s_sq = s_sum + CC;                     // [CC]
  const int b = blockIdx.y;
  const int tiles_t = ceil_div(To, TT), tiles_f = ceil_div(Fo, FR), chunks = ceil_div(C, CC);
  const int tiles_per_chunk = tiles_t * tiles_f;
  const bool need_red = (kPool && pool != nullptr) || (kStats && stat_sum != nullptr);
  const T* inb = in + (size_t)b * F * Tn * C;
  T* outb = out + (size_t)b * Fo * To * C;
  const T* resb = (kRes && res != nullptr) ? res + (size_t)b * Fo * To * C : nullptr;
  wt += (size_t)b * dy.wt_bstride;
  const int tid = threadIdx.x;
  // blockIdx.x enumerates (channel chunk, tile group); each CTA walks its tile group with a stride
  const int groups = gridDim.x / chunks;        // CTAs per channel chunk
  const int chunk = blockIdx.x / groups, grp = blockIdx.x - chunk * groups;
  if (chunk >= chunks) return;
  const int cbase = chunk * CC;
  const int ccv_valid = min(CC, C - cbase) / 4; // valid 4-channel vectors in this chunk
  // ---- weights + reduction scratch
  for (int i = tid; i < K * K * CC; i += kThreads) {
    const int tap = i / CC, c = i % CC;
    const int src = flip ? (K * K - 1 - tap) : tap;
    s_w[i] = (cbase + c < C) ? __ldg(wt + (size_t)src * C + cbase + c) : 0.f;
  }
  if (tid < 2 * CC) s_sum[tid] = 0.f;
  // loader mapping: VPP 16-byte vectors per pixel
  constexpr int VPP = CC / VG;
  const int lv = tid % VPP;                     // this thread's vector slot inside a pixel (fixed)
  const int lc0 = cbase + lv * VG;              // first channel of that vector
  const bool lvalid = lc0 < C;
  float isc[VG], ish[VG];
  if (kXf && xf.scale != nullptr && lvalid) {
#pragma unroll
    for (int i = 0; i < VG; ++i) { isc[i] = xf.scale[lc0 + i]; ish[i] = xf.shift[lc0 + i]; }
  }
  // compute mapping
  const int cvec = tid % CCV;
  const int c0 = cbase + cvec * 4;
  const bool cvalid = cvec < ccv_valid;
  float osc[4], osh[4], lsum[4] = {0.f, 0.f, 0.f, 0.f}, lsq[4] = {0.f, 0.f, 0.f, 0.f};
  DyCoef<DM> dyc[4];
  if (cvalid) {
    if (kAff && scale != nullptr) {
#pragma unroll
      for (int i = 0; i < 4; ++i) { osc[i] = scale[c0 + i]; osh[i] = shift[c0 + i]; }
    }
    if (kDy && dy.theta != nullptr) {
#pragma unroll
      for (int i = 0; i < 4; ++i) dyc[i].load(dy.theta + ((size_t)b * C + c0 + i) * (2 * DM), dy.lam, dy.init, true);
    }
  }
  for (int tile = grp; tile < tiles_per_chunk; tile += groups) {
    const int tf = tile / tiles_t, tt = tile - tf * tiles_t;
    const int f0 = tf * FR, t0 = tt * TT;
    __syncthreads();                            // previous tile's readers are done (also covers the init above)
    // ---- stage the input tile (transform once)
    for (int idx = tid; idx < IR * IT * VPP; idx += kThreads) {
      const int pix = idx / VPP;
      const int ir = pix / IT, it = pix - ir * IT;
      const int f = f0 * S - PAD + ir, t = t0 * S - PAD + it;
      float v[VG];
      if (lvalid && f >= 0 && f < F && t >= 0 && t < Tn) {
        Vec<T>::load(inb + ((size_t)f * Tn + t) * C + lc0, v);
        if (kXf && xf.scale != nullptr) {
#pragma unroll
          for (int i = 0; i < VG; ++i) v[i] = act_fwd(fmaf(v[i], isc[i], ish[i]), xf.act);
        }
      } else {
#pragma unroll
        for (int i = 0; i < VG; ++i) v[i] = 0.f;
      }
      float* dst = s_in + (size_t)pix * CC + lv * VG;
#pragma unroll
      for (int q = 0; q < VG / 4; ++q)
        *reinterpret_cast<float4*>(dst + 4 * q) = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
    }
    __syncthreads();
    // ---- compute
    if (cvalid) {
      for (int item = tid; item < ITEMS; item += kThreads) {
        const int strip = item / CCV;
        const int fl = strip / SPR, ts = strip - fl * SPR;
        const int fo = f0 + fl, to0 = t0 + ts * P;
        if (fo >= Fo || to0 >= To) continue;
        float acc[P][4];
#pragma unroll
        for (int p = 0; p < P; ++p) { acc[p][0] = acc[p][1] = acc[p][2] = acc[p][3] = 0.f; }
#pragma unroll
        for (int ky = 0; ky < K; ++ky) {
          float4 w4[K];
#pragma unroll
          for (int kx = 0; kx < K; ++kx) w4[kx] = *reinterpret_cast<const float4*>(s_w + (ky * K + kx) * CC + cvec * 4);
          const float* rowp = s_in + ((size_t)(fl * S + ky) * IT + ts * P * S) * CC + cvec * 4;
#pragma unroll
          for (int ix = 0; ix < NIN; ++ix) {
            const float4 v = *reinterpret_cast<const float4*>(rowp + (size_t)ix * CC);
#pragma unroll
            for (int p = 0; p < P; ++p) {
              const int kx = ix - p * S;
              if (kx >= 0 && kx < K) {
                acc[p][0] = fmaf(v.x, w4[kx].x, acc[p][0]);
                acc[p][1] = fmaf(v.y, w4[kx].y, acc[p][1]);
                acc[p][2] = fmaf(v.z, w4[kx].z, acc[p][2]);
                acc[p][3] = fmaf(v.w, w4[kx].w, acc[p][3]);
              }
            }
          }
        }
#pragma unroll
        for (int p = 0; p < P; ++p) {
          const int to = to0 + p;
          if (to >= To) break;
          float o[4];
          if (kAff && scale != nullptr) {
#pragma unroll
            for (int i = 0; i < 4; ++i) { o[i] = act_fwd(fmaf(acc[p][i], osc[i], osh[i]), act); lsum[i] += o[i]; }
          } else {
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              o[i] = acc[p][i];
              if (kStats) { lsum[i] += o[i]; lsq[i] = fmaf(o[i], o[i], lsq[i]); }
            }
          }
          if (kDy && dy.theta != nullptr) {
#pragma unroll
            for (int i = 0; i < 4; ++i) o[i] = dyc[i].apply(o[i]);
          }
          if (kDy && dy.ca_f != nullptr) {
            const float4 f4 = __ldg(reinterpret_cast<const float4*>(dy.ca_f + ((size_t)b * Fo + fo) * C + c0));
            const float4 t4 = __ldg(reinterpret_cast<const float4*>(dy.ca_t + ((size_t)b * To + to) * C + c0));
            o[0] *= f4.x * t4.x; o[1] *= f4.y * t4.y; o[2] *= f4.z * t4.z; o[3] *= f4.w * t4.w;
          }
          const size_t off = ((size_t)fo * To + to) * C + c0;
          if (resb != nullptr) {
            float r[4];
            Vec4IO<T>::load(resb + off, r);
#pragma unroll
            for (int i = 0; i < 4; ++i) o[i] += r[i];
          }
          Vec4IO<T>::store(outb + off, o);
        }
      }
    }
  }
  if (need_red) {
    if (cvalid) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        atomicAdd(&s_sum[cvec * 4 + i], lsum[i]);
        if (kStats && stat_sum != nullptr) atomicAdd(&s_sq[cvec * 4 + i], lsq[i]);
      }
    }
    __syncthreads();
    if (tid < CC && cbase + tid < C) {
      if (kPool && pool != nullptr) atomicAdd(pool + (size_t)b * C + cbase + tid, s_sum[tid]);
      if (kStats && stat_sum != nullptr) { atomicAdd(stat_sum + cbase + tid, (double)s_sum[tid]); atomicAdd(stat_sq + cbase + tid, (double)s_sq[tid]); }
    }
  }
}

// [C,1,k,k] -> [k*k][C]
__global__ void dw_repack_kernel(const float* __restrict__ w, float* __restrict__ wt, int C, int kk) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < C * kk) { int c = i / kk, tap = i % kk; wt[(size_t)tap * C + c] = w[i]; }
}

// ------------------------------------------------------------------------------------------
// BatchNorm helpers
__global__ void bn_fold_kernel(const float* __restrict__ gamma, const float* __restrict__ beta,
                               const float* __restrict__ rmean, const float* __restrict__ rvar, float eps,
                               float* __restrict__ scale, float* __restrict__ shift, int C) {
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < C) {
    float s = gamma[c] / sqrtf(rvar[c] + eps);
    scale[c] = s;
    shift[c] = beta[c] - rmean[c] * s;
  }
}

// training: batch statistics -> scale/shift (+ saved mean / invstd), running-stat update
// (nn.BatchNorm2d: running = (1-m) running + m batch, unbiased variance for the running buffer)
__global__ void bn_finalize_kernel(const double* __restrict__ sum, const double* __restrict__ sq, double count,
                                   const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                   float momentum, float* __restrict__ rmean, float* __restrict__ rvar,
                                   long long* __restrict__ nbt, float* __restrict__ scale,
                                   float* __restrict__ shift, float* __restrict__ save_mean,
                                   float* __restrict__ save_invstd, int C) {
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < C) {
    double mean = sum[c] / count;
    double var = sq[c] / count - mean * mean;
    if (var < 0.0) var = 0.0;
    float invstd = (float)(1.0 / sqrt(var + (double)eps));
    float s = gamma[c] * invstd;
    scale[c] = s;
    shift[c] = beta[c] - (float)mean * s;
    save_mean[c] = (float)mean;
    save_invstd[c] = invstd;
    if (rmean != nullptr) {
      double unbiased = count > 1.0 ? var * count / (count - 1.0) : var;
      rmean[c] = (1.f - momentum) * rmean[c] + momentum * (float)mean;
      rvar[c] = (1.f - momentum) * rvar[c] + momentum * (float)unbiased;
    }
  }
  if (nbt != nullptr && blockIdx.x == 0 && threadIdx.x == 0) *nbt += 1;
}

// y = act(z * scale + shift) (+ residual);  elementwise over [rows, C]
template <typename T>
__global__ void __launch_bounds__(kThreads) bn_apply_kernel(const T* __restrict__ z, const float* __restrict__ scale,
                                                            const float* __restrict__ shift, int act,
                                                            const T* __restrict__ res, T* __restrict__ y,
                                                            long long rows, int C) {
  constexpr int V = Vec<T>::N;
  const int cv = C / V;
  const long long nvec = rows * cv;
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < nvec; i += (long long)gridDim.x * kThreads) {
    const int c0 = (int)(i % cv) * V;
    float v[V];
    Vec<T>::load(z + i * V, v);
#pragma unroll
    for (int k = 0; k < V; ++k) v[k] = act_fwd(fmaf(v[k], scale[c0 + k], shift[c0 + k]), act);
    if (res != nullptr) {
      float r[V];
      Vec<T>::load(res + i * V, r);
#pragma unroll
      for (int k = 0; k < V; ++k) v[k] += r[k];
    }
    Vec<T>::store(y + i * V, v);
  }
}

// pool[b, c] += sum_p act(z[b, p, c] * scale[c] + shift[c]);  grid = (chunks, B)
template <typename T>
__global__ void __launch_bounds__(kThreads) bn_act_pool_kernel(const T* __restrict__ z, const float* __restrict__ scale,
                                                               const float* __restrict__ shift, int act,
                                                               float* __restrict__ pool, float mul, int P, int C) {
  constexpr int V = Vec<T>::N;
  extern __shared__ float smem[];
  for (int i = threadIdx.x; i < C; i += kThreads) smem[i] = 0.f;
  __syncthreads();
  const int cv = C / V;
  const int b = blockIdx.y;
  const T* zb = z + (size_t)b * P * C;
  const long long nvec = (long long)P * cv;
  // each thread keeps a fixed channel vector when kThreads % cv == 0 is not guaranteed, so use smem atomics per item
  // but first accumulate privately over a stride that preserves the channel vector: stride = lcm-free trick:
  // iterate pixels for (slot, cvi) pairs as in the conv kernels.
  const int tcv = cv < kThreads ? cv : kThreads;
  const int ppb = kThreads / tcv;
  const int slot = threadIdx.x / tcv;
  if (slot < ppb) {
    for (int cvi = threadIdx.x % tcv; cvi < cv; cvi += tcv) {
      const int c0 = cvi * V;
      float acc[V];
#pragma unroll
      for (int k = 0; k < V; ++k) acc[k] = 0.f;
      for (int p = blockIdx.x * ppb + slot; p < P; p += gridDim.x * ppb) {
        float v[V];
        Vec<T>::load(zb + (size_t)p * C + c0, v);
#pragma unroll
        for (int k = 0; k < V; ++k)
          acc[k] += scale != nullptr ? act_fwd(fmaf(v[k], scale[c0 + k], shift[c0 + k]), act) : v[k];
      }
#pragma unroll
      for (int k = 0; k < V; ++k) atomicAdd(&smem[c0 + k], acc[k]);
    }
  }
  (void)nvec;
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += kThreads) atomicAdd(pool + (size_t)b * C + c, smem[c] * mul);
}

// Second generation (the BatchNorm-backward reduce went the same way): same thread mapping, activation compile-time, the
// two per-channel constants in registers, EIGHT pixels (fp32; four for bf16) = 128 bytes of loads in flight per thread.
template <typename T, int ACT>
__global__ void __launch_bounds__(kThreads, 3) bn_act_pool2_kernel(const T* __restrict__ z, const float* __restrict__ scale,
                                                                   const float* __restrict__ shift,
                                                                   float* __restrict__ pool, float mul, int P, int C) {
  constexpr int V = Vec<T>::N;
  constexpr int U = V == 4 ? 8 : 4;
  extern __shared__ float smem[];
  for (int i = threadIdx.x; i < C; i += kThreads) smem[i] = 0.f;
  __syncthreads();
  const int cv = C / V;
  const int b = blockIdx.y;
  const T* zb = z + (size_t)b * P * C;
  const int tcv = cv < kThreads ? cv : kThreads;
  const int ppb = kThreads / tcv;
  const int slot = threadIdx.x / tcv;
  if (slot < ppb) {
    for (int cvi = threadIdx.x % tcv; cvi < cv; cvi += tcv) {
      const int c0 = cvi * V;
      float sc[V], sh[V], acc[V];
#pragma unroll
      for (int k = 0; k < V; ++k) { sc[k] = scale[c0 + k]; sh[k] = shift[c0 + k]; acc[k] = 0.f; }
      const int step = gridDim.x * ppb;
      int p = blockIdx.x * ppb + slot;
      for (; p + (U - 1) * step < P; p += U * step) {
        float v[U][V];
#pragma unroll
        for (int u = 0; u < U; ++u) Vec<T>::load(zb + (size_t)(p + u * step) * C + c0, v[u]);
#pragma unroll
        for (int u = 0; u < U; ++u)
#pragma unroll
          for (int k = 0; k < V; ++k) acc[k] += act_fwd(fmaf(v[u][k], sc[k], sh[k]), ACT);
      }
      for (; p < P; p += step) {
        float v[V];
        Vec<T>::load(zb + (size_t)p * C + c0, v);
#pragma unroll
        for (int k = 0; k < V; ++k) acc[k] += act_fwd(fmaf(v[k], sc[k], sh[k]), ACT);
      }
#pragma unroll
      for (int k = 0; k < V; ++k) atomicAdd(&smem[c0 + k], acc[k]);
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += kThreads) atomicAdd(pool + (size_t)b * C + c, smem[c] * mul);
}

// ------------------------------------------------------------------------------------------
// Squeeze-excitation MLP: gate[b,:] = sigmoid(W2 relu(W1 (pool[b,:] * inv_count) + b1) + b2)
// one CTA per sample; warp per output row (coalesced weight rows).
__global__ void __launch_bounds__(kThreads) se_fc_kernel(const float* __restrict__ pool, float inv_count,
                                                         const float* __restrict__ w1, const float* __restrict__ b1,
                                                         const float* __restrict__ w2, const float* __restrict__ b2,
                                                         float* __restrict__ gate, float* __restrict__ hidden_out,
                                                         int C, int S) {
  extern __shared__ float smem[];
  float* s_mean = smem;       // [C]
  float* s_hid = smem + C;    // [S]
  const int b = blockIdx.x;
  for (int c = threadIdx.x; c < C; c += kThreads) s_mean[c] = pool[(size_t)b * C + c] * inv_count;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = kThreads / 32;
  for (int s = warp; s < S; s += nwarps) {
    const float* wr = w1 + (size_t)s * C;
    float acc = 0.f;
    for (int c = lane; c < C; c += 32) acc = fmaf(__ldg(wr + c), s_mean[c], acc);
    acc = warp_sum(acc);
    if (lane == 0) {
      float h = fmaxf(acc + b1[s], 0.f);
      s_hid[s] = h;
      if (hidden_out != nullptr) hidden_out[(size_t)b * S + s] = h;
    }
  }
  __syncthreads();
  for (int c = warp; c < C; c += nwarps) {
    const float* wr = w2 + (size_t)c * S;
    float acc = 0.f;
    for (int s = lane; s < S; s += 32) acc = fmaf(__ldg(wr + s), s_hid[s], acc);
    acc = warp_sum(acc);
    if (lane == 0) gate[(size_t)b * C + c] = sigmoidf_(acc + b2[c]);
  }
}

inline int grid_for(long long items, int per_block, int max_blocks = kNumSMs * 16) {
  long long g = ceil_div_ll(items, per_block);
  if (g > max_blocks) g = max_blocks;
  if (g < 1) g = 1;
  return (int)g;
}

}  // namespace

// about six CTAs per SM over all chunks and samples, never more CTAs per chunk than it has tiles
DwTilePlan dw_tile_plan(int B, int Fo, int To, int C, int stride) {
  DwTilePlan pl;
  pl.FR = stride == 1 ? 8 : 4;
  pl.TT = stride == 1 ? 32 : 16;
  pl.chunks = ceil_div(C, 32);
  pl.tiles = ceil_div(Fo, pl.FR) * ceil_div(To, pl.TT);
  pl.groups = max(1, (kNumSMs * 6) / max(B * pl.chunks, 1));
  if (pl.groups > pl.tiles) pl.groups = pl.tiles;
  return pl;
}

namespace {

template <typename T>
int launch_dw(const T* in, const float* wt, T* out, int B, int F, int Tn, int C, int k, int stride, InXform xf,
              const float* scale, const float* shift, int act, const T* res, int flip, float* pool, double* ssum,
              double* ssq, cudaStream_t st, DyEpi dy = DyEpi{nullptr, nullptr, nullptr, nullptr, nullptr, 0}, int dyk = 2) {
  constexpr int V = Vec<T>::N;
  if (C % V != 0) { eat_set_error("dw conv: channels must be a multiple of the vector width"); return EAT_ERR_ARG; }
  const int pad = (k - 1) / 2;
  const int Fo = (F + 2 * pad - k) / stride + 1, To = (Tn + 2 * pad - k) / stride + 1;
  const int mode_ = (scale != nullptr || pool != nullptr || dy.theta != nullptr || dy.ca_f != nullptr) ? 1 : ((flip || res != nullptr) ? 2 : 0);
  // sliding-window kernel (dw_slide.cu) for every 3x3 case and the 5x5 training forward; the 5x5 eval and wide
  // data-gradient cases stay on the shared-memory tile kernel below
  // 5x5 stride-1 data gradient: sliding-window kernel up to 256 channels, tile kernel above
  // (the tile kernel wins on the widest layers); EAT_DW5_DGRAD=slide|tile forces one
  const char* e5 = getenv("EAT_DW5_DGRAD");
  const bool slide5 = e5 != nullptr ? e5[0] == 's' : C <= 256;
  if ((stride == 1 || stride == 2) && (k == 3 || (k == 5 && (mode_ == 0 || (mode_ == 2 && slide5)))) && !(mode_ == 2 && stride != 1))
    return dw_slide_launch(in, wt, out, V == 8 ? EAT_BF16 : EAT_F32, B, F, Tn, C, k, stride, xf, scale, shift, act, res, flip,
                           pool, ssum, ssq, st, dy, dyk);
  if (k != 5) { eat_set_error("dw conv: only k in {3,5}, stride in {1,2}"); return EAT_ERR_UNSUPPORTED; }
  // shared-memory tiled kernel: grid.x = channel chunks x tile groups (each CTA strides over its group's tiles)
  const DwTilePlan pl = dw_tile_plan(B, Fo, To, C, stride);
  const int IR = (pl.FR - 1) * stride + k, IT = (pl.TT - 1) * stride + k;
  dim3 grid(pl.chunks * pl.groups, B);
  size_t smem = ((size_t)IR * IT * 32 + (size_t)k * k * 32 + 64) * sizeof(float);
  const int tmode = (scale != nullptr || pool != nullptr || dy.theta != nullptr || dy.ca_f != nullptr) ? 1 : ((flip || res != nullptr) ? 2 : 0);
#define EAT_DWM(KK, SS, MM, DK)                                                                                 \
  do {                                                                                                          \
    static unsigned long long attr = 0;                                                                         \
    if (int rc = eat_opt_in_smem(dw_tile_kernel<T, KK, SS, MM, DK>, 100 * 1024, attr)) return rc;               \
    dw_tile_kernel<T, KK, SS, MM, DK><<<grid, kThreads, smem, st>>>(in, wt, out, F, Tn, Fo, To, C, xf, scale, shift, act, res, flip, pool, ssum, ssq, dy); \
  } while (0)
  // the eval epilogue's DyReLU-B pieces (dyk, only read when dy.theta is set)
  const int tdk = (tmode == 1 && dy.theta != nullptr) ? dyk : 2;
  if (tdk < 1 || tdk > 4) { eat_set_error("dw conv: DyReLU-B takes 1..4 linear pieces"); return EAT_ERR_UNSUPPORTED; }
#define EAT_DW1(KK, SS)                                                                                         \
  do {                                                                                                          \
    if (tdk == 1) EAT_DWM(KK, SS, 1, 1);                                                                        \
    else if (tdk == 3) EAT_DWM(KK, SS, 1, 3);                                                                   \
    else if (tdk == 4) EAT_DWM(KK, SS, 1, 4);                                                                   \
    else EAT_DWM(KK, SS, 1, 2);                                                                                 \
  } while (0)
#define EAT_DW(KK, SS) do { if (tmode == 0) EAT_DWM(KK, SS, 0, 2); else if (tmode == 1) EAT_DW1(KK, SS); else EAT_DWM(KK, SS, 2, 2); } while (0)
  if (k == 5 && stride == 1) EAT_DW(5, 1);
  else if (k == 5 && stride == 2) EAT_DW(5, 2);
  else { eat_set_error("dw conv: only k in {3,5}, stride in {1,2}"); return EAT_ERR_UNSUPPORTED; }
#undef EAT_DWM
#undef EAT_DW1
#undef EAT_DW
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

}  // namespace

extern "C" {

int eat_stem_fwd(const float* x, const float* w, void* out, int out_dtype, int B, int F, int T, int C, int stride,
                 const float* scale, const float* shift, int act, double* stat_sum, double* stat_sq,
                 cudaStream_t st) {
  const int Fo = (F + 2 - 3) / stride + 1, To = (T + 2 - 3) / stride + 1;
  const int V = out_dtype == EAT_BF16 ? 8 : 4;
  if (C % V != 0 || C / V > kThreads) { eat_set_error("stem: unsupported channel count"); return EAT_ERR_ARG; }
  const long long npix = (long long)B * Fo * To;
  if (npix == 0) return EAT_OK;
  if (npix >= (1ll << 31)) { eat_set_error("stem: B*Fo*To must be below 2^31"); return EAT_ERR_ARG; }
  const int ppb = kThreads / (C / V);
  if (out_dtype == EAT_F32 && C <= 64 && (stride == 1 || stride == 2)) {      // row-oriented kernel (every released width <= 4.0)
    const int rows = B * Fo;
    const int grid_r = rows < kNumSMs * 8 ? rows : kNumSMs * 8;
    if (stride == 2) stem_row_kernel<2><<<grid_r, kThreads, 0, st>>>(x, w, (float*)out, B, F, T, Fo, To, C, scale, shift, act, stat_sum, stat_sq);
    else stem_row_kernel<1><<<grid_r, kThreads, 0, st>>>(x, w, (float*)out, B, F, T, Fo, To, C, scale, shift, act, stat_sum, stat_sq);
    EAT_CHECK_LAUNCH();
    return EAT_OK;
  }
  int grid = grid_for(npix, ppb, kNumSMs * 8);
  size_t smem = (size_t)9 * C * sizeof(float);
  if (out_dtype == EAT_BF16)
    stem_kernel<__nv_bfloat16><<<grid, kThreads, smem, st>>>(x, w, (__nv_bfloat16*)out, B, F, T, Fo, To, C, stride, scale, shift, act, stat_sum, stat_sq);
  else
    stem_kernel<float><<<grid, kThreads, smem, st>>>(x, w, (float*)out, B, F, T, Fo, To, C, stride, scale, shift, act, stat_sum, stat_sq);
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

int eat_dw_repack(const float* w, float* wt, int C, int k, cudaStream_t st) {
  int n = C * k * k;
  dw_repack_kernel<<<ceil_div(n, 256), 256, 0, st>>>(w, wt, C, k * k);
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

int eat_dw_conv_fwd(const void* in, const float* wt, void* out, int dtype, int B, int F, int T, int C, int k,
                    int stride, const float* in_scale, const float* in_shift, int in_act, const float* scale,
                    const float* shift, int act, float* pool, double* stat_sum, double* stat_sq,
                    cudaStream_t st) {
  if (B == 0) return EAT_OK;
  InXform xf{in_scale, in_shift, nullptr, in_act, 0};
  if (dtype == EAT_BF16)
    return launch_dw<__nv_bfloat16>((const __nv_bfloat16*)in, wt, (__nv_bfloat16*)out, B, F, T, C, k, stride, xf, scale, shift, act, nullptr, 0, pool, stat_sum, stat_sq, st);
  return launch_dw<float>((const float*)in, wt, (float*)out, B, F, T, C, k, stride, xf, scale, shift, act, nullptr, 0, pool, stat_sum, stat_sq, st);
}

// DyMN depthwise stage: per-sample weight tables + BN affine + DyReLU-B + coordinate attention in one kernel
int eat_dw_conv_fwd_dy(const void* in, const float* wt, long long wt_bstride, void* out, int dtype, int B, int F, int T,
                       int C, int k, int stride, const float* in_scale, const float* in_shift, int in_act,
                       const float* scale, const float* shift, const float* theta, const float* lam,
                       const float* init, const float* ca_f, const float* ca_t, double* stat_sum, double* stat_sq,
                       cudaStream_t st) {
  if (B == 0) return EAT_OK;
  InXform xf{in_scale, in_shift, nullptr, in_act, 0};
  DyEpi dy{theta, lam, init, ca_f, ca_t, wt_bstride};
  if (dtype == EAT_BF16)
    return launch_dw<__nv_bfloat16>((const __nv_bfloat16*)in, wt, (__nv_bfloat16*)out, B, F, T, C, k, stride, xf, scale, shift, 0, nullptr, 0, nullptr, stat_sum, stat_sq, st, dy);
  return launch_dw<float>((const float*)in, wt, (float*)out, B, F, T, C, k, stride, xf, scale, shift, 0, nullptr, 0, nullptr, stat_sum, stat_sq, st, dy);
}

// eat_dw_conv_fwd_dy with M DyReLU-B pieces: theta [B, C, 2M], lam / init [2M].  Every check comes before any launch.
int eat_dw_conv_fwd_dy_m(const void* in, const float* wt, long long wt_bstride, void* out, int dtype, int B, int F, int T,
                         int C, int k, int stride, const float* in_scale, const float* in_shift, int in_act,
                         const float* scale, const float* shift, const float* theta, const float* lam,
                         const float* init, const float* ca_f, const float* ca_t, int pieces, double* stat_sum,
                         double* stat_sq, cudaStream_t st) {
  char msg[192];
  int rc = EAT_OK;
  const bool eval = scale != nullptr || theta != nullptr || ca_f != nullptr;
  if (dtype != EAT_F32 && dtype != EAT_BF16) { snprintf(msg, sizeof msg, "dw_conv_fwd_dy_m: dtype must be fp32 (0) or bf16 (1)"); rc = EAT_ERR_ARG; }
  else if (B < 0 || F < 1 || T < 1 || C < 1) { snprintf(msg, sizeof msg, "dw_conv_fwd_dy_m: B >= 0 and F, T, C >= 1 required"); rc = EAT_ERR_ARG; }
  else if (pieces < 1 || pieces > 4) {
    snprintf(msg, sizeof msg, "dw_conv_fwd_dy_m: DyReLU-B takes 1..4 linear pieces (got %d)", pieces);
    rc = EAT_ERR_UNSUPPORTED;
  } else if (k != 3 && k != 5) { snprintf(msg, sizeof msg, "dw_conv_fwd_dy_m: k must be 3 or 5 (got %d)", k); rc = EAT_ERR_UNSUPPORTED; }
  else if (stride != 1 && stride != 2) { snprintf(msg, sizeof msg, "dw_conv_fwd_dy_m: stride must be 1 or 2 (got %d)", stride); rc = EAT_ERR_UNSUPPORTED; }
  else if (C % (dtype == EAT_BF16 ? 8 : 4) != 0) {
    snprintf(msg, sizeof msg, "dw_conv_fwd_dy_m: C must be a multiple of %d for %s storage (got %d)", dtype == EAT_BF16 ? 8 : 4,
             dtype == EAT_BF16 ? "bf16" : "fp32", C);
    rc = EAT_ERR_ARG;
  } else if ((scale == nullptr) != (shift == nullptr) || (in_scale == nullptr) != (in_shift == nullptr) ||
             (stat_sum == nullptr) != (stat_sq == nullptr) || (ca_f == nullptr) != (ca_t == nullptr) ||
             (theta == nullptr) != (lam == nullptr) || (theta == nullptr) != (init == nullptr)) {
    snprintf(msg, sizeof msg, "dw_conv_fwd_dy_m: scale/shift, in_scale/in_shift, stat_sum/stat_sq, ca_f/ca_t and "
             "theta/lam/init come in sets");
    rc = EAT_ERR_ARG;
  } else if (eval && (in_scale != nullptr || stat_sum != nullptr)) {
    snprintf(msg, sizeof msg, "dw_conv_fwd_dy_m: the input transform and the statistics are for the training forward "
             "(no scale, theta or ca_f)");
    rc = EAT_ERR_ARG;
  }
  if (rc != EAT_OK) { eat_set_error(msg); return rc; }
  if (B == 0) return EAT_OK;
  InXform xf{in_scale, in_shift, nullptr, in_act, 0};
  DyEpi dy{theta, lam, init, ca_f, ca_t, wt_bstride};
  if (dtype == EAT_BF16)
    return launch_dw<__nv_bfloat16>((const __nv_bfloat16*)in, wt, (__nv_bfloat16*)out, B, F, T, C, k, stride, xf, scale, shift, 0, nullptr, 0, nullptr, stat_sum, stat_sq, st, dy, pieces);
  return launch_dw<float>((const float*)in, wt, (float*)out, B, F, T, C, k, stride, xf, scale, shift, 0, nullptr, 0, nullptr, stat_sum, stat_sq, st, dy, pieces);
}

// stride-1 depthwise data gradient = the forward kernel with mirrored taps (+ residual-gradient add)
int eat_dw_conv_dgrad_s1(const void* dz, const float* wt, long long wt_bstride, const void* res, void* din, int dtype,
                         int B, int F, int T, int C, int k, cudaStream_t st) {
  if (B == 0) return EAT_OK;
  InXform xf{nullptr, nullptr, nullptr, 0, 0};
  DyEpi dy{nullptr, nullptr, nullptr, nullptr, nullptr, wt_bstride};
  if (dtype == EAT_BF16)
    return launch_dw<__nv_bfloat16>((const __nv_bfloat16*)dz, wt, (__nv_bfloat16*)din, B, F, T, C, k, 1, xf, nullptr, nullptr, 0, (const __nv_bfloat16*)res, 1, nullptr, nullptr, nullptr, st, dy);
  return launch_dw<float>((const float*)dz, wt, (float*)din, B, F, T, C, k, 1, xf, nullptr, nullptr, 0, (const float*)res, 1, nullptr, nullptr, nullptr, st, dy);
}

int eat_bn_fold(const float* gamma, const float* beta, const float* rmean, const float* rvar, float eps,
                float* scale, float* shift, int C, cudaStream_t st) {
  bn_fold_kernel<<<ceil_div(C, 128), 128, 0, st>>>(gamma, beta, rmean, rvar, eps, scale, shift, C);
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

int eat_bn_finalize(const double* sum, const double* sq, double count, const float* gamma, const float* beta,
                    float eps, float momentum, float* rmean, float* rvar, long long* nbt, float* scale,
                    float* shift, float* save_mean, float* save_invstd, int C, cudaStream_t st) {
  bn_finalize_kernel<<<ceil_div(C, 128), 128, 0, st>>>(sum, sq, count, gamma, beta, eps, momentum, rmean, rvar, nbt,
                                                        scale, shift, save_mean, save_invstd, C);
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

int eat_bn_apply(const void* z, const float* scale, const float* shift, int act, const void* res, void* y,
                 int dtype, long long rows, int C, cudaStream_t st) {
  if (rows == 0) return EAT_OK;
  const int V = dtype == EAT_BF16 ? 8 : 4;
  if (C % V != 0) { eat_set_error("bn_apply: channels must be a multiple of the vector width"); return EAT_ERR_ARG; }
  int grid = grid_for(rows * (C / V), kThreads * 4);
  if (dtype == EAT_BF16)
    bn_apply_kernel<__nv_bfloat16><<<grid, kThreads, 0, st>>>((const __nv_bfloat16*)z, scale, shift, act, (const __nv_bfloat16*)res, (__nv_bfloat16*)y, rows, C);
  else
    bn_apply_kernel<float><<<grid, kThreads, 0, st>>>((const float*)z, scale, shift, act, (const float*)res, (float*)y, rows, C);
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

int eat_bn_act_pool(const void* z, const float* scale, const float* shift, int act, float* pool, float mul,
                    int dtype, int B, int P, int C, cudaStream_t st) {
  if (B == 0) return EAT_OK;
  const int V = dtype == EAT_BF16 ? 8 : 4;
  if (C % V != 0) { eat_set_error("bn_act_pool: channels must be a multiple of the vector width"); return EAT_ERR_ARG; }
  const int cv = C / V;
  const int tcv = cv < kThreads ? cv : kThreads;
  const int ppb = kThreads / tcv;
  int gx = ceil_div(P, ppb * 8);
  const int cap = max(1, (kNumSMs * 8) / B);
  if (gx > cap) gx = cap;
  if (gx < 1) gx = 1;
  dim3 grid(gx, B);
  size_t smem = (size_t)C * sizeof(float);
  // EAT_POOL=v2|v1 selects the kernel generation (v2: eight pixels in flight, compile-time activation)
  static const bool v2 = [] { const char* e = getenv("EAT_POOL"); return e != nullptr ? strcmp(e, "v2") == 0 : kPoolV2Default; }();
  if (v2 && scale != nullptr && shift != nullptr && (act == EAT_ACT_NONE || act == EAT_ACT_RELU || act == EAT_ACT_HSWISH)) {
    // more pixels per thread in flight: fewer, longer-lived CTAs (~12 per SM over the batch)
    const int U = dtype == EAT_BF16 ? 4 : 8;
    int g2 = ceil_div(P, ppb * U);
    const int cap2 = max(1, (kNumSMs * 12) / B);
    if (g2 > cap2) g2 = cap2;
    if (g2 < 1) g2 = 1;
    dim3 grid2(g2, B);
#define EAT_POOL2(TT, ACT) bn_act_pool2_kernel<TT, ACT><<<grid2, kThreads, smem, st>>>((const TT*)z, scale, shift, pool, mul, P, C)
#define EAT_POOL2_T(TT) do { if (act == EAT_ACT_RELU) EAT_POOL2(TT, EAT_ACT_RELU); else if (act == EAT_ACT_HSWISH) EAT_POOL2(TT, EAT_ACT_HSWISH); \
                             else EAT_POOL2(TT, EAT_ACT_NONE); } while (0)
    if (dtype == EAT_BF16) EAT_POOL2_T(__nv_bfloat16); else EAT_POOL2_T(float);
#undef EAT_POOL2_T
#undef EAT_POOL2
    EAT_CHECK_LAUNCH();
    return EAT_OK;
  }
  if (dtype == EAT_BF16)
    bn_act_pool_kernel<__nv_bfloat16><<<grid, kThreads, smem, st>>>((const __nv_bfloat16*)z, scale, shift, act, pool, mul, P, C);
  else
    bn_act_pool_kernel<float><<<grid, kThreads, smem, st>>>((const float*)z, scale, shift, act, pool, mul, P, C);
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

int eat_se_fc_fwd(const float* pool, float inv_count, const float* w1, const float* b1, const float* w2,
                  const float* b2, float* gate, float* hidden_out, int B, int C, int S, cudaStream_t st) {
  if (B == 0) return EAT_OK;
  size_t smem = (size_t)(C + S) * sizeof(float);
  se_fc_kernel<<<B, kThreads, smem, st>>>(pool, inv_count, w1, b1, w2, b2, gate, hidden_out, C, S);
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

}  // extern "C"
