// Backward-pass kernels of the MobileNetV3 path (training step, reference ex_audioset.py:197
// `loss.backward()` over models/mn/block_types.py:177-181 and models/mn/model.py:212-231).
// BatchNorm backward is two passes over (upstream grad, saved raw conv output):
//   reduce : s1[c] = sum dy, s2[c] = sum dy * xhat      with dy = g * act'(BN(z))
//   apply  : dz = gamma*invstd * (dy - s1/M - xhat * s2/M)
// where the upstream gradient may be composed on the fly, g = gA * gate[b,c] + dpool[b,c]
// (squeeze-excitation gate and the gradient of a spatial mean), so those products are never stored.
#include <cstdlib>
#include <cstring>

#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr bool kBnApplyV2Default = true;    // eat_bn_bwd_apply: kernel generation used when EAT_BN_APPLY is not set (v2: 6.19 -> 5.42 ms per mn10 step)

struct BnCtx {
  const float* scale;   // gamma * invstd      [C]
  const float* shift;   // beta - mean * scale [C]
  const float* mean;    // [C]
  const float* invstd;  // [C]
  int act;
};

template <typename T>
__global__ void __launch_bounds__(kThreads) bn_bwd_reduce_kernel(
    const T* __restrict__ gA, const float* __restrict__ gate, const float* __restrict__ dpool,
    const T* __restrict__ z, BnCtx bn, int B, int P, int C, double* __restrict__ s1, double* __restrict__ s2) {
  constexpr int V = Vec<T>::N;
  extern __shared__ float smem[];   // [2][C]
  for (int i = threadIdx.x; i < 2 * C; i += kThreads) smem[i] = 0.f;
  __syncthreads();
  const int cv = C / V;
  const int tcv = cv < kThreads ? cv : kThreads;
  const int ppb = kThreads / tcv;
  const int slot = threadIdx.x / tcv;
  const int b = blockIdx.y;
  if (slot < ppb) {
    for (int cvi = threadIdx.x % tcv; cvi < cv; cvi += tcv) {
      const int c0 = cvi * V;
      float sc[V], sh[V], mu[V], is[V], gt[V], dp[V], a1[V], a2[V];
#pragma unroll
      for (int k = 0; k < V; ++k) {
        sc[k] = bn.scale[c0 + k]; sh[k] = bn.shift[c0 + k]; mu[k] = bn.mean[c0 + k]; is[k] = bn.invstd[c0 + k];
        gt[k] = gate != nullptr ? gate[(size_t)b * C + c0 + k] : 1.f;
        dp[k] = dpool != nullptr ? dpool[(size_t)b * C + c0 + k] : 0.f;
        a1[k] = 0.f; a2[k] = 0.f;
      }
      auto one = [&](const float (&zv)[V], const float (&gv)[V]) {
#pragma unroll
        for (int k = 0; k < V; ++k) {
          float g = (gA != nullptr ? gv[k] * gt[k] : 0.f) + dp[k];
          float dy = g * act_bwd(fmaf(zv[k], sc[k], sh[k]), bn.act);
          a1[k] += dy;
          a2[k] = fmaf(dy, (zv[k] - mu[k]) * is[k], a2[k]);
        }
      };
      const size_t base = (size_t)b * P * C + c0;
      const int step = gridDim.x * ppb;
      int p = blockIdx.x * ppb + slot;
      for (; p + step < P; p += 2 * step) {          // two pixels per trip: four loads in flight before the math
        const size_t o0 = base + (size_t)p * C, o1 = base + (size_t)(p + step) * C;
        float z0[V], z1[V], g0[V], g1[V];
        Vec<T>::load(z + o0, z0);
        Vec<T>::load(z + o1, z1);
        if (gA != nullptr) { Vec<T>::load(gA + o0, g0); Vec<T>::load(gA + o1, g1); }
        one(z0, g0);
        one(z1, g1);
      }
      if (p < P) {
        const size_t o0 = base + (size_t)p * C;
        float z0[V], g0[V];
        Vec<T>::load(z + o0, z0);
        if (gA != nullptr) Vec<T>::load(gA + o0, g0);
        one(z0, g0);
      }
#pragma unroll
      for (int k = 0; k < V; ++k) { atomicAdd(&smem[c0 + k], a1[k]); atomicAdd(&smem[C + c0 + k], a2[k]); }
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += kThreads) {
    atomicAdd(s1 + c, (double)smem[c]);
    atomicAdd(s2 + c, (double)smem[C + c]);
  }
}

// Second generation of the reduce pass.  Same thread mapping (a thread owns one channel vector and strides over the
// pixels of one sample) but: the activation and the composition of the upstream gradient are compile-time (ACT, GM),
// only three per-channel constants live in the loop (invstd is applied once at the end), and FOUR pixels = eight
// 16-byte loads are in flight per thread before the first use (the v1 kernel was latency bound at 33 % occupancy).
// GM: 0 g = gA;  1 g = gA * gate[b,c] + dpool[b,c] (either may be absent);  2 g = dpool[b,c] only (no gA tensor).
template <typename T, int ACT, int GM>
__global__ void __launch_bounds__(kThreads, 3) bn_bwd_reduce2_kernel(
    const T* __restrict__ gA, const float* __restrict__ gate, const float* __restrict__ dpool,
    const T* __restrict__ z, BnCtx bn, int B, int P, int C, double* __restrict__ s1, double* __restrict__ s2) {
  constexpr int V = Vec<T>::N;
  constexpr int U = V == 4 ? 4 : 2;  // pixels per trip (64 bytes of loads per tensor in flight either way)
  extern __shared__ float smem[];   // [2][C]
  for (int i = threadIdx.x; i < 2 * C; i += kThreads) smem[i] = 0.f;
  __syncthreads();
  const int cv = C / V;
  const int tcv = cv < kThreads ? cv : kThreads;
  const int ppb = kThreads / tcv;
  const int slot = threadIdx.x / tcv;
  const int b = blockIdx.y;
  if (slot < ppb) {
    for (int cvi = threadIdx.x % tcv; cvi < cv; cvi += tcv) {
      const int c0 = cvi * V;
      float sc[V], sh[V], mu[V], gt[V], dp[V], a1[V], a2[V];
#pragma unroll
      for (int k = 0; k < V; ++k) {
        sc[k] = bn.scale[c0 + k]; sh[k] = bn.shift[c0 + k]; mu[k] = bn.mean[c0 + k];
        gt[k] = (GM == 1 && gate != nullptr) ? gate[(size_t)b * C + c0 + k] : 1.f;
        dp[k] = (GM != 0 && dpool != nullptr) ? dpool[(size_t)b * C + c0 + k] : 0.f;
        a1[k] = 0.f; a2[k] = 0.f;
      }
      auto one = [&](const float (&zv)[V], const float (&gv)[V]) {
#pragma unroll
        for (int k = 0; k < V; ++k) {
          float g = GM == 0 ? gv[k] : (GM == 1 ? fmaf(gv[k], gt[k], dp[k]) : dp[k]);
          if (ACT != EAT_ACT_NONE) g *= act_bwd(fmaf(zv[k], sc[k], sh[k]), ACT);
          a1[k] += g;
          a2[k] = fmaf(g, zv[k] - mu[k], a2[k]);
        }
      };
      const size_t base = (size_t)b * P * C + c0;
      const int step = gridDim.x * ppb;
      int p = blockIdx.x * ppb + slot;
      for (; p + (U - 1) * step < P; p += U * step) {
        float zz[U][V], gg[U][V];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const size_t o = base + (size_t)(p + u * step) * C;
          Vec<T>::load(z + o, zz[u]);
          if (GM != 2) Vec<T>::load(gA + o, gg[u]);
        }
#pragma unroll
        for (int u = 0; u < U; ++u) one(zz[u], gg[u]);
      }
      for (; p < P; p += step) {
        const size_t o = base + (size_t)p * C;
        float z0[V], g0[V];
        Vec<T>::load(z + o, z0);
        if (GM != 2) Vec<T>::load(gA + o, g0);
        one(z0, g0);
      }
#pragma unroll
      for (int k = 0; k < V; ++k) { atomicAdd(&smem[c0 + k], a1[k]); atomicAdd(&smem[C + c0 + k], a2[k] * bn.invstd[c0 + k]); }
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += kThreads) {
    atomicAdd(s1 + c, (double)smem[c]);
    atomicAdd(s2 + c, (double)smem[C + c]);
  }
}

// dgamma += s2, dbeta += s1, coef = (s1/M, s2/M)
__global__ void bn_bwd_finalize_kernel(const double* __restrict__ s1, const double* __restrict__ s2, double count,
                                       float* __restrict__ dgamma, float* __restrict__ dbeta,
                                       float* __restrict__ c1, float* __restrict__ c2, int C) {
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < C) {
    if (dgamma != nullptr) dgamma[c] += (float)s2[c];
    if (dbeta != nullptr) dbeta[c] += (float)s1[c];
    c1[c] = (float)(s1[c] / count);
    c2[c] = (float)(s2[c] / count);
  }
}

// pass 2: dz = scale * (dy - c1 - xhat * c2).  A thread keeps one channel vector (its BatchNorm constants live in
// registers) and walks the pixels of one sample two at a time (both pixels' loads in flight before the math).
template <typename T>
__global__ void __launch_bounds__(kThreads) bn_bwd_apply_kernel(
    const T* __restrict__ gA, const float* __restrict__ gate, const float* __restrict__ dpool,
    const T* __restrict__ z, BnCtx bn, const float* __restrict__ c1, const float* __restrict__ c2,
    T* __restrict__ dz, int B, int P, int C) {
  constexpr int V = Vec<T>::N;
  const int cv = C / V;
  const int tcv = cv < kThreads ? cv : kThreads;
  const int ppb = kThreads / tcv;
  const int slot = threadIdx.x / tcv;
  const int b = blockIdx.y;
  if (slot >= ppb) return;
  for (int cvi = threadIdx.x % tcv; cvi < cv; cvi += tcv) {
    const int c0 = cvi * V;
    float sc[V], sh[V], mu[V], is[V], k1[V], k2[V], gt[V], dp[V];
#pragma unroll
    for (int k = 0; k < V; ++k) {
      const int c = c0 + k;
      sc[k] = bn.scale[c]; sh[k] = bn.shift[c]; mu[k] = bn.mean[c]; is[k] = bn.invstd[c];
      k1[k] = c1[c]; k2[k] = c2[c];
      gt[k] = gate != nullptr ? gate[(size_t)b * C + c] : 1.f;
      dp[k] = dpool != nullptr ? dpool[(size_t)b * C + c] : 0.f;
    }
    const size_t base = (size_t)b * P * C + c0;
    const int step = gridDim.x * ppb;
    auto one = [&](const float (&zv)[V], const float (&gv)[V], size_t off) {
      float o[V];
#pragma unroll
      for (int k = 0; k < V; ++k) {
        const float g = (gA != nullptr ? gv[k] * gt[k] : 0.f) + dp[k];
        const float dy = g * act_bwd(fmaf(zv[k], sc[k], sh[k]), bn.act);
        const float xhat = (zv[k] - mu[k]) * is[k];
        o[k] = sc[k] * (dy - k1[k] - xhat * k2[k]);
      }
      Vec<T>::store(dz + off, o);
    };
    int p = blockIdx.x * ppb + slot;
    for (; p + step < P; p += 2 * step) {
      const size_t o0 = base + (size_t)p * C, o1 = base + (size_t)(p + step) * C;
      float z0[V], z1[V], g0[V], g1[V];
      Vec<T>::load(z + o0, z0);
      Vec<T>::load(z + o1, z1);
      if (gA != nullptr) { Vec<T>::load(gA + o0, g0); Vec<T>::load(gA + o1, g1); }
      one(z0, g0, o0);
      one(z1, g1, o1);
    }
    if (p < P) {
      const size_t o0 = base + (size_t)p * C;
      float z0[V], g0[V];
      Vec<T>::load(z + o0, z0);
      if (gA != nullptr) Vec<T>::load(gA + o0, g0);
      one(z0, g0, o0);
    }
  }
}

// Second generation of the apply pass (as bn_bwd_reduce2_kernel for the reduce): activation and gradient composition are
// compile-time (ACT, GM: 0 g = gA; 1 g = gA * gate + dpool; 2 g = dpool), the per-channel constants are folded into four
//   dz = scale * (dy - c1 - xhat * c2) = scale * dy + alpha * z + beta,   alpha = -scale*c2*invstd,  beta = -scale*c1 - alpha*mean
// and FOUR pixels (two for bf16) = eight 16-byte loads are in flight per thread before the first use.
template <typename T, int ACT, int GM>
__global__ void __launch_bounds__(kThreads, 3) bn_bwd_apply2_kernel(
    const T* __restrict__ gA, const float* __restrict__ gate, const float* __restrict__ dpool,
    const T* __restrict__ z, BnCtx bn, const float* __restrict__ c1, const float* __restrict__ c2,
    T* __restrict__ dz, int B, int P, int C) {
  constexpr int V = Vec<T>::N;
  constexpr int U = V == 4 ? 4 : 2;
  const int cv = C / V;
  const int tcv = cv < kThreads ? cv : kThreads;
  const int ppb = kThreads / tcv;
  const int slot = threadIdx.x / tcv;
  const int b = blockIdx.y;
  if (slot >= ppb) return;
  for (int cvi = threadIdx.x % tcv; cvi < cv; cvi += tcv) {
    const int c0 = cvi * V;
    float sc[V], sh[V], al[V], be[V], gt[V], dp[V];
#pragma unroll
    for (int k = 0; k < V; ++k) {
      const int c = c0 + k;
      sc[k] = bn.scale[c]; sh[k] = bn.shift[c];
      al[k] = -sc[k] * c2[c] * bn.invstd[c];
      be[k] = -sc[k] * c1[c] - al[k] * bn.mean[c];
      gt[k] = (GM == 1 && gate != nullptr) ? gate[(size_t)b * C + c] : 1.f;
      dp[k] = (GM != 0 && dpool != nullptr) ? dpool[(size_t)b * C + c] : 0.f;
    }
    const size_t base = (size_t)b * P * C + c0;
    const int step = gridDim.x * ppb;
    auto one = [&](const float (&zv)[V], const float (&gv)[V], size_t off) {
      float o[V];
#pragma unroll
      for (int k = 0; k < V; ++k) {
        float g = GM == 0 ? gv[k] : (GM == 1 ? fmaf(gv[k], gt[k], dp[k]) : dp[k]);
        if (ACT != EAT_ACT_NONE) g *= act_bwd(fmaf(zv[k], sc[k], sh[k]), ACT);
        o[k] = fmaf(sc[k], g, fmaf(al[k], zv[k], be[k]));
      }
      Vec<T>::store(dz + off, o);
    };
    int p = blockIdx.x * ppb + slot;
    for (; p + (U - 1) * step < P; p += U * step) {
      float zz[U][V], gg[U][V];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const size_t o = base + (size_t)(p + u * step) * C;
        Vec<T>::load(z + o, zz[u]);
        if (GM != 2) Vec<T>::load(gA + o, gg[u]);
      }
#pragma unroll
      for (int u = 0; u < U; ++u) one(zz[u], gg[u], base + (size_t)(p + u * step) * C);
    }
    for (; p < P; p += step) {
      const size_t o = base + (size_t)p * C;
      float z0[V], g0[V];
      Vec<T>::load(z + o, z0);
      if (GM != 2) Vec<T>::load(gA + o, g0);
      one(z0, g0, o);
    }
  }
}

// dgate[b,c] += sum_p dp[b,p,c] * act(z[b,p,c] * scale[c] + shift[c])
template <typename T>
__global__ void __launch_bounds__(kThreads) se_bwd_reduce_kernel(const T* __restrict__ dp, const T* __restrict__ z,
                                                                 const float* __restrict__ scale,
                                                                 const float* __restrict__ shift, int act,
                                                                 float* __restrict__ dgate, int P, int C) {
  constexpr int V = Vec<T>::N;
  extern __shared__ float smem[];
  for (int i = threadIdx.x; i < C; i += kThreads) smem[i] = 0.f;
  __syncthreads();
  const int cv = C / V;
  const int tcv = cv < kThreads ? cv : kThreads;
  const int ppb = kThreads / tcv;
  const int slot = threadIdx.x / tcv;
  const int b = blockIdx.y;
  if (slot < ppb) {
    for (int cvi = threadIdx.x % tcv; cvi < cv; cvi += tcv) {
      const int c0 = cvi * V;
      float acc[V];
#pragma unroll
      for (int k = 0; k < V; ++k) acc[k] = 0.f;
      for (int p = blockIdx.x * ppb + slot; p < P; p += gridDim.x * ppb) {
        const size_t off = ((size_t)b * P + p) * C + c0;
        float zv[V], gv[V];
        Vec<T>::load(z + off, zv);
        Vec<T>::load(dp + off, gv);
#pragma unroll
        for (int k = 0; k < V; ++k) acc[k] = fmaf(gv[k], act_fwd(fmaf(zv[k], scale[c0 + k], shift[c0 + k]), act), acc[k]);
      }
#pragma unroll
      for (int k = 0; k < V; ++k) atomicAdd(&smem[c0 + k], acc[k]);
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += kThreads) atomicAdd(dgate + (size_t)b * C + c, smem[c]);
}

// SE block: the squeeze-excitation reduce AND the BatchNorm-backward reduce of the depthwise output in ONE pass over
// (dp, z).  The BatchNorm reduce needs  sum (dp * gate[b,c] + dpool[b,c]) * act'(v) * {1, z - mean}  but dpool is only known
// after the SE MLP backward, which itself needs  dgate = sum_p dp * act(v)  -- so far three passes (dgate, reduce, apply).
// gate and dpool are constant over the pixels of a sample, hence per (b, c)
//   sum_p (dp * gate + dpool) * act' * w  =  gate * sum_p dp * act' * w  +  dpool * sum_p act' * w        (w = 1, z - mean)
// and the four pixel sums can be taken in the same walk that produces dgate; a tiny kernel combines them over the batch
// once dpool exists (se_bn_bwd_combine_kernel).  One read of the two expanded tensors less per SE block.
//   dgate[b,c]          += sum_p dp * act(v)                       (atomics, as se_bwd_reduce_kernel)
//   part[x][0][b][c]     = sum_p dp * act'(v)          part[x][1][b][c] = sum_p dp * act'(v) * (z - mean)
//   part[x][2][b][c]     = sum_p act'(v)               part[x][3][b][c] = sum_p act'(v) * (z - mean)
// x = blockIdx.x (the CTAs of a sample split its pixels; every CTA stores its slice, zeros included: no zero fill needed).
template <typename T, int ACT>
__global__ void __launch_bounds__(kThreads, 2) se_bn_bwd_reduce_kernel(
    const T* __restrict__ dp, const T* __restrict__ z, const float* __restrict__ scale, const float* __restrict__ shift,
    const float* __restrict__ mean, float* __restrict__ dgate, float* __restrict__ part, int B, int P, int C) {
  constexpr int V = Vec<T>::N;
  constexpr int U = V == 4 ? 4 : 2;  // pixels per trip
  extern __shared__ float smem[];    // [5][C], only when several pixel slots of the CTA share a channel vector
  const int cv = C / V;
  const int tcv = cv < kThreads ? cv : kThreads;
  const int ppb = kThreads / tcv;
  const int slot = threadIdx.x / tcv;
  const int b = blockIdx.y;
  const bool shared = ppb > 1;
  if (shared) {
    for (int i = threadIdx.x; i < 5 * C; i += kThreads) smem[i] = 0.f;
    __syncthreads();
  }
  const size_t qs = (size_t)B * C;                                   // stride between the four quantities
  float* const my_part = part + ((size_t)blockIdx.x * 4 * B + b) * C;
  if (slot < ppb) {
    for (int cvi = threadIdx.x % tcv; cvi < cv; cvi += tcv) {
      const int c0 = cvi * V;
      float sc[V], sh[V], mu[V], aD[V], a1[V], a2[V], e1[V], e2[V];
#pragma unroll
      for (int k = 0; k < V; ++k) {
        sc[k] = scale[c0 + k]; sh[k] = shift[c0 + k]; mu[k] = mean[c0 + k];
        aD[k] = 0.f; a1[k] = 0.f; a2[k] = 0.f; e1[k] = 0.f; e2[k] = 0.f;
      }
      auto one = [&](const float (&zv)[V], const float (&gv)[V]) {
#pragma unroll
        for (int k = 0; k < V; ++k) {
          const float v = fmaf(zv[k], sc[k], sh[k]);
          const float d = ACT != EAT_ACT_NONE ? act_bwd(v, ACT) : 1.f;
          const float f = ACT != EAT_ACT_NONE ? act_fwd(v, ACT) : v;
          const float zc = zv[k] - mu[k];
          const float gd = gv[k] * d;
          aD[k] = fmaf(gv[k], f, aD[k]);
          a1[k] += gd;
          a2[k] = fmaf(gd, zc, a2[k]);
          e1[k] += d;
          e2[k] = fmaf(d, zc, e2[k]);
        }
      };
      const size_t base = (size_t)b * P * C + c0;
      const int step = gridDim.x * ppb;
      int p = blockIdx.x * ppb + slot;
      for (; p + (U - 1) * step < P; p += U * step) {
        float zz[U][V], gg[U][V];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const size_t o = base + (size_t)(p + u * step) * C;
          Vec<T>::load(z + o, zz[u]);
          Vec<T>::load(dp + o, gg[u]);
        }
#pragma unroll
        for (int u = 0; u < U; ++u) one(zz[u], gg[u]);
      }
      for (; p < P; p += step) {
        const size_t o = base + (size_t)p * C;
        float z0[V], g0[V];
        Vec<T>::load(z + o, z0);
        Vec<T>::load(dp + o, g0);
        one(z0, g0);
      }
      if (shared) {
#pragma unroll
        for (int k = 0; k < V; ++k) {
          atomicAdd(&smem[c0 + k], aD[k]);
          atomicAdd(&smem[C + c0 + k], a1[k]);
          atomicAdd(&smem[2 * C + c0 + k], a2[k]);
          atomicAdd(&smem[3 * C + c0 + k], e1[k]);
          atomicAdd(&smem[4 * C + c0 + k], e2[k]);
        }
      } else {                                       // this thread is the only owner of the channel vector in the CTA
#pragma unroll
        for (int k = 0; k < V; ++k) {
          atomicAdd(dgate + (size_t)b * C + c0 + k, aD[k]);
          my_part[c0 + k] = a1[k];
          my_part[qs + c0 + k] = a2[k];
          my_part[2 * qs + c0 + k] = e1[k];
          my_part[3 * qs + c0 + k] = e2[k];
        }
      }
    }
  }
  if (shared) {
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += kThreads) {
      atomicAdd(dgate + (size_t)b * C + c, smem[c]);
#pragma unroll
      for (int q = 0; q < 4; ++q) my_part[q * qs + c] = smem[(q + 1) * C + c];
    }
  }
}

// s1[c] += sum_b gate*A1 + dpool*E1,  s2[c] += invstd[c] * sum_b gate*A2 + dpool*E2, with A1, A2, E1, E2 the pixel sums of
// se_bn_bwd_reduce_kernel (added up over its `parts` slices): what bn_bwd_reduce2_kernel<GM = 1> would have produced.
// Block = 32 channels x 8 batch lanes; grid.y splits the batch further (fp64 atomics into the zeroed accumulators).
__global__ void __launch_bounds__(256) se_bn_bwd_combine_kernel(const float* __restrict__ part, int parts,
                                                                const float* __restrict__ gate,
                                                                const float* __restrict__ dpool,
                                                                const float* __restrict__ invstd, int B, int C,
                                                                double* __restrict__ s1, double* __restrict__ s2) {
  __shared__ double r1[8][33], r2[8][33];
  const int c = blockIdx.x * 32 + threadIdx.x;
  const size_t qs = (size_t)B * C;
  double t1 = 0.0, t2 = 0.0;
  if (c < C) {
    for (int b = blockIdx.y * 8 + threadIdx.y; b < B; b += gridDim.y * 8) {
      float A1 = 0.f, A2 = 0.f, E1 = 0.f, E2 = 0.f;
      for (int g = 0; g < parts; ++g) {
        const float* p = part + ((size_t)g * 4 * B + b) * C + c;
        A1 += p[0]; A2 += p[qs]; E1 += p[2 * qs]; E2 += p[3 * qs];
      }
      const double gt = gate != nullptr ? (double)gate[(size_t)b * C + c] : 1.0;
      const double dv = dpool != nullptr ? (double)dpool[(size_t)b * C + c] : 0.0;
      t1 += gt * A1 + dv * E1;
      t2 += gt * A2 + dv * E2;
    }
  }
  r1[threadIdx.y][threadIdx.x] = t1;
  r2[threadIdx.y][threadIdx.x] = t2;
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
    double u1 = 0.0, u2 = 0.0;
#pragma unroll
    for (int j = 0; j < 8; ++j) { u1 += r1[j][threadIdx.x]; u2 += r2[j][threadIdx.x]; }
    atomicAdd(s1 + c, u1);
    atomicAdd(s2 + c, u2 * (double)invstd[c]);
  }
}

// Squeeze-excitation MLP backward for one sample per CTA (block_types.py:72-83):
//   du2 = dgate * gate * (1 - gate); dh = W2^T du2; du1 = dh * (hidden > 0); dmean = W1^T du1
//   dpool_out[b,c] = dmean * inv_count.   du2 / du1 are stored for the weight-gradient GEMMs.
__global__ void __launch_bounds__(kThreads) se_fc_bwd_kernel(const float* __restrict__ dgate,
                                                             const float* __restrict__ gate,
                                                             const float* __restrict__ hidden,
                                                             const float* __restrict__ w1, const float* __restrict__ w2,
                                                             float inv_count, float* __restrict__ du2,
                                                             float* __restrict__ du1, float* __restrict__ dpool,
                                                             int C, int S) {
  extern __shared__ float smem[];
  float* s_du2 = smem;       // [C]
  float* s_du1 = smem + C;   // [S]
  const int b = blockIdx.x;
  for (int c = threadIdx.x; c < C; c += kThreads) {
    float g = gate[(size_t)b * C + c];
    float v = dgate[(size_t)b * C + c] * g * (1.f - g);
    s_du2[c] = v;
    du2[(size_t)b * C + c] = v;
  }
  __syncthreads();
  // dh[s] = sum_c w2[c, s] * du2[c]   (column access of w2: threads over s are coalesced)
  for (int s = threadIdx.x; s < S; s += kThreads) {
    // four independent accumulators: a single fmaf chain over C <= 960 terms is pure FMA latency
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
    int c = 0;
    for (; c + 3 < C; c += 4) {
      a0 = fmaf(__ldg(w2 + (size_t)c * S + s), s_du2[c], a0);
      a1 = fmaf(__ldg(w2 + (size_t)(c + 1) * S + s), s_du2[c + 1], a1);
      a2 = fmaf(__ldg(w2 + (size_t)(c + 2) * S + s), s_du2[c + 2], a2);
      a3 = fmaf(__ldg(w2 + (size_t)(c + 3) * S + s), s_du2[c + 3], a3);
    }
    for (; c < C; ++c) a0 = fmaf(__ldg(w2 + (size_t)c * S + s), s_du2[c], a0);
    const float acc = (a0 + a1) + (a2 + a3);
    float v = hidden[(size_t)b * S + s] > 0.f ? acc : 0.f;
    s_du1[s] = v;
    du1[(size_t)b * S + s] = v;
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += kThreads) {
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
    int s = 0;
    for (; s + 3 < S; s += 4) {
      a0 = fmaf(__ldg(w1 + (size_t)s * C + c), s_du1[s], a0);
      a1 = fmaf(__ldg(w1 + (size_t)(s + 1) * C + c), s_du1[s + 1], a1);
      a2 = fmaf(__ldg(w1 + (size_t)(s + 2) * C + c), s_du1[s + 2], a2);
      a3 = fmaf(__ldg(w1 + (size_t)(s + 3) * C + c), s_du1[s + 3], a3);
    }
    for (; s < S; ++s) a0 = fmaf(__ldg(w1 + (size_t)s * C + c), s_du1[s], a0);
    dpool[(size_t)b * C + c] = ((a0 + a1) + (a2 + a3)) * inv_count;
  }
}

// The same backward as batched products (any batch): the per-sample kernel above re-reads both weight matrices once per
// sample -- at mn40 widths (C = 3840, S = 960: 14.7 MB per matrix) that was 18 % of the training step.
//   du2 = dgate * gate * (1 - gate)                     [B, C]   (se_du2_kernel)
//   dh  = du2 . W2                                       [B, S]   (32 x 32-tile GEMM, W2 = fc2.weight [C, S])
//   du1 = dh * (hidden > 0)                              [B, S]   (se_mask_kernel, in place)
//   dpool = inv_count * du1 . W1                         [B, C]   (W1 = fc1.weight [S, C])
__global__ void se_du2_kernel(const float* __restrict__ dgate, const float* __restrict__ gate, float* __restrict__ du2,
                              long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float g = gate[i];
    du2[i] = dgate[i] * g * (1.f - g);
  }
}
__global__ void se_mask_kernel(float* __restrict__ du1, const float* __restrict__ hidden, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    du1[i] = hidden[i] > 0.f ? du1[i] : 0.f;
}

// ------------------------------------------------------------------------------------------
// Depthwise conv backward.  The data gradients and the fp32 weight gradients live in dw_slide.cu / conv_kernels.cu;
// the kernel below is the weight gradient of the remaining case (bf16 storage, 5x5).
// Shared-memory tiled depthwise weight gradient: dw[c, ky, kx] += sum dz * xf(in).  A CTA stages the transformed
// input tile and the dz tile of one sample / 32-channel chunk in shared memory (BatchNorm+activation applied once
// per input element), keeps all K*K tap accumulators of its channel slice in registers across its tiles, and
// reduces them once at the end (shared atomics, then one global atomic per tap and channel).
template <typename T, int K, int S>
__global__ void __launch_bounds__(kThreads) dw_wgrad_tile_kernel(const T* __restrict__ dz, const T* __restrict__ in,
                                                                 InXform xf, float* __restrict__ dw, int F, int Tn,
                                                                 int Fo, int To, int C, long long dw_bstride) {
  constexpr int VG = Vec<T>::N;
  constexpr int CC = 32;
  constexpr int VW = (K == 3) ? 4 : 2;           // channels per thread (register budget: K*K*VW accumulators)
  constexpr int CCW = CC / VW;
  constexpr int FR = (S == 1) ? 8 : 4;
  constexpr int TT = (S == 1) ? 32 : 16;
  constexpr int P = 4;
  constexpr int SPR = TT / P;
  constexpr int IR = (FR - 1) * S + K, IT = (TT - 1) * S + K;
  constexpr int NIN = (P - 1) * S + K;
  constexpr int PAD = (K - 1) / 2;
  constexpr int KK = K * K;
  constexpr int STRIPS = FR * SPR;
  constexpr int PARTS = kThreads / CCW;
  extern __shared__ __align__(16) float smem[];
  float* s_in = smem;                            // [IR*IT][CC]
  float* s_g = s_in + IR * IT * CC;              // [FR*TT][CC]
  float* s_acc = s_g + FR * TT * CC;             // [KK][CC]
  const int b = blockIdx.y;
  const int tiles_t = ceil_div(To, TT), tiles_f = ceil_div(Fo, FR), chunks = ceil_div(C, CC);
  const int tiles_per_chunk = tiles_t * tiles_f;
  const int groups = gridDim.x / chunks;
  const int chunk = blockIdx.x / groups, grp = blockIdx.x - chunk * groups;
  if (chunk >= chunks) return;
  const int cbase = chunk * CC;
  const int tid = threadIdx.x;
  const T* inb = in + (size_t)b * F * Tn * C;
  const T* dzb = dz + (size_t)b * Fo * To * C;
  for (int i = tid; i < KK * CC; i += kThreads) s_acc[i] = 0.f;
  constexpr int VPP = CC / VG;
  const int lv = tid % VPP;
  const int lc0 = cbase + lv * VG;
  const bool lvalid = lc0 < C;
  float isc[VG], ish[VG];
  if (xf.scale != nullptr && lvalid) {
#pragma unroll
    for (int i = 0; i < VG; ++i) { isc[i] = xf.scale[lc0 + i]; ish[i] = xf.shift[lc0 + i]; }
  }
  const int cw = tid % CCW, part = tid / CCW;
  const bool cvalid = cbase + cw * VW < C;
  float acc[KK][VW];
#pragma unroll
  for (int q = 0; q < KK; ++q)
#pragma unroll
    for (int i = 0; i < VW; ++i) acc[q][i] = 0.f;
  for (int tile = grp; tile < tiles_per_chunk; tile += groups) {
    const int tf = tile / tiles_t, tt = tile - tf * tiles_t;
    const int f0 = tf * FR, t0 = tt * TT;
    __syncthreads();
    for (int idx = tid; idx < IR * IT * VPP; idx += kThreads) {
      const int pix = idx / VPP;
      const int ir = pix / IT, it = pix - ir * IT;
      const int f = f0 * S - PAD + ir, t = t0 * S - PAD + it;
      float v[VG];
      if (lvalid && f >= 0 && f < F && t >= 0 && t < Tn) {
        Vec<T>::load(inb + ((size_t)f * Tn + t) * C + lc0, v);
        if (xf.scale != nullptr) {
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
    for (int idx = tid; idx < FR * TT * VPP; idx += kThreads) {
      const int pix = idx / VPP;
      const int fl = pix / TT, tl = pix - fl * TT;
      const int fo = f0 + fl, to = t0 + tl;
      float v[VG];
      if (lvalid && fo < Fo && to < To) Vec<T>::load(dzb + ((size_t)fo * To + to) * C + lc0, v);
      else {
#pragma unroll
        for (int i = 0; i < VG; ++i) v[i] = 0.f;
      }
      float* dst = s_g + (size_t)pix * CC + lv * VG;
#pragma unroll
      for (int q = 0; q < VG / 4; ++q)
        *reinterpret_cast<float4*>(dst + 4 * q) = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
    }
    __syncthreads();
    if (cvalid) {
      for (int strip = part; strip < STRIPS; strip += PARTS) {
        const int fl = strip / SPR, ts = strip - fl * SPR;
        float g[P][VW];
#pragma unroll
        for (int pp = 0; pp < P; ++pp) {
          const float* gp = s_g + ((size_t)fl * TT + ts * P + pp) * CC + cw * VW;
#pragma unroll
          for (int i = 0; i < VW; ++i) g[pp][i] = gp[i];
        }
#pragma unroll
        for (int ky = 0; ky < K; ++ky) {
          const float* rowp = s_in + ((size_t)(fl * S + ky) * IT + ts * P * S) * CC + cw * VW;
#pragma unroll
          for (int ix = 0; ix < NIN; ++ix) {
            float v[VW];
#pragma unroll
            for (int i = 0; i < VW; ++i) v[i] = rowp[(size_t)ix * CC + i];
#pragma unroll
            for (int pp = 0; pp < P; ++pp) {
              const int kx = ix - pp * S;
              if (kx >= 0 && kx < K) {
#pragma unroll
                for (int i = 0; i < VW; ++i) acc[ky * K + kx][i] = fmaf(g[pp][i], v[i], acc[ky * K + kx][i]);
              }
            }
          }
        }
      }
    }
  }
  if (cvalid) {
#pragma unroll
    for (int q = 0; q < KK; ++q)
#pragma unroll
      for (int i = 0; i < VW; ++i) atomicAdd(&s_acc[q * CC + cw * VW + i], acc[q][i]);
  }
  __syncthreads();
  float* dwb = dw + (size_t)b * dw_bstride;
  for (int i = tid; i < KK * CC; i += kThreads) {
    const int q = i / CC, c = i % CC;
    if (cbase + c < C) atomicAdd(dwb + (size_t)(cbase + c) * KK + q, s_acc[i]);
  }
}

// stem wgrad: dw[c, ky, kx] += sum dz[b,fo,to,c] * x[b, fo*s-1+ky, to*s-1+kx]
template <typename T>
__global__ void __launch_bounds__(kThreads) stem_wgrad_kernel(const T* __restrict__ dz, const float* __restrict__ x,
                                                              float* __restrict__ dw, int B, int F, int Tn, int Fo,
                                                              int To, int C, int stride) {
  constexpr int V = Vec<T>::N;
  extern __shared__ float smem[];   // [9][C]
  for (int i = threadIdx.x; i < 9 * C; i += kThreads) smem[i] = 0.f;
  __syncthreads();
  const int cv = C / V;
  const int ppb = kThreads / cv;
  const int cvi = threadIdx.x % cv, slot = threadIdx.x / cv;
  const long long npix = (long long)B * Fo * To;
  if (slot < ppb) {
    float acc[9][V];
#pragma unroll
    for (int q = 0; q < 9; ++q)
#pragma unroll
      for (int k = 0; k < V; ++k) acc[q][k] = 0.f;
    const unsigned ppx = (unsigned)To * (unsigned)Fo;       // 32-bit index math: npix < 2^31 is checked by the launcher
    for (unsigned pix = blockIdx.x * ppb + slot; pix < (unsigned)npix; pix += gridDim.x * ppb) {
      const unsigned b_ = pix / ppx, rem_ = pix - b_ * ppx;
      const int fo = (int)(rem_ / (unsigned)To), to = (int)(rem_ - (rem_ / (unsigned)To) * (unsigned)To), b = (int)b_;
      float g[V];
      Vec<T>::load(dz + (size_t)pix * C + cvi * V, g);
#pragma unroll
      for (int ky = 0; ky < 3; ++ky) {
        const int f = fo * stride - 1 + ky;
        if (f < 0 || f >= F) continue;
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) {
          const int t = to * stride - 1 + kx;
          if (t < 0 || t >= Tn) continue;
          const float xv = __ldg(x + ((size_t)b * F + f) * Tn + t);
#pragma unroll
          for (int k = 0; k < V; ++k) acc[ky * 3 + kx][k] = fmaf(g[k], xv, acc[ky * 3 + kx][k]);
        }
      }
    }
#pragma unroll
    for (int q = 0; q < 9; ++q)
#pragma unroll
      for (int k = 0; k < V; ++k) atomicAdd(&smem[q * C + cvi * V + k], acc[q][k]);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 9 * C; i += kThreads) {
    const int q = i / C, c = i % C;
    atomicAdd(dw + (size_t)c * 9 + q, smem[i]);
  }
}

// stem data gradient: dx[b,f,t] = sum_{c,ky,kx} w[c,ky,kx] * dz[b,fo,to,c] over the taps with f = fo*S-1+ky,
// t = to*S-1+kx, where dz = scale * (dy * act'(z*scale+shift) - c1 - xhat*c2) is formed on load (eat_bn_bwd_apply's
// formula; c1 = c2 = 0 for BatchNorm on running statistics).  One thread per input pixel, all channels in a fixed order:
// no atomics, so the result is bitwise repeatable.  Lanes of a warp walk the same channel, so the weight and BatchNorm
// loads are broadcasts.
template <typename T, int S>
__global__ void __launch_bounds__(kThreads) stem_dgrad_kernel(const T* __restrict__ dy, const T* __restrict__ z, BnCtx bn,
                                                              const float* __restrict__ c1, const float* __restrict__ c2,
                                                              const float* __restrict__ w, float* __restrict__ dx, int B,
                                                              int F, int Tn, int C) {
  constexpr int V = Vec<T>::N;
  const int Fo = (F - 1) / S + 1, To = (Tn - 1) / S + 1;
  const long long npix = (long long)B * F * Tn;
  for (long long pix = (long long)blockIdx.x * kThreads + threadIdx.x; pix < npix; pix += (long long)gridDim.x * kThreads) {
    const int t = (int)(pix % Tn), f = (int)((pix / Tn) % F), b = (int)(pix / ((long long)Tn * F));
    float acc = 0.f;
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
      const int fs = f + 1 - ky;
      if (fs < 0 || fs % S != 0 || fs / S >= Fo) continue;
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const int ts = t + 1 - kx;
        if (ts < 0 || ts % S != 0 || ts / S >= To) continue;
        const size_t base = (((size_t)b * Fo + fs / S) * To + ts / S) * C;
        for (int c0 = 0; c0 < C; c0 += V) {
          float g[V], zv[V];
          Vec<T>::load(dy + base + c0, g);
          Vec<T>::load(z + base + c0, zv);
#pragma unroll
          for (int k = 0; k < V; ++k) {
            const int c = c0 + k;
            const float sc = __ldg(bn.scale + c);
            const float d = g[k] * act_bwd(fmaf(zv[k], sc, __ldg(bn.shift + c)), bn.act);
            const float xhat = (zv[k] - __ldg(bn.mean + c)) * __ldg(bn.invstd + c);
            acc = fmaf(__ldg(w + c * 9 + ky * 3 + kx), sc * (d - __ldg(c1 + c) - xhat * __ldg(c2 + c)), acc);
          }
        }
      }
    }
    dx[pix] = acc;
  }
}

// Row-oriented stem weight gradient (fp32 dz, C <= 64): same walk as stem_row_kernel; the U = 4 gradient vectors and
// the 36 input values of a trip are requested before the first use (the pixel-at-a-time kernel above has ONE 16-byte
// load in flight per thread).  APPLY: `dz` is the gradient dy at the BatchNorm + activation's output and dz is computed
// on load from (dy, z) with the folded constants of eat_bn_bwd_apply (as bn_bwd_apply2_kernel), so the stem's
// BatchNorm-backward apply pass and its dz tensor are not needed.
template <int S, int APPLY>
__global__ void __launch_bounds__(kThreads, APPLY ? 2 : 1) stem_wgrad_row_kernel(const float* __restrict__ dz, const float* __restrict__ x,
                                                                  float* __restrict__ dw, int B, int F, int Tn, int Fo,
                                                                  int To, int C, const float* __restrict__ z, BnCtx bn,
                                                                  int act, const float* __restrict__ c1,
                                                                  const float* __restrict__ c2) {
  constexpr int V = 4, U = APPLY ? 2 : 4;        // 64 bytes of dz (dy and z) loads in flight either way
  __shared__ float s_acc[9 * 64];
  for (int i = threadIdx.x; i < 9 * C; i += kThreads) s_acc[i] = 0.f;
  __syncthreads();
  const int cv = C / V;
  const int ppb = kThreads / cv;
  const int cvi = threadIdx.x % cv, slot = threadIdx.x / cv;
  if (slot < ppb) {
    float acc[9][V];
#pragma unroll
    for (int q = 0; q < 9; ++q)
#pragma unroll
      for (int k = 0; k < V; ++k) acc[q][k] = 0.f;
    float sc[V], sh[V], al[V], be[V];              // dz = sc * (dy * act'(z * sc + sh)) + al * z + be
    if (APPLY) {
#pragma unroll
      for (int k = 0; k < V; ++k) {
        const int c = cvi * V + k;
        sc[k] = bn.scale[c]; sh[k] = bn.shift[c];
        al[k] = -sc[k] * c2[c] * bn.invstd[c];
        be[k] = -sc[k] * c1[c] - al[k] * bn.mean[c];
      }
    }
    const int rows = B * Fo;
    for (int row = blockIdx.x; row < rows; row += gridDim.x) {
      const int b = row / Fo, fo = row - b * Fo;
      const float* xb = x + (size_t)b * F * Tn;
      const float* grow = dz + (size_t)row * To * C + cvi * V;
      const float* zrow = APPLY ? z + (size_t)row * To * C + cvi * V : nullptr;
      const int f0 = fo * S - 1;
      for (int to0 = slot; to0 < To; to0 += U * ppb) {
        float4 g[U], zz[U];
        float xv[U][9];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int to = to0 + u * ppb, t0 = to * S - 1;
          g[u] = to < To ? *reinterpret_cast<const float4*>(grow + (size_t)to * C) : make_float4(0.f, 0.f, 0.f, 0.f);
          if (APPLY) zz[u] = to < To ? *reinterpret_cast<const float4*>(zrow + (size_t)to * C) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
          for (int ky = 0; ky < 3; ++ky) {
            const int f = f0 + ky;
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) {
              const int t = t0 + kx;
              xv[u][ky * 3 + kx] = (to < To && f >= 0 && f < F && t >= 0 && t < Tn) ? __ldg(xb + (size_t)f * Tn + t) : 0.f;
            }
          }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          float gv[V] = {g[u].x, g[u].y, g[u].z, g[u].w};
          if (APPLY) {
            const float zv[V] = {zz[u].x, zz[u].y, zz[u].z, zz[u].w};
            const bool live = to0 + u * ppb < To;      // past the row's end dz is 0, not beta
#pragma unroll
            for (int k = 0; k < V; ++k) {
              const float gg = gv[k] * act_bwd(fmaf(zv[k], sc[k], sh[k]), act);
              gv[k] = live ? fmaf(sc[k], gg, fmaf(al[k], zv[k], be[k])) : 0.f;
            }
          }
#pragma unroll
          for (int q = 0; q < 9; ++q)
#pragma unroll
            for (int k = 0; k < V; ++k) acc[q][k] = fmaf(gv[k], xv[u][q], acc[q][k]);
        }
      }
    }
#pragma unroll
    for (int q = 0; q < 9; ++q)
#pragma unroll
      for (int k = 0; k < V; ++k) atomicAdd(&s_acc[q * C + cvi * V + k], acc[q][k]);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 9 * C; i += kThreads) {
    const int q = i / C, c = i % C;
    atomicAdd(dw + (size_t)c * 9 + q, s_acc[i]);
  }
}

// head: dpre = dh * mask * act'(pre)   (fp32, [n])
__global__ void act_bwd_kernel(const float* __restrict__ dh, const float* __restrict__ pre,
                               const float* __restrict__ mask, int act, float* __restrict__ dpre, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    dpre[i] = dh[i] * (mask != nullptr ? mask[i] : 1.f) * act_bwd(pre[i], act);
}

inline int grid2(int P, int ppb, int B) {
  int gx = ceil_div(P, ppb * 4);
  const int cap = max(1, (kNumSMs * 8) / max(B, 1));
  if (gx > cap) gx = cap;
  return gx < 1 ? 1 : gx;
}

template <typename T>
int launch_bn_bwd_reduce(const void* gA, const float* gate, const float* dpool, const void* z, BnCtx bn, int B, int P,
                         int C, double* s1, double* s2, cudaStream_t st) {
  constexpr int V = Vec<T>::N;
  const int cv = C / V, tcv = cv < kThreads ? cv : kThreads, ppb = kThreads / tcv;
  static const bool v1 = [] { const char* e = getenv("EAT_BN_REDUCE"); return e != nullptr && strcmp(e, "v1") == 0; }();
  if (v1) {
    dim3 grid(grid2(P, ppb, B), B);
    bn_bwd_reduce_kernel<T><<<grid, kThreads, 2 * C * sizeof(float), st>>>((const T*)gA, gate, dpool, (const T*)z, bn, B, P, C, s1, s2);
    EAT_CHECK_LAUNCH();
    return EAT_OK;
  }
  // ~12 CTAs per SM in total (3 resident at a time), at least 4 pixels per thread
  int gx = ceil_div(P, ppb * 4);
  const int cap = max(1, (kNumSMs * 12) / max(B, 1));
  if (gx > cap) gx = cap;
  dim3 grid(gx < 1 ? 1 : gx, B);
  const size_t sm = 2 * C * sizeof(float);
  const int gm = gA == nullptr ? 2 : ((gate != nullptr || dpool != nullptr) ? 1 : 0);
#define EAT_RED(ACT, GM) bn_bwd_reduce2_kernel<T, ACT, GM><<<grid, kThreads, sm, st>>>((const T*)gA, gate, dpool, (const T*)z, bn, B, P, C, s1, s2)
#define EAT_RED_A(ACT) do { if (gm == 0) EAT_RED(ACT, 0); else if (gm == 1) EAT_RED(ACT, 1); else EAT_RED(ACT, 2); } while (0)
  if (bn.act == EAT_ACT_RELU) EAT_RED_A(EAT_ACT_RELU);
  else if (bn.act == EAT_ACT_HSWISH) EAT_RED_A(EAT_ACT_HSWISH);
  else EAT_RED_A(EAT_ACT_NONE);
#undef EAT_RED_A
#undef EAT_RED
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

template <typename T>
int launch_dw_bwd(int which, const void* dz, const float* wt, const void* in, InXform xf, const void* res, void* din,
                  float* dw, int B, int F, int Tn, int C, int k, int stride, cudaStream_t st, long long wt_bstride = 0,
                  long long dw_bstride = 0) {
  constexpr int V = Vec<T>::N;
  if (C % V != 0) { eat_set_error("dw bwd: channels must be a multiple of the vector width"); return EAT_ERR_ARG; }
  const int pad = (k - 1) / 2;
  const int Fo = (F + 2 * pad - k) / stride + 1, To = (Tn + 2 * pad - k) / stride + 1;
  const int cv = C / V;
  if (which == 0) {
    eat_set_error("dw dgrad: unsupported kernel size / stride");
    return EAT_ERR_UNSUPPORTED;
  } else {
    const int FR = stride == 1 ? 8 : 4, TT = stride == 1 ? 32 : 16;
    const int IR = (FR - 1) * stride + k, IT = (TT - 1) * stride + k;
    const int chunks = ceil_div(C, 32);
    const int tiles = ceil_div(Fo, FR) * ceil_div(To, TT);
    int groups = max(1, (kNumSMs * 4) / max(B * chunks, 1));
    if (groups > tiles) groups = tiles;
    dim3 grid(chunks * groups, B);
    size_t smem = ((size_t)IR * IT * 32 + (size_t)FR * TT * 32 + (size_t)k * k * 32) * sizeof(float);
#define EAT_WG(KK, SS)                                                                                          \
  do {                                                                                                          \
    static unsigned long long attr = 0;                                                                         \
    if (int rc = eat_opt_in_smem(dw_wgrad_tile_kernel<T, KK, SS>, 128 * 1024, attr)) return rc;                 \
    dw_wgrad_tile_kernel<T, KK, SS><<<grid, kThreads, smem, st>>>((const T*)dz, (const T*)in, xf, dw, F, Tn, Fo, To, C, dw_bstride); \
  } while (0)
    if (k == 3 && stride == 1) EAT_WG(3, 1); else if (k == 3 && stride == 2) EAT_WG(3, 2);
    else if (k == 5 && stride == 1) EAT_WG(5, 1); else if (k == 5 && stride == 2) EAT_WG(5, 2);
    else { eat_set_error("dw wgrad: only k in {3,5}, stride in {1,2}"); return EAT_ERR_UNSUPPORTED; }
#undef EAT_WG
  }
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

}  // namespace

extern "C" {

int eat_bn_bwd_reduce(const void* gA, const float* gate, const float* dpool, const void* z, const float* scale,
                      const float* shift, const float* mean, const float* invstd, int act, int dtype, int B, int P,
                      int C, double* s1, double* s2, cudaStream_t st) {
  if (B == 0 || P == 0) return EAT_OK;
  BnCtx bn{scale, shift, mean, invstd, act};
  const int V = dtype == EAT_BF16 ? 8 : 4;
  if (C % V != 0) { eat_set_error("bn_bwd_reduce: channels must be a multiple of the vector width"); return EAT_ERR_ARG; }
  if (dtype == EAT_BF16) return launch_bn_bwd_reduce<__nv_bfloat16>(gA, gate, dpool, z, bn, B, P, C, s1, s2, st);
  return launch_bn_bwd_reduce<float>(gA, gate, dpool, z, bn, B, P, C, s1, s2, st);
}

int eat_bn_bwd_finalize(const double* s1, const double* s2, double count, float* dgamma, float* dbeta, float* c1,
                        float* c2, int C, cudaStream_t st) {
  bn_bwd_finalize_kernel<<<ceil_div(C, 128), 128, 0, st>>>(s1, s2, count, dgamma, dbeta, c1, c2, C);
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

int eat_bn_bwd_apply(const void* gA, const float* gate, const float* dpool, const void* z, const float* scale,
                     const float* shift, const float* mean, const float* invstd, int act, const float* c1,
                     const float* c2, void* dz, int dtype, int B, int P, int C, cudaStream_t st) {
  if (B == 0 || P == 0) return EAT_OK;
  BnCtx bn{scale, shift, mean, invstd, act};
  const int V = dtype == EAT_BF16 ? 8 : 4;
  if (C % V != 0) { eat_set_error("bn_bwd_apply: channels must be a multiple of the vector width"); return EAT_ERR_ARG; }
  const int cv = C / V, tcv = cv < kThreads ? cv : kThreads, ppb = kThreads / tcv;
  // EAT_BN_APPLY=v2|v1 selects the kernel generation
  static const bool v2 = [] { const char* e = getenv("EAT_BN_APPLY"); return e != nullptr ? strcmp(e, "v2") == 0 : kBnApplyV2Default; }();
  if (v2 && (act == EAT_ACT_NONE || act == EAT_ACT_RELU || act == EAT_ACT_HSWISH)) {
    // ~12 CTAs per SM in total (3 resident at a time), at least 4 pixels per thread
    int g2 = ceil_div(P, ppb * 4);
    const int cap2 = max(1, (kNumSMs * 12) / max(B, 1));
    if (g2 > cap2) g2 = cap2;
    dim3 grid2(g2 < 1 ? 1 : g2, B);
    const int gm = gA == nullptr ? 2 : ((gate != nullptr || dpool != nullptr) ? 1 : 0);
#define EAT_APP(TT, ACT, GM) bn_bwd_apply2_kernel<TT, ACT, GM><<<grid2, kThreads, 0, st>>>((const TT*)gA, gate, dpool, (const TT*)z, bn, c1, c2, (TT*)dz, B, P, C)
#define EAT_APP_A(TT, ACT) do { if (gm == 0) EAT_APP(TT, ACT, 0); else if (gm == 1) EAT_APP(TT, ACT, 1); else EAT_APP(TT, ACT, 2); } while (0)
#define EAT_APP_T(TT) do { if (act == EAT_ACT_RELU) EAT_APP_A(TT, EAT_ACT_RELU); else if (act == EAT_ACT_HSWISH) EAT_APP_A(TT, EAT_ACT_HSWISH); \
                           else EAT_APP_A(TT, EAT_ACT_NONE); } while (0)
    if (dtype == EAT_BF16) EAT_APP_T(__nv_bfloat16); else EAT_APP_T(float);
#undef EAT_APP_T
#undef EAT_APP_A
#undef EAT_APP
    EAT_CHECK_LAUNCH();
    return EAT_OK;
  }
  // ~16 CTAs per SM in total, at least 2 pixels per thread
  int gx = ceil_div(P, 2 * ppb);
  const int cap = max(1, (kNumSMs * 16) / max(B, 1));
  if (gx > cap) gx = cap;
  dim3 grid(gx < 1 ? 1 : gx, B);
  if (dtype == EAT_BF16)
    bn_bwd_apply_kernel<__nv_bfloat16><<<grid, kThreads, 0, st>>>((const __nv_bfloat16*)gA, gate, dpool, (const __nv_bfloat16*)z, bn, c1, c2, (__nv_bfloat16*)dz, B, P, C);
  else
    bn_bwd_apply_kernel<float><<<grid, kThreads, 0, st>>>((const float*)gA, gate, dpool, (const float*)z, bn, c1, c2, (float*)dz, B, P, C);
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

int eat_se_bwd_reduce(const void* dp, const void* z, const float* scale, const float* shift, int act, float* dgate,
                      int dtype, int B, int P, int C, cudaStream_t st) {
  if (B == 0) return EAT_OK;
  const int V = dtype == EAT_BF16 ? 8 : 4;
  if (C % V != 0) { eat_set_error("se_bwd_reduce: channels must be a multiple of the vector width"); return EAT_ERR_ARG; }
  const int cv = C / V, tcv = cv < kThreads ? cv : kThreads, ppb = kThreads / tcv;
  dim3 grid(grid2(P, ppb, B), B);
  if (dtype == EAT_BF16)
    se_bwd_reduce_kernel<__nv_bfloat16><<<grid, kThreads, C * sizeof(float), st>>>((const __nv_bfloat16*)dp, (const __nv_bfloat16*)z, scale, shift, act, dgate, P, C);
  else
    se_bwd_reduce_kernel<float><<<grid, kThreads, C * sizeof(float), st>>>((const float*)dp, (const float*)z, scale, shift, act, dgate, P, C);
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

int eat_se_bn_bwd_reduce(const void* dp, const void* z, const float* scale, const float* shift, const float* mean, int act,
                         float* dgate, float* part, int parts, int dtype, int B, int P, int C, cudaStream_t st) {
  if (B == 0) return EAT_OK;
  const int V = dtype == EAT_BF16 ? 8 : 4;
  if (C % V != 0) { eat_set_error("se_bn_bwd_reduce: channels must be a multiple of the vector width"); return EAT_ERR_ARG; }
  if (parts < 1 || P < 1) { eat_set_error("se_bn_bwd_reduce: parts and P must be positive"); return EAT_ERR_ARG; }
  const int cv = C / V, tcv = cv < kThreads ? cv : kThreads, ppb = kThreads / tcv;
  dim3 grid(parts, B);
  const size_t sm = ppb > 1 ? 5 * (size_t)C * sizeof(float) : 0;      // ppb > 1 implies cv <= 128, i.e. at most 20 KB
#define EAT_SEBN(TT, ACT) se_bn_bwd_reduce_kernel<TT, ACT><<<grid, kThreads, sm, st>>>((const TT*)dp, (const TT*)z, scale, shift, mean, dgate, part, B, P, C)
#define EAT_SEBN_T(TT) do { if (act == EAT_ACT_RELU) EAT_SEBN(TT, EAT_ACT_RELU); else if (act == EAT_ACT_HSWISH) EAT_SEBN(TT, EAT_ACT_HSWISH); \
                            else if (act == EAT_ACT_NONE) EAT_SEBN(TT, EAT_ACT_NONE); \
                            else { eat_set_error("se_bn_bwd_reduce: activation must be none / relu / hardswish"); return EAT_ERR_UNSUPPORTED; } } while (0)
  if (dtype == EAT_BF16) EAT_SEBN_T(__nv_bfloat16); else EAT_SEBN_T(float);
#undef EAT_SEBN_T
#undef EAT_SEBN
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

int eat_se_bn_bwd_combine(const float* part, int parts, const float* gate, const float* dpool, const float* invstd, int B,
                          int C, double* s1, double* s2, cudaStream_t st) {
  if (B == 0 || C == 0) return EAT_OK;
  if (parts < 1) { eat_set_error("se_bn_bwd_combine: parts must be positive"); return EAT_ERR_ARG; }
  int gy = ceil_div(B, 8);
  if (gy > 16) gy = 16;
  dim3 grid(ceil_div(C, 32), gy), block(32, 8);
  se_bn_bwd_combine_kernel<<<grid, block, 0, st>>>(part, parts, gate, dpool, invstd, B, C, s1, s2);
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

int eat_se_fc_bwd(const float* dgate, const float* gate, const float* hidden, const float* w1, const float* w2,
                  float inv_count, float* du2, float* du1, float* dpool, int B, int C, int S, cudaStream_t st) {
  if (B == 0) return EAT_OK;
  static const bool per_sample = [] { const char* e = getenv("EAT_SE_BWD"); return e != nullptr && strcmp(e, "persample") == 0; }();
  if (per_sample) {
    se_fc_bwd_kernel<<<B, kThreads, (size_t)(C + S) * sizeof(float), st>>>(dgate, gate, hidden, w1, w2, inv_count, du2, du1, dpool, C, S);
    EAT_CHECK_LAUNCH();
    return EAT_OK;
  }
  const long long nc = (long long)B * C, ns = (long long)B * S;
  se_du2_kernel<<<(int)min((long long)kNumSMs * 4, ceil_div_ll(nc, 256)), 256, 0, st>>>(dgate, gate, du2, nc);
  EAT_CHECK_LAUNCH();
  if (int rc = gemm_small_kn_launch(du2, w2, du1, B, S, C, 1.f, st)) return rc;
  se_mask_kernel<<<(int)min((long long)kNumSMs * 4, ceil_div_ll(ns, 256)), 256, 0, st>>>(du1, hidden, ns);
  EAT_CHECK_LAUNCH();
  return gemm_small_kn_launch(du1, w1, dpool, B, C, S, inv_count, st);
}

extern "C" int eat_dw_conv_dgrad_s1(const void* dz, const float* wt, long long wt_bstride, const void* res, void* din,
                                    int dtype, int B, int F, int T, int C, int k, cudaStream_t st);

int eat_dw_conv_dgrad(const void* dz, const float* wt, long long wt_bstride, const void* res, void* din, int dtype, int B,
                      int F, int T, int C, int k, int stride, cudaStream_t st) {
  if (B == 0) return EAT_OK;
  if (stride == 1 && (k == 3 || k == 5)) return eat_dw_conv_dgrad_s1(dz, wt, wt_bstride, res, din, dtype, B, F, T, C, k, st);
  if (stride == 2 && (k == 3 || k == 5)) return dw_dgrad2_slide_launch(dz, wt, wt_bstride, res, din, dtype, B, F, T, C, k, st);
  InXform xf{nullptr, nullptr, nullptr, 0, 0};
  if (dtype == EAT_BF16) return launch_dw_bwd<__nv_bfloat16>(0, dz, wt, nullptr, xf, res, din, nullptr, B, F, T, C, k, stride, st, wt_bstride);
  return launch_dw_bwd<float>(0, dz, wt, nullptr, xf, res, din, nullptr, B, F, T, C, k, stride, st, wt_bstride);
}

int eat_dw_conv_dgrad_bnred(const void* dz, const float* wt, const void* res, void* din, const void* z, const float* zscale,
                            const float* zshift, const float* zmean, const float* zinvstd, int zact, double* s1, double* s2,
                            int dtype, int B, int F, int T, int C, int k, int stride, cudaStream_t st) {
  if (B == 0) return EAT_OK;
  if (z == nullptr || zscale == nullptr || zshift == nullptr || zmean == nullptr || zinvstd == nullptr || s1 == nullptr ||
      s2 == nullptr) {
    eat_set_error("dw_conv_dgrad_bnred: z, its BatchNorm tables and the accumulators are required");
    return EAT_ERR_ARG;
  }
  if (dtype != EAT_F32 || stride != 2 || (k != 3 && k != 5)) {
    eat_set_error("dw_conv_dgrad_bnred: fp32 storage, stride 2, k in {3,5} only (use eat_dw_conv_dgrad + eat_bn_bwd_reduce)");
    return EAT_ERR_UNSUPPORTED;
  }
  return dw_dgrad2_slide_launch(dz, wt, 0, res, din, dtype, B, F, T, C, k, st, z, zscale, zshift, zmean, zinvstd, zact, s1, s2);
}

int eat_dw_conv_wgrad(const void* dz, const void* in, const float* in_scale, const float* in_shift, int in_act,
                      float* dw, long long dw_bstride, int dtype, int B, int F, int T, int C, int k, int stride,
                      cudaStream_t st) {
  if (B == 0) return EAT_OK;
  InXform xf{in_scale, in_shift, nullptr, in_act, 0};
  if ((k == 3 || (k == 5 && dtype != EAT_BF16)) && (stride == 1 || stride == 2))
    return dw_wgrad_slide_launch(dz, in, xf, dw, dw_bstride, dtype, B, F, T, C, k, stride, st);
  if (dtype == EAT_BF16) return launch_dw_bwd<__nv_bfloat16>(1, dz, nullptr, in, xf, nullptr, nullptr, dw, B, F, T, C, k, stride, st, 0, dw_bstride);
  return launch_dw_bwd<float>(1, dz, nullptr, in, xf, nullptr, nullptr, dw, B, F, T, C, k, stride, st, 0, dw_bstride);
}

int eat_stem_wgrad(const void* dz, int dtype, const float* x, float* dw, int B, int F, int T, int C, int stride,
                   const float* z, const float* scale, const float* shift, const float* mean, const float* invstd, int act,
                   const float* c1, const float* c2, cudaStream_t st) {
  const int Fo = (F + 2 - 3) / stride + 1, To = (T + 2 - 3) / stride + 1;
  const int V = dtype == EAT_BF16 ? 8 : 4;
  if (C % V != 0 || C / V > kThreads) { eat_set_error("stem wgrad: unsupported channel count"); return EAT_ERR_ARG; }
  const bool rowk = dtype == EAT_F32 && C <= 64 && (stride == 1 || stride == 2);
  if (z != nullptr) {
    if (!rowk) {
      eat_set_error("stem wgrad: the BatchNorm apply on load needs fp32 storage, C <= 64 and stride 1 or 2");
      return EAT_ERR_UNSUPPORTED;
    }
    if (scale == nullptr || shift == nullptr || mean == nullptr || invstd == nullptr || c1 == nullptr || c2 == nullptr) {
      eat_set_error("stem wgrad: the BatchNorm apply on load needs scale, shift, mean, invstd, c1 and c2");
      return EAT_ERR_ARG;
    }
  }
  const long long npix = (long long)B * Fo * To;
  if (npix == 0) return EAT_OK;
  if (npix >= (1ll << 31)) { eat_set_error("stem wgrad: B*Fo*To must be below 2^31"); return EAT_ERR_ARG; }
  const int ppb = kThreads / (C / V);
  if (rowk) {
    const int rows = B * Fo;
    const int grid_r = rows < kNumSMs * 6 ? rows : kNumSMs * 6;
    const BnCtx bn{scale, shift, mean, invstd};
#define EAT_STEM_WG(S_, A_) stem_wgrad_row_kernel<S_, A_><<<grid_r, kThreads, 0, st>>>((const float*)dz, x, dw, B, F, T, Fo, To, C, z, bn, act, c1, c2)
    if (stride == 2) { if (z != nullptr) EAT_STEM_WG(2, 1); else EAT_STEM_WG(2, 0); }
    else { if (z != nullptr) EAT_STEM_WG(1, 1); else EAT_STEM_WG(1, 0); }
#undef EAT_STEM_WG
    EAT_CHECK_LAUNCH();
    return EAT_OK;
  }
  int grid = (int)min((long long)kNumSMs * 4, ceil_div_ll(npix, ppb * 8));
  if (grid < 1) grid = 1;
  size_t smem = (size_t)9 * C * sizeof(float);
  if (dtype == EAT_BF16)
    stem_wgrad_kernel<__nv_bfloat16><<<grid, kThreads, smem, st>>>((const __nv_bfloat16*)dz, x, dw, B, F, T, Fo, To, C, stride);
  else
    stem_wgrad_kernel<float><<<grid, kThreads, smem, st>>>((const float*)dz, x, dw, B, F, T, Fo, To, C, stride);
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

int eat_stem_dgrad(const void* dy, int dtype, const void* z, const float* scale, const float* shift, const float* mean,
                   const float* invstd, int act, const float* c1, const float* c2, const float* w, float* dx, int B, int F,
                   int T, int C, int stride, cudaStream_t st) {
  if (dtype != EAT_F32 && dtype != EAT_BF16) { eat_set_error("stem dgrad: dtype must be EAT_F32 or EAT_BF16"); return EAT_ERR_ARG; }
  const int V = dtype == EAT_BF16 ? 8 : 4;
  if (C < V || C % V != 0 || C / V > kThreads) { eat_set_error("stem dgrad: unsupported channel count"); return EAT_ERR_ARG; }
  if (stride != 1 && stride != 2) { eat_set_error("stem dgrad: stride must be 1 or 2"); return EAT_ERR_UNSUPPORTED; }
  if (act != EAT_ACT_NONE && act != EAT_ACT_RELU && act != EAT_ACT_HSWISH) {
    eat_set_error("stem dgrad: act must be none, relu or hardswish"); return EAT_ERR_ARG;
  }
  if (B < 0 || F < 1 || T < 1) { eat_set_error("stem dgrad: bad sizes"); return EAT_ERR_ARG; }
  if (B == 0) return EAT_OK;
  if (dy == nullptr || z == nullptr || scale == nullptr || shift == nullptr || mean == nullptr || invstd == nullptr ||
      c1 == nullptr || c2 == nullptr || w == nullptr || dx == nullptr) {
    eat_set_error("stem dgrad: dy, z, scale, shift, mean, invstd, c1, c2, w and dx are required"); return EAT_ERR_ARG;
  }
  const long long npix = (long long)B * F * T;
  const int grid = (int)min((long long)kNumSMs * 16, ceil_div_ll(npix, kThreads));
  const BnCtx bn{scale, shift, mean, invstd, act};
#define EAT_STEM_DG(TT, S_) stem_dgrad_kernel<TT, S_><<<grid, kThreads, 0, st>>>((const TT*)dy, (const TT*)z, bn, c1, c2, w, dx, B, F, T, C)
  if (dtype == EAT_BF16) { if (stride == 2) EAT_STEM_DG(__nv_bfloat16, 2); else EAT_STEM_DG(__nv_bfloat16, 1); }
  else { if (stride == 2) EAT_STEM_DG(float, 2); else EAT_STEM_DG(float, 1); }
#undef EAT_STEM_DG
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

int eat_act_bwd(const float* dh, const float* pre, const float* mask, int act, float* dpre, long long n,
                cudaStream_t st) {
  if (n == 0) return EAT_OK;
  int grid = (int)min((long long)kNumSMs * 8, ceil_div_ll(n, 256));
  act_bwd_kernel<<<grid, 256, 0, st>>>(dh, pre, mask, act, dpre, n);
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

}  // extern "C"
