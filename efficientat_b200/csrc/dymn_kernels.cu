// Small kernels of the DyMN context path (reference models/dymn/dy_block.py):
//   ContextGen pooling (:236-237), sequence average pooling (:227-233,249), DynamicConv attention
//   softmax(Linear(h_c)/T) (:104-107) and the per-sample depthwise weight mix (:111-117).
#include <cstdio>
#include <type_traits>

#include "common.cuh"

namespace {

// out[b, pos, c]: pos < F -> mean over t < T_b of x[b, pos, t, c];  pos = F + t -> mean over f of x[b, :, t, c] for
// t < T_b, 0 beyond.  T_b = t_valid[b] with LEN (clips of different lengths, see packed.cu), T without.
template <typename T, bool LEN = false>
__global__ void __launch_bounds__(256) ctx_pool_kernel(const T* __restrict__ x, float* __restrict__ out, int F, int Tn,
                                                       int C, const int* __restrict__ t_valid) {
  constexpr int V = Vec<T>::N;
  const int cv = C / V;
  const int b = blockIdx.y;
  const int tb = LEN ? t_valid[b] : Tn;
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
    } else if (!LEN || pos - F < tb) {
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

// AvgPool (kernel 3, stride s, pad 1, count_include_pad) along a sequence, or a plain copy when stride == 1.
// in: rows [row0, row0 + L) of each sample of a [B, Ltot, H] tensor -> out [B, Lo, H]
__global__ void seq_pool_kernel(const float* __restrict__ in, float* __restrict__ out, int Ltot, int row0, int L, int Lo,
                                int H, int stride, const float* __restrict__ scale, const float* __restrict__ shift,
                                int act) {
  const int b = blockIdx.y;
  const int items = Lo * H;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < items; i += gridDim.x * blockDim.x) {
    const int h = i % H, lo = i / H;
    const float* base = in + ((size_t)b * Ltot + row0) * H + h;
    const float sc = scale != nullptr ? scale[h] : 1.f, sh = scale != nullptr ? shift[h] : 0.f;
    float v;
    if (stride == 1) v = act_fwd(fmaf(base[(size_t)lo * H], sc, sh), scale != nullptr ? act : 0);
    else {
      float acc = 0.f;
#pragma unroll
      for (int d = -1; d <= 1; ++d) {
        const int l = lo * stride + d;
        if (l >= 0 && l < L) acc += act_fwd(fmaf(base[(size_t)l * H], sc, sh), scale != nullptr ? act : 0);
      }
      v = acc * (1.f / 3.f);
    }
    out[((size_t)b * Lo + lo) * H + h] = v;
  }
}

// att[b, :] = softmax((Wr h_c[b] + br) / temperature);  one warp per sample, k <= 4
__global__ void dyconv_att_kernel(const float* __restrict__ hc, const float* __restrict__ wr, const float* __restrict__ br,
                                  float inv_temp, float* __restrict__ att, int B, int H, int k) {
  const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (b >= B) return;
  float logit[4];
  for (int j = 0; j < k; ++j) {
    float acc = 0.f;
    for (int h = lane; h < H; h += 32) acc = fmaf(__ldg(wr + (size_t)j * H + h), hc[(size_t)b * H + h], acc);
    logit[j] = (warp_sum(acc) + br[j]) * inv_temp;
  }
  if (lane == 0) {
    float mx = logit[0];
    for (int j = 1; j < k; ++j) mx = fmaxf(mx, logit[j]);
    float e[4], s = 0.f;
    for (int j = 0; j < k; ++j) { e[j] = expf(logit[j] - mx); s += e[j]; }
    for (int j = 0; j < k; ++j) att[(size_t)b * k + j] = e[j] / s;
  }
}

// wt[b, tap, c] = sum_j att[b, j] * W[j, c, tap]     (W: [k][C][kk] as stored by DynamicConv.weight)
__global__ void dyconv_mix_dw_kernel(const float* __restrict__ w, const float* __restrict__ att, float* __restrict__ wt,
                                     int C, int kk, int k) {
  const int b = blockIdx.y;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < C * kk; i += gridDim.x * blockDim.x) {
    const int c = i / kk, tap = i % kk;
    float acc = 0.f;
    for (int j = 0; j < k; ++j) acc = fmaf(att[(size_t)b * k + j], __ldg(w + (size_t)j * C * kk + i), acc);
    wt[((size_t)b * kk + tap) * C + c] = acc;
  }
}


// ------------------------------------------------------------------------------------------ training path
template <typename T> struct V4;
template <> struct V4<float> {
  __device__ __forceinline__ static void load(const float* p, float (&v)[4]) { float4 t = *reinterpret_cast<const float4*>(p); v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w; }
  __device__ __forceinline__ static void store(float* p, const float (&v)[4]) { *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]); }
};
template <> struct V4<__nv_bfloat16> {
  __device__ __forceinline__ static void load(const __nv_bfloat16* p, float (&v)[4]) {
    uint2 t = *reinterpret_cast<const uint2*>(p);
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&t);
    float2 a = __bfloat1622float2(h[0]), b = __bfloat1622float2(h[1]);
    v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y;
  }
  __device__ __forceinline__ static void store(__nv_bfloat16* p, const float (&v)[4]) {
    __nv_bfloat162 a = __floats2bfloat162_rn(v[0], v[1]), b = __floats2bfloat162_rn(v[2], v[3]);
    uint2 t; t.x = *reinterpret_cast<uint32_t*>(&a); t.y = *reinterpret_cast<uint32_t*>(&b);
    *reinterpret_cast<uint2*>(p) = t;
  }
};

struct DyActCtx {
  const float* scale; const float* shift;   // BatchNorm affine of the depthwise output [C]
  const float* theta;                       // [B, C, 2M] sigmoid(coef_net(h_c)), M = DyReLU-B pieces
  const float* lam; const float* init;      // DyReLU buffers [2M]
  const float* ca_f; const float* ca_t;     // [B, Fo, C], [B, To, C]
};

// DyReLU-B with DM linear pieces (dyrelu_k), theta [B, C, 2 DM] channel-major:
// p = max_m (u a_m + b_m) * ca_f * ca_t,  u = z * scale + shift     (dy_block.py:179-188, 400-402); DM = 1 is the affine
// map u a_0 + b_0
template <typename T, int DM = 2>
__global__ void __launch_bounds__(256) dy_act_fwd_kernel(const T* __restrict__ z, T* __restrict__ out, DyActCtx c, int Fo,
                                                         int To, int C) {
  const int b = blockIdx.y;
  const int cv = C / 4;
  const long long nvec = (long long)Fo * To * cv;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
    const int c0 = (int)(i % cv) * 4;
    const long long pix = i / cv;
    const int to = (int)(pix % To), fo = (int)(pix / To);
    const size_t off = ((size_t)b * Fo * To + pix) * C + c0;
    float v[4];
    V4<T>::load(z + off, v);
    const float4 f4 = *reinterpret_cast<const float4*>(c.ca_f + ((size_t)b * Fo + fo) * C + c0);
    const float4 t4 = *reinterpret_cast<const float4*>(c.ca_t + ((size_t)b * To + to) * C + c0);
    const float q[4] = {f4.x * t4.x, f4.y * t4.y, f4.z * t4.z, f4.w * t4.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      DyCoef<DM> co;
      co.load(c.theta + ((size_t)b * C + c0 + k) * (2 * DM), c.lam, c.init, false);
      v[k] = co.apply(fmaf(v[k], c.scale[c0 + k], c.shift[c0 + k])) * q[k];
    }
    V4<T>::store(out + off, v);
  }
}

// Backward of the above.  CTA = (32 output columns x 32 channels) of one sample, each thread walks all Fo rows of
// its (to, 4-channel) column: d(ca_t) is complete in registers, d(ca_f) and the DyReLU coefficient gradients (2 DM sums
// per channel) are reduced in shared memory and added to global memory once per CTA.  Each pixel's gradient goes to the
// one piece that attains the max (the reference's torch.max(dim=-1) also returns one index): the walk moves on to piece m
// when !(r >= l_m), r the max so far, so a tie stays with the lowest index and a NaN on either side moves on.  At DM = 2
// that is piece 0 iff l_0 >= l_1.
template <typename T, int DM = 2>
__global__ void __launch_bounds__(256) dy_act_bwd_kernel(const T* __restrict__ dp, const T* __restrict__ z, DyActCtx c,
                                                         T* __restrict__ du, float* __restrict__ dcaf,
                                                         float* __restrict__ dcat, float* __restrict__ dcoef, int Fo,
                                                         int To, int C) {
  constexpr int NC = 2 * DM;
  extern __shared__ float smem[];
  float* s_caf = smem;              // [Fo][32]
  float* s_coef = smem + Fo * 32;   // [32][NC]
  const int b = blockIdx.y;
  const int chunks = ceil_div(C, 32);
  const int chunk = blockIdx.x % chunks, tblk = blockIdx.x / chunks;
  const int cvec = threadIdx.x & 7, tslot = threadIdx.x >> 3;
  const int c0 = chunk * 32 + cvec * 4, to = tblk * 32 + tslot;
  for (int i = threadIdx.x; i < Fo * 32 + 32 * NC; i += 256) smem[i] = 0.f;
  __syncthreads();
  const bool live = c0 < C && to < To;
  DyCoef<DM> co[4];
  float sc[4], sh[4], ct[4], g_ct[4], g_a[DM][4], g_b[DM][4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    co[k].zero();
    sc[k] = sh[k] = ct[k] = g_ct[k] = 0.f;
#pragma unroll
    for (int m = 0; m < DM; ++m) g_a[m][k] = g_b[m][k] = 0.f;
  }
  if (live) {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      co[k].load(c.theta + ((size_t)b * C + c0 + k) * NC, c.lam, c.init, false);
      sc[k] = c.scale[c0 + k]; sh[k] = c.shift[c0 + k];
    }
    const float4 t4 = *reinterpret_cast<const float4*>(c.ca_t + ((size_t)b * To + to) * C + c0);
    ct[0] = t4.x; ct[1] = t4.y; ct[2] = t4.z; ct[3] = t4.w;
  }
  // every thread walks the rows (the d(ca_f) partial sums of the four output columns a warp holds for one channel vector
  // are combined with shuffles before they reach shared memory: one atomic per channel and warp instead of four
  // conflicting ones -- shared fp32 atomics are compare-and-swap loops)
  for (int fo = 0; fo < Fo; ++fo) {
    float dcf[4] = {0.f, 0.f, 0.f, 0.f};
    if (live) {
      const size_t off = (((size_t)b * Fo + fo) * To + to) * C + c0;
      float g[4], zv[4], o[4];
      V4<T>::load(dp + off, g);
      V4<T>::load(z + off, zv);
      const float4 f4 = *reinterpret_cast<const float4*>(c.ca_f + ((size_t)b * Fo + fo) * C + c0);
      const float cf[4] = {f4.x, f4.y, f4.z, f4.w};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float u = fmaf(zv[k], sc[k], sh[k]);
        float r = fmaf(u, co[k].a[0], co[k].b[0]), slope = co[k].a[0];
        int arg = 0;
#pragma unroll
        for (int m = 1; m < DM; ++m) {
          const float l = fmaf(u, co[k].a[m], co[k].b[m]);
          if (!(r >= l)) { r = l; slope = co[k].a[m]; arg = m; }
        }
        const float dr = g[k] * cf[k] * ct[k];
        dcf[k] = g[k] * r * ct[k];
        g_ct[k] = fmaf(g[k] * r, cf[k], g_ct[k]);
        o[k] = dr * slope;
#pragma unroll
        for (int m = 0; m < DM; ++m)
          if (arg == m) { g_a[m][k] = fmaf(dr, u, g_a[m][k]); g_b[m][k] += dr; }
      }
      V4<T>::store(du + off, o);
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      dcf[k] += __shfl_xor_sync(0xffffffffu, dcf[k], 8);
      dcf[k] += __shfl_xor_sync(0xffffffffu, dcf[k], 16);
    }
    if ((threadIdx.x & 31) < 8) {
#pragma unroll
      for (int k = 0; k < 4; ++k) atomicAdd(&s_caf[fo * 32 + cvec * 4 + k], dcf[k]);
    }
  }
  // DyReLU coefficient gradients: same shuffle combine, then one atomic per coefficient and warp
#pragma unroll
  for (int k = 0; k < 4; ++k) {
#pragma unroll
    for (int j = 0; j < NC; ++j) {
      float v = j < DM ? g_a[j < DM ? j : 0][k] : g_b[j < DM ? 0 : j - DM][k];
      v += __shfl_xor_sync(0xffffffffu, v, 8);
      v += __shfl_xor_sync(0xffffffffu, v, 16);
      if ((threadIdx.x & 31) < 8) atomicAdd(&s_coef[(cvec * 4 + k) * NC + j], v);
    }
  }
  if (live) {
    float* dct = dcat + ((size_t)b * To + to) * C + c0;
#pragma unroll
    for (int k = 0; k < 4; ++k) dct[k] = g_ct[k];
  }
  __syncthreads();
  for (int i = threadIdx.x; i < Fo * 32; i += 256) {
    const int fo = i / 32, cc = chunk * 32 + (i & 31);
    if (cc < C) atomicAdd(dcaf + ((size_t)b * Fo + fo) * C + cc, s_caf[i]);
  }
  if (threadIdx.x < 32 * NC) {
    const int cc = chunk * 32 + threadIdx.x / NC;
    if (cc < C) atomicAdd(dcoef + ((size_t)b * C + cc) * NC + threadIdx.x % NC, s_coef[threadIdx.x]);
  }
}

// dpre[b,c,j] = dcoef[b,c,j] * lam[j] * 2 * s (1 - s),  s = theta[b,c,j], j < 2 DM      (DyReLU coefficient net,
// dy_block.py:157-160,179)
template <int DM = 2>
__global__ void dyrelu_coef_bwd_kernel(const float* __restrict__ dcoef, const float* __restrict__ theta,
                                       const float* __restrict__ lam, float* __restrict__ dpre, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float s = theta[i];
    dpre[i] = dcoef[i] * lam[i % (2 * DM)] * 2.f * s * (1.f - s);
  }
}
// out = g * s * (1 - s)
__global__ void sigmoid_bwd_kernel(const float* __restrict__ g, const float* __restrict__ s, float* __restrict__ out, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float v = s[i];
    out[i] = g[i] * v * (1.f - v);
  }
}

// softmax(Linear(h_c)/T) backward, one warp per sample: dlogit_j = att_j (datt_j - sum_i att_i datt_i) / T;
// dWr += dlogit^T h_c, dbr += dlogit, dh_c[b,:] += dlogit . Wr
__global__ void dyconv_att_bwd_kernel(const float* __restrict__ datt, const float* __restrict__ att, float inv_temp,
                                      const float* __restrict__ hc, const float* __restrict__ wr, float* __restrict__ dwr,
                                      float* __restrict__ dbr, float* __restrict__ dhc, int B, int H, int k) {
  const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (b >= B) return;
  float dl[4] = {0.f, 0.f, 0.f, 0.f};
  float dot = 0.f;
  for (int j = 0; j < k; ++j) dot = fmaf(att[(size_t)b * k + j], datt[(size_t)b * k + j], dot);
  for (int j = 0; j < k; ++j) dl[j] = att[(size_t)b * k + j] * (datt[(size_t)b * k + j] - dot) * inv_temp;
  for (int h = lane; h < H; h += 32) {
    const float x = hc[(size_t)b * H + h];
    float acc = 0.f;
    for (int j = 0; j < k; ++j) { atomicAdd(dwr + (size_t)j * H + h, dl[j] * x); acc = fmaf(dl[j], wr[(size_t)j * H + h], acc); }
    dhc[(size_t)b * H + h] += acc;
  }
  if (lane < k) atomicAdd(dbr + lane, dl[lane]);
}

// transposed sequence pooling: dsrc rows [row0, row0+L) of a [B, Ltot, H] tensor <- d(out [B, Lo, H])
__global__ void seq_pool_bwd_kernel(const float* __restrict__ dout, float* __restrict__ dsrc, int Ltot, int row0, int L,
                                    int Lo, int H, int stride) {
  const int b = blockIdx.y;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < L * H; i += gridDim.x * blockDim.x) {
    const int h = i % H, l = i / H;
    const float* g = dout + (size_t)b * Lo * H + h;
    float v = 0.f;
    if (stride == 1) v = g[(size_t)l * H];
    else {
      for (int lo = 0; lo < Lo; ++lo) { const int d = l - lo * stride; if (d >= -1 && d <= 1) v += g[(size_t)lo * H]; }
      v *= (1.f / 3.f);
    }
    dsrc[((size_t)b * Ltot + row0 + l) * H + h] = v;
  }
}

// dx[b,f,t,c] += dg[b,f,c] / T + dg[b,F+t,c] / F        (gradient of the ContextGen pooling)
template <typename T>
__global__ void __launch_bounds__(256) ctx_pool_bwd_kernel(const float* __restrict__ dg, T* __restrict__ dx, int F, int Tn,
                                                           int C) {
  const int b = blockIdx.y;
  const int cv = C / 4;
  const long long nvec = (long long)F * Tn * cv;
  const float it = 1.f / Tn, iff = 1.f / F;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
    const int c0 = (int)(i % cv) * 4;
    const long long pix = i / cv;
    const int t = (int)(pix % Tn), f = (int)(pix / Tn);
    const size_t off = ((size_t)b * F * Tn + pix) * C + c0;
    float v[4];
    V4<T>::load(dx + off, v);
    const float4 gf = *reinterpret_cast<const float4*>(dg + ((size_t)b * (F + Tn) + f) * C + c0);
    const float4 gt = *reinterpret_cast<const float4*>(dg + ((size_t)b * (F + Tn) + F + t) * C + c0);
    v[0] += gf.x * it + gt.x * iff; v[1] += gf.y * it + gt.y * iff; v[2] += gf.z * it + gt.z * iff; v[3] += gf.w * it + gt.w * iff;
    V4<T>::store(dx + off, v);
  }
}

// DynamicConv weight/attention gradients from per-sample weight gradients S [B, n]:
//   dW[k, i] += sum_b att[b,k] S[b,i]           datt[b,k] = sum_i S[b,i] W[k,i]
// Both passes stream S (B * n floats: 315 MB for the widest dymn20 layer at B = 128): 16-byte loads, four samples / two
// positions in flight per thread.
__global__ void __launch_bounds__(256) dyn_wgrad_mix_kernel(const float* __restrict__ S, const float* __restrict__ att,
                                                            float* __restrict__ dW, int B, long long n, int k) {
  extern __shared__ float s_att[];                     // [B][4]
  for (int i = threadIdx.x; i < B * 4; i += 256) s_att[i] = (i & 3) < k ? att[(size_t)(i >> 2) * k + (i & 3)] : 0.f;
  __syncthreads();
  const long long n4 = n >> 2;                         // n is a multiple of 4 (N, K multiples of 4)
  for (long long i4 = (long long)blockIdx.x * blockDim.x + threadIdx.x; i4 < n4; i4 += (long long)gridDim.x * blockDim.x) {
    float4 acc[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[j] = make_float4(0.f, 0.f, 0.f, 0.f);
    const float4* Sp = reinterpret_cast<const float4*>(S) + i4;
    int b = 0;
    for (; b + 3 < B; b += 4) {
      float4 sv[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) sv[u] = __ldg(Sp + (size_t)(b + u) * n4);
#pragma unroll
      for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float a = s_att[(b + u) * 4 + j];
          acc[j].x = fmaf(a, sv[u].x, acc[j].x); acc[j].y = fmaf(a, sv[u].y, acc[j].y);
          acc[j].z = fmaf(a, sv[u].z, acc[j].z); acc[j].w = fmaf(a, sv[u].w, acc[j].w);
        }
    }
    for (; b < B; ++b) {
      const float4 sv = __ldg(Sp + (size_t)b * n4);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float a = s_att[b * 4 + j];
        acc[j].x = fmaf(a, sv.x, acc[j].x); acc[j].y = fmaf(a, sv.y, acc[j].y);
        acc[j].z = fmaf(a, sv.z, acc[j].z); acc[j].w = fmaf(a, sv.w, acc[j].w);
      }
    }
    for (int j = 0; j < k; ++j) {
      float4* d = reinterpret_cast<float4*>(dW + (size_t)j * n) + i4;
      float4 o = *d;
      o.x += acc[j].x; o.y += acc[j].y; o.z += acc[j].z; o.w += acc[j].w;
      *d = o;
    }
  }
}
// grid (chunks, B): each CTA reduces one slice of sample b and adds its four partial sums to datt (zeroed by the launcher)
__global__ void __launch_bounds__(256) dyn_datt_kernel(const float* __restrict__ S, const float* __restrict__ W,
                                                       float* __restrict__ datt, long long n, int k) {
  const int b = blockIdx.y;
  const long long n4 = n >> 2;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  const float4* Sp = reinterpret_cast<const float4*>(S + (size_t)b * n);
  for (long long i4 = (long long)blockIdx.x * 256 + threadIdx.x; i4 < n4; i4 += (long long)gridDim.x * 256) {
    const float4 sv = __ldg(Sp + i4);
    float4 wv[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) wv[j] = j < k ? __ldg(reinterpret_cast<const float4*>(W + (size_t)j * n) + i4) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[j] += sv.x * wv[j].x + sv.y * wv[j].y + sv.z * wv[j].z + sv.w * wv[j].w;
  }
  __shared__ float red[8][4];
  for (int j = 0; j < 4; ++j) acc[j] = warp_sum(acc[j]);
  if ((threadIdx.x & 31) == 0) for (int j = 0; j < 4; ++j) red[threadIdx.x >> 5][j] = acc[j];
  __syncthreads();
  if (threadIdx.x < k) {
    float s = 0.f;
    for (int w = 0; w < 8; ++w) s += red[w][threadIdx.x];
    atomicAdd(datt + (size_t)b * k + threadIdx.x, s);
  }
}
__global__ void zero_kernel(float* __restrict__ p, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = 0.f;
}

inline int ew_grid(long long n) { long long g = ceil_div_ll(n, 256); return (int)(g > kNumSMs * 16 ? kNumSMs * 16 : (g < 1 ? 1 : g)); }

// f(std::integral_constant<int, M>{}) for M = pieces, which the caller has checked to be 1..4
template <typename Fn>
void with_pieces(int pieces, Fn&& f) {
  switch (pieces) {
    case 1: f(std::integral_constant<int, 1>{}); break;
    case 2: f(std::integral_constant<int, 2>{}); break;
    case 3: f(std::integral_constant<int, 3>{}); break;
    default: f(std::integral_constant<int, 4>{}); break;
  }
}

// launchers of the DyReLU-B kernels, shared by the entry points with 2 and with `pieces` linear pieces; B >= 1
int dy_act_fwd_launch(const void* z, void* out, int dtype, DyActCtx c, int pieces, int B, int Fo, int To, int C,
                      cudaStream_t st) {
  dim3 grid(max(1, min(kNumSMs * 8 / max(B, 1) + 1, (int)ceil_div_ll((long long)Fo * To * (C / 4), 256))), B);
  with_pieces(pieces, [&](auto dm) {
    constexpr int DM = decltype(dm)::value;
    if (dtype == EAT_BF16) dy_act_fwd_kernel<__nv_bfloat16, DM><<<grid, 256, 0, st>>>((const __nv_bfloat16*)z, (__nv_bfloat16*)out, c, Fo, To, C);
    else dy_act_fwd_kernel<float, DM><<<grid, 256, 0, st>>>((const float*)z, (float*)out, c, Fo, To, C);
  });
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

int dy_act_bwd_launch(const void* dp, const void* z, void* du, int dtype, DyActCtx c, float* dcaf, float* dcat,
                      float* dcoef, int pieces, int B, int Fo, int To, int C, cudaStream_t st) {
  dim3 grid(ceil_div(C, 32) * ceil_div(To, 32), B);
  const size_t smem = ((size_t)Fo * 32 + 32 * 2 * pieces) * sizeof(float);
  with_pieces(pieces, [&](auto dm) {
    constexpr int DM = decltype(dm)::value;
    if (dtype == EAT_BF16)
      dy_act_bwd_kernel<__nv_bfloat16, DM><<<grid, 256, smem, st>>>((const __nv_bfloat16*)dp, (const __nv_bfloat16*)z, c, (__nv_bfloat16*)du, dcaf, dcat, dcoef, Fo, To, C);
    else
      dy_act_bwd_kernel<float, DM><<<grid, 256, smem, st>>>((const float*)dp, (const float*)z, c, (float*)du, dcaf, dcat, dcoef, Fo, To, C);
  });
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

int dyrelu_coef_bwd_launch(const float* dcoef, const float* theta, const float* lam, float* dpre, long long n,
                           int pieces, cudaStream_t st) {
  with_pieces(pieces, [&](auto dm) {
    dyrelu_coef_bwd_kernel<decltype(dm)::value><<<ew_grid(n), 256, 0, st>>>(dcoef, theta, lam, dpre, n);
  });
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

}  // namespace

extern "C" {

int eat_ctx_pool(const void* x, int dtype, float* out, int B, int F, int T, int C, cudaStream_t st) {
  if (B == 0) return EAT_OK;
  const int V = dtype == EAT_BF16 ? 8 : 4;
  if (C % V != 0) { eat_set_error("ctx_pool: channels must be a multiple of the vector width"); return EAT_ERR_ARG; }
  dim3 grid(ceil_div((F + T) * (C / V), 256), B);
  if (dtype == EAT_BF16) ctx_pool_kernel<__nv_bfloat16><<<grid, 256, 0, st>>>((const __nv_bfloat16*)x, out, F, T, C, nullptr);
  else ctx_pool_kernel<float><<<grid, 256, 0, st>>>((const float*)x, out, F, T, C, nullptr);
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
  if (dtype == EAT_BF16) ctx_pool_kernel<__nv_bfloat16, true><<<grid, 256, 0, st>>>((const __nv_bfloat16*)x, out, F, T, C, t_valid);
  else ctx_pool_kernel<float, true><<<grid, 256, 0, st>>>((const float*)x, out, F, T, C, t_valid);
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

// shared by eat_seq_pool / eat_seq_pool_bwd: the window [row0, row0 + L) must lie inside [0, Ltot), and the pooling
// stride must be positive (1 = copy, otherwise AvgPool(3, stride, pad 1))
static int seq_pool_check(int B, int Ltot, int row0, int L, int H, int stride) {
  if (stride < 1) { eat_set_error("seq_pool: stride must be at least 1"); return EAT_ERR_ARG; }
  if (B < 0 || L < 1 || H < 1 || row0 < 0 || (long long)row0 + L > Ltot) {
    eat_set_error("seq_pool: rows [row0, row0 + L) must lie inside [0, Ltot), with L >= 1 and H >= 1");
    return EAT_ERR_ARG;
  }
  return EAT_OK;
}

int eat_seq_pool(const float* in, float* out, int B, int Ltot, int row0, int L, int H, int stride, const float* scale,
                 const float* shift, int act, cudaStream_t st) {
  if (B == 0) return EAT_OK;
  if (int rc = seq_pool_check(B, Ltot, row0, L, H, stride)) return rc;
  const int Lo = stride == 1 ? L : (L + 2 - 3) / stride + 1;
  dim3 grid(ceil_div(Lo * H, 256), B);
  seq_pool_kernel<<<grid, 256, 0, st>>>(in, out, Ltot, row0, L, Lo, H, stride, scale, shift, act);
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

int eat_dyconv_att(const float* hc, const float* wr, const float* br, float temperature, float* att, int B, int H, int k,
                   cudaStream_t st) {
  if (B == 0) return EAT_OK;
  if (k < 1 || k > 4) { eat_set_error("dyconv_att: 1..4 kernels supported"); return EAT_ERR_UNSUPPORTED; }
  dyconv_att_kernel<<<ceil_div(B, 4), 128, 0, st>>>(hc, wr, br, 1.f / temperature, att, B, H, k);
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

int eat_dyconv_mix_dw(const float* w, const float* att, float* wt, int B, int C, int ksize, int k, cudaStream_t st) {
  if (B == 0) return EAT_OK;
  dim3 grid(ceil_div(C * ksize * ksize, 256), B);
  dyconv_mix_dw_kernel<<<grid, 256, 0, st>>>(w, att, wt, C, ksize * ksize, k);
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}


int eat_dy_act_fwd(const void* z, void* out, int dtype, const float* scale, const float* shift, const float* theta,
                   const float* lam, const float* init, const float* ca_f, const float* ca_t, int B, int Fo, int To,
                   int C, cudaStream_t st) {
  if (B == 0) return EAT_OK;
  if (C % 4 != 0) { eat_set_error("dy_act: channels must be a multiple of 4"); return EAT_ERR_ARG; }
  return dy_act_fwd_launch(z, out, dtype, DyActCtx{scale, shift, theta, lam, init, ca_f, ca_t}, 2, B, Fo, To, C, st);
}

int eat_dy_act_bwd(const void* dp, const void* z, void* du, int dtype, const float* scale, const float* shift,
                   const float* theta, const float* lam, const float* init, const float* ca_f, const float* ca_t,
                   float* dcaf, float* dcat, float* dcoef, int B, int Fo, int To, int C, cudaStream_t st) {
  if (B == 0) return EAT_OK;
  if (C % 4 != 0) { eat_set_error("dy_act: channels must be a multiple of 4"); return EAT_ERR_ARG; }
  return dy_act_bwd_launch(dp, z, du, dtype, DyActCtx{scale, shift, theta, lam, init, ca_f, ca_t}, dcaf, dcat, dcoef, 2,
                           B, Fo, To, C, st);
}

int eat_dyrelu_coef_bwd(const float* dcoef, const float* theta, const float* lam, float* dpre, long long n, cudaStream_t st) {
  if (n == 0) return EAT_OK;
  return dyrelu_coef_bwd_launch(dcoef, theta, lam, dpre, n, 2, st);
}

// argument checks of the DyReLU-B entry points with M pieces, before any launch
static int dym_check(const char* who, int dtype, int B, int Fo, int To, int C, int pieces, bool null_ptr) {
  char msg[160];
  int rc = EAT_OK;
  if (pieces < 1 || pieces > 4) {
    snprintf(msg, sizeof msg, "%s: DyReLU-B takes 1..4 linear pieces (got %d)", who, pieces);
    rc = EAT_ERR_UNSUPPORTED;
  } else if (dtype != EAT_F32 && dtype != EAT_BF16) { snprintf(msg, sizeof msg, "%s: dtype must be fp32 (0) or bf16 (1)", who); rc = EAT_ERR_ARG; }
  else if (B < 0 || Fo < 1 || To < 1 || C < 1) { snprintf(msg, sizeof msg, "%s: B >= 0 and Fo, To, C >= 1 required", who); rc = EAT_ERR_ARG; }
  else if (C % 4 != 0) { snprintf(msg, sizeof msg, "%s: channels must be a multiple of 4 (got %d)", who, C); rc = EAT_ERR_ARG; }
  else if (null_ptr) { snprintf(msg, sizeof msg, "%s: every tensor pointer is required", who); rc = EAT_ERR_ARG; }
  if (rc != EAT_OK) eat_set_error(msg);
  return rc;
}

int eat_dy_act_fwd_m(const void* z, void* out, int dtype, const float* scale, const float* shift, const float* theta,
                     const float* lam, const float* init, const float* ca_f, const float* ca_t, int pieces, int B, int Fo,
                     int To, int C, cudaStream_t st) {
  const bool null_ptr = !z || !out || !scale || !shift || !theta || !lam || !init || !ca_f || !ca_t;
  if (int rc = dym_check("dy_act_fwd_m", dtype, B, Fo, To, C, pieces, null_ptr)) return rc;
  if (B == 0) return EAT_OK;
  return dy_act_fwd_launch(z, out, dtype, DyActCtx{scale, shift, theta, lam, init, ca_f, ca_t}, pieces, B, Fo, To, C, st);
}

int eat_dy_act_bwd_m(const void* dp, const void* z, void* du, int dtype, const float* scale, const float* shift,
                     const float* theta, const float* lam, const float* init, const float* ca_f, const float* ca_t,
                     float* dcaf, float* dcat, float* dcoef, int pieces, int B, int Fo, int To, int C, cudaStream_t st) {
  const bool null_ptr = !dp || !z || !du || !scale || !shift || !theta || !lam || !init || !ca_f || !ca_t || !dcaf ||
                        !dcat || !dcoef;
  if (int rc = dym_check("dy_act_bwd_m", dtype, B, Fo, To, C, pieces, null_ptr)) return rc;
  if (B == 0) return EAT_OK;
  return dy_act_bwd_launch(dp, z, du, dtype, DyActCtx{scale, shift, theta, lam, init, ca_f, ca_t}, dcaf, dcat, dcoef,
                           pieces, B, Fo, To, C, st);
}

int eat_dyrelu_coef_bwd_m(const float* dcoef, const float* theta, const float* lam, float* dpre, long long n, int pieces,
                          cudaStream_t st) {
  char msg[128];
  if (pieces < 1 || pieces > 4) {
    snprintf(msg, sizeof msg, "dyrelu_coef_bwd_m: DyReLU-B takes 1..4 linear pieces (got %d)", pieces);
    eat_set_error(msg);
    return EAT_ERR_UNSUPPORTED;
  }
  if (n < 0 || n % (2 * pieces) != 0) {
    snprintf(msg, sizeof msg, "dyrelu_coef_bwd_m: n must be a non-negative multiple of 2M = %d (got %lld)", 2 * pieces, n);
    eat_set_error(msg);
    return EAT_ERR_ARG;
  }
  if (!dcoef || !theta || !lam || !dpre) { eat_set_error("dyrelu_coef_bwd_m: every tensor pointer is required"); return EAT_ERR_ARG; }
  if (n == 0) return EAT_OK;
  return dyrelu_coef_bwd_launch(dcoef, theta, lam, dpre, n, pieces, st);
}

int eat_sigmoid_bwd(const float* g, const float* s, float* out, long long n, cudaStream_t st) {
  if (n == 0) return EAT_OK;
  sigmoid_bwd_kernel<<<ew_grid(n), 256, 0, st>>>(g, s, out, n);
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

int eat_dyconv_att_bwd(const float* datt, const float* att, float temperature, const float* hc, const float* wr,
                       float* dwr, float* dbr, float* dhc, int B, int H, int k, cudaStream_t st) {
  if (B == 0) return EAT_OK;
  if (k < 1 || k > 4) { eat_set_error("dyconv_att_bwd: 1..4 kernels supported"); return EAT_ERR_UNSUPPORTED; }
  dyconv_att_bwd_kernel<<<ceil_div(B, 4), 128, 0, st>>>(datt, att, 1.f / temperature, hc, wr, dwr, dbr, dhc, B, H, k);
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

int eat_seq_pool_bwd(const float* dout, float* dsrc, int B, int Ltot, int row0, int L, int H, int stride, cudaStream_t st) {
  if (B == 0) return EAT_OK;
  if (int rc = seq_pool_check(B, Ltot, row0, L, H, stride)) return rc;
  const int Lo = stride == 1 ? L : (L + 2 - 3) / stride + 1;
  dim3 grid(ceil_div(L * H, 256), B);
  seq_pool_bwd_kernel<<<grid, 256, 0, st>>>(dout, dsrc, Ltot, row0, L, Lo, H, stride);
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

int eat_ctx_pool_bwd(const float* dg, void* dx, int dtype, int B, int F, int T, int C, cudaStream_t st) {
  if (B == 0) return EAT_OK;
  if (C % 4 != 0) { eat_set_error("ctx_pool_bwd: channels must be a multiple of 4"); return EAT_ERR_ARG; }
  dim3 grid(max(1, min(kNumSMs * 8 / max(B, 1) + 1, (int)ceil_div_ll((long long)F * T * (C / 4), 256))), B);
  if (dtype == EAT_BF16) ctx_pool_bwd_kernel<__nv_bfloat16><<<grid, 256, 0, st>>>(dg, (__nv_bfloat16*)dx, F, T, C);
  else ctx_pool_bwd_kernel<float><<<grid, 256, 0, st>>>(dg, (float*)dx, F, T, C);
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

int eat_dyn_wgrad_mix(const float* S, const float* att, const float* W, float* dW, float* datt, int B, long long n, int k,
                      cudaStream_t st) {
  if (B == 0 || n == 0) return EAT_OK;
  if (k < 1 || k > 4) { eat_set_error("dyn_wgrad_mix: 1..4 kernels supported"); return EAT_ERR_UNSUPPORTED; }
  if ((n & 3) != 0 || ((((uintptr_t)S) | ((uintptr_t)W) | ((uintptr_t)dW)) & 15)) { eat_set_error("dyn_wgrad_mix: n must be a multiple of 4 and the tensors 16-byte aligned"); return EAT_ERR_ARG; }
  const long long n4 = n >> 2;
  const int gmix = (int)min((long long)kNumSMs * 8, ceil_div_ll(n4, 256));
  dyn_wgrad_mix_kernel<<<gmix, 256, (size_t)B * 4 * sizeof(float), st>>>(S, att, dW, B, n, k);
  zero_kernel<<<ceil_div(B * k, 256), 256, 0, st>>>(datt, B * k);
  int chunks = (int)min((long long)max(1, (kNumSMs * 8) / B), ceil_div_ll(n4, 256 * 4));
  if (chunks < 1) chunks = 1;
  dyn_datt_kernel<<<dim3(chunks, B), 256, 0, st>>>(S, W, datt, n, k);
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

}  // extern "C"
