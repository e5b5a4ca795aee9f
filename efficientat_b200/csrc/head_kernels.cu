// Multi-head attention pooling classifier head (PSLA), reference models/mn/attention_pooling.py:9-56 with the
// defaults MN builds it with (att_activation 'sigmoid', clf_activation 'ident', epsilon 1e-7):
//   m   = mean_f x                     [B, T, C]        (collapse_dim, mn/utils.py:29-41)
//   P   = m . W^T + b                  [B*T, 2*H*K]     column j = s*H*K + h*K + k, s = 0 attention, 1 value
//   a   = clamp(sigmoid(P_att), eps, 1 - eps)
//   out[b,k] = sum_h hw[h] * sum_t a[b,h,t,k] v[b,h,t,k] / sum_t a[b,h,t,k]
// The projection GEMM is the package's 1x1-conv GEMM; this file has the frequency mean (and its backward broadcast) and
// the attention-normalised sum over time (and its backward).
#include <cstdio>

#include "common.cuh"

namespace {

constexpr int kPoolThreads = 128;
constexpr int kAttX = 32;      // classes per CTA: one warp reads 32 consecutive columns of P (128 B)
constexpr int kAttY = 8;       // samples per CTA

// one thread per (sample, vector of V channels): walks t, sums the F rows of each t, writes m and the running total
// over (F, T) for the features output.  scale != nullptr: BatchNorm affine + activation applied on load.
template <typename T>
__global__ void __launch_bounds__(kPoolThreads) freq_pool_kernel(const T* __restrict__ x, const float* __restrict__ scale,
                                                                 const float* __restrict__ shift, int act,
                                                                 float* __restrict__ m, float* __restrict__ feat, int B,
                                                                 int F, int Tn, int C) {
  constexpr int V = Vec<T>::N;
  const int nv = C / V;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)B * nv) return;
  const int b = (int)(idx / nv), c = (int)(idx % nv) * V;
  float sc[V], sh[V];
  if (scale != nullptr) {
#pragma unroll
    for (int i = 0; i < V; ++i) { sc[i] = scale[c + i]; sh[i] = shift[c + i]; }
  }
  const float inv_f = 1.f / (float)F;
  float tot[V];
#pragma unroll
  for (int i = 0; i < V; ++i) tot[i] = 0.f;
  const long long fstride = (long long)Tn * C;
  for (int t = 0; t < Tn; ++t) {
    const T* p = x + ((long long)b * F * Tn + t) * C + c;
    float s[V];
#pragma unroll
    for (int i = 0; i < V; ++i) s[i] = 0.f;
#pragma unroll 4
    for (int f = 0; f < F; ++f) {
      float v[V];
      Vec<T>::load(p + f * fstride, v);
#pragma unroll
      for (int i = 0; i < V; ++i) s[i] += scale != nullptr ? act_fwd(fmaf(v[i], sc[i], sh[i]), act) : v[i];
    }
    float* mo = m + ((long long)b * Tn + t) * C + c;
#pragma unroll
    for (int i = 0; i < V; i += 4)
      *reinterpret_cast<float4*>(mo + i) = make_float4(s[i] * inv_f, s[i + 1] * inv_f, s[i + 2] * inv_f, s[i + 3] * inv_f);
#pragma unroll
    for (int i = 0; i < V; ++i) tot[i] += s[i];
  }
  if (feat != nullptr) {
    const float inv = 1.f / ((float)F * (float)Tn);
    float* fo = feat + (long long)b * C + c;
#pragma unroll
    for (int i = 0; i < V; i += 4)
      *reinterpret_cast<float4*>(fo + i) = make_float4(tot[i] * inv, tot[i + 1] * inv, tot[i + 2] * inv, tot[i + 3] * inv);
  }
}

// dx[b, f, t, c] = dm[b, t, c] * mul for every f: one thread per (sample, t, vector of V channels)
template <typename T>
__global__ void __launch_bounds__(256) freq_pool_bwd_kernel(const float* __restrict__ dm, float mul, T* __restrict__ dx,
                                                            int F, int Tn, int C, long long n_vec) {
  constexpr int V = Vec<T>::N;
  const int nv = C / V;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_vec; i += (long long)gridDim.x * blockDim.x) {
    const long long bt = i / nv;
    const int c = (int)(i % nv) * V;
    const long long b = bt / Tn;
    const int t = (int)(bt % Tn);
    float v[V];
    const float* src = dm + bt * C + c;
#pragma unroll
    for (int j = 0; j < V; j += 4) {
      const float4 q = *reinterpret_cast<const float4*>(src + j);
      v[j] = q.x * mul; v[j + 1] = q.y * mul; v[j + 2] = q.z * mul; v[j + 3] = q.w * mul;
    }
    T* dst = dx + (b * F * Tn + t) * C + c;
    for (int f = 0; f < F; ++f) Vec<T>::store(dst + (long long)f * Tn * C, v);
  }
}

__device__ __forceinline__ float att_of(float s, float eps, float hi) { return fminf(fmaxf(s, eps), hi); }

// one thread per (sample, class): for each head, one walk over t gives S_a = sum a and sum a*v.  kLen
// (eat_att_pool_fwd_len): sample b's walk stops at t_valid[b]
template <bool kLen>
__device__ __forceinline__ void att_pool_fwd_body(const float* __restrict__ P, const float* __restrict__ hw, float eps,
                                                  float hi, float* __restrict__ out, float* __restrict__ sa_out,
                                                  float* __restrict__ r_out, int B, int Tn, int H, int K,
                                                  const int* __restrict__ t_valid) {
  const int k = blockIdx.x * kAttX + threadIdx.x;
  const int b = blockIdx.y * kAttY + threadIdx.y;
  if (k >= K || b >= B) return;
  const long long ld = 2LL * H * K;
  const float* base = P + (long long)b * Tn * ld + k;
  int tb = Tn;
  if constexpr (kLen) tb = t_valid[b];
  float acc = 0.f;
  for (int h = 0; h < H; ++h) {
    const float* pa = base + (long long)h * K;
    const float* pv = pa + (long long)H * K;
    float sa = 0.f, sav = 0.f;
#pragma unroll 4
    for (int t = 0; t < tb; ++t) {
      const float a = att_of(sigmoidf_(pa[t * ld]), eps, hi);
      sa += a;
      sav = fmaf(a, pv[t * ld], sav);
    }
    const float r = sav / sa;
    acc = fmaf(hw[h], r, acc);
    if (sa_out != nullptr) {
      const long long o = ((long long)b * H + h) * K + k;
      sa_out[o] = sa;
      r_out[o] = r;
    }
  }
  out[(long long)b * K + k] = acc;
}

__global__ void __launch_bounds__(kAttX * kAttY) att_pool_fwd_kernel(const float* __restrict__ P, const float* __restrict__ hw,
                                                                    float eps, float hi, float* __restrict__ out,
                                                                    float* __restrict__ sa_out, float* __restrict__ r_out,
                                                                    int B, int Tn, int H, int K) {
  att_pool_fwd_body<false>(P, hw, eps, hi, out, sa_out, r_out, B, Tn, H, K, nullptr);
}

__global__ void __launch_bounds__(kAttX * kAttY) att_pool_fwd_len_kernel(const float* __restrict__ P,
                                                                        const float* __restrict__ hw, float eps, float hi,
                                                                        float* __restrict__ out, int B, int Tn, int H,
                                                                        int K, const int* __restrict__ t_valid) {
  att_pool_fwd_body<true>(P, hw, eps, hi, out, nullptr, nullptr, B, Tn, H, K, t_valid);
}

// dv = g a, da = g (v - r), g = dout hw / S_a; dP_att = da * sigmoid'(x) where the clamp passes (eps <= sigmoid(x) <= 1-eps,
// torch.clamp's gradient mask), dP_val = dv.  dP may alias P: every element is read, then written, by the same thread.
// dbias[j] += sum_{b,t} dP[., j] and dhw[h] += sum_{b,k} dout r are reduced over the CTA's samples in shared memory first.
__global__ void __launch_bounds__(kAttX * kAttY) att_pool_bwd_kernel(const float* __restrict__ dout, const float* P, float* dP,
                                                                    const float* __restrict__ hw, const float* __restrict__ sa_in,
                                                                    const float* __restrict__ r_in, float eps, float hi,
                                                                    float* __restrict__ dhw, float* __restrict__ dbias, int B,
                                                                    int Tn, int H, int K) {
  __shared__ float red[3][kAttY][kAttX];
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int k = blockIdx.x * kAttX + tx;
  const int b = blockIdx.y * kAttY + ty;
  const bool live = k < K && b < B;
  const long long ld = 2LL * H * K;
  const long long row0 = (long long)b * Tn * ld + k;
  const float d = live ? dout[(long long)b * K + k] : 0.f;
  for (int h = 0; h < H; ++h) {
    float sum_a = 0.f, sum_v = 0.f, dh = 0.f;
    if (live) {
      const long long o = ((long long)b * H + h) * K + k;
      const float r = r_in[o];
      const float g = d * hw[h] / sa_in[o];
      dh = d * r;
      const long long ja = row0 + (long long)h * K, jv = ja + (long long)H * K;
#pragma unroll 4
      for (int t = 0; t < Tn; ++t) {
        const float x = P[ja + t * ld], v = P[jv + t * ld];
        const float s = sigmoidf_(x);
        const float a = att_of(s, eps, hi);
        const float ga = (s >= eps && s <= hi) ? g * (v - r) * s * (1.f - s) : 0.f;
        const float gv = g * a;
        dP[ja + t * ld] = ga;
        dP[jv + t * ld] = gv;
        sum_a += ga;
        sum_v += gv;
      }
    }
    red[0][ty][tx] = sum_a;
    red[1][ty][tx] = sum_v;
    red[2][ty][tx] = dh;
    __syncthreads();
    if (ty == 0) {
      float s0 = 0.f, s1 = 0.f, s2 = 0.f;
#pragma unroll
      for (int y = 0; y < kAttY; ++y) { s0 += red[0][y][tx]; s1 += red[1][y][tx]; s2 += red[2][y][tx]; }
      if (k < K) {
        atomicAdd(dbias + (long long)h * K + k, s0);
        atomicAdd(dbias + (long long)(H + h) * K + k, s1);
      }
      s2 = warp_sum(s2);
      if (tx == 0) atomicAdd(dhw + h, s2);
    }
    __syncthreads();
  }
}

bool misaligned(const void* p) { return ((uintptr_t)p & 15) != 0; }

}  // namespace

extern "C" {

int eat_freq_pool(const void* x, int dtype, const float* scale, const float* shift, int act, float* m, float* feat, int B,
                  int F, int T, int C, cudaStream_t st) {
  if (B < 0 || F < 1 || T < 1 || C < 1) { eat_set_error("freq_pool: need B >= 0 and F, T, C >= 1"); return EAT_ERR_ARG; }
  if (dtype != EAT_F32 && dtype != EAT_BF16) { eat_set_error("freq_pool: dtype must be EAT_F32 or EAT_BF16"); return EAT_ERR_ARG; }
  if (act < EAT_ACT_NONE || act > EAT_ACT_HSWISH) { eat_set_error("freq_pool: act must be none, relu or hardswish"); return EAT_ERR_ARG; }
  if ((scale == nullptr) != (shift == nullptr)) { eat_set_error("freq_pool: scale and shift go together"); return EAT_ERR_ARG; }
  const int V = dtype == EAT_BF16 ? 8 : 4;
  if (C % V != 0) { eat_set_error("freq_pool: channels must be a multiple of the vector width (4 fp32, 8 bf16)"); return EAT_ERR_ARG; }
  if (B == 0) return EAT_OK;
  if (x == nullptr || m == nullptr) { eat_set_error("freq_pool: x and m are required"); return EAT_ERR_ARG; }
  if (misaligned(x) || misaligned(m) || misaligned(feat)) { eat_set_error("freq_pool: x, m and feat must be 16-byte aligned"); return EAT_ERR_ARG; }
  const long long threads = (long long)B * (C / V);
  const unsigned grid = (unsigned)ceil_div_ll(threads, kPoolThreads);
  if (dtype == EAT_BF16)
    freq_pool_kernel<__nv_bfloat16><<<grid, kPoolThreads, 0, st>>>((const __nv_bfloat16*)x, scale, shift, act, m, feat, B, F, T, C);
  else
    freq_pool_kernel<float><<<grid, kPoolThreads, 0, st>>>((const float*)x, scale, shift, act, m, feat, B, F, T, C);
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

int eat_freq_pool_bwd(const float* dm, float mul, void* dx, int dtype, int B, int F, int T, int C, cudaStream_t st) {
  if (B < 0 || F < 1 || T < 1 || C < 1) { eat_set_error("freq_pool_bwd: need B >= 0 and F, T, C >= 1"); return EAT_ERR_ARG; }
  if (dtype != EAT_F32 && dtype != EAT_BF16) { eat_set_error("freq_pool_bwd: dtype must be EAT_F32 or EAT_BF16"); return EAT_ERR_ARG; }
  const int V = dtype == EAT_BF16 ? 8 : 4;
  if (C % V != 0) { eat_set_error("freq_pool_bwd: channels must be a multiple of the vector width (4 fp32, 8 bf16)"); return EAT_ERR_ARG; }
  if (B == 0) return EAT_OK;
  if (dm == nullptr || dx == nullptr) { eat_set_error("freq_pool_bwd: dm and dx are required"); return EAT_ERR_ARG; }
  if (misaligned(dm) || misaligned(dx)) { eat_set_error("freq_pool_bwd: dm and dx must be 16-byte aligned"); return EAT_ERR_ARG; }
  const long long n_vec = (long long)B * T * (C / V);
  const unsigned grid = (unsigned)min((long long)kNumSMs * 16, ceil_div_ll(n_vec, 256));
  if (dtype == EAT_BF16)
    freq_pool_bwd_kernel<__nv_bfloat16><<<grid, 256, 0, st>>>(dm, mul, (__nv_bfloat16*)dx, F, T, C, n_vec);
  else
    freq_pool_bwd_kernel<float><<<grid, 256, 0, st>>>(dm, mul, (float*)dx, F, T, C, n_vec);
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

static int att_pool_check(const char* who, float eps, int B, int T, int H, int K) {
  static char msg[160];
  if (B < 0 || T < 1 || H < 1 || K < 1) {
    snprintf(msg, sizeof msg, "%s: need B >= 0 and T, H, K >= 1", who);
    eat_set_error(msg); return EAT_ERR_ARG;
  }
  if (!(eps > 0.f && eps < 0.5f)) { snprintf(msg, sizeof msg, "%s: eps must lie in (0, 0.5)", who); eat_set_error(msg); return EAT_ERR_ARG; }
  if ((B + kAttY - 1) / kAttY > 65535) { snprintf(msg, sizeof msg, "%s: batch too large", who); eat_set_error(msg); return EAT_ERR_ARG; }
  return EAT_OK;
}

int eat_att_pool_fwd(const float* P, const float* hw, float eps, float* out, float* sa, float* r, int B, int T, int H, int K,
                     cudaStream_t st) {
  if (int rc = att_pool_check("att_pool_fwd", eps, B, T, H, K)) return rc;
  if ((sa == nullptr) != (r == nullptr)) { eat_set_error("att_pool_fwd: sa and r go together"); return EAT_ERR_ARG; }
  if (B == 0) return EAT_OK;
  if (P == nullptr || hw == nullptr || out == nullptr) { eat_set_error("att_pool_fwd: P, hw and out are required"); return EAT_ERR_ARG; }
  const dim3 grid((unsigned)ceil_div(K, kAttX), (unsigned)ceil_div(B, kAttY));
  att_pool_fwd_kernel<<<grid, dim3(kAttX, kAttY), 0, st>>>(P, hw, eps, 1.f - eps, out, sa, r, B, T, H, K);
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

int eat_att_pool_fwd_len(const float* P, const float* hw, float eps, float* out, int B, int T, int H, int K,
                         const int* t_valid, cudaStream_t st) {
  if (int rc = att_pool_check("att_pool_fwd_len", eps, B, T, H, K)) return rc;
  if (B == 0) return EAT_OK;
  if (P == nullptr || hw == nullptr || out == nullptr || t_valid == nullptr) {
    eat_set_error("att_pool_fwd_len: P, hw, out and t_valid are required"); return EAT_ERR_ARG;
  }
  const dim3 grid((unsigned)ceil_div(K, kAttX), (unsigned)ceil_div(B, kAttY));
  att_pool_fwd_len_kernel<<<grid, dim3(kAttX, kAttY), 0, st>>>(P, hw, eps, 1.f - eps, out, B, T, H, K, t_valid);
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

int eat_att_pool_bwd(const float* dout, const float* P, float* dP, const float* hw, const float* sa, const float* r, float eps,
                     float* dhw, float* dbias, int B, int T, int H, int K, cudaStream_t st) {
  if (int rc = att_pool_check("att_pool_bwd", eps, B, T, H, K)) return rc;
  if (B == 0) return EAT_OK;
  if (dout == nullptr || P == nullptr || dP == nullptr || hw == nullptr || sa == nullptr || r == nullptr || dhw == nullptr ||
      dbias == nullptr) {
    eat_set_error("att_pool_bwd: every pointer is required"); return EAT_ERR_ARG;
  }
  const dim3 grid((unsigned)ceil_div(K, kAttX), (unsigned)ceil_div(B, kAttY));
  att_pool_bwd_kernel<<<grid, dim3(kAttX, kAttY), 0, st>>>(dout, P, dP, hw, sa, r, eps, 1.f - eps, dhw, dbias, B, T, H, K);
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

}  // extern "C"
