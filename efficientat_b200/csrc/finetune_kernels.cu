// Fine-tuning losses and augmentation (reference ex_esc50.py:96-118, ex_dcase20.py:98-123, ex_openmic.py:97-121 and
// helpers/utils.py:101-121): softmax cross-entropy with index or probability targets, the masked multi-label BCE of
// OpenMIC, and frequency-wise MixStyle.  FSD50K's loss is eat_bce_kd_loss without a teacher (train_kernels.cu).
#include <math.h>

#include "common.cuh"

namespace {

constexpr int kWarpsPerBlock = 8;

// lam[b] * t[b] + (1 - lam[b]) * t[perm[b]] for class c, with t the index or the probability target
__device__ __forceinline__ float ce_target(const int* __restrict__ yi, const float* __restrict__ yp, int b, int pb,
                                           float l, int c, int C) {
  if (yi != nullptr) return (yi[b] == c ? l : 0.f) + (yi[pb] == c ? 1.f - l : 0.f);
  return yp[(size_t)b * C + c] * l + yp[(size_t)pb * C + c] * (1.f - l);
}

// One warp per row b of z [B, C].  Pass 1: m = max_c z.  Pass 2: s = n0 + r with n0 the number of classes at the
// maximum and r = sum of exp(z - m) over the others, and S = sum_c y_mix.  Pass 3: loss_b = sum_c y_mix * (log s - (z - m)),
// dz = (S * exp(z - m) / s - y_mix) / B.  log s - (z - m) is lse - z without the cancellation of lse against z when |z|
// is large, and log s = log1p(n0 - 1 + r) keeps a small loss accurate.  At the maximum, S / s - y_mix is computed as
// (S - y_mix * n0 - y_mix * r) / s: a confident, correct row has softmax = 1 - O(r) there, and 1/s - 1 would lose r.
// loss_acc[0] += loss_b / B.  An index target outside [0, C) makes the loss NaN (torch raises there).
__global__ void ce_kernel(const float* __restrict__ z, const int* __restrict__ yi, const float* __restrict__ yp,
                          const int* __restrict__ perm, const float* __restrict__ lam, int B, int C,
                          float* __restrict__ dz, double* __restrict__ loss_acc) {
  const int lane = threadIdx.x & 31;
  const int b = blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  if (b >= B) return;
  const float* zr = z + (size_t)b * C;
  const int pb = perm != nullptr ? perm[b] : b;
  const float l = lam != nullptr ? lam[b] : 1.f;
  float m = -INFINITY;
  for (int c = lane; c < C; c += 32) m = fmaxf(m, zr[c]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  float r = 0.f, n0 = 0.f, S = 0.f;
  for (int c = lane; c < C; c += 32) {
    const float d = zr[c] - m;
    if (d == 0.f) n0 += 1.f; else r += expf(d);
    S += ce_target(yi, yp, b, pb, l, c, C);
  }
  r = warp_sum(r);
  n0 = warp_sum(n0);
  S = warp_sum(S);
  const float s = n0 + r, log_s = log1pf((n0 - 1.f) + r), inv_s = 1.f / s, invB = 1.f / (float)B;
  double loss = 0.0;
  for (int c = lane; c < C; c += 32) {
    const float d = zr[c] - m;
    const float t = ce_target(yi, yp, b, pb, l, c, C);
    loss += (double)t * (double)(log_s - d);
    if (dz != nullptr) {
      const float g = d == 0.f ? (S - t * n0 - t * r) * inv_s : S * expf(d) * inv_s - t;
      dz[(size_t)b * C + c] = g * invB;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) loss += __shfl_xor_sync(0xffffffffu, loss, o);
  if (lane == 0) {
    if (yi != nullptr && (yi[b] < 0 || yi[b] >= C || yi[pb] < 0 || yi[pb] >= C)) loss = nan("");
    atomicAdd(loss_acc, loss / (double)B);
  }
}

__device__ __forceinline__ float bce_logits_(float z, float t) {
  return fmaxf(z, 0.f) - z * t + log1pf(expf(-fabsf(z)));
}

// loss_acc[0] += mean over all B*C elements of mask[b, c] * BCE(z, y_mix), y_mix the mixup blend of the BINARISED targets
// (y > 0.5) of rows b and perm[b]; the mask is row b's own.  dz = mask * (sigmoid(z) - y_mix) / (B * C).
__global__ void bce_masked_kernel(const float* __restrict__ z, const float* __restrict__ y, int y_stride,
                                  const float* __restrict__ mask, int mask_stride, const int* __restrict__ perm,
                                  const float* __restrict__ lam, int B, int C, float* __restrict__ dz,
                                  double* __restrict__ loss_acc) {
  const long long n = (long long)B * C;
  const float inv = 1.f / (float)n;
  float acc = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int b = (int)(i / C), c = (int)(i % C);
    const float l = lam != nullptr ? lam[b] : 1.f;
    const int pb = perm != nullptr ? perm[b] : b;
    const float ya = y[(size_t)b * y_stride + c] > 0.5f ? 1.f : 0.f;
    const float yb = y[(size_t)pb * y_stride + c] > 0.5f ? 1.f : 0.f;
    const float ym = ya * l + yb * (1.f - l);
    const float mk = mask[(size_t)b * mask_stride + c];
    const float zz = z[i];
    acc += mk * bce_logits_(zz, ym);
    if (dz != nullptr) dz[i] = mk * (sigmoidf_(zz) - ym) * inv;
  }
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) atomicAdd(loss_acc, (double)(acc * inv));
}

// MixStyle statistics: one warp per (b, f) row of x [B*F, T].  Two passes over the row (the second hits L1/L2):
// mu = sum x / T, then var = sum (x - mu)^2 / (T - 1) -- no E[x^2] - E[x]^2 cancellation for rows whose mean is large
// against their spread.  stats[2 r] = mu, stats[2 r + 1] = sqrt(var + eps).
__global__ void mixstyle_stats_kernel(const float* __restrict__ x, long long rows, int T, float eps,
                                      float* __restrict__ stats) {
  const int lane = threadIdx.x & 31;
  const long long r = (long long)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  if (r >= rows) return;
  const float* xr = x + (size_t)r * T;
  float s = 0.f;
  for (int t = lane; t < T; t += 32) s += xr[t];
  const float mu = warp_sum(s) / (float)T;
  float q = 0.f;
  for (int t = lane; t < T; t += 32) {
    const float d = xr[t] - mu;
    q = fmaf(d, d, q);
  }
  const float var = warp_sum(q) / (float)(T - 1);
  if (lane == 0) {
    stats[2 * r] = mu;
    stats[2 * r + 1] = sqrtf(var + eps);
  }
}

// out[b, f, :] = (x[b, f, :] - mu_b) / sig_b * (l sig_b + (1 - l) sig_pb) + l mu_b + (1 - l) mu_pb, l = lam[b],
// pb = perm[b], statistics of row f of samples b and pb.  One warp per row.
__global__ void mixstyle_apply_kernel(const float* __restrict__ x, const float* __restrict__ stats,
                                      const int* __restrict__ perm, const float* __restrict__ lam, int F, long long rows,
                                      int T, float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const long long r = (long long)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  if (r >= rows) return;
  const int b = (int)(r / F), f = (int)(r % F);
  const long long pr = (long long)perm[b] * F + f;
  const float l = lam[b];
  const float mu = stats[2 * r], sig = stats[2 * r + 1];
  const float mu_mix = mu * l + stats[2 * pr] * (1.f - l);
  const float sig_mix = sig * l + stats[2 * pr + 1] * (1.f - l);
  const float* xr = x + (size_t)r * T;
  float* orow = out + (size_t)r * T;
  for (int t = lane; t < T; t += 32) orow[t] = (xr[t] - mu) / sig * sig_mix + mu_mix;
}

}  // namespace

extern "C" {

int eat_ce_loss(const float* logits, const int* y_index, const float* y_prob, const int* perm, const float* lam, int B,
                int C, float* dlogits, double* loss_acc, cudaStream_t st) {
  if (B < 0 || C < 1) { eat_set_error("ce_loss: need B >= 0 and C >= 1"); return EAT_ERR_ARG; }
  if ((y_index == nullptr) == (y_prob == nullptr)) {
    eat_set_error("ce_loss: exactly one of y_index (int32 [B]) and y_prob (fp32 [B, C]) must be given"); return EAT_ERR_ARG;
  }
  if ((perm == nullptr) != (lam == nullptr)) { eat_set_error("ce_loss: perm and lam go together"); return EAT_ERR_ARG; }
  if (B == 0) return EAT_OK;
  if (logits == nullptr || loss_acc == nullptr) { eat_set_error("ce_loss: logits and loss_acc are required"); return EAT_ERR_ARG; }
  ce_kernel<<<ceil_div(B, kWarpsPerBlock), 32 * kWarpsPerBlock, 0, st>>>(logits, y_index, y_prob, perm, lam, B, C, dlogits,
                                                                         loss_acc);
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

int eat_bce_masked_loss(const float* logits, const float* y, int y_stride, const float* mask, int mask_stride,
                        const int* perm, const float* lam, int B, int C, float* dlogits, double* loss_acc,
                        cudaStream_t st) {
  if (B < 0 || C < 1) { eat_set_error("bce_masked_loss: need B >= 0 and C >= 1"); return EAT_ERR_ARG; }
  if (y_stride < C || mask_stride < C) {
    eat_set_error("bce_masked_loss: the row strides of y and mask must be at least C"); return EAT_ERR_ARG;
  }
  if ((perm == nullptr) != (lam == nullptr)) { eat_set_error("bce_masked_loss: perm and lam go together"); return EAT_ERR_ARG; }
  if (B == 0) return EAT_OK;
  if (logits == nullptr || y == nullptr || mask == nullptr || loss_acc == nullptr) {
    eat_set_error("bce_masked_loss: logits, y, mask and loss_acc are required"); return EAT_ERR_ARG;
  }
  const int grid = (int)min((long long)kNumSMs * 2, ceil_div_ll((long long)B * C, 256));
  bce_masked_kernel<<<grid, 256, 0, st>>>(logits, y, y_stride, mask, mask_stride, perm, lam, B, C, dlogits, loss_acc);
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

int eat_mixstyle(const float* x, const int* perm, const float* lam, float eps, float* stats, float* out, int B, int F,
                 int T, cudaStream_t st) {
  if (B < 0 || F < 1) { eat_set_error("mixstyle: need B >= 0 and F >= 1"); return EAT_ERR_ARG; }
  if (T < 2) { eat_set_error("mixstyle: the unbiased variance over time needs T >= 2"); return EAT_ERR_ARG; }
  if (!(eps >= 0.f)) { eat_set_error("mixstyle: eps must be >= 0"); return EAT_ERR_ARG; }
  if (B == 0) return EAT_OK;
  if (x == nullptr || perm == nullptr || lam == nullptr || stats == nullptr || out == nullptr) {
    eat_set_error("mixstyle: x, perm, lam, stats and out are required"); return EAT_ERR_ARG;
  }
  if (x == out) { eat_set_error("mixstyle: out must not alias x"); return EAT_ERR_ARG; }
  const long long rows = (long long)B * F;
  const unsigned grid = (unsigned)ceil_div_ll(rows, kWarpsPerBlock);
  mixstyle_stats_kernel<<<grid, 32 * kWarpsPerBlock, 0, st>>>(x, rows, T, eps, stats);
  EAT_CHECK_LAUNCH();
  mixstyle_apply_kernel<<<grid, 32 * kWarpsPerBlock, 0, st>>>(x, stats, perm, lam, F, rows, T, out);
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

}  // extern "C"
