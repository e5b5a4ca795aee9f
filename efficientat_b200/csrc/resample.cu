// Polyphase resampling with scipy.signal.resample_poly's semantics (the librosa.core.load(path, sr=32000) step of the
// reference's inference.py:45, windowed_inference.py:89 and datasets/esc50.py:115; scripts/run_reference_script.py
// substitutes resample_poly for librosa's resampler).  With h the centred filter of 2 hl + 1 taps:
//   y[m] = sum_i x[i] h[m down - i up + hl]                                   (forward)
//   dx[i] = sum_m dy[m] h[m down - i up + hl] = sum_m dy[m] g[i up - m down + hl],  g = h reversed   (adjoint)
// so the adjoint is the forward gather with up and down exchanged over the reversed filter.  Both are one kernel:
//   out[m] = sum_{k < K} T[k][m mod U] in[i0(m) + k],  i0(m) = floor((m D + off) / U) - (K - 1)
// with T the polyphase table (efficientat_b200/resample.py), tap-major over the output residue m mod U, so that a warp
// of consecutive outputs reads consecutive table words.  Zeros stand in for the input outside [0, len).
//
// A CTA walks tiles of TM = W J consecutive outputs of one clip.  Thread w < W owns outputs m0 + w + W j, j < J: W is a
// multiple of U, so the J outputs share one residue and each table word it loads serves J multiply-adds.  The tile's
// input span goes to shared memory with coalesced 16-byte loads; the table is staged once per CTA when it fits whole
// (every rate pair of DESIGN section 4 does), else in slices of KC taps, together with the matching slice of the span.
// fp32 accumulation; no atomics, so results are bitwise repeatable.
#include <math.h>
#include <stdio.h>

#include <algorithm>

#include "common.cuh"

namespace {

constexpr int kMaxThreads = 1024;
constexpr int kMaxRounds = 2;                                   // work items per thread: W <= max(U, 512) <= 2048
constexpr int kSmemBudget = 227 * 1024;                         // H100 per-block opt-in limit
constexpr int kMaxTable = 43008;                                // floats: K U <= 2 hl + U <= 20 * 2048 + 2048

struct Plan {
  int W, threads, J, KC, span, smem_floats, tiles;
};

// span of input samples a tile of TM outputs reads for KC taps (+ 3 for the 16-byte alignment of its start), in
// whole float4s
long long span_floats(long long TM, int U, int D, int KC) {
  return (((TM - 1) * D + U - 1) / U + 1 + KC + 3 + 3) & ~3LL;
}

// W = U GB work items per tile (GB groups of U consecutive outputs), J outputs per work item; the largest tile whose
// span and table slice of at least min(K, 16) taps fit in shared memory
bool make_plan(int U, int D, int K, long long n_out, Plan& p) {
  for (int GB = std::max(1, 512 / U); GB >= 1; GB /= 2) {
    const int W = U * GB;
    for (int J = 8; J >= 1; J >>= 1) {
      const long long TM = (long long)W * J;
      if (J > 1 && TM > 2 * n_out + 2LL * W) continue;         // a tile far longer than the clip wastes threads
      const long long base = span_floats(TM, U, D, 0);
      const long long room = kSmemBudget / 4 - 4 - base;
      if (room < (long long)(U + 1)) continue;
      const int KC = (int)std::min<long long>(K, room / (U + 1));
      if (KC < std::min(K, 16)) continue;
      p.W = W;
      p.J = J;
      p.KC = KC;
      const int rounds = ceil_div(W, kMaxThreads);
      p.threads = ceil_div(ceil_div(W, rounds), 32) * 32;
      p.span = (int)span_floats(TM, U, D, KC);
      p.smem_floats = ((KC * U + 3) & ~3) + p.span;
      p.tiles = (int)ceil_div_ll(n_out, TM);
      return true;
    }
  }
  return false;
}

// dst[j] = row[s0a + j] for 0 <= s0a + j < len, else 0, j < n; s0a a multiple of 4, dst 16-byte aligned
__device__ __forceinline__ void stage_span(float* __restrict__ dst, const float* __restrict__ row, long long s0a, int n,
                                           int len, bool vec) {
  const int nq = n >> 2;
  for (int q = threadIdx.x; q < nq; q += blockDim.x) {
    const long long s = s0a + 4 * q;
    float4 v;
    if (vec && s >= 0 && s + 4 <= len) {
      v = __ldg(reinterpret_cast<const float4*>(row + s));
    } else {
      v.x = (s >= 0 && s < len) ? row[s] : 0.f;
      v.y = (s + 1 >= 0 && s + 1 < len) ? row[s + 1] : 0.f;
      v.z = (s + 2 >= 0 && s + 2 < len) ? row[s + 2] : 0.f;
      v.w = (s + 3 >= 0 && s + 3 < len) ? row[s + 3] : 0.f;
    }
    reinterpret_cast<float4*>(dst)[q] = v;
  }
}

// in [B, n_in], out [B, n_out]; lens: per-row input length (nullptr: n_in).  Output m of row b is written for every
// m < n_out: the gather for m < ceil(len U / D), 0 past it.  Persistent: CTAs stride over the (tile, row) items.
template <int J>
__global__ void __launch_bounds__(kMaxThreads) resample_gather_kernel(
    const float* __restrict__ in, int n_in, const int* __restrict__ lens, const float* __restrict__ table, int K, int KC,
    int U, int D, long long off, int W, int span, float* __restrict__ out, int n_out, int tiles, int B) {
  extern __shared__ __align__(16) float smem[];
  float* s_tab = smem;                                           // [KC][U]
  float* s_x = smem + ((KC * U + 3) & ~3);                       // [span]
  const bool whole = KC == K;
  if (whole) {
    for (int i = threadIdx.x; i < K * U; i += blockDim.x) s_tab[i] = __ldg(table + i);
  }
  const long long TM = (long long)W * J;
  for (long long item = blockIdx.x; item < (long long)tiles * B; item += gridDim.x) {
    const int b = (int)(item / tiles);
    const long long m0 = (item % tiles) * TM;
    int len = lens != nullptr ? lens[b] : n_in;
    len = min(max(len, 0), n_in);
    const long long n_valid = min((long long)n_out, ceil_div_ll((long long)len * U, D));
    const float* row = in + (long long)b * n_in;
    float* orow = out + (long long)b * n_out;
    if (m0 >= n_valid) {                                         // tile wholly past the clip: zeros, CTA-uniform
      for (long long m = m0 + threadIdx.x; m < min(m0 + TM, (long long)n_out); m += blockDim.x) orow[m] = 0.f;
      continue;
    }
    const bool vec = (reinterpret_cast<uintptr_t>(row) & 15) == 0;
    const long long i0_tile = (m0 * D + off) / U - (K - 1);
    float acc[kMaxRounds][J];
#pragma unroll
    for (int r = 0; r < kMaxRounds; ++r)
#pragma unroll
      for (int j = 0; j < J; ++j) acc[r][j] = 0.f;
    for (int kc = 0; kc < K; kc += KC) {
      const int kn = min(KC, K - kc);
      const long long s0a = (i0_tile + kc) & ~3LL;
      __syncthreads();                                           // the previous tile / slice is consumed
      if (!whole) {
        for (int i = threadIdx.x; i < kn * U; i += blockDim.x) s_tab[i] = __ldg(table + (long long)kc * U + i);
      }
      stage_span(s_x, row, s0a, span, len, vec);
      __syncthreads();
#pragma unroll
      for (int r = 0; r < kMaxRounds; ++r) {
        const int w = threadIdx.x + r * blockDim.x;
        if (w >= W) break;
        const int res = (int)((m0 + w) % U);
        const float* xb = s_x + (int)(((m0 + w) * D + off) / U - (K - 1) + kc - s0a);
        const int jstep = (int)((long long)W / U * D);            // input advance between the thread's outputs
        for (int k = 0; k < kn; ++k) {
          const float t = s_tab[k * U + res];
#pragma unroll
          for (int j = 0; j < J; ++j) acc[r][j] = fmaf(t, xb[j * jstep + k], acc[r][j]);
        }
      }
    }
#pragma unroll
    for (int r = 0; r < kMaxRounds; ++r) {
      const int w = threadIdx.x + r * blockDim.x;
      if (w >= W) break;
#pragma unroll
      for (int j = 0; j < J; ++j) {
        const long long m = m0 + w + (long long)W * j;
        if (m < n_out) orow[m] = m < n_valid ? acc[r][j] : 0.f;
      }
    }
  }
}

template <int J>
int launch_gather(const float* in, int n_in, const int* lens, const float* table, int K, int U, int D, long long off,
                  const Plan& p, float* out, int n_out, int B, cudaStream_t st) {
  static unsigned long long opted = 0;
  const size_t bytes = (size_t)p.smem_floats * 4;
  if (bytes > 48 * 1024) {
    const int rc = eat_opt_in_smem(resample_gather_kernel<J>, (size_t)kSmemBudget, opted);
    if (rc != EAT_OK) return rc;
  }
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, resample_gather_kernel<J>, p.threads, bytes) != cudaSuccess ||
      per_sm < 1) {
    eat_set_error("resample: kernel does not fit on the device"); return EAT_ERR_CUDA;
  }
  const long long items = (long long)p.tiles * B;
  const int grid = (int)std::min<long long>(items, (long long)kNumSMs * per_sm);
  resample_gather_kernel<J><<<grid, p.threads, bytes, st>>>(in, n_in, lens, table, K, p.KC, U, D, off, p.W, p.span, out,
                                                            n_out, p.tiles, B);
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

int gather(const char* who, const float* in, int n_in, const int* lens, const float* table, int K, int U, int D,
           int off, float* out, int n_out, int B, cudaStream_t st) {
  Plan p;
  if (!make_plan(U, D, K, n_out, p) || p.W > kMaxRounds * kMaxThreads) {
    eat_set_error(who); return EAT_ERR_UNSUPPORTED;
  }
  switch (p.J) {
    case 8: return launch_gather<8>(in, n_in, lens, table, K, U, D, off, p, out, n_out, B, st);
    case 4: return launch_gather<4>(in, n_in, lens, table, K, U, D, off, p, out, n_out, B, st);
    case 2: return launch_gather<2>(in, n_in, lens, table, K, U, D, off, p, out, n_out, B, st);
    default: return launch_gather<1>(in, n_in, lens, table, K, U, D, off, p, out, n_out, B, st);
  }
}

// the argument checks both entry points share; the message names the entry point
int check_args(const char* who, int B, int N, int n_out, int up, int down, int taps, int table_rows, int offset) {
  static thread_local char msg[256];
  if (B < 0 || N < 1 || up < 1 || down < 1 || taps < 1 || offset < 0) {
    snprintf(msg, sizeof msg, "%s: need B >= 0, N >= 1, up >= 1, down >= 1, taps >= 1 and offset >= 0", who);
    eat_set_error(msg); return EAT_ERR_ARG;
  }
  if (up > EAT_RESAMPLE_MAX_RATE || down > EAT_RESAMPLE_MAX_RATE || (long long)taps * table_rows > kMaxTable) {
    snprintf(msg, sizeof msg, "%s: up and down must be at most %d and the table at most %d floats (taps x %s)", who,
             EAT_RESAMPLE_MAX_RATE, kMaxTable, table_rows == up ? "up" : "down");
    eat_set_error(msg); return EAT_ERR_UNSUPPORTED;
  }
  if ((long long)N * up > (long long)INT32_MAX * down || (long long)n_out != ceil_div_ll((long long)N * up, down)) {
    snprintf(msg, sizeof msg, "%s: n_out must be ceil(N * up / down) = %lld and fit in int32", who,
             ceil_div_ll((long long)N * up, down));
    eat_set_error(msg); return EAT_ERR_ARG;
  }
  return EAT_OK;
}

}  // namespace

extern "C" {

int eat_resample_poly_fwd(const float* x, int B, int N, const int* lengths, int up, int down, const float* table, int taps,
                          int offset, float* y, int n_out, cudaStream_t st) {
  int rc = check_args("resample_poly_fwd", B, N, n_out, up, down, taps, up, offset);
  if (rc != EAT_OK) return rc;
  if (B == 0) return EAT_OK;
  if (x == nullptr || table == nullptr || y == nullptr) {
    eat_set_error("resample_poly_fwd: x, table and y are required"); return EAT_ERR_ARG;
  }
  return gather("resample_poly_fwd: no launch plan fits in shared memory", x, N, lengths, table, taps, up, down, offset,
                y, n_out, B, st);
}

int eat_resample_poly_bwd(const float* dy, int B, int N, int up, int down, const float* table_adj, int taps_adj,
                          int offset, float* dx, int n_out, cudaStream_t st) {
  int rc = check_args("resample_poly_bwd", B, N, n_out, up, down, taps_adj, down, offset);
  if (rc != EAT_OK) return rc;
  if (B == 0) return EAT_OK;
  if (dy == nullptr || table_adj == nullptr || dx == nullptr) {
    eat_set_error("resample_poly_bwd: dy, table_adj and dx are required"); return EAT_ERR_ARG;
  }
  // dx [B, N] from dy [B, n_out]: the forward gather with up and down exchanged
  return gather("resample_poly_bwd: no launch plan fits in shared memory", dy, n_out, nullptr, table_adj, taps_adj, down,
                up, offset, dx, N, B, st);
}

}  // extern "C"
