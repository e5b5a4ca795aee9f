// Weight gradient of a pointwise (1x1) convolution for fp32 activations as a TMA-fed wgmma GEMM whose reduction runs
// over pixels:     dW[N, K] += G[M, N]^T . xf(X)[M, K]        G: gradient rows (NHWC), X: saved layer input, dW fp32
// (autograd of the 1x1 ConvNormActivation layers, reference models/mn/block_types.py:140-147,167-171, reached from
// ex_audioset.py:197 loss.backward()).  Built like pw_tma.cu:
//
//   warp 12  TMA producer : one thread; per MB-row block of the reduction, cp.async.bulk.tensor lands [MB rows x 32
//                           channels] fp32 boxes of G (2 boxes = 64 output channels) and of X (up to 2 boxes = 64
//                           input channels) in a ring of stages; rows past M are zero-filled by the TMA unit.
//   warps 0-3 fix-up      : the in-place pass of tma_common.cuh: (BatchNorm affine + activation + SE gate on X), then a
//                           row's 32 fp32 values become 32 bf16 hi + 32 bf16 lo values in the same 128 bytes.
//                           Both operands are "MN-major" for the tensor core (the reduction index m is the row index),
//                           and a landed box IS a canonical MN-major SWIZZLE_128B atom column: 8-row groups 1024 B
//                           apart (SBO) -- no transposition, no second buffer.
//   warps 4-11 consumers  : two warpgroups, one per G box: wgmma m64n64k16 (one per X box), K = 16 reduction rows per
//                           instruction, register accumulators.  Because hi and lo sit side by side along the
//                           NON-reduced dimension, the accumulator holds the four products separately: rows
//                           n' = [hi(n) | lo(n)], columns k' = [hi(k) | lo(k)].  Once per CTA: dW[n,k] += hi.hi + hi.lo
//                           (threads on hi(n) rows) and += lo.hi (threads on lo(n) rows) with vector atomics
//                           (lo.lo ~ 2^-32 is dropped).
// Each CTA owns a (64 x 64) tile of dW and one slice of the M range (dW is zeroed by the caller once per step).
// HBM-bound: algorithmic bytes per launch = 4 * (M*N + M*K + N*K).
#include <cstdlib>

#include "tma_common.cuh"

namespace {
using namespace tc;
using namespace tma;

// MB = reduction rows per pipeline stage (template parameter): 64, or 128 for launches with few boxes per stage, where the
// per-block costs (barrier round trips, TMA issue, fix-up prologue) rather than bytes set the pace.
// BOX = MB * 128 bytes: one landed [MB x 32 fp32] box.
constexpr int GB = 2;                   // G boxes per stage: 64 output channels -> 128 accumulator rows
constexpr int XB = 2;                   // X boxes per stage at most: 64 input channels -> 128 accumulator columns
constexpr int kThreads = 416;
constexpr int kFirstCons = 4, kTmaWarp = 12;
// The register accumulators are flushed to dW (and restarted) every kFlushRows reduction rows: the tensor core's fp32
// accumulation rounds toward zero, so a long split with same-signed terms drifts by ~1.5 x 2^-24 of the sum per 16-row
// step; over 31k rows (mn10 block 2 at B = 256) that was 1.5e-4 of sum |terms|, within 30x of a dropped 128-row block.
constexpr int kFlushRows = 4096;

struct WgParams {
  float* dW;
  int M, N, K;
  int n_tiles, k_tiles, xb;             // xb: X boxes reserved per stage (<= XB); a CTA loads only those inside K
  int gbs;                              // G boxes reserved per stage (1 when N <= 32, else 2); a CTA loads only those inside N
  int rows_per_split, sample_rows, splits_per_sample;
  int stages;
  uint32_t stage_bytes, off_f, off_bar;
  const float* in_scale; const float* in_shift; const float* gate; int in_act; int rps;
};

template <int XACT, int MB>
__global__ void __launch_bounds__(kThreads, 1)
wgrad_tma_kernel(const __grid_constant__ CUtensorMap mapG, const __grid_constant__ CUtensorMap mapX, const WgParams p) {
  constexpr int BOX = MB * 128;
  extern __shared__ __align__(1024) unsigned char smem[];
  float* s_isc = reinterpret_cast<float*>(smem + p.off_f);          // [64] in-transform scale of this CTA's channels
  float* s_ish = s_isc + 64;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + p.off_bar);
  const int S = p.stages;
  const uint32_t bar_full = smem_u32(bars), bar_ready = bar_full + 8 * S, bar_empty = bar_ready + 8 * S;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles = p.n_tiles * p.k_tiles;
  const int ot = blockIdx.x % tiles, split = blockIdx.x / tiles;
  const int nt = ot / p.k_tiles, kt = ot - nt * p.k_tiles;
  const int n0 = nt * 64, k0 = kt * (XB * KB);
  long long m_begin, m_end;
  float* __restrict__ dWout = p.dW;
  if (p.sample_rows > 0) {
    const int b = split / p.splits_per_sample, j = split - b * p.splits_per_sample;
    m_begin = (long long)b * p.sample_rows + (long long)j * p.rows_per_split;
    m_end = m_begin + p.rows_per_split;
    if (m_end > (long long)(b + 1) * p.sample_rows) m_end = (long long)(b + 1) * p.sample_rows;
    dWout += (size_t)b * p.N * p.K;
  } else {
    m_begin = (long long)split * p.rows_per_split;
    m_end = m_begin + p.rows_per_split;
    if (m_end > p.M) m_end = p.M;
  }
  const int n_blocks = m_end > m_begin ? (int)((m_end - m_begin + MB - 1) / MB) : 0;
  // boxes of this CTA's tile that hold real channels; MMAs on boxes that are not loaded are skipped
  const int gb = min(p.gbs, (p.N - n0 + KB - 1) / KB);
  const int xb = min(p.xb, (p.K - k0 + KB - 1) / KB);
  const uint32_t x_off = (uint32_t)p.gbs * BOX;
  const uint32_t stage_base = smem_u32(smem);

  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) { mbar_init(bar_full + 8 * s, 1); mbar_init(bar_ready + 8 * s, 4); mbar_init(bar_empty + 8 * s, 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&mapG)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&mapX)) : "memory");
  }
  if (XACT >= 0) {
    for (int i = threadIdx.x; i < 64; i += kThreads) {
      s_isc[i] = k0 + i < p.K ? p.in_scale[k0 + i] : 0.f;          // zero beyond K: act(0) = 0
      s_ish[i] = k0 + i < p.K ? p.in_shift[k0 + i] : 0.f;
    }
  }
  __syncthreads();

  if (warp == kTmaWarp) {
    // ================================================================= TMA producer (one thread)
    if (lane == 0) {
      int s = 0;
      uint32_t ph = 0;
      for (int blk = 0; blk < n_blocks; ++blk) {
        const int m = (int)(m_begin + (long long)blk * MB);
        mbar_wait(bar_empty + 8 * s, ph ^ 1u);
        const uint32_t dst = stage_base + (uint32_t)s * p.stage_bytes;
        mbar_expect_tx(bar_full + 8 * s, (uint32_t)(gb + xb) * BOX);
        for (int b = 0; b < gb; ++b) tma_load_2d(&mapG, bar_full + 8 * s, dst + b * BOX, n0 + b * KB, m);
        for (int b = 0; b < xb; ++b) tma_load_2d(&mapX, bar_full + 8 * s, dst + x_off + b * BOX, k0 + b * KB, m);
        if (++s == S) { s = 0; ph ^= 1u; }
      }
    }
    __syncwarp();
  } else if (warp < kFirstCons) {
    // ================================================================= fix-up warps (128 threads)
    const int ft = threadIdx.x;
    int s = 0;
    uint32_t ph = 0;
    for (int blk = 0; blk < n_blocks; ++blk) {
      const long long mb = m_begin + (long long)blk * MB;
      const int rows_valid = (int)min((long long)MB, m_end - mb);
      int b0 = 0, off0 = 0;
      if (p.gate != nullptr) { b0 = (int)(mb / p.rps); off0 = (int)(mb - (long long)b0 * p.rps); }
      mbar_wait(bar_full + 8 * s, ph);
      unsigned char* st = smem + (size_t)s * p.stage_bytes;
      for (int b = 0; b < gb; ++b)                               // gradient boxes: plain split (rows past the split zeroed)
        fix_a<2, -1, MB>(st + b * BOX, ft, rows_valid, nullptr, nullptr, 0, nullptr, 0, 0, 1, 0);
      for (int b = 0; b < xb; ++b) {
        const int kl = b * KB + (ft & 3) * 8;                      // channel of this thread's chunk pair, local to the CTA
        fix_a<2, XACT, MB>(st + x_off + b * BOX, ft, rows_valid, s_isc - k0, s_ish - k0, k0 + kl, p.gate, off0, b0, p.rps, p.K);
      }
      fence_proxy_async();
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_ready + 8 * s);
      if (++s == S) { s = 0; ph ^= 1u; }
    }
  } else {
    // ================================================================= consumers: MMA, the atomics every kFlushRows rows
    const int cw = warp - kFirstCons;
    const int g = cw >> 2, wq = cw & 3;                        // G box of this warpgroup, warp inside it
    const int ctid = threadIdx.x - kFirstCons * 32;
    float acc[XB][32];
#pragma unroll
    for (int b = 0; b < XB; ++b)
#pragma unroll
      for (int i = 0; i < 32; ++i) acc[b][i] = 0.f;
    // accumulator rows of this thread: r = 16 wq + lane / 4 (+ 8) inside the group's 64 rows [hi(n) 0..31 | lo(n) 0..31]
    auto flush = [&]() {
      if (g < gb) {
        const bool hi_row = wq < 2;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int r = (wq & 1) * 16 + (lane >> 2) + 8 * h;          // channel inside the 32-channel box
          const int n = n0 + g * 32 + r;
          if (n >= p.N) continue;
#pragma unroll
          for (int b = 0; b < XB; ++b) {
            if (b >= xb) continue;
#pragma unroll
            for (int j = 0; j < 4; ++j) {                             // hi(k) columns 8 j + 2 (lane % 4) of box b
              const int k = k0 + b * KB + 8 * j + 2 * (lane & 3);
              float2 v = make_float2(acc[b][4 * j + 2 * h], acc[b][4 * j + 2 * h + 1]);
              if (hi_row) { v.x += acc[b][4 * (j + 4) + 2 * h]; v.y += acc[b][4 * (j + 4) + 2 * h + 1]; }   // + hi.lo
              if (k < p.K) atomicAdd(reinterpret_cast<float2*>(dWout + (size_t)n * p.K + k), v);
            }
          }
        }
      }
#pragma unroll
      for (int b = 0; b < XB; ++b)
#pragma unroll
        for (int i = 0; i < 32; ++i) acc[b][i] = 0.f;
    };
    int s = 0;
    uint32_t ph = 0;
    for (int blk = 0; blk < n_blocks; ++blk) {
      mbar_wait(bar_ready + 8 * s, ph);
      const uint32_t sg = stage_base + (uint32_t)s * p.stage_bytes + (uint32_t)g * BOX, sx = stage_base + (uint32_t)s * p.stage_bytes + x_off;
      const long long mb = m_begin + (long long)blk * MB;
      const int rows = (int)min((long long)MB, m_end - mb);
      const int steps = (rows + 15) >> 4;
      if (g < gb) {
        wgmma_fence();
#pragma unroll
        for (int st = 0; st < MB / 16; ++st) {
          if (st < steps) {                                         // 16 reduction rows = two 8-row groups = 2048 bytes
            const uint64_t da = gmma_desc(sg + st * 2048, BOX, 1024);
#pragma unroll
            for (int b = 0; b < XB; ++b)
              if (b < xb) wgmma_n64<1, 1>(acc[b], da, gmma_desc(sx + b * BOX + st * 2048, BOX, 1024));
          }
        }
        wgmma_commit();
        wgmma_wait<0>();
#pragma unroll
        for (int b = 0; b < XB; ++b) wgmma_fence_regs(acc[b]);
      }
      asm volatile("bar.sync %0, 128;" ::"r"(1 + g) : "memory");   // every warp of the group is past its wait
      if (ctid == g * 128) mbar_arrive(bar_empty + 8 * s);
      if (++s == S) { s = 0; ph ^= 1u; }
      if ((blk + 1) % (kFlushRows / MB) == 0 && blk + 1 < n_blocks) flush();
    }
    if (n_blocks > 0) flush();
  }
  __syncthreads();
}

// The launch plan (fills the tiling / split / stage fields of p) -> MB and the number of reduction splits.  sms: the
// GPU's SM count.  128-row blocks when a stage holds at most three boxes (N <= 64 and K <= 32, or N <= 32 and K <= 64)
// and the reduction is long: the first layers of the network, M in the millions.
int plan_wg(WgParams& p, int sms, int& mb, int& splits) {
  p.n_tiles = ceil_div(p.N, 64);
  p.k_tiles = ceil_div(p.K, XB * KB);
  const int kt = p.K < XB * KB ? p.K : XB * KB;
  p.xb = ceil_div(kt, KB);
  p.gbs = p.N <= KB ? 1 : GB;
  const int boxes = p.gbs + p.xb;
  mb = (boxes <= 3 && p.sample_rows == 0 && p.M >= (1 << 20)) ? 128 : 64;
  if (const char* e = getenv("EAT_WG_MB")) { const int v = atoi(e); if (v == 64 || (v == 128 && boxes <= 3)) mb = v; }
  const int tiles = p.n_tiles * p.k_tiles;
  const int slots = sms;
  if (p.sample_rows > 0) {
    const int B = p.M / p.sample_rows;
    int sps = max(1, (2 * slots) / max(1, tiles * B));
    long long rows = ceil_div_ll(p.sample_rows, sps);
    rows = ceil_div_ll(rows, mb) * mb;
    sps = (int)ceil_div_ll(p.sample_rows, rows);
    p.rows_per_split = (int)rows;
    p.splits_per_sample = sps;
    splits = sps * B;
  } else {
    splits = max(1, (2 * slots) / tiles);
    long long rows = ceil_div_ll(p.M, splits);
    rows = ceil_div_ll(rows, mb) * mb;
    if (rows < 4 * mb) rows = 4 * mb;
    splits = (int)ceil_div_ll(p.M, rows);
    p.rows_per_split = (int)rows;
    p.splits_per_sample = 0;
  }
  p.stage_bytes = (uint32_t)(boxes * mb * 128);
  const size_t budget = 227 * 1024;
  const size_t misc = 2 * 64 * 4 + 3 * 8 * 8 + 16 + 1024;
  p.stages = (int)((budget - misc) / p.stage_bytes);
  if (p.stages > 8) p.stages = 8;
  if (p.stages < 2) { eat_set_error("wgrad_tma: shared-memory budget exceeded"); return EAT_ERR_UNSUPPORTED; }
  return EAT_OK;
}

template <int XACT, int MB>
int launch_wg_mb(const float* G, const float* X, const WgParams& p, int splits, cudaStream_t st) {
  const size_t budget = 227 * 1024;
  size_t off = (size_t)p.stages * p.stage_bytes;
  const uint32_t off_f = (uint32_t)off; off += 2 * 64 * 4;
  const uint32_t off_bar = (uint32_t)off; off += 3 * (size_t)p.stages * 8 + 16;
  const size_t smem = off;
  WgParams q = p;
  q.off_f = off_f; q.off_bar = off_bar;
  CUtensorMap mG, mX;
  if (int rc = make_map(&mG, G, p.M, p.N, MB)) return rc;
  if (int rc = make_map(&mX, X, p.M, p.K, MB)) return rc;
  static unsigned long long attr_mask = 0;
  if (int rc = eat_opt_in_smem(wgrad_tma_kernel<XACT, MB>, budget, attr_mask)) return rc;
  wgrad_tma_kernel<XACT, MB><<<p.n_tiles * p.k_tiles * splits, kThreads, smem, st>>>(mG, mX, q);
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

template <int XACT>
int launch_wg(const float* G, const float* X, WgParams p, cudaStream_t st) {
  int dev = 0, sms = kNumSMs;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  int mb = 64, splits = 1;
  if (int rc = plan_wg(p, sms, mb, splits)) return rc;
  return mb == 128 ? launch_wg_mb<XACT, 128>(G, X, p, splits, st) : launch_wg_mb<XACT, 64>(G, X, p, splits, st);
}

int launch_wg_x(const float* G, const float* X, const WgParams& p, cudaStream_t st) {
  if (p.in_scale == nullptr) return launch_wg<-1>(G, X, p, st);
  if (p.in_act == EAT_ACT_RELU) return launch_wg<1>(G, X, p, st);
  if (p.in_act == EAT_ACT_HSWISH) return launch_wg<2>(G, X, p, st);
  return launch_wg<0>(G, X, p, st);
}

}  // namespace

extern "C" int eat_pw_tma_wgrad(const float* G, const float* X, float* dW, long long M, int N, int K, const float* in_scale,
                                const float* in_shift, int in_act, const float* gate, int rows_per_sample,
                                int per_sample, cudaStream_t st) {
  if (M == 0) return EAT_OK;
  if (K % 4 != 0 || N % 4 != 0) { eat_set_error("pw_tma_wgrad: K and N must be multiples of 4"); return EAT_ERR_ARG; }
  if (M >= (1ll << 31) - 128) { eat_set_error("pw_tma_wgrad: M too large"); return EAT_ERR_ARG; }
  if ((in_scale == nullptr) != (in_shift == nullptr)) { eat_set_error("pw_tma_wgrad: in_scale and in_shift come together"); return EAT_ERR_ARG; }
  if (in_act == EAT_ACT_SIGMOID) { eat_set_error("pw_tma_wgrad: sigmoid input activation is not offered"); return EAT_ERR_UNSUPPORTED; }
  if ((((uintptr_t)G) | ((uintptr_t)X) | ((uintptr_t)dW) | ((uintptr_t)gate)) & 15) { eat_set_error("pw_tma_wgrad: operands must be 16-byte aligned"); return EAT_ERR_ARG; }
  WgParams p{};
  p.dW = dW; p.M = (int)M; p.N = N; p.K = K;
  p.in_scale = in_scale; p.in_shift = in_shift; p.gate = gate; p.in_act = in_act;
  p.rps = rows_per_sample > 0 ? rows_per_sample : 1;
  p.sample_rows = 0;
  if (per_sample) {
    if (rows_per_sample < 1 || M % rows_per_sample != 0) { eat_set_error("pw_tma_wgrad: per-sample mode needs M = B * rows_per_sample"); return EAT_ERR_ARG; }
    p.sample_rows = rows_per_sample;
  }
  return launch_wg_x(G, X, p, st);
}

extern "C" int eat_pw_wgrad_plan(long long M, int N, int K, int rows_per_sample, int per_sample, int sms, int* plan) {
  if (plan == nullptr) { eat_set_error("pw_wgrad_plan: plan is NULL"); return EAT_ERR_ARG; }
  if (M < 1 || N < 1 || K < 1 || sms < 1) { eat_set_error("pw_wgrad_plan: M, N, K and sms must be positive"); return EAT_ERR_ARG; }
  if (M >= (1ll << 31) - 128) { eat_set_error("pw_wgrad_plan: M too large"); return EAT_ERR_ARG; }
  WgParams p{};
  p.M = (int)M; p.N = N; p.K = K;
  if (per_sample) {
    if (rows_per_sample < 1 || M % rows_per_sample != 0) { eat_set_error("pw_wgrad_plan: per-sample mode needs M = B * rows_per_sample"); return EAT_ERR_ARG; }
    p.sample_rows = rows_per_sample;
  }
  int mb = 64, splits = 1;
  if (int rc = plan_wg(p, sms, mb, splits)) return rc;
  plan[0] = mb; plan[1] = p.n_tiles * p.k_tiles; plan[2] = splits; plan[3] = p.rows_per_split;
  plan[4] = p.splits_per_sample; plan[5] = p.stages;
  return EAT_OK;
}
