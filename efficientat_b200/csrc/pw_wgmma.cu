// Pointwise (1x1) convolution / Linear as a wgmma GEMM for sm_90a:
//     C[M,N] = epi( xf(A)[M,K] . W[N,K]^T )        A, C: NHWC activation rows (fp32 or bf16), W: fp32
// Replaces the 1x1 ConvNormActivation layers of the reference (models/mn/block_types.py:140-147,
// 167-171; models/mn/model.py:160-166) -- 90 % of mn10's MACs.
//
// Design (one persistent CTA per SM, 16 warps, warp-specialised, mbarrier pipelines):
//   warps 0-7  producers : two groups of 4 warps that fill alternate pipeline stages, so the global-load
//                          latency of stage s+1 overlaps the conversion of stage s.  global -> registers ->
//                          (BatchNorm affine + activation + SE gate of the producing layer, fused on load)
//                          -> bf16 -> 128B-swizzled K-major smem tiles.  fp32 activations/weights are split
//                          x = hi + lo (two bf16) so that three MMAs (hi*hi + lo*hi + hi*lo) reproduce fp32
//                          products to ~2^-16.  Only the 16-byte chunks the MMAs will read are produced.
//   warps 8-15 consumers : two warpgroups, one per 64-row half of the 128-row tile.  Each issues wgmma.m64nNk16
//                          (bf16, N = 32-column pieces of the tile, K = 16) on shared-memory descriptors into
//                          register accumulators, then runs the epilogue of its rows: fragment -> per-warp smem
//                          transpose -> 16-byte vector path: BN affine / activation / residual (loads issued up
//                          front) -> coalesced stores; per-channel batch statistics (sum, sum of squares) reduced
//                          with two shuffles per chunk and kept in shared memory across tiles.
// The kernel is HBM-bound for mn10 widths (arithmetic intensity below the ridge); algorithmic bytes per
// launch = M*K*sizeof(A) + M*N*sizeof(C) (+ residual) + N*K*4.
#include <cstdlib>
#include <cstring>

#include "tc_common.cuh"


namespace {

constexpr int BM = 128;
constexpr int BK = 64;                 // bf16 elements per k-block (= one 128-byte swizzle row)
constexpr int kGroupThreads = 128;     // one producer group (4 warps) fills one pipeline stage
constexpr int kThreads = 512;          // 8 producer warps + 2 consumer warpgroups
constexpr int kFirstCons = 8;
constexpr int kEpiThreads = 256;
constexpr int STG_LD = 36;             // floats per staged row: 16-byte aligned rows, conflict-free both ways
constexpr int A_TILE_BYTES = BM * 128; // 16 KB

struct TcParams {
  const void* A;
  const float* W;
  void* C;
  const void* residual;
  int M, N, K;
  InXform xf;
  const float* scale;
  const float* shift;
  int act;
  double* stat_sum;
  double* stat_sq;
  int BN;        // columns per N tile (multiple of 16, <= 128)
  int n_tiles, m_tiles, k_blocks;
  // DynamicConv (reference models/dymn/dy_block.py:103-131): per-sample weights W_b = sum_k att[b,k] * W[k],
  // mixed while the weight tile is staged.  Tiles then never straddle samples.
  const float* dyn_att;   // [B, dyn_k] or nullptr
  int dyn_k;              // number of kernels (4)
  int tps;                // M tiles per sample (0: flat tiling over all rows)
  int tile_rps;           // rows per sample used for tiling
};

// first row / row limit / sample of M tile `mt`
template <bool DYN>
__device__ __forceinline__ void tile_rows(const TcParams& p, int mt, long long& m0, long long& m_lim, int& b) {
  if (!DYN) { m0 = (long long)mt * BM; m_lim = p.M; b = 0; return; }
  b = mt / p.tps;
  const int j = mt - b * p.tps;
  m0 = (long long)b * p.tile_rps + (long long)j * BM;
  m_lim = (long long)(b + 1) * p.tile_rps;
}

using namespace tc;

// d[piece] += A(64 x 16) . B(32 or 16 rows x 16)^T for every 32-column piece of a BN-column tile (K-major operands)
template <int NPC>
__device__ __forceinline__ void mma_pieces(float (&d)[NPC][16], uint64_t da, uint64_t db, int BN) {
#pragma unroll
  for (int pc = 0; pc < NPC; ++pc) {
    if (pc * 32 + 32 <= BN) wgmma_n32<0, 0>(d[pc], da, db + (uint64_t)(pc * 256));   // 32 rows x 128 B = 4 KB apart
    else if (pc * 32 < BN) wgmma_n16<0, 0>(reinterpret_cast<float(&)[8]>(d[pc]), da, db + (uint64_t)(pc * 256));
  }
}

// ------------------------------------------------------------------------------------------ kernel
template <typename T> struct OutVec;
template <> struct OutVec<float> {
  __device__ __forceinline__ static void load(const float* p, float (&v)[4]) {
    float4 t = __ldg(reinterpret_cast<const float4*>(p)); v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
  }
  __device__ __forceinline__ static void store(float* p, const float (&v)[4]) {
    *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
  }
};
template <> struct OutVec<__nv_bfloat16> {
  __device__ __forceinline__ static void load(const __nv_bfloat16* p, float (&v)[4]) {
    uint2 t = __ldg(reinterpret_cast<const uint2*>(p));
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&t);
    float2 a = __bfloat1622float2(h[0]), b = __bfloat1622float2(h[1]);
    v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y;
  }
  __device__ __forceinline__ static void store(__nv_bfloat16* p, const float (&v)[4]) {
    uint2 t;
    t.x = pack_bf16(v[0], v[1]); t.y = pack_bf16(v[2], v[3]);
    *reinterpret_cast<uint2*>(p) = t;
  }
};

template <int EPI>
__device__ __forceinline__ float act_epi(float v) {                // compile-time activation of the epilogue
  if (EPI == 2) return fmaxf(v, 0.f);
  if (EPI == 3) return v * fminf(fmaxf(v + 3.f, 0.f), 6.f) * (1.f / 6.f);
  return v;
}

__device__ __forceinline__ float act_sel(float v, int act) {     // branch-free activation
  const float r = fmaxf(v, 0.f);
  const float h = v * fminf(fmaxf(v + 3.f, 0.f), 6.f) * (1.f / 6.f);
  return act == EAT_ACT_HSWISH ? h : (act == EAT_ACT_RELU ? r : v);
}

// input transform applied while the A operand is staged: XACT -1 none, 0 affine, 1 affine + ReLU, 2 affine + Hardswish,
// 3 affine + run-time activation code (only instantiated for the fused-epilogue variants, where it is rare)
template <int XACT>
__device__ __forceinline__ float act_in(float v, int act) {
  if (XACT == 1) return fmaxf(v, 0.f);
  if (XACT == 2) return v * fminf(fmaxf(v + 3.f, 0.f), 6.f) * (1.f / 6.f);
  if (XACT == 3) return act_sel(v, act);
  return v;
}

// T: activation storage type.  NP = 1: operands rounded to bf16 (bf16 mode); NP = 2: hi/lo split (fp32 mode).
// EPI: 0 raw output (+ statistics), 1 affine, 2 affine + ReLU, 3 affine + Hardswish (each + optional residual)
template <typename T, int NP, int STAGES, int BN_MAX, bool DYN, int EPI, int XACT>
__global__ void __launch_bounds__(kThreads, 1) pw_tc_kernel(TcParams p) {
  constexpr bool AFF = EPI != 0;
  constexpr int NPC = BN_MAX / 32;
  constexpr int B_TILE_BYTES = BN_MAX * 128;
  constexpr int STAGE_BYTES = NP * (A_TILE_BYTES + B_TILE_BYTES);
  extern __shared__ __align__(1024) unsigned char smem[];
  unsigned char* stage_base = smem;
  float* s_stage = reinterpret_cast<float*>(smem + STAGES * STAGE_BYTES);      // 8 warps x 32 x STG_LD floats
  float* s_scale = s_stage + 8 * 32 * STG_LD;                                  // [BN_MAX]
  float* s_shift = s_scale + BN_MAX;                                           // [BN_MAX]
  // [8 warps][2][BN_MAX] statistics partials, fp64: a warp adds one 16-row partial per tile to them, over every tile of
  // the CTA (~480 at mn10 block 2 with 256 clips of 10 s); in fp32 the sum of squares would lose the variance to
  // cancellation in E[x^2] - E[x]^2 when the column's mean is many times its std
  double* s_stat = reinterpret_cast<double*>(s_shift + BN_MAX);
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_stat + 8 * 2 * BN_MAX);       // full[S], empty[S]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t bar_full = smem_u32(bars), bar_empty = smem_u32(bars + STAGES);

  if (threadIdx.x == 0) {
    // one elected arrival per producer WARP (after __syncwarp) and one per consumer warpgroup: per-thread arrivals on
    // one shared-memory barrier serialise
    for (int s = 0; s < STAGES; ++s) { mbar_init(bar_full + 8 * s, kGroupThreads / 32); mbar_init(bar_empty + 8 * s, 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  for (int i = threadIdx.x; i < 8 * 2 * BN_MAX; i += kThreads) s_stat[i] = 0.0;
  __syncthreads();

  const int total_tiles = p.m_tiles * p.n_tiles;
  const int K = p.K, N = p.N, BN = p.BN;

  if (warp < 8) {
    // ================================================================= producers (two groups, alternate stages)
    const int grp = warp >> 2;
    const int gtid = threadIdx.x & (kGroupThreads - 1);
    const T* __restrict__ A = reinterpret_cast<const T*>(p.A);
    const int rps = p.xf.rows_per_sample;
    int it = 0;                                                    // global (tile, k-block) counter of this CTA
    // the weight tile of a stage is still valid when the tile that used the stage last had the same (N tile, k-block,
    // sample): true for STAGES / k_blocks tiles back whenever k_blocks divides STAGES (every K <= 64 * STAGES layer)
    const int back = (p.k_blocks <= STAGES && STAGES % p.k_blocks == 0) ? STAGES / p.k_blocks : 0;
    int h0 = -1, h1 = -1, h2 = -1;                                 // keys of the previous three tiles of this CTA
    // tile walk without divisions (m fastest: a CTA stays on one N tile); (nt2, mt2) runs two tiles ahead for the
    // L2 prefetch.  The per-tile scalar work of the producer warps sits on the critical path of every stage hand-over,
    // so it is kept to a minimum and a
    // group skips the tiles it stages nothing for before doing any of it.
    int nt = blockIdx.x / p.m_tiles, mt = blockIdx.x - nt * p.m_tiles;
    int nt2 = nt, mt2 = mt;
    auto advance = [&](int& n, int& m) { m += gridDim.x; while (m >= p.m_tiles) { m -= p.m_tiles; ++n; } };
    advance(nt2, mt2);
    for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
      long long m0, m_lim;
      int bsample;
      tile_rows<DYN>(p, mt, m0, m_lim, bsample);
      if (threadIdx.x == 0) {
        // L2 prefetch of the A rows this CTA stages one (first iteration only) and two tiles from now: a [rows, K]
        // tile is one contiguous range
        if (t == (int)blockIdx.x && t + (int)gridDim.x < total_tiles) {
          long long m2, lim2;
          int b2;
          tile_rows<DYN>(p, mt2, m2, lim2, b2);
          const long long rows2 = lim2 - m2 < BM ? lim2 - m2 : BM;
          l2_prefetch(A + m2 * (long long)K, (uint32_t)(rows2 * K * (long long)sizeof(T)));
        }
      }
      advance(nt2, mt2);
      if (threadIdx.x == 0 && t + 2 * (int)gridDim.x < total_tiles) {
        long long m2, lim2;
        int b2;
        tile_rows<DYN>(p, mt2, m2, lim2, b2);
        const long long rows2 = lim2 - m2 < BM ? lim2 - m2 : BM;
        l2_prefetch(A + m2 * (long long)K, (uint32_t)(rows2 * K * (long long)sizeof(T)));
      }
      const int key = DYN ? (nt * 65536 + bsample) : nt;
      const int hist = back == 1 ? h0 : (back == 2 ? h1 : (back == 3 ? h2 : -1));
      const bool b_resident = (back != 0) && (hist == key);
      h2 = h1; h1 = h0; h0 = key;
      const int n0 = nt * BN;
      advance(nt, mt);                                             // (nt, mt) now describe the NEXT tile
      if (p.k_blocks == 1 && (it & 1) != grp) { ++it; continue; }  // the other group stages this tile
      float datt[4] = {0.f, 0.f, 0.f, 0.f};
      if (DYN) {
#pragma unroll
        for (int j = 0; j < 4; ++j) datt[j] = j < p.dyn_k ? __ldg(p.dyn_att + (size_t)bsample * p.dyn_k + j) : 0.f;
      }
      const int b0 = p.xf.gate != nullptr ? (int)m0 / rps : 0;
      const int off0 = p.xf.gate != nullptr ? (int)m0 - b0 * rps : 0;
      for (int kb = 0; kb < p.k_blocks; ++kb, ++it) {
        if ((it & 1) != grp) continue;
        const int stage = it % STAGES;
        const uint32_t phase = (uint32_t)(it / STAGES) & 1u;
        mbar_wait(bar_empty + 8 * stage, phase ^ 1);
        unsigned char* sA_hi = stage_base + stage * STAGE_BYTES;
        unsigned char* sA_lo = sA_hi + A_TILE_BYTES;                       // only used when NP == 2
        unsigned char* sB_hi = sA_hi + NP * A_TILE_BYTES;
        unsigned char* sB_lo = sB_hi + B_TILE_BYTES;
        // only the 16-byte chunks the MMAs read are produced: nch = 2 per K=16 step
        const int krem = K - kb * BK;
        const int nch = krem >= BK ? 8 : 2 * ((krem + 15) >> 4);
        const int lg = nch <= 2 ? 1 : (nch <= 4 ? 2 : 3);
        const int kc = gtid & ((1 << lg) - 1), r0 = gtid >> lg, rstep = kGroupThreads >> lg;
        const int k = kb * BK + kc * 8;
        const bool kok = kc < nch && k < K;                                // k >= K inside nch: zero fill
        const bool kact = kc < nch;
        float isc[8], ish[8];
        if (XACT >= 0 && kok) {
          const float4 s0 = __ldg(reinterpret_cast<const float4*>(p.xf.scale + k)), s1 = __ldg(reinterpret_cast<const float4*>(p.xf.scale + k) + 1);
          const float4 t0 = __ldg(reinterpret_cast<const float4*>(p.xf.shift + k)), t1 = __ldg(reinterpret_cast<const float4*>(p.xf.shift + k) + 1);
          isc[0] = s0.x; isc[1] = s0.y; isc[2] = s0.z; isc[3] = s0.w; isc[4] = s1.x; isc[5] = s1.y; isc[6] = s1.z; isc[7] = s1.w;
          ish[0] = t0.x; ish[1] = t0.y; ish[2] = t0.z; ish[3] = t0.w; ish[4] = t1.x; ish[5] = t1.y; ish[6] = t1.z; ish[7] = t1.w;
        }
        // ---- A: 128 rows, batches of 4 rows per thread: loads first, then transform + store
        const bool full = m0 + BM <= m_lim;                                  // no row masking needed for this tile
        const T* __restrict__ ap = A + (m0 + r0) * (long long)K + k;
        const size_t astep = (size_t)rstep * K;
        const int nrow = (BM - r0 + rstep - 1) >> (7 - lg);                 // rows this thread covers: r0 + j*rstep
        for (int j0 = 0; j0 < nrow; j0 += 4) {
          float av[4][8];
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int j = j0 + i;
            const bool ok = kok && j < nrow && (full || m0 + r0 + (long long)j * rstep < m_lim);
            if (ok) load_chunk<T>(ap + (size_t)j * astep, av[i]);
            else {
#pragma unroll
              for (int q = 0; q < 8; ++q) av[i][q] = 0.f;
            }
          }
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int j = j0 + i;
            if (j >= nrow || !kact) continue;
            const int row = r0 + j * rstep;
            if (XACT >= 0 || p.xf.gate != nullptr) {
              const bool ok = kok && (full || m0 + row < m_lim);
              if (ok) {
                if (XACT >= 0) {
#pragma unroll
                  for (int q = 0; q < 8; ++q) av[i][q] = act_in<XACT>(fmaf(av[i][q], isc[q], ish[q]), p.xf.act);
                }
                if (p.xf.gate != nullptr) {
                  const int rel = off0 + row;
                  const int bb = b0 + (rps >= BM ? (rel >= rps ? 1 : 0) : rel / rps);
                  const float4* gp = reinterpret_cast<const float4*>(p.xf.gate + (size_t)bb * K + k);
                  const float4 g0 = __ldg(gp), g1 = __ldg(gp + 1);
                  av[i][0] *= g0.x; av[i][1] *= g0.y; av[i][2] *= g0.z; av[i][3] *= g0.w;
                  av[i][4] *= g1.x; av[i][5] *= g1.y; av[i][6] *= g1.z; av[i][7] *= g1.w;
                }
              }
            }
            store_chunk<NP>(sA_hi, sA_lo, swz(row, kc), av[i]);
          }
        }
        // ---- B: BN rows (output channels) of the fp32 weight matrix, batches of 4 rows; skipped while resident
        for (int rb = b_resident ? BN : r0; rb < BN; rb += 4 * rstep) {
          float wv[4][8];
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int r = rb + i * rstep;
            const int n = n0 + r;
            if (kok && r < BN && n < N) {
              if (!DYN) load_chunk<float>(p.W + (size_t)n * K + k, wv[i]);
              else {
#pragma unroll
                for (int j = 0; j < 8; ++j) wv[i][j] = 0.f;
                for (int kk = 0; kk < p.dyn_k; ++kk) {
                  float t8[8];
                  load_chunk<float>(p.W + (size_t)kk * N * K + (size_t)n * K + k, t8);
#pragma unroll
                  for (int j = 0; j < 8; ++j) wv[i][j] = fmaf(datt[kk], t8[j], wv[i][j]);
                }
              }
            } else {
#pragma unroll
              for (int j = 0; j < 8; ++j) wv[i][j] = 0.f;
            }
          }
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int r = rb + i * rstep;
            if (r < BN && kact) store_chunk<NP>(sB_hi, sB_lo, swz(r, kc), wv[i]);
          }
        }
        fence_proxy_async();
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_full + 8 * stage);
          }
    }
  } else {
    // ================================================================= consumers: MMA + epilogue (two warpgroups)
    const int ew = warp - kFirstCons;                             // 0..7
    const int g = ew >> 2;                                        // 64-row half of the tile
    const int wq = ew & 3;                                        // rows 16 wq .. 16 wq + 15 of the half
    float* stg = s_stage + ew * 32 * STG_LD;
    double* my_sum = s_stat + ew * 2 * BN_MAX;
    double* my_sq = my_sum + BN_MAX;
    T* __restrict__ C = reinterpret_cast<T*>(p.C);
    const T* __restrict__ R = reinterpret_cast<const T*>(p.residual);
    const int etid = threadIdx.x - kFirstCons * 32;               // 0..255
    const int col4 = (lane & 7) * 4, rg = lane >> 3;
    const int fr = lane >> 2, fc = 2 * (lane & 3);                // fragment row / column of this lane
    int cur_nt = -1;
    int it = 0;
    const bool do_stats = p.stat_sum != nullptr;
    int ent = blockIdx.x / p.m_tiles, emt = blockIdx.x - ent * p.m_tiles;
    for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
      const int nt = ent, mt = emt;
      emt += gridDim.x;
      while (emt >= p.m_tiles) { emt -= p.m_tiles; ++ent; }
      long long m0, m_lim;
      int bsample;
      tile_rows<DYN>(p, mt, m0, m_lim, bsample);
      const int n0 = nt * BN;
      if (nt != cur_nt) {
        // new N tile: flush the previous tile's statistics, stage this tile's epilogue affine
        asm volatile("bar.sync 1, 256;" ::: "memory");
        for (int i = etid; i < BN; i += kEpiThreads) {
          if (do_stats && cur_nt >= 0) {
            const int n = cur_nt * BN + i;
            double a = 0.0, b = 0.0;
#pragma unroll
            for (int w = 0; w < 8; ++w) { a += s_stat[w * 2 * BN_MAX + i]; b += s_stat[w * 2 * BN_MAX + BN_MAX + i]; }
            if (n < N) { atomicAdd(p.stat_sum + n, a); atomicAdd(p.stat_sq + n, b); }
#pragma unroll
            for (int w = 0; w < 8; ++w) { s_stat[w * 2 * BN_MAX + i] = 0.0; s_stat[w * 2 * BN_MAX + BN_MAX + i] = 0.0; }
          }
          const int n = n0 + i;
          s_scale[i] = (p.scale != nullptr && n < N) ? p.scale[n] : 1.f;
          s_shift[i] = (p.shift != nullptr && n < N) ? p.shift[n] : 0.f;
        }
        cur_nt = nt;
        asm volatile("bar.sync 1, 256;" ::: "memory");
      }
      if (AFF && R != nullptr && p.n_tiles == 1 && etid == 0) {
        const int t2 = t + gridDim.x;                  // residual rows of this CTA's next tile (contiguous: BN == N)
        if (t2 < total_tiles) {
          long long m2, lim2;
          int b2;
          tile_rows<DYN>(p, t2, m2, lim2, b2);
          const long long rows2 = lim2 - m2 < BM ? lim2 - m2 : BM;
          l2_prefetch(R + m2 * (long long)N, (uint32_t)(rows2 * N * (long long)sizeof(T)));
        }
      }
      float acc[NPC][16];
#pragma unroll
      for (int c = 0; c < NPC; ++c)
#pragma unroll
        for (int i = 0; i < 16; ++i) acc[c][i] = 0.f;
      for (int kb = 0; kb < p.k_blocks; ++kb, ++it) {
        const int stage = it % STAGES;
        const uint32_t phase = (uint32_t)(it / STAGES) & 1u;
        mbar_wait(bar_full + 8 * stage, phase);
        const uint32_t sA_hi = smem_u32(stage_base + stage * STAGE_BYTES) + (uint32_t)g * 8192u;   // rows 64 g ..
        const uint32_t sA_lo = sA_hi + A_TILE_BYTES;
        const uint32_t sB_hi = smem_u32(stage_base + stage * STAGE_BYTES) + NP * A_TILE_BYTES;
        const uint32_t sB_lo = sB_hi + B_TILE_BYTES;
        const int krem = K - kb * BK;
        const int nk16 = krem >= BK ? BK / 16 : (krem + 15) / 16;
        wgmma_fence();
        for (int k16 = 0; k16 < nk16; ++k16) {
          const uint32_t ko = k16 * 32;                         // 16 bf16 = 32 bytes along K inside the swizzle row
          mma_pieces<NPC>(acc, gmma_desc(sA_hi + ko), gmma_desc(sB_hi + ko), BN);
          if (NP == 2) {
            mma_pieces<NPC>(acc, gmma_desc(sA_lo + ko), gmma_desc(sB_hi + ko), BN);
            mma_pieces<NPC>(acc, gmma_desc(sA_hi + ko), gmma_desc(sB_lo + ko), BN);
          }
        }
        wgmma_commit();
        wgmma_wait<0>();
#pragma unroll
        for (int c = 0; c < NPC; ++c) wgmma_fence_regs(acc[c]);
        asm volatile("bar.sync %0, 128;" ::"r"(2 + g) : "memory");   // every warp of the group is past its wait
        if (etid == g * 128) mbar_arrive(bar_empty + 8 * stage);   // frees the smem stage
      }
      const long long mrow0 = m0 + g * 64 + wq * 16;
      const int rows_left = (int)(m_lim - mrow0 < 16 ? m_lim - mrow0 : 16);     // valid rows of this warp's slab
#pragma unroll
      for (int c = 0; c < NPC; ++c) {
        if (c * 32 >= BN) break;
        // fragment -> stg[row][col] (16 rows x 32 columns of chunk c)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          *reinterpret_cast<float2*>(stg + fr * STG_LD + 8 * j + fc) = make_float2(acc[c][4 * j], acc[c][4 * j + 1]);
          *reinterpret_cast<float2*>(stg + (fr + 8) * STG_LD + 8 * j + fc) = make_float2(acc[c][4 * j + 2], acc[c][4 * j + 3]);
        }
        __syncwarp();
        // now lane -> (row group rg = lane / 8, 4 columns at col4); 4 iterations cover the 16 rows
        const int cl = c * 32 + col4;
        const int n = n0 + cl;
        const bool nok = cl < BN && n < N;
        const float4 sc4 = *reinterpret_cast<const float4*>(s_scale + (cl < BN_MAX ? cl : 0));
        const float4 sh4 = *reinterpret_cast<const float4*>(s_shift + (cl < BN_MAX ? cl : 0));
        T* __restrict__ cp = C + (mrow0 + rg) * (long long)N + n;
        const size_t cstep = (size_t)4 * N;
        float res[4][4];
        if (AFF && R != nullptr) {
          const T* __restrict__ rp = R + (mrow0 + rg) * (long long)N + n;
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            if (nok && i * 4 + rg < rows_left) OutVec<T>::load(rp + i * cstep, res[i]);
            else { res[i][0] = res[i][1] = res[i][2] = res[i][3] = 0.f; }
          }
        }
        float cs[4] = {0.f, 0.f, 0.f, 0.f}, cq[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int row = i * 4 + rg;
          const float4 v4 = *reinterpret_cast<const float4*>(stg + row * STG_LD + col4);
          float v[4] = {v4.x, v4.y, v4.z, v4.w};
          if (row < rows_left) {
            if (EPI == 0) {
#pragma unroll
              for (int j = 0; j < 4; ++j) { cs[j] += v[j]; cq[j] = fmaf(v[j], v[j], cq[j]); }
            }
            if (nok) {
              if (AFF) {      // folded BatchNorm / bias + activation (+ residual); compiled out for raw outputs
                v[0] = act_epi<EPI>(fmaf(v[0], sc4.x, sh4.x));
                v[1] = act_epi<EPI>(fmaf(v[1], sc4.y, sh4.y));
                v[2] = act_epi<EPI>(fmaf(v[2], sc4.z, sh4.z));
                v[3] = act_epi<EPI>(fmaf(v[3], sc4.w, sh4.w));
                if (R != nullptr) {
#pragma unroll
                  for (int j = 0; j < 4; ++j) v[j] += res[i][j];
                }
              }
              OutVec<T>::store(cp + i * cstep, v);
            }
          }
        }
        if (do_stats) {
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            cs[j] += __shfl_xor_sync(0xffffffffu, cs[j], 8);
            cq[j] += __shfl_xor_sync(0xffffffffu, cq[j], 8);
            cs[j] += __shfl_xor_sync(0xffffffffu, cs[j], 16);
            cq[j] += __shfl_xor_sync(0xffffffffu, cq[j], 16);
          }
          if (lane < 8 && cl < BN) {
#pragma unroll
            for (int j = 0; j < 4; ++j) { my_sum[cl + j] += (double)cs[j]; my_sq[cl + j] += (double)cq[j]; }
          }
        }
        __syncwarp();
      }
    }
    // final statistics flush
    asm volatile("bar.sync 1, 256;" ::: "memory");
    if (do_stats && cur_nt >= 0) {
      for (int i = etid; i < BN; i += kEpiThreads) {
        const int n = cur_nt * BN + i;
        double a = 0.0, b = 0.0;
#pragma unroll
        for (int w = 0; w < 8; ++w) { a += s_stat[w * 2 * BN_MAX + i]; b += s_stat[w * 2 * BN_MAX + BN_MAX + i]; }
        if (n < N) { atomicAdd(p.stat_sum + n, a); atomicAdd(p.stat_sq + n, b); }
      }
    }
  }
  __syncthreads();
}

template <typename T, int NP, int STAGES, int BN_MAX, bool DYN, int EPI, int XACT>
int launch_tc_x(const TcParams& p0, cudaStream_t st) {
  TcParams p = p0;
  p.n_tiles = ceil_div(p.N, BN_MAX);
  p.BN = ceil_div(ceil_div(p.N, p.n_tiles), 16) * 16;
  p.n_tiles = ceil_div(p.N, p.BN);
  if (DYN) {
    p.tps = ceil_div(p.tile_rps, BM);
    p.m_tiles = (p.M / p.tile_rps) * p.tps;
  } else {
    p.tps = 0;
    p.m_tiles = ceil_div(p.M, BM);
  }
  p.k_blocks = ceil_div(p.K, BK);
  constexpr size_t smem = (size_t)STAGES * NP * (A_TILE_BYTES + BN_MAX * 128) + 8 * 32 * STG_LD * sizeof(float) +
                          2 * BN_MAX * sizeof(float) + 16 * BN_MAX * sizeof(double) +
                          2 * STAGES * sizeof(uint64_t) + 16;
  static_assert(smem <= 227 * 1024, "shared memory budget");
  static unsigned long long attr_mask = 0;
  if (int rc = eat_opt_in_smem(pw_tc_kernel<T, NP, STAGES, BN_MAX, DYN, EPI, XACT>, smem, attr_mask)) return rc;
  int dev = 0, sms = kNumSMs;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int tiles = p.m_tiles * p.n_tiles;
  const int grid = tiles < sms ? tiles : sms;
  pw_tc_kernel<T, NP, STAGES, BN_MAX, DYN, EPI, XACT><<<grid, kThreads, smem, st>>>(p);
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

// instantiated input transforms: the raw-output (training / data-gradient) kernel gets compile-time activations, the
// fused-epilogue (eval) kernels normally see already-activated inputs and keep one run-time variant for the rest
template <typename T, int NP, int STAGES, int BN_MAX, bool DYN, int EPI>
int launch_tc_aff(const TcParams& p, cudaStream_t st) {
  if (p.xf.scale == nullptr) return launch_tc_x<T, NP, STAGES, BN_MAX, DYN, EPI, -1>(p, st);
  if constexpr (DYN) {
    eat_set_error("pw_tc_dyn: input BatchNorm/activation on load is not instantiated for DynamicConv");
    return EAT_ERR_UNSUPPORTED;
  } else if constexpr (EPI == 0) {
    if (p.xf.act == EAT_ACT_RELU) return launch_tc_x<T, NP, STAGES, BN_MAX, DYN, EPI, 1>(p, st);
    if (p.xf.act == EAT_ACT_HSWISH) return launch_tc_x<T, NP, STAGES, BN_MAX, DYN, EPI, 2>(p, st);
    return launch_tc_x<T, NP, STAGES, BN_MAX, DYN, EPI, 0>(p, st);
  } else {
    return launch_tc_x<T, NP, STAGES, BN_MAX, DYN, EPI, 3>(p, st);
  }
}

template <typename T, int NP, int STAGES, int BN_MAX, bool DYN>
int launch_tc(const TcParams& p, cudaStream_t st) {
  const bool aff = p.scale != nullptr || p.shift != nullptr || p.act != 0 || p.residual != nullptr;
  if (!aff) return launch_tc_aff<T, NP, STAGES, BN_MAX, DYN, 0>(p, st);
  if (p.act == EAT_ACT_RELU) return launch_tc_aff<T, NP, STAGES, BN_MAX, DYN, 2>(p, st);
  if (p.act == EAT_ACT_HSWISH) return launch_tc_aff<T, NP, STAGES, BN_MAX, DYN, 3>(p, st);
  return launch_tc_aff<T, NP, STAGES, BN_MAX, DYN, 1>(p, st);
}

}  // namespace

extern "C" int eat_pw_tc_fwd(const void* A, int a_dtype, const float* W, int w_trans, void* C, int c_dtype, long long M,
                             int N, int K, const float* in_scale, const float* in_shift, int in_act, const float* gate,
                             int rows_per_sample, const float* scale, const float* shift, int act, const void* residual,
                             double* stat_sum, double* stat_sq, cudaStream_t st) {
  if (M == 0) return EAT_OK;
  if (act == EAT_ACT_SIGMOID || in_act == EAT_ACT_SIGMOID) { eat_set_error("pw_tc: sigmoid epilogues run on the CUDA-core GEMM (eat_gemm_simt_fwd)"); return EAT_ERR_UNSUPPORTED; }
  if (stat_sum != nullptr && (scale != nullptr || shift != nullptr || act != 0 || residual != nullptr)) {
    eat_set_error("pw_tc: batch statistics are produced by the raw-output variant only (no affine/activation/residual)");
    return EAT_ERR_UNSUPPORTED;
  }
  if (w_trans) { eat_set_error("pw_tc: transposed weights are not supported (pre-transpose with eat_transpose_f32)"); return EAT_ERR_UNSUPPORTED; }
  if (a_dtype != c_dtype) { eat_set_error("pw_tc: A and C must share the storage dtype"); return EAT_ERR_UNSUPPORTED; }
  if (K % 8 != 0 || N % 8 != 0) { eat_set_error("pw_tc: K and N must be multiples of 8"); return EAT_ERR_ARG; }
  if (M >= (1ll << 31) - BM) { eat_set_error("pw_tc: M too large"); return EAT_ERR_ARG; }
  if ((((uintptr_t)A) | ((uintptr_t)W) | ((uintptr_t)C) | ((uintptr_t)in_scale) | ((uintptr_t)in_shift)) & 15) { eat_set_error("pw_tc: operands must be 16-byte aligned"); return EAT_ERR_ARG; }
  if (a_dtype == EAT_F32 && !(residual != nullptr && act != EAT_ACT_NONE)) {
    static const bool use_tma = [] { const char* e = getenv("EAT_PW_IMPL"); return e == nullptr || strcmp(e, "tc") != 0; }();
    if (use_tma)     // fp32 storage: the TMA-fed kernel (pw_tma.cu)
      return eat_pw_tma_fwd((const float*)A, W, 0, (float*)C, M, N, K, in_scale, in_shift, in_act, gate, rows_per_sample, scale,
                            shift, act, (const float*)residual, stat_sum, stat_sq, nullptr, 0, st);
  }
  TcParams p;
  p.A = A; p.W = W; p.C = C; p.residual = residual; p.M = (int)M; p.N = N; p.K = K;
  p.xf = InXform{in_scale, in_shift, gate, in_act, rows_per_sample > 0 ? rows_per_sample : 1};
  p.scale = scale; p.shift = shift; p.act = act; p.stat_sum = stat_sum; p.stat_sq = stat_sq;
  p.dyn_att = nullptr; p.dyn_k = 0; p.tps = 0; p.tile_rps = 0;
  if (a_dtype == EAT_BF16) return launch_tc<__nv_bfloat16, 1, 4, 128, false>(p, st);
  return launch_tc<float, 2, 2, 128, false>(p, st);
}

// DynamicConv 1x1 (reference models/dymn/dy_block.py:103-131): W holds dyn_k kernels [dyn_k][N][K]; sample b uses
// sum_k att[b,k] * W[k].  M = B * rows_per_sample; rows of a tile never cross a sample.
extern "C" int eat_pw_tc_dyn_fwd(const void* A, int dtype, const float* W, const float* att, int dyn_k, void* C,
                                 long long M, int N, int K, int rows_per_sample, const float* in_scale,
                                 const float* in_shift, int in_act, const float* scale, const float* shift, int act,
                                 const void* residual, double* stat_sum, double* stat_sq, cudaStream_t st) {
  if (M == 0) return EAT_OK;
  if (dyn_k < 1 || dyn_k > 4) { eat_set_error("pw_tc_dyn: 1..4 kernels supported"); return EAT_ERR_UNSUPPORTED; }
  if (rows_per_sample < 1 || M % rows_per_sample != 0) { eat_set_error("pw_tc_dyn: M must be B * rows_per_sample"); return EAT_ERR_ARG; }
  if (K % 8 != 0 || N % 8 != 0) { eat_set_error("pw_tc_dyn: K and N must be multiples of 8"); return EAT_ERR_ARG; }
  if (M >= (1ll << 31) - BM) { eat_set_error("pw_tc_dyn: M too large"); return EAT_ERR_ARG; }
  TcParams p;
  p.A = A; p.W = W; p.C = C; p.residual = residual; p.M = (int)M; p.N = N; p.K = K;
  p.xf = InXform{in_scale, in_shift, nullptr, in_act, rows_per_sample};
  p.scale = scale; p.shift = shift; p.act = act; p.stat_sum = stat_sum; p.stat_sq = stat_sq;
  p.dyn_att = att; p.dyn_k = dyn_k; p.tile_rps = rows_per_sample; p.tps = 1;
  if (dtype == EAT_BF16) return launch_tc<__nv_bfloat16, 1, 4, 128, true>(p, st);
  return launch_tc<float, 2, 2, 128, true>(p, st);
}

// [R, Cc] fp32 -> [Cc, R]  (weights for the data-gradient GEMM)
namespace {
__global__ void transpose_kernel(const float* __restrict__ in, float* __restrict__ out, int R, int Cc) {
  __shared__ float tile[32][33];
  int x = blockIdx.x * 32 + threadIdx.x, y = blockIdx.y * 32 + threadIdx.y;
  for (int j = 0; j < 32; j += 8)
    if (x < Cc && y + j < R) tile[threadIdx.y + j][threadIdx.x] = in[(size_t)(y + j) * Cc + x];
  __syncthreads();
  x = blockIdx.y * 32 + threadIdx.x;
  y = blockIdx.x * 32 + threadIdx.y;
  for (int j = 0; j < 32; j += 8)
    if (x < R && y + j < Cc) out[(size_t)(y + j) * R + x] = tile[threadIdx.x][threadIdx.y + j];
}
}  // namespace

extern "C" int eat_transpose_f32(const float* in, float* out, int rows, int cols, cudaStream_t st) {
  if (rows == 0 || cols == 0) return EAT_OK;
  dim3 grid(ceil_div(cols, 32), ceil_div(rows, 32)), block(32, 8);
  transpose_kernel<<<grid, block, 0, st>>>(in, out, rows, cols);
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}
