// Pointwise (1x1) convolution / Linear for fp32 activations as a TMA-fed wgmma GEMM (sm_90a), bf16x3 products:
//     C[M,N] = epi( xf(A)[M,K] . W[N,K]^T  (+ R[M,N]) )          A, C, R: NHWC activation rows, fp32; W: fp32
// Same contract and reference call sites as pw_wgmma.cu (models/mn/block_types.py:140-147,167-171;
// models/mn/model.py:160-166; every data-gradient GEMM of loss.backward(), ex_audioset.py:197).
//
// Why a second kernel: in pw_wgmma.cu eight producer warps carry every operand byte global -> registers -> smem.
// Here no thread touches global memory on the operand path:
//
//   warp 12  TMA producer : ONE thread.  cp.async.bulk.tensor (2-D tiled, SWIZZLE_128B) lands raw fp32 tiles of A
//                           [128 rows x 32 k] (and of W, and of the residual R) in a ring of shared-memory stages;
//                           ragged M / K / N edges are zero-filled by the TMA unit.
//   warps 0-3 fix-up      : on-chip pass over a landed tile: (BatchNorm affine + activation + SE gate of the producing
//                           layer for training-mode operands), then the 32 fp32 values of a row (128 bytes) are
//                           replaced IN PLACE by 32 bf16 "hi" values (64 bytes) followed by 32 bf16 "lo" values with
//                           hi + lo = v to ~2^-17 -- the row is then a 64-element bf16 K-major row of the same
//                           128-byte-swizzled tile the TMA wrote, which wgmma reads as is.  No second buffer.
//   warps 4-11 consumers  : two warpgroups, one per 64-row half of the 128-row tile.  Each issues ONE
//                           wgmma.m64nBNk16 (bf16, BN = the whole N tile) per product and K=16 step for the three
//                           products hi*hi + lo*hi + hi*lo (fp32-grade, ~2^-16) -- the A / B descriptors simply point at
//                           the hi or lo half of the row -- into register accumulators, one MMA group kept in flight
//                           while the next stage is waited for.  The tile width (any multiple of 8 up to 128 columns,
//                           planned from N so that no tile is padded by more than 7 columns) is a template parameter,
//                           so every MMA is issued unconditionally and reads the A slab once.  The residual: R tiles ride the same
//                           pipeline as extra k-blocks, get the same in-place hi/lo split, and hi + lo is added to the
//                           accumulator fragments straight from shared memory.
//                           Epilogue from registers: shift + activation -> 128B-swizzled 16-row staging tile per warp
//                           -> cp.async.bulk.tensor store (ragged edges clipped by the TMA unit); the 8 / 16 / 24-column
//                           tail chunk of a tile goes through a tensor map of that box width, so that no store reaches
//                           into the neighbouring N tile.  BatchNorm batch
//                           statistics: each lane sums one column of the staged tile and keeps its partial sums in
//                           registers across all tiles of the CTA.
// The folded-BatchNorm scale of the epilogue is applied to the WEIGHT rows during their fix-up (W is tiny), which is
// what lets the residual go through the accumulator unscaled.  Weights whose hi/lo tiles fit stay resident in shared
// memory for the whole N tile; larger K streams W k-blocks with A.
// HBM-bound at mn10 widths: algorithmic bytes per launch = 4*(M*K + M*N (+ M*N residual) + N*K).
#include <type_traits>
#include <utility>

#include "tma_common.cuh"

namespace {
using namespace tc;
using namespace tma;

constexpr int BM = 128;
constexpr int BN_MAX = 128;             // widest N tile: 64 accumulator registers per consumer thread
constexpr int A_TILE = BM * 128;        // 16 KB
constexpr int kThreads = 416;           // 4 fix-up warps, 8 consumer warps (2 warpgroups), TMA warp
constexpr int kFirstCons = 4, kTmaWarp = 12, kConsThreads = 256;
constexpr int STG_BYTES = 16 * 128;     // one staged 16 x 32 fp32 sub-tile

struct TmaParams {
  int M, N, K;
  int BN, n_tiles, m_tiles, k_blocks, r_blocks;   // r_blocks: residual k-blocks per tile (0: no residual)
  int bnp;                                        // BN_MAX: stride of the per-column shared-memory tables
  int stages, wres;                               // wres != 0: weight hi/lo tiles resident per N tile
  int stg_bufs;                                   // staging buffers per consumer warp (1 or 2)
  int wpre;                                       // weights arrive pre-split (bf16 hi|lo rows, scale folded): no weight fix-up
  int n_samples, tps, tile_rps;                   // M = n_samples * tile_rps rows; tps M tiles per sample (tiles never straddle
                                                  // samples; 1 sample = the whole matrix for ordinary layers)
  int wdyn;                                       // per-sample weights (DynamicConv): the weight map's third coordinate is the sample
  uint32_t stage_bytes, off_w, off_stg, off_f, off_bar;   // shared-memory carve-up (bytes)
  int kpad;                                       // floats reserved for each of the in-transform vectors (0: none)
  const float* in_scale; const float* in_shift; const float* gate; int in_act; int rps;
  const float* scale; const float* shift;        // epilogue affine (scale is folded into W)
  double* stat_sum; double* stat_sq;
};

// EPI : 0 raw output (+ statistics), 1 + shift, 2 + shift + ReLU, 3 + shift + Hardswish   (scale lives in W)
// XACT: -1 raw operand (gate still possible), 0 affine, 1 affine + ReLU, 2 affine + Hardswish on load
// BN  : columns of the N tile, a multiple of 8; the epilogue walks it in 32-column chunks, the last one TAIL wide
// mapCt: output map with a TAIL-column box (unswizzled) for the last chunk of a tile that has another tile after it
template <int EPI, int XACT, int BN>
__global__ void __launch_bounds__(kThreads, 1)   // 13 warps: 4 on one scheduler, so at most 128 registers per thread
pw_tma_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapW,
              const __grid_constant__ CUtensorMap mapC, const __grid_constant__ CUtensorMap mapCt,
              const __grid_constant__ CUtensorMap mapR, const TmaParams p) {
  constexpr int NC = (BN + 31) / 32;                     // 32-column chunks of the epilogue
  constexpr int TAIL = BN % 32;                          // width of the last chunk when it is not a full one
  extern __shared__ __align__(1024) unsigned char smem[];
  unsigned char* s_w = smem + p.off_w;                   // resident weights: [k_blocks][hi | lo][BN rows x 128 B]
  unsigned char* s_stg = smem + p.off_stg;               // [8 consumer warps][stg_bufs][2 KB]
  float* s_isc = reinterpret_cast<float*>(smem + p.off_f);             // [kpad] in-transform scale (0 beyond K)
  float* s_ish = s_isc + p.kpad;                                       // [kpad]
  float* s_shift = s_ish + p.kpad;                                     // [bnp] epilogue shift of the current N tile
  float* s_stat = s_shift + p.bnp;                                     // [8][2][bnp]
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + p.off_bar);
  const int S = p.stages;
  const uint32_t bar_full = smem_u32(bars), bar_ready = bar_full + 8 * S, bar_empty = bar_ready + 8 * S;
  const uint32_t bar_wfull = bar_empty + 8 * S;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    // empty: one arrival per consumer warpgroup once its MMAs on the stage have completed
    for (int s = 0; s < S; ++s) { mbar_init(bar_full + 8 * s, 1); mbar_init(bar_ready + 8 * s, 4); mbar_init(bar_empty + 8 * s, 2); }
    mbar_init(bar_wfull, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&mapA)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&mapW)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&mapC)) : "memory");
    if (TAIL != 0) asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&mapCt)) : "memory");
  }
  // one-time tables: in-transform vectors (zero beyond K: act(0) = 0)
  if (XACT >= 0) {
    for (int i = threadIdx.x; i < p.kpad; i += kThreads) {
      s_isc[i] = i < p.K ? p.in_scale[i] : 0.f;
      s_ish[i] = i < p.K ? p.in_shift[i] : 0.f;
    }
  }
  for (int i = threadIdx.x; i < 16 * p.bnp; i += kThreads) s_stat[i] = 0.f;
  fence_proxy_async();
  __syncthreads();

  const int total_tiles = p.m_tiles * p.n_tiles;
  const int kb_total = p.k_blocks + p.r_blocks;          // pipeline slots per tile
  const uint32_t w_tile = (uint32_t)BN * 128u;           // bytes of one [BN x 32] weight tile
  const uint32_t stage_base = smem_u32(smem);
  // tile walk: the grid is a multiple of n_tiles; CTA b keeps N tile b % n_tiles (its weights stay resident) and takes every
  // cpn-th M tile from b / n_tiles on.  The n_tiles CTAs of one M tile run at about the same time, so its A rows come from
  // HBM once and from L2 for the other N tiles.  A CTA gets as many tiles as t = b, b + gridDim.x, ... < total_tiles counts.
  const int cpn = gridDim.x / p.n_tiles;
  const int nt = blockIdx.x % p.n_tiles;
  int mt = blockIdx.x / p.n_tiles;
  auto next_tile = [&]() { mt += cpn; };
  // (sample, M tile inside the sample) of M tile `m`; one sample = no division on the ordinary path
  auto split_tile = [&](int m, int& bs, int& jt) { if (p.n_samples == 1) { bs = 0; jt = m; } else { bs = m / p.tps; jt = m - bs * p.tps; } };

  if (warp == kTmaWarp) {
    // ================================================================= TMA producer (one thread)
    if (lane == 0) {
      int s = 0, s_prev = 0, cur_nt = -1;
      uint32_t ph = 0, ph_prev = 0;
      bool first = true;
      for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
        int bs, jt;
        split_tile(mt, bs, jt);
        const int m0 = jt * BM, n0 = nt * BN;                    // m0: row inside the sample
        const int wb = p.wdyn ? bs : 0;
        const int wkey = nt * p.n_samples + wb;
        if (p.wres && wkey != cur_nt) {
          // every MMA that reads the old weights has completed once the most recently filled stage was released
          if (!first) mbar_wait(bar_empty + 8 * s_prev, ph_prev);
          mbar_expect_tx(bar_wfull, (uint32_t)p.k_blocks * w_tile);
          for (int kb = 0; kb < p.k_blocks; ++kb)
            tma_load_3d(&mapW, bar_wfull, smem_u32(s_w) + (uint32_t)kb * w_tile, kb * (p.wpre ? 2 * KB : KB), n0, wb);
          cur_nt = wkey;
        }
        next_tile();
        for (int kb = 0; kb < kb_total; ++kb) {
          mbar_wait(bar_empty + 8 * s, ph ^ 1u);
          const uint32_t dst = stage_base + (uint32_t)s * p.stage_bytes;
          if (kb < p.k_blocks) {
            mbar_expect_tx(bar_full + 8 * s, A_TILE + (p.wres ? 0u : w_tile));
            tma_load_3d(&mapA, bar_full + 8 * s, dst, kb * KB, m0, bs);
            if (!p.wres) tma_load_3d(&mapW, bar_full + 8 * s, dst + A_TILE, kb * (p.wpre ? 2 * KB : KB), n0, wb);
          } else {
            mbar_expect_tx(bar_full + 8 * s, A_TILE);
            tma_load_3d(&mapR, bar_full + 8 * s, dst, n0 + (kb - p.k_blocks) * KB, m0, bs);
          }
          s_prev = s; ph_prev = ph; first = false;
          if (++s == S) { s = 0; ph ^= 1u; }
        }
      }
    }
    __syncwarp();
  } else if (warp < kFirstCons) {
    // ================================================================= fix-up warps (128 threads)
    const int ft = threadIdx.x;
    int s = 0, cur_nt = -1;
    uint32_t ph = 0, wphase = 0;
    const bool fold = EPI != 0 && p.scale != nullptr;
    auto do_fix_w = [&](unsigned char* w, int kb, int n0) {
      const int lg = pair_lg(p.K - kb * KB);
      if (fold) {
        if (lg == 2) fix_w<2, true>(w, ft, BN, p.scale, n0, p.N);
        else fix_w<1, true>(w, ft, BN, p.scale, n0, p.N);
      } else {
        if (lg == 2) fix_w<2, false>(w, ft, BN, nullptr, n0, p.N);
        else fix_w<1, false>(w, ft, BN, nullptr, n0, p.N);
      }
    };
    for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
      int bs, jt;
      split_tile(mt, bs, jt);
      const int n0 = nt * BN;
      const int rows_valid = min(BM, p.tile_rps - jt * BM);
      const int wkey = nt * p.n_samples + (p.wdyn ? bs : 0);
      if (p.wres && wkey != cur_nt) {
        mbar_wait(bar_wfull, wphase);
        wphase ^= 1u;
        if (!p.wpre)
          for (int kb = 0; kb < p.k_blocks; ++kb) do_fix_w(s_w + (size_t)kb * w_tile, kb, n0);
        cur_nt = wkey;
      }
      next_tile();
      int b0 = 0, off0 = 0;
      if (p.gate != nullptr) { const int m0 = bs * p.tile_rps + jt * BM; b0 = m0 / p.rps; off0 = m0 - b0 * p.rps; }
      for (int kb = 0; kb < kb_total; ++kb) {
        mbar_wait(bar_full + 8 * s, ph);
        unsigned char* tile = smem + (size_t)s * p.stage_bytes;
        if (kb >= p.k_blocks) {
          fix_a<2, -1>(tile, ft, BM, nullptr, nullptr, 0, nullptr, 0, 0, 1, 0);                   // residual tile: plain split
        } else {
          const int lg = pair_lg(p.K - kb * KB);
          const int k = kb * KB + (ft & ((1 << lg) - 1)) * 8;
          if (lg == 2) fix_a<2, XACT>(tile, ft, rows_valid, s_isc, s_ish, k, p.gate, off0, b0, p.rps, p.K);
          else fix_a<1, XACT>(tile, ft, rows_valid, s_isc, s_ish, k, p.gate, off0, b0, p.rps, p.K);
          if (!p.wres && !p.wpre) do_fix_w(tile + A_TILE, kb, n0);
        }
        fence_proxy_async();
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_ready + 8 * s);
        if (++s == S) { s = 0; ph ^= 1u; }
      }
    }
  } else {
    // ================================================================= consumers: MMA + epilogue (two warpgroups)
    const int cw = warp - kFirstCons;                         // 0..7
    const int g = cw >> 2;                                    // 64-row half of the tile
    const int wq = cw & 3;                                    // warp inside the warpgroup: rows 16 wq .. 16 wq + 15
    const int ctid = threadIdx.x - kFirstCons * 32;           // 0..255
    unsigned char* stg = s_stg + (size_t)cw * p.stg_bufs * STG_BYTES;
    const int bnp = p.bnp;
    float* my_stat = s_stat + cw * 2 * bnp;
    const bool do_stats = EPI == 0 && p.stat_sum != nullptr;
    const uint64_t desc0 = gmma_desc(0);                      // descriptor of address 0: add (address >> 4)
    const uint64_t wres0 = desc0 + (smem_u32(s_w) >> 4);
    const uint32_t w_tile16 = w_tile >> 4;
    float csum[NC], csq[NC];
#pragma unroll
    for (int c = 0; c < NC; ++c) { csum[c] = 0.f; csq[c] = 0.f; }
    int cur_nt = -1, cb = 0, s = 0;
    uint32_t ph = 0;
    auto flush_stats = [&](int nt_old) {
      // lane partials -> shared, combine the eight warps, one fp64 atomic per channel (lanes past a tail chunk hold 0)
#pragma unroll
      for (int c = 0; c < NC; ++c) { my_stat[c * 32 + lane] = csum[c]; my_stat[bnp + c * 32 + lane] = csq[c]; csum[c] = 0.f; csq[c] = 0.f; }
      asm volatile("bar.sync 1, 256;" ::: "memory");
      for (int e = ctid; e < BN; e += kConsThreads) {
        const int n = nt_old * BN + e;
        float a = 0.f, b = 0.f;
#pragma unroll
        for (int w = 0; w < 8; ++w) { a += s_stat[w * 2 * bnp + e]; b += s_stat[w * 2 * bnp + bnp + e]; }
        if (n < p.N) { atomicAdd(p.stat_sum + n, (double)a); atomicAdd(p.stat_sq + n, (double)b); }
      }
      asm volatile("bar.sync 1, 256;" ::: "memory");
    };
    for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
      int bs, jt;
      split_tile(mt, bs, jt);
      const int m0 = jt * BM, n0 = nt * BN;                      // m0: row inside the sample
      if (nt != cur_nt) {
        if (do_stats && cur_nt >= 0) flush_stats(cur_nt);
        if (EPI != 0) {
          asm volatile("bar.sync 2, 256;" ::: "memory");       // everyone is done with the previous tile's shifts
          for (int e = ctid; e < BN; e += kConsThreads) s_shift[e] = (p.shift != nullptr && n0 + e < p.N) ? p.shift[n0 + e] : 0.f;
          asm volatile("bar.sync 2, 256;" ::: "memory");
        }
        cur_nt = nt;
      }
      next_tile();
      // m64nBN fragment: acc[16 c + 4 j + ...] holds columns 32 c + 8 j + fc (+1) of chunk c
      float acc[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
      // the group of MMAs on stage `pend` may still be running; a stage is released once its group has completed
      int pend = -1;
      auto release = [&](int st) {
        asm volatile("bar.sync %0, 128;" ::"r"(3 + g) : "memory");   // every warp of the group is past its wait
        if (ctid == g * 128) mbar_arrive(bar_empty + 8 * st);
      };
      const int fr = lane >> 2, fc = 2 * (lane & 3);           // fragment row / column of this lane
      for (int kb = 0; kb < kb_total; ++kb) {
        mbar_wait(bar_ready + 8 * s, ph);
        const uint32_t sa = stage_base + (uint32_t)s * p.stage_bytes;
        if (kb < p.k_blocks) {
          // row = [hi: 32 bf16 | lo: 32 bf16]; one K=16 MMA step covers 32 bytes: hi steps at +0/+32 B, lo at +64/+96 B.
          // A k-block with <= 16 valid k has the second step's chunks zeroed by the fix-up.
          const uint64_t a_hi = desc0 + ((sa + (uint32_t)g * 8192u) >> 4), a_lo = a_hi + 4;
          const uint64_t w_hi = p.wres ? wres0 + (uint32_t)kb * w_tile16 : desc0 + ((sa + A_TILE) >> 4);
          const uint64_t w_lo = w_hi + 4;
          wgmma_fence();
#pragma unroll
          for (int j = 0; j < 2; ++j) {
            const uint64_t ko = (uint64_t)(j * 2);                // 16 bf16 = 32 bytes along K, in 16-byte units
            wgmma_kk<BN>(acc, a_hi + ko, w_hi + ko);
            wgmma_kk<BN>(acc, a_lo + ko, w_hi + ko);
            wgmma_kk<BN>(acc, a_hi + ko, w_lo + ko);
          }
          wgmma_commit();
          wgmma_wait<1>();                                       // the previous stage's group has completed
          if (pend >= 0) release(pend);
          pend = s;
        } else {
          // residual block jr: D[:, 32 jr .. 32 jr + 31] += R_hi + R_lo, read from the split tile (row r: hi of column c
          // in chunk c / 8, lo in chunk 4 + c / 8, element c % 8)
          wgmma_wait<0>();
          wgmma_fence_regs(acc);
          if (pend >= 0) { release(pend); pend = -1; }
          const int jr = kb - p.k_blocks;
          const unsigned char* tile = smem + (size_t)s * p.stage_bytes;
          const int r0 = g * 64 + wq * 16 + fr;
#pragma unroll
          for (int c = 0; c < NC; ++c) {
            if (c == jr) {
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                if (32 * c + 8 * j < BN) {
#pragma unroll
                  for (int h = 0; h < 2; ++h) {
                    const int r = r0 + 8 * h;
                    const uint32_t e = (uint32_t)fc * 2;
                    const __nv_bfloat162 hi = *reinterpret_cast<const __nv_bfloat162*>(tile + swz(r, j) + e);
                    const __nv_bfloat162 lo = *reinterpret_cast<const __nv_bfloat162*>(tile + swz(r, 4 + j) + e);
                    const float2 fh = __bfloat1622float2(hi), fl = __bfloat1622float2(lo);
                    acc[16 * c + 4 * j + 2 * h] += fh.x + fl.x;
                    acc[16 * c + 4 * j + 2 * h + 1] += fh.y + fl.y;
                  }
                }
              }
            }
          }
          release(s);
        }
        if (++s == S) { s = 0; ph ^= 1u; }
      }
      if (pend >= 0) {
        wgmma_wait<0>();
        release(pend);
      }
      wgmma_fence_regs(acc);
      // ---- epilogue: fragment -> shift + activation -> staging tile -> TMA store.  A chunk is staged as a swizzled
      // 16 x 32 tile and stored through mapC, which clips at N.  A tail chunk (cw < 32 columns) with another N tile after
      // it is staged as plain 16 x cw rows and stored through mapCt instead.
      const int row0 = m0 + g * 64 + wq * 16;
      const int rows_left = min(16, p.tile_rps - row0);        // <= 0: nothing of this warp's slab is inside the sample
#pragma unroll
      for (int c = 0; c < NC; ++c) {
        const int cw = (TAIL != 0 && c == NC - 1) ? TAIL : 32;
        const bool tail = cw < 32 && n0 + BN < p.N;
        if (n0 + c * 32 < p.N) {
          unsigned char* buf = stg + (size_t)cb * STG_BYTES;
          // the store issued from this buffer (two chunks ago, or the previous one with a single buffer) has drained
          if (p.stg_bufs == 2) { cb ^= 1; if (lane == 0) tma_wait_read<1>(); }
          else if (lane == 0) tma_wait_read<0>();
          __syncwarp();
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            if (32 * c + 8 * j < BN) {
              const int cc = 8 * j + fc;
              const float* a4 = acc + 16 * c + 4 * j;
              float2 v0 = make_float2(a4[0], a4[1]), v1 = make_float2(a4[2], a4[3]);
              if (EPI != 0) {
                const float2 sh = *reinterpret_cast<const float2*>(s_shift + c * 32 + cc);
                v0.x = act_out<EPI>(v0.x + sh.x); v0.y = act_out<EPI>(v0.y + sh.y);
                v1.x = act_out<EPI>(v1.x + sh.x); v1.y = act_out<EPI>(v1.y + sh.y);
              }
              if (tail) {
                *reinterpret_cast<float2*>(buf + (fr * cw + cc) * 4) = v0;
                *reinterpret_cast<float2*>(buf + ((fr + 8) * cw + cc) * 4) = v1;
              } else {
                const uint32_t co = (uint32_t)(((cc >> 2) << 4) + (cc & 3) * 4);
                *reinterpret_cast<float2*>(buf + fr * 128 + (co ^ ((fr & 7) << 4))) = v0;
                *reinterpret_cast<float2*>(buf + (fr + 8) * 128 + (co ^ (((fr + 8) & 7) << 4))) = v1;
              }
            }
          }
          if (do_stats) {
            __syncwarp();
            // lane = column: sum the staged column over the rows of this slab that lie inside M
            float s1 = 0.f, s2 = 0.f;
            const int cj = lane >> 2, ci = lane & 3;
            if (lane < cw) {
              for (int r = 0; r < rows_left; ++r) {
                const uint32_t o = tail ? (uint32_t)(r * cw + lane) * 4 : (uint32_t)(r * 128 + ((cj ^ (r & 7)) << 4) + ci * 4);
                const float x = *reinterpret_cast<const float*>(buf + o);
                s1 += x; s2 = fmaf(x, x, s2);
              }
            }
            csum[c] += s1; csq[c] += s2;
          }
          fence_proxy_async();
          __syncwarp();
          if (lane == 0 && rows_left > 0) { tma_store_3d(tail ? &mapCt : &mapC, smem_u32(buf), n0 + c * 32, row0, bs); tma_commit(); }
        }
      }
    }
    if (do_stats && cur_nt >= 0) flush_stats(cur_nt);
    if (lane == 0) tma_wait_read<0>();                        // staging buffers must outlive their stores
    __syncwarp();
  }
  __syncthreads();
}

// ---------------------------------------------------------------------------------------------- host side
// Weights pre-split once per launch: out[n][kb][64 bf16] = 32 hi | 32 lo values of W[n][32 kb ..] (x row_scale[n]), i.e. the
// layout the in-kernel weight fix-up produces, so that the GEMM's TMA loads land finished operand tiles.  W is [N, K], or
// [K, N] when `trans` (the data gradient uses the forward weight transposed; this replaces eat_transpose_f32 there).
__global__ void w_split_kernel(const float* __restrict__ W, const float* __restrict__ row_scale, int trans,
                               uint4* __restrict__ out, int N, int K, int k_blocks) {
  const long long items = (long long)N * k_blocks * 4;             // one item = 8 consecutive k of one row
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < items; i += (long long)gridDim.x * blockDim.x) {
    const int cp = (int)(i & 3);
    const long long t = i >> 2;
    const int kb = (int)(t % k_blocks), n = (int)(t / k_blocks);
    const int k0 = kb * KB + cp * 8;
    float v[8];
    const float sc = row_scale != nullptr ? __ldg(row_scale + n) : 1.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int k = k0 + j;
      v[j] = k < K ? __ldg(trans ? W + (size_t)k * N + n : W + (size_t)n * K + k) * sc : 0.f;
    }
    uint4 hi, lo;
    split8(make_float4(v[0], v[1], v[2], v[3]), make_float4(v[4], v[5], v[6], v[7]), hi, lo);
    uint4* row = out + ((size_t)n * k_blocks + kb) * 8;              // 8 chunks of 16 bytes per (row, k-block)
    row[cp] = hi;
    row[4 + cp] = lo;
  }
}

// DynamicConv (reference models/dymn/dy_block.py:103-131): per-sample kernels W_b = sum_j att[b, j] * W_j, mixed in fp32 and
// written pre-split like above: out[b][n][kb][64 bf16].  W holds dyn_k kernels [dyn_k][N][K] ([dyn_k][K][N] when `trans`).
__global__ void w_mix_split_kernel(const float* __restrict__ W, const float* __restrict__ att, int dyn_k,
                                   const float* __restrict__ row_scale, int trans, uint4* __restrict__ out, int B, int N,
                                   int K, int k_blocks) {
  const long long per = (long long)N * k_blocks * 4;
  const long long items = per * B;
  const size_t bank = (size_t)N * K;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < items; i += (long long)gridDim.x * blockDim.x) {
    const int b = (int)(i / per);
    const long long r = i - (long long)b * per;
    const int cp = (int)(r & 3);
    const long long t = r >> 2;
    const int kb = (int)(t % k_blocks), n = (int)(t / k_blocks);
    const int k0 = kb * KB + cp * 8;
    float a[4] = {0.f, 0.f, 0.f, 0.f};
    for (int j = 0; j < dyn_k; ++j) a[j] = __ldg(att + (size_t)b * dyn_k + j);
    const float sc = row_scale != nullptr ? __ldg(row_scale + n) : 1.f;
    float v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int k = k0 + e;
      float acc = 0.f;
      if (k < K) {
        const size_t off = trans ? (size_t)k * N + n : (size_t)n * K + k;
        for (int j = 0; j < dyn_k; ++j) acc = fmaf(a[j], __ldg(W + j * bank + off), acc);
      }
      v[e] = acc * sc;
    }
    uint4 hi, lo;
    split8(make_float4(v[0], v[1], v[2], v[3]), make_float4(v[4], v[5], v[6], v[7]), hi, lo);
    uint4* row = out + (((size_t)b * N + n) * k_blocks + kb) * 8;
    row[cp] = hi;
    row[4 + cp] = lo;
  }
}

// [rows, cols] bf16 row-major tensor, box = box_rows x 64 columns (128 bytes), SWIZZLE_128B
int make_map_bf16(CUtensorMap* map, const void* ptr, long long rows, long long cols, int box_rows) {
  EncodeTiledFn enc = encode_fn();
  if (enc == nullptr) { eat_set_error("pw_tma: cuTensorMapEncodeTiled is not available from this driver"); return EAT_ERR_CUDA; }
  cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t gstride[1] = {(cuuint64_t)cols * 2};
  cuuint32_t box[2] = {64, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), gdim, gstride, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { eat_set_error("pw_tma: cuTensorMapEncodeTiled (bf16) failed"); return EAT_ERR_CUDA; }
  return EAT_OK;
}

// [samples, rows, cols] fp32 output viewed through a {cw columns, 16 rows, 1} box without swizzle (cw = 8, 16 or 24): the
// store of a tile's tail chunk, which must not write the columns of the next N tile
int make_map_tail(CUtensorMap* map, const void* ptr, long long samples, long long rows, long long cols, int cw) {
  EncodeTiledFn enc = encode_fn();
  if (enc == nullptr) { eat_set_error("pw_tma: cuTensorMapEncodeTiled is not available from this driver"); return EAT_ERR_CUDA; }
  cuuint64_t gdim[3] = {(cuuint64_t)cols, (cuuint64_t)rows, (cuuint64_t)samples};
  cuuint64_t gstride[2] = {(cuuint64_t)cols * 4, (cuuint64_t)(rows * cols * 4)};
  cuuint32_t box[3] = {(cuuint32_t)cw, 16, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<void*>(ptr), gdim, gstride, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { eat_set_error("pw_tma: cuTensorMapEncodeTiled (tail store) failed"); return EAT_ERR_CUDA; }
  return EAT_OK;
}

constexpr size_t kSmemLimit = 227 * 1024;

struct Maps { CUtensorMap A, W, C, Ct, R; };

template <int EPI, int XACT, int BN>
int launch_kernel(const Maps& m, const TmaParams& p, size_t smem, int tiles, cudaStream_t st) {
  static unsigned long long attr_mask = 0;
  if (int rc = eat_opt_in_smem(pw_tma_kernel<EPI, XACT, BN>, kSmemLimit, attr_mask)) return rc;
  int dev = 0, sms = kNumSMs;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  // persistent grid, a multiple of n_tiles (the kernel's tile walk); tiles is one as well
  const int grid = min(tiles, max(p.n_tiles, sms / p.n_tiles * p.n_tiles));
  pw_tma_kernel<EPI, XACT, BN><<<grid, kThreads, smem, st>>>(m.A, m.W, m.C, m.Ct, m.R, p);
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

// Tile widths with a compiled kernel.  The raw-output variant (training forward with batch statistics, every data
// gradient) has one at every multiple of 8; the epilogue variants (inference) keep 32 / 64 / 128.
template <int EPI>
using Widths = std::conditional_t<EPI == 0,
                                  std::integer_sequence<int, 8, 16, 24, 32, 40, 48, 56, 64, 72, 80, 88, 96, 104, 112, 120, 128>,
                                  std::integer_sequence<int, 32, 64, 128>>;

// narrowest compiled width >= bn
template <int... W>
constexpr int fit_width(std::integer_sequence<int, W...>, int bn) {
  int best = BN_MAX;
  for (int w : {W...}) if (w >= bn && w < best) best = w;
  return best;
}

template <int EPI, int XACT, int... W>
int launch_width(std::integer_sequence<int, W...>, const Maps& m, const TmaParams& p, size_t smem, int tiles, cudaStream_t st) {
  int rc = EAT_ERR_UNSUPPORTED;
  const bool found = ((p.BN == W && (rc = launch_kernel<EPI, XACT, W>(m, p, smem, tiles, st), true)) || ...);
  if (!found) eat_set_error("pw_tma: no kernel for this tile width");
  return rc;
}

struct WeightWs { int trans; void* ws; size_t bytes; const float* att; int dyn_k; };   // att != nullptr: DynamicConv kernel mix

template <int EPI, int XACT>
int launch_tma(const void* A, const float* W, void* C, const void* R, TmaParams p, cudaStream_t st, WeightWs ws) {
  // ---- tiling.  Every N tile lands and fixes up the A tile again (TMA write 16 KB + fix-up 32 KB per k-block), so N is
  // cut into as few tiles as the consumer registers allow (a 64 x 128 fp32 accumulator per warpgroup = 64 registers per
  // thread), of equal width rounded up to 8 columns: tensor-core work is padded by at most 7 columns per tile.  A width
  // without a compiled kernel runs on the next wider one (the TMA unit zero-fills the weight rows past N).
  p.n_tiles = ceil_div(p.N, BN_MAX);
  p.BN = fit_width(Widths<EPI>{}, (ceil_div(p.N, p.n_tiles) + 7) & ~7);
  p.n_tiles = ceil_div(p.N, p.BN);
  p.bnp = BN_MAX;
  if (p.n_samples < 1) { p.n_samples = 1; p.tile_rps = p.M; }
  p.tps = ceil_div(p.tile_rps, BM);
  p.m_tiles = p.n_samples * p.tps;
  p.k_blocks = ceil_div(p.K, KB);
  p.r_blocks = R != nullptr ? ceil_div(min(p.BN, p.N), 32) : 0;
  p.kpad = XACT >= 0 ? p.k_blocks * KB : 0;
  // ---- shared-memory carve-up: [stages][resident W][staging][floats][barriers]; one CTA per SM (the
  // accumulators of two warpgroups and the fix-up / TMA warps use the register file).  Weights stay resident when that
  // still leaves four stages.
  const size_t w_tile = (size_t)p.BN * 128;
  const size_t w_res = (size_t)p.k_blocks * w_tile;
  const size_t floats = (2 * (size_t)p.kpad + 17 * (size_t)p.bnp) * 4;
  const size_t barsz = (3 * 8 + 1) * 8 + 16;
  p.stg_bufs = 2;
  const size_t fixed = (size_t)p.stg_bufs * 8 * STG_BYTES + floats + barsz + 1024 /*alignment slack*/;
  p.wres = (fixed + w_res + 4 * (size_t)A_TILE <= kSmemLimit) ? 1 : 0;
  p.stage_bytes = (uint32_t)(A_TILE + (p.wres ? 0 : w_tile));
  const size_t avail = kSmemLimit - fixed - (p.wres ? w_res : 0);
  p.stages = (int)(avail / p.stage_bytes);
  if (p.stages > 8) p.stages = 8;
  if (p.stages < 2) { eat_set_error("pw_tma: shared-memory budget exceeded (K too large for the in-transform tables)"); return EAT_ERR_UNSUPPORTED; }
  size_t off = (size_t)p.stages * p.stage_bytes;
  p.off_w = (uint32_t)off; off += p.wres ? w_res : 0;
  p.off_stg = (uint32_t)off; off += (size_t)p.stg_bufs * 8 * STG_BYTES;
  p.off_f = (uint32_t)off; off += floats;
  off = (off + 7) & ~(size_t)7;
  p.off_bar = (uint32_t)off; off += (3 * (size_t)p.stages + 1) * 8 + 16;
  const size_t smem = off;
  if (smem > kSmemLimit) { eat_set_error("pw_tma: shared-memory carve-up exceeds its budget"); return EAT_ERR_UNSUPPORTED; }
  // ---- tensor maps
  Maps m;
  CUtensorMap &mA = m.A, &mW = m.W, &mC = m.C, &mR = m.R;
  const long long ns = p.n_samples, rps = p.tile_rps;
  if (int rc = make_map3(&mA, A, ns, rps, p.K, BM, 4)) return rc;
  p.wpre = 0;
  p.wdyn = 0;
  if (ws.ws != nullptr) {
    // pre-split the weights (scale folded, optionally transposed, per sample for DynamicConv) into the caller's workspace
    // and read THAT through TMA
    const long long wsamples = ws.att != nullptr ? ns : 1;
    const size_t need = (size_t)wsamples * p.N * p.k_blocks * 128;
    if (ws.bytes < need || (((uintptr_t)ws.ws) & 127)) { eat_set_error("pw_tma: weight workspace too small or not 128-byte aligned"); return EAT_ERR_ARG; }
    const long long items = wsamples * p.N * p.k_blocks * 4;
    const int grid = (int)min((long long)kNumSMs * 8, ceil_div_ll(items, 256));
    const float* fold = (EPI != 0) ? p.scale : nullptr;
    if (ws.att != nullptr) {
      w_mix_split_kernel<<<grid, 256, 0, st>>>(W, ws.att, ws.dyn_k, fold, ws.trans, reinterpret_cast<uint4*>(ws.ws), (int)ns, p.N, p.K, p.k_blocks);
      p.wdyn = 1;
    } else {
      w_split_kernel<<<grid, 256, 0, st>>>(W, fold, ws.trans, reinterpret_cast<uint4*>(ws.ws), p.N, p.K, p.k_blocks);
    }
    EAT_CHECK_LAUNCH();
    p.wpre = 1;
    if (int rc = make_map3(&mW, ws.ws, wsamples, p.N, (long long)p.k_blocks * 64, p.BN, 2)) return rc;
  } else {
    if (ws.trans || ws.att != nullptr) { eat_set_error("pw_tma: transposed / per-sample weights need the weight workspace"); return EAT_ERR_ARG; }
    if (int rc = make_map3(&mW, W, 1, p.N, p.K, p.BN, 4)) return rc;
  }
  if (int rc = make_map3(&mC, C, ns, rps, p.N, 16, 4)) return rc;
  if (p.n_tiles > 1 && p.BN % 32 != 0) {
    if (int rc = make_map_tail(&m.Ct, C, ns, rps, p.N, p.BN % 32)) return rc;
  } else {
    m.Ct = mC;                                               // unused: every chunk is a full one
  }
  if (int rc = make_map3(&mR, R != nullptr ? R : C, ns, rps, p.N, BM, 4)) return rc;
  return launch_width<EPI, XACT>(Widths<EPI>{}, m, p, smem, p.m_tiles * p.n_tiles, st);
}

template <int EPI>
int launch_tma_x(const void* A, const float* W, void* C, const void* R, const TmaParams& p, cudaStream_t st, WeightWs ws) {
  if (p.in_scale == nullptr) return launch_tma<EPI, -1>(A, W, C, R, p, st, ws);
  if (p.in_act == EAT_ACT_RELU) return launch_tma<EPI, 1>(A, W, C, R, p, st, ws);
  if (p.in_act == EAT_ACT_HSWISH) return launch_tma<EPI, 2>(A, W, C, R, p, st, ws);
  return launch_tma<EPI, 0>(A, W, C, R, p, st, ws);
}

}  // namespace

extern "C" int eat_pw_tma_fwd(const float* A, const float* W, int w_trans, float* C, long long M, int N, int K,
                              const float* in_scale, const float* in_shift, int in_act, const float* gate,
                              int rows_per_sample, const float* scale, const float* shift, int act, const float* residual,
                              double* stat_sum, double* stat_sq, void* w_ws, long long w_ws_bytes, cudaStream_t st) {
  if (M == 0) return EAT_OK;
  if (act == EAT_ACT_SIGMOID || in_act == EAT_ACT_SIGMOID) { eat_set_error("pw_tma: sigmoid epilogues run on the CUDA-core GEMM (eat_gemm_simt_fwd)"); return EAT_ERR_UNSUPPORTED; }
  const bool aff = scale != nullptr || shift != nullptr || act != 0;
  if (residual != nullptr && act != EAT_ACT_NONE) { eat_set_error("pw_tma: the residual is accumulated before the activation; residual + activation is not offered"); return EAT_ERR_UNSUPPORTED; }
  if (stat_sum != nullptr && (aff || residual != nullptr)) {
    eat_set_error("pw_tma: batch statistics are produced by the raw-output variant only (no affine/activation/residual)");
    return EAT_ERR_UNSUPPORTED;
  }
  if ((in_scale == nullptr) != (in_shift == nullptr)) { eat_set_error("pw_tma: in_scale and in_shift come together"); return EAT_ERR_ARG; }
  if (K % 4 != 0 || N % 4 != 0) { eat_set_error("pw_tma: K and N must be multiples of 4 (16-byte row pitch for TMA)"); return EAT_ERR_ARG; }
  if (M >= (1ll << 31) - BM) { eat_set_error("pw_tma: M too large"); return EAT_ERR_ARG; }
  if ((((uintptr_t)A) | ((uintptr_t)W) | ((uintptr_t)C) | ((uintptr_t)residual) | ((uintptr_t)gate)) & 15) { eat_set_error("pw_tma: operands must be 16-byte aligned"); return EAT_ERR_ARG; }
  TmaParams p{};
  p.M = (int)M; p.N = N; p.K = K;
  p.in_scale = in_scale; p.in_shift = in_shift; p.gate = gate; p.in_act = in_act; p.rps = rows_per_sample > 0 ? rows_per_sample : 1;
  p.scale = scale; p.shift = shift; p.stat_sum = stat_sum; p.stat_sq = stat_sq;
  const WeightWs ws{w_trans, w_ws, (size_t)(w_ws_bytes > 0 ? w_ws_bytes : 0), nullptr, 0};
  if (!aff) return launch_tma_x<0>(A, W, C, residual, p, st, ws);
  if (act == EAT_ACT_RELU) return launch_tma_x<2>(A, W, C, residual, p, st, ws);
  if (act == EAT_ACT_HSWISH) return launch_tma_x<3>(A, W, C, residual, p, st, ws);
  return launch_tma_x<1>(A, W, C, residual, p, st, ws);
}

// DynamicConv 1x1 (reference models/dymn/dy_block.py:103-131) on the TMA kernel: W holds dyn_k kernels [dyn_k][N][K]
// ([dyn_k][K][N] with w_trans = 1, the data gradient); sample b uses sum_j att[b, j] * W[j], mixed and pre-split once per
// launch into w_ws (B * N * ceil(K/32) * 128 bytes).  M = B * rows_per_sample; tiles, loads and stores never cross a
// sample (3-D tensor maps).
extern "C" int eat_pw_tma_dyn_fwd(const float* A, const float* W, const float* att, int dyn_k, int w_trans, float* C,
                                  long long M, int N, int K, int rows_per_sample, const float* scale, const float* shift,
                                  int act, const float* residual, double* stat_sum, double* stat_sq, void* w_ws,
                                  long long w_ws_bytes, cudaStream_t st) {
  if (M == 0) return EAT_OK;
  if (dyn_k < 1 || dyn_k > 4) { eat_set_error("pw_tma_dyn: 1..4 kernels supported"); return EAT_ERR_UNSUPPORTED; }
  if (rows_per_sample < 1 || M % rows_per_sample != 0) { eat_set_error("pw_tma_dyn: M must be B * rows_per_sample"); return EAT_ERR_ARG; }
  if (act == EAT_ACT_SIGMOID) { eat_set_error("pw_tma_dyn: sigmoid epilogue is not offered"); return EAT_ERR_UNSUPPORTED; }
  const bool aff = scale != nullptr || shift != nullptr || act != 0;
  if (residual != nullptr && act != EAT_ACT_NONE) { eat_set_error("pw_tma_dyn: residual + activation is not offered"); return EAT_ERR_UNSUPPORTED; }
  if (stat_sum != nullptr && (aff || residual != nullptr)) { eat_set_error("pw_tma_dyn: statistics come from the raw-output variant only"); return EAT_ERR_UNSUPPORTED; }
  if (K % 4 != 0 || N % 4 != 0) { eat_set_error("pw_tma_dyn: K and N must be multiples of 4"); return EAT_ERR_ARG; }
  if (M >= (1ll << 31) - BM) { eat_set_error("pw_tma_dyn: M too large"); return EAT_ERR_ARG; }
  if (w_ws == nullptr || att == nullptr) { eat_set_error("pw_tma_dyn: attention weights and the weight workspace are required"); return EAT_ERR_ARG; }
  if ((((uintptr_t)A) | ((uintptr_t)W) | ((uintptr_t)C) | ((uintptr_t)residual)) & 15) { eat_set_error("pw_tma_dyn: operands must be 16-byte aligned"); return EAT_ERR_ARG; }
  TmaParams p{};
  p.M = (int)M; p.N = N; p.K = K;
  p.rps = 1;
  p.scale = scale; p.shift = shift; p.stat_sum = stat_sum; p.stat_sq = stat_sq;
  p.n_samples = (int)(M / rows_per_sample); p.tile_rps = rows_per_sample;
  const WeightWs ws{w_trans, w_ws, (size_t)(w_ws_bytes > 0 ? w_ws_bytes : 0), att, dyn_k};
  if (!aff) return launch_tma_x<0>(A, W, C, residual, p, st, ws);
  if (act == EAT_ACT_RELU) return launch_tma_x<2>(A, W, C, residual, p, st, ws);
  if (act == EAT_ACT_HSWISH) return launch_tma_x<3>(A, W, C, residual, p, st, ws);
  return launch_tma_x<1>(A, W, C, residual, p, st, ws);
}
