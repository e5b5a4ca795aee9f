// Backward of an InvertedResidual's expand stage (1x1 conv + BatchNorm + activation, reference
// models/mn/block_types.py:140-147, reached from ex_audioset.py:197 loss.backward()) in ONE pass over its tensors:
//
//     dz        = scale * (da * act'(z*scale+shift)) + alpha * z + beta        (the folded constants of eat_bn_bwd_apply)
//     dX[M,cin] = dz . W (+ res)                                                W: expand weight [cexp, cin]
//     dW[cexp,cin] += dz^T . X
//
// dz is computed on chip and never stored.  The three-pass route (apply, weight-gradient GEMM, data-gradient GEMM) reads
// and writes the expanded tensor five times; this kernel reads da and z once each.  Built from the pieces of pw_tma.cu
// (data gradient) and wgrad_tma.cu (weight gradient):
//
//   warp 12  TMA producer : one thread.  Per 128-row tile: the X box (cin <= 32 channels) and, with a residual, the
//                           residual box into one of two tile slots; then the cexp dimension one 32-channel k-block at
//                           a time, as a da box plus a z box, into a ring of stages.
//   warps 0-3 fix-up      : the X box gets the plain in-place hi/lo split of tma_common.cuh; each k-block's dz is
//                           computed from (da, z) and split hi/lo in place into the da box (the z box is then dead).
//   warps 4-11 consumers  : two warpgroups.  The split dz box is BOTH the K-major A operand of the data gradient (each
//                           warpgroup takes one 64-row half, bf16x3 products hi.hi + lo.hi + hi.lo exactly as pw_tma)
//                           AND the MN-major operand of the weight gradient (k-block kb belongs to warpgroup kb % 2,
//                           which reduces all 128 rows of the tile against the split X box; accumulator rows
//                           [hi(n) | lo(n)], columns [hi(k) | lo(k)] as wgrad_tma).  The weight-gradient accumulators
//                           stay in registers for the CTA's whole row range and are flushed once with vector atomics
//                           (hi.hi + hi.lo on hi rows, lo.hi on lo rows, lo.lo ~ 2^-32 dropped).  The data gradient goes
//                           out per tile through the pw_tma epilogue (staging tile + TMA store), the residual added in
//                           fp32 straight from its landed box.
// The register budget decides the coverage: 13 warps cap a thread at 128 registers; a consumer holds 16 data-gradient
// and up to 2 x 32 weight-gradient accumulators, so cin <= 32 (one X box) and cexp <= 128 (four k-blocks).  The expand
// weight (at most 128 x 32) is split into its resident hi/lo tiles by every CTA in the prologue, from L2.
// HBM-bound: algorithmic bytes per launch = 4 * (2 M cexp + M cin (X) + M cin (dX) (+ M cin residual) + 2 cexp cin).
#include <cstdarg>
#include <cstdio>

#include "tma_common.cuh"

namespace {
using namespace tc;
using namespace tma;

constexpr int BM = 128;
constexpr int BOX = BM * 128;           // one landed [128 rows x 32 fp32] box, 16 KB
constexpr int kThreads = 416;           // 4 fix-up warps, 8 consumer warps (2 warpgroups), TMA warp
constexpr int kFirstCons = 4, kTmaWarp = 12;
constexpr int STG_BYTES = 16 * 128;     // one staged 16 x 32 fp32 sub-tile
constexpr int kMaxKb = 4;               // k-blocks of cexp: 2 per warpgroup x 32 weight-gradient registers each
constexpr int kMaxStages = 6;
constexpr size_t kSmemLimit = 227 * 1024;

struct PbParams {
  const float *scale, *shift, *mean, *invstd, *c1, *c2, *W;
  float* dW;
  int M, cexp, cin, m_tiles, stages, res;
  uint32_t off_x, off_w, off_stg, off_f, off_bar;
};

struct PbPlan { int splits, rows_per_split, stages, smem, nkb; uint32_t off_x, off_w, off_stg, off_s, off_f, off_bar; };

void plan_error(const char* fmt, ...) {
  char buf[256];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  eat_set_error(buf);
}

// Both kernels of this file (expand: cn = cin; project, PROJ: cn = cout) share one layout:
// shared memory: [stages][2 boxes of the streamed k-block] [2 tile slots][2 boxes of the tile] [k-blocks][32 weight rows
//                x 128 B] [8 consumer warps][2][staging] (PROJ: [8 consumer warps][2][k-blocks * 32] fp64 sums)
//                [per-channel tables]
//                [barriers].  The tables are 4 x (k-blocks * 32) floats, PROJ 4 x 32 (BN3) + 3 x (k-blocks * 32) (BN2).
int plan_pb(long long M, int cexp, int cn, int sms, bool proj, PbPlan& pl) {
  const char* name = proj ? "pw_proj_bwd_fused" : "pw_conv_bwd_fused";
  const char* cname = proj ? "cout" : "cin";
  if (M < 1 || cexp < 1 || cn < 1) { plan_error("%s: M, cexp and %s must be positive", name, cname); return EAT_ERR_ARG; }
  if (cexp % 4 != 0 || cn % 4 != 0) {
    plan_error("%s: cexp and %s must be multiples of 4 (16-byte row pitch for TMA)", name, cname);
    return EAT_ERR_ARG;
  }
  if (M >= (1ll << 31) - BM) { plan_error("%s: M too large", name); return EAT_ERR_ARG; }
  if (cn > KB || cexp > kMaxKb * KB) {
    plan_error("%s: %s <= 32 and cexp <= 128 only (register-resident weight gradient)", name, cname);
    return EAT_ERR_UNSUPPORTED;
  }
  pl.nkb = (cexp + KB - 1) / KB;
  const int m_tiles = (int)((M + BM - 1) / BM);
  pl.splits = m_tiles < sms ? m_tiles : sms;
  pl.rows_per_split = ((m_tiles + pl.splits - 1) / pl.splits) * BM;
  const size_t kp = (size_t)pl.nkb * KB;
  const size_t x_bytes = 2 * 2 * (size_t)BOX, w_bytes = kp * 128, stg = 8 * 2 * (size_t)STG_BYTES;
  const size_t sums = proj ? 8 * 2 * kp * 8 : 0, floats = (proj ? 4 * KB + 3 * kp : 4 * kp) * 4;
  const size_t bars = (3 * (size_t)kMaxStages + 6) * 8;
  const size_t fixed = x_bytes + w_bytes + stg + sums + floats + bars + 1024 /*alignment slack*/;
  pl.stages = (int)((kSmemLimit - fixed) / (2 * BOX));
  if (pl.stages > kMaxStages) pl.stages = kMaxStages;
  if (pl.stages < 2) { plan_error("%s: shared-memory budget exceeded", name); return EAT_ERR_UNSUPPORTED; }
  size_t off = (size_t)pl.stages * 2 * BOX;
  pl.off_x = (uint32_t)off; off += x_bytes;
  pl.off_w = (uint32_t)off; off += w_bytes;
  pl.off_stg = (uint32_t)off; off += stg;
  pl.off_s = (uint32_t)off; off += sums;
  pl.off_f = (uint32_t)off; off += floats;
  pl.off_bar = (uint32_t)off; off += (3 * (size_t)pl.stages + 6) * 8;
  pl.smem = (int)off;
  return EAT_OK;
}

// the barriers of the pipeline, from bar_full on: per stage full (TMA), ready (4 fix-up warps), empty (2 consumer
// warpgroups); then the same three per tile slot
__device__ __forceinline__ void init_bars(uint32_t bar_full, int S) {
  const uint32_t bar_ready = bar_full + 8 * S, bar_empty = bar_ready + 8 * S;
  const uint32_t bar_tfull = bar_empty + 8 * S, bar_tready = bar_tfull + 16, bar_tempty = bar_tready + 16;
  for (int s = 0; s < S; ++s) { mbar_init(bar_full + 8 * s, 1); mbar_init(bar_ready + 8 * s, 4); mbar_init(bar_empty + 8 * s, 2); }
  for (int s = 0; s < 2; ++s) { mbar_init(bar_tfull + 8 * s, 1); mbar_init(bar_tready + 8 * s, 4); mbar_init(bar_tempty + 8 * s, 2); }
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}

// the CTA's contiguous range of 128-row tiles
__device__ __forceinline__ void tile_range(int m_tiles, int& t_begin, int& t_end) {
  t_begin = (int)((long long)blockIdx.x * m_tiles / gridDim.x);
  t_end = (int)((long long)(blockIdx.x + 1) * m_tiles / gridDim.x);
}

// dz of one k-block from the landed (da, z) boxes, split hi/lo in place into the da box; rows >= rows_valid become zero
// (beta != 0 would otherwise leak into the weight gradient).  Thread layout of fix_a<2>: chunk pair cp of rows r0 + 32 i.
template <int ACT>
__device__ __forceinline__ void fix_dz(unsigned char* dat, const unsigned char* zt, int ft, int rows_valid, const float* s_sc,
                                       const float* s_sh, const float* s_al, const float* s_be, int k) {
  const int cp = ft & 3, r0 = ft >> 2;
  const uint32_t row_off = (uint32_t)((r0 >> 3) * 1024 + (r0 & 7) * 128);
  const int x = r0 & 7;
  const uint32_t in0 = row_off + (((2 * cp) ^ x) << 4), in1 = row_off + (((2 * cp + 1) ^ x) << 4);
  const uint32_t out_hi = row_off + ((cp ^ x) << 4), out_lo = row_off + (((4 + cp) ^ x) << 4);
  float sc[8], sh[8], al[8], be[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) { sc[j] = s_sc[k + j]; sh[j] = s_sh[k + j]; al[j] = s_al[k + j]; be[j] = s_be[k + j]; }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const uint32_t o = (uint32_t)i * 32 * 128;
    const float4 ga = *reinterpret_cast<const float4*>(dat + in0 + o), gb = *reinterpret_cast<const float4*>(dat + in1 + o);
    const float4 za = *reinterpret_cast<const float4*>(zt + in0 + o), zb = *reinterpret_cast<const float4*>(zt + in1 + o);
    const float g[8] = {ga.x, ga.y, ga.z, ga.w, gb.x, gb.y, gb.z, gb.w};
    const float zv[8] = {za.x, za.y, za.z, za.w, zb.x, zb.y, zb.z, zb.w};
    float d[8];
    const bool live = r0 + 32 * i < rows_valid;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float gg = g[j] * act_bwd(fmaf(zv[j], sc[j], sh[j]), ACT);
      d[j] = live ? fmaf(sc[j], gg, fmaf(al[j], zv[j], be[j])) : 0.f;
    }
    __syncwarp();                                   // every lane of the row has its inputs before anyone overwrites them
    uint4 h, l;
    split8(make_float4(d[0], d[1], d[2], d[3]), make_float4(d[4], d[5], d[6], d[7]), h, l);
    *reinterpret_cast<uint4*>(dat + out_hi + o) = h;
    *reinterpret_cast<uint4*>(dat + out_lo + o) = l;
  }
}

// the weight-gradient accumulators of one consumer thread, once per CTA.  Warpgroup g holds k-blocks g, g + 2 of the
// streamed dimension (n < N); accumulator rows r = 16 wq + lane / 4 (+ 8) of [hi(n) 0..31 | lo(n) 0..31], columns
// [hi(k) 0..31 | lo(k) 0..31] of the tile's channels (k < K).  hi.hi + hi.lo go out on hi rows, lo.hi on lo rows (lo.lo
// ~ 2^-32 is dropped), into dW [N, K] with vector atomics or, TRANS, into dW [K, N].
template <int NKB, bool TRANS>
__device__ __forceinline__ void flush_wgrad(float (&accW)[(NKB + 1) / 2][32], int g, int wq, int lane, float* dW, int N,
                                            int K) {
  const bool hi_row = wq < 2;
#pragma unroll
  for (int w = 0; w < (NKB + 1) / 2; ++w) {
    const int kb = 2 * w + g;
    if (kb >= NKB) continue;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int n = kb * KB + (wq & 1) * 16 + (lane >> 2) + 8 * h;
      if (n >= N) continue;
#pragma unroll
      for (int j = 0; j < 4; ++j) {                      // hi(k) columns 8 j + 2 (lane % 4)
        const int k = 8 * j + 2 * (lane & 3);
        float2 v = make_float2(accW[w][4 * j + 2 * h], accW[w][4 * j + 2 * h + 1]);
        if (hi_row) { v.x += accW[w][4 * (j + 4) + 2 * h]; v.y += accW[w][4 * (j + 4) + 2 * h + 1]; }   // + hi.lo
        if (k >= K) continue;
        if (TRANS) {
          atomicAdd(dW + (size_t)k * N + n, v.x);
          atomicAdd(dW + (size_t)(k + 1) * N + n, v.y);   // K is a multiple of 4: k + 1 < K
        } else {
          atomicAdd(reinterpret_cast<float2*>(dW + (size_t)n * K + k), v);
        }
      }
    }
  }
}

template <int NKB, int ACT>
__global__ void __launch_bounds__(kThreads, 1)   // 13 warps: 4 on one scheduler, so at most 128 registers per thread
pw_bwd_fused_kernel(const __grid_constant__ CUtensorMap mapDA, const __grid_constant__ CUtensorMap mapZ,
                    const __grid_constant__ CUtensorMap mapX, const __grid_constant__ CUtensorMap mapR,
                    const __grid_constant__ CUtensorMap mapC, const PbParams p) {
  constexpr int KP = NKB * KB;                           // padded channel count of the per-channel tables
  constexpr int NWA = (NKB + 1) / 2;                     // weight-gradient accumulators per warpgroup
  extern __shared__ __align__(1024) unsigned char smem[];
  unsigned char* s_x = smem + p.off_x;                   // [2 slots][X | residual]
  unsigned char* s_w = smem + p.off_w;                   // [NKB][32 rows x (32 hi | 32 lo) bf16]
  unsigned char* s_stg = smem + p.off_stg;
  float* s_sc = reinterpret_cast<float*>(smem + p.off_f);
  float* s_sh = s_sc + KP;
  float* s_al = s_sh + KP;
  float* s_be = s_al + KP;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + p.off_bar);
  const int S = p.stages;
  const uint32_t bar_full = smem_u32(bars), bar_ready = bar_full + 8 * S, bar_empty = bar_ready + 8 * S;
  const uint32_t bar_tfull = bar_empty + 8 * S, bar_tready = bar_tfull + 16, bar_tempty = bar_tready + 16;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int t_begin, t_end;
  tile_range(p.m_tiles, t_begin, t_end);
  if (threadIdx.x == 0) {
    init_bars(bar_full, S);
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&mapDA)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&mapZ)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&mapX)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&mapC)) : "memory");
  }
  // per-channel constants of the BatchNorm-backward apply (as bn_bwd_apply2_kernel), zero beyond cexp: dz = 0 there
  for (int c = threadIdx.x; c < KP; c += kThreads) {
    float sc = 0.f, sh = 0.f, al = 0.f, be = 0.f;
    if (c < p.cexp) {
      sc = p.scale[c]; sh = p.shift[c];
      al = -sc * p.c2[c] * p.invstd[c];
      be = -sc * p.c1[c] - al * p.mean[c];
    }
    s_sc[c] = sc; s_sh[c] = sh; s_al[c] = al; s_be[c] = be;
  }
  // the data gradient's B operand: W^T as K-major rows, row n (input channel) of k-block kb = 32 hi | 32 lo bf16 values of
  // W[32 kb .., n] -- the tiles eat_pw_tma_fwd's weight pre-split (w_trans = 1) produces
  for (int i = threadIdx.x; i < NKB * KB * 4; i += kThreads) {
    const int cp = i & 3, n = (i >> 2) & (KB - 1), kb = i >> 7;
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int k = kb * KB + cp * 8 + j;
      v[j] = (n < p.cin && k < p.cexp) ? __ldg(p.W + (size_t)k * p.cin + n) : 0.f;
    }
    uint4 hi, lo;
    split8(make_float4(v[0], v[1], v[2], v[3]), make_float4(v[4], v[5], v[6], v[7]), hi, lo);
    unsigned char* wt = s_w + (size_t)kb * KB * 128;
    *reinterpret_cast<uint4*>(wt + swz(n, cp)) = hi;
    *reinterpret_cast<uint4*>(wt + swz(n, 4 + cp)) = lo;
  }
  fence_proxy_async();
  __syncthreads();
  const uint32_t stage_base = smem_u32(smem), x_base = smem_u32(s_x);

  if (warp == kTmaWarp) {
    // ================================================================= TMA producer (one thread)
    if (lane == 0) {
      int s = 0;
      uint32_t ph = 0;
      for (int t = t_begin, i = 0; t < t_end; ++t, ++i) {
        const int slot = i & 1;
        const uint32_t tph = (uint32_t)(i >> 1) & 1u;
        const int m0 = t * BM;
        mbar_wait(bar_tempty + 8 * slot, tph ^ 1u);
        const uint32_t xd = x_base + (uint32_t)slot * 2 * BOX;
        mbar_expect_tx(bar_tfull + 8 * slot, (uint32_t)(p.res ? 2 : 1) * BOX);
        tma_load_2d(&mapX, bar_tfull + 8 * slot, xd, 0, m0);
        if (p.res) tma_load_2d(&mapR, bar_tfull + 8 * slot, xd + BOX, 0, m0);
        for (int kb = 0; kb < NKB; ++kb) {
          mbar_wait(bar_empty + 8 * s, ph ^ 1u);
          const uint32_t dst = stage_base + (uint32_t)s * 2 * BOX;
          mbar_expect_tx(bar_full + 8 * s, 2 * BOX);
          tma_load_2d(&mapDA, bar_full + 8 * s, dst, kb * KB, m0);
          tma_load_2d(&mapZ, bar_full + 8 * s, dst + BOX, kb * KB, m0);
          if (++s == S) { s = 0; ph ^= 1u; }
        }
      }
    }
    __syncwarp();
  } else if (warp < kFirstCons) {
    // ================================================================= fix-up warps (128 threads)
    const int ft = threadIdx.x;
    int s = 0;
    uint32_t ph = 0;
    for (int t = t_begin, i = 0; t < t_end; ++t, ++i) {
      const int slot = i & 1;
      const uint32_t tph = (uint32_t)(i >> 1) & 1u;
      const int rows_valid = min(BM, p.M - t * BM);
      mbar_wait(bar_tfull + 8 * slot, tph);
      fix_a<2, -1>(s_x + (size_t)slot * 2 * BOX, ft, rows_valid, nullptr, nullptr, 0, nullptr, 0, 0, 1, 0);
      fence_proxy_async();
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_tready + 8 * slot);
      for (int kb = 0; kb < NKB; ++kb) {
        mbar_wait(bar_full + 8 * s, ph);
        unsigned char* st = smem + (size_t)s * 2 * BOX;
        fix_dz<ACT>(st, st + BOX, ft, rows_valid, s_sc, s_sh, s_al, s_be, kb * KB + (ft & 3) * 8);
        fence_proxy_async();
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_ready + 8 * s);
        if (++s == S) { s = 0; ph ^= 1u; }
      }
    }
  } else {
    // ================================================================= consumers: MMAs, data-gradient epilogue, weight-gradient flush
    const int cw = warp - kFirstCons;
    const int g = cw >> 2, wq = cw & 3;                  // warpgroup (64-row half of the data gradient), warp inside it
    const int ctid = threadIdx.x - kFirstCons * 32;
    unsigned char* stg = s_stg + (size_t)cw * 2 * STG_BYTES;
    const uint64_t desc0 = gmma_desc(0);
    const uint64_t w0 = desc0 + (smem_u32(s_w) >> 4);
    const int fr = lane >> 2, fc = 2 * (lane & 3);       // fragment row / column of this lane
    float accW[NWA][32];
#pragma unroll
    for (int w = 0; w < NWA; ++w)
#pragma unroll
      for (int e = 0; e < 32; ++e) accW[w][e] = 0.f;
    int s = 0, cb = 0;
    uint32_t ph = 0;
    for (int t = t_begin, i = 0; t < t_end; ++t, ++i) {
      const int slot = i & 1;
      const uint32_t tph = (uint32_t)(i >> 1) & 1u;
      mbar_wait(bar_tready + 8 * slot, tph);
      if (p.res) mbar_wait(bar_tfull + 8 * slot, tph);
      const uint32_t sx = x_base + (uint32_t)slot * 2 * BOX;
      float acc[16];
#pragma unroll
      for (int e = 0; e < 16; ++e) acc[e] = 0.f;
#pragma unroll
      for (int kb = 0; kb < NKB; ++kb) {
        mbar_wait(bar_ready + 8 * s, ph);
        const uint32_t sa = stage_base + (uint32_t)s * 2 * BOX;
        // data gradient: row = [hi: 32 bf16 | lo: 32 bf16]; K=16 steps at +0/+32 B (hi) and +64/+96 B (lo)
        const uint64_t a_hi = desc0 + ((sa + (uint32_t)g * 8192u) >> 4), a_lo = a_hi + 4;
        const uint64_t w_hi = w0 + (uint64_t)(kb * KB * 128 / 16), w_lo = w_hi + 4;
        wgmma_fence();
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const uint64_t ko = (uint64_t)(j * 2);
          wgmma_n32<0, 0>(acc, a_hi + ko, w_hi + ko);
          wgmma_n32<0, 0>(acc, a_lo + ko, w_hi + ko);
          wgmma_n32<0, 0>(acc, a_hi + ko, w_lo + ko);
        }
        // weight gradient of this k-block's 32 channels: 16 reduction rows (two 8-row groups, 2048 B) per instruction
        if ((kb & 1) == g) {
#pragma unroll
          for (int st = 0; st < BM / 16; ++st)
            wgmma_n64<1, 1>(accW[kb >> 1], gmma_desc(sa + st * 2048, BOX, 1024), gmma_desc(sx + st * 2048, BOX, 1024));
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(acc);
#pragma unroll
        for (int w = 0; w < NWA; ++w) wgmma_fence_regs(accW[w]);
        asm volatile("bar.sync %0, 128;" ::"r"(1 + g) : "memory");   // every warp of the group is past its wait
        if (ctid == g * 128) mbar_arrive(bar_empty + 8 * s);
        if (++s == S) { s = 0; ph ^= 1u; }
      }
      // ---- epilogue: fragment (+ residual) -> swizzled 16 x 32 staging tile -> TMA store (rows past M clipped)
      const int rl = g * 64 + wq * 16;                   // first row of this warp's slab inside the tile
      const int row0 = t * BM + rl;
      unsigned char* buf = stg + (size_t)cb * STG_BYTES;
      cb ^= 1;
      if (lane == 0) tma_wait_read<1>();                 // the store issued from this buffer two tiles ago has drained
      __syncwarp();
      const unsigned char* rt = s_x + (size_t)slot * 2 * BOX + BOX;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int cc = 8 * j + fc;
        float2 v0 = make_float2(acc[4 * j], acc[4 * j + 1]), v1 = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
        if (p.res) {
          const float2 r0 = *reinterpret_cast<const float2*>(rt + swz(rl + fr, cc >> 2) + (cc & 3) * 4);
          const float2 r1 = *reinterpret_cast<const float2*>(rt + swz(rl + fr + 8, cc >> 2) + (cc & 3) * 4);
          v0.x += r0.x; v0.y += r0.y; v1.x += r1.x; v1.y += r1.y;
        }
        const uint32_t co = (uint32_t)(((cc >> 2) << 4) + (cc & 3) * 4);
        *reinterpret_cast<float2*>(buf + fr * 128 + (co ^ ((fr & 7) << 4))) = v0;
        *reinterpret_cast<float2*>(buf + (fr + 8) * 128 + (co ^ (((fr + 8) & 7) << 4))) = v1;
      }
      fence_proxy_async();
      __syncwarp();
      if (lane == 0 && row0 < p.M) { tma_store_2d(&mapC, smem_u32(buf), 0, row0); tma_commit(); }
      // the tile slot (split X, residual) is free once both groups are past it
      asm volatile("bar.sync %0, 128;" ::"r"(1 + g) : "memory");
      if (ctid == g * 128) mbar_arrive(bar_tempty + 8 * slot);
    }
    if (t_end > t_begin) flush_wgrad<NKB, false>(accW, g, wq, lane, p.dW, p.cexp, p.cin);
    if (lane == 0) tma_wait_read<0>();                   // staging buffers must outlive their stores
    __syncwarp();
  }
  __syncthreads();
}

template <int NKB, int ACT>
int launch_pb(const CUtensorMap& mDA, const CUtensorMap& mZ, const CUtensorMap& mX, const CUtensorMap& mR,
              const CUtensorMap& mC, const PbParams& p, const PbPlan& pl, cudaStream_t st) {
  static unsigned long long attr_mask = 0;
  if (int rc = eat_opt_in_smem(pw_bwd_fused_kernel<NKB, ACT>, kSmemLimit, attr_mask)) return rc;
  pw_bwd_fused_kernel<NKB, ACT><<<pl.splits, kThreads, pl.smem, st>>>(mDA, mZ, mX, mR, mC, p);
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

template <int ACT>
int launch_pb_act(const CUtensorMap& mDA, const CUtensorMap& mZ, const CUtensorMap& mX, const CUtensorMap& mR,
                  const CUtensorMap& mC, const PbParams& p, const PbPlan& pl, cudaStream_t st) {
  switch (pl.nkb) {
    case 1: return launch_pb<1, ACT>(mDA, mZ, mX, mR, mC, p, pl, st);
    case 2: return launch_pb<2, ACT>(mDA, mZ, mX, mR, mC, p, pl, st);
    case 3: return launch_pb<3, ACT>(mDA, mZ, mX, mR, mC, p, pl, st);
    default: return launch_pb<4, ACT>(mDA, mZ, mX, mR, mC, p, pl, st);
  }
}

// ===================================================================================================================
// Backward of an InvertedResidual's project stage (1x1 conv + BatchNorm, no activation) below its BatchNorm, for blocks
// without squeeze-excitation, in ONE pass -- the roles of the expand kernel above mirrored:
//
//     dz3        = scale3 * dy + alpha3 * z3 + beta3                            (the folded constants of eat_bn_bwd_apply)
//     dp[M,cexp] = dz3 . Wp                                                      Wp: project weight [cout, cexp]
//     dWp       += dz3^T . xf,  xf = act(z2 * scale2 + shift2)
//     s1[c]     += sum_m g,  s2[c] += invstd2[c] * sum_m g * (z2 - mean2[c]),  g = dp * act'(z2 * scale2 + shift2)
//
// (s1, s2: what eat_bn_bwd_reduce(dp, NULL, NULL, z2, ...) adds, the depthwise BatchNorm's backward sums.)  dz3 is never
// stored and dp is not read back.  The tile slot holds the dy and z3 boxes (cout <= 32); the fix-up turns them into the
// split dz3 in place.  The stages stream the raw z2 box of one 32-channel k-block of cexp; the fix-up writes the split
// xf into the stage's second box and leaves the raw box for the epilogue.  Per k-block the consumers compute one
// [128 x 32] chunk of dp (A = split dz3, K = cout; B = the resident Wp^T tile of the k-block's channels) and, in warpgroup
// kb % 2, the k-block's weight gradient (A = split xf, B = split dz3, accumulators = dWp^T, flushed transposed).  The
// per-k-block epilogue stores the dp chunk (staging tile + TMA store) and takes the BatchNorm sums from the fp32 dp
// fragments and the raw z2 box: fp32 over one warp's 16 rows, then fp64 in the warp's own slice of shared memory (plain
// read-modify-write: shared fp64 atomics are compare-and-swap loops), added up over the warps and flushed with fp64
// atomics once per CTA.
// HBM-bound: algorithmic bytes per launch = 4 * (2 M cexp (z2, dp) + 2 M cout (dy, z3) + 2 cout cexp).

struct PpParams {
  const float *scale3, *shift3, *mean3, *invstd3, *c1, *c2;      // BN3 and its backward coefficients
  const float *scale2, *shift2, *mean2, *invstd2, *W;            // BN2 and the project weight
  float* dW;
  double *s1, *s2;
  int M, cexp, cout, m_tiles, stages;
  uint32_t off_x, off_w, off_stg, off_s, off_f, off_bar;
};

// xf = act(z * scale + shift) of one landed k-block of the raw z box, split hi/lo into the box `out`; the raw box stays
// intact.  Rows >= rows_valid become zero.  Thread layout as fix_dz.
template <int ACT>
__device__ __forceinline__ void fix_xf(const unsigned char* zt, unsigned char* out, int ft, int rows_valid,
                                       const float* s_sc, const float* s_sh, int k) {
  const int cp = ft & 3, r0 = ft >> 2;
  const uint32_t row_off = (uint32_t)((r0 >> 3) * 1024 + (r0 & 7) * 128);
  const int x = r0 & 7;
  const uint32_t in0 = row_off + (((2 * cp) ^ x) << 4), in1 = row_off + (((2 * cp + 1) ^ x) << 4);
  const uint32_t out_hi = row_off + ((cp ^ x) << 4), out_lo = row_off + (((4 + cp) ^ x) << 4);
  float sc[8], sh[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) { sc[j] = s_sc[k + j]; sh[j] = s_sh[k + j]; }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const uint32_t o = (uint32_t)i * 32 * 128;
    const float4 za = *reinterpret_cast<const float4*>(zt + in0 + o), zb = *reinterpret_cast<const float4*>(zt + in1 + o);
    const float zv[8] = {za.x, za.y, za.z, za.w, zb.x, zb.y, zb.z, zb.w};
    float v[8];
    const bool live = r0 + 32 * i < rows_valid;
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = live ? act_in<ACT>(fmaf(zv[j], sc[j], sh[j])) : 0.f;
    uint4 h, l;
    split8(make_float4(v[0], v[1], v[2], v[3]), make_float4(v[4], v[5], v[6], v[7]), h, l);
    *reinterpret_cast<uint4*>(out + out_hi + o) = h;
    *reinterpret_cast<uint4*>(out + out_lo + o) = l;
  }
}

template <int NKB, int ACT>
__global__ void __launch_bounds__(kThreads, 1)   // 13 warps: 4 on one scheduler, so at most 128 registers per thread
pw_proj_bwd_kernel(const __grid_constant__ CUtensorMap mapDY, const __grid_constant__ CUtensorMap mapZ3,
                   const __grid_constant__ CUtensorMap mapZ2, const __grid_constant__ CUtensorMap mapC, const PpParams p) {
  constexpr int KP = NKB * KB;                           // padded channel count of the BN2 tables
  constexpr int NWA = (NKB + 1) / 2;                     // weight-gradient accumulators per warpgroup
  extern __shared__ __align__(1024) unsigned char smem[];
  unsigned char* s_x = smem + p.off_x;                   // [2 slots][dy | z3], then [split dz3 | dead]
  unsigned char* s_w = smem + p.off_w;                   // [NKB][32 rows x (32 hi | 32 lo) bf16]
  unsigned char* s_stg = smem + p.off_stg;
  double* s_sum = reinterpret_cast<double*>(smem + p.off_s);     // [8 consumer warps][2][KP]
  float* s_sc3 = reinterpret_cast<float*>(smem + p.off_f);
  float* s_sh3 = s_sc3 + KB;
  float* s_al3 = s_sh3 + KB;
  float* s_be3 = s_al3 + KB;
  float* s_sc2 = s_be3 + KB;
  float* s_sh2 = s_sc2 + KP;
  float* s_mu2 = s_sh2 + KP;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + p.off_bar);
  const int S = p.stages;
  const uint32_t bar_full = smem_u32(bars), bar_ready = bar_full + 8 * S, bar_empty = bar_ready + 8 * S;
  const uint32_t bar_tfull = bar_empty + 8 * S, bar_tready = bar_tfull + 16, bar_tempty = bar_tready + 16;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int t_begin, t_end;
  tile_range(p.m_tiles, t_begin, t_end);
  if (threadIdx.x == 0) {
    init_bars(bar_full, S);
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&mapDY)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&mapZ3)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&mapZ2)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&mapC)) : "memory");
  }
  // BN3's backward apply (as bn_bwd_apply2_kernel, no activation) and BN2's forward tables; zero beyond cout / cexp
  for (int c = threadIdx.x; c < KB; c += kThreads) {
    float sc = 0.f, sh = 0.f, al = 0.f, be = 0.f;
    if (c < p.cout) {
      sc = p.scale3[c]; sh = p.shift3[c];
      al = -sc * p.c2[c] * p.invstd3[c];
      be = -sc * p.c1[c] - al * p.mean3[c];
    }
    s_sc3[c] = sc; s_sh3[c] = sh; s_al3[c] = al; s_be3[c] = be;
  }
  for (int c = threadIdx.x; c < KP; c += kThreads) {
    const bool in = c < p.cexp;
    s_sc2[c] = in ? p.scale2[c] : 0.f;
    s_sh2[c] = in ? p.shift2[c] : 0.f;
    s_mu2[c] = in ? p.mean2[c] : 0.f;
  }
  for (int i = threadIdx.x; i < 8 * 2 * KP; i += kThreads) s_sum[i] = 0.0;
  // the data gradient's B operand: Wp^T as K-major rows, row n (channel of k-block kb) = 32 hi | 32 lo bf16 values of
  // Wp[0 .. 31, 32 kb + n]
  for (int i = threadIdx.x; i < NKB * KB * 4; i += kThreads) {
    const int cp = i & 3, n = (i >> 2) & (KB - 1), kb = i >> 7;
    const int c = kb * KB + n;
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int o = cp * 8 + j;
      v[j] = (o < p.cout && c < p.cexp) ? __ldg(p.W + (size_t)o * p.cexp + c) : 0.f;
    }
    uint4 hi, lo;
    split8(make_float4(v[0], v[1], v[2], v[3]), make_float4(v[4], v[5], v[6], v[7]), hi, lo);
    unsigned char* wt = s_w + (size_t)kb * KB * 128;
    *reinterpret_cast<uint4*>(wt + swz(n, cp)) = hi;
    *reinterpret_cast<uint4*>(wt + swz(n, 4 + cp)) = lo;
  }
  fence_proxy_async();
  __syncthreads();
  const uint32_t stage_base = smem_u32(smem), x_base = smem_u32(s_x);

  if (warp == kTmaWarp) {
    // ================================================================= TMA producer (one thread)
    if (lane == 0) {
      int s = 0;
      uint32_t ph = 0;
      for (int t = t_begin, i = 0; t < t_end; ++t, ++i) {
        const int slot = i & 1;
        const uint32_t tph = (uint32_t)(i >> 1) & 1u;
        const int m0 = t * BM;
        mbar_wait(bar_tempty + 8 * slot, tph ^ 1u);
        const uint32_t xd = x_base + (uint32_t)slot * 2 * BOX;
        mbar_expect_tx(bar_tfull + 8 * slot, 2 * BOX);
        tma_load_2d(&mapDY, bar_tfull + 8 * slot, xd, 0, m0);
        tma_load_2d(&mapZ3, bar_tfull + 8 * slot, xd + BOX, 0, m0);
        for (int kb = 0; kb < NKB; ++kb) {
          mbar_wait(bar_empty + 8 * s, ph ^ 1u);
          mbar_expect_tx(bar_full + 8 * s, BOX);
          tma_load_2d(&mapZ2, bar_full + 8 * s, stage_base + (uint32_t)s * 2 * BOX, kb * KB, m0);
          if (++s == S) { s = 0; ph ^= 1u; }
        }
      }
    }
    __syncwarp();
  } else if (warp < kFirstCons) {
    // ================================================================= fix-up warps (128 threads)
    const int ft = threadIdx.x;
    int s = 0;
    uint32_t ph = 0;
    for (int t = t_begin, i = 0; t < t_end; ++t, ++i) {
      const int slot = i & 1;
      const uint32_t tph = (uint32_t)(i >> 1) & 1u;
      const int rows_valid = min(BM, p.M - t * BM);
      mbar_wait(bar_tfull + 8 * slot, tph);
      unsigned char* xt = s_x + (size_t)slot * 2 * BOX;
      fix_dz<EAT_ACT_NONE>(xt, xt + BOX, ft, rows_valid, s_sc3, s_sh3, s_al3, s_be3, (ft & 3) * 8);
      fence_proxy_async();
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_tready + 8 * slot);
      for (int kb = 0; kb < NKB; ++kb) {
        mbar_wait(bar_full + 8 * s, ph);
        unsigned char* st = smem + (size_t)s * 2 * BOX;
        fix_xf<ACT>(st, st + BOX, ft, rows_valid, s_sc2, s_sh2, kb * KB + (ft & 3) * 8);
        fence_proxy_async();
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_ready + 8 * s);
        if (++s == S) { s = 0; ph ^= 1u; }
      }
    }
  } else {
    // ================================================================= consumers: MMAs, per-k-block epilogue, weight-gradient flush
    const int cw = warp - kFirstCons;
    const int g = cw >> 2, wq = cw & 3;                  // warpgroup (64-row half of dp), warp inside it
    const int ctid = threadIdx.x - kFirstCons * 32;
    unsigned char* stg = s_stg + (size_t)cw * 2 * STG_BYTES;
    const uint64_t desc0 = gmma_desc(0);
    const uint64_t w0 = desc0 + (smem_u32(s_w) >> 4);
    const int fr = lane >> 2, fc = 2 * (lane & 3);       // fragment row / column of this lane
    const int rl = g * 64 + wq * 16;                     // first row of this warp's slab inside the tile
    float accW[NWA][32];
#pragma unroll
    for (int w = 0; w < NWA; ++w)
#pragma unroll
      for (int e = 0; e < 32; ++e) accW[w][e] = 0.f;
    int s = 0, cb = 0;
    uint32_t ph = 0;
    for (int t = t_begin, i = 0; t < t_end; ++t, ++i) {
      const int slot = i & 1;
      const uint32_t tph = (uint32_t)(i >> 1) & 1u;
      mbar_wait(bar_tready + 8 * slot, tph);
      const uint32_t sx = x_base + (uint32_t)slot * 2 * BOX;
      // data gradient's A: row = [hi: 32 bf16 | lo: 32 bf16]; K=16 steps at +0/+32 B (hi) and +64/+96 B (lo)
      const uint64_t a_hi = desc0 + ((sx + (uint32_t)g * 8192u) >> 4), a_lo = a_hi + 4;
      const int row0 = t * BM + rl;
#pragma unroll
      for (int kb = 0; kb < NKB; ++kb) {
        mbar_wait(bar_ready + 8 * s, ph);
        const uint32_t sa = stage_base + (uint32_t)s * 2 * BOX;  // raw z2 box; the split xf box follows at + BOX
        const uint64_t w_hi = w0 + (uint64_t)(kb * KB * 128 / 16), w_lo = w_hi + 4;
        float acc[16];
#pragma unroll
        for (int e = 0; e < 16; ++e) acc[e] = 0.f;
        wgmma_fence();
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const uint64_t ko = (uint64_t)(j * 2);
          wgmma_n32<0, 0>(acc, a_hi + ko, w_hi + ko);
          wgmma_n32<0, 0>(acc, a_lo + ko, w_hi + ko);
          wgmma_n32<0, 0>(acc, a_hi + ko, w_lo + ko);
        }
        // weight gradient (transposed) of this k-block's 32 channels: 16 reduction rows (2048 B) per instruction
        if ((kb & 1) == g) {
#pragma unroll
          for (int st = 0; st < BM / 16; ++st)
            wgmma_n64<1, 1>(accW[kb >> 1], gmma_desc(sa + BOX + st * 2048, BOX, 1024), gmma_desc(sx + st * 2048, BOX, 1024));
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(acc);
#pragma unroll
        for (int w = 0; w < NWA; ++w) wgmma_fence_regs(accW[w]);
        // ---- epilogue of the k-block: fragment -> swizzled 16 x 32 staging tile -> TMA store (rows / columns past the
        // tensor clipped); BN2 sums against the raw z2 box.  Rows past M hold dp = 0 (dz3 is zeroed there).
        unsigned char* buf = stg + (size_t)cb * STG_BYTES;
        cb ^= 1;
        if (lane == 0) tma_wait_read<1>();               // the store issued from this buffer two k-blocks ago has drained
        __syncwarp();
        const unsigned char* zt = smem + (size_t)s * 2 * BOX;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int cc = 8 * j + fc, c = kb * KB + cc;
          const float2 v0 = make_float2(acc[4 * j], acc[4 * j + 1]), v1 = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
          const uint32_t co = (uint32_t)(((cc >> 2) << 4) + (cc & 3) * 4);
          *reinterpret_cast<float2*>(buf + fr * 128 + (co ^ ((fr & 7) << 4))) = v0;
          *reinterpret_cast<float2*>(buf + (fr + 8) * 128 + (co ^ (((fr + 8) & 7) << 4))) = v1;
          const float2 z0 = *reinterpret_cast<const float2*>(zt + swz(rl + fr, cc >> 2) + (cc & 3) * 4);
          const float2 z1 = *reinterpret_cast<const float2*>(zt + swz(rl + fr + 8, cc >> 2) + (cc & 3) * 4);
          const float2 sc = *reinterpret_cast<const float2*>(s_sc2 + c), sh = *reinterpret_cast<const float2*>(s_sh2 + c);
          const float2 mu = *reinterpret_cast<const float2*>(s_mu2 + c);
          const float g0x = v0.x * act_bwd(fmaf(z0.x, sc.x, sh.x), ACT), g0y = v0.y * act_bwd(fmaf(z0.y, sc.y, sh.y), ACT);
          const float g1x = v1.x * act_bwd(fmaf(z1.x, sc.x, sh.x), ACT), g1y = v1.y * act_bwd(fmaf(z1.y, sc.y, sh.y), ACT);
          float a1x = g0x + g1x, a1y = g0y + g1y;
          float a2x = fmaf(g0x, z0.x - mu.x, g1x * (z1.x - mu.x)), a2y = fmaf(g0y, z0.y - mu.y, g1y * (z1.y - mu.y));
#pragma unroll
          for (int m = 4; m < 32; m <<= 1) {             // over the 8 fragment rows of the column pair
            a1x += __shfl_xor_sync(0xffffffffu, a1x, m); a1y += __shfl_xor_sync(0xffffffffu, a1y, m);
            a2x += __shfl_xor_sync(0xffffffffu, a2x, m); a2y += __shfl_xor_sync(0xffffffffu, a2y, m);
          }
          if (fr == 0) {                                 // lanes 0-3: distinct columns of the warp's slice
            double* ws = s_sum + (size_t)cw * 2 * KP;
            ws[c] += (double)a1x; ws[c + 1] += (double)a1y;
            ws[KP + c] += (double)a2x; ws[KP + c + 1] += (double)a2y;
          }
        }
        fence_proxy_async();
        __syncwarp();
        if (lane == 0 && row0 < p.M) { tma_store_2d(&mapC, smem_u32(buf), kb * KB, row0); tma_commit(); }
        // the stage (raw and split z2) is free once both groups are past it
        asm volatile("bar.sync %0, 128;" ::"r"(1 + g) : "memory");
        if (ctid == g * 128) mbar_arrive(bar_empty + 8 * s);
        if (++s == S) { s = 0; ph ^= 1u; }
      }
      // the tile slot (split dz3) is free: every warp of the group passed the last k-block's barrier after its MMAs
      if (ctid == g * 128) mbar_arrive(bar_tempty + 8 * slot);
    }
    if (t_end > t_begin) flush_wgrad<NKB, true>(accW, g, wq, lane, p.dW, p.cexp, p.cout);
    if (lane == 0) tma_wait_read<0>();                   // staging buffers must outlive their stores
    __syncwarp();
  }
  __syncthreads();
  // the CTA's BN2 sums, once
  if (t_end > t_begin) {
    for (int c = threadIdx.x; c < p.cexp; c += kThreads) {
      double a1 = 0.0, a2 = 0.0;
#pragma unroll
      for (int w = 0; w < 8; ++w) { a1 += s_sum[w * 2 * KP + c]; a2 += s_sum[w * 2 * KP + KP + c]; }
      atomicAdd(p.s1 + c, a1);
      atomicAdd(p.s2 + c, a2 * (double)p.invstd2[c]);
    }
  }
}

template <int NKB, int ACT>
int launch_pp(const CUtensorMap& mDY, const CUtensorMap& mZ3, const CUtensorMap& mZ2, const CUtensorMap& mC,
              const PpParams& p, const PbPlan& pl, cudaStream_t st) {
  static unsigned long long attr_mask = 0;
  if (int rc = eat_opt_in_smem(pw_proj_bwd_kernel<NKB, ACT>, kSmemLimit, attr_mask)) return rc;
  pw_proj_bwd_kernel<NKB, ACT><<<pl.splits, kThreads, pl.smem, st>>>(mDY, mZ3, mZ2, mC, p);
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

template <int ACT>
int launch_pp_act(const CUtensorMap& mDY, const CUtensorMap& mZ3, const CUtensorMap& mZ2, const CUtensorMap& mC,
                  const PpParams& p, const PbPlan& pl, cudaStream_t st) {
  switch (pl.nkb) {
    case 1: return launch_pp<1, ACT>(mDY, mZ3, mZ2, mC, p, pl, st);
    case 2: return launch_pp<2, ACT>(mDY, mZ3, mZ2, mC, p, pl, st);
    case 3: return launch_pp<3, ACT>(mDY, mZ3, mZ2, mC, p, pl, st);
    default: return launch_pp<4, ACT>(mDY, mZ3, mZ2, mC, p, pl, st);
  }
}

}  // namespace

extern "C" int eat_pw_bwd_plan(long long M, int cexp, int cin, int* plan) {
  if (plan == nullptr) { eat_set_error("pw_bwd_plan: plan is NULL"); return EAT_ERR_ARG; }
  PbPlan pl;
  if (int rc = plan_pb(M, cexp, cin, kNumSMs, false, pl)) return rc;
  plan[0] = pl.splits; plan[1] = pl.rows_per_split; plan[2] = pl.stages; plan[3] = pl.smem;
  return EAT_OK;
}

extern "C" int eat_pw_conv_bwd_fused(const float* da, const float* z, const float* scale, const float* shift,
                                     const float* mean, const float* invstd, int act, const float* c1, const float* c2,
                                     const float* X, const float* W, const float* res, float* dX, float* dW, int dtype,
                                     long long M, int cexp, int cin, cudaStream_t st) {
  if (dtype != EAT_F32) { eat_set_error("pw_conv_bwd_fused: fp32 storage only"); return EAT_ERR_UNSUPPORTED; }
  if (act != EAT_ACT_RELU && act != EAT_ACT_HSWISH) { eat_set_error("pw_conv_bwd_fused: activation must be relu or hardswish"); return EAT_ERR_UNSUPPORTED; }
  if (M < 0) { eat_set_error("pw_conv_bwd_fused: negative M"); return EAT_ERR_ARG; }
  if (da == nullptr || z == nullptr || scale == nullptr || shift == nullptr || mean == nullptr || invstd == nullptr ||
      c1 == nullptr || c2 == nullptr || X == nullptr || W == nullptr || dX == nullptr || dW == nullptr) {
    eat_set_error("pw_conv_bwd_fused: da, z, the BatchNorm tables, c1/c2, X, W, dX and dW are required");
    return EAT_ERR_ARG;
  }
  if ((((uintptr_t)da) | ((uintptr_t)z) | ((uintptr_t)X) | ((uintptr_t)res) | ((uintptr_t)dX)) & 15) {
    eat_set_error("pw_conv_bwd_fused: activation tensors must be 16-byte aligned");
    return EAT_ERR_ARG;
  }
  if (((uintptr_t)dW) & 7) { eat_set_error("pw_conv_bwd_fused: dW must be 8-byte aligned"); return EAT_ERR_ARG; }
  PbPlan pl;
  if (int rc = plan_pb(M > 0 ? M : 1, cexp, cin, kNumSMs, false, pl)) return rc;
  if (M == 0) return EAT_OK;
  int dev = 0, sms = kNumSMs;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (int rc = plan_pb(M, cexp, cin, sms, false, pl)) return rc;
  CUtensorMap mDA, mZ, mX, mR, mC;
  if (int rc = make_map(&mDA, da, M, cexp, BM)) return rc;
  if (int rc = make_map(&mZ, z, M, cexp, BM)) return rc;
  if (int rc = make_map(&mX, X, M, cin, BM)) return rc;
  if (int rc = make_map(&mR, res != nullptr ? res : X, M, cin, BM)) return rc;
  if (int rc = make_map(&mC, dX, M, cin, 16)) return rc;
  PbParams p;
  p.scale = scale; p.shift = shift; p.mean = mean; p.invstd = invstd; p.c1 = c1; p.c2 = c2; p.W = W; p.dW = dW;
  p.M = (int)M; p.cexp = cexp; p.cin = cin; p.m_tiles = (int)((M + BM - 1) / BM); p.stages = pl.stages;
  p.res = res != nullptr ? 1 : 0;
  p.off_x = pl.off_x; p.off_w = pl.off_w; p.off_stg = pl.off_stg; p.off_f = pl.off_f; p.off_bar = pl.off_bar;
  if (act == EAT_ACT_RELU) return launch_pb_act<EAT_ACT_RELU>(mDA, mZ, mX, mR, mC, p, pl, st);
  return launch_pb_act<EAT_ACT_HSWISH>(mDA, mZ, mX, mR, mC, p, pl, st);
}

extern "C" int eat_pw_proj_bwd_plan(long long M, int cexp, int cout, int* plan) {
  if (plan == nullptr) { eat_set_error("pw_proj_bwd_plan: plan is NULL"); return EAT_ERR_ARG; }
  PbPlan pl;
  if (int rc = plan_pb(M, cexp, cout, kNumSMs, true, pl)) return rc;
  plan[0] = pl.splits; plan[1] = pl.rows_per_split; plan[2] = pl.stages; plan[3] = pl.smem;
  return EAT_OK;
}

extern "C" int eat_pw_proj_bwd_fused(const float* dy, const float* z3, const float* scale3, const float* shift3,
                                     const float* mean3, const float* invstd3, const float* c1, const float* c2,
                                     const float* z2, const float* scale2, const float* shift2, const float* mean2,
                                     const float* invstd2, int act, const float* W, float* dp, float* dW, double* s1,
                                     double* s2, int dtype, long long M, int cexp, int cout, cudaStream_t st) {
  if (dtype != EAT_F32) { eat_set_error("pw_proj_bwd_fused: fp32 storage only"); return EAT_ERR_UNSUPPORTED; }
  if (act != EAT_ACT_RELU && act != EAT_ACT_HSWISH) { eat_set_error("pw_proj_bwd_fused: activation must be relu or hardswish"); return EAT_ERR_UNSUPPORTED; }
  if (M < 0) { eat_set_error("pw_proj_bwd_fused: negative M"); return EAT_ERR_ARG; }
  if (dy == nullptr || z3 == nullptr || scale3 == nullptr || shift3 == nullptr || mean3 == nullptr || invstd3 == nullptr ||
      c1 == nullptr || c2 == nullptr || z2 == nullptr || scale2 == nullptr || shift2 == nullptr || mean2 == nullptr ||
      invstd2 == nullptr || W == nullptr || dp == nullptr || dW == nullptr || s1 == nullptr || s2 == nullptr) {
    eat_set_error("pw_proj_bwd_fused: dy, z3, both BatchNorms' tables, c1/c2, z2, W, dp, dW, s1 and s2 are required");
    return EAT_ERR_ARG;
  }
  if ((((uintptr_t)dy) | ((uintptr_t)z3) | ((uintptr_t)z2) | ((uintptr_t)dp)) & 15) {
    eat_set_error("pw_proj_bwd_fused: activation tensors must be 16-byte aligned");
    return EAT_ERR_ARG;
  }
  if ((((uintptr_t)s1) | ((uintptr_t)s2)) & 7) { eat_set_error("pw_proj_bwd_fused: s1 and s2 must be 8-byte aligned"); return EAT_ERR_ARG; }
  PbPlan pl;
  if (int rc = plan_pb(M > 0 ? M : 1, cexp, cout, kNumSMs, true, pl)) return rc;
  if (M == 0) return EAT_OK;
  int dev = 0, sms = kNumSMs;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (int rc = plan_pb(M, cexp, cout, sms, true, pl)) return rc;
  CUtensorMap mDY, mZ3, mZ2, mC;
  if (int rc = make_map(&mDY, dy, M, cout, BM)) return rc;
  if (int rc = make_map(&mZ3, z3, M, cout, BM)) return rc;
  if (int rc = make_map(&mZ2, z2, M, cexp, BM)) return rc;
  if (int rc = make_map(&mC, dp, M, cexp, 16)) return rc;
  PpParams p;
  p.scale3 = scale3; p.shift3 = shift3; p.mean3 = mean3; p.invstd3 = invstd3; p.c1 = c1; p.c2 = c2;
  p.scale2 = scale2; p.shift2 = shift2; p.mean2 = mean2; p.invstd2 = invstd2; p.W = W; p.dW = dW; p.s1 = s1; p.s2 = s2;
  p.M = (int)M; p.cexp = cexp; p.cout = cout; p.m_tiles = (int)((M + BM - 1) / BM); p.stages = pl.stages;
  p.off_x = pl.off_x; p.off_w = pl.off_w; p.off_stg = pl.off_stg; p.off_s = pl.off_s; p.off_f = pl.off_f;
  p.off_bar = pl.off_bar;
  if (act == EAT_ACT_RELU) return launch_pp_act<EAT_ACT_RELU>(mDY, mZ3, mZ2, mC, p, pl, st);
  return launch_pp_act<EAT_ACT_HSWISH>(mDY, mZ3, mZ2, mC, p, pl, st);
}
