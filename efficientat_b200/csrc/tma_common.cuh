// Shared pieces of the TMA-fed wgmma kernels (pw_tma.cu, wgrad_tma.cu): cp.async.bulk.tensor / mbarrier PTX wrappers,
// the host-side tensor-map encoder (cuTensorMapEncodeTiled fetched through the runtime, no libcuda link), and the
// on-chip "fix-up" pass that turns a TMA-landed fp32 tile into bf16 hi/lo operands IN PLACE.
#pragma once
#include <cuda.h>

#include "tc_common.cuh"

namespace tma {
using namespace tc;

constexpr int KB = 32;                  // fp32 elements per landed row = one 128-byte swizzle row

__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_load_2d(const CUtensorMap* map, uint32_t bar, uint32_t dst, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, uint32_t src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(map)), "r"(src), "r"(c0), "r"(c1) : "memory");
}
// 3-D variants: the third coordinate is the sample, so that boxes never cross a sample boundary (rows past the end of a
// sample are zero-filled on load and clipped on store by the TMA unit)
__device__ __forceinline__ void tma_load_3d(const CUtensorMap* map, uint32_t bar, uint32_t dst, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* map, uint32_t src, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(map)), "r"(src), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ void tma_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void tma_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}

template <int XACT> __device__ __forceinline__ float act_in(float v) {
  if (XACT == 1) return fmaxf(v, 0.f);
  if (XACT == 2) return v * fminf(fmaxf(v + 3.f, 0.f), 6.f) * (1.f / 6.f);
  return v;
}
template <int EPI> __device__ __forceinline__ float act_out(float v) {
  if (EPI == 2) return fmaxf(v, 0.f);
  if (EPI == 3) return v * fminf(fmaxf(v + 3.f, 0.f), 6.f) * (1.f / 6.f);
  return v;
}
// 8 fp32 values -> 8 bf16 hi (one 16-byte chunk) + 8 bf16 lo with hi + lo = v to ~2^-17
__device__ __forceinline__ void split8(const float4 a, const float4 b, uint4& hi, uint4& lo) {
  hi.x = pack_bf16(a.x, a.y); hi.y = pack_bf16(a.z, a.w); hi.z = pack_bf16(b.x, b.y); hi.w = pack_bf16(b.z, b.w);
  // bf16 -> fp32 is a 16-bit shift: element 0 of a pair sits in the low half
  lo.x = pack_bf16(a.x - __uint_as_float(hi.x << 16), a.y - __uint_as_float(hi.x & 0xFFFF0000u));
  lo.y = pack_bf16(a.z - __uint_as_float(hi.y << 16), a.w - __uint_as_float(hi.y & 0xFFFF0000u));
  lo.z = pack_bf16(b.x - __uint_as_float(hi.z << 16), b.y - __uint_as_float(hi.z & 0xFFFF0000u));
  lo.w = pack_bf16(b.z - __uint_as_float(hi.w << 16), b.w - __uint_as_float(hi.w & 0xFFFF0000u));
}

// ---- fix-up passes over a landed 128-byte-swizzled fp32 tile [rows][32 k].  128 fix-up threads; a thread owns the chunk
// PAIR cp (fp32 chunks 2cp, 2cp+1 = 8 consecutive k) of 2^LG rows (r0 + i * (128 >> LG)) and writes, into the SAME row,
// the bf16 hi chunk at logical position cp and the lo chunk at 4 + cp.  The threads of a row are neighbouring lanes of
// one warp: all loads are issued first, a __syncwarp separates them from the in-place stores.
template <int LG, int TR = 128>
struct FixMap {
  static constexpr int RSTEP = 128 >> LG;         // rows per pass: a multiple of 8, so (row & 7) is the same for all rows of a thread
  static constexpr int ROWS = TR / RSTEP;         // rows per thread (TR = rows of the tile: 128, or 64 for the weight-gradient blocks)
  static constexpr int STRIDE = RSTEP * 128;      // bytes between a thread's rows
  static_assert(ROWS >= 1, "tile too short for this chunk-pair count");
};

// LG = 1 (a k-block with <= 16 valid k): the second K=16 step's hi / lo chunks (2 + cp, 6 + cp) still hold raw fp32 bits of
// the landed row; zero them so that the MMAs can always run both steps of a k-block
__device__ __forceinline__ void zero_upper(unsigned char* row, int cp, int x) {
  const uint4 z = make_uint4(0u, 0u, 0u, 0u);
  *reinterpret_cast<uint4*>(row + (((2 + cp) ^ x) << 4)) = z;
  *reinterpret_cast<uint4*>(row + (((6 + cp) ^ x) << 4)) = z;
}

// The reading half of fix_a, for fix_pair: this thread's 8 fp32 values (va, vb) of each of its rows of a landed tile, with
// the optional BatchNorm affine + activation (XACT >= 0) and SE gate applied and rows >= rows_valid forced to zero.
// fix_a keeps its own copy so that the kernels built on it compile to the same instructions as before.
template <int LG, int XACT, int TR>
__device__ __forceinline__ void fix_load(const unsigned char* tile, int ft, int rows_valid, const float* s_isc,
                                         const float* s_ish, int k, const float* gate, int off0, int b0, int rps, int K,
                                         float4 (&va)[FixMap<LG, TR>::ROWS], float4 (&vb)[FixMap<LG, TR>::ROWS]) {
  using M = FixMap<LG, TR>;
  const int cp = ft & ((1 << LG) - 1), r0 = ft >> LG;
  const uint32_t row_off = (uint32_t)((r0 >> 3) * 1024 + (r0 & 7) * 128);
  const int x = r0 & 7;
  const uint32_t in0 = row_off + (((2 * cp) ^ x) << 4), in1 = row_off + (((2 * cp + 1) ^ x) << 4);
#pragma unroll
  for (int i = 0; i < M::ROWS; ++i) {
    va[i] = *reinterpret_cast<const float4*>(tile + in0 + i * M::STRIDE);
    vb[i] = *reinterpret_cast<const float4*>(tile + in1 + i * M::STRIDE);
  }
  if (XACT >= 0) {
    const float4 sa = *reinterpret_cast<const float4*>(s_isc + k), sb = *reinterpret_cast<const float4*>(s_isc + k + 4);
    const float4 ha = *reinterpret_cast<const float4*>(s_ish + k), hb = *reinterpret_cast<const float4*>(s_ish + k + 4);
#pragma unroll
    for (int i = 0; i < M::ROWS; ++i) {
      va[i].x = act_in<XACT>(fmaf(va[i].x, sa.x, ha.x)); va[i].y = act_in<XACT>(fmaf(va[i].y, sa.y, ha.y));
      va[i].z = act_in<XACT>(fmaf(va[i].z, sa.z, ha.z)); va[i].w = act_in<XACT>(fmaf(va[i].w, sa.w, ha.w));
      vb[i].x = act_in<XACT>(fmaf(vb[i].x, sb.x, hb.x)); vb[i].y = act_in<XACT>(fmaf(vb[i].y, sb.y, hb.y));
      vb[i].z = act_in<XACT>(fmaf(vb[i].z, sb.z, hb.z)); vb[i].w = act_in<XACT>(fmaf(vb[i].w, sb.w, hb.w));
    }
  }
  if (rows_valid < TR) {                          // rows past the end of the tensor / of the split stay (or become) zero
#pragma unroll
    for (int i = 0; i < M::ROWS; ++i)
      if (r0 + i * M::RSTEP >= rows_valid) { va[i] = make_float4(0.f, 0.f, 0.f, 0.f); vb[i] = va[i]; }
  }
  if (gate != nullptr && k < K) {
    const bool k2 = k + 4 < K;
    const float4 one = make_float4(1.f, 1.f, 1.f, 1.f);
    if (rps >= TR) {
      // a 128-row tile touches at most two samples: both gate vectors are requested up front (L1/L2 hits) instead of
      // one dependent load per row
      const float4* gp0 = reinterpret_cast<const float4*>(gate + (size_t)b0 * K + k);
      const bool two = off0 + rows_valid > rps;
      const float4* gp1 = two ? reinterpret_cast<const float4*>(gate + (size_t)(b0 + 1) * K + k) : gp0;
      const float4 g0a = __ldg(gp0), g0b = k2 ? __ldg(gp0 + 1) : one, g1a = __ldg(gp1), g1b = k2 ? __ldg(gp1 + 1) : one;
#pragma unroll
      for (int i = 0; i < M::ROWS; ++i) {
        const bool hi_b = off0 + r0 + i * M::RSTEP >= rps;
        const float4 ga = hi_b ? g1a : g0a, gb = hi_b ? g1b : g0b;
        va[i].x *= ga.x; va[i].y *= ga.y; va[i].z *= ga.z; va[i].w *= ga.w;
        vb[i].x *= gb.x; vb[i].y *= gb.y; vb[i].z *= gb.z; vb[i].w *= gb.w;
      }
    } else {
#pragma unroll
      for (int i = 0; i < M::ROWS; ++i) {
        const int r = r0 + i * M::RSTEP;
        if (r < rows_valid) {
          const float4* gp = reinterpret_cast<const float4*>(gate + (size_t)((off0 + r) / rps + b0) * K + k);
          const float4 ga = __ldg(gp), gb = k2 ? __ldg(gp + 1) : one;
          va[i].x *= ga.x; va[i].y *= ga.y; va[i].z *= ga.z; va[i].w *= ga.w;
          vb[i].x *= gb.x; vb[i].y *= gb.y; vb[i].z *= gb.z; vb[i].w *= gb.w;
        }
      }
    }
  }
}

// A-operand tile: optional BatchNorm affine + activation (XACT >= 0) and SE gate, rows >= rows_valid forced to zero
template <int LG, int XACT, int TR = 128>
__device__ __forceinline__ void fix_a(unsigned char* tile, int ft, int rows_valid, const float* s_isc, const float* s_ish,
                                      int k, const float* gate, int off0, int b0, int rps, int K) {
  using M = FixMap<LG, TR>;
  const int cp = ft & ((1 << LG) - 1), r0 = ft >> LG;
  const uint32_t row_off = (uint32_t)((r0 >> 3) * 1024 + (r0 & 7) * 128);
  const int x = r0 & 7;
  const uint32_t in0 = row_off + (((2 * cp) ^ x) << 4), in1 = row_off + (((2 * cp + 1) ^ x) << 4);
  const uint32_t out_hi = row_off + ((cp ^ x) << 4), out_lo = row_off + (((4 + cp) ^ x) << 4);
  float4 va[M::ROWS], vb[M::ROWS];
#pragma unroll
  for (int i = 0; i < M::ROWS; ++i) {
    va[i] = *reinterpret_cast<const float4*>(tile + in0 + i * M::STRIDE);
    vb[i] = *reinterpret_cast<const float4*>(tile + in1 + i * M::STRIDE);
  }
  if (XACT >= 0) {
    const float4 sa = *reinterpret_cast<const float4*>(s_isc + k), sb = *reinterpret_cast<const float4*>(s_isc + k + 4);
    const float4 ha = *reinterpret_cast<const float4*>(s_ish + k), hb = *reinterpret_cast<const float4*>(s_ish + k + 4);
#pragma unroll
    for (int i = 0; i < M::ROWS; ++i) {
      va[i].x = act_in<XACT>(fmaf(va[i].x, sa.x, ha.x)); va[i].y = act_in<XACT>(fmaf(va[i].y, sa.y, ha.y));
      va[i].z = act_in<XACT>(fmaf(va[i].z, sa.z, ha.z)); va[i].w = act_in<XACT>(fmaf(va[i].w, sa.w, ha.w));
      vb[i].x = act_in<XACT>(fmaf(vb[i].x, sb.x, hb.x)); vb[i].y = act_in<XACT>(fmaf(vb[i].y, sb.y, hb.y));
      vb[i].z = act_in<XACT>(fmaf(vb[i].z, sb.z, hb.z)); vb[i].w = act_in<XACT>(fmaf(vb[i].w, sb.w, hb.w));
    }
  }
  if (rows_valid < TR) {                          // rows past the end of the tensor / of the split stay (or become) zero
#pragma unroll
    for (int i = 0; i < M::ROWS; ++i)
      if (r0 + i * M::RSTEP >= rows_valid) { va[i] = make_float4(0.f, 0.f, 0.f, 0.f); vb[i] = va[i]; }
  }
  if (gate != nullptr && k < K) {
    const bool k2 = k + 4 < K;
    const float4 one = make_float4(1.f, 1.f, 1.f, 1.f);
    if (rps >= TR) {
      // a 128-row tile touches at most two samples: both gate vectors are requested up front (L1/L2 hits) instead of
      // one dependent load per row
      const float4* gp0 = reinterpret_cast<const float4*>(gate + (size_t)b0 * K + k);
      const bool two = off0 + rows_valid > rps;
      const float4* gp1 = two ? reinterpret_cast<const float4*>(gate + (size_t)(b0 + 1) * K + k) : gp0;
      const float4 g0a = __ldg(gp0), g0b = k2 ? __ldg(gp0 + 1) : one, g1a = __ldg(gp1), g1b = k2 ? __ldg(gp1 + 1) : one;
#pragma unroll
      for (int i = 0; i < M::ROWS; ++i) {
        const bool hi_b = off0 + r0 + i * M::RSTEP >= rps;
        const float4 ga = hi_b ? g1a : g0a, gb = hi_b ? g1b : g0b;
        va[i].x *= ga.x; va[i].y *= ga.y; va[i].z *= ga.z; va[i].w *= ga.w;
        vb[i].x *= gb.x; vb[i].y *= gb.y; vb[i].z *= gb.z; vb[i].w *= gb.w;
      }
    } else {
#pragma unroll
      for (int i = 0; i < M::ROWS; ++i) {
        const int r = r0 + i * M::RSTEP;
        if (r < rows_valid) {
          const float4* gp = reinterpret_cast<const float4*>(gate + (size_t)((off0 + r) / rps + b0) * K + k);
          const float4 ga = __ldg(gp), gb = k2 ? __ldg(gp + 1) : one;
          va[i].x *= ga.x; va[i].y *= ga.y; va[i].z *= ga.z; va[i].w *= ga.w;
          vb[i].x *= gb.x; vb[i].y *= gb.y; vb[i].z *= gb.z; vb[i].w *= gb.w;
        }
      }
    }
  }
  __syncwarp();                                   // every lane of the row has its inputs before anyone overwrites them
#pragma unroll
  for (int i = 0; i < M::ROWS; ++i) {
    uint4 h, l;
    split8(va[i], vb[i], h, l);
    *reinterpret_cast<uint4*>(tile + out_hi + i * M::STRIDE) = h;
    *reinterpret_cast<uint4*>(tile + out_lo + i * M::STRIDE) = l;
    if (LG == 1) zero_upper(tile + row_off + i * M::STRIDE, cp, x);
  }
}

// PAIR fix-up of two landed [TR rows x 32 channels] fp32 tiles of the same rows, channels c .. c+31 (ta) and c+32 .. c+63
// (tb): afterwards each row of ta holds the 64 bf16 hi values of the 64 channels and the same row of tb their 64 bf16 lo
// values, channel j at logical chunk j / 8.  Each tile is then a canonical MN-major SWIZZLE_128B atom column of 64
// channels, all hi or all lo.  The transforms are fix_a's (k: channel of this thread's first value in ta).  tb_landed =
// false: tb holds no data (its channels lie past the tensor) and counts as zeros.  Thread layout of fix_a<2>.
template <int XACT, int TR>
__device__ __forceinline__ void fix_pair(unsigned char* ta, unsigned char* tb, bool tb_landed, int ft, int rows_valid,
                                         const float* s_isc, const float* s_ish, int k, const float* gate, int off0,
                                         int b0, int rps, int K) {
  using M = FixMap<2, TR>;
  const int cp = ft & 3, r0 = ft >> 2;
  const uint32_t row_off = (uint32_t)((r0 >> 3) * 1024 + (r0 & 7) * 128);
  const int x = r0 & 7;
  const uint32_t out_a = row_off + ((cp ^ x) << 4), out_b = row_off + (((4 + cp) ^ x) << 4);
  float4 va[M::ROWS], vb[M::ROWS], wa[M::ROWS], wb[M::ROWS];
  fix_load<2, XACT, TR>(ta, ft, rows_valid, s_isc, s_ish, k, gate, off0, b0, rps, K, va, vb);
  if (tb_landed) {
    fix_load<2, XACT, TR>(tb, ft, rows_valid, s_isc, s_ish, k + 32, gate, off0, b0, rps, K, wa, wb);
  } else {
#pragma unroll
    for (int i = 0; i < M::ROWS; ++i) { wa[i] = make_float4(0.f, 0.f, 0.f, 0.f); wb[i] = wa[i]; }
  }
  __syncwarp();                                   // every lane of the row has read both tiles before anyone overwrites them
#pragma unroll
  for (int i = 0; i < M::ROWS; ++i) {
    uint4 h0, l0, h1, l1;
    split8(va[i], vb[i], h0, l0);
    split8(wa[i], wb[i], h1, l1);
    *reinterpret_cast<uint4*>(ta + out_a + i * M::STRIDE) = h0;
    *reinterpret_cast<uint4*>(ta + out_b + i * M::STRIDE) = h1;
    *reinterpret_cast<uint4*>(tb + out_a + i * M::STRIDE) = l0;
    *reinterpret_cast<uint4*>(tb + out_b + i * M::STRIDE) = l1;
  }
}

// weight tile [rows < BN]: row n scaled by the folded-BatchNorm scale of the epilogue (FOLD), split hi/lo in place
template <int LG, bool FOLD>
__device__ __forceinline__ void fix_w(unsigned char* tile, int ft, int BN, const float* scale, int n0, int N) {
  using M = FixMap<LG>;
  const int cp = ft & ((1 << LG) - 1), r0 = ft >> LG;
  const uint32_t row_off = (uint32_t)((r0 >> 3) * 1024 + (r0 & 7) * 128);
  const int x = r0 & 7;
  const uint32_t in0 = row_off + (((2 * cp) ^ x) << 4), in1 = row_off + (((2 * cp + 1) ^ x) << 4);
  const uint32_t out_hi = row_off + ((cp ^ x) << 4), out_lo = row_off + (((4 + cp) ^ x) << 4);
  float4 va[M::ROWS], vb[M::ROWS];
  float sc[M::ROWS];
#pragma unroll
  for (int i = 0; i < M::ROWS; ++i) {
    const int r = r0 + i * M::RSTEP;
    const bool ok = r < BN;
    va[i] = ok ? *reinterpret_cast<const float4*>(tile + in0 + i * M::STRIDE) : make_float4(0.f, 0.f, 0.f, 0.f);
    vb[i] = ok ? *reinterpret_cast<const float4*>(tile + in1 + i * M::STRIDE) : make_float4(0.f, 0.f, 0.f, 0.f);
    sc[i] = (FOLD && ok && n0 + r < N) ? __ldg(scale + n0 + r) : 0.f;
  }
  __syncwarp();
#pragma unroll
  for (int i = 0; i < M::ROWS; ++i) {
    const int r = r0 + i * M::RSTEP;
    if (r < BN) {
      if (FOLD) {
        va[i].x *= sc[i]; va[i].y *= sc[i]; va[i].z *= sc[i]; va[i].w *= sc[i];
        vb[i].x *= sc[i]; vb[i].y *= sc[i]; vb[i].z *= sc[i]; vb[i].w *= sc[i];
      }
      uint4 h, l;
      split8(va[i], vb[i], h, l);
      *reinterpret_cast<uint4*>(tile + out_hi + i * M::STRIDE) = h;
      *reinterpret_cast<uint4*>(tile + out_lo + i * M::STRIDE) = l;
      if (LG == 1) zero_upper(tile + row_off + i * M::STRIDE, cp, x);
    }
  }
}

// log2 of the 8-element chunk pairs of a k-block that are converted, rounded up to 2 or 4: a K=16 MMA step reads two hi
// chunks, so an odd pair count must still overwrite the (zero-filled) partner chunk -- it holds raw fp32 bits otherwise;
// with 2 pairs the chunks of the second K=16 step are zeroed (zero_upper)
__device__ __forceinline__ int pair_lg(int krem) {
  return krem > 16 ? 2 : 1;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn == nullptr) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(ptr);
  }
  return fn;
}

// [rows, cols] fp32 row-major tensor, box = box_rows x 32 columns (128 bytes), SWIZZLE_128B, zero fill outside
inline int make_map(CUtensorMap* map, const void* ptr, long long rows, int cols, int box_rows) {
  EncodeTiledFn enc = encode_fn();
  if (enc == nullptr) { eat_set_error("pw_tma: cuTensorMapEncodeTiled is not available from this driver"); return EAT_ERR_CUDA; }
  cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t gstride[1] = {(cuuint64_t)cols * 4};
  cuuint32_t box[2] = {32, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(ptr), gdim, gstride, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { eat_set_error("pw_tma: cuTensorMapEncodeTiled failed (pointer / stride alignment?)"); return EAT_ERR_CUDA; }
  return EAT_OK;
}

// [samples, rows, cols] row-major tensor viewed through a {128-byte, box_rows, 1} box, SWIZZLE_128B; elem_bytes 4 (fp32,
// 32 columns per box) or 2 (bf16, 64 columns per box)
inline int make_map3(CUtensorMap* map, const void* ptr, long long samples, long long rows, long long cols, int box_rows,
                     int elem_bytes) {
  EncodeTiledFn enc = encode_fn();
  if (enc == nullptr) { eat_set_error("tma: cuTensorMapEncodeTiled is not available from this driver"); return EAT_ERR_CUDA; }
  cuuint64_t gdim[3] = {(cuuint64_t)cols, (cuuint64_t)rows, (cuuint64_t)samples};
  cuuint64_t gstride[2] = {(cuuint64_t)cols * elem_bytes, (cuuint64_t)rows * cols * elem_bytes};
  cuuint32_t box[3] = {(cuuint32_t)(128 / elem_bytes), (cuuint32_t)box_rows, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(map, elem_bytes == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3,
                   const_cast<void*>(ptr), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { eat_set_error("tma: cuTensorMapEncodeTiled (3-D) failed (pointer / stride alignment?)"); return EAT_ERR_CUDA; }
  return EAT_OK;
}

}  // namespace tma
