// Shared wgmma / mbarrier inline-PTX helpers and operand-staging utilities (sm_90a).
#pragma once
#include "common.cuh"

namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "LAB_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1, %2;\n"     // suspends up to the time hint
      "@P1 bra DONE;\n"
      "bra LAB_WAIT;\n"
      "DONE:\n"
      "}\n" ::"r"(bar), "r"(parity), "r"(0x989680) : "memory");
}
// asynchronous L2 prefetch of a contiguous global range (16-byte aligned, size a multiple of 16): issued by ONE thread
// a few tiles ahead, it turns the register-limited loads of the producer warps into L2 hits
__device__ __forceinline__ void l2_prefetch(const void* p, uint32_t bytes) {
  asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(p), "r"(bytes) : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- Hopper warpgroup MMA (wgmma).  A warpgroup (4 consecutive warps, the first a multiple of 4) issues
// m64nNk16 bf16 x bf16 -> fp32 with both operands read from shared memory through descriptors; the accumulator lives in
// the registers of the 128 threads.  Fragment of thread t (warp w = t / 32, lane l): rows 16 w + l / 4 and 16 w + l / 4 + 8,
// columns 8 j + 2 (l % 4) + {0, 1}; d[4 j + {0, 1}] is the first row, d[4 j + {2, 3}] the second.
// Shared-memory descriptor, SWIZZLE_128B: start >> 4 [0,14), LBO >> 4 [16,30), SBO >> 4 [32,46), layout 1 [62,64).
// K-major: SBO = 1024 (8 rows x 128 B), LBO unused.  MN-major: LBO between 64-element atoms along MN, SBO between
// 8-row groups along K.
__device__ __forceinline__ uint64_t gmma_desc(uint32_t saddr, uint32_t lbo_bytes = 16, uint32_t sbo_bytes = 1024) {
  uint64_t d = (uint64_t)((saddr & 0x3FFFF) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator accesses across an asynchronous MMA
template <int R> __device__ __forceinline__ void wgmma_fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// TA / TB: 0 K-major, 1 MN-major operand
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n16(float (&d)[8], uint64_t da, uint64_t db) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %10, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, %11, %12;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(da), "l"(db), "r"(1), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n32(float (&d)[16], uint64_t da, uint64_t db) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, %19, %20;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(da), "l"(db), "r"(1), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n64(float (&d)[32], uint64_t da, uint64_t db) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(1), "n"(TA), "n"(TB));
}

// m64nNk16 for any N = 8, 16, ..., 128: d[N / 2] is the fragment above with j = 0 .. N / 8 - 1; TA / TB as above (both
// K-major by default).  EAT_WG_S<N> / EAT_WG_O<N> spell out the N / 2 accumulator placeholders and operands; the
// descriptors, the scale-d flag and the two layout immediates follow them as operands N / 2 .. N / 2 + 4.
#define EAT_WG_S8 "%0, %1, %2, %3"
#define EAT_WG_S16 EAT_WG_S8 ", %4, %5, %6, %7"
#define EAT_WG_S24 EAT_WG_S16 ", %8, %9, %10, %11"
#define EAT_WG_S32 EAT_WG_S24 ", %12, %13, %14, %15"
#define EAT_WG_S40 EAT_WG_S32 ", %16, %17, %18, %19"
#define EAT_WG_S48 EAT_WG_S40 ", %20, %21, %22, %23"
#define EAT_WG_S56 EAT_WG_S48 ", %24, %25, %26, %27"
#define EAT_WG_S64 EAT_WG_S56 ", %28, %29, %30, %31"
#define EAT_WG_S72 EAT_WG_S64 ", %32, %33, %34, %35"
#define EAT_WG_S80 EAT_WG_S72 ", %36, %37, %38, %39"
#define EAT_WG_S88 EAT_WG_S80 ", %40, %41, %42, %43"
#define EAT_WG_S96 EAT_WG_S88 ", %44, %45, %46, %47"
#define EAT_WG_S104 EAT_WG_S96 ", %48, %49, %50, %51"
#define EAT_WG_S112 EAT_WG_S104 ", %52, %53, %54, %55"
#define EAT_WG_S120 EAT_WG_S112 ", %56, %57, %58, %59"
#define EAT_WG_S128 EAT_WG_S120 ", %60, %61, %62, %63"
#define EAT_WG_O8 "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
#define EAT_WG_O16 EAT_WG_O8, "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
#define EAT_WG_O24 EAT_WG_O16, "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11])
#define EAT_WG_O32 EAT_WG_O24, "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
#define EAT_WG_O40 EAT_WG_O32, "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19])
#define EAT_WG_O48 EAT_WG_O40, "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
#define EAT_WG_O56 EAT_WG_O48, "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27])
#define EAT_WG_O64 EAT_WG_O56, "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
#define EAT_WG_O72 EAT_WG_O64, "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35])
#define EAT_WG_O80 EAT_WG_O72, "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39])
#define EAT_WG_O88 EAT_WG_O80, "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43])
#define EAT_WG_O96 EAT_WG_O88, "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
#define EAT_WG_O104 EAT_WG_O96, "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51])
#define EAT_WG_O112 EAT_WG_O104, "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55])
#define EAT_WG_O120 EAT_WG_O112, "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59])
#define EAT_WG_O128 EAT_WG_O120, "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
#define EAT_WG_CASE(W, DA, DB, ONE, TAI, TBI)                                                                           \
  if constexpr (N == W)                                                                                                 \
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %" #ONE ", 0;\n"                                                     \
                 "wgmma.mma_async.sync.aligned.m64n" #W "k16.f32.bf16.bf16 {" EAT_WG_S##W "}, %" #DA ", %" #DB ", p, 1, 1, %" #TAI ", %" #TBI ";\n}\n" \
                 : EAT_WG_O##W : "l"(da), "l"(db), "r"(1), "n"(TA), "n"(TB));
template <int N, int TA = 0, int TB = 0>
__device__ __forceinline__ void wgmma_kk(float (&d)[N / 2], uint64_t da, uint64_t db) {
  static_assert(N % 8 == 0 && N >= 8 && N <= 128, "m64nNk16: N is a multiple of 8 up to 128 here");
  EAT_WG_CASE(8, 4, 5, 6, 7, 8) EAT_WG_CASE(16, 8, 9, 10, 11, 12) EAT_WG_CASE(24, 12, 13, 14, 15, 16)
  EAT_WG_CASE(32, 16, 17, 18, 19, 20) EAT_WG_CASE(40, 20, 21, 22, 23, 24) EAT_WG_CASE(48, 24, 25, 26, 27, 28)
  EAT_WG_CASE(56, 28, 29, 30, 31, 32) EAT_WG_CASE(64, 32, 33, 34, 35, 36) EAT_WG_CASE(72, 36, 37, 38, 39, 40)
  EAT_WG_CASE(80, 40, 41, 42, 43, 44) EAT_WG_CASE(88, 44, 45, 46, 47, 48) EAT_WG_CASE(96, 48, 49, 50, 51, 52)
  EAT_WG_CASE(104, 52, 53, 54, 55, 56) EAT_WG_CASE(112, 56, 57, 58, 59, 60) EAT_WG_CASE(120, 60, 61, 62, 63, 64)
  EAT_WG_CASE(128, 64, 65, 66, 67, 68)
}
#undef EAT_WG_CASE

__device__ __forceinline__ uint32_t swz(int row, int chunk) {   // byte offset of a 16-byte chunk in a [rows][128 B] tile
  return (uint32_t)((row >> 3) * 1024 + (row & 7) * 128 + ((chunk ^ (row & 7)) << 4));
}

__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

template <int NP>
__device__ __forceinline__ void store_chunk(unsigned char* hi_tile, unsigned char* lo_tile, uint32_t off, const float (&v)[8]) {
  uint4 h;
  h.x = pack_bf16(v[0], v[1]); h.y = pack_bf16(v[2], v[3]); h.z = pack_bf16(v[4], v[5]); h.w = pack_bf16(v[6], v[7]);
  *reinterpret_cast<uint4*>(hi_tile + off) = h;
  if (NP == 2) {
    float r[8];
    const __nv_bfloat162* hh = reinterpret_cast<const __nv_bfloat162*>(&h);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float2 f = __bfloat1622float2(hh[i]);
      r[2 * i] = v[2 * i] - f.x;
      r[2 * i + 1] = v[2 * i + 1] - f.y;
    }
    uint4 l;
    l.x = pack_bf16(r[0], r[1]); l.y = pack_bf16(r[2], r[3]); l.z = pack_bf16(r[4], r[5]); l.w = pack_bf16(r[6], r[7]);
    *reinterpret_cast<uint4*>(lo_tile + off) = l;
  }
}

template <typename T>
__device__ __forceinline__ void load_chunk(const T* p, float (&v)[8]);
template <>
__device__ __forceinline__ void load_chunk<float>(const float* p, float (&v)[8]) {
  float4 a = __ldg(reinterpret_cast<const float4*>(p)), b = __ldg(reinterpret_cast<const float4*>(p) + 1);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
template <>
__device__ __forceinline__ void load_chunk<__nv_bfloat16>(const __nv_bfloat16* p, float (&v)[8]) {
  uint4 t = __ldg(reinterpret_cast<const uint4*>(p));
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&t);
#pragma unroll
  for (int i = 0; i < 4; ++i) { float2 f = __bfloat1622float2(h[i]); v[2 * i] = f.x; v[2 * i + 1] = f.y; }
}


}  // namespace tc
