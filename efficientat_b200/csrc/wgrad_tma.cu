// Weight gradient of a pointwise (1x1) convolution for fp32 activations as a TMA-fed wgmma GEMM whose reduction runs
// over pixels:     dW[N, K] += G[M, N]^T . xf(X)[M, K]        G: gradient rows (NHWC), X: saved layer input, dW fp32
// (autograd of the 1x1 ConvNormActivation layers, reference models/mn/block_types.py:140-147,167-171, reached from
// ex_audioset.py:197 loss.backward()).  Built like pw_tma.cu.  One of G and X is the "m" operand (64 channels per
// consumer warpgroup, 128 per CTA), the other the "n" operand (BN channels, a multiple of 8 up to 128; the planner puts the
// ragged channel count there):
//
//   warps 0-3 fix-up      : thread 0 issues the loads: per MB-row block of the reduction, cp.async.bulk.tensor lands
//                           [MB rows x 32 channels] fp32 boxes of both operands (up to 4 per operand) in a ring of stages,
//                           S - 1 blocks ahead; rows past M and channels past N / K are zero-filled by the TMA unit.  (A
//                           13th producer warp would put 4 warps on one SM sub-partition and cap every thread at 128
//                           registers; the accumulators of a 64 x 128 dW block need more.)  Then the pair pass of tma_common.cuh (fix_pair): (BatchNorm affine + activation + SE gate on X),
//                           then the boxes of channels c .. c+31 and c+32 .. c+63 become the bf16 hi and the bf16 lo values
//                           of those 64 channels, in the same bytes.  Both operands are "MN-major" for the tensor core (the
//                           reduction index m is the row index), and each box IS a canonical MN-major SWIZZLE_128B atom
//                           column: 8-row groups 1024 B apart (SBO), the n operand's next 64 channels 2 boxes further (LBO).
//   warps 4-11 consumers  : two warpgroups, one per 64 m channels: per 16 reduction rows hi.hi + lo.hi + hi.lo as three
//                           wgmma m64nBNk16 into one register accumulator that holds dW itself (lo.lo ~ 2^-32 is dropped);
//                           added into dW with atomics every kFlushRows rows and at the end.
// Each CTA owns a (128 x BN) tile of dW and one slice of the M range (dW is zeroed by the caller once per step).
// Algorithmic bytes per launch = 4 * (M*N + M*K + N*K).
#include <cstdlib>

#include "tma_common.cuh"

namespace {
using namespace tc;
using namespace tma;

// MB = reduction rows per pipeline stage (template parameter): 64, or 128 for launches with few boxes per stage, where the
// per-block costs (barrier round trips, TMA issue, fix-up prologue) rather than bytes set the pace.
// BOX = MB * 128 bytes: one landed [MB x 32 fp32] box.
constexpr int kMB = 4;                  // m-operand boxes per stage at most: 2 pairs = 128 channels, one per warpgroup
constexpr int kThreads = 384;
constexpr int kFirstCons = 4;
// The register accumulators are flushed to dW (and restarted) every kFlushRows reduction rows: the tensor core's fp32
// accumulation rounds toward zero, so a long split with same-signed terms drifts by ~1.5 x 2^-24 of the sum per 16-row
// step; over 31k rows (mn10 block 2 at B = 256) that was 1.5e-4 of sum |terms|, within 30x of a dropped 128-row block.
constexpr int kFlushRows = 4096;

struct WgParams {
  float* dW;
  int M, N, K;
  int xm;                               // 1: X is the m operand (dW^T is accumulated), 0: G is
  int m_dim, n_dim, bn;                 // channels of the m / n operand, n tile width
  int m_tiles, n_tiles, mbs, nbs;       // tiles; boxes reserved per stage for the m / n operand
  int rows_per_split, sample_rows, splits_per_sample;
  int stages;
  uint32_t stage_bytes, off_f, off_bar;
  const float* in_scale; const float* in_shift; const float* gate; int in_act; int rps;
};

template <int XACT, int MB, int BN>
__global__ void __launch_bounds__(kThreads, 1)
wgrad_tma_kernel(const __grid_constant__ CUtensorMap mapM, const __grid_constant__ CUtensorMap mapN, const WgParams p) {
  constexpr int BOX = MB * 128;
  extern __shared__ __align__(1024) unsigned char smem[];
  float* s_isc = reinterpret_cast<float*>(smem + p.off_f);          // [128] in-transform scale of this CTA's X channels
  float* s_ish = s_isc + 128;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + p.off_bar);
  const int S = p.stages;
  const uint32_t bar_full = smem_u32(bars), bar_ready = bar_full + 8 * S, bar_empty = bar_ready + 8 * S;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles = p.m_tiles * p.n_tiles;
  const int ot = blockIdx.x % tiles, split = blockIdx.x / tiles;
  const int mt = ot / p.n_tiles, nt = ot - mt * p.n_tiles;
  const int m0 = mt * (kMB * KB), n0 = nt * BN;
  const int x0 = p.xm ? m0 : n0;                                     // first X channel of this CTA
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
  // boxes of this CTA that hold real channels (only those are loaded); gm: warpgroups with m channels
  const int mb = min(p.mbs, (p.m_dim - m0 + KB - 1) / KB);
  const int nb = min(p.nbs, (min(BN, p.n_dim - n0) + KB - 1) / KB);
  const int gm = (mb + 1) >> 1;
  const uint32_t n_off = (uint32_t)p.mbs * BOX;
  const uint32_t stage_base = smem_u32(smem);

  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) { mbar_init(bar_full + 8 * s, 1); mbar_init(bar_ready + 8 * s, 4); mbar_init(bar_empty + 8 * s, 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&mapM)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&mapN)) : "memory");
  }
  if (XACT >= 0) {
    for (int i = threadIdx.x; i < 128; i += kThreads) {
      s_isc[i] = x0 + i < p.K ? p.in_scale[x0 + i] : 0.f;          // zero beyond K: act(0) = 0
      s_ish[i] = x0 + i < p.K ? p.in_shift[x0 + i] : 0.f;
    }
  }
  __syncthreads();

  if (warp < kFirstCons) {
    // ================================================================= fix-up warps (128 threads); thread 0 also issues
    // the TMA loads: block b goes to stage b % S once the consumers have released that stage's previous block
    const int ft = threadIdx.x;
    auto issue = [&](int b) {
      const int sb = b % S;
      const int m = (int)(m_begin + (long long)b * MB);
      mbar_wait(bar_empty + 8 * sb, ((uint32_t)(b / S) & 1u) ^ 1u);
      const uint32_t dst = stage_base + (uint32_t)sb * p.stage_bytes;
      mbar_expect_tx(bar_full + 8 * sb, (uint32_t)(mb + nb) * BOX);
      for (int i = 0; i < mb; ++i) tma_load_2d(&mapM, bar_full + 8 * sb, dst + i * BOX, m0 + i * KB, m);
      for (int i = 0; i < nb; ++i) tma_load_2d(&mapN, bar_full + 8 * sb, dst + n_off + i * BOX, n0 + i * KB, m);
    };
    if (ft == 0)
      for (int b = 0; b < min(S - 1, n_blocks); ++b) issue(b);
    const int kc = (ft & 3) * 8;                                   // channel of this thread's chunk pair inside a box
    int s = 0;
    uint32_t ph = 0;
    for (int blk = 0; blk < n_blocks; ++blk) {
      const long long mbeg = m_begin + (long long)blk * MB;
      const int rows_valid = (int)min((long long)MB, m_end - mbeg);
      int b0 = 0, off0 = 0;
      if (p.gate != nullptr) { b0 = (int)(mbeg / p.rps); off0 = (int)(mbeg - (long long)b0 * p.rps); }
      mbar_wait(bar_full + 8 * s, ph);
      unsigned char* st = smem + (size_t)s * p.stage_bytes;
      // the X boxes get the input transform, the gradient boxes only the split (rows past the split zeroed in both)
      for (int b = 0; b < mb; b += 2) {
        unsigned char* t = st + b * BOX;
        if (p.xm) fix_pair<XACT, MB>(t, t + BOX, b + 1 < mb, ft, rows_valid, s_isc - x0, s_ish - x0, m0 + b * KB + kc, p.gate, off0, b0, p.rps, p.K);
        else fix_pair<-1, MB>(t, t + BOX, b + 1 < mb, ft, rows_valid, nullptr, nullptr, 0, nullptr, 0, 0, 1, 0);
      }
      for (int b = 0; b < nb; b += 2) {
        unsigned char* t = st + n_off + b * BOX;
        if (p.xm) fix_pair<-1, MB>(t, t + BOX, b + 1 < nb, ft, rows_valid, nullptr, nullptr, 0, nullptr, 0, 0, 1, 0);
        else fix_pair<XACT, MB>(t, t + BOX, b + 1 < nb, ft, rows_valid, s_isc - x0, s_ish - x0, n0 + b * KB + kc, p.gate, off0, b0, p.rps, p.K);
      }
      fence_proxy_async();
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_ready + 8 * s);
      if (++s == S) { s = 0; ph ^= 1u; }
      // S - 1 blocks ahead: the stage of block blk - 1, whose MMAs ran while this block was fixed up
      if (ft == 0 && blk + S - 1 < n_blocks) issue(blk + S - 1);
    }
  } else {
    // ================================================================= consumers: MMA, the atomics every kFlushRows rows
    const int cw = warp - kFirstCons;
    const int g = cw >> 2, wq = cw & 3;                        // m pair of this warpgroup, warp inside it
    const int ctid = threadIdx.x - kFirstCons * 32;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    // accumulator rows of this thread: m channels m0 + 64 g + 16 wq + lane / 4 (+ 8); columns n0 + 8 j + 2 (lane % 4) (+ 1)
    auto flush = [&]() {
      if (g < gm) {
        const int c0 = 2 * (lane & 3);
        const int lim = p.n_dim - n0 - c0;                           // columns 8 j + c0 (+ 1) exist while 8 j < lim
        const bool odd = (lane >> 2) & 1;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int mi = m0 + 64 * g + 16 * wq + (lane >> 2) + 8 * h;
          if (p.xm) {
            // dW[n][m]: lanes l and l ^ 4 hold rows mi and mi ^ 1 (mi even in the even lane) of the same two columns;
            // one exchange gives the even lane column n's pair of rows, the odd lane column n + 1's, as float2
            const int me = mi & ~1;
            float2* q = reinterpret_cast<float2*>(dWout + (size_t)(n0 + c0 + (odd ? 1 : 0)) * p.K + me);
            const size_t step = (size_t)4 * p.K;                     // 8 columns, in float2
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
              const float vx = acc[4 * j + 2 * h], vy = acc[4 * j + 2 * h + 1];
              const float r = __shfl_xor_sync(0xffffffffu, odd ? vx : vy, 4);
              if (8 * j < lim && me < p.m_dim) atomicAdd(q + j * step, odd ? make_float2(r, vy) : make_float2(vx, r));
            }
          } else if (mi < p.m_dim) {                                  // dW[mi][n0 + 8 j + c0 (+ 1)]
            float2* q = reinterpret_cast<float2*>(dWout + (size_t)mi * p.K + n0 + c0);
#pragma unroll
            for (int j = 0; j < BN / 8; ++j)
              if (8 * j < lim) atomicAdd(q + 4 * j, make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]));
          }
        }
      }
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    };
    int s = 0;
    uint32_t ph = 0;
    for (int blk = 0; blk < n_blocks; ++blk) {
      mbar_wait(bar_ready + 8 * s, ph);
      const uint32_t sm = stage_base + (uint32_t)s * p.stage_bytes + (uint32_t)(2 * g) * BOX, sn = stage_base + (uint32_t)s * p.stage_bytes + n_off;
      if (g < gm) {
        wgmma_fence();
#pragma unroll
        for (int st = 0; st < MB / 16; ++st) {                      // 16 reduction rows = two 8-row groups = 2048 bytes
          const uint64_t ah = gmma_desc(sm + st * 2048, BOX, 1024), al = gmma_desc(sm + BOX + st * 2048, BOX, 1024);
          const uint64_t bh = gmma_desc(sn + st * 2048, 2 * BOX, 1024), bl = gmma_desc(sn + BOX + st * 2048, 2 * BOX, 1024);
          wgmma_kk<BN, 1, 1>(acc, ah, bh);
          wgmma_kk<BN, 1, 1>(acc, al, bh);
          wgmma_kk<BN, 1, 1>(acc, ah, bl);
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(acc);
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

// padded tensor work of one orientation: m channels in 64-channel warpgroup tiles, n channels in the planner's BN tiles
long long wg_cost(int m_dim, int n_dim) {
  const int nt = ceil_div(n_dim, 128);
  return (long long)ceil_div(m_dim, 64) * 64 * nt * (ceil_div(ceil_div(n_dim, nt), 8) * 8);
}

// The launch plan (fills the orientation / tiling / split / stage fields of p) -> MB and the number of reduction splits.
// sms: the GPU's SM count.  The operand whose channel count pads less as n tile goes on the n side (ties: X, so that
// the flush adds float2 pairs along dW rows).  128-row blocks when the stage holds one pair of each operand (m and n
// channels <= 64) and the reduction is long: the first layers of the network, M in the millions.
int plan_wg(WgParams& p, int sms, int& mb, int& splits) {
  p.xm = wg_cost(p.K, p.N) < wg_cost(p.N, p.K) ? 1 : 0;
  p.m_dim = p.xm ? p.K : p.N;
  p.n_dim = p.xm ? p.N : p.K;
  p.m_tiles = ceil_div(p.m_dim, kMB * KB);
  p.n_tiles = ceil_div(p.n_dim, 128);
  p.bn = ceil_div(ceil_div(p.n_dim, p.n_tiles), 8) * 8;
  p.mbs = p.m_dim <= 2 * KB ? 2 : kMB;
  p.nbs = p.bn <= 2 * KB ? 2 : 4;
  const int boxes = p.mbs + p.nbs;
  mb = (boxes <= 4 && p.sample_rows == 0 && p.M >= (1 << 20)) ? 128 : 64;
  if (const char* e = getenv("EAT_WG_MB")) { const int v = atoi(e); if (v == 64 || (v == 128 && boxes <= 4)) mb = v; }
  const int tiles = p.m_tiles * p.n_tiles;
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
  const size_t misc = 2 * 128 * 4 + 3 * 8 * 8 + 16 + 1024;
  p.stages = (int)((budget - misc) / p.stage_bytes);
  if (p.stages > 8) p.stages = 8;
  if (p.stages < 2) { eat_set_error("wgrad_tma: shared-memory budget exceeded"); return EAT_ERR_UNSUPPORTED; }
  return EAT_OK;
}

template <int XACT, int MB, int BN>
int launch_wg_bn(const float* G, const float* X, const WgParams& p, int splits, cudaStream_t st) {
  const size_t budget = 227 * 1024;
  size_t off = (size_t)p.stages * p.stage_bytes;
  const uint32_t off_f = (uint32_t)off; off += 2 * 128 * 4;
  const uint32_t off_bar = (uint32_t)off; off += 3 * (size_t)p.stages * 8 + 16;
  const size_t smem = off;
  WgParams q = p;
  q.off_f = off_f; q.off_bar = off_bar;
  CUtensorMap mM, mN;
  if (int rc = make_map(&mM, p.xm ? X : G, p.M, p.m_dim, MB)) return rc;
  if (int rc = make_map(&mN, p.xm ? G : X, p.M, p.n_dim, MB)) return rc;
  static unsigned long long attr_mask = 0;
  if (int rc = eat_opt_in_smem(wgrad_tma_kernel<XACT, MB, BN>, budget, attr_mask)) return rc;
  wgrad_tma_kernel<XACT, MB, BN><<<p.m_tiles * p.n_tiles * splits, kThreads, smem, st>>>(mM, mN, q);
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

// n tile widths: every multiple of 8 up to 128 at 64-row blocks; 128-row blocks only run n tiles of <= 64 channels
template <int XACT, int MB, int BN = 8>
int launch_wg_mb(const float* G, const float* X, const WgParams& p, int splits, cudaStream_t st) {
  if constexpr (BN > (MB == 128 ? 64 : 128)) {
    eat_set_error("wgrad_tma: no instance for this n tile width");
    return EAT_ERR_UNSUPPORTED;
  } else {
    if (p.bn == BN) return launch_wg_bn<XACT, MB, BN>(G, X, p, splits, st);
    return launch_wg_mb<XACT, MB, BN + 8>(G, X, p, splits, st);
  }
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
  plan[0] = mb; plan[1] = p.m_tiles * p.n_tiles; plan[2] = splits; plan[3] = p.rows_per_split;
  plan[4] = p.splits_per_sample; plan[5] = p.stages;
  return EAT_OK;
}
