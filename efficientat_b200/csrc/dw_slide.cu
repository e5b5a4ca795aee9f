// Depthwise k x k convolution as a register sliding window (sm_90a).
//
// Replaces the depthwise ConvNormActivation of the reference's InvertedResidual / DY_Block
// (models/mn/block_types.py:155-165, models/dymn/dy_block.py:255-262) for forward (training and eval) and,
// with mirrored taps, the stride-1 data gradient.
//
// One thread owns one 16-byte channel vector and a strip of P output columns, and walks DOWN the rows of its
// segment: each input row (NIN = (P-1)*S + K vectors) is loaded and BatchNorm+activation-transformed exactly once,
// then scattered into the L = ceil(K/S) output rows it contributes to, which live in registers.  When an output
// row has received its last kernel row it runs the epilogue, is stored, and the window shifts by one slot.
// Compared with the per-output-row strip kernel (conv_kernels.cu: dw_kernel) this removes the K-fold reload and
// re-transform of every input row, all per-load bounds checks (the column mask of a strip is loop invariant and
// rows outside the image are skipped whole) and most address arithmetic: ~4x fewer instructions per output.
// No shared-memory staging of activations and no CTA barriers in the main loop; weights sit in shared memory.
//
// Algorithmic bytes: B*F*T*C + B*Fo*To*C elements (+ residual in the data-gradient mode), HBM bound.
#include <cstdio>
#include <cstdlib>
#include <type_traits>

#include "common.cuh"

namespace {

constexpr int kST = 128;        // threads per CTA
constexpr int kChMax = 512;     // channels per CTA (bounds the shared-memory weight table: 25 * 512 * 4 B = 50 KB)

// c += a * b over a channel vector (H100 has no packed fp32 FMA: one fmaf per channel)
template <int V>
__device__ __forceinline__ void fma_vec(const float (&a)[V], const float (&b)[V], float (&c)[V]) {
#pragma unroll
  for (int i = 0; i < V; ++i) c[i] = fmaf(a[i], b[i], c[i]);
}

template <int XACT>
__device__ __forceinline__ float xact(float v) {
  if (XACT == EAT_ACT_RELU) return fmaxf(v, 0.f);
  if (XACT == EAT_ACT_HSWISH) return v * fminf(fmaxf(v + 3.f, 0.f), 6.f) * (1.f / 6.f);
  return v;
}


// Per-thread prefetch ring (cp.async): a thread's loads of the NEXT `depth` input rows are in flight while it multiplies
// the current one.  Each thread reads back only what it copied itself, so cp.async.wait_group is the only synchronisation
// (no CTA barrier); slot layout [depth][vectors][thread] keeps both the copies and the read-back conflict-free.
template <int BYTES>
__device__ __forceinline__ void cp_async(uint32_t dst, const void* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], %2;" ::"r"(dst), "l"(src), "n"(BYTES) : "memory");
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_wait_pending(int n) {      // n = depth - 1 groups may stay in flight
  switch (n) {
    case 0: asm volatile("cp.async.wait_group 0;" ::: "memory"); break;
    case 1: asm volatile("cp.async.wait_group 1;" ::: "memory"); break;
    case 2: asm volatile("cp.async.wait_group 2;" ::: "memory"); break;
    case 3: asm volatile("cp.async.wait_group 3;" ::: "memory"); break;
    case 4: asm volatile("cp.async.wait_group 4;" ::: "memory"); break;
    default: asm volatile("cp.async.wait_group 5;" ::: "memory"); break;
  }
}
constexpr int kRingMax = 6;
// ring depth (<= maxd) that fits `budget` bytes of shared memory next to `fixed` bytes of tables; 0: ring off.
// Measured (profiles/r02_dw_ring_microbench_b256.txt): two rows ahead is the sweet spot -- deeper rings take shared memory
// away from the L1 that serves the column halo of neighbouring strips, and any ring that costs a resident CTA loses.
inline int ring_depth(size_t budget, size_t fixed, size_t slot_bytes, int maxd) {
  if (const char* e = getenv("EAT_DW_RING")) { const int v = atoi(e); if (v <= 0) return 0; if (v <= kRingMax) { return (fixed + v * slot_bytes <= 200 * 1024) ? v : 0; } }
  if (maxd < 2 || budget <= fixed) return 0;
  const size_t d = (budget - fixed) / slot_bytes;
  return d >= 2 ? (int)(d > (size_t)maxd ? (size_t)maxd : d) : 0;
}

struct SlideArgs {
  const void* in;
  const float* wt;
  void* out;
  int F, Tn, Fo, To, C;
  int B;
  int cvc;          // channel vectors per CTA chunk
  int chunks;       // channel chunks (gridDim.x = chunks * groups)
  int seg_rows;     // output rows per segment
  int per_sample;   // 1: blockIdx.y is the sample (per-sample weights / pooling / DyMN epilogue); 0: CTAs stride over samples
  int depth;        // prefetch ring depth in rows (RING kernels)
  const float* xscale;
  const float* xshift;
  const float* scale;
  const float* shift;
  int act;
  const void* res;
  int flip;
  float* pool;
  double* stat_sum;
  double* stat_sq;
  DyEpi dy;
};

// MODE 0: training forward (optional input BN+act XACT >= 0, raw output + batch statistics)
// MODE 1: eval forward (folded BN + act epilogue, SE pooling, DyMN DyReLU-B / coordinate attention)
// MODE 2: stride-1 data gradient (mirrored taps, optional residual-gradient add)
// D = 2: dilation 2 at stride 1.  Such a layer is four independent undilated K x K convolutions, one on each (row parity,
// column parity) sub-grid of the image, so a unit walks rows and columns of one parity: the same walk with row and column
// steps of two pixels.  Each sample has D * D times the units of one sub-grid; D = 1 is the undilated kernel.
// DM: DyReLU-B pieces of the MODE 1 DyMN epilogue.  DM = 2 is the four-register form; 1, 3 and 4 hold 2 DM coefficients
// per channel in registers (DyCoef, common.cuh).
template <typename T, int K, int S, int P, int MODE, int XACT, int MINB, bool RING, int D = 1, int DM = 2>
__global__ void __launch_bounds__(kST, MINB) dw_slide_kernel(const SlideArgs a) {
  static_assert(D == 1 || (D == 2 && S == 1), "dilation 2 is stride 1 only");
  static_assert(DM >= 1 && DM <= 4 && (DM == 2 || (MODE == 1 && D == 1)), "DyReLU-B pieces: 1..4, eval epilogue only");
  constexpr int V = Vec<T>::N;
  constexpr int NIN = (P - 1) * S + K, PAD = (K - 1) / 2, KK = K * K;
  constexpr int L = (K + S - 1) / S;           // output rows alive at once
  constexpr bool kAff = MODE == 1, kStats = MODE == 0, kRes = MODE == 2, kDy = MODE == 1, kPool = MODE == 1;
  constexpr bool kXf = MODE == 0 && XACT >= 0;
  extern __shared__ __align__(16) float smem[];
  const int F = a.F, Tn = a.Tn, Fo = a.Fo, To = a.To, C = a.C;
  const int chunk = blockIdx.x % a.chunks, grp = blockIdx.x / a.chunks, groups = gridDim.x / a.chunks;
  const int cv = C / V;
  const int cv0 = chunk * a.cvc;
  const int ncv = min(a.cvc, cv - cv0);       // channel vectors of this CTA
  const int cc = ncv * V;                      // channels of this CTA
  float* s_w = smem;                           // [KK][cc]
  float* s_sum = s_w + KK * a.cvc * V;         // [cc]
  float* s_sq = s_sum + a.cvc * V;             // [cc]
  const int b = blockIdx.y;
  const int tid = threadIdx.x;
  // prefetch ring: [depth][NIN][kST] 16-byte vectors behind the tables
  const uint32_t ring0 = (uint32_t)__cvta_generic_to_shared(s_sq + a.cvc * V) + (uint32_t)tid * 16u;
  const unsigned char* ringp = reinterpret_cast<const unsigned char*>(s_sq + a.cvc * V) + tid * 16;
  {
    const float* wsrc = a.wt + (size_t)b * a.dy.wt_bstride + (size_t)cv0 * V;
    for (int i = tid; i < KK * cc; i += kST) {
      const int tap = i / cc, c = i - tap * cc;
      s_w[i] = __ldg(wsrc + (size_t)(a.flip ? KK - 1 - tap : tap) * C + c);
    }
    for (int i = tid; i < 2 * a.cvc * V; i += kST) s_sum[i] = 0.f;
  }
  __syncthreads();
  const bool need_red = (kPool && a.pool != nullptr) || (kStats && a.stat_sum != nullptr);
  const int ppb = kST / ncv;
  const int cvl = tid % ncv, slot = tid / ncv;
  if (slot < ppb) {
    const int c0 = (cv0 + cvl) * V;
    const float* wl = s_w + cvl * V;

    float isc[V], ish[V];
    if (kXf) {
#pragma unroll
      for (int i = 0; i < V; ++i) { isc[i] = __ldg(a.xscale + c0 + i); ish[i] = __ldg(a.xshift + c0 + i); }
    }
    float osc[V], osh[V];
    if (kAff && a.scale != nullptr) {
#pragma unroll
      for (int i = 0; i < V; ++i) { osc[i] = __ldg(a.scale + c0 + i); osh[i] = __ldg(a.shift + c0 + i); }
    }
    float da1[V], da2[V], db1[V], db2[V];
    DyCoef<DM> dyc[V];
    if (kDy && a.dy.theta != nullptr) {
      if constexpr (DM == 2) {
        const float* th = a.dy.theta + ((size_t)b * C + c0) * 4;
#pragma unroll
        for (int i = 0; i < V; ++i) {
          const float4 t4 = __ldg(reinterpret_cast<const float4*>(th) + i);
          da1[i] = (2.f * t4.x - 1.f) * a.dy.lam[0] + a.dy.init[0];
          da2[i] = (2.f * t4.y - 1.f) * a.dy.lam[1] + a.dy.init[1];
          db1[i] = (2.f * t4.z - 1.f) * a.dy.lam[2] + a.dy.init[2];
          db2[i] = (2.f * t4.w - 1.f) * a.dy.lam[3] + a.dy.init[3];
        }
      } else {
#pragma unroll
        for (int i = 0; i < V; ++i) dyc[i].load(a.dy.theta + ((size_t)b * C + c0 + i) * (2 * DM), a.dy.lam, a.dy.init);
      }
    }
    float lsum[V], lsq[V];
#pragma unroll
    for (int i = 0; i < V; ++i) { lsum[i] = 0.f; lsq[i] = 0.f; }
    int bb = b;                                  // sample of the current unit
    const T* inb = nullptr;
    T* outb = nullptr;
    const T* resb = nullptr;
    // D = 2: strips and segments of the largest sub-grid, ceil(Fo / 2) x ceil(To / 2)
    const int strips = ceil_div(D == 1 ? To : (To + 1) / 2, P), segs = ceil_div(D == 1 ? Fo : (Fo + 1) / 2, a.seg_rows);
    const int units = D * D * strips * segs;
    const long long rowstride = (long long)Tn * C * D;
    const int cstep = C * D;                     // elements between the columns a unit reads
    int Fs = Fo, Ts = To;                        // rows / columns of the unit's sub-grid (D = 1: the image)

    // epilogue of one finished output row (P vectors), then the row is stored
    auto finish = [&](float (&o)[P][V], int fo, int to0) {
#pragma unroll
      for (int p = 0; p < P; ++p) {
        const int to = to0 + p;
        if (to < Ts) {
          if (kAff && a.scale != nullptr) {
#pragma unroll
            for (int i = 0; i < V; ++i) { o[p][i] = act_fwd(fmaf(o[p][i], osc[i], osh[i]), a.act); lsum[i] += o[p][i]; }
          } else if (kStats) {
#pragma unroll
            for (int i = 0; i < V; ++i) { lsum[i] += o[p][i]; lsq[i] = fmaf(o[p][i], o[p][i], lsq[i]); }
          }
          if (kDy && a.dy.theta != nullptr) {
            if constexpr (DM == 2) {
#pragma unroll
              for (int i = 0; i < V; ++i) o[p][i] = fmaxf(fmaf(o[p][i], da1[i], db1[i]), fmaf(o[p][i], da2[i], db2[i]));
            } else {
#pragma unroll
              for (int i = 0; i < V; ++i) o[p][i] = dyc[i].apply(o[p][i]);
            }
          }
          if (kDy && a.dy.ca_f != nullptr) {
            const float* cf = a.dy.ca_f + ((size_t)bb * Fo + fo) * C + c0;
            const float* ct = a.dy.ca_t + ((size_t)bb * To + to) * C + c0;
#pragma unroll
            for (int q = 0; q < V / 4; ++q) {
              const float4 f4 = __ldg(reinterpret_cast<const float4*>(cf) + q), t4 = __ldg(reinterpret_cast<const float4*>(ct) + q);
              o[p][4 * q] *= f4.x * t4.x; o[p][4 * q + 1] *= f4.y * t4.y;
              o[p][4 * q + 2] *= f4.z * t4.z; o[p][4 * q + 3] *= f4.w * t4.w;
            }
          }
          const size_t off = D == 1 ? ((size_t)fo * To + to) * C : ((size_t)(D * fo) * To + D * to) * C;
          if (kRes && resb != nullptr) {
            float r[V];
            Vec<T>::load(resb + off, r);
#pragma unroll
            for (int i = 0; i < V; ++i) o[p][i] += r[i];
          }
          Vec<T>::store(outb + off, o[p]);
        }
      }
    };

    // flat (sample, unit) index space; a thread strides over it so every thread gets the same number of units +-1
    long long g = a.per_sample ? (long long)b * units + grp * ppb + slot : ((long long)blockIdx.y * groups + grp) * ppb + slot;
    const long long gend = a.per_sample ? (long long)(b + 1) * units : (long long)a.B * units;
    const long long gstep = a.per_sample ? (long long)groups * ppb : (long long)gridDim.y * groups * ppb;
    for (; g < gend; g += gstep) {
      bb = (int)(g / units);
      int u = (int)(g - (long long)bb * units);
      inb = reinterpret_cast<const T*>(a.in) + (size_t)bb * F * Tn * C + c0;
      outb = reinterpret_cast<T*>(a.out) + (size_t)bb * Fo * To * C + c0;
      if (kRes && a.res != nullptr) resb = reinterpret_cast<const T*>(a.res) + (size_t)bb * Fo * To * C + c0;
      if constexpr (D == 2) {                               // sub-grid (pr, pc): image rows pr, pr+2, .. and columns pc, pc+2, ..
        const int par = u / (strips * segs), pr = par >> 1, pc = par & 1;
        u -= par * strips * segs;
        Fs = (Fo - pr + 1) >> 1;
        Ts = (To - pc + 1) >> 1;
        const size_t poff = ((size_t)pr * To + pc) * C;    // stride 1: input and output share the pixel grid
        inb += poff;
        outb += poff;
        if (kRes && a.res != nullptr) resb += poff;
      }
      const int seg = u / strips, strip = u - seg * strips;
      const int fo_a = seg * a.seg_rows;
      const int nrows = min(a.seg_rows, Fs - fo_a);
      const int to0 = strip * P;
      if (D == 2 && (nrows <= 0 || to0 >= Ts)) continue;    // past the end of a smaller sub-grid
      const int t0 = to0 * S - PAD;
      const int Fin = D == 1 ? F : Fs, Tin = D == 1 ? Tn : Ts;
      unsigned cmask = 0;
#pragma unroll
      for (int j = 0; j < NIN; ++j) cmask |= (t0 + j >= 0 && t0 + j < Tin) ? (1u << j) : 0u;
      const int i0 = fo_a * S - PAD;                        // input row of step 0
      const T* colp = inb + (long long)t0 * cstep;          // column j of input row i: colp + i*rowstride + j*cstep
      float acc[L][P][V];
#pragma unroll
      for (int l = 0; l < L; ++l)
#pragma unroll
        for (int p = 0; p < P; ++p)
#pragma unroll
          for (int i = 0; i < V; ++i) acc[l][p][i] = 0.f;

      // ring: feed q of this unit reads input row i0 + q (S = 2: even rows are the Ph0 feeds, odd rows the Ph1 feeds)
      const int steps = nrows + L - 1;
      const int nfeed = S == 1 ? steps : 2 * steps - 1;
      int rs = 0;                                             // ring slot of the next feed
      auto issue = [&](int q, int slot_) {
        if (RING) {
          const int irow = i0 + q;
          if (q < nfeed && irow >= 0 && irow < Fin) {
            const T* rp = colp + (long long)irow * rowstride;
            const uint32_t dst = ring0 + (uint32_t)(slot_ * NIN) * (kST * 16u);
#pragma unroll
            for (int j = 0; j < NIN; ++j)
              if ((cmask >> j) & 1u) cp_async<16>(dst + (uint32_t)j * (kST * 16u), rp + (size_t)j * cstep);
          }
          cp_commit();
        }
      };
      if (RING) {
        for (int q = 0; q < a.depth; ++q) issue(q, q);
      }
      int fq = 0;                                             // feeds consumed so far
      // one input row: load, transform once, scatter into the live output rows.  PH = row parity for S = 2.
      auto feed_row = [&](int irow, auto ph_tag) {
        constexpr int PH = decltype(ph_tag)::value;
        if (irow < 0 || irow >= Fin) return;
        const T* rp = colp + (long long)irow * rowstride;
        float v[NIN][V];
#pragma unroll
        for (int j = 0; j < NIN; ++j) {
          if ((cmask >> j) & 1u) {
            if (RING) Vec<T>::load(reinterpret_cast<const T*>(ringp + (size_t)(rs * NIN + j) * (kST * 16)), v[j]);
            else Vec<T>::load(rp + (size_t)j * cstep, v[j]);
          } else {
#pragma unroll
            for (int i = 0; i < V; ++i) v[j][i] = 0.f;
          }
        }
        if (kXf) {
#pragma unroll
          for (int j = 0; j < NIN; ++j) {
            const bool ok = (cmask >> j) & 1u;
#pragma unroll
            for (int i = 0; i < V; ++i) {
              const float tv = xact<XACT>(fmaf(v[j][i], isc[i], ish[i]));
              v[j][i] = ok ? tv : 0.f;                      // zero padding applies to the activated tensor
            }
          }
        }
#pragma unroll
        for (int ky = 0; ky < K; ++ky) {
          if ((ky % S) != PH) continue;
          // slot of the output row this kernel row feeds (see the loop below)
          const int sl = (S == 1) ? (K - 1 - ky) : (PH == 0 ? (L - 1 - ky / 2) : (L - 2 - (ky - 1) / 2));
          float w[K][V];
#pragma unroll
          for (int kx = 0; kx < K; ++kx) {
#pragma unroll
            for (int q = 0; q < V / 4; ++q) {
              const float4 t4 = *reinterpret_cast<const float4*>(wl + (ky * K + kx) * cc + 4 * q);
              w[kx][4 * q] = t4.x; w[kx][4 * q + 1] = t4.y; w[kx][4 * q + 2] = t4.z; w[kx][4 * q + 3] = t4.w;
            }
          }
#pragma unroll
          for (int ix = 0; ix < NIN; ++ix) {
#pragma unroll
            for (int p = 0; p < P; ++p) {
              const int kx = ix - p * S;
              if (kx >= 0 && kx < K) {
                fma_vec<V>(v[ix], w[kx], acc[sl][p]);
              }
            }
          }
        }
      };
      auto feed = [&](int irow, auto ph_tag) {
        if (RING) cp_wait_pending(a.depth - 1);               // this feed's row has landed (own copies only)
        feed_row(irow, ph_tag);
        if (RING) {                                           // the slot just consumed takes the row `depth` feeds ahead
          issue(fq + a.depth, rs);
          ++fq;
          if (++rs == a.depth) rs = 0;
        }
      };
      using Ph0 = std::integral_constant<int, 0>;
      using Ph1 = std::integral_constant<int, 1>;

      // step n: before the shift, slot j holds output row  n - (L-1) + j  (relative to fo_a).
      //   S = 1: input row i0 + n, kernel row ky feeds slot K-1-ky; slot 0 is complete afterwards.
      //   S = 2: input row i0 + 2n (even kernel rows) completes slot 0; after the shift row i0 + 2n + 1 feeds
      //          the odd kernel rows.
      for (int n = 0; n < steps; ++n) {
        feed(i0 + n * S, Ph0{});
        const int orel = n - (L - 1);
        if (orel >= 0) finish(acc[0], fo_a + orel, to0);
#pragma unroll
        for (int l = 0; l + 1 < L; ++l)
#pragma unroll
          for (int p = 0; p < P; ++p)
#pragma unroll
            for (int i = 0; i < V; ++i) acc[l][p][i] = acc[l + 1][p][i];
#pragma unroll
        for (int p = 0; p < P; ++p)
#pragma unroll
          for (int i = 0; i < V; ++i) acc[L - 1][p][i] = 0.f;
        if (S == 2 && n + 1 < steps) feed(i0 + 2 * n + 1, Ph1{});   // the last odd row only feeds rows past the segment
      }
    }
    if (need_red) {
#pragma unroll
      for (int i = 0; i < V; ++i) atomicAdd(&s_sum[cvl * V + i], lsum[i]);
      if (kStats) {
#pragma unroll
        for (int i = 0; i < V; ++i) atomicAdd(&s_sq[cvl * V + i], lsq[i]);
      }
    }
  }
  if (need_red) {
    __syncthreads();
    for (int c = tid; c < cc; c += kST) {
      const int cg = cv0 * V + c;
      if (kPool && a.pool != nullptr) atomicAdd(a.pool + (size_t)b * C + cg, s_sum[c]);
      if (kStats && a.stat_sum != nullptr) { atomicAdd(a.stat_sum + cg, (double)s_sum[c]); atomicAdd(a.stat_sq + cg, (double)s_sq[c]); }
    }
  }
}


// Grid plan shared by the forward and weight-gradient kernels.  All CTAs are resident at once (ctas_per_sm per SM),
// every thread walks its share of the flat (sample, unit) space.  The segment length trades the K-S halo rows
// re-read at each segment start against the rounding loss of "ceil(units per thread)": both are evaluated for every
// candidate length and the cheapest wins.
struct SlidePlan { int chunks, cvc, seg_rows, groups, gy; };

// grids: independent sub-grids of Fo x To per sample (4 for a dilation-2 layer, see dw_slide_kernel)
inline SlidePlan plan_slide(int B, int Fo, int To, int cv, int V, int P, int S, int K, int ctas_per_sm, bool per_sample,
                            int cvc_cap = kST, int grids = 1) {
  SlidePlan pl;
  const int cvc_max = min(kChMax / V < kST ? kChMax / V : kST, cvc_cap);
  pl.chunks = ceil_div(cv, cvc_max);
  pl.cvc = ceil_div(cv, pl.chunks);
  const int ppb = kST / pl.cvc > 0 ? kST / pl.cvc : 1;
  const int strips = ceil_div(To, P);
  const long long ctas = (long long)kNumSMs * ctas_per_sm;
  // CTAs available to one channel chunk (per sample when blockIdx.y must be the sample)
  const long long lanes = per_sample ? max(1LL, ctas / ((long long)B * pl.chunks)) : max(1LL, ctas / pl.chunks);
  const long long work_items = (per_sample ? 1LL : (long long)B) * grids;
  // makespan model: rounds of units per thread slot x row steps per unit (segment rows + the L-1 halo steps)
  const int L = (K + S - 1) / S;
  const long long slots = lanes * ppb;
  long long best = -1;
  pl.seg_rows = Fo;
  for (int seg = 1; seg <= min(Fo, 64); ++seg) {
    const long long units = (long long)strips * ceil_div(Fo, seg) * work_items;
    const long long cost = ((units + slots - 1) / slots) * (seg + L - 1);
    if (best < 0 || cost < best) { best = cost; pl.seg_rows = seg; }
  }
  const long long units1 = (long long)strips * ceil_div(Fo, pl.seg_rows) * grids;     // units of one sample
  if (per_sample) {
    pl.gy = B;
    pl.groups = (int)min(lanes, (long long)ceil_div((int)units1, ppb));
  } else {
    const long long need = (units1 * B + ppb - 1) / ppb;                       // CTAs (per chunk) that have any work
    pl.gy = (int)max(1LL, min(lanes, need));                                   // flat index space: any factorisation works
    pl.groups = 1;
  }
  if (pl.groups < 1) pl.groups = 1;
  return pl;
}

template <typename T, int K, int S, int P, int MODE, int XACT, int MINB, int D = 1, int DM = 2>
void launch_one(SlideArgs a, dim3 grid, size_t smem, cudaStream_t st) {
  constexpr int NIN = (P - 1) * S + K;
  const size_t slot = (size_t)NIN * kST * 16;
  a.depth = ring_depth((size_t)(227 * 1024) / MINB - 1024, smem, slot, a.cvc * Vec<T>::N <= 32 ? 3 : 2);
  static unsigned long long mask0 = 0, mask1 = 0;
  if (a.depth > 0) {
    auto kern = dw_slide_kernel<T, K, S, P, MODE, XACT, MINB, true, D, DM>;
    if (eat_opt_in_smem(kern, 200 * 1024, mask1) != EAT_OK) return;
    kern<<<grid, kST, smem + a.depth * slot, st>>>(a);
  } else {
    auto kern = dw_slide_kernel<T, K, S, P, MODE, XACT, MINB, false, D, DM>;
    if (eat_opt_in_smem(kern, 64 * 1024, mask0) != EAT_OK) return;
    kern<<<grid, kST, smem, st>>>(a);
  }
}

// the eval epilogue with DyReLU-B pieces other than two: the 3x3 layers of D = 1 only (a 5x5 eval runs in the tile kernel,
// conv_kernels.cu, and DyMN has no dilated layer)
constexpr int kDyMinB = 2;
template <typename T, int K, int S, int P, int MINB, int D = 1>
int launch_mode(const SlideArgs& a, int mode, int xact_code, dim3 grid, size_t smem, cudaStream_t st, int dyk = 2) {
  if (mode == 1 && dyk != 2 && a.dy.theta != nullptr) {
    if constexpr (K == 3 && D == 1) {
      // 2 DM coefficients per channel vector on top of the window: these instances run at kDyMinB CTAs per SM, where
      // they keep everything in registers (no spills, DESIGN.md section 4)
      switch (dyk) {
        case 1: launch_one<T, K, S, P, 1, -1, kDyMinB, D, 1>(a, grid, smem, st); break;
        case 3: launch_one<T, K, S, P, 1, -1, kDyMinB, D, 3>(a, grid, smem, st); break;
        case 4: launch_one<T, K, S, P, 1, -1, kDyMinB, D, 4>(a, grid, smem, st); break;
        default: eat_set_error("dw slide: DyReLU-B takes 1..4 linear pieces"); return EAT_ERR_UNSUPPORTED;
      }
      return EAT_OK;
    }
    eat_set_error("dw slide: DyReLU-B pieces other than two need a 3x3 undilated layer");
    return EAT_ERR_UNSUPPORTED;
  }
  if (mode == 1) launch_one<T, K, S, P, 1, -1, MINB, D>(a, grid, smem, st);
  else if (mode == 2) {
    if (S != 1) { eat_set_error("dw slide: data-gradient mode is stride 1 only"); return EAT_ERR_UNSUPPORTED; }
    launch_one<T, K, 1, P, 2, -1, MINB, D>(a, grid, smem, st);
  } else {
    switch (xact_code) {
      case -1: launch_one<T, K, S, P, 0, -1, MINB, D>(a, grid, smem, st); break;
      case EAT_ACT_NONE: launch_one<T, K, S, P, 0, EAT_ACT_NONE, MINB, D>(a, grid, smem, st); break;
      case EAT_ACT_RELU: launch_one<T, K, S, P, 0, EAT_ACT_RELU, MINB, D>(a, grid, smem, st); break;
      case EAT_ACT_HSWISH: launch_one<T, K, S, P, 0, EAT_ACT_HSWISH, MINB, D>(a, grid, smem, st); break;
      default: eat_set_error("dw slide: unsupported input activation"); return EAT_ERR_UNSUPPORTED;
    }
  }
  return EAT_OK;
}

template <typename T, int D = 1>
int launch_slide(SlideArgs a, int B, int k, int stride, int mode, int xact_code, cudaStream_t st, int dyk = 2) {
  constexpr int V = Vec<T>::N;
  constexpr bool kF32 = V == 4;
  const int cv = a.C / V;
  // 3x3 stride 1 -> 4-wide strips at 4 CTAs/SM; 3x3 stride 2 -> 2-wide strips (the 4-wide input span of 9 vectors costs
  // too many registers) at 5 CTAs/SM; 5x5 -> 2-wide strips at 3 CTAs/SM
  const int P = (k == 3 && stride == 1) ? (kF32 ? 4 : 2) : (kF32 ? 2 : 1);
  const int minb = k == 3 ? (stride == 1 ? 4 : 5) : 3;
  a.B = B;
  a.per_sample = (a.pool != nullptr || a.dy.theta != nullptr || a.dy.ca_f != nullptr || a.dy.wt_bstride != 0) ? 1 : 0;
  const SlidePlan pl = plan_slide(B, ceil_div(a.Fo, D), ceil_div(a.To, D), cv, V, P, stride, k, minb, a.per_sample != 0, kST,
                                  D * D);
  a.chunks = pl.chunks; a.cvc = pl.cvc; a.seg_rows = pl.seg_rows;
  dim3 grid(pl.chunks * pl.groups, pl.gy);
  const size_t smem = ((size_t)k * k + 2) * a.cvc * V * sizeof(float);
  int rc = EAT_OK;
  if (D == 2) {
    if (k == 3 && stride == 1) rc = launch_mode<T, 3, 1, kF32 ? 4 : 2, 4, 2>(a, mode, xact_code, grid, smem, st);
    else if (k == 5 && stride == 1) rc = launch_mode<T, 5, 1, kF32 ? 2 : 1, 3, 2>(a, mode, xact_code, grid, smem, st);
    else { eat_set_error("dw slide: dilation 2 needs k in {3,5} and stride 1"); return EAT_ERR_UNSUPPORTED; }
  } else if (k == 3 && stride == 1) rc = launch_mode<T, 3, 1, kF32 ? 4 : 2, 4>(a, mode, xact_code, grid, smem, st, dyk);
  else if (k == 3 && stride == 2) rc = launch_mode<T, 3, 2, kF32 ? 2 : 1, 5>(a, mode, xact_code, grid, smem, st, dyk);
  else if (k == 5 && stride == 1) rc = launch_mode<T, 5, 1, kF32 ? 2 : 1, 3>(a, mode, xact_code, grid, smem, st);
  else if (k == 5 && stride == 2) rc = launch_mode<T, 5, 2, kF32 ? 2 : 1, 3>(a, mode, xact_code, grid, smem, st);
  else { eat_set_error("dw slide: only k in {3,5}, stride in {1,2}"); return EAT_ERR_UNSUPPORTED; }
  if (rc != EAT_OK) return rc;
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}


// ------------------------------------------------------------------------------------------ weight gradient (3x3)
// dw[c, ky, kx] += sum_{b,o,t} dz[b,o,t,c] * xf(in)[b, o*S-1+ky, t*S-1+kx, c]
// Same walk as the forward kernel: a thread keeps the 9 tap accumulators of its channel vector in registers for
// its whole life (all strips, segments and samples it visits), slides a window of the L = ceil(3/S) most recent dz
// rows, and loads + transforms every input row once.  One shared-memory / global atomic flush per CTA at the end.
// V channels per thread as one vector load: the 5x5 weight gradient keeps 25 tap accumulators per channel, so it
// takes 2 fp32 channels (8-byte loads) per thread instead of 4 to stay in registers
template <typename T, int VW> struct VecW;
template <> struct VecW<float, 4> {
  __device__ __forceinline__ static void load(const float* p, float (&v)[4]) { Vec<float>::load(p, v); }
};
template <> struct VecW<float, 2> {
  __device__ __forceinline__ static void load(const float* p, float (&v)[2]) {
    const float2 t = *reinterpret_cast<const float2*>(p);
    v[0] = t.x; v[1] = t.y;
  }
};
template <> struct VecW<__nv_bfloat16, 8> {
  __device__ __forceinline__ static void load(const __nv_bfloat16* p, float (&v)[8]) { Vec<__nv_bfloat16>::load(p, v); }
};
template <> struct VecW<__nv_bfloat16, 4> {      // the dilated bf16 5x5 weight gradient: 25 x 4 tap accumulators
  __device__ __forceinline__ static void load(const __nv_bfloat16* p, float (&v)[4]) {
    const uint2 t = *reinterpret_cast<const uint2*>(p);
    const float2 lo = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&t.x));
    const float2 hi = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&t.y));
    v[0] = lo.x; v[1] = lo.y; v[2] = hi.x; v[3] = hi.y;
  }
};

struct WgArgs {
  const void* dz;
  const void* in;
  float* dw;
  long long dw_bstride;
  int B, F, Tn, Fo, To, C;
  int cvc, chunks, seg_rows;
  int per_sample;   // 1: blockIdx.y is the sample (per-sample gradient tables, DyMN)
  int depth;        // prefetch ring depth in steps (RING kernels)
  const float* xscale;
  const float* xshift;
};

// D = 2: dilation 2 at stride 1, walked sub-grid by sub-grid as in dw_slide_kernel
template <typename T, int K, int S, int P, int V, int XACT, int MINB, bool RING, int D = 1>
__global__ void __launch_bounds__(kST, MINB) dw_wgrad_slide_kernel(const WgArgs a) {
  static_assert(D == 1 || (D == 2 && S == 1), "dilation 2 is stride 1 only");
  constexpr int KK = K * K, PAD = (K - 1) / 2;
  constexpr int NIN = (P - 1) * S + K;
  constexpr int L = (K + S - 1) / S;
  constexpr bool kXf = XACT >= 0;
  extern __shared__ __align__(16) float smem[];
  const int F = a.F, Tn = a.Tn, Fo = a.Fo, To = a.To, C = a.C;
  const int chunk = blockIdx.x % a.chunks, grp = blockIdx.x / a.chunks, groups = gridDim.x / a.chunks;
  const int cv = C / V;
  const int cv0 = chunk * a.cvc;
  const int ncv = min(a.cvc, cv - cv0);
  const int cc = ncv * V;
  float* s_acc = smem;                         // [KK][cc]
  const int tid = threadIdx.x;
  // prefetch ring behind the table: [depth][NV][kST] vectors of VB bytes; NV = P dz vectors + NIN input vectors per row
  constexpr int VB = V * (int)sizeof(T), NV = P + NIN * S;
  const uint32_t ring0 = (uint32_t)__cvta_generic_to_shared(s_acc + KK * a.cvc * V) + (uint32_t)tid * VB;
  const unsigned char* ringp = reinterpret_cast<const unsigned char*>(s_acc + KK * a.cvc * V) + tid * VB;
  for (int i = tid; i < KK * cc; i += kST) s_acc[i] = 0.f;
  __syncthreads();
  const int ppb = kST / ncv;
  const int cvl = tid % ncv, slot = tid / ncv;
  if (slot < ppb) {
    const int c0 = (cv0 + cvl) * V;
    float isc[V], ish[V];
    if (kXf) {
#pragma unroll
      for (int i = 0; i < V; ++i) { isc[i] = __ldg(a.xscale + c0 + i); ish[i] = __ldg(a.xshift + c0 + i); }
    }
    float wacc[KK][V];
#pragma unroll
    for (int q = 0; q < KK; ++q)
#pragma unroll
      for (int i = 0; i < V; ++i) wacc[q][i] = 0.f;
    const int strips = ceil_div(D == 1 ? To : (To + 1) / 2, P), segs = ceil_div(D == 1 ? Fo : (Fo + 1) / 2, a.seg_rows);
    const int units = D * D * strips * segs;
    const long long rowstride = (long long)Tn * C * D;
    const int cstep = C * D;
    long long g = a.per_sample ? (long long)blockIdx.y * units + grp * ppb + slot : ((long long)blockIdx.y * groups + grp) * ppb + slot;
    const long long gend = a.per_sample ? (long long)(blockIdx.y + 1) * units : (long long)a.B * units;
    const long long gstep = a.per_sample ? (long long)groups * ppb : (long long)gridDim.y * groups * ppb;
    {
      for (; g < gend; g += gstep) {
        const int b = (int)(g / units);
        int u = (int)(g - (long long)b * units);
        const T* inb = reinterpret_cast<const T*>(a.in) + (size_t)b * F * Tn * C + c0;
        const T* dzb = reinterpret_cast<const T*>(a.dz) + (size_t)b * Fo * To * C + c0;
        int Fs = Fo, Ts = To;                   // rows / columns of the unit's sub-grid (D = 1: the image)
        if constexpr (D == 2) {
          const int par = u / (strips * segs), pr = par >> 1, pc = par & 1;
          u -= par * strips * segs;
          Fs = (Fo - pr + 1) >> 1;
          Ts = (To - pc + 1) >> 1;
          const size_t poff = ((size_t)pr * To + pc) * C;
          inb += poff;
          dzb += poff;
        }
        const int seg = u / strips, strip = u - seg * strips;
        const int fo_a = seg * a.seg_rows;
        const int nrows = min(a.seg_rows, Fs - fo_a);
        const int to0 = strip * P;
        if (D == 2 && (nrows <= 0 || to0 >= Ts)) continue;
        const int t0 = to0 * S - PAD;
        const int Fin = D == 1 ? F : Fs, Tin = D == 1 ? Tn : Ts;
        unsigned cmask = 0;
#pragma unroll
        for (int j = 0; j < NIN; ++j) cmask |= (t0 + j >= 0 && t0 + j < Tin) ? (1u << j) : 0u;
        const int i0 = fo_a * S - PAD;
        const T* colp = inb + (long long)t0 * cstep;
        const T* dzp = dzb + (D == 1 ? ((size_t)fo_a * To + to0) * C : ((size_t)(D * fo_a) * To + D * to0) * C);
        float dzw[L][P][V];
#pragma unroll
        for (int l = 0; l < L; ++l)
#pragma unroll
          for (int p = 0; p < P; ++p)
#pragma unroll
            for (int i = 0; i < V; ++i) dzw[l][p][i] = 0.f;

        // an input row is loaded (raw) by ld() and later transformed + multiplied by mac(); for S = 2 the even and the
        // odd row of a step are both requested before either is used (twice the bytes in flight per thread)
        float ve[NIN][V], vo[NIN][V];            // two row buffers: even/odd row of a stride-2 step, ping-pong for stride 1
        auto ld = [&](int irow, auto buf_tag) {
          constexpr int BUF = decltype(buf_tag)::value;
          float (&v)[NIN][V] = *reinterpret_cast<float (*)[NIN][V]>(BUF == 0 ? &ve[0][0] : &vo[0][0]);
          const T* rp = colp + (long long)irow * rowstride;
#pragma unroll
          for (int j = 0; j < NIN; ++j) {
            if ((cmask >> j) & 1u) VecW<T, V>::load(rp + (size_t)j * cstep, v[j]);
            else {
#pragma unroll
              for (int i = 0; i < V; ++i) v[j][i] = 0.f;
            }
          }
        };
        auto mac = [&](auto buf_tag, auto ph_tag) {
          constexpr int BUF = decltype(buf_tag)::value;
          constexpr int PH = decltype(ph_tag)::value;
          float (&v)[NIN][V] = *reinterpret_cast<float (*)[NIN][V]>(BUF == 0 ? &ve[0][0] : &vo[0][0]);
          if (kXf) {
#pragma unroll
            for (int j = 0; j < NIN; ++j) {
              const bool ok = (cmask >> j) & 1u;
#pragma unroll
              for (int i = 0; i < V; ++i) {
                const float tv = xact<XACT>(fmaf(v[j][i], isc[i], ish[i]));
                v[j][i] = ok ? tv : 0.f;
              }
            }
          }
#pragma unroll
          for (int ky = 0; ky < K; ++ky) {
            if ((ky % S) != PH) continue;
            const int sl = (S == 1) ? (L - 1 - ky) : (PH == 0 ? (L - 1 - ky / 2) : (L - 1 - (ky - 1) / 2));
#pragma unroll
            for (int kx = 0; kx < K; ++kx)
#pragma unroll
              for (int p = 0; p < P; ++p)
                fma_vec<V>(dzw[sl][p], v[p * S + kx], wacc[ky * K + kx]);
          }
        };
        using Ph0 = std::integral_constant<int, 0>;
        using Ph1 = std::integral_constant<int, 1>;

        // step n: the window slides to dz rows n-(L-1) .. n (relative to fo_a), then input row i0 + n*S (and, for
        // S = 2, i0 + 2n + 1 with the middle kernel row) meets the dz rows it was multiplied with in the forward pass
        const int steps = nrows + L - 1;
        auto slide_window = [&](int n) {
#pragma unroll
          for (int l = 0; l + 1 < L; ++l)
#pragma unroll
            for (int p = 0; p < P; ++p)
#pragma unroll
              for (int i = 0; i < V; ++i) dzw[l][p][i] = dzw[l + 1][p][i];
          if (n < nrows) {
            const T* gp = dzp + (size_t)n * To * C * D;
#pragma unroll
            for (int p = 0; p < P; ++p) {
              if (to0 + p < Ts) VecW<T, V>::load(gp + (size_t)p * cstep, dzw[L - 1][p]);
              else {
#pragma unroll
                for (int i = 0; i < V; ++i) dzw[L - 1][p][i] = 0.f;
              }
            }
          } else {
#pragma unroll
            for (int p = 0; p < P; ++p)
#pragma unroll
              for (int i = 0; i < V; ++i) dzw[L - 1][p][i] = 0.f;
          }
        };
        if constexpr (RING) {
          // step n's operands (dz row n, input row i0 + n, or rows i0 + 2n and i0 + 2n + 1 for stride 2) travel as ONE
          // cp.async group into slot n % depth; the thread reads back only its own copies
          auto rows_of = [&](int n, int& ie, bool& ev, bool& od) {
            ie = i0 + n * S;
            ev = ie >= 0 && ie < Fin;
            od = S == 2 && (n < nrows + (K - 3) / 2) && ie + 1 >= 0 && ie + 1 < Fin;
          };
          auto issue = [&](int n, int slot_) {
            if (n < steps) {
              const uint32_t dst = ring0 + (uint32_t)(slot_ * NV) * (kST * VB);
              if (n < nrows) {
                const T* gp = dzp + (size_t)n * To * C * D;
#pragma unroll
                for (int p = 0; p < P; ++p)
                  if (to0 + p < Ts) cp_async<VB>(dst + (uint32_t)p * (kST * VB), gp + (size_t)p * cstep);
              }
              int ie; bool ev, od;
              rows_of(n, ie, ev, od);
              if (ev) {
                const T* rp = colp + (long long)ie * rowstride;
#pragma unroll
                for (int j = 0; j < NIN; ++j)
                  if ((cmask >> j) & 1u) cp_async<VB>(dst + (uint32_t)(P + j) * (kST * VB), rp + (size_t)j * cstep);
              }
              if (od) {
                const T* rp = colp + (long long)(ie + 1) * rowstride;
#pragma unroll
                for (int j = 0; j < NIN; ++j)
                  if ((cmask >> j) & 1u) cp_async<VB>(dst + (uint32_t)(P + NIN + j) * (kST * VB), rp + (size_t)j * cstep);
              }
            }
            cp_commit();
          };
          auto fetch = [&](int slot_, int first, float (&v)[NIN][V]) {
#pragma unroll
            for (int j = 0; j < NIN; ++j) {
              if ((cmask >> j) & 1u) VecW<T, V>::load(reinterpret_cast<const T*>(ringp + (size_t)(slot_ * NV + first + j) * (kST * VB)), v[j]);
              else {
#pragma unroll
                for (int i = 0; i < V; ++i) v[j][i] = 0.f;
              }
            }
          };
          for (int q = 0; q < a.depth; ++q) issue(q, q);
          int rs = 0;
          for (int n = 0; n < steps; ++n) {
            cp_wait_pending(a.depth - 1);
#pragma unroll
            for (int l = 0; l + 1 < L; ++l)
#pragma unroll
              for (int p = 0; p < P; ++p)
#pragma unroll
                for (int i = 0; i < V; ++i) dzw[l][p][i] = dzw[l + 1][p][i];
#pragma unroll
            for (int p = 0; p < P; ++p) {
              if (n < nrows && to0 + p < Ts) VecW<T, V>::load(reinterpret_cast<const T*>(ringp + (size_t)(rs * NV + p) * (kST * VB)), dzw[L - 1][p]);
              else {
#pragma unroll
                for (int i = 0; i < V; ++i) dzw[L - 1][p][i] = 0.f;
              }
            }
            int ie; bool ev, od;
            rows_of(n, ie, ev, od);
            if (ev) { fetch(rs, P, ve); mac(Ph0{}, Ph0{}); }
            if (od) { fetch(rs, P + NIN, ve); mac(Ph0{}, Ph1{}); }
            issue(n + a.depth, rs);
            if (++rs == a.depth) rs = 0;
          }
        } else if (S == 2) {
          for (int n = 0; n < steps; ++n) {
            slide_window(n);
            const int ie = i0 + 2 * n, io = ie + 1;                   // odd kernel rows reach dz rows n .. n-(K-3)/2
            const bool ev = ie >= 0 && ie < F;
            const bool od = (n < nrows + (K - 3) / 2) && io >= 0 && io < F;
            if (ev) ld(ie, Ph0{});
            if (od) ld(io, Ph1{});
            if (ev) mac(Ph0{}, Ph0{});
            if (od) mac(Ph1{}, Ph1{});
          }
        } else {
          // stride 1: row n+1 is requested into the other buffer before row n is multiplied
          auto step = [&](int n, auto cur, auto nxt) {
            slide_window(n);
            const int ie = i0 + n;
            if (n + 1 < steps && ie + 1 >= 0 && ie + 1 < Fin) ld(ie + 1, nxt);
            if (ie >= 0 && ie < Fin) mac(cur, Ph0{});
          };
          if (i0 >= 0 && i0 < Fin) ld(i0, Ph0{});
          for (int n = 0; n < steps; n += 2) {
            step(n, Ph0{}, Ph1{});
            if (n + 1 < steps) step(n + 1, Ph1{}, Ph0{});
          }
        }
      }
    }
#pragma unroll
    for (int q = 0; q < KK; ++q)
#pragma unroll
      for (int i = 0; i < V; ++i) atomicAdd(&s_acc[q * cc + cvl * V + i], wacc[q][i]);
  }
  __syncthreads();
  float* dwb = a.dw + (a.dw_bstride != 0 ? (size_t)blockIdx.y * a.dw_bstride : 0);
  for (int i = tid; i < KK * cc; i += kST) {
    const int q = i / cc, c = i - q * cc;
    atomicAdd(dwb + (size_t)(cv0 * V + c) * KK + q, s_acc[i]);
  }
}

template <typename T, int K, int S, int P, int V, int XACT, int MINB, int D>
int launch_wg_one(WgArgs a, dim3 grid, size_t smem, cudaStream_t st) {
  constexpr int NIN = (P - 1) * S + K;
  const size_t slot = (size_t)(P + NIN * S) * kST * V * sizeof(T);
  a.depth = ring_depth((size_t)(227 * 1024) / MINB - 1024, smem, slot, S == 1 ? 2 : 0);   // stride 2: a slot holds two input rows, the ring costs a CTA
  static unsigned long long mask1 = 0;
  if (a.depth > 0) {
    auto kern = dw_wgrad_slide_kernel<T, K, S, P, V, XACT, MINB, true, D>;
    if (int rc = eat_opt_in_smem(kern, 200 * 1024, mask1)) return rc;
    kern<<<grid, kST, smem + a.depth * slot, st>>>(a);
  } else {
    dw_wgrad_slide_kernel<T, K, S, P, V, XACT, MINB, false, D><<<grid, kST, smem, st>>>(a);
  }
  return EAT_OK;
}

template <typename T, int K, int S, int P, int V, int MINB, int D = 1>
int launch_wg_act(const WgArgs& a, int xact_code, dim3 grid, size_t smem, cudaStream_t st) {
  switch (xact_code) {
    case -1: return launch_wg_one<T, K, S, P, V, -1, MINB, D>(a, grid, smem, st);
    case EAT_ACT_NONE: return launch_wg_one<T, K, S, P, V, EAT_ACT_NONE, MINB, D>(a, grid, smem, st);
    case EAT_ACT_RELU: return launch_wg_one<T, K, S, P, V, EAT_ACT_RELU, MINB, D>(a, grid, smem, st);
    case EAT_ACT_HSWISH: return launch_wg_one<T, K, S, P, V, EAT_ACT_HSWISH, MINB, D>(a, grid, smem, st);
    default: eat_set_error("dw wgrad slide: unsupported input activation"); return EAT_ERR_UNSUPPORTED;
  }
}

// K = 3: 4 fp32 (8 bf16) channels per thread; K = 5 (fp32 only): 2 channels per thread, 25 x 2 tap accumulators
template <typename T, int K, int V, int P, int MINB, int D = 1>
int launch_wg_slide(WgArgs a, int stride, int xact_code, cudaStream_t st) {
  const int cv = a.C / V;
  a.per_sample = a.dw_bstride != 0 ? 1 : 0;
  const SlidePlan pl = plan_slide(a.B, ceil_div(a.Fo, D), ceil_div(a.To, D), cv, V, P, stride, K, stride == 2 ? 3 : MINB,
                                  a.per_sample != 0, kST, D * D);
  a.chunks = pl.chunks; a.cvc = pl.cvc; a.seg_rows = pl.seg_rows;
  dim3 grid(pl.chunks * pl.groups, pl.gy);
  const size_t smem = (size_t)K * K * a.cvc * V * sizeof(float);
  int rc;
  if (D == 2) {
    if (stride != 1) { eat_set_error("dw wgrad slide: dilation 2 is stride 1 only"); return EAT_ERR_UNSUPPORTED; }
    rc = launch_wg_act<T, K, 1, P, V, MINB, 2>(a, xact_code, grid, smem, st);
  } else if (stride == 1) rc = launch_wg_act<T, K, 1, P, V, MINB>(a, xact_code, grid, smem, st);
  else rc = launch_wg_act<T, K, 2, P, V, 3>(a, xact_code, grid, smem, st);     // two row buffers: 168 registers
  if (rc != EAT_OK) return rc;
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}


// ------------------------------------------------------------------------------------------ stride-2 data gradient
// din[i, t] = sum_{ky, kx : i+PAD-ky and t+PAD-kx even} dz[(i+PAD-ky)/2, (t+PAD-kx)/2] * w[ky, kx]   (+ res)
// A thread owns a channel vector and Q = 4 input-gradient columns, walks down PAIRS of din rows (2m, 2m+1) and keeps
// the (K+1)/2 dz rows they read in a register window, so every dz row is loaded once per strip; the parity
// conditions are resolved at compile time (no divisions / bounds tests per tap as in the gather kernel).
struct Dg2Args {
  const void* dz;
  const float* wt;
  long long wt_bstride;
  const void* res;
  void* din;
  int B, F, Tn, Fo, To, C;
  int cvc, chunks, seg_rows;   // seg_rows counts row PAIRS
  int per_sample;
  int depth;                   // prefetch ring depth in dz rows (RING kernels)
  // RED kernels: din is the upstream gradient of a BatchNorm + activation whose raw input z has din's shape; the
  // BatchNorm-backward reduce (s1 += sum g, s2 += invstd * sum g * (z - mean), g = din * act'(z*scale+shift)) is taken
  // in the epilogue, while the din values are still in registers -- the separate reduce pass would read din and z again
  const void* z;
  const float* zscale;
  const float* zshift;
  const float* zmean;
  const float* zinvstd;
  int zact;
  double* s1;
  double* s2;
};

template <typename T, int K, int MINB, bool RING, bool RED = false>
__global__ void __launch_bounds__(kST, MINB) dw_dgrad2_slide_kernel(const Dg2Args a) {
  constexpr int V = Vec<T>::N;
  constexpr int Q = 4, PAD = (K - 1) / 2, KK = K * K;
  constexpr int LW = (K + 1) / 2;               // dz rows read by one pair of din rows
  constexpr int NDZ = Q / 2 + PAD / 2 + 1;      // dz columns read by Q din columns
  extern __shared__ __align__(16) float smem[];
  const int F = a.F, Tn = a.Tn, Fo = a.Fo, To = a.To, C = a.C;
  const int chunk = blockIdx.x % a.chunks, grp = blockIdx.x / a.chunks, groups = gridDim.x / a.chunks;
  const int cv = C / V;
  const int cv0 = chunk * a.cvc;
  const int ncv = min(a.cvc, cv - cv0);
  const int cc = ncv * V;
  float* s_w = smem;                             // [KK][cc]
  const int tid = threadIdx.x;
  const int cst = a.cvc * V;                     // channel stride of the per-CTA tables
  float* s_bn = s_w + KK * cst;                  // RED: [3][cst] scale, shift, mean of the BatchNorm behind din
  float* s_red = s_bn + 3 * cst;                 // RED: [2][cst] CTA partial sums
  float* s_end = RED ? s_red + 2 * cst : s_bn;   // the prefetch ring follows the tables
  const uint32_t ring0 = (uint32_t)__cvta_generic_to_shared(s_end) + (uint32_t)tid * 16u;   // [depth][NDZ][kST] x 16 B
  const unsigned char* ringp = reinterpret_cast<const unsigned char*>(s_end) + tid * 16;
  {
    const float* wsrc = a.wt + (a.per_sample ? (size_t)blockIdx.y * a.wt_bstride : 0) + (size_t)cv0 * V;
    for (int i = tid; i < KK * cc; i += kST) {
      const int tap = i / cc, c = i - tap * cc;
      s_w[i] = __ldg(wsrc + (size_t)tap * C + c);
    }
    if (RED) {
      for (int c = tid; c < cc; c += kST) {
        const int cg = cv0 * V + c;
        s_bn[c] = __ldg(a.zscale + cg); s_bn[cst + c] = __ldg(a.zshift + cg); s_bn[2 * cst + c] = __ldg(a.zmean + cg);
        s_red[c] = 0.f; s_red[cst + c] = 0.f;
      }
    }
  }
  __syncthreads();
  const int ppb = kST / ncv;
  const int cvl = tid % ncv, slot = tid / ncv;
  if (!RED && slot >= ppb) return;               // RED: idle threads still take part in the final CTA reduction
  const int c0 = (cv0 + cvl) * V;
  const float* wl = s_w + cvl * V;
  float lsum[V], lsq[V];                         // RED: this thread's share of sum g, sum g * (z - mean)
#pragma unroll
  for (int i = 0; i < V; ++i) { lsum[i] = 0.f; lsq[i] = 0.f; }
  const int pairs = (F + 1) / 2;
  const int strips = ceil_div(Tn, Q), segs = ceil_div(pairs, a.seg_rows), units = strips * segs;
  long long g = a.per_sample ? (long long)blockIdx.y * units + grp * ppb + slot : ((long long)blockIdx.y * groups + grp) * ppb + slot;
  const long long gend = a.per_sample ? (long long)(blockIdx.y + 1) * units : (long long)a.B * units;
  const long long gstep = a.per_sample ? (long long)groups * ppb : (long long)gridDim.y * groups * ppb;
  if (RED && slot >= ppb) g = gend;
  for (; g < gend; g += gstep) {
    const int b = (int)(g / units);
    const int u = (int)(g - (long long)b * units);
    const T* dzb = reinterpret_cast<const T*>(a.dz) + (size_t)b * Fo * To * C + c0;
    T* dinb = reinterpret_cast<T*>(a.din) + (size_t)b * F * Tn * C + c0;
    const T* resb = a.res != nullptr ? reinterpret_cast<const T*>(a.res) + (size_t)b * F * Tn * C + c0 : nullptr;
    const T* zb = RED ? reinterpret_cast<const T*>(a.z) + (size_t)b * F * Tn * C + c0 : nullptr;
    const int seg = u / strips, strip = u - seg * strips;
    const int m_a = seg * a.seg_rows;
    const int npair = min(a.seg_rows, pairs - m_a);
    const int t_a = strip * Q;                               // even
    const int to_base = t_a / 2 - PAD / 2;                   // dz column of window index 0
    unsigned cmask = 0;
#pragma unroll
    for (int j = 0; j < NDZ; ++j) cmask |= (to_base + j >= 0 && to_base + j < To) ? (1u << j) : 0u;
    const T* colp = dzb + (long long)to_base * C;
    float win[LW][NDZ][V];                                   // slot l <-> dz row m - PAD/2 + l
    auto load_row = [&](int o, float (&dst)[NDZ][V]) {
      if (o >= 0 && o < Fo) {
        const T* rp = colp + (long long)o * To * C;
#pragma unroll
        for (int j = 0; j < NDZ; ++j) {
          if ((cmask >> j) & 1u) Vec<T>::load(rp + (size_t)j * C, dst[j]);
          else {
#pragma unroll
            for (int i = 0; i < V; ++i) dst[j][i] = 0.f;
          }
        }
      } else {
#pragma unroll
        for (int j = 0; j < NDZ; ++j)
#pragma unroll
          for (int i = 0; i < V; ++i) dst[j][i] = 0.f;
      }
    };
    // prefill: rows m_a - PAD/2 .. m_a + LW - 2 - PAD/2 go to slots 1 .. LW-1 (they shift down by one in step 0)
    // ring: step mm needs dz row m_a + mm - PAD/2 + LW - 1; one cp.async group per step, own copies only
    auto issue = [&](int mm, int slot_) {
      if (RING) {
        const int o = m_a + mm - PAD / 2 + LW - 1;
        if (mm < npair && o >= 0 && o < Fo) {
          const T* rp = colp + (long long)o * To * C;
          const uint32_t dst = ring0 + (uint32_t)(slot_ * NDZ) * (kST * 16u);
#pragma unroll
          for (int j = 0; j < NDZ; ++j)
            if ((cmask >> j) & 1u) cp_async<16>(dst + (uint32_t)j * (kST * 16u), rp + (size_t)j * C);
        }
        cp_commit();
      }
    };
    if (RING) {
      for (int q = 0; q < a.depth; ++q) issue(q, q);
    }
#pragma unroll
    for (int l = 1; l < LW; ++l) load_row(m_a - PAD / 2 + l - 1, win[l]);
    int rs = 0;
    for (int mm = 0; mm < npair; ++mm) {
      const int m = m_a + mm;
#pragma unroll
      for (int l = 0; l + 1 < LW; ++l)
#pragma unroll
        for (int j = 0; j < NDZ; ++j)
#pragma unroll
          for (int i = 0; i < V; ++i) win[l][j][i] = win[l + 1][j][i];
      if (RING) {
        cp_wait_pending(a.depth - 1);
        const int o = m - PAD / 2 + LW - 1;
#pragma unroll
        for (int j = 0; j < NDZ; ++j) {
          if (o >= 0 && o < Fo && ((cmask >> j) & 1u)) Vec<T>::load(reinterpret_cast<const T*>(ringp + (size_t)(rs * NDZ + j) * (kST * 16)), win[LW - 1][j]);
          else {
#pragma unroll
            for (int i = 0; i < V; ++i) win[LW - 1][j][i] = 0.f;
          }
        }
        issue(mm + a.depth, rs);
        if (++rs == a.depth) rs = 0;
      } else {
        load_row(m - PAD / 2 + LW - 1, win[LW - 1]);
      }
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int irow = 2 * m + r;
        if (irow >= F) continue;
        float acc[Q][V];
#pragma unroll
        for (int q = 0; q < Q; ++q)
#pragma unroll
          for (int i = 0; i < V; ++i) acc[q][i] = 0.f;
#pragma unroll
        for (int ky = 0; ky < K; ++ky) {
          if (((r + PAD - ky) & 1) != 0) continue;
          const int sl = (r + PAD - ky) / 2 + PAD / 2;         // compile-time after unrolling (numerator even, may be < 0)
#pragma unroll
          for (int kx = 0; kx < K; ++kx) {
            float w[V];
#pragma unroll
            for (int qq = 0; qq < V / 4; ++qq) {
              const float4 t4 = *reinterpret_cast<const float4*>(wl + (ky * K + kx) * cc + 4 * qq);
              w[4 * qq] = t4.x; w[4 * qq + 1] = t4.y; w[4 * qq + 2] = t4.z; w[4 * qq + 3] = t4.w;
            }
#pragma unroll
            for (int q = 0; q < Q; ++q) {
              if (((q + PAD - kx) & 1) != 0) continue;
              const int j = (q + PAD - kx) / 2 + PAD / 2;
              fma_vec<V>(win[sl][j], w, acc[q]);
            }
          }
        }
#pragma unroll
        for (int q = 0; q < Q; ++q) {
          const int t = t_a + q;
          if (t < Tn) {
            const size_t off = ((size_t)irow * Tn + t) * C;
            if (resb != nullptr) {
              float rv[V];
              Vec<T>::load(resb + off, rv);
#pragma unroll
              for (int i = 0; i < V; ++i) acc[q][i] += rv[i];
            }
            Vec<T>::store(dinb + off, acc[q]);
            if (RED) {
              float zv[V];
              Vec<T>::load(zb + off, zv);
              const float* bn = s_bn + cvl * V;
#pragma unroll
              for (int i = 0; i < V; ++i) {
                const float gd = acc[q][i] * act_bwd(fmaf(zv[i], bn[i], bn[cst + i]), a.zact);
                lsum[i] += gd;
                lsq[i] = fmaf(gd, zv[i] - bn[2 * cst + i], lsq[i]);
              }
            }
          }
        }
      }
    }
  }
  if (RED) {
    if (slot < ppb) {
#pragma unroll
      for (int i = 0; i < V; ++i) { atomicAdd(&s_red[cvl * V + i], lsum[i]); atomicAdd(&s_red[cst + cvl * V + i], lsq[i]); }
    }
    __syncthreads();
    for (int c = tid; c < cc; c += kST) {
      const int cg = cv0 * V + c;
      atomicAdd(a.s1 + cg, (double)s_red[c]);
      atomicAdd(a.s2 + cg, (double)s_red[cst + c] * (double)__ldg(a.zinvstd + cg));
    }
  }
}

// resident CTAs per SM of the RED variants (the epilogue needs ~16 more registers than the plain kernels' 104 / 160)
constexpr int kDg2RedMinB3 = 4, kDg2RedMinB5 = 3;

template <typename T>
int launch_dg2_slide(Dg2Args a, int k, cudaStream_t st) {
  constexpr int V = Vec<T>::N;
  const int cv = a.C / V;
  const int minb = a.z != nullptr ? (k == 3 ? kDg2RedMinB3 : kDg2RedMinB5) : (k == 3 ? 4 : 3);
  a.per_sample = a.wt_bstride != 0 ? 1 : 0;
  const int pairs = (a.F + 1) / 2;
  const SlidePlan pl = plan_slide(a.B, pairs, a.Tn, cv, V, 4, 1, (k + 1) / 2, minb, a.per_sample != 0);
  a.chunks = pl.chunks; a.cvc = pl.cvc; a.seg_rows = pl.seg_rows;
  dim3 grid(pl.chunks * pl.groups, pl.gy);
  constexpr int NDZ3 = 4 / 2 + 1 / 2 + 1, NDZ5 = 4 / 2 + 2 / 2 + 1;
  if (a.z != nullptr) {
    // BatchNorm-backward reduce in the epilogue (fp32 storage only): five more per-channel tables in shared memory
    if constexpr (std::is_same<T, float>::value) {
      const size_t smem_r = (size_t)(k * k + 5) * a.cvc * V * sizeof(float);
      static unsigned long long r3 = 0, r5 = 0, r5n = 0;
      if (k == 3) {
        a.depth = 0;
        if (int rc = eat_opt_in_smem(dw_dgrad2_slide_kernel<T, 3, kDg2RedMinB3, false, true>, 64 * 1024, r3)) return rc;
        dw_dgrad2_slide_kernel<T, 3, kDg2RedMinB3, false, true><<<grid, kST, smem_r, st>>>(a);
      } else {
        const size_t slot = (size_t)NDZ5 * kST * 16;
        a.depth = ring_depth((size_t)(227 * 1024) / kDg2RedMinB5 - 1024, smem_r, slot, 2);
        if (a.depth > 0) {
          if (int rc = eat_opt_in_smem(dw_dgrad2_slide_kernel<T, 5, kDg2RedMinB5, true, true>, 200 * 1024, r5)) return rc;
          dw_dgrad2_slide_kernel<T, 5, kDg2RedMinB5, true, true><<<grid, kST, smem_r + a.depth * slot, st>>>(a);
        } else {
          if (int rc = eat_opt_in_smem(dw_dgrad2_slide_kernel<T, 5, kDg2RedMinB5, false, true>, 64 * 1024, r5n)) return rc;
          dw_dgrad2_slide_kernel<T, 5, kDg2RedMinB5, false, true><<<grid, kST, smem_r, st>>>(a);
        }
      }
      EAT_CHECK_LAUNCH();
      return EAT_OK;
    } else {
      eat_set_error("dw dgrad with BatchNorm reduce: fp32 storage only");
      return EAT_ERR_UNSUPPORTED;
    }
  }
  const size_t smem = (size_t)k * k * a.cvc * V * sizeof(float);
  static unsigned long long m3 = 0, m5 = 0, m5n = 0;
  if (k == 3) {
    const size_t slot = (size_t)NDZ3 * kST * 16;
    a.depth = ring_depth((size_t)(227 * 1024) / 4 - 1024, smem, slot, 0);       // 3x3: no ring (a slot would hold two input rows)
    if (a.depth > 0) {
      if (int rc = eat_opt_in_smem(dw_dgrad2_slide_kernel<T, 3, 4, true>, 200 * 1024, m3)) return rc;
      dw_dgrad2_slide_kernel<T, 3, 4, true><<<grid, kST, smem + a.depth * slot, st>>>(a);
    } else dw_dgrad2_slide_kernel<T, 3, 4, false><<<grid, kST, smem, st>>>(a);
  } else {
    const size_t slot = (size_t)NDZ5 * kST * 16;
    a.depth = ring_depth((size_t)(227 * 1024) / 3 - 1024, smem, slot, 2);
    if (a.depth > 0) {
      if (int rc = eat_opt_in_smem(dw_dgrad2_slide_kernel<T, 5, 3, true>, 200 * 1024, m5)) return rc;
      dw_dgrad2_slide_kernel<T, 5, 3, true><<<grid, kST, smem + a.depth * slot, st>>>(a);
    } else {
      if (int rc = eat_opt_in_smem(dw_dgrad2_slide_kernel<T, 5, 3, false>, 64 * 1024, m5n)) return rc;
      dw_dgrad2_slide_kernel<T, 5, 3, false><<<grid, kST, smem, st>>>(a);
    }
  }
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}


// ------------------------------------------------------------------------------------------ fused depthwise backward
// The whole backward of a depthwise stage whose raw output z2 feeds a BatchNorm + activation (BN2), in one walk:
//   dz   = BN2-backward apply of (dp, z2): scale2 * g * act'(z2*scale2+shift2) + alpha * z2 + beta, g = dp*gate + dpool
//          (the constants of bn_bwd_apply2_kernel), computed as each dz element is loaded and never stored
//   din  = depthwise data gradient of dz (+ res), stored
//   dW  += sum dz * xf(in),  xf = act(in*in_scale+in_shift) (the expand stage's BatchNorm + activation) or identity
//   s1  += sum g1, s2 += invstd1 * sum g1*(in-mean1),  g1 = din * act'(in*in_scale+in_shift)  (optional: the expand
//          BatchNorm's backward reduce, what eat_bn_bwd_reduce(gA = din) yields)
// The data and the weight gradient visit the same (din element, dz element, tap) triples, so both come out of a walk
// organised by din elements, as dw_dgrad2_slide_kernel: a thread owns a channel vector and Q din columns, walks down its
// segment (single din rows for stride 1, row pairs for stride 2) and keeps the LW dz rows they read in a register
// window.  Per step ONE cp.async group brings the new dz row (dp and z2 over the strip and its halo) and the step's S input
// rows (own columns only) into the thread's ring slot, two steps ahead.
// Algorithmic bytes: dp, z2, in read once, din written once (2*T2 + 2*T1 elements); the separate passes (BN2 apply,
// weight gradient, data gradient, BN1 reduce) move 5*T2 + 4*T1.
struct FusedBwdArgs {
  const float* dp;
  const float* gate;
  const float* dpool;
  const float* z2;
  const float* scale;
  const float* shift;
  const float* mean;
  const float* invstd;
  const float* c1;
  const float* c2;
  const float* wt;
  const float* in;
  const float* in_scale;
  const float* in_shift;
  const float* res;
  float* din;
  float* dw;
  const float* zmean;
  const float* zinvstd;
  double* s1;
  double* s2;
  int B, F, Tn, Fo, To, C;
  int cvc, chunks, seg_rows;   // seg_rows counts steps (din rows for stride 1, row pairs for stride 2)
};

template <int V> struct VecF;
template <> struct VecF<4> {
  __device__ __forceinline__ static void load(const float* p, float (&v)[4]) { Vec<float>::load(p, v); }
  __device__ __forceinline__ static void store(float* p, const float (&v)[4]) { Vec<float>::store(p, v); }
};
template <> struct VecF<2> {
  __device__ __forceinline__ static void load(const float* p, float (&v)[2]) {
    const float2 t = *reinterpret_cast<const float2*>(p);
    v[0] = t.x; v[1] = t.y;
  }
  __device__ __forceinline__ static void store(float* p, const float (&v)[2]) {
    *reinterpret_cast<float2*>(p) = make_float2(v[0], v[1]);
  }
};

constexpr int kFbCvcMax = 32;   // channel vectors per CTA: keeps the five per-CTA tables small next to the ring
constexpr int kFbDepth = 2;     // ring depth in steps

// V: channels per thread (the 5x5 kernels keep 25 x V tap accumulators, so they take 2); Q: din columns per strip
template <int K, int S> struct FbShape {
  static constexpr int V = K == 3 ? 4 : 2;
  static constexpr int Q = (S == 2 && K == 5) ? 4 : 2;
  static constexpr int PAD = (K - 1) / 2;
  static constexpr int LW = S == 1 ? K : (K + 1) / 2;                   // dz rows read by one step
  static constexpr int NDZ = S == 1 ? Q + 2 * PAD : Q / 2 + PAD / 2 + 1;  // dz columns read by Q din columns
  static constexpr int OB0 = S == 1 ? PAD : PAD / 2;                    // window slot 0 <-> dz row m - OB0
  static constexpr int NV = 2 * NDZ + S * Q;                            // ring vectors per step: dp, z2, input rows
  // resident CTAs per SM the register budget is planned for: 3 (<= 168 registers) fits the 3x3 stride-2 walk; the
  // stride-1 windows (K dz rows) and the 25 tap accumulators of the 5x5 spill there, so they take 2 (<= 255 registers)
  static constexpr int MINB = (K == 3 && S == 2) ? 3 : 2;
};

template <int K, int S, int ACT, bool XF>
__global__ void __launch_bounds__(kST, FbShape<K, S>::MINB) dw_bwd_fused_kernel(const FusedBwdArgs a) {
  using Sh = FbShape<K, S>;
  constexpr int V = Sh::V, Q = Sh::Q, PAD = Sh::PAD, LW = Sh::LW, NDZ = Sh::NDZ, OB0 = Sh::OB0, NV = Sh::NV;
  constexpr int KK = K * K, VB = V * (int)sizeof(float);
  extern __shared__ __align__(16) float smem[];
  const int F = a.F, Tn = a.Tn, Fo = a.Fo, To = a.To, C = a.C;
  const int chunk = blockIdx.x % a.chunks, grp = blockIdx.x / a.chunks, groups = gridDim.x / a.chunks;
  const int cv = C / V;
  const int cv0 = chunk * a.cvc;
  const int ncv = min(a.cvc, cv - cv0);
  const int cc = ncv * V;
  const int cst = a.cvc * V;                     // channel stride of the per-CTA tables
  float* s_w = smem;                             // [KK][cst] taps
  float* s_acc = s_w + KK * cst;                 // [KK][cst] weight-gradient partial sums
  float* s_bn = s_acc + KK * cst;                // [7][cst] BN2 scale, shift, alpha, beta; xf scale, shift; BN1 mean
  float* s_red = s_bn + 7 * cst;                 // [2][cst] BN1 partial sums
  float* s_end = s_red + 2 * cst;                // the prefetch ring follows: [depth][NV][kST] vectors
  const int tid = threadIdx.x;
  const uint32_t ring0 = (uint32_t)__cvta_generic_to_shared(s_end) + (uint32_t)tid * VB;
  const unsigned char* ringp = reinterpret_cast<const unsigned char*>(s_end) + tid * VB;
  const bool red = XF && a.s1 != nullptr;
  for (int i = tid; i < KK * cc; i += kST) {
    const int tap = i / cc, c = i - tap * cc;
    s_w[tap * cst + c] = __ldg(a.wt + (size_t)tap * C + cv0 * V + c);
    s_acc[tap * cst + c] = 0.f;
  }
  for (int c = tid; c < cc; c += kST) {
    const int cg = cv0 * V + c;
    const float sc = __ldg(a.scale + cg);
    const float al = -sc * __ldg(a.c2 + cg) * __ldg(a.invstd + cg);
    s_bn[c] = sc;
    s_bn[cst + c] = __ldg(a.shift + cg);
    s_bn[2 * cst + c] = al;
    s_bn[3 * cst + c] = -sc * __ldg(a.c1 + cg) - al * __ldg(a.mean + cg);
    if (XF) {
      s_bn[4 * cst + c] = __ldg(a.in_scale + cg);
      s_bn[5 * cst + c] = __ldg(a.in_shift + cg);
      s_bn[6 * cst + c] = red ? __ldg(a.zmean + cg) : 0.f;
    }
    s_red[c] = 0.f;
    s_red[cst + c] = 0.f;
  }
  __syncthreads();
  const int ppb = kST / ncv;
  const int cvl = tid % ncv, slot = tid / ncv;
  float wacc[KK][V];
  float lsum[V], lsq[V];
#pragma unroll
  for (int q = 0; q < KK; ++q)
#pragma unroll
    for (int i = 0; i < V; ++i) wacc[q][i] = 0.f;
#pragma unroll
  for (int i = 0; i < V; ++i) { lsum[i] = 0.f; lsq[i] = 0.f; }
  if (slot < ppb) {
    const int c0 = (cv0 + cvl) * V;
    const float* wl = s_w + cvl * V;
    const float* bnl = s_bn + cvl * V;
    const int rows = S == 1 ? F : (F + 1) / 2;
    const int strips = ceil_div(Tn, Q), segs = ceil_div(rows, a.seg_rows), units = strips * segs;
    long long g = ((long long)blockIdx.y * groups + grp) * ppb + slot;
    const long long gend = (long long)a.B * units;
    const long long gstep = (long long)gridDim.y * groups * ppb;
    for (; g < gend; g += gstep) {
      const int b = (int)(g / units);
      const int u = (int)(g - (long long)b * units);
      const int seg = u / strips, strip = u - seg * strips;
      const int m_a = seg * a.seg_rows;
      const int nstep = min(a.seg_rows, rows - m_a);
      const int t_a = strip * Q;                                 // even
      const int to_base = S == 1 ? t_a - PAD : t_a / 2 - PAD / 2;  // dz column of window index 0
      unsigned cmask = 0, qmask = 0;
#pragma unroll
      for (int j = 0; j < NDZ; ++j) cmask |= (to_base + j >= 0 && to_base + j < To) ? (1u << j) : 0u;
#pragma unroll
      for (int q = 0; q < Q; ++q) qmask |= (t_a + q < Tn) ? (1u << q) : 0u;
      float gt[V], dpl[V];
#pragma unroll
      for (int i = 0; i < V; ++i) {
        gt[i] = a.gate != nullptr ? __ldg(a.gate + (size_t)b * C + c0 + i) : 1.f;
        dpl[i] = a.dpool != nullptr ? __ldg(a.dpool + (size_t)b * C + c0 + i) : 0.f;
      }
      const size_t zoff = (size_t)b * Fo * To * C + c0, ioff = (size_t)b * F * Tn * C + c0;
      const float* dpp = a.dp + zoff + (long long)to_base * C;   // column j of dz row o: + (o * To + j) * C
      const float* zzp = a.z2 + zoff + (long long)to_base * C;
      const float* inp = a.in + ioff + (size_t)t_a * C;           // column q of input row i: + (i * Tn + q) * C
      float* dinp = a.din + ioff + (size_t)t_a * C;
      const float* resp = a.res != nullptr ? a.res + ioff + (size_t)t_a * C : nullptr;

      auto dz_of = [&](const float (&p)[V], const float (&z)[V], float (&o)[V]) {
        float sc[V], sh[V], al[V], be[V];
        VecF<V>::load(bnl, sc);
        VecF<V>::load(bnl + cst, sh);
        VecF<V>::load(bnl + 2 * cst, al);
        VecF<V>::load(bnl + 3 * cst, be);
#pragma unroll
        for (int i = 0; i < V; ++i) {
          const float gg = fmaf(p[i], gt[i], dpl[i]) * act_bwd(fmaf(z[i], sc[i], sh[i]), ACT);
          o[i] = fmaf(sc[i], gg, fmaf(al[i], z[i], be[i]));
        }
      };
      auto load_dz = [&](int o, float (&dst)[NDZ][V]) {          // synchronous: the window rows before the first step
#pragma unroll
        for (int j = 0; j < NDZ; ++j) {
          if (o >= 0 && o < Fo && ((cmask >> j) & 1u)) {
            float p[V], z[V];
            VecF<V>::load(dpp + ((size_t)o * To + j) * C, p);
            VecF<V>::load(zzp + ((size_t)o * To + j) * C, z);
            dz_of(p, z, dst[j]);
          } else {
#pragma unroll
            for (int i = 0; i < V; ++i) dst[j][i] = 0.f;
          }
        }
      };
      // step mm: dz row m - OB0 + LW - 1 (vectors 0 .. 2*NDZ-1: dp, z2) and input rows S*m .. S*m+S-1 (own columns)
      auto issue = [&](int mm, int slot_) {
        if (mm < nstep) {
          const int m = m_a + mm;
          const int o = m - OB0 + LW - 1;
          const uint32_t dst = ring0 + (uint32_t)(slot_ * NV) * (kST * VB);
          if (o >= 0 && o < Fo) {
#pragma unroll
            for (int j = 0; j < NDZ; ++j) {
              if ((cmask >> j) & 1u) {
                cp_async<VB>(dst + (uint32_t)j * (kST * VB), dpp + ((size_t)o * To + j) * C);
                cp_async<VB>(dst + (uint32_t)(NDZ + j) * (kST * VB), zzp + ((size_t)o * To + j) * C);
              }
            }
          }
#pragma unroll
          for (int r = 0; r < S; ++r) {
            const int irow = S * m + r;
            if (irow < F) {
#pragma unroll
              for (int q = 0; q < Q; ++q)
                if ((qmask >> q) & 1u) cp_async<VB>(dst + (uint32_t)(2 * NDZ + r * Q + q) * (kST * VB), inp + ((size_t)irow * Tn + q) * C);
            }
          }
        }
        cp_commit();
      };
      auto ring = [&](int slot_, int v, float (&dst)[V]) {
        VecF<V>::load(reinterpret_cast<const float*>(ringp + (size_t)(slot_ * NV + v) * (kST * VB)), dst);
      };

      for (int q = 0; q < kFbDepth; ++q) issue(q, q);
      float win[LW][NDZ][V];
#pragma unroll
      for (int l = 1; l < LW; ++l) load_dz(m_a - OB0 + l - 1, win[l]);
      int rs = 0;
      for (int mm = 0; mm < nstep; ++mm) {
        const int m = m_a + mm;
#pragma unroll
        for (int l = 0; l + 1 < LW; ++l)
#pragma unroll
          for (int j = 0; j < NDZ; ++j)
#pragma unroll
            for (int i = 0; i < V; ++i) win[l][j][i] = win[l + 1][j][i];
        cp_wait_pending(kFbDepth - 1);                          // this step's group has landed (own copies only)
        const int o = m - OB0 + LW - 1;
#pragma unroll
        for (int j = 0; j < NDZ; ++j) {
          if (o < Fo && ((cmask >> j) & 1u)) {
            float p[V], z[V];
            ring(rs, j, p);
            ring(rs, NDZ + j, z);
            dz_of(p, z, win[LW - 1][j]);
          } else {
#pragma unroll
            for (int i = 0; i < V; ++i) win[LW - 1][j][i] = 0.f;
          }
        }
        float xr[S][Q][V];                                      // raw input (z1 or the block input) at the own columns
#pragma unroll
        for (int r = 0; r < S; ++r)
#pragma unroll
          for (int q = 0; q < Q; ++q) {
            if (S * m + r < F && ((qmask >> q) & 1u)) ring(rs, 2 * NDZ + r * Q + q, xr[r][q]);
            else {
#pragma unroll
              for (int i = 0; i < V; ++i) xr[r][q][i] = 0.f;
            }
          }
        issue(mm + kFbDepth, rs);                               // the slot just read takes the step `depth` ahead
        if (++rs == kFbDepth) rs = 0;
        float isc[V], ish[V];
        if (XF) {
          VecF<V>::load(bnl + 4 * cst, isc);
          VecF<V>::load(bnl + 5 * cst, ish);
        }
#pragma unroll
        for (int r = 0; r < S; ++r) {
          const int irow = S * m + r;
          if (irow >= F) continue;
          float xf[Q][V];
#pragma unroll
          for (int q = 0; q < Q; ++q) {
            const bool ok = (qmask >> q) & 1u;
#pragma unroll
            for (int i = 0; i < V; ++i) xf[q][i] = XF ? (ok ? xact<ACT>(fmaf(xr[r][q][i], isc[i], ish[i])) : 0.f) : xr[r][q][i];
          }
          float acc[Q][V];
#pragma unroll
          for (int q = 0; q < Q; ++q)
#pragma unroll
            for (int i = 0; i < V; ++i) acc[q][i] = 0.f;
#pragma unroll
          for (int ky = 0; ky < K; ++ky) {
            if (S == 2 && ((r + PAD - ky) & 1) != 0) continue;
            const int sl = S == 1 ? 2 * PAD - ky : (r + PAD - ky) / 2 + PAD / 2;   // dz row (i + PAD - ky) / S
#pragma unroll
            for (int kx = 0; kx < K; ++kx) {
              float w[V];
              VecF<V>::load(wl + (ky * K + kx) * cst, w);
#pragma unroll
              for (int q = 0; q < Q; ++q) {
                if (S == 2 && ((q + PAD - kx) & 1) != 0) continue;
                const int j = S == 1 ? q + 2 * PAD - kx : (q + PAD - kx) / 2 + PAD / 2;   // dz column (t + PAD - kx) / S
                fma_vec<V>(win[sl][j], w, acc[q]);
                fma_vec<V>(win[sl][j], xf[q], wacc[ky * K + kx]);
              }
            }
          }
#pragma unroll
          for (int q = 0; q < Q; ++q) {
            if (!((qmask >> q) & 1u)) continue;
            const size_t off = ((size_t)irow * Tn + q) * C;
            if (resp != nullptr) {
              float rv[V];
              VecF<V>::load(resp + off, rv);
#pragma unroll
              for (int i = 0; i < V; ++i) acc[q][i] += rv[i];
            }
            VecF<V>::store(dinp + off, acc[q]);
            if (red) {
              float mu[V];
              VecF<V>::load(bnl + 6 * cst, mu);
#pragma unroll
              for (int i = 0; i < V; ++i) {
                const float gd = acc[q][i] * act_bwd(fmaf(xr[r][q][i], isc[i], ish[i]), ACT);
                lsum[i] += gd;
                lsq[i] = fmaf(gd, xr[r][q][i] - mu[i], lsq[i]);
              }
            }
          }
        }
      }
    }
#pragma unroll
    for (int q = 0; q < KK; ++q)
#pragma unroll
      for (int i = 0; i < V; ++i) atomicAdd(&s_acc[q * cst + cvl * V + i], wacc[q][i]);
    if (red) {
#pragma unroll
      for (int i = 0; i < V; ++i) { atomicAdd(&s_red[cvl * V + i], lsum[i]); atomicAdd(&s_red[cst + cvl * V + i], lsq[i]); }
    }
  }
  __syncthreads();
  for (int i = tid; i < KK * cc; i += kST) {
    const int q = i / cc, c = i - q * cc;
    atomicAdd(a.dw + (size_t)(cv0 * V + c) * KK + q, s_acc[q * cst + c]);
  }
  if (red) {
    for (int c = tid; c < cc; c += kST) {
      const int cg = cv0 * V + c;
      atomicAdd(a.s1 + cg, (double)s_red[c]);
      atomicAdd(a.s2 + cg, (double)s_red[cst + c] * (double)__ldg(a.zinvstd + cg));
    }
  }
}

template <int K, int S, int ACT, bool XF>
int launch_fb_one(const FusedBwdArgs& a, dim3 grid, size_t smem, cudaStream_t st) {
  static unsigned long long mask = 0;
  if (int rc = eat_opt_in_smem(dw_bwd_fused_kernel<K, S, ACT, XF>, 64 * 1024, mask)) return rc;
  dw_bwd_fused_kernel<K, S, ACT, XF><<<grid, kST, smem, st>>>(a);
  EAT_CHECK_LAUNCH();
  return EAT_OK;
}

// a step reads LW dz rows, consecutive steps share LW - 1 of them: the plan of a stride-1 walk with an LW-row kernel over
// the steps (din rows, or row pairs for stride 2) and Q-wide din strips
template <int K, int S>
SlidePlan plan_fb(int B, int F, int Tn, int C) {
  using Sh = FbShape<K, S>;
  const int rows = S == 1 ? F : (F + 1) / 2;
  return plan_slide(B, rows, Tn, C / Sh::V, Sh::V, Sh::Q, 1, Sh::LW, Sh::MINB, false, kFbCvcMax);
}

template <int K, int S>
int launch_fb(FusedBwdArgs a, int act, bool xf, cudaStream_t st) {
  using Sh = FbShape<K, S>;
  const SlidePlan pl = plan_fb<K, S>(a.B, a.F, a.Tn, a.C);
  a.chunks = pl.chunks; a.cvc = pl.cvc; a.seg_rows = pl.seg_rows;
  dim3 grid(pl.chunks * pl.groups, pl.gy);
  const size_t smem = (size_t)(2 * K * K + 9) * a.cvc * Sh::V * sizeof(float) +
                      (size_t)kFbDepth * Sh::NV * kST * Sh::V * sizeof(float);
  if (act == EAT_ACT_RELU) return xf ? launch_fb_one<K, S, EAT_ACT_RELU, true>(a, grid, smem, st)
                                     : launch_fb_one<K, S, EAT_ACT_RELU, false>(a, grid, smem, st);
  return xf ? launch_fb_one<K, S, EAT_ACT_HSWISH, true>(a, grid, smem, st)
            : launch_fb_one<K, S, EAT_ACT_HSWISH, false>(a, grid, smem, st);
}

}  // namespace

extern "C" int eat_dw_conv_bwd_fused(const float* dp, const float* gate, const float* dpool, const float* z2,
                                     const float* scale, const float* shift, const float* mean, const float* invstd, int act,
                                     const float* c1, const float* c2, const float* wt, const float* in,
                                     const float* in_scale, const float* in_shift, int in_act, const float* res, float* din,
                                     float* dw, const float* zmean, const float* zinvstd, double* s1, double* s2, int dtype,
                                     int B, int F, int T, int C, int k, int stride, cudaStream_t st) {
  if (dtype != EAT_F32) { eat_set_error("dw_conv_bwd_fused: fp32 storage only"); return EAT_ERR_UNSUPPORTED; }
  if ((k != 3 && k != 5) || (stride != 1 && stride != 2)) {
    eat_set_error("dw_conv_bwd_fused: k in {3,5}, stride in {1,2} only");
    return EAT_ERR_UNSUPPORTED;
  }
  const int V = k == 3 ? 4 : 2;
  if (C <= 0 || C % V != 0) {
    eat_set_error(k == 3 ? "dw_conv_bwd_fused: 3x3 needs channels in multiples of 4" : "dw_conv_bwd_fused: 5x5 needs channels in multiples of 2");
    return EAT_ERR_UNSUPPORTED;
  }
  if (act != EAT_ACT_RELU && act != EAT_ACT_HSWISH) { eat_set_error("dw_conv_bwd_fused: activation must be relu or hardswish"); return EAT_ERR_UNSUPPORTED; }
  if (in_scale != nullptr && (in_shift == nullptr || in_act != act)) {
    eat_set_error("dw_conv_bwd_fused: the input transform needs in_shift and the block's activation (in_act == act)");
    return EAT_ERR_UNSUPPORTED;
  }
  if (dp == nullptr || z2 == nullptr || scale == nullptr || shift == nullptr || mean == nullptr || invstd == nullptr ||
      c1 == nullptr || c2 == nullptr || wt == nullptr || in == nullptr || din == nullptr || dw == nullptr) {
    eat_set_error("dw_conv_bwd_fused: dp, z2, the BN2 tables, c1/c2, wt, in, din and dw are required");
    return EAT_ERR_ARG;
  }
  if (s1 != nullptr && (s2 == nullptr || zmean == nullptr || zinvstd == nullptr || in_scale == nullptr)) {
    eat_set_error("dw_conv_bwd_fused: the BN1 reduce needs s2, zmean, zinvstd and the input transform");
    return EAT_ERR_ARG;
  }
  if (B < 0 || F < 0 || T < 0) { eat_set_error("dw_conv_bwd_fused: negative shape"); return EAT_ERR_ARG; }
  if (B == 0 || F == 0 || T == 0) return EAT_OK;
  const int pad = (k - 1) / 2;
  FusedBwdArgs a;
  a.dp = dp; a.gate = gate; a.dpool = dpool; a.z2 = z2;
  a.scale = scale; a.shift = shift; a.mean = mean; a.invstd = invstd; a.c1 = c1; a.c2 = c2;
  a.wt = wt; a.in = in; a.in_scale = in_scale; a.in_shift = in_shift; a.res = res; a.din = din; a.dw = dw;
  a.zmean = zmean; a.zinvstd = zinvstd; a.s1 = s1; a.s2 = s2;
  a.B = B; a.F = F; a.Tn = T; a.C = C;
  a.Fo = (F + 2 * pad - k) / stride + 1;
  a.To = (T + 2 * pad - k) / stride + 1;
  const bool xf = in_scale != nullptr;
  if (k == 3) return stride == 1 ? launch_fb<3, 1>(a, act, xf, st) : launch_fb<3, 2>(a, act, xf, st);
  return stride == 1 ? launch_fb<5, 1>(a, act, xf, st) : launch_fb<5, 2>(a, act, xf, st);
}

namespace {
// dil 2 (stride 1, padding 2 * (k-1)/2): the output has the input's size
int slide_launch(const void* in, const float* wt, void* out, int dtype, int B, int F, int Tn, int C, int k, int stride,
                 int dil, InXform xf, const float* scale, const float* shift, int act, const void* res, int flip,
                 float* pool, double* ssum, double* ssq, cudaStream_t st, DyEpi dy, int dyk = 2) {
  const int V = dtype == EAT_BF16 ? 8 : 4;
  if (C % V != 0) { eat_set_error("dw conv: channels must be a multiple of the vector width"); return EAT_ERR_ARG; }
  const int pad = (k - 1) / 2 * dil;
  SlideArgs a;
  a.in = in; a.wt = wt; a.out = out;
  a.F = F; a.Tn = Tn; a.C = C;
  a.Fo = (F + 2 * pad - dil * (k - 1) - 1) / stride + 1;
  a.To = (Tn + 2 * pad - dil * (k - 1) - 1) / stride + 1;
  a.xscale = xf.scale; a.xshift = xf.shift;
  a.scale = scale; a.shift = shift; a.act = act;
  a.res = res; a.flip = flip; a.pool = pool; a.stat_sum = ssum; a.stat_sq = ssq; a.dy = dy;
  const int mode = (scale != nullptr || pool != nullptr || dy.theta != nullptr || dy.ca_f != nullptr) ? 1 : ((flip || res != nullptr) ? 2 : 0);
  const int xact_code = xf.scale != nullptr ? xf.act : -1;
  if (mode != 0 && xf.scale != nullptr) { eat_set_error("dw slide: input transform only in training-forward mode"); return EAT_ERR_UNSUPPORTED; }
  if (dil == 2) {
    if (dtype == EAT_BF16) return launch_slide<__nv_bfloat16, 2>(a, B, k, stride, mode, xact_code, st);
    return launch_slide<float, 2>(a, B, k, stride, mode, xact_code, st);
  }
  if (dtype == EAT_BF16) return launch_slide<__nv_bfloat16>(a, B, k, stride, mode, xact_code, st, dyk);
  return launch_slide<float>(a, B, k, stride, mode, xact_code, st, dyk);
}

int wgrad_slide_launch(const void* dz, const void* in, InXform xf, float* dw, long long dw_bstride, int dtype, int B,
                       int F, int Tn, int C, int k, int stride, int dil, cudaStream_t st) {
  const int V = dtype == EAT_BF16 ? 8 : 4;
  if (C % V != 0) { eat_set_error("dw wgrad: channels must be a multiple of the vector width"); return EAT_ERR_ARG; }
  if (dil == 1 && !((k == 3 || (k == 5 && dtype != EAT_BF16)) && (stride == 1 || stride == 2))) {
    eat_set_error("dw wgrad slide: 3x3 (fp32, bf16) or 5x5 (fp32), stride 1 or 2");
    return EAT_ERR_UNSUPPORTED;
  }
  const int pad = (k - 1) / 2 * dil;
  WgArgs a;
  a.dz = dz; a.in = in; a.dw = dw; a.dw_bstride = dw_bstride;
  a.B = B; a.F = F; a.Tn = Tn; a.C = C;
  a.Fo = (F + 2 * pad - dil * (k - 1) - 1) / stride + 1;
  a.To = (Tn + 2 * pad - dil * (k - 1) - 1) / stride + 1;
  a.xscale = xf.scale; a.xshift = xf.shift;
  const int xact_code = xf.scale != nullptr ? xf.act : -1;
  if (dil == 2) {          // the bf16 5x5 instance takes 4 channels per thread: 25 x 8 accumulators would spill
    if (dtype == EAT_BF16) return k == 5 ? launch_wg_slide<__nv_bfloat16, 5, 4, 1, 3, 2>(a, stride, xact_code, st)
                                         : launch_wg_slide<__nv_bfloat16, 3, 8, 1, 3, 2>(a, stride, xact_code, st);
    if (k == 5) return launch_wg_slide<float, 5, 2, 4, 3, 2>(a, stride, xact_code, st);
    return launch_wg_slide<float, 3, 4, 4, 3, 2>(a, stride, xact_code, st);
  }
  if (dtype == EAT_BF16) return launch_wg_slide<__nv_bfloat16, 3, 8, 1, 3>(a, stride, xact_code, st);
  if (k == 5) return launch_wg_slide<float, 5, 2, 4, 3>(a, stride, xact_code, st);
  return launch_wg_slide<float, 3, 4, 4, 3>(a, stride, xact_code, st);
}

// argument checks of the dilated entry points, before any launch
int dil_check(const char* who, int dtype, int B, int F, int T, int C, int k, int stride, int dilation) {
  char msg[160];
  int rc = EAT_OK;
  if (dtype != EAT_F32 && dtype != EAT_BF16) { snprintf(msg, sizeof msg, "%s: dtype must be fp32 (0) or bf16 (1)", who); rc = EAT_ERR_ARG; }
  else if (B < 0 || F < 1 || T < 1 || C < 1) { snprintf(msg, sizeof msg, "%s: B >= 0 and F, T, C >= 1 required", who); rc = EAT_ERR_ARG; }
  else if (dilation != 2) { snprintf(msg, sizeof msg, "%s: dilation must be 2 (got %d)", who, dilation); rc = EAT_ERR_UNSUPPORTED; }
  else if (stride != 1) { snprintf(msg, sizeof msg, "%s: a dilated layer runs at stride 1 (got %d)", who, stride); rc = EAT_ERR_UNSUPPORTED; }
  else if (k != 3 && k != 5) { snprintf(msg, sizeof msg, "%s: k must be 3 or 5 (got %d)", who, k); rc = EAT_ERR_UNSUPPORTED; }
  else if (C % (dtype == EAT_BF16 ? 8 : 4) != 0) {
    snprintf(msg, sizeof msg, "%s: C must be a multiple of %d for %s storage (got %d)", who, dtype == EAT_BF16 ? 8 : 4,
             dtype == EAT_BF16 ? "bf16" : "fp32", C);
    rc = EAT_ERR_ARG;
  }
  if (rc != EAT_OK) eat_set_error(msg);
  return rc;
}
}  // namespace

int dw_slide_launch(const void* in, const float* wt, void* out, int dtype, int B, int F, int Tn, int C, int k, int stride,
                    InXform xf, const float* scale, const float* shift, int act, const void* res, int flip, float* pool,
                    double* ssum, double* ssq, cudaStream_t st, DyEpi dy, int dyk) {
  return slide_launch(in, wt, out, dtype, B, F, Tn, C, k, stride, 1, xf, scale, shift, act, res, flip, pool, ssum, ssq, st, dy,
                      dyk);
}

int dw_wgrad_slide_launch(const void* dz, const void* in, InXform xf, float* dw, long long dw_bstride, int dtype, int B,
                          int F, int Tn, int C, int k, int stride, cudaStream_t st) {
  return wgrad_slide_launch(dz, in, xf, dw, dw_bstride, dtype, B, F, Tn, C, k, stride, 1, st);
}

extern "C" int eat_dw_conv_fwd_dil(const void* in, const float* wt, void* out, int dtype, int B, int F, int T, int C, int k,
                                   int stride, int dilation, const float* in_scale, const float* in_shift, int in_act,
                                   const float* scale, const float* shift, int act, float* pool, double* stat_sum,
                                   double* stat_sq, cudaStream_t st) {
  if (int rc = dil_check("dw_conv_fwd_dil", dtype, B, F, T, C, k, stride, dilation)) return rc;
  if (in_scale != nullptr && (scale != nullptr || pool != nullptr)) {
    eat_set_error("dw_conv_fwd_dil: the input transform is for the training forward (no scale, shift or pool)");
    return EAT_ERR_ARG;
  }
  if ((scale == nullptr) != (shift == nullptr) || (in_scale == nullptr) != (in_shift == nullptr) ||
      (stat_sum == nullptr) != (stat_sq == nullptr)) {
    eat_set_error("dw_conv_fwd_dil: scale/shift, in_scale/in_shift and stat_sum/stat_sq come in pairs");
    return EAT_ERR_ARG;
  }
  if (B == 0) return EAT_OK;
  InXform xf{in_scale, in_shift, nullptr, in_act, 0};
  return slide_launch(in, wt, out, dtype, B, F, T, C, k, stride, dilation, xf, scale, shift, act, nullptr, 0, pool,
                      stat_sum, stat_sq, st, DyEpi{nullptr, nullptr, nullptr, nullptr, nullptr, 0});
}

extern "C" int eat_dw_conv_dgrad_dil(const void* dz, const float* wt, const void* res, void* din, int dtype, int B, int F,
                                     int T, int C, int k, int stride, int dilation, cudaStream_t st) {
  if (int rc = dil_check("dw_conv_dgrad_dil", dtype, B, F, T, C, k, stride, dilation)) return rc;
  if (B == 0) return EAT_OK;
  InXform xf{nullptr, nullptr, nullptr, 0, 0};
  return slide_launch(dz, wt, din, dtype, B, F, T, C, k, stride, dilation, xf, nullptr, nullptr, 0, res, 1, nullptr,
                      nullptr, nullptr, st, DyEpi{nullptr, nullptr, nullptr, nullptr, nullptr, 0});
}

extern "C" int eat_dw_conv_wgrad_dil(const void* dz, const void* in, const float* in_scale, const float* in_shift,
                                     int in_act, float* dw, int dtype, int B, int F, int T, int C, int k, int stride,
                                     int dilation, cudaStream_t st) {
  if (int rc = dil_check("dw_conv_wgrad_dil", dtype, B, F, T, C, k, stride, dilation)) return rc;
  if ((in_scale == nullptr) != (in_shift == nullptr)) {
    eat_set_error("dw_conv_wgrad_dil: in_scale and in_shift come in pairs");
    return EAT_ERR_ARG;
  }
  if (B == 0) return EAT_OK;
  InXform xf{in_scale, in_shift, nullptr, in_act, 0};
  return wgrad_slide_launch(dz, in, xf, dw, 0, dtype, B, F, T, C, k, stride, dilation, st);
}

int dw_dgrad2_slide_launch(const void* dz, const float* wt, long long wt_bstride, const void* res, void* din, int dtype,
                           int B, int F, int Tn, int C, int k, cudaStream_t st, const void* z, const float* zscale,
                           const float* zshift, const float* zmean, const float* zinvstd, int zact, double* s1,
                           double* s2) {
  const int V = dtype == EAT_BF16 ? 8 : 4;
  if (C % V != 0) { eat_set_error("dw dgrad: channels must be a multiple of the vector width"); return EAT_ERR_ARG; }
  if (k != 3 && k != 5) { eat_set_error("dw dgrad slide: k in {3,5} only"); return EAT_ERR_UNSUPPORTED; }
  const int pad = (k - 1) / 2;
  Dg2Args a;
  a.dz = dz; a.wt = wt; a.wt_bstride = wt_bstride; a.res = res; a.din = din;
  a.z = z; a.zscale = zscale; a.zshift = zshift; a.zmean = zmean; a.zinvstd = zinvstd; a.zact = zact; a.s1 = s1; a.s2 = s2;
  a.B = B; a.F = F; a.Tn = Tn; a.C = C;
  a.Fo = (F + 2 * pad - k) / 2 + 1;
  a.To = (Tn + 2 * pad - k) / 2 + 1;
  if (dtype == EAT_BF16) return launch_dg2_slide<__nv_bfloat16>(a, k, st);
  return launch_dg2_slide<float>(a, k, st);
}

extern "C" int eat_dw_plan(int kind, int dtype, int B, int F, int T, int C, int k, int stride, int per_sample, int* plan) {
  const int V0 = kind == 3 ? (k == 5 ? 2 : 4) : (dtype == EAT_BF16 ? 8 : 4);
  if (plan == nullptr || B < 1 || F < 1 || T < 1 || C % V0 != 0 || (k != 3 && k != 5) || (stride != 1 && stride != 2)) {
    eat_set_error("dw_plan: invalid arguments");
    return EAT_ERR_ARG;
  }
  if (kind == 3) {                                   // dw_bwd_fused_kernel: steps (din rows / row pairs), Q din columns
    if (dtype != EAT_F32) { eat_set_error("dw_plan: the fused depthwise backward is fp32 only"); return EAT_ERR_UNSUPPORTED; }
    SlidePlan pl;
    int Q;
    if (k == 3 && stride == 1) { pl = plan_fb<3, 1>(B, F, T, C); Q = FbShape<3, 1>::Q; }
    else if (k == 3) { pl = plan_fb<3, 2>(B, F, T, C); Q = FbShape<3, 2>::Q; }
    else if (stride == 1) { pl = plan_fb<5, 1>(B, F, T, C); Q = FbShape<5, 1>::Q; }
    else { pl = plan_fb<5, 2>(B, F, T, C); Q = FbShape<5, 2>::Q; }
    plan[0] = pl.chunks; plan[1] = pl.cvc; plan[2] = pl.seg_rows; plan[3] = pl.groups; plan[4] = pl.gy; plan[5] = Q;
    return EAT_OK;
  }
  const bool f32 = dtype != EAT_BF16;
  const int pad = (k - 1) / 2;
  const int Fo = (F + 2 * pad - k) / stride + 1, To = (T + 2 * pad - k) / stride + 1;
  int V = V0, P, minb, rows, cols, S = stride, Kp = k;
  if (kind == 0) {                                   // launch_slide
    P = (k == 3 && stride == 1) ? (f32 ? 4 : 2) : (f32 ? 2 : 1);
    minb = k == 3 ? (stride == 1 ? 4 : 5) : 3;
    rows = Fo; cols = To;
  } else if (kind == 1) {                            // launch_wg_slide
    if (k == 5 && !f32) { eat_set_error("dw_plan: the bf16 5x5 weight gradient uses the tile kernel"); return EAT_ERR_UNSUPPORTED; }
    V = f32 ? (k == 5 ? 2 : 4) : 8;
    P = f32 ? 4 : 1;
    minb = 3;
    rows = Fo; cols = To;
  } else if (kind == 2) {                            // launch_dg2_slide: pairs of din rows, 4 din columns per strip
    if (stride != 2) { eat_set_error("dw_plan: kind 2 is the stride-2 data gradient"); return EAT_ERR_ARG; }
    P = 4; minb = k == 3 ? 4 : 3;
    rows = (F + 1) / 2; cols = T; S = 1; Kp = (k + 1) / 2;
  } else {
    eat_set_error("dw_plan: kind must be 0, 1, 2 or 3");
    return EAT_ERR_ARG;
  }
  const SlidePlan pl = plan_slide(B, rows, cols, C / V, V, P, S, Kp, minb, per_sample != 0);
  plan[0] = pl.chunks; plan[1] = pl.cvc; plan[2] = pl.seg_rows; plan[3] = pl.groups; plan[4] = pl.gy; plan[5] = P;
  return EAT_OK;
}
