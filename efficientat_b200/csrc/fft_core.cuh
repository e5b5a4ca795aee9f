// Stockham passes for an M-point complex FFT (= 2M-point real FFT after the split step), M a power of two
// in [128, 2048]: floor(log8 M) radix-8 passes, then one radix-2 or radix-4 pass when log2 M is not a multiple
// of 3.  A work group of M/8 threads holds 8 complex values per thread.  Written __host__ __device__ so the exact
// index/twiddle logic is unit-tested on the CPU (tests/test_fft_core.py and tests/test_fft_sizes.py compile this
// header with g++).
#pragma once
#if defined(__CUDACC__)
#define EAT_HD __host__ __device__ __forceinline__
#else
#define EAT_HD inline
struct float2 { float x, y; };
static inline float2 make_float2(float x, float y) { float2 r; r.x = x; r.y = y; return r; }
#endif

EAT_HD float2 cmul(float2 a, float2 b) { return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }
EAT_HD float2 cadd(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
EAT_HD float2 csub(float2 a, float2 b) { return make_float2(a.x - b.x, a.y - b.y); }
EAT_HD float2 cmul_mi(float2 a) { return make_float2(a.y, -a.x); }   // a * (-i)

EAT_HD void bfly2(float2& a, float2& b) { float2 t = a; a = cadd(t, b); b = csub(t, b); }

// in-register 8-point DFT (forward, e^{-i...}); result in natural order in v[0..7]
EAT_HD void fft8(float2 (&v)[8]) {
  const float h = 0.70710678118654752440f;
  bfly2(v[0], v[4]); bfly2(v[1], v[5]); bfly2(v[2], v[6]); bfly2(v[3], v[7]);
  v[5] = cmul(v[5], make_float2(h, -h));
  v[6] = cmul_mi(v[6]);
  v[7] = cmul(v[7], make_float2(-h, -h));
  // two 4-point DFTs on (0,1,2,3) and (4,5,6,7)
  bfly2(v[0], v[2]); bfly2(v[1], v[3]); v[3] = cmul_mi(v[3]); bfly2(v[0], v[1]); bfly2(v[2], v[3]);
  bfly2(v[4], v[6]); bfly2(v[5], v[7]); v[7] = cmul_mi(v[7]); bfly2(v[4], v[5]); bfly2(v[6], v[7]);
  // outputs are bit-reversed: X0=v0 X1=v4 X2=v2 X3=v6 X4=v1 X5=v5 X6=v3 X7=v7
  float2 t1 = v[1], t3 = v[3], t4 = v[4], t6 = v[6];
  v[1] = t4; v[3] = t6; v[4] = t1; v[6] = t3;
}

// One radix-8 Stockham pass of an M-point FFT, work item j in [0, M/8): twiddle + butterfly on 8 values already
// in v (v[r] = in[j + (M/8) r]), Ns = 8^pass < M; tw[m] = exp(-2 pi i m / M).
EAT_HD void stockham8_compute_m(float2 (&v)[8], int j, int Ns, int M, const float2* tw) {
  if (Ns > 1) {
    int k = j & (Ns - 1);
    int step = M / (Ns * 8);
#pragma unroll
    for (int r = 1; r < 8; ++r) v[r] = cmul(v[r], tw[r * k * step]);
  }
  fft8(v);
}
// the M = 512 case (1024-point real FFT), Ns in {1, 8, 64}
EAT_HD void stockham8_compute(float2 (&v)[8], int j, int Ns, const float2* tw) { stockham8_compute_m(v, j, Ns, 512, tw); }

// destination index of output r of work item j (any M)
EAT_HD int stockham8_dst(int j, int Ns, int r) {
  int k = j & (Ns - 1);
  return (j - k) * 8 + k + r * Ns;
}

// Last pass when log2 M = 3p + 1: radix 2 at Ns = M/2.  Thread j of M/8 holds v[r] = in[j + (M/8) r]; its four
// work items are jj = j + (M/8) q, q < 4, on the pairs (v[q], v[q+4]), twiddle exp(-2 pi i jj / M).  Every output
// lands where its work item's inputs came from (dst = jj + r M/2), so the pass is in place: v[r] -> out[j + (M/8) r].
EAT_HD void stockham2_tail(float2 (&v)[8], int j, int M, const float2* tw) {
  const int g = M / 8;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    float2 a = v[q], b = cmul(v[q + 4], tw[j + g * q]);
    v[q] = cadd(a, b);
    v[q + 4] = csub(a, b);
  }
}

// Last pass when log2 M = 3p + 2: radix 4 at Ns = M/4.  Work items jj = j + (M/8) q, q < 2, on
// (v[q], v[q+2], v[q+4], v[q+6]), twiddles exp(-2 pi i r jj / M); in place like the radix-2 tail (dst = jj + r M/4).
EAT_HD void stockham4_tail(float2 (&v)[8], int j, int M, const float2* tw) {
  const int g = M / 8;
#pragma unroll
  for (int q = 0; q < 2; ++q) {
    const int jj = j + g * q;
    float2 a0 = v[q], a1 = cmul(v[q + 2], tw[jj]), a2 = cmul(v[q + 4], tw[2 * jj]), a3 = cmul(v[q + 6], tw[3 * jj]);
    float2 t0 = cadd(a0, a2), t1 = csub(a0, a2), t2 = cadd(a1, a3), t3 = cmul_mi(csub(a1, a3));
    v[q] = cadd(t0, t2);
    v[q + 2] = cadd(t1, t3);
    v[q + 4] = csub(t0, t2);
    v[q + 6] = csub(t1, t3);
  }
}

// Real-FFT split: given Z = FFT_M(x[2n] + i x[2n+1]), returns X[k] of the 2M-point real FFT for k in [0, M);
// w = exp(-2 pi i k / 2M).  (X[M] = Re Z0 - Im Z0.)
EAT_HD float2 rfft_split(float2 zk, float2 zmk, float2 w) {
  // E = (Zk + conj(Zmk))/2 ; O = -i (Zk - conj(Zmk))/2 ; X = E + w O
  float2 e = make_float2(0.5f * (zk.x + zmk.x), 0.5f * (zk.y - zmk.y));
  float2 d = make_float2(0.5f * (zk.x - zmk.x), 0.5f * (zk.y + zmk.y));
  float2 o = make_float2(d.y, -d.x);
  return cadd(e, cmul(w, o));
}
