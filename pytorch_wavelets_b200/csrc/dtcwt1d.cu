// dtcwt1d.cu -- the 1-D dual-tree complex wavelet transform's level kernels (sm_90a), float and double.
//
// One kernel per level and direction computes both filters of the level (both trees at levels >= 2):
//   FWD1  lo = colfilter(x, h0), hi = colfilter(x, h1)                     12 B / sample (float)
//   FWD2  lo = coldfilt(x, h0b, h0a), hi = coldfilt(x, h1b, h1a, hp)        8 B / input sample
//   INV1  y = colfilter(lo, g0) + colfilter(hi, g1)                        12 B / sample
//   INV2  y = colifilt(lo, g0b, g0a) + colifilt(hi, g1b, g1a, hp)          16 B / low-pass coefficient
// A CTA stages the input window of its outputs -- the segment plus a halo on each side -- in shared memory once: the
// 16-byte aligned middle with cp.async.cg, the unaligned head and tail and the positions outside the row with scalar
// loads that resolve the symmetric (any number of reflections) or zero extension.  Both branches read the staged copy.
// Work is counted in units: one output sample (FWD1 / INV1), one output pair of each of lo and hi (FWD2, 4 input
// samples) or four output samples (INV2, 2 samples of each input).  Two CTA shapes:
//   long rows   one segment of KindInfo::seg units (2048 samples of each input) of one row per CTA;
//   packed      whole rows, as many as fit KindInfo::seg units and kPackSmem bytes of staging, per CTA, when at
//               least two fit.
// Consecutive threads take consecutive units, so every warp stores contiguous runs.  Accumulation is the oracle's and
// k_prims.cu's: a product, then fused multiply-adds in stored-tap order; the inverses round each branch and add them
// with add_rn, so the results are bit-identical to the oracle primitives in both precisions.
// k_scat1d runs FWD1 / FWD2 with the scattering epilogue of ScatLayer1D / ScatLayer1Dj2 (pooled low-pass, smoothed
// magnitude of each (re, im) band-pass pair, optionally its derivatives) on the same body, so its filter outputs are
// those of k_dt1d; k_dt1d itself compiles to the same code as without the epilogue.
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.h"
#include "launch.cuh"

namespace b200w {
namespace dt1d {

enum Kind { FWD1 = 0, FWD2 = 1, INV1 = 2, INV2 = 3 };

constexpr int kThreads = 256;
constexpr int kPackSmem = 48 * 1024;   // staging budget of a packed CTA

// Scattering epilogue of the forward kernels (k_scat1d): SC = 0 none, SC_MAG smoothed magnitude, SC_DER magnitude and
// its derivatives.  A level-1 unit is then one output pair (x[2q], x[2q + 1]) of each filter.
enum Scat { SC_NONE = 0, SC_MAG = 1, SC_DER = 2 };

// input samples per unit, staged inputs, units per long-row segment (2048 input samples of each input)
template <int K, int SC = SC_NONE> struct KindInfo {
  static constexpr int ipu = K == FWD2 ? 4 : (K == INV2 || (K == FWD1 && SC != SC_NONE) ? 2 : 1);
  static constexpr int nin = (K == INV1 || K == INV2) ? 2 : 1;
  static constexpr int seg = 2048 / ipu;
};

template <class T>
struct Dt1dParams {
  const T* in0; long long pitch0;   // x (forward) / lo (inverse; may be null)
  const T* in1;                     // hi (inverse; may be null), row pitch nin
  T* out0; T* out1;                 // lo, hi (forward; hi may be null) / y (inverse; out1 unused)
  int rows, nin, nout;              // rows, input and output row lengths
  int units, seg, rpc, nseg;        // units per row; units per CTA row segment; rows per CTA; segments per row
  int halo, srow;                   // staged halo on each side; shared-memory row stride (elements)
  int L0, L1;                       // level 1: filter lengths; levels >= 2: L0 = m
  int sym;                          // 1 symmetric extension, 0 zero padding (level 1 only)
  // level 1: a0 = branch-0 filter (h0 / g0), a1 = branch-1 filter (h1 / g1);
  // levels >= 2: (ha, hb) of the coldfilt / colifilt call of branch 0 (low-pass) and branch 1 (high-pass)
  TapsT<T> a0, b0, a1, b1;
};

// The scattering forms append their outputs, so the plain kernels' parameter layout is the one above.  Row r = b * C + c
// of an output of row length m (= units) is at base + b * bstride + c * m: out0 = low-pass (2x pooled, or at level 1
// the full-length low-pass when !pool), mag = sqrt(re^2 + im^2 + b^2) - b, dre / dim = re / r, im / r (SC_DER).
template <class T>
struct Scat1dParams : Dt1dParams<T> {
  T* mag; T* dre; T* dim;
  long long bs_lo, bs_mag, bs_dre, bs_dim;
  int C, pool;
  T magbias, magbias2;              // b and T(b * b), the product in double
};

__device__ __forceinline__ void cp_async16(void* sdst, const void* gsrc) {
  const unsigned s = (unsigned)__cvta_generic_to_shared(sdst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(__cvta_generic_to_global(gsrc)) : "memory");
}

// element misalignment of a row start w.r.t. 16 bytes
template <class T>
__device__ __forceinline__ int misalign(const T* row) {
  return (int)(((uintptr_t)row / sizeof(T)) & (16 / sizeof(T) - 1));
}

// a = h[0] x[0] then a = fma(h[j * TS], x[j * XS], a) for j < count; LC > 0: count compiled in
template <int LC, int TS, int XS, class T>
__device__ __forceinline__ T corr(const T* h, const T* x, int count) {
  T a = mul_rn(h[0], x[0]);
  if (LC > 0) {
#pragma unroll
    for (int j = 1; j < LC; ++j) a = fma_rn(h[j * TS], x[j * XS], a);
  } else {
    for (int j = 1; j < count; ++j) a = fma_rn(h[j * TS], x[j * XS], a);
  }
  return a;
}

// One of the four y[4t + s] of colifilt (k_prims.cu k_ifilt): x at window index of 2t - m2 (step 2).
template <int M2, bool HP, int S, class T>
__device__ __forceinline__ T ifilt_phase(const T* ha, const T* hb, const T* x, int m2) {
  const bool even = ((m2 & 1) == 0);
  const int par = even ? (S >= 2 ? 1 : 0) : (S < 2 ? 1 : 0);
  const int o = even ? (HP ? (S ^ 1) : S) : (HP ? (2 - (S & 1)) : (1 + (S & 1)));
  const T* h = (S & 1) ? hb : ha;
  return corr<M2, 2, 2>(h + par, x + o, m2);
}

template <bool HP, int M2, class T>
__device__ __forceinline__ void ifilt4(const T* ha, const T* hb, const T* x, int m2, T* y) {
  y[0] = ifilt_phase<M2, HP, 0>(ha, hb, x, m2);
  y[1] = ifilt_phase<M2, HP, 1>(ha, hb, x, m2);
  y[2] = ifilt_phase<M2, HP, 2>(ha, hb, x, m2);
  y[3] = ifilt_phase<M2, HP, 3>(ha, hb, x, m2);
}

template <class T>
__device__ __forceinline__ T sum2(bool h0, T a, bool h1, T b) {
  return h0 ? (h1 ? add_rn(a, b) : a) : (h1 ? b : (T)0);
}

// One (lo, hi) output pair of a forward level into the scattering outputs of row `row`, position q.
template <int SC, class T>
__device__ __forceinline__ void scat_store(const Scat1dParams<T>& p, int row, int q, T lo0, T lo1, T re, T im) {
  const int b = row / p.C, c = row - b * p.C;
  const long long o = (long long)c * p.units + q;
  if (p.pool) {
    p.out0[b * p.bs_lo + o] = mul_rn(add_rn(lo0, lo1), (T)0.5);
  } else {
    const long long ol = b * p.bs_lo + 2 * o;
    p.out0[ol] = lo0;
    p.out0[ol + 1] = lo1;
  }
  const T r = sqrt_rn(add_rn(add_rn(mul_rn(re, re), mul_rn(im, im)), p.magbias2));
  p.mag[b * p.bs_mag + o] = sub_rn(r, p.magbias);
  if (SC == SC_DER) {
    p.dre[b * p.bs_dre + o] = div_rn(re, r);
    p.dim[b * p.bs_dim + o] = div_rn(im, r);
  }
}

// The body of every level kernel.  LA, LB: level-1 filter lengths (branch 0, branch 1); levels >= 2: LA = m.
// 0 = runtime length.  P is Dt1dParams<T>, or Scat1dParams<T> when SC != SC_NONE.
template <class T, int K, int LA, int LB, bool PACK, int SC, class P>
__device__ __forceinline__ void dt1d_body(const P& p) {
  using KI = KindInfo<K, SC>;
  constexpr int VEC = 16 / (int)sizeof(T);
  extern __shared__ __align__(16) unsigned char smem_raw[];
  T* smem = reinterpret_cast<T*>(smem_raw);

  int row0, u0, useg, nrows;
  if (PACK) {
    row0 = blockIdx.x * p.rpc; u0 = 0; useg = p.units; nrows = imin(p.rpc, p.rows - row0);
  } else {
    row0 = blockIdx.x / p.nseg; u0 = (blockIdx.x - row0 * p.nseg) * p.seg; useg = imin(p.seg, p.units - u0); nrows = 1;
  }
  const int g0 = u0 * KI::ipu - p.halo;           // input index of window position 0
  const int win = useg * KI::ipu + 2 * p.halo;    // window length

  // ---- stage the windows ----
#pragma unroll
  for (int a = 0; a < KI::nin; ++a) {
    const T* base = a == 0 ? p.in0 : p.in1;
    if (!base) continue;
    const long long pitch = a == 0 ? p.pitch0 : p.nin;
    T* sa = smem + (size_t)a * p.rpc * p.srow;
    const int cpr = win / VEC + 2;                // 16-byte chunks per row, upper bound
    const int epr = 2 * p.halo + 2 * VEC;         // scalar positions per row, upper bound
    for (int e = threadIdx.x; e < nrows * (cpr + epr); e += kThreads) {
      const int r = e / (cpr + epr), c = e - r * (cpr + epr);
      const T* xr = base + (long long)(row0 + r) * pitch;
      const int mis = misalign(xr);
      const int lo = imax(g0, 0), hi = imin(g0 + win, p.nin);   // in-row part of the window
      int alo = lo + ((VEC - ((mis + lo) & (VEC - 1))) & (VEC - 1));
      int ahi = hi - ((mis + hi) & (VEC - 1));
      if (ahi <= alo) alo = ahi = lo;
      T* sr = sa + (size_t)r * p.srow + ((mis + g0) & (VEC - 1)) - g0;   // sr[g] = staged sample g
      if (c < cpr) {
        const int g = alo + c * VEC;
        if (g < ahi) cp_async16(sr + g, xr + g);
      } else {
        const int k = c - cpr, left = alo - g0, right = g0 + win - ahi;
        int g;
        if (k < left) g = g0 + k;
        else if (k - left < right) g = ahi + (k - left);
        else continue;
        const int i = sym_or_zero(g, p.nin, p.sym);
        sr[g] = i < 0 ? (T)0 : xr[i];
      }
    }
  }
  asm volatile("cp.async.commit_group;\n" ::: "memory");
  asm volatile("cp.async.wait_group 0;\n" ::: "memory");
  __syncthreads();

  // ---- compute: consecutive threads take consecutive units ----
  for (int e = threadIdx.x; e < nrows * useg; e += kThreads) {
    const int r = PACK ? e / useg : 0;
    const int u = e - r * useg;
    const int row = row0 + r;
    const T* s0 = nullptr;
    const T* s1 = nullptr;
    if (p.in0 || K == FWD1 || K == FWD2)
      s0 = smem + (size_t)r * p.srow + ((misalign(p.in0 + (long long)row * p.pitch0) + g0) & (VEC - 1));
    if (KI::nin == 2 && p.in1)
      s1 = smem + (size_t)(p.rpc + r) * p.srow + ((misalign(p.in1 + (long long)row * p.nin) + g0) & (VEC - 1));
    if constexpr (SC != SC_NONE) {
      // the filter outputs of the FWD1 / FWD2 branches below, one output pair of each filter per unit
      const int q = u0 + u;
      if (K == FWD1) {
        const int w = 2 * u + p.halo;
        const int l0 = LA > 0 ? LA : p.L0, l1 = LB > 0 ? LB : p.L1;
        const T* xa = s0 + w - l0 / 2;
        const T* xb = s0 + w - l1 / 2;
        scat_store<SC>(p, row, q, corr<LA, 1, 1>(p.a0.t, xa, l0), corr<LA, 1, 1>(p.a0.t, xa + 1, l0),
                       corr<LB, 1, 1>(p.a1.t, xb, l1), corr<LB, 1, 1>(p.a1.t, xb + 1, l1));
      } else {   // FWD2
        const int m = LA > 0 ? LA : p.L0;
        const T* xa = s0 + 4 * u + 2;
        scat_store<SC>(p, row, q, corr<LA, 1, 2>(p.a0.t, xa, m), corr<LA, 1, 2>(p.b0.t, xa + 1, m),
                       corr<LA, 1, 2>(p.b1.t, xa + 1, m), corr<LA, 1, 2>(p.a1.t, xa, m));
      }
    } else if (K == FWD1) {
      const int i = u0 + u, w = u + p.halo;
      const int l0 = LA > 0 ? LA : p.L0, l1 = LB > 0 ? LB : p.L1;
      p.out0[(long long)row * p.nout + i] = corr<LA, 1, 1>(p.a0.t, s0 + w - l0 / 2, l0);
      if (p.out1) p.out1[(long long)row * p.nout + i] = corr<LB, 1, 1>(p.a1.t, s0 + w - l1 / 2, l1);
    } else if (K == INV1) {
      const int i = u0 + u, w = u + p.halo;
      const int l0 = LA > 0 ? LA : p.L0, l1 = LB > 0 ? LB : p.L1;
      T a = 0, b = 0;
      if (s0) a = corr<LA, 1, 1>(p.a0.t, s0 + w - l0 / 2, l0);
      if (s1) b = corr<LB, 1, 1>(p.a1.t, s1 + w - l1 / 2, l1);
      p.out0[(long long)row * p.nout + i] = sum2(s0 != nullptr, a, s1 != nullptr, b);
    } else if (K == FWD2) {
      const int q = u0 + u, m = LA > 0 ? LA : p.L0;
      const T* xa = s0 + 4 * u + 2;               // window of x[4q + 2 - m + 2j]
      const long long o = (long long)row * p.nout + 2 * q;
      p.out0[o] = corr<LA, 1, 2>(p.a0.t, xa, m);
      p.out0[o + 1] = corr<LA, 1, 2>(p.b0.t, xa + 1, m);
      if (p.out1) {
        p.out1[o] = corr<LA, 1, 2>(p.b1.t, xa + 1, m);
        p.out1[o + 1] = corr<LA, 1, 2>(p.a1.t, xa, m);
      }
    } else {   // INV2
      constexpr int M2 = LA / 2;
      const int m2 = (LA > 0 ? LA : p.L0) / 2;
      const int w = 2 * u + p.halo - m2;          // window index of 2t - m2
      T ya[4] = {0, 0, 0, 0}, yb[4] = {0, 0, 0, 0};
      if (s0) ifilt4<false, M2>(p.a0.t, p.b0.t, s0 + w, m2, ya);
      if (s1) ifilt4<true, M2>(p.a1.t, p.b1.t, s1 + w, m2, yb);
      const long long o = (long long)row * p.nout + 4 * (u0 + u);
#pragma unroll
      for (int k = 0; k < 4; ++k) p.out0[o + k] = sum2(s0 != nullptr, ya[k], s1 != nullptr, yb[k]);
    }
  }
}

template <class T, int K, int LA, int LB, bool PACK>
__global__ void __launch_bounds__(kThreads) k_dt1d(const __grid_constant__ Dt1dParams<T> p) {
  dt1d_body<T, K, LA, LB, PACK, SC_NONE>(p);
}

// K = FWD1 or FWD2 with the scattering epilogue
template <class T, int K, int LA, int LB, bool PACK, int SC>
__global__ void __launch_bounds__(kThreads) k_scat1d(const __grid_constant__ Scat1dParams<T> p) {
  dt1d_body<T, K, LA, LB, PACK, SC>(p);
}

// ---- host side -------------------------------------------------------------------------------------------------

template <class T>
static void set_taps(TapsT<T>& d, const T* src, int L) {
  for (int i = 0; i < kMaxTaps; ++i) d.t[i] = (i < L) ? src[i] : (T)0;
}

template <class T, int K, int LA, int LB, bool PACK, int SC>
static auto kernel_of() {
  if constexpr (SC == SC_NONE) return k_dt1d<T, K, LA, LB, PACK>;
  else return k_scat1d<T, K, LA, LB, PACK, SC>;
}

template <class T, int K, int LA, int LB, int SC, class P>
static int launch_kind(P& p, void* stream) {
  using KI = KindInfo<K, SC>;
  constexpr int VEC = 16 / (int)sizeof(T);
  auto srow_of = [&](int units) { return ((units * KI::ipu + 2 * p.halo + 2 * VEC - 1) / VEC) * VEC; };
  // packed CTA: at least two whole rows within KindInfo::seg units and the staging budget
  int rpc = KI::seg / p.units;
  const int srow = srow_of(p.units);
  rpc = imin(rpc, kPackSmem / (KI::nin * srow * (int)sizeof(T)));
  if (rpc >= 2) {
    p.seg = p.units; p.rpc = rpc; p.nseg = 1; p.srow = srow;
    const long long blocks = (p.rows + rpc - 1) / rpc;
    return launch(kernel_of<T, K, LA, LB, true, SC>(), p, blocks, kThreads, (size_t)KI::nin * rpc * srow * sizeof(T),
                  stream);
  }
  p.seg = KI::seg; p.rpc = 1; p.nseg = (p.units + KI::seg - 1) / KI::seg; p.srow = srow_of(imin(p.units, KI::seg));
  const long long blocks = (long long)p.rows * p.nseg;
  if (blocks > 2147483647LL) return B200W_ESIZE;
  return launch(kernel_of<T, K, LA, LB, false, SC>(), p, blocks, kThreads, (size_t)KI::nin * p.srow * sizeof(T), stream);
}

// level 1: the (L0, L1) pairs of the biorthogonal tables, in both orders (the backward passes swap directions)
template <class T, int K, int SC = SC_NONE, class P>
static int dispatch_j1(P& p, void* stream) {
  const int a = p.L0, b = p.L1;
#define B200W_DT1D_PAIR(X, Y) if (a == X && b == Y) return launch_kind<T, K, X, Y, SC>(p, stream);
  B200W_DT1D_PAIR(5, 7) B200W_DT1D_PAIR(7, 5)      // near_sym_a
  B200W_DT1D_PAIR(9, 7) B200W_DT1D_PAIR(7, 9)      // antonini
  B200W_DT1D_PAIR(5, 3) B200W_DT1D_PAIR(3, 5)      // legall
  B200W_DT1D_PAIR(13, 19) B200W_DT1D_PAIR(19, 13)  // near_sym_b
#undef B200W_DT1D_PAIR
  return launch_kind<T, K, 0, 0, SC>(p, stream);
}

// levels >= 2: the q-shift table lengths
template <class T, int K, int SC = SC_NONE, class P>
static int dispatch_j2(P& p, void* stream) {
  switch (p.L0) {
    case 10: return launch_kind<T, K, 10, 0, SC>(p, stream);   // qshift_06, qshift_a
    case 14: return launch_kind<T, K, 14, 0, SC>(p, stream);   // qshift_b
    case 16: return launch_kind<T, K, 16, 0, SC>(p, stream);   // qshift_c
    case 18: return launch_kind<T, K, 18, 0, SC>(p, stream);   // qshift_d
    case 32: return launch_kind<T, K, 32, 0, SC>(p, stream);   // qshift_32
    default: return launch_kind<T, K, 0, 0, SC>(p, stream);
  }
}

static bool l1_ok(int L) { return L >= 1 && L <= kMaxTaps && (L & 1); }
static bool qs_ok(int m) { return m >= 2 && m <= kMaxTaps && !(m & 1); }

template <class T>
static int fwd_j1(const T* x, long long pitch, int rows, int n, T* lo, T* hi, const T* h0, int L0, const T* h1, int L1,
                  int mode, void* stream) {
  if (mode != B200W_MODE_SYMMETRIC && mode != B200W_MODE_ZERO) return B200W_EMODE;
  if (!x || !lo || !h0 || !h1) return B200W_EARG;
  if (rows < 0 || n < 2 || (n & 1)) return B200W_ESIZE;
  if (pitch < n) return B200W_EARG;
  if (!l1_ok(L0) || !l1_ok(L1)) return B200W_EFILTER;
  if (rows == 0) return B200W_OK;
  Dt1dParams<T> p = {};
  p.rows = rows; p.nin = n; p.nout = n; p.units = n;
  p.in0 = x; p.pitch0 = pitch; p.in1 = nullptr; p.out0 = lo; p.out1 = hi;
  p.L0 = L0; p.L1 = L1; p.halo = imax(L0, L1) / 2; p.sym = mode == B200W_MODE_SYMMETRIC;
  set_taps(p.a0, h0, L0); set_taps(p.a1, h1, L1);
  return dispatch_j1<T, FWD1>(p, stream);
}

template <class T>
static int inv_j1(const T* lo, long long pitch, const T* hi, int rows, int n, T* y, const T* g0, int L0, const T* g1,
                  int L1, int mode, void* stream) {
  if (mode != B200W_MODE_SYMMETRIC && mode != B200W_MODE_ZERO) return B200W_EMODE;
  if (!y || !g0 || !g1) return B200W_EARG;
  if (rows < 0 || n < 2 || (n & 1)) return B200W_ESIZE;
  if (lo && pitch < n) return B200W_EARG;
  if (!l1_ok(L0) || !l1_ok(L1)) return B200W_EFILTER;
  if (rows == 0) return B200W_OK;
  Dt1dParams<T> p = {};
  p.rows = rows; p.nin = n; p.nout = n; p.units = n;
  p.in0 = lo; p.pitch0 = lo ? pitch : n; p.in1 = hi; p.out0 = y; p.out1 = nullptr;
  p.L0 = L0; p.L1 = L1; p.halo = imax(L0, L1) / 2; p.sym = mode == B200W_MODE_SYMMETRIC;
  set_taps(p.a0, g0, L0); set_taps(p.a1, g1, L1);
  return dispatch_j1<T, INV1>(p, stream);
}

template <class T>
static int fwd_j2(const T* x, long long pitch, int rows, int n, T* lo, T* hi, const T* h0a, const T* h1a, const T* h0b,
                  const T* h1b, int m, void* stream) {
  if (!x || !lo || !h0a || !h1a || !h0b || !h1b) return B200W_EARG;
  if (rows < 0 || n < 4 || (n % 4)) return B200W_ESIZE;
  if (pitch < n) return B200W_EARG;
  if (!qs_ok(m)) return B200W_EFILTER;
  if (rows == 0) return B200W_OK;
  Dt1dParams<T> p = {};
  p.rows = rows; p.nin = n; p.nout = n / 2; p.units = n / 4;
  p.in0 = x; p.pitch0 = pitch; p.in1 = nullptr; p.out0 = lo; p.out1 = hi;
  p.L0 = m; p.L1 = m; p.halo = m; p.sym = 1;
  // lo = coldfilt(x, h0b, h0a), hi = coldfilt(x, h1b, h1a, highpass)
  set_taps(p.a0, h0b, m); set_taps(p.b0, h0a, m); set_taps(p.a1, h1b, m); set_taps(p.b1, h1a, m);
  return dispatch_j2<T, FWD2>(p, stream);
}

template <class T>
static int inv_j2(const T* lo, long long pitch, const T* hi, int rows, int n, T* y, const T* g0a, const T* g1a,
                  const T* g0b, const T* g1b, int m, void* stream) {
  if (!y || !g0a || !g1a || !g0b || !g1b) return B200W_EARG;
  if (rows < 0 || n < 4 || (n % 4)) return B200W_ESIZE;
  if (lo && pitch < n / 2) return B200W_EARG;
  if (!qs_ok(m)) return B200W_EFILTER;
  if (rows == 0) return B200W_OK;
  Dt1dParams<T> p = {};
  p.rows = rows; p.nin = n / 2; p.nout = n; p.units = n / 4;
  p.in0 = lo; p.pitch0 = lo ? pitch : n / 2; p.in1 = hi; p.out0 = y; p.out1 = nullptr;
  p.L0 = m; p.L1 = m; p.halo = m / 2 + 2; p.sym = 1;
  // y = colifilt(lo, g0b, g0a) + colifilt(hi, g1b, g1a, highpass)
  set_taps(p.a0, g0b, m); set_taps(p.b0, g0a, m); set_taps(p.a1, g1b, m); set_taps(p.b1, g1a, m);
  return dispatch_j2<T, INV2>(p, stream);
}

// Shared argument checks and output fields of the scattering entries; m = output row length.  Returns 1 when there is
// a launch to make, else B200W_OK or an error code.
template <class T>
static int scat_setup(Scat1dParams<T>& p, const T* x, long long pitch, int N, int C, int n, T* lo, long long bs_lo,
                      int m_lo, T* mag, long long bs_mag, T* dre, long long bs_dre, T* dim, long long bs_dim, int m,
                      double magbias) {
  if (!x || !lo || !mag || (!dre != !dim)) return B200W_EARG;
  if (N < 0 || C < 0 || (long long)N * C > 2147483647LL) return B200W_ESIZE;
  const long long cm = (long long)C * m;
  if (pitch < n || bs_lo < (long long)C * m_lo || bs_mag < cm || (dre && (bs_dre < cm || bs_dim < cm)))
    return B200W_EARG;
  p.rows = N * C; p.nin = n; p.units = m;
  p.in0 = x; p.pitch0 = pitch; p.in1 = nullptr; p.out0 = lo; p.out1 = nullptr;
  p.mag = mag; p.dre = dre; p.dim = dim;
  p.bs_lo = bs_lo; p.bs_mag = bs_mag; p.bs_dre = bs_dre; p.bs_dim = bs_dim;
  p.C = C; p.pool = m_lo == m;
  p.magbias = (T)magbias; p.magbias2 = (T)(magbias * magbias);
  return 1;
}

template <class T>
static int scat_j1(const T* x, long long pitch, int N, int C, int n, T* lo, long long bs_lo, int pool, T* mag,
                   long long bs_mag, T* dre, long long bs_dre, T* dim, long long bs_dim, const T* h0, int L0,
                   const T* h1, int L1, int mode, double magbias, void* stream) {
  if (mode != B200W_MODE_SYMMETRIC && mode != B200W_MODE_ZERO) return B200W_EMODE;
  if (!h0 || !h1) return B200W_EARG;
  if (n < 2 || (n & 1)) return B200W_ESIZE;
  Scat1dParams<T> p = {};
  const int rc = scat_setup(p, x, pitch, N, C, n, lo, bs_lo, pool ? n / 2 : n, mag, bs_mag, dre, bs_dre, dim, bs_dim,
                            n / 2, magbias);
  if (rc <= 0) return rc;
  if (!l1_ok(L0) || !l1_ok(L1)) return B200W_EFILTER;
  if (p.rows == 0) return B200W_OK;
  p.L0 = L0; p.L1 = L1; p.halo = imax(L0, L1) / 2; p.sym = mode == B200W_MODE_SYMMETRIC;
  set_taps(p.a0, h0, L0); set_taps(p.a1, h1, L1);
  return dre ? dispatch_j1<T, FWD1, SC_DER>(p, stream) : dispatch_j1<T, FWD1, SC_MAG>(p, stream);
}

template <class T>
static int scat_j2(const T* x, long long pitch, int N, int C, int n, T* lo, long long bs_lo, T* mag, long long bs_mag,
                   T* dre, long long bs_dre, T* dim, long long bs_dim, const T* h0a, const T* h1a, const T* h0b,
                   const T* h1b, int m, double magbias, void* stream) {
  if (!h0a || !h1a || !h0b || !h1b) return B200W_EARG;
  if (n < 4 || (n % 4)) return B200W_ESIZE;
  Scat1dParams<T> p = {};
  const int rc = scat_setup(p, x, pitch, N, C, n, lo, bs_lo, n / 4, mag, bs_mag, dre, bs_dre, dim, bs_dim, n / 4,
                            magbias);
  if (rc <= 0) return rc;
  if (!qs_ok(m)) return B200W_EFILTER;
  if (p.rows == 0) return B200W_OK;
  p.L0 = m; p.L1 = m; p.halo = m; p.sym = 1;
  set_taps(p.a0, h0b, m); set_taps(p.b0, h0a, m); set_taps(p.a1, h1b, m); set_taps(p.b1, h1a, m);
  return dre ? dispatch_j2<T, FWD2, SC_DER>(p, stream) : dispatch_j2<T, FWD2, SC_MAG>(p, stream);
}

}  // namespace dt1d
}  // namespace b200w

using namespace b200w::dt1d;

extern "C" {

int b200w_dtcwt1d_fwd_j1(const float* x, long long x_pitch, int rows, int n, float* lo, float* hi, const float* h0,
                         int L0, const float* h1, int L1, int mode, void* stream) {
  return fwd_j1<float>(x, x_pitch, rows, n, lo, hi, h0, L0, h1, L1, mode, stream);
}
int b200w_dtcwt1d_fwd_j1_f64(const double* x, long long x_pitch, int rows, int n, double* lo, double* hi,
                             const double* h0, int L0, const double* h1, int L1, int mode, void* stream) {
  return fwd_j1<double>(x, x_pitch, rows, n, lo, hi, h0, L0, h1, L1, mode, stream);
}
int b200w_dtcwt1d_fwd_j2plus(const float* x, long long x_pitch, int rows, int n, float* lo, float* hi,
                             const float* h0a, const float* h1a, const float* h0b, const float* h1b, int m,
                             void* stream) {
  return fwd_j2<float>(x, x_pitch, rows, n, lo, hi, h0a, h1a, h0b, h1b, m, stream);
}
int b200w_dtcwt1d_fwd_j2plus_f64(const double* x, long long x_pitch, int rows, int n, double* lo, double* hi,
                                 const double* h0a, const double* h1a, const double* h0b, const double* h1b, int m,
                                 void* stream) {
  return fwd_j2<double>(x, x_pitch, rows, n, lo, hi, h0a, h1a, h0b, h1b, m, stream);
}
int b200w_dtcwt1d_inv_j1(const float* lo, long long lo_pitch, const float* hi, int rows, int n, float* y,
                         const float* g0, int L0, const float* g1, int L1, int mode, void* stream) {
  return inv_j1<float>(lo, lo_pitch, hi, rows, n, y, g0, L0, g1, L1, mode, stream);
}
int b200w_dtcwt1d_inv_j1_f64(const double* lo, long long lo_pitch, const double* hi, int rows, int n, double* y,
                             const double* g0, int L0, const double* g1, int L1, int mode, void* stream) {
  return inv_j1<double>(lo, lo_pitch, hi, rows, n, y, g0, L0, g1, L1, mode, stream);
}
int b200w_dtcwt1d_inv_j2plus(const float* lo, long long lo_pitch, const float* hi, int rows, int n, float* y,
                             const float* g0a, const float* g1a, const float* g0b, const float* g1b, int m,
                             void* stream) {
  return inv_j2<float>(lo, lo_pitch, hi, rows, n, y, g0a, g1a, g0b, g1b, m, stream);
}
int b200w_dtcwt1d_inv_j2plus_f64(const double* lo, long long lo_pitch, const double* hi, int rows, int n, double* y,
                                 const double* g0a, const double* g1a, const double* g0b, const double* g1b, int m,
                                 void* stream) {
  return inv_j2<double>(lo, lo_pitch, hi, rows, n, y, g0a, g1a, g0b, g1b, m, stream);
}

int b200w_scat1d_j1(const float* x, long long x_pitch, int N, int C, int n, float* lo, long long lo_bstride, int pool_lo,
                    float* mag, long long mag_bstride, float* dre, long long dre_bstride, float* dim,
                    long long dim_bstride, const float* h0, int L0, const float* h1, int L1, int mode, double magbias,
                    void* stream) {
  return scat_j1<float>(x, x_pitch, N, C, n, lo, lo_bstride, pool_lo, mag, mag_bstride, dre, dre_bstride, dim,
                        dim_bstride, h0, L0, h1, L1, mode, magbias, stream);
}
int b200w_scat1d_j1_f64(const double* x, long long x_pitch, int N, int C, int n, double* lo, long long lo_bstride,
                        int pool_lo, double* mag, long long mag_bstride, double* dre, long long dre_bstride,
                        double* dim, long long dim_bstride, const double* h0, int L0, const double* h1, int L1,
                        int mode, double magbias, void* stream) {
  return scat_j1<double>(x, x_pitch, N, C, n, lo, lo_bstride, pool_lo, mag, mag_bstride, dre, dre_bstride, dim,
                         dim_bstride, h0, L0, h1, L1, mode, magbias, stream);
}
int b200w_scat1d_j2plus(const float* x, long long x_pitch, int N, int C, int n, float* lo, long long lo_bstride,
                        float* mag, long long mag_bstride, float* dre, long long dre_bstride, float* dim,
                        long long dim_bstride, const float* h0a, const float* h1a, const float* h0b, const float* h1b,
                        int m, double magbias, void* stream) {
  return scat_j2<float>(x, x_pitch, N, C, n, lo, lo_bstride, mag, mag_bstride, dre, dre_bstride, dim, dim_bstride,
                        h0a, h1a, h0b, h1b, m, magbias, stream);
}
int b200w_scat1d_j2plus_f64(const double* x, long long x_pitch, int N, int C, int n, double* lo, long long lo_bstride,
                            double* mag, long long mag_bstride, double* dre, long long dre_bstride, double* dim,
                            long long dim_bstride, const double* h0a, const double* h1a, const double* h0b,
                            const double* h1b, int m, double magbias, void* stream) {
  return scat_j2<double>(x, x_pitch, N, C, n, lo, lo_bstride, mag, mag_bstride, dre, dre_bstride, dim, dim_bstride,
                         h0a, h1a, h0b, h1b, m, magbias, stream);
}

}  // extern "C"
