// dwt1d.cu -- 1-D DWT analysis / synthesis levels (sm_90a): AFB1D / SFB1D of the reference (dwt/lowlevel.py:368-424,
// 697-743 = afb1d / sfb1d along the last dimension of (N, C, L) signals), the callers' side of the 2-D banks
// (SURVEY.md 8(f) rank 4).  HBM-bound and tiny per element: one CTA stages a contiguous segment of one signal (with
// the boundary extension resolved by index arithmetic while staging) in shared memory with coalesced loads, every thread
// produces one output position of both bands, stores are coalesced.  Accumulation order = the oracle's (stored tap
// order, first term a product, then fused multiply-adds), so the analysis is bit-identical to it.  The kernels are
// templates on the element type; this unit defines both the float and the `_f64` entry points.
#include <cuda_runtime.h>

#include <type_traits>

#include "launch.cuh"
#include "launch_params.h"

namespace b200w {

constexpr int kT1 = 256;   // outputs per CTA (= threads)

// The staged segment: one dynamic shared array per element type.  (Cast from a single byte array, as the tile kernels
// do it, nvcc 12.9 schedules these two kernels differently.)
extern __shared__ __align__(16) float g_seg_f32[];
extern __shared__ __align__(16) double g_seg_f64[];
template <class T> __device__ __forceinline__ T* seg_smem() {
  if constexpr (std::is_same_v<T, float>) return g_seg_f32;
  else return g_seg_f64;
}

template <class T>
struct Afb1dParams {
  const T* x; long long xpitch;
  T* lo; T* hi;
  int rows, N, K, L, mode, tiles;
  TapsT<T> f0, f1;
};

template <class T>
struct Sfb1dParams {
  const T* lo; const T* hi;
  T* y;
  int rows, K, Nout, L, mode, tiles;
  TapsT<T> g0, g1;
};

// out[k] = sum_j f[j] xe[2k + j - pl]  (reference afb1d :134-168)
template <class T>
__global__ void __launch_bounds__(kT1) afb1d_rows(const __grid_constant__ Afb1dParams<T> p) {
  T* seg = seg_smem<T>();
  const int tile = blockIdx.x % p.tiles, row = blockIdx.x / p.tiles;
  const int k0 = tile * kT1;
  const int pl = (p.mode == B200W_MODE_PERIODIZATION) ? (p.L - 1 - p.L / 2) : (p.L - 2);
  const int nseg = 2 * kT1 + p.L;                       // extended positions [2*k0 - pl, 2*k0 - pl + nseg)
  const T* xr = p.x + (long long)row * p.xpitch;
  for (int i = threadIdx.x; i < nseg; i += kT1) {
    const int g = ext_index(2 * k0 - pl + i, p.N, p.mode);
    seg[i] = (g >= 0) ? xr[g] : T(0);
  }
  __syncthreads();
  const int k = k0 + threadIdx.x;
  if (k >= p.K) return;
  const T* s = seg + 2 * threadIdx.x;
  T a0 = mul_rn(p.f0.t[0], s[0]), a1 = mul_rn(p.f1.t[0], s[0]);
  for (int j = 1; j < p.L; ++j) {
    a0 = fma_rn(p.f0.t[j], s[j], a0);
    a1 = fma_rn(p.f1.t[j], s[j], a1);
  }
  p.lo[(long long)row * p.K + k] = a0;
  p.hi[(long long)row * p.K + k] = a1;
}

// y[n] = sum_k lo[k] g0[s - 2k] + sum_k hi[k] g1[s - 2k], s = n + off  (reference sfb1d :252-267)
template <class T>
__global__ void __launch_bounds__(kT1) sfb1d_rows(const __grid_constant__ Sfb1dParams<T> p) {
  T* seg = seg_smem<T>();
  const int tile = blockIdx.x % p.tiles, row = blockIdx.x / p.tiles;
  const int n0 = tile * kT1;
  const bool per = (p.mode == B200W_MODE_PERIODIZATION);
  const int off = per ? (p.L / 2 - 1) : (p.L - 2);
  // coefficient indices needed by the tile: k in [floor((n0 + off - L + 2) / 2), floor((n0 + kT1 - 1 + off) / 2)]
  const int kb = floordiv2(n0 + off - p.L + 2);
  const int nk = kT1 / 2 + p.L / 2 + 2;
  T* slo = seg;
  T* shi = seg + nk;
  const T* lo = p.lo + (long long)row * p.K;
  const T* hi = p.hi ? p.hi + (long long)row * p.K : nullptr;
  for (int i = threadIdx.x; i < nk; i += kT1) {
    int k = kb + i;
    bool ok = true;
    if (per) { k %= p.K; if (k < 0) k += p.K; }
    else ok = (k >= 0 && k < p.K);
    slo[i] = ok ? lo[k] : T(0);
    shi[i] = (ok && hi) ? hi[k] : T(0);
  }
  __syncthreads();
  const int n = n0 + threadIdx.x;
  if (n >= p.Nout) return;
  const int s = n + off;
  const int kmin = floordiv2(s - p.L + 2), kmax = floordiv2(s);
  T a0 = 0, a1 = 0;
  bool first = true;
  for (int k = kmin; k <= kmax; ++k) {
    if (!per && (k < 0 || k >= p.K)) continue;          // the oracle skips them too (they do not start the sum)
    const int t = s - 2 * k;
    const T vl = slo[k - kb], vh = shi[k - kb];
    if (first) { a0 = mul_rn(vl, p.g0.t[t]); a1 = mul_rn(vh, p.g1.t[t]); first = false; }
    else { a0 = fma_rn(vl, p.g0.t[t], a0); a1 = fma_rn(vh, p.g1.t[t], a1); }
  }
  p.y[(long long)row * p.Nout + n] = add_rn(a0, a1);
}

}  // namespace b200w

using namespace b200w;

namespace {

template <class T>
int afb1d_impl(const T* x, long long x_pitch, int rows, int N, T* lo, T* hi, const T* f0, const T* f1, int L, int mode,
               void* stream) {
  if (!dwt_mode_ok(mode)) return B200W_EMODE;
  if (!x || !lo || !hi) return B200W_EARG;
  if (rows < 0 || N < 1 || x_pitch < N) return B200W_ESIZE;
  if (L < 2) return B200W_EFILTER;
  Afb1dParams<T> p;
  int rc;
  if ((rc = set_taps(p.f0, f0, L)) || (rc = set_taps(p.f1, f1, L))) return rc;
  p.x = x; p.xpitch = x_pitch; p.lo = lo; p.hi = hi;
  p.rows = rows; p.N = N; p.K = coeff_len(N, L, mode); p.L = L; p.mode = mode;
  p.tiles = cdiv(p.K, kT1);
  const long long blocks = (long long)rows * p.tiles;
  if (!grid_ok(blocks)) return B200W_ESIZE;
  return launch(afb1d_rows<T>, p, blocks, kT1, (2 * kT1 + L) * sizeof(T), stream);
}

template <class T>
int sfb1d_impl(const T* lo, const T* hi, int rows, int K, T* y, int Nout, const T* g0, const T* g1, int L, int mode,
               void* stream) {
  if (!dwt_mode_ok(mode)) return B200W_EMODE;
  if (!lo || !y) return B200W_EARG;
  if (rows < 0 || K < 1) return B200W_ESIZE;
  if (L < 2) return B200W_EFILTER;
  if (Nout < 1 || Nout > rec_len(K, L, mode)) return B200W_ESIZE;
  Sfb1dParams<T> p;
  int rc;
  if ((rc = set_taps(p.g0, g0, L)) || (rc = set_taps(p.g1, g1, L))) return rc;
  p.lo = lo; p.hi = hi; p.y = y;
  p.rows = rows; p.K = K; p.Nout = Nout; p.L = L; p.mode = mode;
  p.tiles = cdiv(Nout, kT1);
  const long long blocks = (long long)rows * p.tiles;
  if (!grid_ok(blocks)) return B200W_ESIZE;
  return launch(sfb1d_rows<T>, p, blocks, kT1, 2 * (kT1 / 2 + L / 2 + 2) * sizeof(T), stream);
}

}  // namespace

extern "C" {

int b200w_dwt_afb1d(const float* x, long long x_pitch, int rows, int N, float* lo, float* hi, const float* f0,
                    const float* f1, int L, int mode, void* stream) {
  return afb1d_impl(x, x_pitch, rows, N, lo, hi, f0, f1, L, mode, stream);
}
int b200w_dwt_afb1d_f64(const double* x, long long x_pitch, int rows, int N, double* lo, double* hi, const double* f0,
                        const double* f1, int L, int mode, void* stream) {
  return afb1d_impl(x, x_pitch, rows, N, lo, hi, f0, f1, L, mode, stream);
}

int b200w_dwt_sfb1d(const float* lo, const float* hi, int rows, int K, float* y, int Nout, const float* g0,
                    const float* g1, int L, int mode, void* stream) {
  return sfb1d_impl(lo, hi, rows, K, y, Nout, g0, g1, L, mode, stream);
}
int b200w_dwt_sfb1d_f64(const double* lo, const double* hi, int rows, int K, double* y, int Nout, const double* g0,
                        const double* g1, int L, int mode, void* stream) {
  return sfb1d_impl(lo, hi, rows, K, y, Nout, g0, g1, L, mode, stream);
}

}  // extern "C"
