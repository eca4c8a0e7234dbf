// k_prims.cu -- the reference's standalone 1-D DTCWT primitives as CUDA kernels (sm_90a):
//   colfilter / rowfilter   (dtcwt/lowlevel.py:70-94;  any filter length -- an EVEN length gives N + 1 outputs)
//   coldfilt / rowdfilt     (:97-151, decimating q-shift pair)
//   colifilt / rowifilt     (:154-239, interpolating q-shift pair)
// In the transforms these passes are fused into the per-level kernels (the hot path); the standalone forms exist for
// callers of the reference's low-level API and for its unit tests (tests/test_colfilter.py, test_coldfilt.py, ...).
// One thread per output element, threads consecutive along W (coalesced stores; loads coalesced for the column forms and
// stride-1 windows for the row forms, which the L1 serves).  Accumulation = the oracle's: first term a product, then fused
// multiply-adds in stored-tap order, so float32 / float64 results are bit-identical to oracle/wave_oracle_impl.h.
#include <cuda_runtime.h>

#include "common.h"
#include "launch.cuh"

namespace b200w {
namespace prims {

template <class T> struct PTaps { T t[kMaxTaps]; };

template <class T>
struct PrimParams {
  const T* x; T* y;
  long long total;        // output elements
  int H, W, Ho, Wo;       // input / output plane size
  int L, sym, along_w, highpass;
  PTaps<T> ha, hb;
};

// y[n] = sum_j h[j] x[ext(n + j - m)], m = L / 2, n in [0, N + 2m - L + 1)
template <class T>
__global__ void __launch_bounds__(256) k_filter(const __grid_constant__ PrimParams<T> p) {
  const long long idx = (long long)blockIdx.x * 256 + threadIdx.x;
  if (idx >= p.total) return;
  const int c = (int)(idx % p.Wo);
  const long long t = idx / p.Wo;
  const int r = (int)(t % p.Ho);
  const long long plane = t / p.Ho;
  const T* xp = p.x + plane * p.H * p.W;
  const int m = p.L / 2;
  const int N = p.along_w ? p.W : p.H;
  const int n = p.along_w ? c : r;
  T a = 0;
  for (int j = 0; j < p.L; ++j) {
    const int i = sym_or_zero(n + j - m, N, p.sym);
    const T v = (i < 0) ? (T)0 : (p.along_w ? xp[(long long)r * p.W + i] : xp[(long long)i * p.W + c]);
    a = (j == 0) ? mul_rn(p.ha.t[0], v) : fma_rn(p.ha.t[j], v, a);
  }
  p.y[idx] = a;
}

// Ya[q] = sum_j ha[j] x[sym(4q + 2j + 2 - m)], Yb[q] = sum_j hb[j] x[sym(4q + 2j + 3 - m)];
// low-pass: y[2q] = Ya, y[2q+1] = Yb; high-pass: swapped
template <class T>
__global__ void __launch_bounds__(256) k_dfilt(const __grid_constant__ PrimParams<T> p) {
  const long long idx = (long long)blockIdx.x * 256 + threadIdx.x;
  if (idx >= p.total) return;
  const int c = (int)(idx % p.Wo);
  const long long t = idx / p.Wo;
  const int r = (int)(t % p.Ho);
  const long long plane = t / p.Ho;
  const T* xp = p.x + plane * p.H * p.W;
  const int m = p.L;
  const int N = p.along_w ? p.W : p.H;
  const int k = p.along_w ? c : r;            // output index along the filtered dimension
  const int q = k >> 1;
  const bool use_b = ((k & 1) != 0) != (p.highpass != 0);
  const T* h = use_b ? p.hb.t : p.ha.t;
  const int base = 4 * q + (use_b ? 3 : 2) - m;
  T a = 0;
  for (int j = 0; j < m; ++j) {
    const int i = ext_index(base + 2 * j, N, B200W_MODE_SYMMETRIC);
    const T v = p.along_w ? xp[(long long)r * p.W + i] : xp[(long long)i * p.W + c];
    a = (j == 0) ? mul_rn(h[0], v) : fma_rn(h[j], v, a);
  }
  p.y[idx] = a;
}

// y[4t+s] = sum_{j<m2} f_s[j] x[sym(2(t+j) + o_s - m2)]   (phase tables: dtcwt/lowlevel.py:169-186)
template <class T>
__global__ void __launch_bounds__(256) k_ifilt(const __grid_constant__ PrimParams<T> p) {
  const long long idx = (long long)blockIdx.x * 256 + threadIdx.x;
  if (idx >= p.total) return;
  const int c = (int)(idx % p.Wo);
  const long long tt = idx / p.Wo;
  const int r = (int)(tt % p.Ho);
  const long long plane = tt / p.Ho;
  const T* xp = p.x + plane * p.H * p.W;
  const int m2 = p.L / 2;
  const int N = p.along_w ? p.W : p.H;
  const int k = p.along_w ? c : r;
  const int t = k >> 2, s = k & 3;
  int o, par;
  if ((m2 & 1) == 0) { par = (s >= 2) ? 1 : 0; o = p.highpass ? (s ^ 1) : s; }
  else { par = (s < 2) ? 1 : 0; o = p.highpass ? (2 - (s & 1)) : (1 + (s & 1)); }
  const T* h = (s & 1) ? p.hb.t : p.ha.t;
  T a = 0;
  for (int j = 0; j < m2; ++j) {
    const int i = ext_index(2 * (t + j) + o - m2, N, B200W_MODE_SYMMETRIC);
    const T v = p.along_w ? xp[(long long)r * p.W + i] : xp[(long long)i * p.W + c];
    const T cf = h[2 * j + par];
    a = (j == 0) ? mul_rn(cf, v) : fma_rn(cf, v, a);
  }
  p.y[idx] = a;
}

template <class T>
static int set_ptaps(PTaps<T>& d, const T* src, int L) {
  if (!src) return B200W_EARG;
  if (L < 1 || L > kMaxTaps) return B200W_EFILTER;
  for (int i = 0; i < kMaxTaps; ++i) d.t[i] = (i < L) ? src[i] : (T)0;
  return 0;
}

template <class T, class K>
static int launch_prim(K kernel, PrimParams<T>& p, int planes, void* stream) {
  p.total = (long long)planes * p.Ho * p.Wo;
  const long long blocks = (p.total + 255) / 256;
  if (blocks > 2147483647LL) return B200W_ESIZE;
  return launch(kernel, p, blocks, 256, 0, stream);
}

template <class T>
static int filter_impl(const T* x, T* y, int planes, int H, int W, const T* h, int L, int symmetric, int along_w,
                       void* stream) {
  if (!x || !y) return B200W_EARG;
  if (planes < 0 || H < 1 || W < 1) return B200W_ESIZE;
  PrimParams<T> p;
  int rc = set_ptaps(p.ha, h, L);
  if (rc) return rc;
  p.hb = p.ha;
  const int ext = 2 * (L / 2) - L + 1;     // 0 for odd lengths, 1 for even ones
  p.x = x; p.y = y; p.H = H; p.W = W; p.Ho = along_w ? H : H + ext; p.Wo = along_w ? W + ext : W;
  p.L = L; p.sym = symmetric ? 1 : 0; p.along_w = along_w ? 1 : 0; p.highpass = 0;
  return launch_prim<T>(k_filter<T>, p, planes, stream);
}

template <class T>
static int dfilt_impl(const T* x, T* y, int planes, int H, int W, const T* ha, const T* hb, int m, int highpass,
                      int along_w, void* stream) {
  if (!x || !y) return B200W_EARG;
  if (planes < 0 || H < 1 || W < 1 || ((along_w ? W : H) % 4)) return B200W_ESIZE;   // reference ValueError
  if (m < 2 || (m & 1)) return B200W_EFILTER;
  PrimParams<T> p;
  int rc;
  if ((rc = set_ptaps(p.ha, ha, m)) || (rc = set_ptaps(p.hb, hb, m))) return rc;
  p.x = x; p.y = y; p.H = H; p.W = W; p.Ho = along_w ? H : H / 2; p.Wo = along_w ? W / 2 : W;
  p.L = m; p.sym = 1; p.along_w = along_w ? 1 : 0; p.highpass = highpass ? 1 : 0;
  return launch_prim<T>(k_dfilt<T>, p, planes, stream);
}

template <class T>
static int ifilt_impl(const T* x, T* y, int planes, int H, int W, const T* ha, const T* hb, int m, int highpass,
                      int along_w, void* stream) {
  if (!x || !y) return B200W_EARG;
  if (planes < 0 || H < 1 || W < 1 || ((along_w ? W : H) % 2)) return B200W_ESIZE;   // reference ValueError
  if (m < 2 || (m & 1)) return B200W_EFILTER;
  PrimParams<T> p;
  int rc;
  if ((rc = set_ptaps(p.ha, ha, m)) || (rc = set_ptaps(p.hb, hb, m))) return rc;
  p.x = x; p.y = y; p.H = H; p.W = W; p.Ho = along_w ? H : 2 * H; p.Wo = along_w ? 2 * W : W;
  p.L = m; p.sym = 1; p.along_w = along_w ? 1 : 0; p.highpass = highpass ? 1 : 0;
  return launch_prim<T>(k_ifilt<T>, p, planes, stream);
}

}  // namespace prims
}  // namespace b200w

using namespace b200w::prims;

extern "C" {

int b200w_dtcwt_filter(const float* x, float* y, int planes, int H, int W, const float* h, int L, int symmetric,
                       int along_w, void* stream) {
  return filter_impl<float>(x, y, planes, H, W, h, L, symmetric, along_w, stream);
}
int b200w_dtcwt_filter_f64(const double* x, double* y, int planes, int H, int W, const double* h, int L, int symmetric,
                           int along_w, void* stream) {
  return filter_impl<double>(x, y, planes, H, W, h, L, symmetric, along_w, stream);
}
int b200w_dtcwt_dfilt(const float* x, float* y, int planes, int H, int W, const float* ha, const float* hb, int m,
                      int highpass, int along_w, void* stream) {
  return dfilt_impl<float>(x, y, planes, H, W, ha, hb, m, highpass, along_w, stream);
}
int b200w_dtcwt_dfilt_f64(const double* x, double* y, int planes, int H, int W, const double* ha, const double* hb, int m,
                          int highpass, int along_w, void* stream) {
  return dfilt_impl<double>(x, y, planes, H, W, ha, hb, m, highpass, along_w, stream);
}
int b200w_dtcwt_ifilt(const float* x, float* y, int planes, int H, int W, const float* ha, const float* hb, int m,
                      int highpass, int along_w, void* stream) {
  return ifilt_impl<float>(x, y, planes, H, W, ha, hb, m, highpass, along_w, stream);
}
int b200w_dtcwt_ifilt_f64(const double* x, double* y, int planes, int H, int W, const double* ha, const double* hb, int m,
                          int highpass, int along_w, void* stream) {
  return ifilt_impl<double>(x, y, planes, H, W, ha, hb, m, highpass, along_w, stream);
}

}  // extern "C"
