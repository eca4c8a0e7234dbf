// dwt_adjoint.cu -- the transpose of the mode-extended DWT analysis bank, A_m^T, in 1-D and 2-D (sm_90a).
//
// A_m(x)[k] = sum_j f[j] x[ext_m(2k + j - pl)] (dwt1d.cu afb1d_rows, pl = L - 2, or L - 1 - L/2 in periodization).
// Its transpose sums, for every output i, the transposed convolution z[p] = sum_k f[p + pl - 2k] c[k] over every
// extended position p with ext_m(p) == i ("the images of i").  It is what autograd differentiates when a caller takes
// the gradient of SFB1D / SFB2D's backward pass (reference dwt/lowlevel.py:683-694, 732-743).
//
// Away from the edges the only image of i is p = i, and z[i] is the synthesis bank's output cropped to n.  So one
// launch is:
//   1. the existing synthesis level (b200w_dwt_sfb2d / b200w_dwt_sfb1d with the crop, on the streaming kernels where
//      they apply) writes z[i] to every output;
//   2. a border kernel overwrites the outputs within `depth` = L rows / columns of an edge (the whole axis when it is
//      shorter than 2L) with the full sum over every image, evaluated straight from the coefficients.
// Outside those borders no output has a second image, and in periodization the synthesis kernel's own wrap-around
// (k taken mod K) only reaches them too.  Zero mode and even-size periodization have no images beyond p = i (the
// synthesis level is then the whole answer), so the border kernel is not launched.  In periodization with an odd
// filter length the synthesis offset (L/2 - 1) differs from pl, so that axis is recomputed in full.
#include <cuda_runtime.h>

#include "launch.cuh"
#include "launch_params.h"

namespace b200w {

constexpr int kAdjT = 256;   // outputs per CTA (= threads)

// The images of output i along one axis of length n: every p in [plo, phi] congruent to one of `nb` bases modulo `per`
// (ext_index, common.h, inverted).
struct Images {
  int b0, b1, nb, per;
  __device__ __forceinline__ int base(int a) const { return a ? b1 : b0; }   // (no local-memory array)
};

__device__ __forceinline__ Images images_of(int i, int n, int mode) {
  Images im;
  im.nb = 1;
  im.b0 = im.b1 = i;
  switch (mode) {
    case B200W_MODE_SYMMETRIC:
      im.per = 2 * n; im.b1 = 2 * n - 1 - i; im.nb = 2;
      break;
    case B200W_MODE_REFLECT:
      if (n == 1) { im.per = 1; break; }
      im.per = 2 * n - 2;
      if (i > 0 && i < n - 1) { im.b1 = 2 * n - 2 - i; im.nb = 2; }
      break;
    case B200W_MODE_PERIODIC:
      im.per = n;
      break;
    case B200W_MODE_PERIODIZATION:   // period n + (n & 1); the appended sample n repeats n - 1
      im.per = n + (n & 1);
      if ((n & 1) && i == n - 1) { im.b1 = n; im.nb = 2; }
      break;
    default:                         // zero: p = i only
      im.per = 1 << 29;
  }
  return im;
}

// first p >= plo with p == base (mod per)
__device__ __forceinline__ int first_image(int base, int per, int plo) {
  int r = (base - plo) % per;
  if (r < 0) r += per;
  return plo + r;
}

// Output position t of a plane's border region -> (row, col).  The region is the first and last `dh` rows at full width
// (all rows when 2 dh >= H), then, on the rows between, the first and last `dw` columns (all columns when 2 dw >= W).
__device__ __forceinline__ void border_pos(int t, int H, int W, int dh, int dw, int& r, int& c) {
  const int full = (2 * dh >= H) ? H : 2 * dh;
  if (t < full * W) {
    const int a = t / W;
    c = t - a * W;
    r = (full == H || a < dh) ? a : H - 2 * dh + a;
    return;
  }
  t -= full * W;
  const int ew = (2 * dw >= W) ? W : 2 * dw;
  const int a = t / ew, b = t - a * ew;
  r = dh + a;
  c = (ew == W || b < dw) ? b : W - 2 * dw + b;
}

__host__ __device__ __forceinline__ long long border_count(int H, int W, int dh, int dw) {
  const int full = (2 * dh >= H) ? H : 2 * dh;
  const int ew = (2 * dw >= W) ? W : 2 * dw;
  return (long long)full * W + (long long)(H - full) * ew;
}

template <class T>
struct Adj2dParams {
  const T* ll; long long llps; int llpitch;
  const T* highs;                          // (planes, 3, Hc, Wc) contiguous, or null = zeros
  T* y; long long yps; int ypitch;
  int planes, Hc, Wc, H, W, Lh, Lw, mode, plh, plw, dh, dw, count, tiles;
  TapsT<T> fh_lo, fh_hi, fw_lo, fw_hi;
};

template <class T>
struct Adj1dParams {
  const T* lo; const T* hi;                // (rows, K) contiguous; hi may be null = zeros
  T* y;                                    // (rows, N) contiguous
  int rows, K, N, L, mode, pl, depth, count, tiles;
  TapsT<T> f0, f1;
};

// y[i, j] = sum over the images (p, q) of (i, j) of sum_{kh, kw} fH[p + plh - 2kh] fW[q + plw - 2kw] c[kh, kw], summed
// over the four bands (ll: H lo W lo, highs[0]: H hi W lo, highs[1]: H lo W hi, highs[2]: H hi W hi).  The W sums
// of one coefficient row are accumulated first, then weighted by the H taps, as the synthesis does it per axis.
template <class T>
__global__ void __launch_bounds__(kAdjT) afb2d_adjoint_border(const __grid_constant__ Adj2dParams<T> p) {
  // the taps in shared memory: the lanes of a warp index them at different positions, which the constant bank
  // behind the kernel parameters would serialise
  __shared__ T fhl[kMaxTaps], fhh[kMaxTaps], fwl[kMaxTaps], fwh[kMaxTaps];
  for (int q = threadIdx.x; q < kMaxTaps; q += kAdjT) {
    fhl[q] = p.fh_lo.t[q]; fhh[q] = p.fh_hi.t[q]; fwl[q] = p.fw_lo.t[q]; fwh[q] = p.fw_hi.t[q];
  }
  __syncthreads();
  const int tile = blockIdx.x % p.tiles;
  const long long plane = blockIdx.x / p.tiles;
  const int t = tile * kAdjT + threadIdx.x;
  if (t >= p.count) return;
  int i, j;
  border_pos(t, p.H, p.W, p.dh, p.dw, i, j);
  const T* ll = p.ll + plane * p.llps;
  const long long bs = (long long)p.Hc * p.Wc;
  const T* hs = p.highs ? p.highs + plane * 3 * bs : nullptr;
  const Images ih = images_of(i, p.H, p.mode), iw = images_of(j, p.W, p.mode);
  const int phh = 2 * p.Hc - 3 + p.Lh - p.plh, phw = 2 * p.Wc - 3 + p.Lw - p.plw;   // last extended positions
  T acc = T(0);
  for (int a = 0; a < ih.nb; ++a) {
    for (int ph = first_image(ih.base(a), ih.per, -p.plh); ph <= phh; ph += ih.per) {
      const int khmin = imax(0, floordiv2(ph + p.plh - p.Lh + 2)), khmax = imin(p.Hc - 1, floordiv2(ph + p.plh));
      for (int kh = khmin; kh <= khmax; ++kh) {
        const T* rl = ll + (long long)kh * p.llpitch;
        const T* r1 = hs ? hs + (long long)kh * p.Wc : nullptr;
        T slo = T(0), shi = T(0);
        for (int b = 0; b < iw.nb; ++b) {
          for (int pw = first_image(iw.base(b), iw.per, -p.plw); pw <= phw; pw += iw.per) {
            const int kwmin = imax(0, floordiv2(pw + p.plw - p.Lw + 2)), kwmax = imin(p.Wc - 1, floordiv2(pw + p.plw));
            for (int kw = kwmin; kw <= kwmax; ++kw) {
              const int tw = pw + p.plw - 2 * kw;
              const T wl = fwl[tw], wh = fwh[tw];
              slo = fma_rn(wl, rl[kw], slo);
              if (r1) {
                slo = fma_rn(wh, r1[bs + kw], slo);
                shi = fma_rn(wl, r1[kw], shi);
                shi = fma_rn(wh, r1[2 * bs + kw], shi);
              }
            }
          }
        }
        const int th = ph + p.plh - 2 * kh;
        acc = fma_rn(fhl[th], slo, acc);
        acc = fma_rn(fhh[th], shi, acc);
      }
    }
  }
  p.y[plane * p.yps + (long long)i * p.ypitch + j] = acc;
}

// y[i] = sum over the images p of i of sum_k (f0[p + pl - 2k] lo[k] + f1[p + pl - 2k] hi[k]); the first and last
// `depth` outputs of each row (all of them when 2 depth >= N).
template <class T>
__global__ void __launch_bounds__(kAdjT) afb1d_adjoint_border(const __grid_constant__ Adj1dParams<T> p) {
  __shared__ T f0[kMaxTaps], f1[kMaxTaps];   // (as in the 2-D kernel)
  for (int q = threadIdx.x; q < kMaxTaps; q += kAdjT) { f0[q] = p.f0.t[q]; f1[q] = p.f1.t[q]; }
  __syncthreads();
  const int tile = blockIdx.x % p.tiles;
  const long long row = blockIdx.x / p.tiles;
  const int t = tile * kAdjT + threadIdx.x;
  if (t >= p.count) return;
  const int i = (p.count == p.N || t < p.depth) ? t : p.N - 2 * p.depth + t;
  const T* lo = p.lo + row * p.K;
  const T* hi = p.hi ? p.hi + row * p.K : nullptr;
  const Images im = images_of(i, p.N, p.mode);
  const int phi = 2 * p.K - 3 + p.L - p.pl;
  T acc = T(0);
  for (int a = 0; a < im.nb; ++a) {
    for (int q = first_image(im.base(a), im.per, -p.pl); q <= phi; q += im.per) {
      const int kmin = imax(0, floordiv2(q + p.pl - p.L + 2)), kmax = imin(p.K - 1, floordiv2(q + p.pl));
      for (int k = kmin; k <= kmax; ++k) {
        const int tt = q + p.pl - 2 * k;
        acc = fma_rn(f0[tt], lo[k], acc);
        if (hi) acc = fma_rn(f1[tt], hi[k], acc);
      }
    }
  }
  p.y[row * p.N + i] = acc;
}

}  // namespace b200w

using namespace b200w;

namespace {

int sfb2d_entry(const float* ll, long long llps, int llpitch, const float* highs, float* y, long long yps, int ypitch,
                int planes, int Hc, int Wc, int Ho, int Wo, const float* gh_lo, const float* gh_hi, int Lh,
                const float* gw_lo, const float* gw_hi, int Lw, int mode, void* stream) {
  return b200w_dwt_sfb2d(ll, llps, llpitch, highs, y, yps, ypitch, planes, Hc, Wc, Ho, Wo, gh_lo, gh_hi, Lh, gw_lo,
                         gw_hi, Lw, mode, stream);
}
int sfb2d_entry(const double* ll, long long llps, int llpitch, const double* highs, double* y, long long yps,
                int ypitch, int planes, int Hc, int Wc, int Ho, int Wo, const double* gh_lo, const double* gh_hi,
                int Lh, const double* gw_lo, const double* gw_hi, int Lw, int mode, void* stream) {
  return b200w_dwt_sfb2d_f64(ll, llps, llpitch, highs, y, yps, ypitch, planes, Hc, Wc, Ho, Wo, gh_lo, gh_hi, Lh,
                             gw_lo, gw_hi, Lw, mode, stream);
}
int sfb1d_entry(const float* lo, const float* hi, int rows, int K, float* y, int N, const float* f0, const float* f1,
                int L, int mode, void* stream) {
  return b200w_dwt_sfb1d(lo, hi, rows, K, y, N, f0, f1, L, mode, stream);
}
int sfb1d_entry(const double* lo, const double* hi, int rows, int K, double* y, int N, const double* f0,
                const double* f1, int L, int mode, void* stream) {
  return b200w_dwt_sfb1d_f64(lo, hi, rows, K, y, N, f0, f1, L, mode, stream);
}

int ext_pl(int L, int mode) { return mode == B200W_MODE_PERIODIZATION ? L - 1 - L / 2 : L - 2; }

// Outputs within this many of an edge can differ from the cropped synthesis (see the file comment).
int border_depth(int n, int L, int mode) { return (mode == B200W_MODE_PERIODIZATION && (L & 1)) ? n : L; }

// The synthesis level alone is A_m^T along an axis: zero mode, and periodization with n and L even.
bool synthesis_exact(int n, int L, int mode) {
  return mode == B200W_MODE_ZERO || (mode == B200W_MODE_PERIODIZATION && !(n & 1) && !(L & 1));
}

template <class T>
int afb2d_adjoint_impl(const T* ll, long long ll_plane_stride, int ll_pitch, const T* highs, T* y,
                       long long y_plane_stride, int y_pitch, int planes, int Hc, int Wc, int H, int W, const T* fh_lo,
                       const T* fh_hi, int Lh, const T* fw_lo, const T* fw_hi, int Lw, int mode, void* stream) {
  if (!dwt_mode_ok(mode)) return B200W_EMODE;
  if (!ll || !y) return B200W_EARG;
  if (planes < 0 || H < 1 || W < 1) return B200W_ESIZE;
  if (Lh < 2 || Lw < 2) return B200W_EFILTER;
  Adj2dParams<T> p;
  int rc;
  if ((rc = set_taps(p.fh_lo, fh_lo, Lh)) || (rc = set_taps(p.fh_hi, fh_hi, Lh)) ||
      (rc = set_taps(p.fw_lo, fw_lo, Lw)) || (rc = set_taps(p.fw_hi, fw_hi, Lw)))
    return rc;
  if (Hc != coeff_len(H, Lh, mode) || Wc != coeff_len(W, Lw, mode)) return B200W_ESIZE;
  if (ll_pitch < Wc || y_pitch < W) return B200W_EARG;
  p.ll = ll; p.llps = ll_plane_stride; p.llpitch = ll_pitch; p.highs = highs;
  p.y = y; p.yps = y_plane_stride; p.ypitch = y_pitch;
  p.planes = planes; p.Hc = Hc; p.Wc = Wc; p.H = H; p.W = W; p.Lh = Lh; p.Lw = Lw; p.mode = mode;
  p.plh = ext_pl(Lh, mode); p.plw = ext_pl(Lw, mode);
  p.dh = border_depth(H, Lh, mode); p.dw = border_depth(W, Lw, mode);
  const long long count = border_count(H, W, p.dh, p.dw);
  p.count = (int)count;
  p.tiles = cdiv(p.count, kAdjT);
  const long long blocks = (long long)planes * p.tiles;
  if (count > 2147483647LL || !grid_ok(blocks)) return B200W_ESIZE;
  if ((rc = sfb2d_entry(ll, ll_plane_stride, ll_pitch, highs, y, y_plane_stride, y_pitch, planes, Hc, Wc, H, W, fh_lo,
                        fh_hi, Lh, fw_lo, fw_hi, Lw, mode, stream)))
    return rc;
  if (synthesis_exact(H, Lh, mode) && synthesis_exact(W, Lw, mode)) return B200W_OK;
  return launch(afb2d_adjoint_border<T>, p, blocks, kAdjT, 0, stream);
}

template <class T>
int afb1d_adjoint_impl(const T* lo, const T* hi, int rows, int K, T* y, int N, const T* f0, const T* f1, int L,
                       int mode, void* stream) {
  if (!dwt_mode_ok(mode)) return B200W_EMODE;
  if (!lo || !y) return B200W_EARG;
  if (rows < 0 || N < 1) return B200W_ESIZE;
  if (L < 2) return B200W_EFILTER;
  Adj1dParams<T> p;
  int rc;
  if ((rc = set_taps(p.f0, f0, L)) || (rc = set_taps(p.f1, f1, L))) return rc;
  if (K != coeff_len(N, L, mode)) return B200W_ESIZE;
  p.lo = lo; p.hi = hi; p.y = y;
  p.rows = rows; p.K = K; p.N = N; p.L = L; p.mode = mode; p.pl = ext_pl(L, mode);
  p.depth = border_depth(N, L, mode);
  p.count = (2 * p.depth >= N) ? N : 2 * p.depth;
  p.tiles = cdiv(p.count, kAdjT);
  const long long blocks = (long long)rows * p.tiles;
  if (!grid_ok(blocks)) return B200W_ESIZE;
  if ((rc = sfb1d_entry(lo, hi, rows, K, y, N, f0, f1, L, mode, stream))) return rc;
  if (synthesis_exact(N, L, mode)) return B200W_OK;
  return launch(afb1d_adjoint_border<T>, p, blocks, kAdjT, 0, stream);
}

}  // namespace

extern "C" {

int b200w_dwt_afb2d_adjoint(const float* ll, long long ll_plane_stride, int ll_pitch, const float* highs, float* y,
                            long long y_plane_stride, int y_pitch, int planes, int Hc, int Wc, int H, int W,
                            const float* fh_lo, const float* fh_hi, int Lh, const float* fw_lo, const float* fw_hi,
                            int Lw, int mode, void* stream) {
  return afb2d_adjoint_impl(ll, ll_plane_stride, ll_pitch, highs, y, y_plane_stride, y_pitch, planes, Hc, Wc, H, W,
                            fh_lo, fh_hi, Lh, fw_lo, fw_hi, Lw, mode, stream);
}
int b200w_dwt_afb2d_adjoint_f64(const double* ll, long long ll_plane_stride, int ll_pitch, const double* highs,
                                double* y, long long y_plane_stride, int y_pitch, int planes, int Hc, int Wc, int H,
                                int W, const double* fh_lo, const double* fh_hi, int Lh, const double* fw_lo,
                                const double* fw_hi, int Lw, int mode, void* stream) {
  return afb2d_adjoint_impl(ll, ll_plane_stride, ll_pitch, highs, y, y_plane_stride, y_pitch, planes, Hc, Wc, H, W,
                            fh_lo, fh_hi, Lh, fw_lo, fw_hi, Lw, mode, stream);
}

int b200w_dwt_afb1d_adjoint(const float* lo, const float* hi, int rows, int K, float* y, int N, const float* f0,
                            const float* f1, int L, int mode, void* stream) {
  return afb1d_adjoint_impl(lo, hi, rows, K, y, N, f0, f1, L, mode, stream);
}
int b200w_dwt_afb1d_adjoint_f64(const double* lo, const double* hi, int rows, int K, double* y, int N,
                                const double* f0, const double* f1, int L, int mode, void* stream) {
  return afb1d_adjoint_impl(lo, hi, rows, K, y, N, f0, f1, L, mode, stream);
}

}  // extern "C"
