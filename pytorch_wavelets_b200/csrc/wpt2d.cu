// wpt2d.cu -- 2-D wavelet packet levels (sm_90a): b200w_wpt_afb2d / b200w_wpt_sfb2d and their _generic / _f64 twins.
//
// A packet level applies one DWT level (AFB2D / SFB2D arithmetic) to every plane.  Layout: the four children of plane p
// (ll, lh, hl, hh) are nodes 4p .. 4p+3 of the output, so the level's (P, 4, Ho, Wo) output is the next level's list of
// 4P planes.  Three routes, chosen per level:
//   * streaming (wpt_afb2d_stream / wpt_sfb2d_stream / wpt_sfb2d_stream4): the float32 DWT streaming kernels compiled
//     for the packet layout (afb_stream_kernel.cuh, sfb_stream_kernel.cuh, k_wpt_stream.cu), wherever they apply.
//   * packed (wpt_afb2d_packed / wpt_sfb2d_packed, below): small planes, float and double.  A CTA stages several WHOLE
//     planes in shared memory with the boundary extension resolved by index arithmetic, runs both 1-D passes there and
//     writes its planes' outputs, which in the packet layout are one contiguous span (coalesced loads and stores).
//     Synthesis levels of at most 8 coefficient columns, and small levels the streaming kernels do not cover.
//   * tile (k_wpt_afb2d_tile / k_wpt_sfb2d_tile): the generic tile kernels compiled for the packet layout, for
//     everything else and for the _generic entries.
// The packed kernel was written for the deep levels, where a streaming warp (64 output columns of one plane) idles most
// of its lanes.  Measured, the streaming kernels still win there from 16 columns up (and the analysis one at 8): they
// keep many more bytes in flight.  The packed kernel beats the tile kernel at every small size measured.
// The packed kernels accumulate exactly as the tile kernels (stored-tap order from a zero accumulator, FMA; synthesis
// H pass then W pass, one rounded add per pass), so analysis is bit-identical to the oracle and to the tile kernel,
// and synthesis bit-identical to the tile kernel.
#include <cuda_runtime.h>

#include <type_traits>

#include "fast_api.h"
#include "launch.cuh"
#include "launch_params.h"

namespace b200w {
namespace {

constexpr int kWptNT = 256;                      // threads per CTA of the tile and packed kernels
// Routes (measured on an H100, DESIGN.md section 4g): the streaming kernel wherever it applies, except synthesis levels
// of at most kWptPackedFirstW coefficient columns, which take the packed kernel; where the streaming kernel does not
// apply (float64, unequal filter lengths, unaligned analysis input, more than 20 taps) the packed kernel for levels whose
// small side (analysis Wo, synthesis Wc) is at most kWptPackedMaxW, the tile kernel otherwise.  The packed kernel also
// needs one plane's working set to fit kWptPlaneMaxBytes of shared memory.
constexpr int kWptPackedFirstW = 8;
constexpr int kWptPackedMaxW = 40;
constexpr long long kWptPlaneMaxBytes = 64 * 1024;
constexpr long long kWptCtaBytes = 48 * 1024;     // planes are packed up to this much shared memory per CTA ...
constexpr long long kWptCtaOutputs = 4096;       // ... or until the CTA writes this many outputs

extern __shared__ __align__(16) unsigned char g_wpt_smem[];

template <class T> __global__ void __launch_bounds__(kWptNT) k_wpt_afb2d_tile(const __grid_constant__ AfbParamsT<T> p) { afb2d_tile<kWptNT, T, true>(p, blockIdx.x, reinterpret_cast<T*>(g_wpt_smem)); }
template <class T> __global__ void __launch_bounds__(kWptNT) k_wpt_sfb2d_tile(const __grid_constant__ SfbParamsT<T> p) { sfb2d_tile<kWptNT, T, true>(p, blockIdx.x, reinterpret_cast<T*>(g_wpt_smem)); }

// ---- packed small-plane analysis -----------------------------------------------------------------------------------
// Per plane: the extended input (IH x IW, rows IWp apart), then the W-pass low / high (IH x Wo each).
B200W_HD long long afb_packed_floats(int Ho, int Wo, int Lw, int Lh) {
  const int IW = 2 * Wo + Lw - 2, IH = 2 * Ho + Lh - 2;
  return (long long)IH * (IW | 1) + 2LL * IH * Wo;
}

// LC: filter length compiled in (Lw == Lh == LC), 0 = the runtime lengths p.Lw / p.Lh.  ppc planes per CTA.
template <class T, int LC>
__global__ void __launch_bounds__(kWptNT, 1) wpt_afb2d_packed(const __grid_constant__ AfbParamsT<T> p, int ppc) {
  T* smem = reinterpret_cast<T*>(g_wpt_smem);
  const int Lw = LC ? LC : p.Lw, Lh = LC ? LC : p.Lh, mode = p.mode;
  const int Ho = p.Ho, Wo = p.Wo;
  const int plw = (mode == B200W_MODE_PERIODIZATION) ? (Lw - 1 - Lw / 2) : (Lw - 2);
  const int plh = (mode == B200W_MODE_PERIODIZATION) ? (Lh - 1 - Lh / 2) : (Lh - 2);
  const int IW = 2 * Wo + Lw - 2, IH = 2 * Ho + Lh - 2, IWp = IW | 1;
  const int plane0 = blockIdx.x * ppc;
  const int np = imin(ppc, p.planes - plane0);
  T* s_in = smem;
  T* s_lo = s_in + (long long)np * IH * IWp;
  T* s_hi = s_lo + (long long)np * IH * Wo;

  // stage every row of the CTA's planes, boundary extension by index arithmetic (as afb2d_tile)
  for (int rr = threadIdx.x / 32; rr < np * IH; rr += kWptNT / 32) {
    const int q = rr / IH, r = rr - q * IH;
    const int gr = ext_index(r - plh, p.H, mode);
    const T* src = p.x + (long long)(plane0 + q) * p.xps + (long long)(gr < 0 ? 0 : gr) * p.xpitch;
    for (int c = threadIdx.x & 31; c < IW; c += 32) {
      const int gc = ext_index(c - plw, p.W, mode);
      s_in[rr * IWp + c] = (gr < 0 || gc < 0) ? T(0) : src[gc];
    }
  }
  __syncthreads();

  // W pass: every staged row -> low / high of each output column
  for (int idx = threadIdx.x; idx < np * IH * Wo; idx += kWptNT) {
    const int rr = idx / Wo, k = idx - rr * Wo;
    const T* row = s_in + rr * IWp + 2 * k;
    T a0 = 0, a1 = 0;
    auto tap = [&](int j) {
      const T v = row[j];
      a0 = fma_rn(p.fw_lo.t[j], v, a0);
      a1 = fma_rn(p.fw_hi.t[j], v, a1);
    };
    if (LC) {
#pragma unroll
      for (int j = 0; j < (LC ? LC : 1); ++j) tap(j);
    } else {
      for (int j = 0; j < Lw; ++j) tap(j);
    }
    s_lo[idx] = a0;
    s_hi[idx] = a1;
  }
  __syncthreads();

  // H pass and store: consecutive threads take consecutive output columns, so with rows Wo apart (the packet layout's
  // contiguous case) each band's stores of a warp are one contiguous run
  const long long ns = p.llps >> 2;   // node stride
  for (int idx = threadIdx.x; idx < np * Ho * Wo; idx += kWptNT) {
    const int t = idx / Wo, kc = idx - t * Wo;
    const int q = t / Ho, kr = t - q * Ho;
    const T* lo = s_lo + ((long long)q * IH + 2 * kr) * Wo + kc;
    const T* hi = s_hi + ((long long)q * IH + 2 * kr) * Wo + kc;
    T all = 0, alh = 0, ahl = 0, ahh = 0;
    auto tap = [&](int j) {
      const T vlo = lo[j * Wo], vhi = hi[j * Wo];
      const T f0 = p.fh_lo.t[j], f1 = p.fh_hi.t[j];
      all = fma_rn(f0, vlo, all);
      alh = fma_rn(f1, vlo, alh);
      ahl = fma_rn(f0, vhi, ahl);
      ahh = fma_rn(f1, vhi, ahh);
    };
    if (LC) {
#pragma unroll
      for (int j = 0; j < (LC ? LC : 1); ++j) tap(j);
    } else {
      for (int j = 0; j < Lh; ++j) tap(j);
    }
    T* y = p.ll + 4LL * (plane0 + q) * ns + (long long)kr * p.llpitch + kc;
    y[0] = all;
    y[ns] = alh;
    y[2 * ns] = ahl;
    y[3 * ns] = ahh;
  }
}

// ---- packed small-plane synthesis ----------------------------------------------------------------------------------
// Per plane: the four children over the coefficient rows / columns any output touches (KH x KW each, wrapped for
// periodization, zero outside otherwise), then the H-pass low / high (Ho x KW each).
struct SfbSpan { int k0, n; };
B200W_HD SfbSpan sfb_packed_span(int No, int L, bool per) {
  const int off = per ? (L / 2 - 1) : (L - 2);
  const int k0 = floordiv2(off - L + 2);
  return {k0, floordiv2(No - 1 + off) - k0 + 1};
}
B200W_HD long long sfb_packed_floats(int Ho, int Wo, int Lh, int Lw, int mode) {
  const bool per = (mode == B200W_MODE_PERIODIZATION);
  const SfbSpan sh = sfb_packed_span(Ho, Lh, per), sw = sfb_packed_span(Wo, Lw, per);
  return 4LL * sh.n * sw.n + 2LL * Ho * sw.n;
}

template <class T, int LC>
__global__ void __launch_bounds__(kWptNT) wpt_sfb2d_packed(const __grid_constant__ SfbParamsT<T> p, int ppc) {
  T* smem = reinterpret_cast<T*>(g_wpt_smem);
  const int Lh = LC ? LC : p.Lh, Lw = LC ? LC : p.Lw;
  const bool per = (p.mode == B200W_MODE_PERIODIZATION);
  const int offh = per ? (Lh / 2 - 1) : (Lh - 2);
  const int offw = per ? (Lw / 2 - 1) : (Lw - 2);
  const int Hc = p.Hc, Wc = p.Wc, Ho = p.Ho, Wo = p.Wo;
  const SfbSpan sh = sfb_packed_span(Ho, Lh, per), sw = sfb_packed_span(Wo, Lw, per);
  const int KH = sh.n, KW = sw.n, kh0 = sh.k0, kw0 = sw.k0;
  const int plane0 = blockIdx.x * ppc;
  const int np = imin(ppc, p.planes - plane0);
  const long long band = (long long)Hc * Wc;
  T* s_b = smem;                                   // [plane][child][KH][KW]
  T* s_lo = s_b + 4LL * np * KH * KW;              // [plane][Ho][KW]
  T* s_hi = s_lo + (long long)np * Ho * KW;

  // the children of the CTA's planes are 4 * np consecutive nodes: one contiguous span of the input
  const T* c = p.ll + 4LL * plane0 * band;
  for (int idx = threadIdx.x; idx < 4 * np * KH * KW; idx += kWptNT) {
    const int t = idx / KW, j = idx - t * KW;
    const int node = t / KH, i = t - node * KH;
    int kr = kh0 + i, kc = kw0 + j;
    bool ok = true;
    if (per) {
      kr %= Hc; if (kr < 0) kr += Hc;
      kc %= Wc; if (kc < 0) kc += Wc;
    } else {
      ok = (kr >= 0 && kr < Hc && kc >= 0 && kc < Wc);
    }
    s_b[idx] = ok ? c[node * band + (long long)kr * Wc + kc] : T(0);
  }
  __syncthreads();

  // H pass: lo = S(ll, lh), hi = S(hl, hh)
  for (int idx = threadIdx.x; idx < np * Ho * KW; idx += kWptNT) {
    const int t = idx / KW, j = idx - t * KW;
    const int q = t / Ho, n = t - q * Ho;
    const T* b0 = s_b + 4LL * q * KH * KW + j;
    const T* b1 = b0 + KH * KW;
    const T* b2 = b1 + KH * KW;
    const T* b3 = b2 + KH * KW;
    const int s = n + offh;
    const int kmin = floordiv2(s - Lh + 2), kmax = floordiv2(s);
    T a0 = 0, a1 = 0, c0 = 0, c1 = 0;
    auto tap = [&](int k) {
      const int tt = s - 2 * k;
      const int o = (k - kh0) * KW;
      const T g0 = p.gh_lo.t[tt], g1 = p.gh_hi.t[tt];
      a0 = fma_rn(b0[o], g0, a0);
      a1 = fma_rn(b1[o], g1, a1);
      c0 = fma_rn(b2[o], g0, c0);
      c1 = fma_rn(b3[o], g1, c1);
    };
    if (LC) {   // an even length: always LC / 2 coefficients
#pragma unroll
      for (int u = 0; u < (LC ? LC / 2 : 1); ++u) tap(kmin + u);
    } else {
      for (int k = kmin; k <= kmax; ++k) tap(k);
    }
    s_lo[idx] = add_rn(a0, a1);
    s_hi[idx] = add_rn(c0, c1);
  }
  __syncthreads();

  // W pass and store
  for (int idx = threadIdx.x; idx < np * Ho * Wo; idx += kWptNT) {
    const int t = idx / Wo, m = idx - t * Wo;
    const int q = t / Ho, n = t - q * Ho;
    const T* lo = s_lo + (long long)t * KW - kw0;
    const T* hi = s_hi + (long long)t * KW - kw0;
    const int s = m + offw;
    const int kmin = floordiv2(s - Lw + 2), kmax = floordiv2(s);
    T a0 = 0, a1 = 0;
    auto tap = [&](int k) {
      const int tt = s - 2 * k;
      a0 = fma_rn(lo[k], p.gw_lo.t[tt], a0);
      a1 = fma_rn(hi[k], p.gw_hi.t[tt], a1);
    };
    if (LC) {
#pragma unroll
      for (int u = 0; u < (LC ? LC / 2 : 1); ++u) tap(kmin + u);
    } else {
      for (int k = kmin; k <= kmax; ++k) tap(k);
    }
    p.y[(long long)(plane0 + q) * p.yps + (long long)n * p.ypitch + m] = add_rn(a0, a1);
  }
}

// ---- routing --------------------------------------------------------------------------------------------------------

// planes per CTA of the packed route, or 0 when it does not apply (small side above max_w, or a plane's working set too
// large)
template <class T>
int packed_ppc(int planes, int w_small, int max_w, long long plane_floats, long long plane_outputs) {
  const long long bytes = plane_floats * (long long)sizeof(T);
  if (w_small > max_w || bytes > kWptPlaneMaxBytes) return 0;
  long long ppc = kWptCtaBytes / bytes;
  const long long by_out = (kWptCtaOutputs + plane_outputs - 1) / plane_outputs;
  if (by_out < ppc) ppc = by_out;
  if (ppc > planes) ppc = planes;
  return ppc < 1 ? 1 : (int)ppc;
}

template <class T, class P>
int launch_packed(void (*kernel)(P, int), const P& p, int ppc, long long floats_per_plane, void* stream) {
  const long long blocks = ((long long)p.planes + ppc - 1) / ppc;
  if (!grid_ok(blocks)) return B200W_ESIZE;
  const size_t smem = (size_t)(floats_per_plane * ppc) * sizeof(T);
  if (smem > 48 * 1024) {
    const int rc = check_cuda(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    if (rc) return rc;
  }
  kernel<<<(unsigned)blocks, kWptNT, smem, (cudaStream_t)stream>>>(p, ppc);
  return check_launch();
}

// the compiled instantiation for Lw == Lh of a named even length, else the runtime-length one
template <class T>
auto afb_packed_kernel(int Lw, int Lh) -> void (*)(AfbParamsT<T>, int) {
  if (Lw == Lh) {
    switch (Lw) {
      case 2: return wpt_afb2d_packed<T, 2>;
      case 4: return wpt_afb2d_packed<T, 4>;
      case 6: return wpt_afb2d_packed<T, 6>;
      case 8: return wpt_afb2d_packed<T, 8>;
      case 10: return wpt_afb2d_packed<T, 10>;
      case 12: return wpt_afb2d_packed<T, 12>;
      case 14: return wpt_afb2d_packed<T, 14>;
      case 16: return wpt_afb2d_packed<T, 16>;
      case 18: return wpt_afb2d_packed<T, 18>;
      case 20: return wpt_afb2d_packed<T, 20>;
      default: break;
    }
  }
  return wpt_afb2d_packed<T, 0>;
}

template <class T>
auto sfb_packed_kernel(int Lh, int Lw) -> void (*)(SfbParamsT<T>, int) {
  if (Lw == Lh) {
    switch (Lw) {
      case 2: return wpt_sfb2d_packed<T, 2>;
      case 4: return wpt_sfb2d_packed<T, 4>;
      case 6: return wpt_sfb2d_packed<T, 6>;
      case 8: return wpt_sfb2d_packed<T, 8>;
      case 10: return wpt_sfb2d_packed<T, 10>;
      case 12: return wpt_sfb2d_packed<T, 12>;
      case 14: return wpt_sfb2d_packed<T, 14>;
      case 16: return wpt_sfb2d_packed<T, 16>;
      case 18: return wpt_sfb2d_packed<T, 18>;
      case 20: return wpt_sfb2d_packed<T, 20>;
      default: break;
    }
  }
  return wpt_sfb2d_packed<T, 0>;
}

// generic: the _generic entry (float32 tile kernel only)
template <class T>
int wpt_afb2d_impl(const T* x, long long x_plane_stride, int x_pitch, T* y, long long y_node_stride, int y_pitch,
                   int planes, int H, int W, const T* fw_lo, const T* fw_hi, int Lw, const T* fh_lo, const T* fh_hi,
                   int Lh, int mode, void* stream, bool generic) {
  if (!dwt_mode_ok(mode)) return B200W_EMODE;
  if (!x || !y) return B200W_EARG;
  if (Lw < 2 || Lh < 2 || Lw > kMaxTaps || Lh > kMaxTaps) return B200W_EFILTER;
  AfbParamsT<T> p;
  int rc = build_afb(p, x, x_plane_stride, x_pitch, y, 4 * y_node_stride, y_pitch, y + y_node_stride, planes, H, W,
                     fw_lo, fw_hi, Lw, fh_lo, fh_hi, Lh, mode);
  if (rc) return rc;
  if (y_node_stride < (long long)p.Ho * y_pitch) return B200W_EARG;
  p.hipitch = y_pitch;
  if (planes == 0) return B200W_OK;
  if (!generic) {
    if constexpr (std::is_same_v<T, float>) {
      rc = fast::try_launch_wpt_afb(p, (cudaStream_t)stream);
      if (rc != fast::kNoFastPath) return rc ? rc : check_launch();
    }
    const long long fl = afb_packed_floats(p.Ho, p.Wo, Lw, Lh);
    const int ppc = packed_ppc<T>(planes, p.Wo, kWptPackedMaxW, fl, 4LL * p.Ho * p.Wo);
    if (ppc > 0) return launch_packed<T>(afb_packed_kernel<T>(Lw, Lh), p, ppc, fl, stream);
  }
  return launch(k_wpt_afb2d_tile<T>, p, (long long)planes * p.tiles_x * p.tiles_y, kWptNT,
                (size_t)afb_smem_floats(Lw, Lh) * sizeof(T), stream);
}

template <class T>
int wpt_sfb2d_impl(const T* c, T* y, long long y_plane_stride, int y_pitch, int planes, int Hc, int Wc, int Ho, int Wo,
                   const T* gh_lo, const T* gh_hi, int Lh, const T* gw_lo, const T* gw_hi, int Lw, int mode,
                   void* stream, bool generic) {
  if (!dwt_mode_ok(mode)) return B200W_EMODE;
  if (!c || !y) return B200W_EARG;
  if (Lw < 2 || Lh < 2 || Lw > kMaxTaps || Lh > kMaxTaps) return B200W_EFILTER;
  if (Hc < 1 || Wc < 1) return B200W_ESIZE;
  const long long band = (long long)Hc * Wc;
  SfbParamsT<T> p;
  int rc = build_sfb(p, c, 4 * band, Wc, c + band, y, y_plane_stride, y_pitch, planes, Hc, Wc, Ho, Wo, gh_lo, gh_hi,
                     Lh, gw_lo, gw_hi, Lw, mode);
  if (rc) return rc;
  if (y_plane_stride < (long long)Ho * y_pitch) return B200W_EARG;
  if (planes == 0) return B200W_OK;
  if (!generic) {
    const long long fl = sfb_packed_floats(Ho, Wo, Lh, Lw, mode);
    const auto packed = [&](int max_w) {
      const int ppc = packed_ppc<T>(planes, Wc, max_w, fl, (long long)Ho * Wo);
      return ppc > 0 ? launch_packed<T>(sfb_packed_kernel<T>(Lh, Lw), p, ppc, fl, stream) : fast::kNoFastPath;
    };
    if ((rc = packed(kWptPackedFirstW)) != fast::kNoFastPath) return rc;
    if constexpr (std::is_same_v<T, float>) {
      rc = fast::try_launch_wpt_sfb(p, (cudaStream_t)stream);
      if (rc != fast::kNoFastPath) return rc ? rc : check_launch();
    }
    if ((rc = packed(kWptPackedMaxW)) != fast::kNoFastPath) return rc;
  }
  return launch(k_wpt_sfb2d_tile<T>, p, (long long)planes * p.tiles_x * p.tiles_y, kWptNT,
                (size_t)sfb_smem_floats(Lh, Lw) * sizeof(T), stream);
}

}  // namespace
}  // namespace b200w

using namespace b200w;

extern "C" {

int b200w_wpt_afb2d(const float* x, long long x_plane_stride, int x_pitch, float* y, long long y_node_stride,
                    int y_pitch, int planes, int H, int W, const float* fw_lo, const float* fw_hi, int Lw,
                    const float* fh_lo, const float* fh_hi, int Lh, int mode, void* stream) {
  return wpt_afb2d_impl<float>(x, x_plane_stride, x_pitch, y, y_node_stride, y_pitch, planes, H, W, fw_lo, fw_hi, Lw,
                               fh_lo, fh_hi, Lh, mode, stream, false);
}
int b200w_wpt_afb2d_generic(const float* x, long long x_plane_stride, int x_pitch, float* y, long long y_node_stride,
                            int y_pitch, int planes, int H, int W, const float* fw_lo, const float* fw_hi, int Lw,
                            const float* fh_lo, const float* fh_hi, int Lh, int mode, void* stream) {
  return wpt_afb2d_impl<float>(x, x_plane_stride, x_pitch, y, y_node_stride, y_pitch, planes, H, W, fw_lo, fw_hi, Lw,
                               fh_lo, fh_hi, Lh, mode, stream, true);
}
int b200w_wpt_afb2d_f64(const double* x, long long x_plane_stride, int x_pitch, double* y, long long y_node_stride,
                        int y_pitch, int planes, int H, int W, const double* fw_lo, const double* fw_hi, int Lw,
                        const double* fh_lo, const double* fh_hi, int Lh, int mode, void* stream) {
  return wpt_afb2d_impl<double>(x, x_plane_stride, x_pitch, y, y_node_stride, y_pitch, planes, H, W, fw_lo, fw_hi, Lw,
                                fh_lo, fh_hi, Lh, mode, stream, false);
}

int b200w_wpt_sfb2d(const float* c, float* y, long long y_plane_stride, int y_pitch, int planes, int Hc, int Wc,
                    int Ho, int Wo, const float* gh_lo, const float* gh_hi, int Lh, const float* gw_lo,
                    const float* gw_hi, int Lw, int mode, void* stream) {
  return wpt_sfb2d_impl<float>(c, y, y_plane_stride, y_pitch, planes, Hc, Wc, Ho, Wo, gh_lo, gh_hi, Lh, gw_lo, gw_hi,
                               Lw, mode, stream, false);
}
int b200w_wpt_sfb2d_generic(const float* c, float* y, long long y_plane_stride, int y_pitch, int planes, int Hc,
                            int Wc, int Ho, int Wo, const float* gh_lo, const float* gh_hi, int Lh, const float* gw_lo,
                            const float* gw_hi, int Lw, int mode, void* stream) {
  return wpt_sfb2d_impl<float>(c, y, y_plane_stride, y_pitch, planes, Hc, Wc, Ho, Wo, gh_lo, gh_hi, Lh, gw_lo, gw_hi,
                               Lw, mode, stream, true);
}
int b200w_wpt_sfb2d_f64(const double* c, double* y, long long y_plane_stride, int y_pitch, int planes, int Hc, int Wc,
                        int Ho, int Wo, const double* gh_lo, const double* gh_hi, int Lh, const double* gw_lo,
                        const double* gw_hi, int Lw, int mode, void* stream) {
  return wpt_sfb2d_impl<double>(c, y, y_plane_stride, y_pitch, planes, Hc, Wc, Ho, Wo, gh_lo, gh_hi, Lh, gw_lo, gw_hi,
                                Lw, mode, stream, false);
}

}  // extern "C"
