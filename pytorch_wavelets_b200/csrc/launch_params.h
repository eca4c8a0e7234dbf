// launch_params.h -- host-side validation and parameter-block construction for every C-ABI entry
// point (plain C++, no CUDA): shared by the CUDA launchers (b200wave.cu) and by the host
// emulation used in CPU tests (tests/emu/emu.cpp), so the argument checking and tiling logic the
// tests exercise is the code that ships.
#pragma once
#include <string.h>

#include "tile_kernels.h"

namespace b200w {

inline bool dwt_mode_ok(int mode) {
  // modes accepted by afb1d / sfb1d (reference dwt/lowlevel.py:134,155,165,263-264)
  return mode == B200W_MODE_ZERO || mode == B200W_MODE_SYMMETRIC || mode == B200W_MODE_PERIODIZATION ||
         mode == B200W_MODE_REFLECT || mode == B200W_MODE_PERIODIC;
}

inline int coeff_len(int n, int flen, int mode) {
  if (n < 1 || flen < 1) return B200W_ESIZE;
  return mode == B200W_MODE_PERIODIZATION ? (n + 1) / 2 : (n + flen - 1) / 2;
}
inline int rec_len(int k, int flen, int mode) {
  if (k < 1 || flen < 1) return B200W_ESIZE;
  return mode == B200W_MODE_PERIODIZATION ? 2 * k : 2 * k - flen + 2;
}

template <class T>
inline int set_taps(TapsT<T>& dst, const T* src, int L) {
  if (!src) return B200W_EARG;
  if (L < 1 || L > kMaxTaps) return B200W_EFILTER;
  memset(&dst, 0, sizeof(dst));
  for (int i = 0; i < L; ++i) dst.t[i] = src[i];
  return 0;
}

inline int cdiv(int a, int b) { return (a + b - 1) / b; }

// Total CTA count must fit a 1-D grid.
inline bool grid_ok(long long blocks) { return blocks >= 0 && blocks <= 2147483647LL; }

template <class T>
inline int build_afb(AfbParamsT<T>& p, const T* x, long long xps, int xpitch, T* ll, long long llps,
                     int llpitch, T* highs, int planes, int H, int W, const T* fw_lo,
                     const T* fw_hi, int Lw, const T* fh_lo, const T* fh_hi, int Lh, int mode) {
  if (!dwt_mode_ok(mode)) return B200W_EMODE;
  if (!x || !ll || !highs) return B200W_EARG;
  if (planes < 0 || H < 1 || W < 1) return B200W_ESIZE;
  if (Lw < 2 || Lh < 2) return B200W_EFILTER;
  int rc;
  if ((rc = set_taps(p.fw_lo, fw_lo, Lw)) || (rc = set_taps(p.fw_hi, fw_hi, Lw)) ||
      (rc = set_taps(p.fh_lo, fh_lo, Lh)) || (rc = set_taps(p.fh_hi, fh_hi, Lh)))
    return rc;
  for (int i = 0; i < kMaxTaps; ++i) { p.fwp[2 * i] = p.fw_lo.t[i]; p.fwp[2 * i + 1] = p.fw_hi.t[i]; }
  p.x = x; p.xps = xps; p.xpitch = xpitch;
  p.ll = ll; p.llps = llps; p.llpitch = llpitch;
  p.hipitch = 0;
  p.highs = highs;
  p.planes = planes; p.H = H; p.W = W;
  p.Ho = coeff_len(H, Lh, mode); p.Wo = coeff_len(W, Lw, mode);
  p.Lw = Lw; p.Lh = Lh; p.mode = mode;
  if (xpitch < W || llpitch < p.Wo) return B200W_EARG;
  p.tiles_x = cdiv(p.Wo, kAfbTW);
  p.tiles_y = cdiv(p.Ho, kAfbTH);
  if (!grid_ok((long long)planes * p.tiles_x * p.tiles_y)) return B200W_ESIZE;
  return 0;
}

template <class T>
inline int build_sfb(SfbParamsT<T>& p, const T* ll, long long llps, int llpitch, const T* highs, T* y,
                     long long yps, int ypitch, int planes, int Hc, int Wc, int Ho, int Wo, const T* gh_lo,
                     const T* gh_hi, int Lh, const T* gw_lo, const T* gw_hi, int Lw, int mode) {
  if (!dwt_mode_ok(mode)) return B200W_EMODE;
  if (!ll || !y) return B200W_EARG;
  if (planes < 0 || Hc < 1 || Wc < 1) return B200W_ESIZE;
  if (Lw < 2 || Lh < 2) return B200W_EFILTER;
  const int Hn = rec_len(Hc, Lh, mode), Wn = rec_len(Wc, Lw, mode);
  if (Ho < 1 || Wo < 1 || Ho > Hn || Wo > Wn) return B200W_ESIZE;
  int rc;
  if ((rc = set_taps(p.gh_lo, gh_lo, Lh)) || (rc = set_taps(p.gh_hi, gh_hi, Lh)) ||
      (rc = set_taps(p.gw_lo, gw_lo, Lw)) || (rc = set_taps(p.gw_hi, gw_hi, Lw)))
    return rc;
  p.ll = ll; p.llps = llps; p.llpitch = llpitch;
  p.highs = highs;
  p.y = y; p.yps = yps; p.ypitch = ypitch;
  p.planes = planes; p.Hc = Hc; p.Wc = Wc; p.Ho = Ho; p.Wo = Wo;
  p.Lh = Lh; p.Lw = Lw; p.mode = mode;
  if (llpitch < Wc || ypitch < Wo) return B200W_EARG;
  p.tiles_x = cdiv(Wo, kSfbTW);
  p.tiles_y = cdiv(Ho, kSfbTH);
  if (!grid_ok((long long)planes * p.tiles_x * p.tiles_y)) return B200W_ESIZE;
  return 0;
}

template <class T>
inline void dt_clear(DtParamsT<T>& p) { memset(&p, 0, sizeof(p)); }

template <class T>
inline int build_fwd_j1(DtParamsT<T>& p, const T* x, long long xps, int xpitch, T* ll, long long llps,
                        int llpitch, T* highs, const long long hs[6], int N, int C, int H, int W,
                        const T* h0, int L0, const T* h1, int L1, int mode) {
  dt_clear(p);
  if (!x || !ll) return B200W_EARG;
  if (highs && !hs) return B200W_EARG;
  if (N < 0 || C < 1 || H < 2 || W < 2 || (H & 1) || (W & 1)) return B200W_ESIZE;
  if (!(L0 & 1) || !(L1 & 1)) return B200W_EFILTER;  // even-length level-1 filters change the output size (+1)
  int rc;
  if ((rc = set_taps(p.f0, h0, L0)) || (rc = set_taps(p.f1, h1, L1))) return rc;
  if (xpitch < W || llpitch < W) return B200W_EARG;
  p.in = x; p.inps = xps; p.inpitch = xpitch;
  p.out = ll; p.outps = llps; p.outpitch = llpitch;
  p.highs = highs;
  if (highs) for (int i = 0; i < 6; ++i) p.hs[i] = hs[i];
  p.N = N; p.C = C; p.H = H; p.W = W; p.L0 = L0; p.L1 = L1;
  p.sym = (mode == B200W_MODE_SYMMETRIC);
  p.tiles_x = cdiv(W, kJ1TW);
  p.tiles_y = cdiv(H, kJ1TH);
  if (!grid_ok((long long)N * C * p.tiles_x * p.tiles_y)) return B200W_ESIZE;
  return 0;
}

template <class T>
inline int build_scat_j1(DtParamsT<T>& p, const T* x, T* z, T* dre, T* dim, int N, int C, int H,
                         int W, const T* h0, int L0, const T* h1, int L1, int mode, T magbias) {
  dt_clear(p);
  if (!x || !z) return B200W_EARG;
  if ((dre == nullptr) != (dim == nullptr)) return B200W_EARG;
  if (N < 0 || C < 1 || H < 2 || W < 2 || (H & 1) || (W & 1)) return B200W_ESIZE;
  if (!(L0 & 1) || !(L1 & 1)) return B200W_EFILTER;
  int rc;
  if ((rc = set_taps(p.f0, h0, L0)) || (rc = set_taps(p.f1, h1, L1))) return rc;
  p.in = x; p.inps = (long long)H * W; p.inpitch = W;
  p.z = z; p.dre = dre; p.dim = dim;
  p.N = N; p.C = C; p.H = H; p.W = W; p.L0 = L0; p.L1 = L1;
  p.sym = (mode == B200W_MODE_SYMMETRIC);
  p.magbias = magbias;
  p.magbias2 = (T)((double)magbias * (double)magbias);
  p.tiles_x = cdiv(W, kJ1TW);
  p.tiles_y = cdiv(H, kJ1TH);
  if (!grid_ok((long long)N * C * p.tiles_x * p.tiles_y)) return B200W_ESIZE;
  return 0;
}

template <class T>
inline int build_fwd_j2plus(DtParamsT<T>& p, const T* x, long long xps, int xpitch, T* ll, long long llps,
                            int llpitch, T* highs, const long long hs[6], int N, int C, int H, int W,
                            const T* h0a, const T* h1a, const T* h0b, const T* h1b, int m) {
  dt_clear(p);
  if (!x || !ll) return B200W_EARG;
  if (highs && !hs) return B200W_EARG;
  if (N < 0 || C < 1 || H < 4 || W < 4 || (H % 4) || (W % 4)) return B200W_ESIZE;  // reference ValueError
  if (m < 2 || (m & 1)) return B200W_EFILTER;
  int rc;
  if ((rc = set_taps(p.f0, h0a, m)) || (rc = set_taps(p.f1, h1a, m)) || (rc = set_taps(p.f2, h0b, m)) ||
      (rc = set_taps(p.f3, h1b, m)))
    return rc;
  for (int i = 0; i < kMaxTaps; ++i) {
    p.qlo[2 * i] = p.f2.t[i]; p.qlo[2 * i + 1] = p.f0.t[i];
    p.qhi[2 * i] = p.f3.t[i]; p.qhi[2 * i + 1] = p.f1.t[i];
  }
  if (xpitch < W || llpitch < W / 2) return B200W_EARG;
  p.in = x; p.inps = xps; p.inpitch = xpitch;
  p.out = ll; p.outps = llps; p.outpitch = llpitch;
  p.highs = highs;
  if (highs) for (int i = 0; i < 6; ++i) p.hs[i] = hs[i];
  p.N = N; p.C = C; p.H = H; p.W = W; p.L0 = m; p.L1 = m; p.sym = 1;
  p.tiles_x = cdiv(W / 2, kJ2TW);
  p.tiles_y = cdiv(H / 2, kJ2TH);
  if (!grid_ok((long long)N * C * p.tiles_x * p.tiles_y)) return B200W_ESIZE;
  return 0;
}

template <class T>
inline int build_inv_j1(DtParamsT<T>& p, const T* ll, long long llps, int llpitch, const T* highs,
                        const long long hs[6], T* y, long long yps, int ypitch, int N, int C, int H, int W,
                        const T* g0, int L0, const T* g1, int L1, int mode) {
  dt_clear(p);
  if (!y || (!ll && !highs)) return B200W_EARG;
  if (highs && !hs) return B200W_EARG;
  if (N < 0 || C < 1 || H < 2 || W < 2 || (H & 1) || (W & 1)) return B200W_ESIZE;
  if (!(L0 & 1) || !(L1 & 1)) return B200W_EFILTER;
  int rc;
  if ((rc = set_taps(p.f0, g0, L0)) || (rc = set_taps(p.f1, g1, L1))) return rc;
  if ((ll && llpitch < W) || ypitch < W) return B200W_EARG;
  p.in = ll; p.inps = llps; p.inpitch = llpitch;
  p.out = y; p.outps = yps; p.outpitch = ypitch;
  p.highs = const_cast<T*>(highs);
  if (highs) for (int i = 0; i < 6; ++i) p.hs[i] = hs[i];
  p.N = N; p.C = C; p.H = H; p.W = W; p.L0 = L0; p.L1 = L1;
  p.sym = (mode == B200W_MODE_SYMMETRIC);
  p.tiles_x = cdiv(W, kI1TW);
  p.tiles_y = cdiv(H, kI1TH);
  if (!grid_ok((long long)N * C * p.tiles_x * p.tiles_y)) return B200W_ESIZE;
  return 0;
}

template <class T>
inline int build_inv_j2plus(DtParamsT<T>& p, const T* ll, long long llps, int llpitch, const T* highs,
                            const long long hs[6], T* y, long long yps, int ypitch, int N, int C, int H,
                            int W, const T* g0a, const T* g1a, const T* g0b, const T* g1b,
                            int m) {
  dt_clear(p);
  if (!y || (!ll && !highs)) return B200W_EARG;
  if (highs && !hs) return B200W_EARG;
  if (N < 0 || C < 1 || H < 2 || W < 2 || (H & 1) || (W & 1)) return B200W_ESIZE;  // reference ValueError
  if (m < 2 || (m & 1)) return B200W_EFILTER;
  int rc;
  if ((rc = set_taps(p.f0, g0a, m)) || (rc = set_taps(p.f1, g1a, m)) || (rc = set_taps(p.f2, g0b, m)) ||
      (rc = set_taps(p.f3, g1b, m)))
    return rc;
  if ((ll && llpitch < W) || ypitch < 2 * W) return B200W_EARG;
  p.in = ll; p.inps = llps; p.inpitch = llpitch;
  p.out = y; p.outps = yps; p.outpitch = ypitch;
  p.highs = const_cast<T*>(highs);
  if (highs) for (int i = 0; i < 6; ++i) p.hs[i] = hs[i];
  p.N = N; p.C = C; p.H = H; p.W = W; p.L0 = m; p.L1 = m; p.sym = 1;
  p.tiles_x = cdiv(2 * W, kI2TW);
  p.tiles_y = cdiv(2 * H, kI2TH);
  if (!grid_ok((long long)N * C * p.tiles_x * p.tiles_y)) return B200W_ESIZE;
  return 0;
}

}  // namespace b200w
