// emu.cpp -- host emulation of the generic tile kernels (TEST ONLY).
//
// Compiles pytorch_wavelets_b200/csrc/tile_kernels.h + launch_params.h with g++: every CTA is run
// as a loop over its threads, phase by phase (B200W_FOR_THREADS / B200W_SYNC), on host buffers.
// This checks the index arithmetic, tiling, boundary handling and argument validation of the
// shipped kernel source against the oracle on a machine without a GPU.  It is never loaded by the
// package; the product path is libb200wave.so (CUDA) only.
#include <stdlib.h>

#include <vector>

#include "../../pytorch_wavelets_b200/csrc/launch_params.h"
#include "../../pytorch_wavelets_b200/csrc/pyramid_plan.h"

using namespace b200w;

namespace {
constexpr int NT = 256;

template <class T, class P, class F>
void run_blocks(const P& p, long long blocks, int smem_elems, F body) {
#pragma omp parallel
  {
    std::vector<T> smem((size_t)smem_elems + 64, T(0));
#pragma omp for schedule(static)
    for (long long b = 0; b < blocks; ++b) body(p, (int)b, smem.data());
  }
}

template <class T>
int dwt_afb2d(const T* x, long long xps, int xpitch, T* ll, long long llps, int llpitch,
              T* highs, int planes, int H, int W, const T* fw_lo, const T* fw_hi, int Lw,
              const T* fh_lo, const T* fh_hi, int Lh, int mode) {
  AfbParamsT<T> p;
  int rc = build_afb(p, x, xps, xpitch, ll, llps, llpitch, highs, planes, H, W, fw_lo, fw_hi, Lw, fh_lo, fh_hi, Lh, mode);
  if (rc) return rc;
  run_blocks<T>(p, (long long)planes * p.tiles_x * p.tiles_y, afb_smem_floats(Lw, Lh),
                [](const AfbParamsT<T>& q, int b, T* s) { afb2d_tile<NT>(q, b, s); });
  return 0;
}

template <class T>
int dwt_sfb2d(const T* ll, long long llps, int llpitch, const T* highs, T* y, long long yps,
              int ypitch, int planes, int Hc, int Wc, int Ho, int Wo, const T* gh_lo,
              const T* gh_hi, int Lh, const T* gw_lo, const T* gw_hi, int Lw, int mode) {
  SfbParamsT<T> p;
  int rc = build_sfb(p, ll, llps, llpitch, highs, y, yps, ypitch, planes, Hc, Wc, Ho, Wo, gh_lo, gh_hi, Lh, gw_lo, gw_hi, Lw, mode);
  if (rc) return rc;
  run_blocks<T>(p, (long long)planes * p.tiles_x * p.tiles_y, sfb_smem_floats(Lh, Lw),
                [](const SfbParamsT<T>& q, int b, T* s) { sfb2d_tile<NT>(q, b, s); });
  return 0;
}

template <class T>
int dtcwt_fwd_j1(const T* x, long long xps, int xpitch, T* ll, long long llps, int llpitch,
                 T* highs, const long long hs[6], int N, int C, int H, int W, const T* h0, int L0,
                 const T* h1, int L1, int mode) {
  DtParamsT<T> p;
  int rc = build_fwd_j1(p, x, xps, xpitch, ll, llps, llpitch, highs, hs, N, C, H, W, h0, L0, h1, L1, mode);
  if (rc) return rc;
  run_blocks<T>(p, (long long)N * C * p.tiles_x * p.tiles_y, fwdj1_smem_floats(L0, L1),
                [](const DtParamsT<T>& q, int b, T* s) { fwd_j1_tile<NT, false>(q, b, s); });
  return 0;
}

template <class T>
int scat_j1(const T* x, T* z, T* dre, T* dim, int N, int C, int H, int W, const T* h0,
            int L0, const T* h1, int L1, int mode, T magbias) {
  DtParamsT<T> p;
  int rc = build_scat_j1(p, x, z, dre, dim, N, C, H, W, h0, L0, h1, L1, mode, magbias);
  if (rc) return rc;
  run_blocks<T>(p, (long long)N * C * p.tiles_x * p.tiles_y, fwdj1_smem_floats(L0, L1),
                [](const DtParamsT<T>& q, int b, T* s) { fwd_j1_tile<NT, true>(q, b, s); });
  return 0;
}

template <class T>
int dtcwt_fwd_j2plus(const T* x, long long xps, int xpitch, T* ll, long long llps, int llpitch,
                     T* highs, const long long hs[6], int N, int C, int H, int W, const T* h0a,
                     const T* h1a, const T* h0b, const T* h1b, int m) {
  DtParamsT<T> p;
  int rc = build_fwd_j2plus(p, x, xps, xpitch, ll, llps, llpitch, highs, hs, N, C, H, W, h0a, h1a, h0b, h1b, m);
  if (rc) return rc;
  run_blocks<T>(p, (long long)N * C * p.tiles_x * p.tiles_y, fwdj2_smem_floats(m),
                [](const DtParamsT<T>& q, int b, T* s) { fwd_j2plus_tile<NT>(q, b, s); });
  return 0;
}

template <class T>
int dtcwt_inv_j1(const T* ll, long long llps, int llpitch, const T* highs, const long long hs[6],
                 T* y, long long yps, int ypitch, int N, int C, int H, int W, const T* g0, int L0,
                 const T* g1, int L1, int mode) {
  DtParamsT<T> p;
  int rc = build_inv_j1(p, ll, llps, llpitch, highs, hs, y, yps, ypitch, N, C, H, W, g0, L0, g1, L1, mode);
  if (rc) return rc;
  run_blocks<T>(p, (long long)N * C * p.tiles_x * p.tiles_y, invj1_smem_floats(L0, L1),
                [](const DtParamsT<T>& q, int b, T* s) { inv_j1_tile<NT>(q, b, s); });
  return 0;
}

template <class T>
int dtcwt_inv_j2plus(const T* ll, long long llps, int llpitch, const T* highs, const long long hs[6],
                     T* y, long long yps, int ypitch, int N, int C, int H, int W, const T* g0a,
                     const T* g1a, const T* g0b, const T* g1b, int m) {
  DtParamsT<T> p;
  int rc = build_inv_j2plus(p, ll, llps, llpitch, highs, hs, y, yps, ypitch, N, C, H, W, g0a, g1a, g0b, g1b, m);
  if (rc) return rc;
  run_blocks<T>(p, (long long)N * C * p.tiles_x * p.tiles_y, invj2_smem_floats(m),
                [](const DtParamsT<T>& q, int b, T* s) { inv_j2plus_tile<NT>(q, b, s); });
  return 0;
}
}  // namespace

extern "C" {

// float32 entry points under the names of the C ABI, double precision with the `_f64` suffix
int emu_dwt_afb2d(const float* x, long long xps, int xpitch, float* ll, long long llps, int llpitch,
                  float* highs, int planes, int H, int W, const float* fw_lo, const float* fw_hi, int Lw,
                  const float* fh_lo, const float* fh_hi, int Lh, int mode) {
  return dwt_afb2d<float>(x, xps, xpitch, ll, llps, llpitch, highs, planes, H, W, fw_lo, fw_hi, Lw, fh_lo, fh_hi, Lh, mode);
}
int emu_dwt_afb2d_f64(const double* x, long long xps, int xpitch, double* ll, long long llps, int llpitch,
                      double* highs, int planes, int H, int W, const double* fw_lo, const double* fw_hi, int Lw,
                      const double* fh_lo, const double* fh_hi, int Lh, int mode) {
  return dwt_afb2d<double>(x, xps, xpitch, ll, llps, llpitch, highs, planes, H, W, fw_lo, fw_hi, Lw, fh_lo, fh_hi, Lh, mode);
}
int emu_dwt_sfb2d(const float* ll, long long llps, int llpitch, const float* highs, float* y, long long yps,
                  int ypitch, int planes, int Hc, int Wc, int Ho, int Wo, const float* gh_lo,
                  const float* gh_hi, int Lh, const float* gw_lo, const float* gw_hi, int Lw, int mode) {
  return dwt_sfb2d<float>(ll, llps, llpitch, highs, y, yps, ypitch, planes, Hc, Wc, Ho, Wo, gh_lo, gh_hi, Lh, gw_lo, gw_hi, Lw, mode);
}
int emu_dwt_sfb2d_f64(const double* ll, long long llps, int llpitch, const double* highs, double* y, long long yps,
                      int ypitch, int planes, int Hc, int Wc, int Ho, int Wo, const double* gh_lo,
                      const double* gh_hi, int Lh, const double* gw_lo, const double* gw_hi, int Lw, int mode) {
  return dwt_sfb2d<double>(ll, llps, llpitch, highs, y, yps, ypitch, planes, Hc, Wc, Ho, Wo, gh_lo, gh_hi, Lh, gw_lo, gw_hi, Lw, mode);
}
int emu_dtcwt_fwd_j1(const float* x, long long xps, int xpitch, float* ll, long long llps, int llpitch,
                     float* highs, const long long hs[6], int N, int C, int H, int W, const float* h0, int L0,
                     const float* h1, int L1, int mode) {
  return dtcwt_fwd_j1<float>(x, xps, xpitch, ll, llps, llpitch, highs, hs, N, C, H, W, h0, L0, h1, L1, mode);
}
int emu_dtcwt_fwd_j1_f64(const double* x, long long xps, int xpitch, double* ll, long long llps, int llpitch,
                         double* highs, const long long hs[6], int N, int C, int H, int W, const double* h0, int L0,
                         const double* h1, int L1, int mode) {
  return dtcwt_fwd_j1<double>(x, xps, xpitch, ll, llps, llpitch, highs, hs, N, C, H, W, h0, L0, h1, L1, mode);
}
int emu_scat_j1(const float* x, float* z, float* dre, float* dim, int N, int C, int H, int W, const float* h0,
                int L0, const float* h1, int L1, int mode, float magbias) {
  return scat_j1<float>(x, z, dre, dim, N, C, H, W, h0, L0, h1, L1, mode, magbias);
}
int emu_scat_j1_f64(const double* x, double* z, double* dre, double* dim, int N, int C, int H, int W, const double* h0,
                    int L0, const double* h1, int L1, int mode, double magbias) {
  return scat_j1<double>(x, z, dre, dim, N, C, H, W, h0, L0, h1, L1, mode, magbias);
}
int emu_dtcwt_fwd_j2plus(const float* x, long long xps, int xpitch, float* ll, long long llps, int llpitch,
                         float* highs, const long long hs[6], int N, int C, int H, int W, const float* h0a,
                         const float* h1a, const float* h0b, const float* h1b, int m) {
  return dtcwt_fwd_j2plus<float>(x, xps, xpitch, ll, llps, llpitch, highs, hs, N, C, H, W, h0a, h1a, h0b, h1b, m);
}
int emu_dtcwt_fwd_j2plus_f64(const double* x, long long xps, int xpitch, double* ll, long long llps, int llpitch,
                             double* highs, const long long hs[6], int N, int C, int H, int W, const double* h0a,
                             const double* h1a, const double* h0b, const double* h1b, int m) {
  return dtcwt_fwd_j2plus<double>(x, xps, xpitch, ll, llps, llpitch, highs, hs, N, C, H, W, h0a, h1a, h0b, h1b, m);
}
int emu_dtcwt_inv_j1(const float* ll, long long llps, int llpitch, const float* highs, const long long hs[6],
                     float* y, long long yps, int ypitch, int N, int C, int H, int W, const float* g0, int L0,
                     const float* g1, int L1, int mode) {
  return dtcwt_inv_j1<float>(ll, llps, llpitch, highs, hs, y, yps, ypitch, N, C, H, W, g0, L0, g1, L1, mode);
}
int emu_dtcwt_inv_j1_f64(const double* ll, long long llps, int llpitch, const double* highs, const long long hs[6],
                         double* y, long long yps, int ypitch, int N, int C, int H, int W, const double* g0, int L0,
                         const double* g1, int L1, int mode) {
  return dtcwt_inv_j1<double>(ll, llps, llpitch, highs, hs, y, yps, ypitch, N, C, H, W, g0, L0, g1, L1, mode);
}
int emu_dtcwt_inv_j2plus(const float* ll, long long llps, int llpitch, const float* highs, const long long hs[6],
                         float* y, long long yps, int ypitch, int N, int C, int H, int W, const float* g0a,
                         const float* g1a, const float* g0b, const float* g1b, int m) {
  return dtcwt_inv_j2plus<float>(ll, llps, llpitch, highs, hs, y, yps, ypitch, N, C, H, W, g0a, g1a, g0b, g1b, m);
}
int emu_dtcwt_inv_j2plus_f64(const double* ll, long long llps, int llpitch, const double* highs, const long long hs[6],
                             double* y, long long yps, int ypitch, int N, int C, int H, int W, const double* g0a,
                             const double* g1a, const double* g0b, const double* g1b, int m) {
  return dtcwt_inv_j2plus<double>(ll, llps, llpitch, highs, hs, y, yps, ypitch, N, C, H, W, g0a, g1a, g0b, g1b, m);
}

// The shipped host-side plan of the fused pyramid kernel (pyramid_plan.h), flattened for the CPU tests:
// out = {rc, smem_bytes, threads, n_bars, zero_off, then per level: H, W, Ho, Wo, n_stage, warp0, nwarps, in_off,
//        in_pitch, in_rows, n_in, bar_in, st_off, st_cap, nbands, bar_out}
int emu_plan_pyramid(int planes, int H, int W, int J, int L, int mode, int xpitch, int max_smem, int ll_pitch, int* out) {
  PyrParams p;
  memset(&p, 0, sizeof(p));
  alignas(16) static float dummy[4];
  const int rc = plan_pyramid_best(p, planes, H, W, J, L, mode, (long long)H * xpitch, xpitch, dummy, max_smem, 228 * 1024, ll_pitch);
  out[0] = rc; out[1] = p.smem_bytes; out[2] = p.threads; out[3] = p.n_bars; out[4] = p.zero_off;
  out[5 + 16 * 4] = p.nslot; out[6 + 16 * 4] = p.split; out[7 + 16 * 4] = p.ll_pitch;
  if (rc) return rc;
  for (int l = 0; l < J; ++l) {
    const PyrLevel& v = p.lv[l];
    const int f[16] = {v.H, v.W, v.Ho, v.Wo, v.n_stage, v.warp0, v.nwarps, v.in_off, v.in_pitch, v.in_rows, v.n_in,
                       v.bar_in, v.st_off, v.st_cap, v.nbands, v.bar_out};
    for (int i = 0; i < 16; ++i) out[5 + 16 * l + i] = f[i];
  }
  return 0;
}

}  // extern "C"
