// b200wave.cu -- libb200wave.so: C ABI (include/b200wave.h) + CUDA launchers, sm_90a only.
//
// Build (see pytorch_wavelets_b200/_build.py): every .cu of this directory is compiled with
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -Xcompiler -fPIC -c
// in parallel and linked into libb200wave.so.  This unit holds the C ABI and the generic tile kernels in float and
// double; the float32 streaming kernels live in k_*.cu behind fast_api.h.  Double precision (the `_f64` entry points,
// for torch.float64 callers, as the reference computes in the default dtype) always runs the generic tile kernels:
// same source, index logic and accumulation order as float, IEEE double arithmetic.
#include <cuda_runtime.h>
#include <stdio.h>

#include <type_traits>

#include "launch_params.h"
#include "launch.cuh"
#include "fast_api.h"

namespace b200w {
constexpr int NT = 256;
// ---- __global__ wrappers of the generic tile bodies ---------------------------------------------
extern __shared__ __align__(16) unsigned char g_smem[];   // one byte array, cast to T* by every instantiation

template <class T> __global__ void __launch_bounds__(NT) k_afb2d_tile(const __grid_constant__ AfbParamsT<T> p) { afb2d_tile<NT>(p, blockIdx.x, reinterpret_cast<T*>(g_smem)); }
template <class T> __global__ void __launch_bounds__(NT) k_sfb2d_tile(const __grid_constant__ SfbParamsT<T> p) { sfb2d_tile<NT>(p, blockIdx.x, reinterpret_cast<T*>(g_smem)); }
template <class T> __global__ void __launch_bounds__(NT) k_fwd_j1_tile(const __grid_constant__ DtParamsT<T> p) { fwd_j1_tile<NT, false>(p, blockIdx.x, reinterpret_cast<T*>(g_smem)); }
template <class T> __global__ void __launch_bounds__(NT) k_scat_j1_tile(const __grid_constant__ DtParamsT<T> p) { fwd_j1_tile<NT, true>(p, blockIdx.x, reinterpret_cast<T*>(g_smem)); }
template <class T> __global__ void __launch_bounds__(NT) k_fwd_j2plus_tile(const __grid_constant__ DtParamsT<T> p) { fwd_j2plus_tile<NT>(p, blockIdx.x, reinterpret_cast<T*>(g_smem)); }
template <class T> __global__ void __launch_bounds__(NT) k_inv_j1_tile(const __grid_constant__ DtParamsT<T> p) { inv_j1_tile<NT>(p, blockIdx.x, reinterpret_cast<T*>(g_smem)); }
template <class T> __global__ void __launch_bounds__(NT) k_inv_j2plus_tile(const __grid_constant__ DtParamsT<T> p) { inv_j2plus_tile<NT>(p, blockIdx.x, reinterpret_cast<T*>(g_smem)); }

// the one buffer behind b200w_last_cuda_error(), written by every launch of the library (launch.cuh)
thread_local char g_last_cuda_error[256] = "";

int check_cuda(cudaError_t e) {
  if (e == cudaSuccess) return B200W_OK;
  snprintf(g_last_cuda_error, sizeof(g_last_cuda_error), "%s: %s", cudaGetErrorName(e), cudaGetErrorString(e));
  return B200W_ECUDA;
}

}  // namespace b200w

using namespace b200w;

namespace {

// One level of one transform: the float32 streaming kernel `try_fast` when it covers p (unless the caller asked for
// the generic kernel), else the generic tile kernel.  Double precision always runs the tile kernel.
template <class T, class P, class F, class K>
int run_level(const P& p, bool generic, F try_fast, K tile, long long blocks, int smem_elems, void* stream) {
  if constexpr (std::is_same_v<T, float>) {
    if (!generic) {
      const int rc = try_fast(p, (cudaStream_t)stream);
      if (rc != fast::kNoFastPath) return rc ? rc : check_launch();
    }
  }
  return launch(tile, p, blocks, NT, (size_t)smem_elems * sizeof(T), stream);
}

template <class T>
int dwt_afb2d_impl(const T* x, long long x_plane_stride, int x_pitch, T* ll, long long ll_plane_stride, int ll_pitch,
                   T* highs, int planes, int H, int W, const T* fw_lo, const T* fw_hi, int Lw, const T* fh_lo,
                   const T* fh_hi, int Lh, int mode, void* stream, bool generic) {
  AfbParamsT<T> p;
  const int rc = build_afb(p, x, x_plane_stride, x_pitch, ll, ll_plane_stride, ll_pitch, highs, planes, H, W, fw_lo,
                           fw_hi, Lw, fh_lo, fh_hi, Lh, mode);
  return rc ? rc : run_level<T>(p, generic, fast::try_launch_afb, k_afb2d_tile<T>,
                                (long long)planes * p.tiles_x * p.tiles_y, afb_smem_floats(Lw, Lh), stream);
}

template <class T>
int dwt_sfb2d_impl(const T* ll, long long ll_plane_stride, int ll_pitch, const T* highs, T* y, long long y_plane_stride,
                   int y_pitch, int planes, int Hc, int Wc, int Ho, int Wo, const T* gh_lo, const T* gh_hi, int Lh,
                   const T* gw_lo, const T* gw_hi, int Lw, int mode, void* stream, bool generic) {
  SfbParamsT<T> p;
  const int rc = build_sfb(p, ll, ll_plane_stride, ll_pitch, highs, y, y_plane_stride, y_pitch, planes, Hc, Wc, Ho, Wo,
                           gh_lo, gh_hi, Lh, gw_lo, gw_hi, Lw, mode);
  return rc ? rc : run_level<T>(p, generic, fast::try_launch_sfb, k_sfb2d_tile<T>,
                                (long long)planes * p.tiles_x * p.tiles_y, sfb_smem_floats(Lh, Lw), stream);
}

template <class T>
int dtcwt_fwd_j1_impl(const T* x, long long x_plane_stride, int x_pitch, T* ll, long long ll_plane_stride, int ll_pitch,
                      T* highs, const long long hs[6], int N, int C, int H, int W, const T* h0, int L0, const T* h1,
                      int L1, int mode, void* stream, bool generic) {
  DtParamsT<T> p;
  const int rc = build_fwd_j1(p, x, x_plane_stride, x_pitch, ll, ll_plane_stride, ll_pitch, highs, hs, N, C, H, W, h0,
                              L0, h1, L1, mode);
  return rc ? rc : run_level<T>(p, generic, fast::try_launch_fwd_j1, k_fwd_j1_tile<T>,
                                (long long)N * C * p.tiles_x * p.tiles_y, fwdj1_smem_floats(L0, L1), stream);
}

template <class T>
int dtcwt_fwd_j2plus_impl(const T* x, long long x_plane_stride, int x_pitch, T* ll, long long ll_plane_stride,
                          int ll_pitch, T* highs, const long long hs[6], int N, int C, int H, int W, const T* h0a,
                          const T* h1a, const T* h0b, const T* h1b, int m, void* stream, bool generic) {
  DtParamsT<T> p;
  const int rc = build_fwd_j2plus(p, x, x_plane_stride, x_pitch, ll, ll_plane_stride, ll_pitch, highs, hs, N, C, H, W,
                                  h0a, h1a, h0b, h1b, m);
  return rc ? rc : run_level<T>(p, generic, fast::try_launch_fwd_j2plus, k_fwd_j2plus_tile<T>,
                                (long long)N * C * p.tiles_x * p.tiles_y, fwdj2_smem_floats(m), stream);
}

template <class T>
int dtcwt_inv_j1_impl(const T* ll, long long ll_plane_stride, int ll_pitch, const T* highs, const long long hs[6], T* y,
                      long long y_plane_stride, int y_pitch, int N, int C, int H, int W, const T* g0, int L0,
                      const T* g1, int L1, int mode, void* stream, bool generic) {
  DtParamsT<T> p;
  const int rc = build_inv_j1(p, ll, ll_plane_stride, ll_pitch, highs, hs, y, y_plane_stride, y_pitch, N, C, H, W, g0,
                              L0, g1, L1, mode);
  return rc ? rc : run_level<T>(p, generic, fast::try_launch_inv_j1, k_inv_j1_tile<T>,
                                (long long)N * C * p.tiles_x * p.tiles_y, invj1_smem_floats(L0, L1), stream);
}

template <class T>
int dtcwt_inv_j2plus_impl(const T* ll, long long ll_plane_stride, int ll_pitch, const T* highs, const long long hs[6],
                          T* y, long long y_plane_stride, int y_pitch, int N, int C, int H, int W, const T* g0a,
                          const T* g1a, const T* g0b, const T* g1b, int m, void* stream, bool generic) {
  DtParamsT<T> p;
  const int rc = build_inv_j2plus(p, ll, ll_plane_stride, ll_pitch, highs, hs, y, y_plane_stride, y_pitch, N, C, H, W,
                                  g0a, g1a, g0b, g1b, m);
  return rc ? rc : run_level<T>(p, generic, fast::try_launch_inv_j2plus, k_inv_j2plus_tile<T>,
                                (long long)N * C * p.tiles_x * p.tiles_y, invj2_smem_floats(m), stream);
}

template <class T>
int scat_j1_impl(const T* x, T* z, T* dre_dr, T* dim_dr, int N, int C, int H, int W, const T* h0, int L0, const T* h1,
                 int L1, int mode, T magbias, void* stream, bool generic) {
  DtParamsT<T> p;
  const int rc = build_scat_j1(p, x, z, dre_dr, dim_dr, N, C, H, W, h0, L0, h1, L1, mode, magbias);
  return rc ? rc : run_level<T>(p, generic, fast::try_launch_scat_j1, k_scat_j1_tile<T>,
                                (long long)N * C * p.tiles_x * p.tiles_y, fwdj1_smem_floats(L0, L1), stream);
}

}  // namespace

extern "C" {

int b200w_version(void) { return B200W_VERSION; }

const char* b200w_strerror(int code) {
  switch (code) {
    case B200W_OK: return "ok";
    case B200W_EMODE: return "Unkown pad type";  // (sic) the reference's message, dwt/lowlevel.py:88
    case B200W_ESIZE: return "bad tensor size";
    case B200W_EARG: return "bad argument";
    case B200W_EFILTER: return "unsupported filter length";
    case B200W_ECUDA: return "CUDA error";
    case B200W_ENOTIMPL: return "not implemented";
    default: return "unknown error";
  }
}

const char* b200w_last_cuda_error(void) { return g_last_cuda_error; }

int b200w_dwt_coeff_len(int n, int flen, int mode) { return coeff_len(n, flen, mode); }
int b200w_dwt_rec_len(int k, int flen, int mode) { return rec_len(k, flen, mode); }

// ---- per-level entry points: float (streaming kernel when one applies), float generic, double ------------------

int b200w_dwt_afb2d(const float* x, long long x_plane_stride, int x_pitch, float* ll, long long ll_plane_stride,
                    int ll_pitch, float* highs, int planes, int H, int W, const float* fw_lo, const float* fw_hi,
                    int Lw, const float* fh_lo, const float* fh_hi, int Lh, int mode, void* stream) {
  return dwt_afb2d_impl<float>(x, x_plane_stride, x_pitch, ll, ll_plane_stride, ll_pitch, highs, planes, H, W, fw_lo, fw_hi, Lw, fh_lo, fh_hi, Lh, mode, stream, false);
}
int b200w_dwt_afb2d_generic(const float* x, long long x_plane_stride, int x_pitch, float* ll, long long ll_plane_stride,
                            int ll_pitch, float* highs, int planes, int H, int W, const float* fw_lo, const float* fw_hi,
                            int Lw, const float* fh_lo, const float* fh_hi, int Lh, int mode, void* stream) {
  return dwt_afb2d_impl<float>(x, x_plane_stride, x_pitch, ll, ll_plane_stride, ll_pitch, highs, planes, H, W, fw_lo, fw_hi, Lw, fh_lo, fh_hi, Lh, mode, stream, true);
}
int b200w_dwt_afb2d_f64(const double* x, long long x_plane_stride, int x_pitch, double* ll, long long ll_plane_stride,
                        int ll_pitch, double* highs, int planes, int H, int W, const double* fw_lo, const double* fw_hi,
                        int Lw, const double* fh_lo, const double* fh_hi, int Lh, int mode, void* stream) {
  return dwt_afb2d_impl<double>(x, x_plane_stride, x_pitch, ll, ll_plane_stride, ll_pitch, highs, planes, H, W, fw_lo, fw_hi, Lw, fh_lo, fh_hi, Lh, mode, stream, true);
}

int b200w_dwt_sfb2d(const float* ll, long long ll_plane_stride, int ll_pitch, const float* highs, float* y,
                    long long y_plane_stride, int y_pitch, int planes, int Hc, int Wc, int Ho, int Wo,
                    const float* gh_lo, const float* gh_hi, int Lh, const float* gw_lo, const float* gw_hi, int Lw,
                    int mode, void* stream) {
  return dwt_sfb2d_impl<float>(ll, ll_plane_stride, ll_pitch, highs, y, y_plane_stride, y_pitch, planes, Hc, Wc, Ho, Wo, gh_lo, gh_hi, Lh, gw_lo, gw_hi, Lw, mode, stream, false);
}
int b200w_dwt_sfb2d_generic(const float* ll, long long ll_plane_stride, int ll_pitch, const float* highs, float* y,
                            long long y_plane_stride, int y_pitch, int planes, int Hc, int Wc, int Ho, int Wo,
                            const float* gh_lo, const float* gh_hi, int Lh, const float* gw_lo, const float* gw_hi, int Lw,
                            int mode, void* stream) {
  return dwt_sfb2d_impl<float>(ll, ll_plane_stride, ll_pitch, highs, y, y_plane_stride, y_pitch, planes, Hc, Wc, Ho, Wo, gh_lo, gh_hi, Lh, gw_lo, gw_hi, Lw, mode, stream, true);
}
int b200w_dwt_sfb2d_f64(const double* ll, long long ll_plane_stride, int ll_pitch, const double* highs, double* y,
                        long long y_plane_stride, int y_pitch, int planes, int Hc, int Wc, int Ho, int Wo,
                        const double* gh_lo, const double* gh_hi, int Lh, const double* gw_lo, const double* gw_hi, int Lw,
                        int mode, void* stream) {
  return dwt_sfb2d_impl<double>(ll, ll_plane_stride, ll_pitch, highs, y, y_plane_stride, y_pitch, planes, Hc, Wc, Ho, Wo, gh_lo, gh_hi, Lh, gw_lo, gw_hi, Lw, mode, stream, true);
}

int b200w_dtcwt_fwd_j1(const float* x, long long x_plane_stride, int x_pitch, float* ll, long long ll_plane_stride,
                       int ll_pitch, float* highs, const long long hs[6], int N, int C, int H, int W,
                       const float* h0, int L0, const float* h1, int L1, int mode, void* stream) {
  return dtcwt_fwd_j1_impl<float>(x, x_plane_stride, x_pitch, ll, ll_plane_stride, ll_pitch, highs, hs, N, C, H, W, h0, L0, h1, L1, mode, stream, false);
}
int b200w_dtcwt_fwd_j1_generic(const float* x, long long x_plane_stride, int x_pitch, float* ll, long long ll_plane_stride,
                               int ll_pitch, float* highs, const long long hs[6], int N, int C, int H, int W,
                               const float* h0, int L0, const float* h1, int L1, int mode, void* stream) {
  return dtcwt_fwd_j1_impl<float>(x, x_plane_stride, x_pitch, ll, ll_plane_stride, ll_pitch, highs, hs, N, C, H, W, h0, L0, h1, L1, mode, stream, true);
}
int b200w_dtcwt_fwd_j1_f64(const double* x, long long x_plane_stride, int x_pitch, double* ll, long long ll_plane_stride,
                           int ll_pitch, double* highs, const long long hs[6], int N, int C, int H, int W,
                           const double* h0, int L0, const double* h1, int L1, int mode, void* stream) {
  return dtcwt_fwd_j1_impl<double>(x, x_plane_stride, x_pitch, ll, ll_plane_stride, ll_pitch, highs, hs, N, C, H, W, h0, L0, h1, L1, mode, stream, true);
}

int b200w_dtcwt_fwd_j2plus(const float* x, long long x_plane_stride, int x_pitch, float* ll,
                           long long ll_plane_stride, int ll_pitch, float* highs, const long long hs[6], int N,
                           int C, int H, int W, const float* h0a, const float* h1a, const float* h0b,
                           const float* h1b, int m, void* stream) {
  return dtcwt_fwd_j2plus_impl<float>(x, x_plane_stride, x_pitch, ll, ll_plane_stride, ll_pitch, highs, hs, N, C, H, W, h0a, h1a, h0b, h1b, m, stream, false);
}
int b200w_dtcwt_fwd_j2plus_generic(const float* x, long long x_plane_stride, int x_pitch, float* ll,
                                   long long ll_plane_stride, int ll_pitch, float* highs, const long long hs[6], int N,
                                   int C, int H, int W, const float* h0a, const float* h1a, const float* h0b,
                                   const float* h1b, int m, void* stream) {
  return dtcwt_fwd_j2plus_impl<float>(x, x_plane_stride, x_pitch, ll, ll_plane_stride, ll_pitch, highs, hs, N, C, H, W, h0a, h1a, h0b, h1b, m, stream, true);
}
int b200w_dtcwt_fwd_j2plus_f64(const double* x, long long x_plane_stride, int x_pitch, double* ll,
                               long long ll_plane_stride, int ll_pitch, double* highs, const long long hs[6], int N,
                               int C, int H, int W, const double* h0a, const double* h1a, const double* h0b,
                               const double* h1b, int m, void* stream) {
  return dtcwt_fwd_j2plus_impl<double>(x, x_plane_stride, x_pitch, ll, ll_plane_stride, ll_pitch, highs, hs, N, C, H, W, h0a, h1a, h0b, h1b, m, stream, true);
}

int b200w_dtcwt_inv_j1(const float* ll, long long ll_plane_stride, int ll_pitch, const float* highs,
                       const long long hs[6], float* y, long long y_plane_stride, int y_pitch, int N, int C, int H,
                       int W, const float* g0, int L0, const float* g1, int L1, int mode, void* stream) {
  return dtcwt_inv_j1_impl<float>(ll, ll_plane_stride, ll_pitch, highs, hs, y, y_plane_stride, y_pitch, N, C, H, W, g0, L0, g1, L1, mode, stream, false);
}
int b200w_dtcwt_inv_j1_generic(const float* ll, long long ll_plane_stride, int ll_pitch, const float* highs,
                               const long long hs[6], float* y, long long y_plane_stride, int y_pitch, int N, int C, int H,
                               int W, const float* g0, int L0, const float* g1, int L1, int mode, void* stream) {
  return dtcwt_inv_j1_impl<float>(ll, ll_plane_stride, ll_pitch, highs, hs, y, y_plane_stride, y_pitch, N, C, H, W, g0, L0, g1, L1, mode, stream, true);
}
int b200w_dtcwt_inv_j1_f64(const double* ll, long long ll_plane_stride, int ll_pitch, const double* highs,
                           const long long hs[6], double* y, long long y_plane_stride, int y_pitch, int N, int C, int H,
                           int W, const double* g0, int L0, const double* g1, int L1, int mode, void* stream) {
  return dtcwt_inv_j1_impl<double>(ll, ll_plane_stride, ll_pitch, highs, hs, y, y_plane_stride, y_pitch, N, C, H, W, g0, L0, g1, L1, mode, stream, true);
}

int b200w_dtcwt_inv_j2plus(const float* ll, long long ll_plane_stride, int ll_pitch, const float* highs,
                           const long long hs[6], float* y, long long y_plane_stride, int y_pitch, int N, int C,
                           int H, int W, const float* g0a, const float* g1a, const float* g0b, const float* g1b,
                           int m, void* stream) {
  return dtcwt_inv_j2plus_impl<float>(ll, ll_plane_stride, ll_pitch, highs, hs, y, y_plane_stride, y_pitch, N, C, H, W, g0a, g1a, g0b, g1b, m, stream, false);
}
int b200w_dtcwt_inv_j2plus_generic(const float* ll, long long ll_plane_stride, int ll_pitch, const float* highs,
                                   const long long hs[6], float* y, long long y_plane_stride, int y_pitch, int N, int C,
                                   int H, int W, const float* g0a, const float* g1a, const float* g0b, const float* g1b,
                                   int m, void* stream) {
  return dtcwt_inv_j2plus_impl<float>(ll, ll_plane_stride, ll_pitch, highs, hs, y, y_plane_stride, y_pitch, N, C, H, W, g0a, g1a, g0b, g1b, m, stream, true);
}
int b200w_dtcwt_inv_j2plus_f64(const double* ll, long long ll_plane_stride, int ll_pitch, const double* highs,
                               const long long hs[6], double* y, long long y_plane_stride, int y_pitch, int N, int C,
                               int H, int W, const double* g0a, const double* g1a, const double* g0b, const double* g1b,
                               int m, void* stream) {
  return dtcwt_inv_j2plus_impl<double>(ll, ll_plane_stride, ll_pitch, highs, hs, y, y_plane_stride, y_pitch, N, C, H, W, g0a, g1a, g0b, g1b, m, stream, true);
}

int b200w_scat_j1(const float* x, float* z, float* dre_dr, float* dim_dr, int N, int C, int H, int W,
                  const float* h0, int L0, const float* h1, int L1, int mode, float magbias, void* stream) {
  return scat_j1_impl<float>(x, z, dre_dr, dim_dr, N, C, H, W, h0, L0, h1, L1, mode, magbias, stream, false);
}
int b200w_scat_j1_generic(const float* x, float* z, float* dre_dr, float* dim_dr, int N, int C, int H, int W,
                          const float* h0, int L0, const float* h1, int L1, int mode, float magbias, void* stream) {
  return scat_j1_impl<float>(x, z, dre_dr, dim_dr, N, C, H, W, h0, L0, h1, L1, mode, magbias, stream, true);
}
int b200w_scat_j1_f64(const double* x, double* z, double* dre_dr, double* dim_dr, int N, int C, int H, int W,
                      const double* h0, int L0, const double* h1, int L1, int mode, double magbias, void* stream) {
  return scat_j1_impl<double>(x, z, dre_dr, dim_dr, N, C, H, W, h0, L0, h1, L1, mode, magbias, stream, true);
}

/* ---- whole-transform entry point: all J analysis levels of DWTForward.forward (reference dwt/transform2d.py:68-74) */

static long long align256(long long n) { return (n + 255) / 256 * 256; }

// intermediate low-pass buffers of the level-by-level path: level j writes buffer j % 2 with a 128-byte row pitch
static void dwt_ws_layout(int planes, int H, int W, int J, int Lw, int Lh, int mode, long long bytes[2]) {
  bytes[0] = bytes[1] = 0;
  int h = H, w = W;
  for (int j = 0; j + 1 < J; ++j) {
    h = coeff_len(h, Lh, mode); w = coeff_len(w, Lw, mode);
    if (h < 1 || w < 1) break;
    const long long need = align256(4LL * planes * h * ((w + 31) / 32 * 32));
    if (need > bytes[j & 1]) bytes[j & 1] = need;
  }
}

// How the levels of one DWTForward call are executed (one policy, decided from the arguments alone):
//   kPyramidAll   all J levels in the fused pyramid kernel (one launch, no inter-level low-pass in device memory)
//   kPyramidFirst level 1 in the pyramid kernel (TMA loads, bulk stores, writes the padded low-pass into the
//                 workspace), deeper levels one streaming kernel each
//   kLevels       one K1 launch per level
// Why (tools/policy_probe.py, J = 2 / 3 db4 symmetric, 268 Mpix per call, on an H100 80GB HBM3): below 512 columns a
// multi-level CTA is register / shared-memory bound to 2 per SM, which costs more than the hand-off traffic it saves
// (256^2, J = 3: 1.64 ms fused vs 1.52 ms level 1 fused + streaming levels); from 512 columns up the single launch wins
// (512^2: 0.99 vs 1.39 ms; 1024^2: 0.88 vs 1.21 ms).
enum DwtPolicy { kLevels = 0, kPyramidFirst = 1, kPyramidAll = 2 };

#ifndef B200W_PYR_FUSE_ALL_MIN_WIDTH
#define B200W_PYR_FUSE_ALL_MIN_WIDTH 512    /* planes at least this wide run every level in the pyramid kernel */
#endif

static DwtPolicy dwt_policy(PyrParams& pp, const float* x, long long xps, int xpitch, int planes, int H, int W, int J,
                            int Lw, int Lh, int mode, bool generic) {
  if (generic || Lw != Lh) return kLevels;
  const bool wide = (W >= B200W_PYR_FUSE_ALL_MIN_WIDTH);
  if ((J == 1 || wide) && fast::plan_dwt_pyramid(pp, x, xps, xpitch, planes, H, W, J, Lw, mode, 0) == 0)
    return kPyramidAll;
  if (J >= 2) {
    const int wo = coeff_len(W, Lw, mode);
    if (wo > 0 && fast::plan_dwt_pyramid(pp, x, xps, xpitch, planes, H, W, 1, Lw, mode, (wo + 31) / 32 * 32) == 0)
      return kPyramidFirst;
  }
  return kLevels;
}

long long b200w_dwt_forward_workspace(const float* x, long long x_plane_stride, int x_pitch, int planes, int H, int W,
                                      int J, int Lw, int Lh, int mode) {
  if (!dwt_mode_ok(mode)) return B200W_EMODE;
  if (planes < 0 || H < 1 || W < 1 || J < 1) return B200W_ESIZE;
  if (Lw < 2 || Lh < 2 || Lw > kMaxTaps || Lh > kMaxTaps) return B200W_EFILTER;
  PyrParams pp;
  if (dwt_policy(pp, x, x_plane_stride, x_pitch, planes, H, W, J, Lw, Lh, mode, false) == kPyramidAll) return 0;
  long long b[2];
  dwt_ws_layout(planes, H, W, J, Lw, Lh, mode, b);
  return b[0] + b[1];
}

static void pyr_set_taps(PyrParams& pp, const float* fw_lo, const float* fw_hi, const float* fh_lo, const float* fh_hi,
                         int L) {
  for (int i = 0; i < kPyrMaxTaps; ++i) {
    const bool on = i < L;
    pp.fw[2 * i] = on ? fw_lo[i] : 0.f; pp.fw[2 * i + 1] = on ? fw_hi[i] : 0.f;
    pp.fh_lo[i] = on ? fh_lo[i] : 0.f; pp.fh_hi[i] = on ? fh_hi[i] : 0.f;
  }
}

static int dwt_forward_impl(const float* x, long long x_plane_stride, int x_pitch, int planes, int H, int W, int J,
                            float* yl, float* const* highs, const float* fw_lo, const float* fw_hi, int Lw,
                            const float* fh_lo, const float* fh_hi, int Lh, int mode, void* workspace,
                            long long workspace_bytes, void* stream, bool generic) {
  if (!dwt_mode_ok(mode)) return B200W_EMODE;
  if (!x || !yl || !highs || !fw_lo || !fw_hi || !fh_lo || !fh_hi) return B200W_EARG;
  if (planes < 0 || H < 1 || W < 1 || J < 1) return B200W_ESIZE;
  if (Lw < 2 || Lh < 2) return B200W_EFILTER;
  for (int j = 0; j < J; ++j)
    if (!highs[j]) return B200W_EARG;
  PyrParams pp;
  DwtPolicy pol = dwt_policy(pp, x, x_plane_stride, x_pitch, planes, H, W, J, Lw, Lh, mode, generic);
  if (pol == kPyramidAll) {
    pyr_set_taps(pp, fw_lo, fw_hi, fh_lo, fh_hi, Lw);
    pp.yl = yl;
    for (int j = 0; j < kPyrMaxLevels; ++j) pp.highs[j] = (j < J) ? highs[j] : nullptr;
    const int rc = fast::launch_dwt_pyramid(pp, (cudaStream_t)stream);
    if (rc != fast::kNoFastPath) return rc ? rc : check_launch();
    pol = kLevels;
  }
  long long wb[2];
  dwt_ws_layout(planes, H, W, J, Lw, Lh, mode, wb);
  if (wb[0] + wb[1] > 0 && (!workspace || workspace_bytes < wb[0] + wb[1])) return B200W_EARG;
  float* buf[2] = {static_cast<float*>(workspace), reinterpret_cast<float*>(static_cast<char*>(workspace) + wb[0])};
  const float* src = x;
  long long sps = x_plane_stride;
  int spitch = x_pitch, h = H, w = W;
  for (int j = 0; j < J; ++j) {
    const int ho = coeff_len(h, Lh, mode), wo = coeff_len(w, Lw, mode);
    if (ho < 1 || wo < 1) return B200W_ESIZE;
    const bool last = (j == J - 1);
    const int wp = last ? wo : (wo + 31) / 32 * 32;
    float* ll = last ? yl : buf[j & 1];
    int rc = fast::kNoFastPath;
    if (j == 0 && pol == kPyramidFirst) {   // (J >= 2, so ll is the padded workspace buffer the plan was made for)
      pyr_set_taps(pp, fw_lo, fw_hi, fh_lo, fh_hi, Lw);
      pp.yl = ll;
      for (int i = 0; i < kPyrMaxLevels; ++i) pp.highs[i] = (i == 0) ? highs[0] : nullptr;
      rc = fast::launch_dwt_pyramid(pp, (cudaStream_t)stream);
      if (rc == 0) rc = check_launch();
    }
    if (rc == fast::kNoFastPath)
      rc = dwt_afb2d_impl<float>(src, sps, spitch, ll, (long long)ho * wp, wp, highs[j], planes, h, w, fw_lo, fw_hi, Lw, fh_lo,
                          fh_hi, Lh, mode, stream, generic);
    if (rc) return rc;
    src = ll; sps = (long long)ho * wp; spitch = wp; h = ho; w = wo;
  }
  return B200W_OK;
}

int b200w_dwt_forward(const float* x, long long x_plane_stride, int x_pitch, int planes, int H, int W, int J, float* yl,
                      float* const* highs, const float* fw_lo, const float* fw_hi, int Lw, const float* fh_lo,
                      const float* fh_hi, int Lh, int mode, void* workspace, long long workspace_bytes, void* stream) {
  return dwt_forward_impl(x, x_plane_stride, x_pitch, planes, H, W, J, yl, highs, fw_lo, fw_hi, Lw, fh_lo, fh_hi, Lh,
                          mode, workspace, workspace_bytes, stream, false);
}
int b200w_dwt_forward_generic(const float* x, long long x_plane_stride, int x_pitch, int planes, int H, int W, int J,
                              float* yl, float* const* highs, const float* fw_lo, const float* fw_hi, int Lw,
                              const float* fh_lo, const float* fh_hi, int Lh, int mode, void* workspace,
                              long long workspace_bytes, void* stream) {
  return dwt_forward_impl(x, x_plane_stride, x_pitch, planes, H, W, J, yl, highs, fw_lo, fw_hi, Lw, fh_lo, fh_hi, Lh,
                          mode, workspace, workspace_bytes, stream, true);
}

}  // extern "C"
