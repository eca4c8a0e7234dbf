// common.h -- shared host/device definitions for libb200wave (sm_90a).
//
// The kernel bodies in tile_kernels.h are templates on the element type T (float or double), written once and
// compiled twice:
//   * by nvcc for sm_90a (the product: b200wave.cu and dwt1d.cu instantiate them for float and double), and
//   * by g++ as a block/thread-loop emulation (tests/emu/, CPU tests of the index logic and arithmetic).
// B200W_FOR_THREADS / B200W_SYNC express "every thread of the CTA runs this phase, then barrier".
#pragma once
#include <math.h>
#include <stdint.h>

#include "../../include/b200wave.h"

#ifdef __CUDACC__
#define B200W_HD __host__ __device__ __forceinline__
#define B200W_D __device__ __forceinline__
#define B200W_FOR_THREADS(tid, NT) { const int tid = (int)threadIdx.x;
#define B200W_END_THREADS }
#define B200W_SYNC() __syncthreads()
#else
#define B200W_HD inline
#define B200W_D inline
#define B200W_FOR_THREADS(tid, NT) for (int tid = 0; tid < (NT); ++tid) {
#define B200W_END_THREADS }
#define B200W_SYNC() ((void)0)
#endif

namespace b200w {

// IEEE round-to-nearest arithmetic in either precision.  On the device the explicit intrinsics keep the compiler from
// contracting a product and a sum into one FMA; the host emulation is built with -ffp-contract=off and uses the plain
// operators.  fma_rn is the one fused multiply-add of the accumulation loops.
#ifdef __CUDACC__
B200W_D float mul_rn(float a, float b) { return __fmul_rn(a, b); }
B200W_D double mul_rn(double a, double b) { return __dmul_rn(a, b); }
B200W_D float add_rn(float a, float b) { return __fadd_rn(a, b); }
B200W_D double add_rn(double a, double b) { return __dadd_rn(a, b); }
B200W_D float sub_rn(float a, float b) { return __fsub_rn(a, b); }
B200W_D double sub_rn(double a, double b) { return __dsub_rn(a, b); }
B200W_D float div_rn(float a, float b) { return __fdiv_rn(a, b); }
B200W_D double div_rn(double a, double b) { return __ddiv_rn(a, b); }
B200W_D float sqrt_rn(float a) { return __fsqrt_rn(a); }
B200W_D double sqrt_rn(double a) { return __dsqrt_rn(a); }
#else
template <class T> inline T mul_rn(T a, T b) { return a * b; }
template <class T> inline T add_rn(T a, T b) { return a + b; }
template <class T> inline T sub_rn(T a, T b) { return a - b; }
template <class T> inline T div_rn(T a, T b) { return a / b; }
inline float sqrt_rn(float a) { return sqrtf(a); }
inline double sqrt_rn(double a) { return sqrt(a); }
#endif
B200W_D float fma_rn(float a, float b, float c) { return fmaf(a, b, c); }
B200W_D double fma_rn(double a, double b, double c) { return fma(a, b, c); }

constexpr int kMaxTaps = B200W_MAX_TAPS;
// 1/sqrt(2) rounded once to the element type
template <class T> constexpr T kInvSqrt2T = (T)0.70710678118654752440;
constexpr float kInvSqrt2 = kInvSqrt2T<float>;

// Filter taps travel as kernel parameters (constant bank): with a compile-time tap index the FFMA
// takes its coefficient straight from c[0x0][..]; with a runtime index it is one LDC.
template <class T>
struct alignas(16) TapsT {
  T t[kMaxTaps];
};
using Taps = TapsT<float>;

// Boundary extension: index of the extended signal -> index in [0,N), or -1 meaning "zero".
// Same closed forms as the oracle (reference utils.py:146-163 reflect; dwt/lowlevel.py:28-88 mypad;
// :135-141 periodization pre-extension).
B200W_HD int ext_index(int i, int N, int mode) {
  if ((unsigned)i < (unsigned)N) return i;
  int p, r;
  switch (mode) {
    case B200W_MODE_SYMMETRIC:
      p = 2 * N;
      r = i % p;
      if (r < 0) r += p;
      return r < N ? r : p - 1 - r;
    case B200W_MODE_REFLECT:
      if (N == 1) return 0;
      p = 2 * N - 2;
      r = i % p;
      if (r < 0) r += p;
      return r < N ? r : p - r;
    case B200W_MODE_PERIODIC:
      r = i % N;
      if (r < 0) r += N;
      return r;
    case B200W_MODE_PERIODIZATION:
      p = N + (N & 1);
      r = i % p;
      if (r < 0) r += p;
      return r < N ? r : N - 1;
    default:
      return -1;
  }
}

// DTCWT level-1 extension: symmetric, or zero padding (reference dtcwt/lowlevel.py:75-79)
B200W_HD int sym_or_zero(int i, int N, int sym) {
  return sym ? ext_index(i, N, B200W_MODE_SYMMETRIC) : (((unsigned)i < (unsigned)N) ? i : -1);
}

B200W_HD int floordiv2(int a) { return a >> 1; }  // arithmetic shift == floor division by 2
B200W_HD int imax(int a, int b) { return a > b ? a : b; }
B200W_HD int imin(int a, int b) { return a < b ? a : b; }

// ---- parameter blocks (plain data, passed by value) ------------------------------------------
// Templates on the element type; the float32 blocks, which the streaming and pyramid kernels also take, keep the
// plain names.

template <class T>
struct AfbParamsT {  // K1
  const T* x; long long xps; int xpitch;
  T* ll; long long llps; int llpitch;
  T* highs;
  int planes, H, W, Ho, Wo, Lw, Lh, mode;
  int tiles_x, tiles_y;
  TapsT<T> fw_lo, fw_hi, fh_lo, fh_hi;
  int hipitch;        // experiments only (streaming kernel): row pitch of the band-pass planes, 0 = Wo
  // the W-pass taps once more as interleaved {low-pass, high-pass} pairs: one aligned 64-bit constant load feeds a
  // packed FMA (pairs built from two separate arrays cost two extra uniform moves per FMA pair)
  alignas(16) T fwp[2 * kMaxTaps];
};

template <class T>
struct SfbParamsT {  // K2
  const T* ll; long long llps; int llpitch;
  const T* highs;
  T* y; long long yps; int ypitch;
  int planes, Hc, Wc, Ho, Wo, Lh, Lw, mode;
  int tiles_x, tiles_y;
  TapsT<T> gh_lo, gh_hi, gw_lo, gw_hi;
};

template <class T>
struct DtParamsT {  // K3..K7
  const T* in; long long inps; int inpitch;       // x (forward) / ll (inverse, may be null)
  T* out; long long outps; int outpitch;          // ll (forward) / y (inverse)
  T* highs;                                        // band-pass tensor (output forward, input inverse); may be null
  long long hs[6];                                 // element strides n,c,o,row,col,ri
  T* z; T* dre; T* dim;                            // scat outputs
  int N, C, H, W;                                  // forward: input dims; inverse: dims of the ll / quad grid
  int L0, L1;                                      // level-1 filter lengths, or L0 = m for q-shift
  int sym;                                         // 1 symmetric extension, 0 zero padding
  T magbias, magbias2;
  int tiles_x, tiles_y;
  TapsT<T> f0, f1, f2, f3;                         // level 1: f0=h0/g0, f1=h1/g1; q-shift: f0=*0a f1=*1a f2=*0b f3=*1b
  // q-shift forward: interleaved pairs {f2[j], f0[j]} (low-pass trees b, a) and {f3[j], f1[j]} (high-pass trees)
  alignas(16) T qlo[2 * kMaxTaps];
  alignas(16) T qhi[2 * kMaxTaps];
};

using AfbParams = AfbParamsT<float>;
using SfbParams = SfbParamsT<float>;
using DtParams = DtParamsT<float>;

}  // namespace b200w
