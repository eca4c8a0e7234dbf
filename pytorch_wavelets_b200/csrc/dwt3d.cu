// dwt3d.cu -- 3-D DWT levels (sm_90a): b200w_dwt_afb3d / b200w_dwt_sfb3d and their _generic / _f64 variants.
//
// One level is the 1-D filter bank along W, H and D with one filter pair.  Two routes:
//   * fused (float32, L in {2, 4, 6, 8}): afb3d_stream / sfb3d_stream.  A CTA owns a tile of (h, w) positions of one
//     volume and marches along D.  Every slice of the tile's window is staged once in shared memory (cp.async, double
//     buffered), the two in-plane passes run from shared memory, and each thread keeps the last few slices of its
//     positions in a register window whose indices are compile-time (one unrolled window period per loop trip).  The
//     input is read once (plus tile halos) and every output is written once.
//   * two-step (everything else, and the _generic / _f64 entries): the 2-D level over all volumes*D planes into the
//     workspace, then a 1-D pass along D (afb1d_strided), or the reverse for synthesis (sfb1d_strided, then the 2-D
//     synthesis level).  The strided kernels are templates on the element type.
// Analysis accumulates in the oracle's order (stored tap order, first term a product, then fused multiply-adds) on both
// routes, so both are bit-identical to the oracle composition.  The fused synthesis runs the in-plane passes before the
// pass along D (the two-step route runs D first); both agree within the fp32 error bound of the tests.
#include <cuda_runtime.h>

#include <type_traits>

#include "launch.cuh"
#include "launch_params.h"
#include "stream_common.cuh"

namespace b200w {

// ---- two-step route: 1-D passes along a strided axis ------------------------------------------------------------------

constexpr int kD3T = 256;   // threads per CTA = positions of the contiguous (h, w) plane per CTA

// Up to four (W, H) band groups per launch.  Group g reads src[g] + vol * svs[g] + d * sds[g] and writes lo[g] / hi[g]
// + vol * dvs + k * P (plane-contiguous outputs).
template <class T>
struct D3AfbParams {
  const T* src[4]; long long svs[4], sds[4];
  T* lo[4]; T* hi[4]; long long lvs[4], hvs[4];
  int vols, D, Do, P, L, mode, tiles;
  TapsT<T> f0, f1;
};

template <class T>
struct D3SfbParams {
  const T* lo[4]; const T* hi[4]; long long lvs[4], hvs[4];   // d stride P; hi[g] may be null (zeros)
  T* dst[4]; long long dvs[4], dds[4];
  int vols, K, Nout, P, L, mode, tiles;
  TapsT<T> g0, g1;
};

// out[k] = sum_j f[j] xe[2k + j - pl] along D (the afb1d_rows sum, dwt1d.cu), one thread per (k, h, w)
template <class T>
__global__ void __launch_bounds__(kD3T) afb1d_strided(const __grid_constant__ D3AfbParams<T> p) {
  long long b = blockIdx.x;
  const int tile = (int)(b % p.tiles); b /= p.tiles;
  const int k = (int)(b % p.Do); b /= p.Do;
  const int vol = (int)(b % p.vols);
  const int g = (int)(b / p.vols);
  const int idx = tile * kD3T + threadIdx.x;
  if (idx >= p.P) return;
  const int pl = (p.mode == B200W_MODE_PERIODIZATION) ? (p.L - 1 - p.L / 2) : (p.L - 2);
  const T* s = p.src[g] + (long long)vol * p.svs[g] + idx;
  T a0 = 0, a1 = 0;
  for (int j = 0; j < p.L; ++j) {
    const int d = ext_index(2 * k - pl + j, p.D, p.mode);
    const T v = (d >= 0) ? s[(long long)d * p.sds[g]] : T(0);
    if (j == 0) { a0 = mul_rn(p.f0.t[0], v); a1 = mul_rn(p.f1.t[0], v); }
    else { a0 = fma_rn(p.f0.t[j], v, a0); a1 = fma_rn(p.f1.t[j], v, a1); }
  }
  p.lo[g][(long long)vol * p.lvs[g] + (long long)k * p.P + idx] = a0;
  p.hi[g][(long long)vol * p.hvs[g] + (long long)k * p.P + idx] = a1;
}

// y[n] = sum_k lo[k] g0[s - 2k] + sum_k hi[k] g1[s - 2k], s = n + off, along D (the sfb1d_rows sum)
template <class T>
__global__ void __launch_bounds__(kD3T) sfb1d_strided(const __grid_constant__ D3SfbParams<T> p) {
  long long b = blockIdx.x;
  const int tile = (int)(b % p.tiles); b /= p.tiles;
  const int n = (int)(b % p.Nout); b /= p.Nout;
  const int vol = (int)(b % p.vols);
  const int g = (int)(b / p.vols);
  const int idx = tile * kD3T + threadIdx.x;
  if (idx >= p.P) return;
  const bool per = (p.mode == B200W_MODE_PERIODIZATION);
  const int s = n + (per ? (p.L / 2 - 1) : (p.L - 2));
  const T* lo = p.lo[g] + (long long)vol * p.lvs[g] + idx;
  const T* hi = p.hi[g] ? p.hi[g] + (long long)vol * p.hvs[g] + idx : nullptr;
  T a0 = 0, a1 = 0;
  bool first = true;
  for (int k = floordiv2(s - p.L + 2); k <= floordiv2(s); ++k) {
    int kk = k;
    if (per) { kk %= p.K; if (kk < 0) kk += p.K; }
    else if (k < 0 || k >= p.K) continue;
    const int t = s - 2 * k;
    const T vl = lo[(long long)kk * p.P], vh = hi ? hi[(long long)kk * p.P] : T(0);
    if (first) { a0 = mul_rn(vl, p.g0.t[t]); a1 = mul_rn(vh, p.g1.t[t]); first = false; }
    else { a0 = fma_rn(vl, p.g0.t[t], a0); a1 = fma_rn(vh, p.g1.t[t], a1); }
  }
  p.dst[g][(long long)vol * p.dvs[g] + (long long)n * p.dds[g] + idx] = add_rn(a0, a1);
}

// ---- fused float32 route ------------------------------------------------------------------------------------------------

constexpr int kF3T = 256;                  // threads per CTA: 32 lanes along W x 8 rows
constexpr int kA3TW = 32, kA3TH = 16;      // analysis tile of output (h, w) positions; a thread owns 2 rows of one column
constexpr int kS3TW = 64, kS3TH = 32;      // synthesis tile of output positions; a thread owns 2 columns x 4 rows

struct Afb3dParams {
  const float* x; long long xvs;
  float* yl; float* highs;
  int vols, D, H, W, Do, Ho, Wo, mode;
  int tiles_x, tiles_y, n_chunks, CH;
  Taps f0, f1;
};

struct Sfb3dParams {
  const float* yl; long long ylvs;
  const float* highs;   // null: low-pass only
  float* y;
  int vols, Dc, Hc, Wc, Do, Ho, Wo, mode;
  int tiles_x, tiles_y, n_chunks, CH;
  Taps g0, g1;
};

template <int L>
struct Afb3dCfg {
  static constexpr int WR = 2 * kA3TH + L - 2, WC = 2 * kA3TW + L - 2, WN = WR * WC;   // staged input window
  static constexpr int SMEM_BYTES = (2 * WN + 2 * WR * kA3TW) * 4 + (WR + WC) * 4;
};

template <int L>
struct Sfb3dCfg {
  static constexpr int FR = kS3TH / 2 + L / 2 + 1, FC = kS3TW / 2 + L / 2 + 1, FN = FR * FC;   // coefficient footprint
  static constexpr int P = L / 2;          // register window: coefficient slices per output slice
  static constexpr int SMEM_BYTES = (2 * 8 * FN + 4 * kS3TH * FC) * 4 + (FR + FC) * 4;
};

// Analysis.  Slice i of a chunk is extended D index 2*k0 - pl + i; output slice k0 + m is emitted after slice 2m + L - 1
// from register window slots (u + 1 + j) mod L, u = i mod L.
template <int L>
__global__ void __launch_bounds__(kF3T, 2) afb3d_stream(const __grid_constant__ Afb3dParams p) {
  using C = Afb3dCfg<L>;
  extern __shared__ __align__(16) float sm3[];
  float* buf = sm3;                        // [2][WR][WC]
  float* wlo = sm3 + 2 * C::WN;            // [WR][TW] W-pass low-pass
  float* whi = wlo + C::WR * kA3TW;        // [WR][TW] W-pass high-pass
  int* rsrc = reinterpret_cast<int*>(whi + C::WR * kA3TW);
  int* csrc = rsrc + C::WR;
  const int tid = threadIdx.x, tx = tid & 31, ty = tid >> 5;
  long long item = blockIdx.x;
  const int bx = (int)(item % p.tiles_x); item /= p.tiles_x;
  const int by = (int)(item % p.tiles_y); item /= p.tiles_y;
  const int chunk = (int)(item % p.n_chunks);
  const int vol = (int)(item / p.n_chunks);
  const int pl = (p.mode == B200W_MODE_PERIODIZATION) ? (L - 1 - L / 2) : (L - 2);
  const int h0 = by * kA3TH, w0 = bx * kA3TW;
  for (int i = tid; i < C::WR; i += kF3T) rsrc[i] = ext_index(2 * h0 - pl + i, p.H, p.mode);
  for (int i = tid; i < C::WC; i += kF3T) csrc[i] = ext_index(2 * w0 - pl + i, p.W, p.mode);
  __syncthreads();
  const int k0 = chunk * p.CH, k1 = imin(k0 + p.CH, p.Do);
  const int n = 2 * (k1 - k0) + L - 2;
  const float* xv = p.x + (long long)vol * p.xvs;
  const long long plane = (long long)p.H * p.W;

  auto stage = [&](int i, float* dst) {
    const int gd = ext_index(2 * k0 - pl + i, p.D, p.mode);
    const float* xs = xv + (long long)gd * plane;
    for (int e = tid; e < C::WN; e += kF3T) {
      const int r = e / C::WC, c = e - r * C::WC;
      const int gr = rsrc[r], gc = csrc[c];
      if (gd >= 0 && gr >= 0 && gc >= 0) fast::cp_async4(dst + e, xs + (long long)gr * p.W + gc);
      else dst[e] = 0.f;
    }
    fast::cp_async_commit();
  };

  float ring[L][2][4];
#pragma unroll
  for (int a = 0; a < L; ++a)
#pragma unroll
    for (int q = 0; q < 2; ++q)
#pragma unroll
      for (int v = 0; v < 4; ++v) ring[a][q][v] = 0.f;

  const long long band = (long long)p.Do * p.Ho * p.Wo;
  const int wo = w0 + tx;
  stage(0, buf);
#pragma unroll 1
  for (int base = 0; base < n; base += L) {
#pragma unroll
    for (int u = 0; u < L; ++u) {
      const int i = base + u;
      if (i >= n) break;
      fast::cp_async_wait<0>();
      __syncthreads();
      if (i + 1 < n) stage(i + 1, buf + ((i + 1) & 1) * C::WN);
      const float* cur = buf + (i & 1) * C::WN;
      for (int r = ty; r < C::WR; r += kF3T / 32) {        // W pass: one output column, both filters
        const float* s = cur + r * C::WC + 2 * tx;
        float lo = mul_rn(p.f0.t[0], s[0]), hi = mul_rn(p.f1.t[0], s[0]);
#pragma unroll
        for (int j = 1; j < L; ++j) { lo = fma_rn(p.f0.t[j], s[j], lo); hi = fma_rn(p.f1.t[j], s[j], hi); }
        wlo[r * kA3TW + tx] = lo;
        whi[r * kA3TW + tx] = hi;
      }
      __syncthreads();
#pragma unroll
      for (int q = 0; q < 2; ++q) {                       // H pass: {ll, lh, hl, hh} of rows ty and ty + 8
        const float* cl = wlo + 2 * (ty + 8 * q) * kA3TW + tx;
        const float* ch = whi + 2 * (ty + 8 * q) * kA3TW + tx;
        float ll = mul_rn(p.f0.t[0], cl[0]), lh = mul_rn(p.f1.t[0], cl[0]);
        float hl = mul_rn(p.f0.t[0], ch[0]), hh = mul_rn(p.f1.t[0], ch[0]);
#pragma unroll
        for (int j = 1; j < L; ++j) {
          ll = fma_rn(p.f0.t[j], cl[j * kA3TW], ll); lh = fma_rn(p.f1.t[j], cl[j * kA3TW], lh);
          hl = fma_rn(p.f0.t[j], ch[j * kA3TW], hl); hh = fma_rn(p.f1.t[j], ch[j * kA3TW], hh);
        }
        ring[u][q][0] = ll; ring[u][q][1] = lh; ring[u][q][2] = hl; ring[u][q][3] = hh;
      }
      if ((u & 1) && i >= L - 1) {                        // D pass: output slice k0 + (i - L + 1) / 2
        const int k = k0 + (i - L + 1) / 2;
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          const int ho = h0 + ty + 8 * q;
          if (ho >= p.Ho || wo >= p.Wo) continue;
          const long long o = (long long)k * p.Ho * p.Wo + (long long)ho * p.Wo + wo;
          float* hb = p.highs + (long long)vol * 7 * band + o;
#pragma unroll
          for (int v = 0; v < 4; ++v) {
            float dl = mul_rn(p.f0.t[0], ring[(u + 1) % L][q][v]), dh = mul_rn(p.f1.t[0], ring[(u + 1) % L][q][v]);
#pragma unroll
            for (int j = 1; j < L; ++j) {
              dl = fma_rn(p.f0.t[j], ring[(u + 1 + j) % L][q][v], dl);
              dh = fma_rn(p.f1.t[j], ring[(u + 1 + j) % L][q][v], dh);
            }
            // band 4aW + 2aH + aD - 1 with v = 2aW + aH: (v, low) -> 2v - 1 (v = 0: yl), (v, high) -> 2v
            if (v == 0) p.yl[(long long)vol * band + o] = dl;
            else hb[(2 * v - 1) * band] = dl;
            hb[2 * v * band] = dh;
          }
        }
      }
    }
  }
}

__device__ __forceinline__ int coef_index(int k, int K, bool per) {
  if (per) { k %= K; return k < 0 ? k + K : k; }
  return (k >= 0 && k < K) ? k : -1;
}

// Synthesis.  Per coefficient slice: the 2-D synthesis (H, then W) of the D-low bands {yl, 1, 3, 5} and of the D-high
// bands {0, 2, 4, 6} at every output position of the tile, kept for the last L/2 slices; after slice k the output slices
// 2k - off and 2k + 1 - off are complete.
template <int L>
__global__ void __launch_bounds__(kF3T, 2) sfb3d_stream(const __grid_constant__ Sfb3dParams p) {
  using C = Sfb3dCfg<L>;
  constexpr int FC = C::FC, FN = C::FN, PP = C::P;
  extern __shared__ __align__(16) float sm3[];
  float* buf = sm3;                        // [2][8][FR][FC]: 0 = yl, 1 + b = band b
  float* hp = sm3 + 2 * 8 * FN;            // [4][TH][FC]: (D group, H low / high)
  int* rsrc = reinterpret_cast<int*>(hp + 4 * kS3TH * FC);
  int* csrc = rsrc + C::FR;
  const int tid = threadIdx.x, tx = tid & 31, ty = tid >> 5;
  long long item = blockIdx.x;
  const int bx = (int)(item % p.tiles_x); item /= p.tiles_x;
  const int by = (int)(item % p.tiles_y); item /= p.tiles_y;
  const int chunk = (int)(item % p.n_chunks);
  const int vol = (int)(item / p.n_chunks);
  const bool per = (p.mode == B200W_MODE_PERIODIZATION);
  const bool has_hi = p.highs != nullptr;
  const int off = per ? (L / 2 - 1) : (L - 2);
  const int h0 = by * kS3TH, w0 = bx * kS3TW;
  const int kbh = floordiv2(h0 + off - L + 2), kbw = floordiv2(w0 + off - L + 2);
  for (int i = tid; i < C::FR; i += kF3T) rsrc[i] = coef_index(kbh + i, p.Hc, per);
  for (int i = tid; i < FC; i += kF3T) csrc[i] = coef_index(kbw + i, p.Wc, per);
  __syncthreads();
  const int n0 = chunk * p.CH, n1 = imin(n0 + p.CH, p.Do);
  const int ks = floordiv2(n0 + off - L + 2);
  const int nk = floordiv2(n1 - 1 + off) - ks + 1;
  const long long pc = (long long)p.Hc * p.Wc;
  const float* ylv = p.yl + (long long)vol * p.ylvs;
  const float* hv = has_hi ? p.highs + (long long)vol * 7 * p.Dc * pc : nullptr;

  auto stage = [&](int i, float* dst) {
    const int kd = coef_index(ks + i, p.Dc, per);
    const int nb = has_hi ? 8 : 1;
    for (int e = tid; e < nb * FN; e += kF3T) {
      const int bb = e / FN, f = e - bb * FN;
      const int r = f / FC, c = f - r * FC;
      const int gr = rsrc[r], gc = csrc[c];
      if (kd >= 0 && gr >= 0 && gc >= 0) {
        const float* src = (bb == 0) ? ylv : hv + (long long)(bb - 1) * p.Dc * pc;
        fast::cp_async4(dst + e, src + (long long)kd * pc + (long long)gr * p.Wc + gc);
      } else {
        dst[e] = 0.f;
      }
    }
    fast::cp_async_commit();
  };

  float ylo[PP][8], yhi[PP][8];            // in-plane synthesis of the last L/2 slices, D-low and D-high groups
#pragma unroll
  for (int a = 0; a < PP; ++a)
#pragma unroll
    for (int q = 0; q < 8; ++q) ylo[a][q] = yhi[a][q] = 0.f;

  stage(0, buf);
#pragma unroll 1
  for (int base = 0; base < nk; base += PP) {
#pragma unroll
    for (int u = 0; u < PP; ++u) {
      const int i = base + u;
      if (i >= nk) break;
      fast::cp_async_wait<0>();
      __syncthreads();
      if (i + 1 < nk) stage(i + 1, buf + ((i + 1) & 1) * 8 * FN);
      const float* cur = buf + (i & 1) * 8 * FN;
      for (int e = tid; e < kS3TH * FC; e += kF3T) {      // H pass of both D groups
        const int r = e / FC, c = e - r * FC;
        const int s = h0 + r + off;
        const int fi = floordiv2(s - L + 2) - kbh, t0 = (s & 1) + L - 2;
#pragma unroll
        for (int d = 0; d < 2; ++d) {
          float lo = 0.f, hi = 0.f;
          if (has_hi) {
            float a_ll = 0.f, a_lh = 0.f, a_hl = 0.f, a_hh = 0.f;
#pragma unroll
            for (int m = 0; m < PP; ++m) {
              const int at = (fi + m) * FC + c;
              const float g0 = p.g0.t[t0 - 2 * m], g1 = p.g1.t[t0 - 2 * m];
              a_ll = fma_rn(cur[d * FN + at], g0, a_ll);
              a_lh = fma_rn(cur[(2 + d) * FN + at], g1, a_lh);
              a_hl = fma_rn(cur[(4 + d) * FN + at], g0, a_hl);
              a_hh = fma_rn(cur[(6 + d) * FN + at], g1, a_hh);
            }
            lo = add_rn(a_ll, a_lh);
            hi = add_rn(a_hl, a_hh);
          } else if (d == 0) {
#pragma unroll
            for (int m = 0; m < PP; ++m) lo = fma_rn(cur[(fi + m) * FC + c], p.g0.t[t0 - 2 * m], lo);
          }
          hp[(2 * d) * kS3TH * FC + e] = lo;
          hp[(2 * d + 1) * kS3TH * FC + e] = hi;
        }
      }
      __syncthreads();
#pragma unroll
      for (int q = 0; q < 8; ++q) {                       // W pass: column tx + 32 * (q & 1), row ty + 8 * (q >> 1)
        const int r = ty + 8 * (q >> 1), cw = tx + 32 * (q & 1);
        const int s = w0 + cw + off;
        const int fi = floordiv2(s - L + 2) - kbw, t0 = (s & 1) + L - 2;
        float v[2];
#pragma unroll
        for (int d = 0; d < 2; ++d) {
          const float* lo = hp + (2 * d) * kS3TH * FC + r * FC + fi;
          const float* hi = lo + kS3TH * FC;
          float a0 = 0.f, a1 = 0.f;
#pragma unroll
          for (int m = 0; m < PP; ++m) {
            a0 = fma_rn(lo[m], p.g0.t[t0 - 2 * m], a0);
            a1 = fma_rn(hi[m], p.g1.t[t0 - 2 * m], a1);
          }
          v[d] = add_rn(a0, a1);
        }
        ylo[u][q] = v[0];
        yhi[u][q] = v[1];
      }
      const int k = ks + i;
#pragma unroll
      for (int dd = 0; dd < 2; ++dd) {                    // D pass: output slice 2k + dd - off from slices k-L/2+1..k
        const int nd = 2 * k + dd - off;
        if (nd < n0 || nd >= n1) continue;
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          const int ho = h0 + ty + 8 * (q >> 1), wo = w0 + tx + 32 * (q & 1);
          if (ho >= p.Ho || wo >= p.Wo) continue;
          float a0 = 0.f, a1 = 0.f;
#pragma unroll
          for (int m = PP - 1; m >= 0; --m) {
            a0 = fma_rn(ylo[(u - m + PP) % PP][q], p.g0.t[dd + 2 * m], a0);
            a1 = fma_rn(yhi[(u - m + PP) % PP][q], p.g1.t[dd + 2 * m], a1);
          }
          p.y[(((long long)vol * p.Do + nd) * p.Ho + ho) * p.Wo + wo] = add_rn(a0, a1);
        }
      }
    }
  }
}

namespace {

inline bool fused_len(int L) { return L == 2 || L == 4 || L == 6 || L == 8; }

// resident CTAs of a fused kernel on the whole device (chunking decision, as the 2-D streaming kernels make it)
template <class K>
int resident_ctas(fast::ConcCache& cc, K kernel, int smem) {
  return imax(1, fast::resident_warps_dev(cc, kernel, smem, kF3T) / (kF3T / 32));
}

// D chunks: every chunk pays the window's prologue again (pro, in output slices)
inline void d_chunks(long long items, int Dout, int pro, int conc, int* n_chunks, int* CH) {
  fast::pick_chunks(items, Dout, 4, pro, conc, n_chunks, CH);
}

template <int L>
int launch_afb3d(Afb3dParams& p, void* stream) {
  using C = Afb3dCfg<L>;
  static_assert(C::SMEM_BYTES <= 48 * 1024, "analysis window must fit the default shared-memory size");
  static fast::ConcCache cc;
  const long long items = (long long)p.vols * p.tiles_x * p.tiles_y;
  d_chunks(items, p.Do, (L - 2) / 2, resident_ctas(cc, afb3d_stream<L>, C::SMEM_BYTES), &p.n_chunks, &p.CH);
  const long long blocks = items * p.n_chunks;
  if (!grid_ok(blocks)) return B200W_ESIZE;
  return launch(afb3d_stream<L>, p, blocks, kF3T, C::SMEM_BYTES, stream);
}

template <int L>
int launch_sfb3d(Sfb3dParams& p, void* stream) {
  using C = Sfb3dCfg<L>;
  static fast::ConcCache cc;
  const long long items = (long long)p.vols * p.tiles_x * p.tiles_y;
  // the occupancy query needs the opt-in above 48 KB first (launch() repeats it)
  const int rc = check_cuda(cudaFuncSetAttribute(sfb3d_stream<L>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                 C::SMEM_BYTES));
  if (rc) return rc;
  d_chunks(items, p.Do, L - 2, resident_ctas(cc, sfb3d_stream<L>, C::SMEM_BYTES), &p.n_chunks, &p.CH);
  const long long blocks = items * p.n_chunks;
  if (!grid_ok(blocks)) return B200W_ESIZE;
  return launch(sfb3d_stream<L>, p, blocks, kF3T, C::SMEM_BYTES, stream);
}

long long align256(long long n) { return (n + 255) / 256 * 256; }

// ---- the 2-D levels of the two-step route (the library's own K1 / K2 entry points) ----------------------------------
int afb2d_entry(const float* x, long long xps, int xpitch, float* ll, long long llps, int llpitch, float* highs,
                int planes, int H, int W, const float* f0, const float* f1, int L, int mode, void* stream) {
  return b200w_dwt_afb2d(x, xps, xpitch, ll, llps, llpitch, highs, planes, H, W, f0, f1, L, f0, f1, L, mode, stream);
}
int afb2d_entry(const double* x, long long xps, int xpitch, double* ll, long long llps, int llpitch, double* highs,
                int planes, int H, int W, const double* f0, const double* f1, int L, int mode, void* stream) {
  return b200w_dwt_afb2d_f64(x, xps, xpitch, ll, llps, llpitch, highs, planes, H, W, f0, f1, L, f0, f1, L, mode, stream);
}
int sfb2d_entry(const float* ll, long long llps, int llpitch, const float* highs, float* y, long long yps, int ypitch,
                int planes, int Hc, int Wc, int Ho, int Wo, const float* g0, const float* g1, int L, int mode,
                void* stream) {
  return b200w_dwt_sfb2d(ll, llps, llpitch, highs, y, yps, ypitch, planes, Hc, Wc, Ho, Wo, g0, g1, L, g0, g1, L, mode,
                         stream);
}
int sfb2d_entry(const double* ll, long long llps, int llpitch, const double* highs, double* y, long long yps,
                int ypitch, int planes, int Hc, int Wc, int Ho, int Wo, const double* g0, const double* g1, int L,
                int mode, void* stream) {
  return b200w_dwt_sfb2d_f64(ll, llps, llpitch, highs, y, yps, ypitch, planes, Hc, Wc, Ho, Wo, g0, g1, L, g0, g1, L,
                             mode, stream);
}

// ---- argument checks and workspace sizes (no CUDA call) -------------------------------------------------------------

int check_afb3d(long long xvs, int vols, int D, int H, int W, int L, int mode) {
  if (!dwt_mode_ok(mode)) return B200W_EMODE;
  if (vols < 0 || D < 1 || H < 1 || W < 1) return B200W_ESIZE;
  if (L < 2 || L > kMaxTaps) return B200W_EFILTER;
  if (xvs < (long long)D * H * W) return B200W_EARG;
  return B200W_OK;
}

int check_sfb3d(int vols, int Dc, int Hc, int Wc, int Do, int Ho, int Wo, int L, int mode) {
  if (!dwt_mode_ok(mode)) return B200W_EMODE;
  if (vols < 0 || Dc < 1 || Hc < 1 || Wc < 1) return B200W_ESIZE;
  if (L < 2 || L > kMaxTaps) return B200W_EFILTER;
  if (Do < 1 || Ho < 1 || Wo < 1 || Do > rec_len(Dc, L, mode) || Ho > rec_len(Hc, L, mode) || Wo > rec_len(Wc, L, mode))
    return B200W_ESIZE;
  return B200W_OK;
}

// two-step analysis: ll and highs of the 2-D level over volumes*D planes
long long afb3d_ws(int vols, int D, int H, int W, int L, int mode, int elem) {
  const long long n = (long long)vols * D * coeff_len(H, L, mode) * coeff_len(W, L, mode) * elem;
  return align256(n) + align256(3 * n);
}
// two-step synthesis: ll and highs of the 2-D level over volumes*Do planes
long long sfb3d_ws(int vols, int Hc, int Wc, int Do, int elem) {
  const long long n = (long long)vols * Do * Hc * Wc * elem;
  return align256(n) + align256(3 * n);
}

template <class T>
long long afb3d_workspace(const T* x, long long xvs, int vols, int D, int H, int W, int L, int mode, bool generic) {
  (void)x;   // (no alignment precondition: the answer depends on the sizes alone)
  const int rc = check_afb3d(xvs, vols, D, H, W, L, mode);
  if (rc) return rc;
  if (std::is_same_v<T, float> && !generic && fused_len(L)) return 0;
  return afb3d_ws(vols, D, H, W, L, mode, (int)sizeof(T));
}

template <class T>
long long sfb3d_workspace(int vols, int Dc, int Hc, int Wc, int Do, int Ho, int Wo, int L, int mode, bool generic) {
  const int rc = check_sfb3d(vols, Dc, Hc, Wc, Do, Ho, Wo, L, mode);
  if (rc) return rc;
  if (std::is_same_v<T, float> && !generic && fused_len(L)) return 0;
  return sfb3d_ws(vols, Hc, Wc, Do, (int)sizeof(T));
}

// ---- one level, either route ------------------------------------------------------------------------------------------

template <class T>
int afb3d_impl(const T* x, long long xvs, T* yl, T* highs, int vols, int D, int H, int W, const T* f_lo, const T* f_hi,
               int L, int mode, void* ws, long long wsb, void* stream, bool generic) {
  if (!dwt_mode_ok(mode)) return B200W_EMODE;
  if (!x || !yl || !highs || !f_lo || !f_hi) return B200W_EARG;
  int rc = check_afb3d(xvs, vols, D, H, W, L, mode);
  if (rc) return rc;
  const int Do = coeff_len(D, L, mode), Ho = coeff_len(H, L, mode), Wo = coeff_len(W, L, mode);
  const long long P = (long long)Ho * Wo;
  if constexpr (std::is_same_v<T, float>) {
    if (!generic && fused_len(L)) {
      Afb3dParams p;
      if ((rc = set_taps(p.f0, f_lo, L)) || (rc = set_taps(p.f1, f_hi, L))) return rc;
      if (vols == 0) return B200W_OK;
      p.x = x; p.xvs = xvs; p.yl = yl; p.highs = highs;
      p.vols = vols; p.D = D; p.H = H; p.W = W; p.Do = Do; p.Ho = Ho; p.Wo = Wo; p.mode = mode;
      p.tiles_x = cdiv(Wo, kA3TW); p.tiles_y = cdiv(Ho, kA3TH);
      switch (L) {
        case 2: return launch_afb3d<2>(p, stream);
        case 4: return launch_afb3d<4>(p, stream);
        case 6: return launch_afb3d<6>(p, stream);
        default: return launch_afb3d<8>(p, stream);
      }
    }
  }
  D3AfbParams<T> q;
  if ((rc = set_taps(q.f0, f_lo, L)) || (rc = set_taps(q.f1, f_hi, L))) return rc;
  const long long need = afb3d_ws(vols, D, H, W, L, mode, (int)sizeof(T));
  if (!ws || wsb < need) return B200W_EARG;
  if (vols == 0) return B200W_OK;
  const long long planes = (long long)vols * D;
  if (planes > 2147483647LL) return B200W_ESIZE;
  T* ll2 = static_cast<T*>(ws);
  T* hi2 = reinterpret_cast<T*>(static_cast<char*>(ws) + align256(planes * P * (long long)sizeof(T)));
  const long long xps = (long long)H * W;
  if (xvs == (long long)D * xps) {
    rc = afb2d_entry(x, xps, W, ll2, P, Wo, hi2, (int)planes, H, W, f_lo, f_hi, L, mode, stream);
  } else {   // volumes further apart than D planes: one 2-D call per volume
    for (int v = 0; v < vols && !rc; ++v)
      rc = afb2d_entry(x + (long long)v * xvs, xps, W, ll2 + (long long)v * D * P, P, Wo, hi2 + (long long)v * D * 3 * P,
                       D, H, W, f_lo, f_hi, L, mode, stream);
  }
  if (rc) return rc;
  const long long band = (long long)Do * P;
  for (int g = 0; g < 4; ++g) {
    q.src[g] = g == 0 ? ll2 : hi2 + (g - 1) * P;
    q.svs[g] = (g == 0 ? 1 : 3) * D * P;
    q.sds[g] = (g == 0 ? 1 : 3) * P;
    q.lo[g] = g == 0 ? yl : highs + (2 * g - 1) * band;
    q.lvs[g] = g == 0 ? band : 7 * band;
    q.hi[g] = highs + 2 * g * band;
    q.hvs[g] = 7 * band;
  }
  q.vols = vols; q.D = D; q.Do = Do; q.P = (int)P; q.L = L; q.mode = mode;
  if (P > 2147483647LL) return B200W_ESIZE;
  q.tiles = cdiv((int)P, kD3T);
  const long long blocks = 4LL * vols * Do * q.tiles;
  if (!grid_ok(blocks)) return B200W_ESIZE;
  return launch(afb1d_strided<T>, q, blocks, kD3T, 0, stream);
}

template <class T>
int sfb3d_impl(const T* yl, long long ylvs, const T* highs, T* y, int vols, int Dc, int Hc, int Wc, int Do, int Ho,
               int Wo, const T* g_lo, const T* g_hi, int L, int mode, void* ws, long long wsb, void* stream,
               bool generic) {
  if (!dwt_mode_ok(mode)) return B200W_EMODE;
  if (!yl || !y || !g_lo || !g_hi) return B200W_EARG;
  int rc = check_sfb3d(vols, Dc, Hc, Wc, Do, Ho, Wo, L, mode);
  if (rc) return rc;
  const long long pc = (long long)Hc * Wc;
  if (ylvs < Dc * pc) return B200W_EARG;
  if constexpr (std::is_same_v<T, float>) {
    if (!generic && fused_len(L)) {
      Sfb3dParams p;
      if ((rc = set_taps(p.g0, g_lo, L)) || (rc = set_taps(p.g1, g_hi, L))) return rc;
      if (vols == 0) return B200W_OK;
      p.yl = yl; p.ylvs = ylvs; p.highs = highs; p.y = y;
      p.vols = vols; p.Dc = Dc; p.Hc = Hc; p.Wc = Wc; p.Do = Do; p.Ho = Ho; p.Wo = Wo; p.mode = mode;
      p.tiles_x = cdiv(Wo, kS3TW); p.tiles_y = cdiv(Ho, kS3TH);
      switch (L) {
        case 2: return launch_sfb3d<2>(p, stream);
        case 4: return launch_sfb3d<4>(p, stream);
        case 6: return launch_sfb3d<6>(p, stream);
        default: return launch_sfb3d<8>(p, stream);
      }
    }
  }
  D3SfbParams<T> q;
  if ((rc = set_taps(q.g0, g_lo, L)) || (rc = set_taps(q.g1, g_hi, L))) return rc;
  const long long need = sfb3d_ws(vols, Hc, Wc, Do, (int)sizeof(T));
  if (!ws || wsb < need) return B200W_EARG;
  if (vols == 0) return B200W_OK;
  const long long planes = (long long)vols * Do;
  if (planes > 2147483647LL || pc > 2147483647LL) return B200W_ESIZE;
  T* ll2 = static_cast<T*>(ws);
  T* hi2 = reinterpret_cast<T*>(static_cast<char*>(ws) + align256(planes * pc * (long long)sizeof(T)));
  const long long band = (long long)Dc * pc;
  const int groups = highs ? 4 : 1;   // without band-passes the three (W, H) band-pass groups are zeros
  for (int g = 0; g < 4; ++g) {
    q.lo[g] = g == 0 ? yl : (highs ? highs + (2 * g - 1) * band : nullptr);
    q.lvs[g] = g == 0 ? ylvs : 7 * band;
    q.hi[g] = highs ? highs + 2 * g * band : nullptr;
    q.hvs[g] = 7 * band;
    q.dst[g] = g == 0 ? ll2 : hi2 + (g - 1) * pc;
    q.dvs[g] = (g == 0 ? 1 : 3) * Do * pc;
    q.dds[g] = (g == 0 ? 1 : 3) * pc;
  }
  q.vols = vols; q.K = Dc; q.Nout = Do; q.P = (int)pc; q.L = L; q.mode = mode;
  q.tiles = cdiv((int)pc, kD3T);
  const long long blocks = (long long)groups * vols * Do * q.tiles;
  if (!grid_ok(blocks)) return B200W_ESIZE;
  if ((rc = launch(sfb1d_strided<T>, q, blocks, kD3T, 0, stream))) return rc;
  return sfb2d_entry(ll2, pc, Wc, highs ? hi2 : nullptr, y, (long long)Ho * Wo, Wo, (int)planes, Hc, Wc, Ho, Wo, g_lo,
                     g_hi, L, mode, stream);
}

}  // namespace
}  // namespace b200w

using namespace b200w;

extern "C" {

long long b200w_dwt_afb3d_workspace(const float* x, long long x_vol_stride, int volumes, int D, int H, int W, int L,
                                    int mode) {
  return afb3d_workspace(x, x_vol_stride, volumes, D, H, W, L, mode, false);
}
long long b200w_dwt_afb3d_workspace_generic(const float* x, long long x_vol_stride, int volumes, int D, int H, int W,
                                            int L, int mode) {
  return afb3d_workspace(x, x_vol_stride, volumes, D, H, W, L, mode, true);
}
long long b200w_dwt_afb3d_workspace_f64(const double* x, long long x_vol_stride, int volumes, int D, int H, int W,
                                        int L, int mode) {
  return afb3d_workspace(x, x_vol_stride, volumes, D, H, W, L, mode, true);
}

int b200w_dwt_afb3d(const float* x, long long x_vol_stride, float* yl, float* highs, int volumes, int D, int H, int W,
                    const float* f_lo, const float* f_hi, int L, int mode, void* workspace, long long workspace_bytes,
                    void* stream) {
  return afb3d_impl(x, x_vol_stride, yl, highs, volumes, D, H, W, f_lo, f_hi, L, mode, workspace, workspace_bytes,
                    stream, false);
}
int b200w_dwt_afb3d_generic(const float* x, long long x_vol_stride, float* yl, float* highs, int volumes, int D, int H,
                            int W, const float* f_lo, const float* f_hi, int L, int mode, void* workspace,
                            long long workspace_bytes, void* stream) {
  return afb3d_impl(x, x_vol_stride, yl, highs, volumes, D, H, W, f_lo, f_hi, L, mode, workspace, workspace_bytes,
                    stream, true);
}
int b200w_dwt_afb3d_f64(const double* x, long long x_vol_stride, double* yl, double* highs, int volumes, int D, int H,
                        int W, const double* f_lo, const double* f_hi, int L, int mode, void* workspace,
                        long long workspace_bytes, void* stream) {
  return afb3d_impl(x, x_vol_stride, yl, highs, volumes, D, H, W, f_lo, f_hi, L, mode, workspace, workspace_bytes,
                    stream, true);
}

long long b200w_dwt_sfb3d_workspace(int volumes, int Dc, int Hc, int Wc, int Do, int Ho, int Wo, int L, int mode) {
  return sfb3d_workspace<float>(volumes, Dc, Hc, Wc, Do, Ho, Wo, L, mode, false);
}
long long b200w_dwt_sfb3d_workspace_generic(int volumes, int Dc, int Hc, int Wc, int Do, int Ho, int Wo, int L,
                                            int mode) {
  return sfb3d_workspace<float>(volumes, Dc, Hc, Wc, Do, Ho, Wo, L, mode, true);
}
long long b200w_dwt_sfb3d_workspace_f64(int volumes, int Dc, int Hc, int Wc, int Do, int Ho, int Wo, int L, int mode) {
  return sfb3d_workspace<double>(volumes, Dc, Hc, Wc, Do, Ho, Wo, L, mode, true);
}

int b200w_dwt_sfb3d(const float* yl, long long yl_vol_stride, const float* highs, float* y, int volumes, int Dc,
                    int Hc, int Wc, int Do, int Ho, int Wo, const float* g_lo, const float* g_hi, int L, int mode,
                    void* workspace, long long workspace_bytes, void* stream) {
  return sfb3d_impl(yl, yl_vol_stride, highs, y, volumes, Dc, Hc, Wc, Do, Ho, Wo, g_lo, g_hi, L, mode, workspace,
                    workspace_bytes, stream, false);
}
int b200w_dwt_sfb3d_generic(const float* yl, long long yl_vol_stride, const float* highs, float* y, int volumes,
                            int Dc, int Hc, int Wc, int Do, int Ho, int Wo, const float* g_lo, const float* g_hi, int L,
                            int mode, void* workspace, long long workspace_bytes, void* stream) {
  return sfb3d_impl(yl, yl_vol_stride, highs, y, volumes, Dc, Hc, Wc, Do, Ho, Wo, g_lo, g_hi, L, mode, workspace,
                    workspace_bytes, stream, true);
}
int b200w_dwt_sfb3d_f64(const double* yl, long long yl_vol_stride, const double* highs, double* y, int volumes, int Dc,
                        int Hc, int Wc, int Do, int Ho, int Wo, const double* g_lo, const double* g_hi, int L,
                        int mode, void* workspace, long long workspace_bytes, void* stream) {
  return sfb3d_impl(yl, yl_vol_stride, highs, y, volumes, Dc, Hc, Wc, Do, Ho, Wo, g_lo, g_hi, L, mode, workspace,
                    workspace_bytes, stream, true);
}

}  // extern "C"
