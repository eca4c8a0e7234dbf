#pragma once
#include "stream_common.cuh"

namespace b200w {
namespace fast {

// sfb_stream.cuh -- streaming DWT synthesis kernels (included inside namespace b200w::fast).
//
// One warp owns 64 coefficient columns (= 128 output columns) of one plane and marches down the
// coefficient rows.  The four subband rows (ll, lh, hl, hh) of each coefficient row are staged in a
// per-warp shared-memory ring with 4-byte cp.async (the band-pass tensors the caller hands in are
// contiguous with odd widths, so 16-byte alignment cannot be assumed).  The pass along W runs first on
// the staged rows (64-bit conflict-free LDS), the pass along H runs in a rotating register window --
// the two passes commute exactly in real arithmetic; in fp32 the result differs from the H-then-W order
// of the generic kernel / oracle by rounding only (<= 1e-6 relative, tests use the 1e-5 tolerance).
//   y[2c+ph] = sum_{i<L/2} a[c+i] g[L-2-2i+ph]   (non-periodization synthesis, reference sfb1d :263-267)

template <int L>
struct SfbCfg {
  static constexpr int HALF = L / 2;
  static constexpr int SWB = 96;                                  // staged floats per band row (3 x 32 lanes)
  static constexpr int KR = (HALF % 2 == 0) ? 2 : 1;              // coefficient rows per stage
  static constexpr int UNS = HALF / KR;                           // window period in stages
  static constexpr int NS = 3;
  static constexpr int STAGE = KR * 4 * SWB;                      // floats per stage
  static constexpr int SMEM_BYTES = NS * STAGE * 4;
  static constexpr int NVB = (HALF + 1 + 1) / 2;                  // 64-bit loads per band row per lane
  static_assert(HALF - 1 <= 32, "halo must fit the third 32-lane copy");
};

// one coefficient row: W pass into window slot U, then (if emit) the H pass for the output row pair.
// Packed FMA throughout: along W a coefficient times the (even, odd)-phase tap pair gives both output columns it
// feeds; along H a tap times a window column pair gives two adjacent outputs of one row.
// PER (periodization): the same sums over the periodic extension of the coefficients give y[(n' + L/2 - 1) mod 2K]
// (reference sfb1d :252-261 re-indexed: 2k + j - (L/2 - 1) = n  <=>  n' = n - L/2 + 1 with n' = 2c + phase,
// a[(c + i) mod K]); only the staging (wrapped rows / columns) and the store positions differ.
template <int L, int U, bool PER>
__device__ __forceinline__ void sfb_row(const SfbParams& p, const float* srow, float2 (&wP)[L / 2][2],
                                        float2 (&wQ)[L / 2][2], bool emit, float*& y_ptr, int ypitch, int nv4,
                                        bool row1_ok, const int (&ncol)[4], int nr0, int nr1) {
  using C = SfbCfg<L>;
  constexpr int HALF = C::HALF;
  float a[4][2 * C::NVB];  // [band][window]
#pragma unroll
  for (int b = 0; b < 4; ++b)
#pragma unroll
    for (int q = 0; q < C::NVB; ++q) {
      const float2 v = *reinterpret_cast<const float2*>(srow + b * C::SWB + 2 * q);
      a[b][2 * q] = v.x; a[b][2 * q + 1] = v.y;
    }
  // W pass: P = S(ll; gw_lo) + S(hl; gw_hi), Q = S(lh; gw_lo) + S(hh; gw_hi)   (bands: 0 ll, 1 lh, 2 hl, 3 hh)
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    float2 s_ll = make_float2(0.f, 0.f), s_lh = s_ll, s_hl = s_ll, s_hh = s_ll;   // {phase 0, phase 1}
#pragma unroll
    for (int i = 0; i < HALF; ++i) {
      const float2 g0 = make_float2(p.gw_lo.t[L - 2 - 2 * i], p.gw_lo.t[L - 1 - 2 * i]);
      const float2 g1 = make_float2(p.gw_hi.t[L - 2 - 2 * i], p.gw_hi.t[L - 1 - 2 * i]);
      s_ll = ffma2_s(a[0][e + i], g0, s_ll);
      s_lh = ffma2_s(a[1][e + i], g0, s_lh);
      s_hl = ffma2_s(a[2][e + i], g1, s_hl);
      s_hh = ffma2_s(a[3][e + i], g1, s_hh);
    }
    wP[U][e] = make_float2(__fadd_rn(s_ll.x, s_hl.x), __fadd_rn(s_ll.y, s_hl.y));
    wQ[U][e] = make_float2(__fadd_rn(s_lh.x, s_hh.x), __fadd_rn(s_lh.y, s_hh.y));
  }
  if (emit) {
    float2 o[2][2];  // [output row of the pair][column pair]
#pragma unroll
    for (int ph = 0; ph < 2; ++ph)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        float2 s0 = make_float2(0.f, 0.f), s1 = s0;
#pragma unroll
        for (int i = 0; i < HALF; ++i) {
          const int sl = (U + 1 + i) % HALF;
          s0 = ffma2_s(p.gh_lo.t[L - 2 - 2 * i + ph], wP[sl][e], s0);
          s1 = ffma2_s(p.gh_hi.t[L - 2 - 2 * i + ph], wQ[sl][e], s1);
        }
        o[ph][e] = make_float2(__fadd_rn(s0.x, s1.x), __fadd_rn(s0.y, s1.y));
      }
    if constexpr (PER) {
      // y_ptr = plane base; nr0 / nr1 = rotated output rows of the pair (-1: outside the requested output),
      // ncol[] = rotated output columns of the lane's four values
#pragma unroll
      for (int ph = 0; ph < 2; ++ph) {
        const int nr = ph ? nr1 : nr0;
        if (nr < 0) continue;
        float* q = y_ptr + (long long)nr * ypitch;
        if (ncol[0] >= 0) q[ncol[0]] = o[ph][0].x;
        if (ncol[1] >= 0) q[ncol[1]] = o[ph][0].y;
        if (ncol[2] >= 0) q[ncol[2]] = o[ph][1].x;
        if (ncol[3] >= 0) q[ncol[3]] = o[ph][1].y;
      }
    } else {
#pragma unroll
      for (int ph = 0; ph < 2; ++ph) {
        if (ph == 1 && !row1_ok) break;
        float* q = y_ptr + ph * ypitch;
        if (0 < nv4) q[0] = o[ph][0].x;
        if (1 < nv4) q[1] = o[ph][0].y;
        if (2 < nv4) q[2] = o[ph][1].x;
        if (3 < nv4) q[3] = o[ph][1].y;
      }
      y_ptr += 2 * ypitch;
    }
  }
}

template <int L, int V, bool PER>
__device__ __forceinline__ void sfb_stage_dispatch(int vv, const SfbParams& p, const float* stage,
                                                   float2 (&wP)[L / 2][2], float2 (&wQ)[L / 2][2], int rho0,
                                                   int rho_end, int m0, float*& y_ptr, int ypitch, int nv4,
                                                   const int (&ncol)[4]) {
  using C = SfbCfg<L>;
  if constexpr (V < C::UNS) {
    if (vv == V) {
#pragma unroll
      for (int r = 0; r < C::KR; ++r) {
        const int rho = rho0 + r;                         // coefficient row index relative to the chunk start
        const bool emit = (rho >= C::HALF - 1) && (rho < rho_end);
        const int n0 = 2 * (m0 + rho - (C::HALF - 1));    // first output row of the pair (before rotation if PER)
        int nr0 = -1, nr1 = -1;
        if (PER && emit) {
          const int N = 2 * p.Hc;
          // true modulo: for planes smaller than the filter (full-depth pyramids) the rotation L/2-1 can exceed N
          nr0 = (n0 + C::HALF - 1) % N;
          nr1 = (n0 + C::HALF) % N;
          if (nr0 >= p.Ho) nr0 = -1;
          if (nr1 >= p.Ho) nr1 = -1;
        }
        if (r == 0)
          sfb_row<L, C::KR * V, PER>(p, stage, wP, wQ, emit, y_ptr, ypitch, nv4, n0 + 1 < p.Ho, ncol, nr0, nr1);
        else
          sfb_row<L, C::KR * V + (C::KR - 1), PER>(p, stage + 4 * C::SWB, wP, wQ, emit, y_ptr, ypitch, nv4, n0 + 1 < p.Ho,
                                                   ncol, nr0, nr1);
      }
    } else {
      sfb_stage_dispatch<L, V + 1, PER>(vv, p, stage, wP, wQ, rho0, rho_end, m0, y_ptr, ypitch, nv4, ncol);
    }
  }
}

#define B200W_SFB_KERNEL sfb2d_stream
#define B200W_SFB_PLANE_BANDS 3
#include "sfb_stream_kernel.cuh"
#undef B200W_SFB_KERNEL
#undef B200W_SFB_PLANE_BANDS
#define B200W_SFB_KERNEL wpt_sfb2d_stream
#define B200W_SFB_PLANE_BANDS 4
#include "sfb_stream_kernel.cuh"
#undef B200W_SFB_KERNEL
#undef B200W_SFB_PLANE_BANDS

// ------------------------------------------------------------------------------------------------------------------
// Wide form (filters up to 8 taps, every mode except periodization): a lane owns FOUR coefficient columns (eight
// output columns), a strip is 128 coefficient columns.  Why: the 2-column form above is bound by its shared-memory /
// LSU instruction stream (`mio_throttle` is its main stall reason): per 4 outputs it issues 12 LDGSTS.32 + 12 LDS.64.  Here a lane's window of a band row is 4 + L/2 - 1
// adjacent coefficients = two aligned LDS.128, and the staged row costs 5 LDGSTS.32 per 128 + 3 columns (-33 %
// shared-memory wavefronts); the 512-wide level is exactly two strips (no remainder strip).  Same arithmetic and
// summation order as the 2-column form.
// Outputs are written with 32-bit stores in both forms.  Built for sm_90a with nvcc 12.9, the earlier form that used
// 128-bit stores (float4, when the output rows were 16-byte aligned) gave wrong values on the H100 in some 16-byte groups
// of the first columns of a plane (zeros or partial sums), the same from run to run, in both kernels;
// test_wide_synthesis_kernel_every_width_matches_generic_and_oracle and test_synthesis_streaming_kernels_multi_chunk
// (tests/test_gpu_parity.py) catch it.  The cause is NOT known: the SASS of that path is the expected
// STG.E.128 of the same registers to the same address as the scalar stores, and a fence after the ring zeroing did not
// change the result, so a race elsewhere in the kernel that only this schedule exposes has not been ruled out.
// ------------------------------------------------------------------------------------------------------------------
template <int L>
struct Sfb4Cfg {
  static constexpr int HALF = L / 2;
  static constexpr int CW = 128;                                   // coefficient columns per strip (4 per lane)
  static constexpr int NCOPY = (CW + HALF - 1 + 31) / 32;          // 32-lane copies per staged band row
  static constexpr int SWB = (CW + HALF - 1 + 3) / 4 * 4;         // staged floats per band row (16-byte multiple)
  static constexpr int KR = (HALF % 2 == 0) ? 2 : 1;               // coefficient rows per stage
  static constexpr int UNS = HALF / KR;                            // window period in stages
  static constexpr int NS = 2;                                     // ring depth in stages
  static constexpr int STAGE = KR * 4 * SWB;
  static constexpr int SMEM_BYTES = NS * STAGE * 4;
  static constexpr int NW = 4 + HALF - 1;                          // window of a lane in a band row
  static constexpr int NV4 = (NW + 3) / 4;                         // ... as 128-bit loads
  static_assert(4 * 31 + 4 * NV4 <= SWB, "the last lane's window must lie inside the staged row");
};

template <int L, int U>
__device__ __forceinline__ void sfb4_row(const SfbParams& p, const float* srow, float2 (&wP)[L / 2][4],
                                         float2 (&wQ)[L / 2][4], bool emit, float*& y_ptr, int ypitch, int nv8,
                                         bool row1_ok) {
  using C = Sfb4Cfg<L>;
  constexpr int HALF = C::HALF;
  float a[4][4 * C::NV4];  // [band][window]
#pragma unroll
  for (int b = 0; b < 4; ++b)
#pragma unroll
    for (int q = 0; q < C::NV4; ++q) {
      const float4 v = *reinterpret_cast<const float4*>(srow + b * C::SWB + 4 * q);
      a[b][4 * q] = v.x; a[b][4 * q + 1] = v.y; a[b][4 * q + 2] = v.z; a[b][4 * q + 3] = v.w;
    }
  // W pass: P = S(ll; gw_lo) + S(hl; gw_hi), Q = S(lh; gw_lo) + S(hh; gw_hi)   (bands: 0 ll, 1 lh, 2 hl, 3 hh)
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    float2 s_ll = make_float2(0.f, 0.f), s_lh = s_ll, s_hl = s_ll, s_hh = s_ll;   // {phase 0, phase 1}
#pragma unroll
    for (int i = 0; i < HALF; ++i) {
      const float2 g0 = make_float2(p.gw_lo.t[L - 2 - 2 * i], p.gw_lo.t[L - 1 - 2 * i]);
      const float2 g1 = make_float2(p.gw_hi.t[L - 2 - 2 * i], p.gw_hi.t[L - 1 - 2 * i]);
      s_ll = ffma2_s(a[0][e + i], g0, s_ll);
      s_lh = ffma2_s(a[1][e + i], g0, s_lh);
      s_hl = ffma2_s(a[2][e + i], g1, s_hl);
      s_hh = ffma2_s(a[3][e + i], g1, s_hh);
    }
    wP[U][e] = make_float2(__fadd_rn(s_ll.x, s_hl.x), __fadd_rn(s_ll.y, s_hl.y));
    wQ[U][e] = make_float2(__fadd_rn(s_lh.x, s_hh.x), __fadd_rn(s_lh.y, s_hh.y));
  }
  if (emit) {
#pragma unroll
    for (int ph = 0; ph < 2; ++ph) {
      float2 o[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float2 s0 = make_float2(0.f, 0.f), s1 = s0;
#pragma unroll
        for (int i = 0; i < HALF; ++i) {
          const int sl = (U + 1 + i) % HALF;
          s0 = ffma2_s(p.gh_lo.t[L - 2 - 2 * i + ph], wP[sl][e], s0);
          s1 = ffma2_s(p.gh_hi.t[L - 2 - 2 * i + ph], wQ[sl][e], s1);
        }
        o[e] = make_float2(__fadd_rn(s0.x, s1.x), __fadd_rn(s0.y, s1.y));
      }
      if (ph == 1 && !row1_ok) break;
      float* q = y_ptr + ph * ypitch;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        if (2 * e < nv8) q[2 * e] = o[e].x;
        if (2 * e + 1 < nv8) q[2 * e + 1] = o[e].y;
      }
    }
    y_ptr += 2 * ypitch;
  }
}

template <int L, int V>
__device__ __forceinline__ void sfb4_stage_dispatch(int vv, const SfbParams& p, const float* stage,
                                                    float2 (&wP)[L / 2][4], float2 (&wQ)[L / 2][4], int rho0,
                                                    int rho_end, int m0, float*& y_ptr, int ypitch, int nv8) {
  using C = Sfb4Cfg<L>;
  if constexpr (V < C::UNS) {
    if (vv == V) {
#pragma unroll
      for (int r = 0; r < C::KR; ++r) {
        const int rho = rho0 + r;                         // coefficient row index relative to the chunk start
        const bool emit = (rho >= C::HALF - 1) && (rho < rho_end);
        const int n0 = 2 * (m0 + rho - (C::HALF - 1));    // first output row of the pair
        if (r == 0) sfb4_row<L, C::KR * V>(p, stage, wP, wQ, emit, y_ptr, ypitch, nv8, n0 + 1 < p.Ho);
        else sfb4_row<L, C::KR * V + (C::KR - 1)>(p, stage + 4 * C::SWB, wP, wQ, emit, y_ptr, ypitch, nv8, n0 + 1 < p.Ho);
      }
    } else {
      sfb4_stage_dispatch<L, V + 1>(vv, p, stage, wP, wQ, rho0, rho_end, m0, y_ptr, ypitch, nv8);
    }
  }
}

#define B200W_SFB4_KERNEL sfb2d_stream4
#define B200W_SFB_PLANE_BANDS 3
#include "sfb_stream4_kernel.cuh"
#undef B200W_SFB4_KERNEL
#undef B200W_SFB_PLANE_BANDS
#define B200W_SFB4_KERNEL wpt_sfb2d_stream4
#define B200W_SFB_PLANE_BANDS 4
#include "sfb_stream4_kernel.cuh"
#undef B200W_SFB4_KERNEL
#undef B200W_SFB_PLANE_BANDS

// the DWT-layout or the packet-layout kernel (only the one asked for is instantiated)
template <int L, bool PER, bool PK, bool WIDE>
constexpr auto sfb_kernel_of() {
  if constexpr (WIDE) {
    if constexpr (PK) return wpt_sfb2d_stream4<L>;
    else return sfb2d_stream4<L>;
  } else {
    if constexpr (PK) return wpt_sfb2d_stream<L, PER>;
    else return sfb2d_stream<L, PER>;
  }
}

template <int L, bool PK>
inline int launch_sfb_stream4(const SfbParams& p, cudaStream_t stream, int n_strips) {
  using C = Sfb4Cfg<L>;
  constexpr auto kernel = sfb_kernel_of<L, false, PK, true>();
  const int npairs_h = (p.Ho + 1) >> 1;
  int n_chunks, CH;
  static ConcCache conc_cache;
  const int conc = resident_warps_dev(conc_cache, kernel, C::SMEM_BYTES);
  pick_chunks((long long)p.planes * n_strips, npairs_h, 16, L / 2 + 8, conc, &n_chunks, &CH);
  const long long blocks = (long long)p.planes * n_strips * n_chunks;
  if (blocks <= 0) return 0;
  if (blocks > 2147483647LL) return kNoFastPath;
  kernel<<<(unsigned)blocks, 32, C::SMEM_BYTES, stream>>>(p, n_strips, n_chunks, CH);
  return 0;
}

template <int L, bool PER, bool PK>
inline int launch_sfb_stream_m(const SfbParams& p, cudaStream_t stream) {
  using C = SfbCfg<L>;
  constexpr auto kernel = sfb_kernel_of<L, PER, PK, false>();
  const int npairs_w = PER ? p.Wc : (p.Wo + 1) >> 1;
  const int npairs_h = PER ? p.Hc : (p.Ho + 1) >> 1;
  const int n_strips = (npairs_w + 63) / 64;
  int n_chunks, CH;
  static ConcCache conc_cache;
  const int conc = resident_warps_dev(conc_cache, kernel, C::SMEM_BYTES);
  pick_chunks((long long)p.planes * n_strips, npairs_h, 16, L / 2 + 8, conc, &n_chunks, &CH);
  const long long blocks = (long long)p.planes * n_strips * n_chunks;
  if (blocks <= 0) return 0;
  if (blocks > 2147483647LL) return kNoFastPath;
  kernel<<<(unsigned)blocks, 32, C::SMEM_BYTES, stream>>>(p, n_strips, n_chunks, CH);
  return 0;
}

template <int L, bool PK>
inline int launch_sfb_stream(const SfbParams& p, cudaStream_t stream) {
  if (p.mode == B200W_MODE_PERIODIZATION) return launch_sfb_stream_m<L, true, PK>(p, stream);
  if constexpr (L <= 8) {
    // 128-column strips for every plane with more than 64 column pairs, remainder strip included: routing a narrow
    // remainder to the 2-column kernel in a second launch costs more than it saves, and one 67-pair wide strip beats a
    // 64 + 3 pair of narrow ones
    const int npairs_w = (p.Wo + 1) >> 1;
    if (npairs_w > 64) return launch_sfb_stream4<L, PK>(p, stream, (npairs_w + 127) / 128);
  }
  return launch_sfb_stream_m<L, false, PK>(p, stream);
}

template <bool PK>
inline int try_launch_sfb_layout(const SfbParams& p, cudaStream_t stream) {
  if (p.Lw != p.Lh) return kNoFastPath;
  if (p.planes == 0) return 0;
  switch (p.Lw) {
    case 2: return launch_sfb_stream<2, PK>(p, stream);
    case 4: return launch_sfb_stream<4, PK>(p, stream);
    case 6: return launch_sfb_stream<6, PK>(p, stream);
    case 8: return launch_sfb_stream<8, PK>(p, stream);
    case 10: return launch_sfb_stream<10, PK>(p, stream);
    case 12: return launch_sfb_stream<12, PK>(p, stream);
    case 14: return launch_sfb_stream<14, PK>(p, stream);
    case 16: return launch_sfb_stream<16, PK>(p, stream);
    case 18: return launch_sfb_stream<18, PK>(p, stream);
    case 20: return launch_sfb_stream<20, PK>(p, stream);
    default: return kNoFastPath;
  }
}



}  // namespace fast
}  // namespace b200w
