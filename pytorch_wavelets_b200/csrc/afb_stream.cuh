// afb_stream.cuh -- streaming DWT analysis level (K1); see stream_common.cuh for the design notes.
#pragma once
#include "stream_common.cuh"

namespace b200w {
namespace fast {

// ================================================================================================
// K1 fast: DWT analysis level, Lw == Lh == L (even), modes zero / symmetric / reflect / periodic.
//   strip = 64 output columns per warp (2 per lane) = 128 input columns + (L-2) halo;
//   stage = 2 input rows = 1 output row.
// ================================================================================================
// XM: 0 = zero / symmetric / reflect (border sources inside the strip), 1 = periodic, 2 = periodization
// (wrap-around modes: border columns come from the other end of the row, fetched with the stage)
template <int L, int PW = 32, int HSM = 2, int XM = 0>
struct AfbCfg {
  static constexpr bool PER = (XM == 2);
  // PW = column pairs per plane handled by one warp: 32 -> the warp owns one 64-column strip of one plane;
  // PW < 32 -> a narrow remainder strip, the warp's lanes are split over G = 32/PW planes.
  static constexpr int G = 32 / PW;
  // out[k] = sum_j f[j] xe[2k + j - PL]: PL = L-2, or L/2-1 for periodization (reference afb1d :134-154)
  static constexpr int PL = PER ? (L - 1 - L / 2) : (L - 2);
  static constexpr int HLA = (PL + 3) / 4 * 4;       // left halo rounded up to 16 bytes
  static constexpr int OFF = HLA - PL;               // lane window offset inside its aligned read
  static constexpr int NX = OFF + L + 2;             // floats a lane needs per row
  static constexpr int NV = (NX + 3) / 4;            // ... as 128-bit loads
  static constexpr int SW = 4 * (PW - 1) + 4 * NV;   // staged floats per row (per plane)
  static constexpr int RH = L - 2 - PL;              // columns needed right of the last output's 2k+1
  // half-stages (2 input rows = 1 output row) per stage: the largest of 4, 2, 1 dividing the window period
  static constexpr int HS0 = ((L / 2) % 4 == 0) ? 4 : (((L / 2) % 2 == 0) ? 2 : 1);
  static constexpr int HS = (HS0 < HSM) ? HS0 : HSM;
  static constexpr int RPS = 2 * HS;                 // image rows per stage
#ifndef B200W_AFB_NS
#define B200W_AFB_NS 4   /* 2: -4.5 %, 3 -> 4: +0.4..0.8 % (levels 2/3 of configs[1], configs[4]) */
#endif
  static constexpr int NS = (HS == 4) ? 2 : ((HS == 2) ? B200W_AFB_NS : 4);  // ring depth in stages
  static constexpr int NFIX = (PW == 32) ? (RPS * 2 * (HLA + L) + 31) / 32 : 8;  // border fix-ups per lane per stage
  static constexpr int SMEM_BYTES = NS * RPS * G * SW * 4;
  static constexpr int PRO = (L - 2) / 2;            // prologue half-stages before the first output row
  static constexpr int UNR = L / 2;                  // window period in half-stages
  static constexpr int UNS = UNR / HS;               // ... in stages: copies of the stage body
  using Loader = StripLoader<RPS * G, SW, NS, NFIX, RPS, (XM != 0)>;
};

// ---- where a finished output row goes -------------------------------------------------------------------------
// DirectOut: straight from registers to global memory (each lane stores its two adjacent columns of each band).
struct DirectOut {
  float* ll_ptr; float* hi_ptr; long long band; int llpitch, Wo, nv;
  // Rows of the reference's contiguous outputs start at any 4-byte phase (Wo = 259: every other row is 8-byte
  // misaligned).  `par` bit b = this row of plane b (0 = ll, 1..3 = the band-pass planes) is misaligned; the value is
  // the same in every lane (lanes are 8 bytes apart), and it flips with `flip` from row to row.  One bit test per
  // store replaces an address test + divergence bookkeeping around each of them.
  unsigned par, flip;
  __device__ __forceinline__ void init_parity() {
    par = (unsigned)((reinterpret_cast<uintptr_t>(ll_ptr) >> 2) & 1) |
          (unsigned)((reinterpret_cast<uintptr_t>(hi_ptr) >> 2) & 1) << 1 |
          (unsigned)((reinterpret_cast<uintptr_t>(hi_ptr + band) >> 2) & 1) << 2 |
          (unsigned)((reinterpret_cast<uintptr_t>(hi_ptr + 2 * band) >> 2) & 1) << 3;
    flip = (unsigned)(llpitch & 1) | ((Wo & 1) ? 14u : 0u);
  }
  __device__ __forceinline__ void pair(float* ptr, float v0, float v1, unsigned odd, bool stream) {
    stream = stream && (B200W_STREAM_STORES != 0);
    if (!odd) {
      if (stream) __stcs(reinterpret_cast<float2*>(ptr), make_float2(v0, v1));
      else *reinterpret_cast<float2*>(ptr) = make_float2(v0, v1);
    } else {
      if (stream) { __stcs(ptr, v0); __stcs(ptr + 1, v1); }
      else { ptr[0] = v0; ptr[1] = v1; }
    }
  }
  __device__ __forceinline__ void row(float2 lo0, float2 lo1, float2 hi0, float2 hi1) {
    // {column low-pass of (l, h)} = {ll, band 1}; {column high-pass} = {band 0, band 2}   (reference order lh, hl, hh)
    if (nv == 2) {
      pair(ll_ptr, lo0.x, lo1.x, par & 1u, false);
      pair(hi_ptr, hi0.x, hi1.x, par & 2u, true);
      pair(hi_ptr + band, lo0.y, lo1.y, par & 4u, true);
      pair(hi_ptr + 2 * band, hi0.y, hi1.y, par & 8u, true);
    } else if (nv == 1) {   // the last column of an odd-width plane
      ll_ptr[0] = lo0.x;
      hi_ptr[0] = hi0.x;
      hi_ptr[band] = lo0.y;
      hi_ptr[2 * band] = hi0.y;
    }
    par ^= flip;
    ll_ptr += llpitch;
    hi_ptr += Wo;
  }
};

// one half-stage of compute: row pass on the two staged rows into window slots (2U, 2U+1) mod L, then (if emit)
// the column pass reading tap j from slot (2U+2+j) mod L, and the output row.  U is the position inside the
// window period, so every window index is a compile-time constant: the window never moves.
template <int L, int PW, int HSM, int XM, int U, class Out>
__device__ __forceinline__ void afb_stage(const AfbParams& p, const float* s0, float2 (&w)[L][2], bool emit, Out& out) {
  using C = AfbCfg<L, PW, HSM, XM>;
  float xa[4 * C::NV], xb[4 * C::NV];
#pragma unroll
  for (int q = 0; q < C::NV; ++q) {
    const float4 a = *reinterpret_cast<const float4*>(s0 + 4 * q);
    const float4 b = *reinterpret_cast<const float4*>(s0 + C::SW + 4 * q);
    xa[4 * q] = a.x; xa[4 * q + 1] = a.y; xa[4 * q + 2] = a.z; xa[4 * q + 3] = a.w;
    xb[4 * q] = b.x; xb[4 * q + 1] = b.y; xb[4 * q + 2] = b.z; xb[4 * q + 3] = b.w;
  }
  // window entries are {row-lowpass, row-highpass} pairs: one packed FMA per tap feeds both
  constexpr int SA = (2 * U) % L, SB = (2 * U + 1) % L;
#pragma unroll
  for (int o = 0; o < 2; ++o) {
    float2 ra = make_float2(0.f, 0.f), rb = make_float2(0.f, 0.f);
#pragma unroll
    for (int j = 0; j < L; ++j) {
      const float2 f = make_float2(p.fwp[2 * j], p.fwp[2 * j + 1]);
      ra = ffma2_s(xa[C::OFF + 2 * o + j], f, ra);
      rb = ffma2_s(xb[C::OFF + 2 * o + j], f, rb);
    }
    w[SA][o] = ra;
    w[SB][o] = rb;
  }
  if (emit) {
    float2 lo[2], hi[2];  // column low-pass of {l, h} -> {ll, hl}; column high-pass -> {lh, hh}
#pragma unroll
    for (int o = 0; o < 2; ++o) {
      float2 a0 = make_float2(0.f, 0.f), a1 = make_float2(0.f, 0.f);
#pragma unroll
      for (int j = 0; j < L; ++j) {
        constexpr int base = 2 * U + 2;
        a0 = ffma2_s(p.fh_lo.t[j], w[(base + j) % L][o], a0);
        a1 = ffma2_s(p.fh_hi.t[j], w[(base + j) % L][o], a1);
      }
      lo[o] = a0; hi[o] = a1;
    }
    out.row(lo[0], lo[1], hi[0], hi[1]);
  }
}

template <int L, int PW, int HSM, int XM, int V, class Out>
__device__ __forceinline__ void afb_stage_dispatch(int vv, const AfbParams& p, const float* s0, float2 (&w)[L][2],
                                                   int h0, int h_emit_end, Out& out) {
  using C = AfbCfg<L, PW, HSM, XM>;
  if constexpr (V < C::UNS) {
    if (vv == V) {
      // h0 = index of this stage's first half-stage; output rows are emitted for PRO <= h < h_emit_end
      afb_stage<L, PW, HSM, XM, C::HS * V>(p, s0, w, h0 >= C::PRO && h0 < h_emit_end, out);
      if constexpr (C::HS >= 2)
        afb_stage<L, PW, HSM, XM, C::HS * V + 1>(p, s0 + 2 * C::SW, w, h0 + 1 >= C::PRO && h0 + 1 < h_emit_end, out);
      if constexpr (C::HS == 4) {
        afb_stage<L, PW, HSM, XM, C::HS * V + 2>(p, s0 + 4 * C::SW, w, h0 + 2 >= C::PRO && h0 + 2 < h_emit_end, out);
        afb_stage<L, PW, HSM, XM, C::HS * V + 3>(p, s0 + 6 * C::SW, w, h0 + 3 >= C::PRO && h0 + 3 < h_emit_end, out);
      }
    } else {
      afb_stage_dispatch<L, PW, HSM, XM, V + 1>(vv, p, s0, w, h0, h_emit_end, out);
    }
  }
}

#define B200W_AFB_KERNEL afb2d_stream
#define B200W_PK 0
#include "afb_stream_kernel.cuh"
#undef B200W_AFB_KERNEL
#undef B200W_PK
#define B200W_AFB_KERNEL wpt_afb2d_stream
#define B200W_PK 1
#include "afb_stream_kernel.cuh"
#undef B200W_AFB_KERNEL
#undef B200W_PK

template <int L, int PW, int MINB, int HSM, bool PK>
constexpr auto afb_kernel_of() {
  if constexpr (PK) return wpt_afb2d_stream<L, PW, MINB, HSM, 0>;
  else return afb2d_stream<L, PW, MINB, HSM, 0>;
}

template <int L, int PW, int MINB, int HSM, int XM = 0, bool PK = false>
inline void launch_afb_kernel(const AfbParams& p, cudaStream_t stream, long long blocks, int n_strips, int n_chunks,
                              int CH, int k_rem) {
  using C = AfbCfg<L, PW, HSM, XM>;
  // strips are 64 columns wide; splitting the columns evenly over the strips instead (g_tune_balanced) gives more row
  // segments that straddle 128-byte lines
  const int swid = 64;
  if constexpr (PK)
    wpt_afb2d_stream<L, PW, MINB, HSM, XM><<<(unsigned)blocks, 32, C::SMEM_BYTES, stream>>>(p, n_strips, n_chunks, CH, k_rem, swid);
  else
    afb2d_stream<L, PW, MINB, HSM, XM><<<(unsigned)blocks, 32, C::SMEM_BYTES, stream>>>(p, n_strips, n_chunks, CH, k_rem, swid);
}

#ifndef B200W_AFB_SHORT_MINB
#define B200W_AFB_SHORT_MINB 1
#endif
#ifndef B200W_AFB_LONG_MINB
#define B200W_AFB_LONG_MINB 12  /* resident one-warp CTAs per SM the >= 14-tap instantiations are compiled for
                                  * (a register cap that does not spill; 16 spills) */
#endif
template <int L, int PW, bool PK = false>
inline int launch_afb_part(const AfbParams& p, cudaStream_t stream, int n_strips, int k_rem) {
  constexpr int G = 32 / PW;
  const long long groups = ((long long)p.planes + G - 1) / G;
  int n_chunks, CH;
  static ConcCache conc_cache;
  const int conc = resident_warps_dev(conc_cache, afb_kernel_of<L, PW, (L >= 14 ? B200W_AFB_LONG_MINB : B200W_AFB_SHORT_MINB), 2, PK>(),
                                      AfbCfg<L, PW, 2, 0>::SMEM_BYTES);
  pick_chunks(groups * n_strips, p.Ho, 16, (L - 2) / 2 + 8, conc, &n_chunks, &CH);
  const long long blocks = groups * n_strips * n_chunks;
  if (blocks <= 0) return 0;
  if (blocks > 2147483647LL) return B200W_ESIZE;
  if (p.mode == B200W_MODE_PERIODIZATION) {
    launch_afb_kernel<L, PW, 1, 2, 2, PK>(p, stream, blocks, n_strips, n_chunks, CH, k_rem);
    return 0;
  }
  if (p.mode == B200W_MODE_PERIODIC) {
    launch_afb_kernel<L, PW, 1, 2, 1, PK>(p, stream, blocks, n_strips, n_chunks, CH, k_rem);
    return 0;
  }
  // tried and not kept: register caps (__launch_bounds__(32, 18..32): faster on the small levels only, slower on the
  // large one) and 8-row stages
  launch_afb_kernel<L, PW, (L >= 14 ? B200W_AFB_LONG_MINB : B200W_AFB_SHORT_MINB), 2, 0, PK>(p, stream, blocks, n_strips, n_chunks, CH, k_rem);
  return 0;
}

template <int L, bool PK = false>
inline int launch_afb_stream(const AfbParams& p, cudaStream_t stream) {
  // aligned 16-byte staging needs an aligned source; anything else takes the generic kernel
  if (!aligned_plane(p.x, p.xps, p.xpitch)) return kNoFastPath;
  // Every 64-column strip (including a narrow last one) is an ordinary warp item: the kernel is
  // latency/occupancy-bound, not issue-bound, so a mostly-idle last strip costs almost nothing, while packing it
  // across planes (AfbCfg<L, PW<32>, kept for reference) needs a second launch that costs more than it saves.
  const int n_strips = (p.Wo + 63) / 64;
  return launch_afb_part<L, 32, PK>(p, stream, n_strips, 0);
}

template <bool PK>
inline int try_launch_afb_layout(const AfbParams& p, cudaStream_t stream) {
  if (p.Lw != p.Lh) return kNoFastPath;
  if (p.planes == 0) return 0;
  switch (p.Lw) {
    case 2: return launch_afb_stream<2, PK>(p, stream);
    case 4: return launch_afb_stream<4, PK>(p, stream);
    case 6: return launch_afb_stream<6, PK>(p, stream);
    case 8: return launch_afb_stream<8, PK>(p, stream);
    case 10: return launch_afb_stream<10, PK>(p, stream);
    case 12: return launch_afb_stream<12, PK>(p, stream);
    case 14: return launch_afb_stream<14, PK>(p, stream);
    case 16: return launch_afb_stream<16, PK>(p, stream);
    case 18: return launch_afb_stream<18, PK>(p, stream);
    case 20: return launch_afb_stream<20, PK>(p, stream);
    default: return kNoFastPath;
  }
}


}  // namespace fast
}  // namespace b200w
