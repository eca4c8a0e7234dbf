// dtcwt_fwd12.cuh -- DTCWT forward levels 1 and 2 in one kernel (sm_90a), included from k_dtcwt_fwd.cu after
// dtcwt_fwd_stream.cuh, whose stage functions it runs: the full-resolution level-1 low-pass (LL1) never goes to HBM.
//
// One CTA owns one plane's band of rows across the full plane width (schedule and shared-memory layout:
// dtcwt_fwd12_plan.h).  Thread i owns two of j1_stage's column pairs at level 1 (columns 2i and W/2 + 2i, each pair
// with its own register window, so a warp reads and writes consecutive 8-byte words) and the complex column q = i at
// level 2, as a lane of fwd_j2plus_stream.  The CTA marches down its band one step of 4 input rows at a time:
//   phase A  two level-1 stages on input rows staged by cp.async in the input ring: yh0 to HBM (q2c_emit), the step's
//            group of 4 LL1 rows into the LL ring with level 2's mirrored halo columns, and, at the plane's top and
//            bottom edges, into the mirrored virtual group as well;
//   phase B  one level-2 stage on a group of the LL ring: LL2 and yh1 to HBM.
// CTA barriers separate the phases; there are no warp roles and no mbarriers.  Every output comes from the stage
// functions of the per-level kernels, with the same taps in the same order, so the two routes agree bit for bit.
#pragma once
#include "dtcwt_fwd12_plan.h"
#include "dtcwt_fwd_stream.cuh"
#include "launch.cuh"

namespace b200w {
namespace fast {

struct Fwd12Params {
  DtParams p1;         // level 1: in = x, highs = yh0, f0 / f1 = h0o / h1o, sym
  DtParams p2;         // level 2: out = LL2, highs = yh1 (or null), the q-shift taps
  Fwd12Plan pl;
  int CH, n_bands;     // LL2 quad rows per band, bands per plane
};

// one LL1 value pair (columns c, c + 1 of a ring row whose column 0 is at `row`) and its mirrored halo copies
__device__ __forceinline__ void fwd12_put(float* row, int c, int W, int HL, float v0, float v1) {
  *reinterpret_cast<float2*>(row + c) = make_float2(v0, v1);
  if (c < HL) { row[-1 - c] = v0; row[-2 - c] = v1; }                  // column -1 - k <- k
  if (c >= W - HL) { row[2 * W - 1 - c] = v0; row[2 * W - 2 - c] = v1; }  // column W + k <- W - 1 - k
}

template <int L0, int L1, int MQ>
__global__ void __launch_bounds__(kF12MaxThreads, 1) dtcwt_fwd12_band(const __grid_constant__ Fwd12Params P) {
  using C1 = J1Cfg<L0, L1>;
  using C2 = J2Cfg<MQ>;
  constexpr int M = C1::M, HLA1 = C1::HLA, HLA2 = C2::HLA, HL = C2::HL, NMG = HL / 4, NS1 = kF12InStages;
  constexpr int RING = 4 * NMG;
  static_assert(HL % 4 == 0, "level 2's mirrored rows must come in whole groups");
  static_assert(HLA1 == fwd12_hla1(L0, L1) && HLA2 == fwd12_hla2(MQ) && RING == fwd12_ring(MQ), "plan / kernel shape");
  extern __shared__ __align__(16) float smem[];
  const DtParams& p1 = P.p1;
  const DtParams& p2 = P.p2;
  const int tid = threadIdx.x;
  const int H = p1.H, W = p1.W, Hq = H >> 2, W2 = W >> 1, W4 = W >> 2;
  const int SW1 = P.pl.sw1, SW2 = P.pl.sw2;
  const int band = (int)(blockIdx.x % (unsigned)P.n_bands);
  const int plane = (int)(blockIdx.x / (unsigned)P.n_bands);
  const int n = plane / p1.C, ch = plane - n * p1.C;
  const Fwd12Band b = fwd12_band(band, P.CH, Hq, NMG);
  const bool active = tid < W4;
  float* const in_ring = smem;
  float* const ll_ring = smem + P.pl.ll_off;

  // ---- input ring: level-1 stage t = input rows r1 + 2t, r1 + 2t + 1, full width plus HLA1 pad columns per side
  const float* const xp = p1.in + (long long)plane * p1.inps;
  const int r1 = 4 * b.a0 - M;
  const int n1 = 2 * (b.a1 - b.a0) + M;
  if (!p1.sym) {   // zero padding: the pad columns are never copied to, so they stay zero
    for (int e = tid; e < NS1 * 2 * 2 * HLA1; e += blockDim.x) {
      const int row = e / (2 * HLA1), k = e - row * (2 * HLA1);
      in_ring[row * SW1 + (k < HLA1 ? k : W + k)] = 0.f;
    }
  }
  auto issue = [&](int t) {
    if (t < n1) {
      float* const dst = in_ring + (t % NS1) * 2 * SW1;
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        const int r = r1 + 2 * t + k;
        const int gr = sym_or_zero(r, H, p1.sym);
        float* const d = dst + k * SW1;
        if (gr < 0) {
          if (active) *reinterpret_cast<float4*>(d + HLA1 + 4 * tid) = make_float4(0.f, 0.f, 0.f, 0.f);
        } else {
          const float* const src = xp + (long long)gr * p1.inpitch;
          if (active) cp_async16(d + HLA1 + 4 * tid, src + 4 * tid);
          if (p1.sym && tid < 2 * HLA1) {   // symmetric pad columns: -1 - j <- j, W + j <- W - 1 - j
            if (tid < HLA1) cp_async4(d + HLA1 - 1 - tid, src + tid);
            else cp_async4(d + HLA1 + W + (tid - HLA1), src + W - 1 - (tid - HLA1));
          }
        }
      }
    }
    cp_async_commit();
  };
#pragma unroll 1
  for (int t = 0; t < NS1 - 1; ++t) issue(t);

  // ---- level 1: two column pairs per thread, register windows as in fwd_j1_stream
  float2 w0[C1::WR][2], w1[C1::WR][2];
#pragma unroll
  for (int j = 0; j < C1::WR; ++j) { w0[j][0] = w0[j][1] = w1[j][0] = w1[j][1] = make_float2(0.f, 0.f); }
  const int c0 = 2 * tid, c1 = W2 + 2 * tid;   // the pairs' first columns
  float* hq0 = p1.highs + n * p1.hs[0] + ch * p1.hs[1] + (long long)(2 * b.a0) * p1.hs[3] + (long long)tid * p1.hs[4];
  const long long hq0_pair1 = (long long)(W4) * p1.hs[4];
  const bool vec0 = (p1.hs[5] == 1) && ((p1.hs[4] & 1) == 0) && ((p1.hs[3] & 1) == 0) && ((p1.hs[2] & 1) == 0) &&
                    ((p1.hs[1] & 1) == 0) && ((p1.hs[0] & 1) == 0) && ((reinterpret_cast<uintptr_t>(p1.highs) & 7) == 0);

  // ---- level 2: one complex column per thread, register windows as in fwd_j2plus_stream
  float2 wl[C2::WR], wh[C2::WR];
#pragma unroll
  for (int j = 0; j < C2::WR; ++j) { wl[j] = wh[j] = make_float2(0.f, 0.f); }
  const bool want_hi = (p2.highs != nullptr);
  float* ll_ptr = p2.out + (long long)plane * p2.outps + (long long)(2 * b.qy0) * p2.outpitch + 2 * tid;
  float* hq1 = nullptr;
  bool vec1 = false;
  if (want_hi) {
    hq1 = p2.highs + n * p2.hs[0] + ch * p2.hs[1] + (long long)b.qy0 * p2.hs[3] + (long long)tid * p2.hs[4];
    vec1 = (p2.hs[5] == 1) && ((p2.hs[4] & 1) == 0) && ((p2.hs[3] & 1) == 0) && ((p2.hs[2] & 1) == 0) &&
           ((p2.hs[1] & 1) == 0) && ((p2.hs[0] & 1) == 0) && ((reinterpret_cast<uintptr_t>(p2.highs) & 7) == 0);
  }

  // one level-1 pair's outputs: yh0 (owned groups only) and the LL1 rows into the ring (+ mirrored virtual group)
  auto emit1 = [&](const J1Quads& v, int c, float* hq, int g, int rr) {
    if (g >= b.qy0 && g < b.qy1) {
      const long long so = p1.hs[2], sr = p1.hs[5];
      q2c_emit(v.vlh[0][0], v.vlh[0][1], v.vlh[1][0], v.vlh[1][1], hq, so, sr, vec0, 0, 5);  // lh -> 15, 165
      q2c_emit(v.vhh[0][0], v.vhh[0][1], v.vhh[1][0], v.vhh[1][1], hq, so, sr, vec0, 1, 4);  // hh -> 45, 135
      q2c_emit(v.vhl[0][0], v.vhl[0][1], v.vhl[1][0], v.vhl[1][1], hq, so, sr, vec0, 2, 3);  // hl -> 75, 105
    }
    float* const row = ll_ring + fwd12_slot(g, RING) * 4 * SW2 + rr * SW2 + HLA2;
    fwd12_put(row, c, W, HL, v.vll[0][0], v.vll[0][1]);
    fwd12_put(row + SW2, c, W, HL, v.vll[1][0], v.vll[1][1]);
    // rows 4g + rr + dr mirrored: virtual row -1 - r (top) / 2H - 1 - r (bottom) = row 3 - rr - dr of the mirror group
    const int vt = -1 - g, vb = 2 * Hq - 1 - g;
    if (g < NMG && vt >= b.g0) {
      float* const mrow = ll_ring + fwd12_slot(vt, RING) * 4 * SW2 + (3 - rr) * SW2 + HLA2;
      fwd12_put(mrow, c, W, HL, v.vll[0][0], v.vll[0][1]);
      fwd12_put(mrow - SW2, c, W, HL, v.vll[1][0], v.vll[1][1]);
    }
    if (g >= Hq - NMG && vb < b.g0 + b.n2) {
      float* const mrow = ll_ring + fwd12_slot(vb, RING) * 4 * SW2 + (3 - rr) * SW2 + HLA2;
      fwd12_put(mrow, c, W, HL, v.vll[0][0], v.vll[0][1]);
      fwd12_put(mrow - SW2, c, W, HL, v.vll[1][0], v.vll[1][1]);
    }
  };

  // ticks: one level-1 stage each (the first M fill the window); every second tick after those ends a step
  const int n_ticks = M + 2 * (b.lag + b.n2);
  int uu1 = 0, uu2 = 0;
#pragma unroll 1
  for (int t = 0; t < n_ticks; ++t) {
    if (t < n1) {   // phase A: level-1 stage t
      cp_async_wait<NS1 - 2>();
      __syncthreads();
      issue(t + NS1 - 1);
      const float* const st = in_ring + (t % NS1) * 2 * SW1;
      const bool emit = (t >= M);
      const int g = b.a0 + ((t - M) >> 1), rr = 2 * ((t - M) & 1);
      if (active) {
        J1Quads v;
        j1_dispatch<L0, L1, 0>(uu1, p1, st + c0, w0, emit, v, SW1);
        if (emit) emit1(v, c0, hq0, g, rr);
        j1_dispatch<L0, L1, 0>(uu1, p1, st + c1, w1, emit, v, SW1);
        if (emit) emit1(v, c1, hq0 + hq0_pair1, g, rr);
      }
      if (emit) hq0 += p1.hs[3];
      uu1 = (uu1 + 1 == C1::UNR) ? 0 : uu1 + 1;
    }
    if (t >= M && ((t - M) & 1)) {   // end of step s: phase B, level-2 stage s - lag
      const int s = (t - M) >> 1;
      __syncthreads();
      if (s >= b.lag) {
        const int t2 = s - b.lag;
        const float* const st2 = ll_ring + fwd12_slot(b.g0 + t2, RING) * 4 * SW2 + 4 * tid;
        if (active) j2_dispatch<MQ, 0>(uu2, p2, st2, wl, wh, t2 >= C2::PRO, want_hi, ll_ptr, hq1, true, vec1, SW2);
        uu2 = (uu2 + 1 == C2::UNR) ? 0 : uu2 + 1;
      }
    }
  }
  cp_async_wait<0>();
}

// CTAs of one kernel shape resident on the current device (occupancy query, cached per device / threads / bytes)
template <class K>
inline int fwd12_resident_ctas(K kernel, int threads, int smem_bytes) {
  struct Entry { int dev, threads, smem, ctas; };
  static Entry cache[16];
  static int n_cache = 0;
  int dev = 0, sms = 132, per_sm = 0;
  (void)cudaGetDevice(&dev);
  for (int i = 0; i < n_cache; ++i)
    if (cache[i].dev == dev && cache[i].threads == threads && cache[i].smem == smem_bytes) return cache[i].ctas;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, smem_bytes) != cudaSuccess || per_sm < 1) {
    (void)cudaGetLastError();
    per_sm = 1;
  }
  (void)cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int ctas = per_sm * sms;
  if (n_cache < 16) cache[n_cache++] = Entry{dev, threads, smem_bytes, ctas};
  return ctas;
}

template <int L0, int L1, int MQ>
inline int launch_fwd12(Fwd12Params& P, cudaStream_t stream) {
  auto kernel = dtcwt_fwd12_band<L0, L1, MQ>;
  static bool smem_set[64] = {};
  int dev = 0;
  (void)cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64 || !smem_set[dev]) {
    const int rc = check_cuda(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kF12MaxSmem));
    if (rc) return rc;
    if (dev >= 0 && dev < 64) smem_set[dev] = true;
  }
  const long long planes = (long long)P.p1.N * P.p1.C;
  const int nmg = fwd12_nmg(MQ);
  // every band recomputes 2 * NMG groups of level 1 and fills the level-1 window (M rows): its overhead in steps
  pick_chunks(planes, P.p1.H >> 2, 2 * nmg, 2 * nmg + (fwd12_m(L0, L1) + 1) / 2,
              fwd12_resident_ctas(kernel, P.pl.threads, P.pl.smem_bytes), &P.n_bands, &P.CH);
  const long long blocks = planes * P.n_bands;
  if (blocks <= 0) return 0;
  if (blocks > 2147483647LL) return kNoFastPath;
  kernel<<<(unsigned)blocks, P.pl.threads, P.pl.smem_bytes, stream>>>(P);
  return 0;
}

int try_launch_fwd12(const DtParams& p1, const DtParams& p2, cudaStream_t stream) {
  Fwd12Params P;
  if (fwd12_route(P.pl, p1.in, p1.inps, p1.inpitch, p1.H, p1.W, p1.L0, p1.L1, p2.L0, p1.highs != nullptr))
    return kNoFastPath;
  if ((long long)p1.N * p1.C == 0) return 0;
  P.p1 = p1;
  P.p2 = p2;
  if (p1.L0 == 5 && p1.L1 == 7 && p2.L0 == 10) return launch_fwd12<5, 7, 10>(P, stream);   // near_sym_a + qshift_a
  return kNoFastPath;
}

}  // namespace fast
}  // namespace b200w
