// afb_stream_kernel.cuh -- the streaming DWT analysis kernel (K1), included twice by afb_stream.cuh (deliberately no
// include guard): as afb2d_stream with B200W_PK 0 (the DWT layout: ll, then the three band-pass planes of plane p at
// highs + (3p + b) * Ho * hipitch) and as wpt_afb2d_stream with B200W_PK 1 (the wavelet-packet layout: child b of plane
// p at ll + (4p + b) * llps / 4, highs = ll + llps / 4, rows hipitch apart).  One source, two kernels with their own
// names, and the DWT kernel's code is exactly what it was before the packet layout existed.
// strip0 / n_strips: the 64-column strips this launch covers (PW == 32), or the single remainder strip
// starting at output column k_rem (PW < 32, n_strips == 1).
template <int L, int PW, int MINB, int HSM, int XM>
__global__ void __launch_bounds__(32, (MINB > 1 ? MINB : 0)) B200W_AFB_KERNEL(const __grid_constant__ AfbParams p, int n_strips, int n_chunks,
                                                   int CH, int k_rem, int swid) {
  using C = AfbCfg<L, PW, HSM, XM>;
  extern __shared__ __align__(16) float ring[];  // this warp's staging ring
  const int lane = threadIdx.x;
  long long item = blockIdx.x;                    // one warp per CTA: no intra-CTA load imbalance
  const int strip = (int)(item % n_strips);
  item /= n_strips;
  const int chunk = (int)(item % n_chunks);
  const int pgroup = (int)(item / n_chunks);
  const int g = lane / PW, jp = lane % PW;        // plane within the group, column pair within the plane
  const int plane0 = pgroup * C::G;
  const int nplanes = imin(C::G, p.planes - plane0);
  const int plane = plane0 + g;

  // swid = output columns per strip (even, <= 64)
  const int k0 = (PW == 32) ? strip * swid : k_rem;
  const int ky0 = chunk * CH;
  const int ky1 = imin(ky0 + CH, p.Ho);
  const int n_half = (ky1 - ky0) + C::PRO;             // half-stages: PRO of warm-up, then one output row each
  const int n_stage = (n_half + C::HS - 1) / C::HS;
  const int nvalid = imin((PW == 32) ? swid : 2 * PW, p.Wo - k0);

  const int sh = (XM == 0 && PW == 32) ? widen_left(2 * k0 - C::HLA, C::HLA + 2 * nvalid + C::RH, p.W, p.mode,
                                                         C::SW - 4 * C::NV - 4 * ((nvalid + 1) / 2 - 1)) : 0;
  typename C::Loader ld;
  ld.init(ring, p.x + (long long)plane0 * p.xps, p.xps, nplanes, p.H, p.W, p.xpitch, p.mode, 2 * k0 - C::HLA - sh,
          C::HLA + 2 * nvalid + C::RH + sh, 2 * ky0 - C::PL, n_stage, lane);
  ld.prologue();

  float2 w[L][2];
#pragma unroll
  for (int j = 0; j < L; ++j) { w[j][0] = w[j][1] = make_float2(0.f, 0.f); }

  DirectOut out;
  const int hipitch = p.hipitch > 0 ? p.hipitch : p.Wo;
#if B200W_PK
  out.band = p.llps >> 2;
#else
  out.band = (long long)p.Ho * hipitch;
#endif
  out.ll_ptr = p.ll + (long long)plane * p.llps + (long long)ky0 * p.llpitch + k0 + 2 * jp;
#if B200W_PK
  out.hi_ptr = p.highs + (long long)plane * p.llps + (long long)ky0 * hipitch + k0 + 2 * jp;
#else
  out.hi_ptr = p.highs + (long long)plane * 3 * out.band + (long long)ky0 * hipitch + k0 + 2 * jp;
#endif
  out.nv = (g < nplanes) ? imax(0, imin(2, k0 + nvalid - (k0 + 2 * jp))) : 0;
  out.llpitch = p.llpitch;
  out.Wo = hipitch;
  out.init_parity();
  const int lane_off = g * (C::RPS * C::SW) + ((sh > 0 && out.nv == 0) ? 0 : 4 * jp + sh);

  int vv = 0;
#pragma unroll 1
  for (int t = 0; t < n_stage; ++t) {
    const float* stage = ld.acquire(t);
    ld.issue(t + C::NS - 1);
    afb_stage_dispatch<L, PW, HSM, XM, 0>(vv, p, stage + lane_off, w, C::HS * t, n_half, out);
    vv = (vv + 1 == C::UNS) ? 0 : vv + 1;
  }
  cp_async_wait<0>();
}

