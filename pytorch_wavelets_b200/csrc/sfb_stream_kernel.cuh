// sfb_stream_kernel.cuh -- the streaming DWT synthesis kernel (2 columns per lane), included twice by sfb_stream.cuh
// (deliberately no include guard): as sfb2d_stream with B200W_SFB_PLANE_BANDS 3 (the DWT layout: the three band-pass
// planes of plane p at highs + (3p + b) * Hc * Wc) and as wpt_sfb2d_stream with B200W_SFB_PLANE_BANDS 4 (the
// wavelet-packet layout: the children of plane p are planes 4p .. 4p+3 of one contiguous (4P, Hc, Wc) tensor, ll = its
// base with llps = 4 Hc Wc, highs = ll + Hc Wc).  One source, two kernels with their own names, and the DWT kernel's
// code is exactly what it was before the packet layout existed.
template <int L, bool PER = false>
__global__ void __launch_bounds__(32) B200W_SFB_KERNEL(const __grid_constant__ SfbParams p, int n_strips, int n_chunks,
                                                   int CH /* output row pairs per chunk */) {
  using C = SfbCfg<L>;
  extern __shared__ __align__(16) float ring[];
  const int lane = threadIdx.x;
  long long item = blockIdx.x;
  const int strip = (int)(item % n_strips);
  item /= n_strips;
  const int chunk = (int)(item % n_chunks);
  const int plane = (int)(item / n_chunks);

  const int c0 = strip * 64;                       // first coefficient column (= pair index) of the strip
  const int npairs_h = PER ? p.Hc : (p.Ho + 1) >> 1;
  const int m0 = chunk * CH;
  const int m1 = imin(m0 + CH, npairs_h);
  const int n_rows = (m1 - m0) + C::HALF - 1;      // coefficient rows m0 .. m1-1+HALF-1
  const int n_stage = (n_rows + C::KR - 1) / C::KR;

  // zero the ring once: positions that are never copied (columns beyond Wc, absent band-passes) must read 0
  for (int i = lane; i < C::NS * C::STAGE; i += 32) ring[i] = 0.f;
  __syncwarp();

  const long long band = (long long)p.Hc * p.Wc;
  const float* bptr[4];
  int bpitch[4];
  bptr[0] = p.ll + (long long)plane * p.llps;
  bpitch[0] = p.llpitch;
#pragma unroll
  for (int b = 1; b < 4; ++b) {
    bptr[b] = p.highs ? p.highs + ((long long)plane * B200W_SFB_PLANE_BANDS + (b - 1)) * band : nullptr;
    bpitch[b] = p.Wc;
  }
  // the three 32-lane column copies of a band row: coefficient columns c0 + lane + {0, 32, 64}; PER wraps them
  int colw[3];
  bool okc[3];
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    const int cidx = c0 + lane + 32 * j;
    const bool in_lanes = (j < 2) || (lane < C::HALF - 1);
    okc[j] = in_lanes && (PER ? (cidx < p.Wc + C::HALF - 1) : (cidx < p.Wc));
    colw[j] = PER ? cidx % p.Wc : cidx;
  }

  const unsigned ring_s = (unsigned)__cvta_generic_to_shared(ring) + 4 * lane;
  int slot_i = 0;
  auto issue = [&](int t) {
    const int slot = slot_i;
    slot_i = (slot_i + 1 == C::NS) ? 0 : slot_i + 1;
    if (t < n_stage) {
      const unsigned dst = ring_s + slot * (C::STAGE * 4);
#pragma unroll
      for (int r = 0; r < C::KR; ++r) {
        int k = m0 + C::KR * t + r;
        bool row_ok = (C::KR * t + r < n_rows);
        if (PER) k %= p.Hc; else row_ok = row_ok && (k < p.Hc);
        if (row_ok) {
#pragma unroll
          for (int b = 0; b < 4; ++b) {
            if (bptr[b] == nullptr) continue;
            const float* src = bptr[b] + (long long)k * bpitch[b];
            const unsigned d = dst + (r * 4 + b) * (C::SWB * 4);
            if (okc[0]) cp_async4_s(d, src + colw[0]);
            if (okc[1]) cp_async4_s(d + 128, src + colw[1]);
            if (okc[2]) cp_async4_s(d + 256, src + colw[2]);
          }
        }
      }
    }
    cp_async_commit();
  };
#pragma unroll 1
  for (int t = 0; t < C::NS - 1; ++t) issue(t);

  float2 wP[C::HALF][2], wQ[C::HALF][2];
#pragma unroll
  for (int j = 0; j < C::HALF; ++j)
#pragma unroll
    for (int c = 0; c < 2; ++c) { wP[j][c] = make_float2(0.f, 0.f); wQ[j][c] = make_float2(0.f, 0.f); }

  const int col0 = 2 * c0 + 4 * lane;
  float* y_ptr = PER ? p.y + (long long)plane * p.yps
                     : p.y + (long long)plane * p.yps + (long long)(2 * m0) * p.ypitch + col0;
  const int nv4 = imax(0, imin(4, p.Wo - col0));
  int ncol[4] = {-1, -1, -1, -1};
  if (PER) {
    const int N = 2 * p.Wc;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int c = (col0 + q + C::HALF - 1) % N;
      ncol[q] = (col0 + q < N && c < p.Wo) ? c : -1;
    }
  }

  int vv = 0, slot_a = 0;
#pragma unroll 1
  for (int t = 0; t < n_stage; ++t) {
    cp_async_wait<C::NS - 2>();
    __syncwarp();
    issue(t + C::NS - 1);
    const float* stage = ring + slot_a * C::STAGE + 2 * lane;
    slot_a = (slot_a + 1 == C::NS) ? 0 : slot_a + 1;
    sfb_stage_dispatch<L, 0, PER>(vv, p, stage, wP, wQ, C::KR * t, n_rows, m0, y_ptr, p.ypitch, nv4, ncol);
    vv = (vv + 1 == C::UNS) ? 0 : vv + 1;
  }
  cp_async_wait<0>();
}
