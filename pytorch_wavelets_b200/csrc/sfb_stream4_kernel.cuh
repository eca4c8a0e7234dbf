// sfb_stream4_kernel.cuh -- the wide streaming DWT synthesis kernel (4 columns per lane), included twice by
// sfb_stream.cuh (deliberately no include guard), as sfb2d_stream4 and wpt_sfb2d_stream4; see sfb_stream_kernel.cuh.
template <int L>
__global__ void __launch_bounds__(32) B200W_SFB4_KERNEL(const __grid_constant__ SfbParams p, int n_strips, int n_chunks,
                                                    int CH /* output row pairs per chunk */) {
  using C = Sfb4Cfg<L>;
  extern __shared__ __align__(16) float ring[];
  const int lane = threadIdx.x;
  long long item = blockIdx.x;
  const int strip = (int)(item % n_strips);
  item /= n_strips;
  const int chunk = (int)(item % n_chunks);
  const int plane = (int)(item / n_chunks);

  const int c0 = strip * C::CW;                    // first coefficient column (= output column pair) of the strip
  const int npairs_h = (p.Ho + 1) >> 1;
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
  // the 32-lane column copies of a band row: coefficient columns c0 + lane + 32 j
  unsigned okmask = 0;
#pragma unroll
  for (int j = 0; j < C::NCOPY; ++j)
    if ((lane + 32 * j < C::CW + C::HALF - 1) && (c0 + lane + 32 * j < p.Wc)) okmask |= 1u << j;

  const unsigned ring_s = (unsigned)__cvta_generic_to_shared(ring) + 4 * lane;
  int slot_i = 0;
  auto issue = [&](int t) {
    const int slot = slot_i;
    slot_i = (slot_i + 1 == C::NS) ? 0 : slot_i + 1;
    if (t < n_stage) {
      const unsigned dst = ring_s + slot * (C::STAGE * 4);
#pragma unroll
      for (int r = 0; r < C::KR; ++r) {
        const int k = m0 + C::KR * t + r;
        if ((C::KR * t + r < n_rows) && (k < p.Hc)) {
#pragma unroll
          for (int b = 0; b < 4; ++b) {
            if (bptr[b] == nullptr) continue;
            const float* src = bptr[b] + (long long)k * bpitch[b] + c0 + lane;
            const unsigned d = dst + (r * 4 + b) * (C::SWB * 4);
#pragma unroll
            for (int j = 0; j < C::NCOPY; ++j)
              if (okmask & (1u << j)) cp_async4_s(d + 128 * j, src + 32 * j);
          }
        }
      }
    }
    cp_async_commit();
  };
#pragma unroll 1
  for (int t = 0; t < C::NS - 1; ++t) issue(t);

  float2 wP[C::HALF][4], wQ[C::HALF][4];
#pragma unroll
  for (int j = 0; j < C::HALF; ++j)
#pragma unroll
    for (int c = 0; c < 4; ++c) { wP[j][c] = make_float2(0.f, 0.f); wQ[j][c] = make_float2(0.f, 0.f); }

  const int col0 = 2 * c0 + 8 * lane;
  float* y_ptr = p.y + (long long)plane * p.yps + (long long)(2 * m0) * p.ypitch + col0;
  const int nv8 = imax(0, imin(8, p.Wo - col0));

  int vv = 0, slot_a = 0;
#pragma unroll 1
  for (int t = 0; t < n_stage; ++t) {
    cp_async_wait<C::NS - 2>();
    __syncwarp();
    issue(t + C::NS - 1);
    const float* stage = ring + slot_a * C::STAGE + 4 * lane;
    slot_a = (slot_a + 1 == C::NS) ? 0 : slot_a + 1;
    sfb4_stage_dispatch<L, 0>(vv, p, stage, wP, wQ, C::KR * t, n_rows, m0, y_ptr, p.ypitch, nv8);
    vv = (vv + 1 == C::UNS) ? 0 : vv + 1;
  }
  cp_async_wait<0>();
}
