// dtcwt_fwd12_plan.h -- host-side plan (and the schedule rules shared with the device code) of the fused DTCWT
// forward levels 1 + 2 kernel (dtcwt_fwd12.cuh): one launch computes yh0, yh1 and LL2, and the full-resolution
// level-1 low-pass (LL1) lives only in shared memory.
//
// One CTA owns one plane's band of LL2 quad rows across the full plane width.  Rows are handed from level 1 to level 2
// in GROUPS of 4 LL1 rows: group g = LL1 rows [4g, 4g + 4) = the rows one level-2 stage reads, and the level-1 output of
// one step of 4 input rows.  Level 2's symmetric extension reaches HL = MQ - 2 rows past each plane edge, i.e.
// NMG = HL / 4 whole groups (MQ % 4 == 2): "virtual" group -1 - g is group g mirrored, and so is 2*Hq - 1 - g at the
// bottom (Hq = H / 4 groups).  Level 1 writes those mirrored copies into the LL ring as it produces the real group.
//
// Band schedule (band = LL2 quad rows [qy0, qy1)):
//   level 2 consumes virtual groups g0 = qy0 - NMG ... g0 + n2 - 1, n2 = (qy1 - qy0) + 2*NMG (its stage prologue);
//   level 1 produces real groups a0 = max(0, g0) ... a1 - 1, a1 = min(Hq, qy1 + NMG), and emits yh0 only for the
//   groups the band owns (qy0 ... qy1 - 1; the others are the band's halo, recomputed by the neighbouring band);
//   step s produces group a0 + s (while any are left) and then consumes virtual group g0 + s - lag (once s >= lag):
//   a top band first needs group NMG - 1 (the mirror of its first virtual group), so it lags by NMG - 1 steps.
// A virtual group occupies ring slot (v mod ring) from the step that produces its source to the step that consumes it.
// The widest span of live groups is a top band that also reaches the bottom edge: producing group Hq - NMG writes its
// mirror Hq + NMG - 1 while level 2, NMG - 1 steps behind, still needs group Hq - 3*NMG + 1, i.e. 4*NMG - 1 groups, so
// ring = 4*NMG; planes of fewer than 3*NMG groups would also keep top mirrors alive then and run the level kernels
// instead (tests/test_dtcwt_fwd12_plan.py replays every band of many (H, band height) pairs).
#pragma once
#include <stdint.h>

#include "common.h"

namespace b200w {

constexpr int kF12MaxThreads = 256;     // one thread per 4 columns: planes up to 1024 columns wide
constexpr int kF12InStages = 8;         // input-ring slots (one level-1 stage = 2 input rows each): 7 stages in flight
constexpr int kF12MaxSmem = 227 * 1024;

// the (level-1, q-shift) filter lengths compiled into the fused kernel: near_sym_a with qshift_a / qshift_06
constexpr bool fwd12_pair_compiled(int L0, int L1, int MQ) { return L0 == 5 && L1 == 7 && MQ == 10; }

constexpr int fwd12_m(int L0, int L1) { return (L0 > L1 ? L0 : L1) / 2; }   // level-1 half filter length (J1Cfg::M)
constexpr int fwd12_hla1(int L0, int L1) { return (fwd12_m(L0, L1) + 3) / 4 * 4; }   // input-row pad (J1Cfg::HLA)
constexpr int fwd12_hla2(int MQ) { return (MQ - 2 + 3) / 4 * 4; }                    // LL-row pad (J2Cfg::HLA)
constexpr int fwd12_nmg(int MQ) { return (MQ - 2) / 4; }
constexpr int fwd12_ring(int MQ) { return 4 * fwd12_nmg(MQ); }

struct Fwd12Plan {
  int threads;           // CTA size: W / 4 rounded up to whole warps
  int sw1;               // input ring: row pitch (floats) = HLA1 + W + HLA1; kF12InStages slots of 2 rows
  int sw2;               // LL ring: row pitch (floats) = HLA2 + W + HLA2; `ring` slots of one group (4 rows)
  int ring;              // LL ring depth in groups
  int ll_off;            // float offset of the LL ring (the input ring starts at 0)
  int smem_bytes;
};

struct Fwd12Band {
  int qy0, qy1;          // LL2 quad rows (= LL1 groups) the band owns
  int g0, n2;            // virtual groups level 2 consumes: g0 ... g0 + n2 - 1
  int a0, a1;            // real groups level 1 produces: a0 ... a1 - 1
  int lag;               // steps level 2 waits before its first stage
};

B200W_HD Fwd12Band fwd12_band(int band, int CH, int Hq, int nmg) {
  Fwd12Band b;
  b.qy0 = band * CH;
  b.qy1 = imin(b.qy0 + CH, Hq);
  b.g0 = b.qy0 - nmg;
  b.n2 = b.qy1 - b.qy0 + 2 * nmg;
  b.a0 = imax(0, b.g0);
  b.a1 = imin(Hq, b.qy1 + nmg);
  b.lag = imax(0, -1 - b.g0);
  return b;
}

B200W_HD int fwd12_slot(int v, int ring) {
  const int s = v % ring;
  return s < 0 ? s + ring : s;
}

// Returns 0 and fills pl when the fused kernel covers an (H, W) plane with these filter lengths, 1 otherwise.
inline int fwd12_plan(Fwd12Plan& pl, int H, int W, int L0, int L1, int MQ) {
  if (!fwd12_pair_compiled(L0, L1, MQ)) return 1;
  if ((MQ - 2) % 4) return 1;                   // mirrored rows must come in whole groups
  if ((H & 3) || (W & 3)) return 1;             // no replicate padding between the levels
  const int HL = MQ - 2, hla1 = fwd12_hla1(L0, L1), hla2 = fwd12_hla2(MQ);
  // one reflection covers every halo: level 2's rows and columns (HL), the input ring's pad columns (hla1); and with
  // at least 3*NMG groups no top mirror is still waiting in the ring when the bottom mirrors arrive (ring depth above)
  if (H < 3 * HL || W < imax(HL, hla1)) return 1;
  // (every narrower plane class measured runs faster fused, 128 columns included: tools/bench_dtcwt_fwd12.py)
  if (W > 4 * kF12MaxThreads) return 1;
  pl.threads = ((W / 4) + 31) / 32 * 32;
  pl.sw1 = hla1 + W + hla1;
  pl.sw2 = hla2 + W + hla2;
  pl.ring = fwd12_ring(MQ);
  pl.ll_off = kF12InStages * 2 * pl.sw1;
  pl.smem_bytes = (pl.ll_off + pl.ring * 4 * pl.sw2) * 4;
  if (pl.smem_bytes > kF12MaxSmem) return 1;
  return 0;
}

// The route of one b200w_dtcwt_fwd_j12 call: 0 (and the plan) when the fused kernel runs it, 1 when the two level
// kernels run through an LL1 workspace.  The fused kernel stages input rows with 16-byte cp.async copies.
inline int fwd12_route(Fwd12Plan& pl, const void* x, long long xps, int xpitch, int H, int W, int L0, int L1, int MQ,
                       bool has_highs0) {
  if (!has_highs0) return 1;
  if ((reinterpret_cast<uintptr_t>(x) & 15) || (xpitch & 3) || (xps & 3)) return 1;
  return fwd12_plan(pl, H, W, L0, L1, MQ);
}

}  // namespace b200w
