// tile_kernels.h -- generic (any filter length, any mode) fused per-level kernels, one CTA per
// (plane, output tile).  Each body: stage the input tile + halo into shared memory with the
// boundary extension applied by index arithmetic, run the first 1-D pass into a shared-memory
// intermediate, run the second pass from it, apply the pack/unpack epilogue, store.  One HBM read
// of the input and one write of every output per level; no intermediate tensor in global memory.
//
// These are the correctness-complete kernels (every L <= 40, every mode, every layout), templated on
// the element type: b200wave.cu instantiates them for float and double.  The specialised float32
// streaming kernels (afb_stream.cuh, sfb_stream.cuh, dtcwt_*_stream.cuh, behind fast_api.h) take over
// for the headline configurations.
//
// Accumulation order = the oracle's (= the reference CPU result's): increasing stored-tap index,
// fused multiply-add, pass order exactly as the reference (W then H for analysis, H then W for
// synthesis), so results are bit-identical to oracle/wave_oracle.c except for (a) the sign of
// zeros and (b) the q2c / c2q scale, applied here as x * (1/sqrt 2) like the reference's own CUDA
// path (ATen multiplies by the reciprocal of a scalar divisor) instead of a true division.
#pragma once
#include "common.h"

namespace b200w {

// ================================================================================================
// K1  DWT analysis level (reference AFB2D.forward, dwt/lowlevel.py:336-347)
//   out[k] = sum_j f[j] xe[2k + j - pl], pl = L-2 (or L-1-L/2 for periodization); W pass then H pass.
// ================================================================================================
constexpr int kAfbTH = 16, kAfbTW = 32;

B200W_HD int afb_smem_floats(int Lw, int Lh) {
  const int IW = 2 * kAfbTW + Lw - 2, IH = 2 * kAfbTH + Lh - 2;
  const int IWp = IW | 1;
  return IH * IWp + 2 * IH * kAfbTW;
}

// PK (packet layout): child b of plane p goes to ll + (4p + b) * (llps / 4) with row pitch llpitch; `highs` is then
// ll + llps / 4 and `hipitch` the row pitch of the band-pass children.
template <int NT, class T, bool PK = false>
B200W_D void afb2d_tile(const AfbParamsT<T>& p, int bid, T* smem) {
  constexpr int TH = kAfbTH, TW = kAfbTW;
  const int tx = bid % p.tiles_x;
  const int t2 = bid / p.tiles_x;
  const int ty = t2 % p.tiles_y;
  const int plane = t2 / p.tiles_y;
  const int Lw = p.Lw, Lh = p.Lh, mode = p.mode;
  const int plw = (mode == B200W_MODE_PERIODIZATION) ? (Lw - 1 - Lw / 2) : (Lw - 2);
  const int plh = (mode == B200W_MODE_PERIODIZATION) ? (Lh - 1 - Lh / 2) : (Lh - 2);
  const int k0 = tx * TW, r0 = ty * TH;
  const int IW = 2 * TW + Lw - 2, IH = 2 * TH + Lh - 2, IWp = IW | 1;
  const int c_in0 = 2 * k0 - plw, r_in0 = 2 * r0 - plh;
  T* s_in = smem;
  T* s_lo = s_in + IH * IWp;
  T* s_hi = s_lo + IH * TW;
  const T* xp = p.x + (long long)plane * p.xps;

  B200W_FOR_THREADS(tid, NT)
    const int wid = tid >> 5, lane = tid & 31;
    for (int r = wid; r < IH; r += NT / 32) {
      const int gr = ext_index(r_in0 + r, p.H, mode);
      const T* src = xp + (long long)(gr < 0 ? 0 : gr) * p.xpitch;
      for (int c = lane; c < IW; c += 32) {
        const int gc = ext_index(c_in0 + c, p.W, mode);
        s_in[r * IWp + c] = (gr < 0 || gc < 0) ? T(0) : src[gc];
      }
    }
  B200W_END_THREADS
  B200W_SYNC();

  B200W_FOR_THREADS(tid, NT)
    for (int idx = tid; idx < IH * TW; idx += NT) {
      const int r = idx / TW, k = idx - r * TW;
      const T* row = s_in + r * IWp + 2 * k;
      T a0 = 0, a1 = 0;
      for (int j = 0; j < Lw; ++j) {
        const T v = row[j];
        a0 = fma_rn(p.fw_lo.t[j], v, a0);
        a1 = fma_rn(p.fw_hi.t[j], v, a1);
      }
      s_lo[idx] = a0;
      s_hi[idx] = a1;
    }
  B200W_END_THREADS
  B200W_SYNC();

  B200W_FOR_THREADS(tid, NT)
    for (int idx = tid; idx < TH * TW; idx += NT) {
      const int kr = idx / TW, kc = idx - kr * TW;
      const int orow = r0 + kr, ocol = k0 + kc;
      if (orow >= p.Ho || ocol >= p.Wo) continue;
      T all = 0, alh = 0, ahl = 0, ahh = 0;
      for (int j = 0; j < Lh; ++j) {
        const T vlo = s_lo[(2 * kr + j) * TW + kc];
        const T vhi = s_hi[(2 * kr + j) * TW + kc];
        const T f0 = p.fh_lo.t[j], f1 = p.fh_hi.t[j];
        all = fma_rn(f0, vlo, all);
        alh = fma_rn(f1, vlo, alh);
        ahl = fma_rn(f0, vhi, ahl);
        ahh = fma_rn(f1, vhi, ahh);
      }
      p.ll[(long long)plane * p.llps + (long long)orow * p.llpitch + ocol] = all;
      long long band;
      T* hp;
      if constexpr (PK) {
        band = p.llps >> 2;
        hp = p.highs + (long long)plane * p.llps + (long long)orow * p.hipitch + ocol;
      } else {
        band = (long long)p.Ho * p.Wo;
        hp = p.highs + (long long)plane * 3 * band + (long long)orow * p.Wo + ocol;
      }
      hp[0] = alh;
      hp[band] = ahl;
      hp[2 * band] = ahh;
    }
  B200W_END_THREADS
}

// ================================================================================================
// K2  DWT synthesis level (reference SFB2D.forward, dwt/lowlevel.py:671-680)
//   y[n] = sum_k lo[k] g0[s-2k] + sum_k hi[k] g1[s-2k], s = n + off, off = L-2 (or L/2-1, k mod K
//   for periodization); H pass on (ll,lh) and (hl,hh), then W pass.
// ================================================================================================
constexpr int kSfbTH = 32, kSfbTW = 32;

B200W_HD int sfb_kspan(int T, int L) { return T / 2 + L / 2 + 2; }
B200W_HD int sfb_smem_floats(int Lh, int Lw) {
  const int KH = sfb_kspan(kSfbTH, Lh), KW = sfb_kspan(kSfbTW, Lw);
  return 4 * KH * KW + 2 * kSfbTH * KW;
}

// PK (packet layout): the four children of plane p are planes 4p .. 4p+3 of one contiguous (4P, Hc, Wc) tensor: `ll`
// = its base with llps = 4 Hc Wc, `highs` = ll + Hc Wc.
template <int NT, class T, bool PK = false>
B200W_D void sfb2d_tile(const SfbParamsT<T>& p, int bid, T* smem) {
  constexpr int TH = kSfbTH, TW = kSfbTW;
  const int tx = bid % p.tiles_x;
  const int t2 = bid / p.tiles_x;
  const int ty = t2 % p.tiles_y;
  const int plane = t2 / p.tiles_y;
  const int Lh = p.Lh, Lw = p.Lw;
  const bool per = (p.mode == B200W_MODE_PERIODIZATION);
  const int offh = per ? (Lh / 2 - 1) : (Lh - 2);
  const int offw = per ? (Lw / 2 - 1) : (Lw - 2);
  const int n0 = ty * TH, m0 = tx * TW;
  const int KH = sfb_kspan(TH, Lh), KW = sfb_kspan(TW, Lw);
  const int kh0 = floordiv2(n0 + offh - Lh + 2);  // first coefficient row any output row of the tile can touch
  const int kw0 = floordiv2(m0 + offw - Lw + 2);
  T* s_b[4];
  s_b[0] = smem;
  s_b[1] = s_b[0] + KH * KW;
  s_b[2] = s_b[1] + KH * KW;
  s_b[3] = s_b[2] + KH * KW;
  T* s_lo = s_b[3] + KH * KW;
  T* s_hi = s_lo + TH * KW;
  const T* llp = p.ll + (long long)plane * p.llps;
  const long long band = (long long)p.Hc * p.Wc;
  const T* hp = p.highs ? p.highs + (long long)plane * (PK ? 4 : 3) * band : nullptr;

  B200W_FOR_THREADS(tid, NT)
    for (int idx = tid; idx < KH * KW; idx += NT) {
      const int i = idx / KW, j = idx - i * KW;
      int kr = kh0 + i, kc = kw0 + j;
      bool ok = true;
      if (per) {
        kr %= p.Hc; if (kr < 0) kr += p.Hc;
        kc %= p.Wc; if (kc < 0) kc += p.Wc;
      } else {
        ok = (kr >= 0 && kr < p.Hc && kc >= 0 && kc < p.Wc);
      }
      T v0 = 0, v1 = 0, v2 = 0, v3 = 0;
      if (ok) {
        v0 = llp[(long long)kr * p.llpitch + kc];
        if (hp) {
          const long long o = (long long)kr * p.Wc + kc;
          v1 = hp[o];
          v2 = hp[band + o];
          v3 = hp[2 * band + o];
        }
      }
      s_b[0][idx] = v0; s_b[1][idx] = v1; s_b[2][idx] = v2; s_b[3][idx] = v3;
    }
  B200W_END_THREADS
  B200W_SYNC();

  // H pass: lo = S(ll, lh), hi = S(hl, hh)
  B200W_FOR_THREADS(tid, NT)
    for (int idx = tid; idx < TH * KW; idx += NT) {
      const int n = idx / KW, j = idx - n * KW;
      const int s = n0 + n + offh;
      const int kmin = floordiv2(s - Lh + 2), kmax = floordiv2(s);
      T a0 = 0, a1 = 0, b0 = 0, b1 = 0;
      for (int k = kmin; k <= kmax; ++k) {
        const int t = s - 2 * k;
        const int i = k - kh0;
        const T g0 = p.gh_lo.t[t], g1 = p.gh_hi.t[t];
        a0 = fma_rn(s_b[0][i * KW + j], g0, a0);
        a1 = fma_rn(s_b[1][i * KW + j], g1, a1);
        b0 = fma_rn(s_b[2][i * KW + j], g0, b0);
        b1 = fma_rn(s_b[3][i * KW + j], g1, b1);
      }
      s_lo[idx] = add_rn(a0, a1);
      s_hi[idx] = add_rn(b0, b1);
    }
  B200W_END_THREADS
  B200W_SYNC();

  // W pass
  B200W_FOR_THREADS(tid, NT)
    for (int idx = tid; idx < TH * TW; idx += NT) {
      const int n = idx / TW, m = idx - n * TW;
      const int orow = n0 + n, ocol = m0 + m;
      if (orow >= p.Ho || ocol >= p.Wo) continue;
      const int s = ocol + offw;
      const int kmin = floordiv2(s - Lw + 2), kmax = floordiv2(s);
      T a0 = 0, a1 = 0;
      for (int k = kmin; k <= kmax; ++k) {
        const int t = s - 2 * k;
        const int j = k - kw0;
        a0 = fma_rn(s_lo[n * KW + j], p.gw_lo.t[t], a0);
        a1 = fma_rn(s_hi[n * KW + j], p.gw_hi.t[t], a1);
      }
      p.y[(long long)plane * p.yps + (long long)orow * p.ypitch + ocol] = add_rn(a0, a1);
    }
  B200W_END_THREADS
}

// ================================================================================================
// DTCWT helpers
// ================================================================================================
// q2c + orientation store (reference dtcwt/lowlevel.py:243-260, transform_funcs.py:61-72).
// a,b / c,d = the 2x2 quad of one real subband; o1/o2 = orientation slots of w1 = (a-d, b+c), w2 = (a+d, b-c).
template <class T>
B200W_D void q2c_store(T a, T b, T c, T d, T* hq, const long long* hs, int o1, int o2) {
  a = mul_rn(a, kInvSqrt2T<T>); b = mul_rn(b, kInvSqrt2T<T>);
  c = mul_rn(c, kInvSqrt2T<T>); d = mul_rn(d, kInvSqrt2T<T>);
  hq[o1 * hs[2]] = sub_rn(a, d);
  hq[o1 * hs[2] + hs[5]] = add_rn(b, c);
  hq[o2 * hs[2]] = add_rn(a, d);
  hq[o2 * hs[2] + hs[5]] = sub_rn(b, c);
}

// c2q (reference dtcwt/lowlevel.py:263-295 via orientations_to_highs, transform_funcs.py:75-95):
// value of the real quad-domain subband at (gr, gc) from the complex pair (o1 -> w1, o2 -> w2).
template <class T>
B200W_D T c2q_load(const T* hb, const long long* hs, int gr, int gc, int o1, int o2) {
  const int pr = gr & 1, pc = gc & 1;
  const long long q = (long long)(gr >> 1) * hs[3] + (long long)(gc >> 1) * hs[4];
  const long long ri = (pr ^ pc) ? hs[5] : 0;  // (0,0),(1,1) use the real parts; (0,1),(1,0) the imaginary parts
  const T w1 = hb[q + o1 * hs[2] + ri];
  const T w2 = hb[q + o2 * hs[2] + ri];
  T v;
  if (pr == 0) v = add_rn(w1, w2);       // a = w1r + w2r ; b = w1i + w2i
  else if (pc == 0) v = sub_rn(w1, w2);  // c = w1i - w2i
  else v = sub_rn(w2, w1);               // d = -w1r + w2r
  return mul_rn(v, kInvSqrt2T<T>);
}

// ================================================================================================
// K3 / K7  DTCWT level-1 forward (reference FWD_J1.forward, dtcwt/transform_funcs.py:346-358) and
//          the ScatLayer epilogue on top of it (scatternet/lowlevel.py:76-111).
//   y[n] = sum_j h[j] x[ext(n + j - L/2)], undecimated; rows then columns; q2c on 2x2 quads.
// ================================================================================================
constexpr int kJ1TH = 32, kJ1TW = 32;

B200W_HD int fwdj1_smem_floats(int L0, int L1) {
  const int M = imax(L0 / 2, L1 / 2);
  const int IH = kJ1TH + 2 * M, IW = kJ1TW + 2 * M, IWp = IW | 1;
  return IH * IWp + 2 * IH * kJ1TW;
}

template <int NT, bool SCAT, class T>
B200W_D void fwd_j1_tile(const DtParamsT<T>& p, int bid, T* smem) {
  constexpr int TH = kJ1TH, TW = kJ1TW;
  const int tx = bid % p.tiles_x;
  const int t2 = bid / p.tiles_x;
  const int ty = t2 % p.tiles_y;
  const int plane = t2 / p.tiles_y;
  const int L0 = p.L0, L1 = p.L1, M0 = L0 / 2, M1 = L1 / 2, M = imax(M0, M1);
  const int r0 = ty * TH, c0 = tx * TW;
  const int IH = TH + 2 * M, IW = TW + 2 * M, IWp = IW | 1;
  T* s_in = smem;
  T* s_lo = s_in + IH * IWp;
  T* s_hi = s_lo + IH * TW;
  const T* xp = p.in + (long long)plane * p.inps;
  const bool want_highs = SCAT || (p.highs != nullptr);

  B200W_FOR_THREADS(tid, NT)
    const int wid = tid >> 5, lane = tid & 31;
    for (int r = wid; r < IH; r += NT / 32) {
      const int gr = sym_or_zero(r0 - M + r, p.H, p.sym);
      const T* src = xp + (long long)(gr < 0 ? 0 : gr) * p.inpitch;
      for (int c = lane; c < IW; c += 32) {
        const int gc = sym_or_zero(c0 - M + c, p.W, p.sym);
        s_in[r * IWp + c] = (gr < 0 || gc < 0) ? T(0) : src[gc];
      }
    }
  B200W_END_THREADS
  B200W_SYNC();

  // row pass (rowfilter, dtcwt/lowlevel.py:83-94)
  B200W_FOR_THREADS(tid, NT)
    for (int idx = tid; idx < IH * TW; idx += NT) {
      const int r = idx / TW, c = idx - r * TW;
      const T* row = s_in + r * IWp + c + M;
      T a0 = 0;
      for (int j = 0; j < L0; ++j) a0 = fma_rn(p.f0.t[j], row[j - M0], a0);
      s_lo[idx] = a0;
      if (want_highs) {
        T a1 = 0;
        for (int j = 0; j < L1; ++j) a1 = fma_rn(p.f1.t[j], row[j - M1], a1);
        s_hi[idx] = a1;
      }
    }
  B200W_END_THREADS
  B200W_SYNC();

  // column pass (colfilter :70-80) on one 2x2 quad per thread, then q2c / magnitude epilogue
  B200W_FOR_THREADS(tid, NT)
    for (int idx = tid; idx < (TH / 2) * (TW / 2); idx += NT) {
      const int qr = idx / (TW / 2), qc = idx - qr * (TW / 2);
      const int gr = r0 + 2 * qr, gc = c0 + 2 * qc;
      if (gr >= p.H || gc >= p.W) continue;
      const int n = plane / p.C, ch = plane - n * p.C;
      T v[4][4];  // [band ll,lh,hl,hh][quad position a,b,c,d]
      for (int dr = 0; dr < 2; ++dr)
        for (int dc = 0; dc < 2; ++dc) {
          const int r = 2 * qr + dr + M, c = 2 * qc + dc;
          T all = 0, alh = 0, ahl = 0, ahh = 0;
          for (int j = 0; j < L0; ++j) {
            const T f = p.f0.t[j];
            all = fma_rn(f, s_lo[(r - M0 + j) * TW + c], all);
            if (want_highs) ahl = fma_rn(f, s_hi[(r - M0 + j) * TW + c], ahl);
          }
          if (want_highs)
            for (int j = 0; j < L1; ++j) {
              const T f = p.f1.t[j];
              alh = fma_rn(f, s_lo[(r - M1 + j) * TW + c], alh);
              ahh = fma_rn(f, s_hi[(r - M1 + j) * TW + c], ahh);
            }
          v[0][dr * 2 + dc] = all; v[1][dr * 2 + dc] = alh; v[2][dr * 2 + dc] = ahl; v[3][dr * 2 + dc] = ahh;
        }
      if (!SCAT) {
        T* lp = p.out + (long long)plane * p.outps + (long long)gr * p.outpitch + gc;
        lp[0] = v[0][0]; lp[1] = v[0][1];
        lp[p.outpitch] = v[0][2]; lp[p.outpitch + 1] = v[0][3];
        if (p.highs) {
          T* hq = p.highs + n * p.hs[0] + ch * p.hs[1] + (long long)(gr >> 1) * p.hs[3] + (long long)(gc >> 1) * p.hs[4];
          q2c_store(v[1][0], v[1][1], v[1][2], v[1][3], hq, p.hs, 0, 5);  // lh -> 15, 165
          q2c_store(v[3][0], v[3][1], v[3][2], v[3][3], hq, p.hs, 1, 4);  // hh -> 45, 135
          q2c_store(v[2][0], v[2][1], v[2][2], v[2][3], hq, p.hs, 2, 3);  // hl -> 75, 105
        }
      } else {
        // z (N,7,C,h,w): slot 0 = 2x2 mean of ll (F.avg_pool2d, scatternet/lowlevel.py:88), slots 1..6 = smoothed magnitudes
        const int h = p.H >> 1, w = p.W >> 1;
        const long long hw = (long long)h * w;
        const long long pix = (long long)(gr >> 1) * w + (gc >> 1);
        T s = add_rn(v[0][0], v[0][1]);
        s = add_rn(s, v[0][2]);
        s = add_rn(s, v[0][3]);
        p.z[(((long long)n * 7 + 0) * p.C + ch) * hw + pix] = mul_rn(s, T(0.25));
        const int band_of[3] = {1, 3, 2};            // lh, hh, hl
        const int o1s[3] = {0, 1, 2}, o2s[3] = {5, 4, 3};
#pragma unroll
        for (int b = 0; b < 3; ++b) {
          const T a = mul_rn(v[band_of[b]][0], kInvSqrt2T<T>), bb = mul_rn(v[band_of[b]][1], kInvSqrt2T<T>);
          const T c = mul_rn(v[band_of[b]][2], kInvSqrt2T<T>), d = mul_rn(v[band_of[b]][3], kInvSqrt2T<T>);
          const T re[2] = {sub_rn(a, d), add_rn(a, d)};
          const T im[2] = {add_rn(bb, c), sub_rn(bb, c)};
          const int os[2] = {o1s[b], o2s[b]};
#pragma unroll
          for (int k = 0; k < 2; ++k) {
            const T rr = mul_rn(re[k], re[k]), ii = mul_rn(im[k], im[k]);
            const T r = sqrt_rn(add_rn(add_rn(rr, ii), p.magbias2));
            p.z[(((long long)n * 7 + 1 + os[k]) * p.C + ch) * hw + pix] = sub_rn(r, p.magbias);
            if (p.dre) {
              const long long o6 = (((long long)n * 6 + os[k]) * p.C + ch) * hw + pix;
              p.dre[o6] = div_rn(re[k], r);
              p.dim[o6] = div_rn(im[k], r);
            }
          }
        }
      }
    }
  B200W_END_THREADS
}

// ================================================================================================
// K4  DTCWT level>=2 forward (reference FWD_J2PLUS.forward, dtcwt/transform_funcs.py:380-392)
//   rowdfilt / coldfilt (dtcwt/lowlevel.py:97-151): Ya[q] = sum_j ha[j] x[sym(4q+2j+2-m)],
//   Yb[q] = sum_j hb[j] x[sym(4q+2j+3-m)], interleaved (a,b) for low-pass, (b,a) for high-pass.
//   taps: f0=h0a f1=h1a f2=h0b f3=h1b (stored); low: (ha,hb)=(h0b,h0a), high: (ha,hb)=(h1b,h1a).
// ================================================================================================
constexpr int kJ2TH = 16, kJ2TW = 32;  // tile of the half-resolution ll output

B200W_HD int fwdj2_smem_floats(int m) {
  const int IH = 2 * kJ2TH + 2 * m - 4, IW = 2 * kJ2TW + 2 * m - 4, IWp = IW | 1;
  return IH * IWp + 2 * IH * kJ2TW;
}

template <int NT, class T>
B200W_D void fwd_j2plus_tile(const DtParamsT<T>& p, int bid, T* smem) {
  constexpr int TH = kJ2TH, TW = kJ2TW;
  const int tx = bid % p.tiles_x;
  const int t2 = bid / p.tiles_x;
  const int ty = t2 % p.tiles_y;
  const int plane = t2 / p.tiles_y;
  const int m = p.L0;
  const int y0 = ty * TH, x0 = tx * TW;  // origin in the half-res output
  const int IH = 2 * TH + 2 * m - 4, IW = 2 * TW + 2 * m - 4, IWp = IW | 1;
  const int r_in0 = 2 * y0 + 2 - m, c_in0 = 2 * x0 + 2 - m;
  const int H2 = p.H >> 1, W2 = p.W >> 1;
  T* s_in = smem;
  T* s_lo = s_in + IH * IWp;
  T* s_hi = s_lo + IH * TW;
  const T* xp = p.in + (long long)plane * p.inps;
  const bool want_highs = (p.highs != nullptr);

  B200W_FOR_THREADS(tid, NT)
    const int wid = tid >> 5, lane = tid & 31;
    for (int r = wid; r < IH; r += NT / 32) {
      const int gr = ext_index(r_in0 + r, p.H, B200W_MODE_SYMMETRIC);
      const T* src = xp + (long long)gr * p.inpitch;
      for (int c = lane; c < IW; c += 32) {
        const int gc = ext_index(c_in0 + c, p.W, B200W_MODE_SYMMETRIC);
        s_in[r * IWp + c] = src[gc];
      }
    }
  B200W_END_THREADS
  B200W_SYNC();

  // row pass: lo = rowdfilt(x, h0b, h0a, False), hi = rowdfilt(x, h1b, h1a, True)
  B200W_FOR_THREADS(tid, NT)
    for (int idx = tid; idx < IH * (TW / 2); idx += NT) {
      const int r = idx / (TW / 2), q = idx - r * (TW / 2);
      const T* row = s_in + r * IWp + 4 * q;
      T la = 0, lb = 0, ha = 0, hb = 0;
      for (int j = 0; j < m; ++j) {
        const T ve = row[2 * j], vo = row[2 * j + 1];
        la = fma_rn(p.f2.t[j], ve, la);  // Ya with h0b
        lb = fma_rn(p.f0.t[j], vo, lb);  // Yb with h0a
        if (want_highs) {
          ha = fma_rn(p.f3.t[j], ve, ha);  // Ya with h1b
          hb = fma_rn(p.f1.t[j], vo, hb);  // Yb with h1a
        }
      }
      s_lo[r * TW + 2 * q] = la;
      s_lo[r * TW + 2 * q + 1] = lb;
      if (want_highs) {
        s_hi[r * TW + 2 * q] = hb;      // high-pass: (b, a)
        s_hi[r * TW + 2 * q + 1] = ha;
      }
    }
  B200W_END_THREADS
  B200W_SYNC();

  // column pass on one quad (2x2 of the half-res bands) per thread
  B200W_FOR_THREADS(tid, NT)
    for (int idx = tid; idx < (TH / 2) * (TW / 2); idx += NT) {
      const int qr = idx / (TW / 2), qc = idx - qr * (TW / 2);
      const int gy = y0 + 2 * qr, gx = x0 + 2 * qc;  // half-res coordinates of the quad's top-left
      if (gy >= H2 || gx >= W2) continue;
      const int n = plane / p.C, ch = plane - n * p.C;
      T v[4][4];
      for (int dc = 0; dc < 2; ++dc) {
        const int c = 2 * qc + dc;
        T ll0 = 0, ll1 = 0, lh0 = 0, lh1 = 0, hl0 = 0, hl1 = 0, hh0 = 0, hh1 = 0;
        for (int j = 0; j < m; ++j) {
          const T le = s_lo[(4 * qr + 2 * j) * TW + c], lo_ = s_lo[(4 * qr + 2 * j + 1) * TW + c];
          ll0 = fma_rn(p.f2.t[j], le, ll0);   // ll[2q]   = Ya(h0b) on lo
          ll1 = fma_rn(p.f0.t[j], lo_, ll1);  // ll[2q+1] = Yb(h0a)
          if (want_highs) {
            const T he = s_hi[(4 * qr + 2 * j) * TW + c], ho = s_hi[(4 * qr + 2 * j + 1) * TW + c];
            lh0 = fma_rn(p.f1.t[j], lo_, lh0);  // lh[2q]   = Yb(h1a) on lo   (high-pass interleave)
            lh1 = fma_rn(p.f3.t[j], le, lh1);   // lh[2q+1] = Ya(h1b)
            hl0 = fma_rn(p.f2.t[j], he, hl0);   // hl[2q]   = Ya(h0b) on hi
            hl1 = fma_rn(p.f0.t[j], ho, hl1);   // hl[2q+1] = Yb(h0a)
            hh0 = fma_rn(p.f1.t[j], ho, hh0);   // hh[2q]   = Yb(h1a) on hi
            hh1 = fma_rn(p.f3.t[j], he, hh1);   // hh[2q+1] = Ya(h1b)
          }
        }
        v[0][dc] = ll0; v[0][2 + dc] = ll1;
        v[1][dc] = lh0; v[1][2 + dc] = lh1;
        v[2][dc] = hl0; v[2][2 + dc] = hl1;
        v[3][dc] = hh0; v[3][2 + dc] = hh1;
      }
      T* lp = p.out + (long long)plane * p.outps + (long long)gy * p.outpitch + gx;
      lp[0] = v[0][0]; lp[1] = v[0][1];
      lp[p.outpitch] = v[0][2]; lp[p.outpitch + 1] = v[0][3];
      if (want_highs) {
        T* hq = p.highs + n * p.hs[0] + ch * p.hs[1] + (long long)(gy >> 1) * p.hs[3] + (long long)(gx >> 1) * p.hs[4];
        q2c_store(v[1][0], v[1][1], v[1][2], v[1][3], hq, p.hs, 0, 5);
        q2c_store(v[3][0], v[3][1], v[3][2], v[3][3], hq, p.hs, 1, 4);
        q2c_store(v[2][0], v[2][1], v[2][2], v[2][3], hq, p.hs, 2, 3);
      }
    }
  B200W_END_THREADS
}

// ================================================================================================
// K5  DTCWT level-1 inverse (reference INV_J1.forward, dtcwt/transform_funcs.py:419-431 / inv_j1 :152-184)
//   hi = colfilter(hh,g1) + colfilter(hl,g0); lo = colfilter(lh,g1) [+ colfilter(ll,g0)];
//   y  = rowfilter(hi,g1) + rowfilter(lo,g0).   f0 = g0 (L0 taps), f1 = g1 (L1 taps).
//   highs == null: y = rowfilter(colfilter(ll,g0),g0) with symmetric extension (:159).
// ================================================================================================
constexpr int kI1TH = 16, kI1TW = 32;

B200W_HD int invj1_smem_floats(int L0, int L1) {
  const int M = imax(L0 / 2, L1 / 2);
  const int IH = kI1TH + 2 * M, IW = kI1TW + 2 * M;
  return 4 * IH * IW + 2 * kI1TH * IW;
}

template <int NT, class T>
B200W_D void inv_j1_tile(const DtParamsT<T>& p, int bid, T* smem) {
  constexpr int TH = kI1TH, TW = kI1TW;
  const int tx = bid % p.tiles_x;
  const int t2 = bid / p.tiles_x;
  const int ty = t2 % p.tiles_y;
  const int plane = t2 / p.tiles_y;
  const int L0 = p.L0, L1 = p.L1, M0 = L0 / 2, M1 = L1 / 2, M = imax(M0, M1);
  const int r0 = ty * TH, c0 = tx * TW;
  const int IH = TH + 2 * M, IW = TW + 2 * M;
  T* s_ll = smem;
  T* s_lh = s_ll + IH * IW;
  T* s_hl = s_lh + IH * IW;
  T* s_hh = s_hl + IH * IW;
  T* s_lo = s_hh + IH * IW;
  T* s_hi = s_lo + TH * IW;
  const T* llp = p.in ? p.in + (long long)plane * p.inps : nullptr;
  const int n = plane / p.C, ch = plane - n * p.C;
  const T* hb = p.highs ? p.highs + n * p.hs[0] + ch * p.hs[1] : nullptr;
  const int sym = hb ? p.sym : 1;

  B200W_FOR_THREADS(tid, NT)
    for (int idx = tid; idx < IH * IW; idx += NT) {
      const int r = idx / IW, c = idx - r * IW;
      const int gr = sym_or_zero(r0 - M + r, p.H, sym), gc = sym_or_zero(c0 - M + c, p.W, sym);
      T vll = 0, vlh = 0, vhl = 0, vhh = 0;
      if (gr >= 0 && gc >= 0) {
        if (llp) vll = llp[(long long)gr * p.inpitch + gc];
        if (hb) {
          vlh = c2q_load(hb, p.hs, gr, gc, 0, 5);
          vhl = c2q_load(hb, p.hs, gr, gc, 2, 3);
          vhh = c2q_load(hb, p.hs, gr, gc, 1, 4);
        }
      }
      s_ll[idx] = vll; s_lh[idx] = vlh; s_hl[idx] = vhl; s_hh[idx] = vhh;
    }
  B200W_END_THREADS
  B200W_SYNC();

  B200W_FOR_THREADS(tid, NT)
    for (int idx = tid; idx < TH * IW; idx += NT) {
      const int r = idx / IW, c = idx - r * IW;
      const int rr = r + M;
      T a_ll = 0, a_hl = 0, a_lh = 0, a_hh = 0;
      for (int j = 0; j < L0; ++j) {
        const T f = p.f0.t[j];
        a_ll = fma_rn(f, s_ll[(rr - M0 + j) * IW + c], a_ll);
        a_hl = fma_rn(f, s_hl[(rr - M0 + j) * IW + c], a_hl);
      }
      for (int j = 0; j < L1; ++j) {
        const T f = p.f1.t[j];
        a_lh = fma_rn(f, s_lh[(rr - M1 + j) * IW + c], a_lh);
        a_hh = fma_rn(f, s_hh[(rr - M1 + j) * IW + c], a_hh);
      }
      if (hb) {
        s_hi[idx] = add_rn(a_hh, a_hl);
        s_lo[idx] = llp ? add_rn(a_lh, a_ll) : a_lh;
      } else {
        s_lo[idx] = a_ll;
        s_hi[idx] = 0;
      }
    }
  B200W_END_THREADS
  B200W_SYNC();

  B200W_FOR_THREADS(tid, NT)
    for (int idx = tid; idx < TH * TW; idx += NT) {
      const int r = idx / TW, c = idx - r * TW;
      const int gr = r0 + r, gc = c0 + c;
      if (gr >= p.H || gc >= p.W) continue;
      const T* rl = s_lo + r * IW + c + M;
      const T* rh = s_hi + r * IW + c + M;
      T a0 = 0, a1 = 0;
      for (int j = 0; j < L0; ++j) a0 = fma_rn(p.f0.t[j], rl[j - M0], a0);
      T yv = a0;
      if (hb) {
        for (int j = 0; j < L1; ++j) a1 = fma_rn(p.f1.t[j], rh[j - M1], a1);
        yv = add_rn(a1, a0);
      }
      p.out[(long long)plane * p.outps + (long long)gr * p.outpitch + gc] = yv;
    }
  B200W_END_THREADS
}

// ================================================================================================
// K6  DTCWT level>=2 inverse (reference INV_J2PLUS.forward, transform_funcs.py:455-468 / inv_j2plus :279-307)
//   colifilt / rowifilt (dtcwt/lowlevel.py:154-239): y[4t+s] = sum_{j<m2} f_s[j] x[sym(2(t+j) + o_s - m2)].
//   taps: f0=g0a f1=g1a f2=g0b f3=g1b (stored); low call (ha,hb)=(g0b,g0a), high call (ha,hb)=(g1b,g1a).
// ================================================================================================
constexpr int kI2TH = 32, kI2TW = 32;  // tile of the 2x-resolution output

B200W_HD int invj2_smem_floats(int m) {
  const int m2 = m / 2;
  const int IH = kI2TH / 2 + 2 * m2, IW = kI2TW / 2 + 2 * m2;
  return 4 * IH * IW + 2 * kI2TH * IW;
}

// phase table of colifilt/rowifilt: tap parity and input offset for output phase s
B200W_HD void ifilt_phase(int m2, int highpass, int s, int* par, int* o) {
  if ((m2 & 1) == 0) {  // (hae, hbe, hao, hbo), o = (0,1,2,3) low / (1,0,3,2) high
    *par = (s >= 2);
    *o = highpass ? (s ^ 1) : s;
  } else {              // (hao, hbo, hae, hbe), o = (1,2,1,2) low / (2,1,2,1) high
    *par = (s < 2);
    *o = highpass ? (2 - (s & 1)) : (1 + (s & 1));
  }
}

template <int NT, class T>
B200W_D void inv_j2plus_tile(const DtParamsT<T>& p, int bid, T* smem) {
  constexpr int TH = kI2TH, TW = kI2TW;
  const int tx = bid % p.tiles_x;
  const int t2 = bid / p.tiles_x;
  const int ty = t2 % p.tiles_y;
  const int plane = t2 / p.tiles_y;
  const int m = p.L0, m2 = m / 2;
  const int R0 = ty * TH, C0 = tx * TW;  // output origin
  const int t0 = R0 / 4, u0 = C0 / 4;
  const int IH = TH / 2 + 2 * m2, IW = TW / 2 + 2 * m2;
  const int r_in0 = 2 * t0 - m2, c_in0 = 2 * u0 - m2;
  T* s_ll = smem;
  T* s_lh = s_ll + IH * IW;
  T* s_hl = s_lh + IH * IW;
  T* s_hh = s_hl + IH * IW;
  T* s_lo = s_hh + IH * IW;
  T* s_hi = s_lo + TH * IW;
  const T* llp = p.in ? p.in + (long long)plane * p.inps : nullptr;
  const int n = plane / p.C, ch = plane - n * p.C;
  const T* hb = p.highs ? p.highs + n * p.hs[0] + ch * p.hs[1] : nullptr;

  B200W_FOR_THREADS(tid, NT)
    for (int idx = tid; idx < IH * IW; idx += NT) {
      const int r = idx / IW, c = idx - r * IW;
      const int gr = ext_index(r_in0 + r, p.H, B200W_MODE_SYMMETRIC);
      const int gc = ext_index(c_in0 + c, p.W, B200W_MODE_SYMMETRIC);
      T vll = 0, vlh = 0, vhl = 0, vhh = 0;
      if (llp) vll = llp[(long long)gr * p.inpitch + gc];
      if (hb) {
        vlh = c2q_load(hb, p.hs, gr, gc, 0, 5);
        vhl = c2q_load(hb, p.hs, gr, gc, 2, 3);
        vhh = c2q_load(hb, p.hs, gr, gc, 1, 4);
      }
      s_ll[idx] = vll; s_lh[idx] = vlh; s_hl[idx] = vhl; s_hh[idx] = vhh;
    }
  B200W_END_THREADS
  B200W_SYNC();

  // column pass: rows of the 2x output, all staged columns
  B200W_FOR_THREADS(tid, NT)
    for (int idx = tid; idx < TH * IW; idx += NT) {
      const int r = idx / IW, c = idx - r * IW;
      const int tt = r >> 2, s = r & 3;
      int parl, ol, parh, oh;
      ifilt_phase(m2, 0, s, &parl, &ol);
      ifilt_phase(m2, 1, s, &parh, &oh);
      // s even -> ha, s odd -> hb;  low call: ha=g0b(f2) hb=g0a(f0);  high call: ha=g1b(f3) hb=g1a(f1)
      const T* fl = (s & 1) ? p.f0.t : p.f2.t;
      const T* fh = (s & 1) ? p.f1.t : p.f3.t;
      T a_ll = 0, a_hl = 0, a_lh = 0, a_hh = 0;
      for (int j = 0; j < m2; ++j) {
        const int il = (2 * (tt + j) + ol) * IW + c;
        const int ih = (2 * (tt + j) + oh) * IW + c;
        const T cl = fl[2 * j + parl], chh = fh[2 * j + parh];
        a_ll = fma_rn(cl, s_ll[il], a_ll);
        a_hl = fma_rn(cl, s_hl[il], a_hl);
        a_lh = fma_rn(chh, s_lh[ih], a_lh);
        a_hh = fma_rn(chh, s_hh[ih], a_hh);
      }
      if (hb) {
        s_hi[idx] = add_rn(a_hh, a_hl);
        s_lo[idx] = llp ? add_rn(a_lh, a_ll) : a_lh;
      } else {
        s_lo[idx] = a_ll;
        s_hi[idx] = 0;
      }
    }
  B200W_END_THREADS
  B200W_SYNC();

  B200W_FOR_THREADS(tid, NT)
    for (int idx = tid; idx < TH * TW; idx += NT) {
      const int r = idx / TW, c = idx - r * TW;
      const int gr = R0 + r, gc = C0 + c;
      if (gr >= 2 * p.H || gc >= 2 * p.W) continue;
      const int uu = c >> 2, s = c & 3;
      int parl, ol, parh, oh;
      ifilt_phase(m2, 0, s, &parl, &ol);
      ifilt_phase(m2, 1, s, &parh, &oh);
      const T* fl = (s & 1) ? p.f0.t : p.f2.t;
      const T* fh = (s & 1) ? p.f1.t : p.f3.t;
      T a0 = 0, a1 = 0;
      for (int j = 0; j < m2; ++j) a0 = fma_rn(fl[2 * j + parl], s_lo[r * IW + 2 * (uu + j) + ol], a0);
      T yv = a0;
      if (hb) {
        for (int j = 0; j < m2; ++j) a1 = fma_rn(fh[2 * j + parh], s_hi[r * IW + 2 * (uu + j) + oh], a1);
        yv = add_rn(a1, a0);
      }
      p.out[(long long)plane * p.outps + (long long)gr * p.outpitch + gc] = yv;
    }
  B200W_END_THREADS
}

}  // namespace b200w
