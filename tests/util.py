"""Shared helpers for the parity tests."""
import glob
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')

# fp32 parity tolerance, relative to max|ref| of the tensor compared.  Same-algorithm fp32
# differences (FMA contraction, summation order of the transposed convolutions, x*(1/sqrt2) vs
# x/sqrt2) are ~1e-7..1e-6; the reference's own tests use decimal=3..4 (SURVEY section 4).
RTOL_F32 = 1e-5


def fixtures(prefix):
    return sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN, prefix + '*.npz')))


def load(name):
    d = np.load(os.path.join(GOLDEN, name + '.npz'), allow_pickle=False)
    return {k: d[k] for k in d.files}


def rel_err(a, b):
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    assert a.shape == b.shape, (a.shape, b.shape)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def bit_equal_fraction(a, b):
    a = np.asarray(a)
    b = np.asarray(b)
    return float((a == b).mean())


def assert_close(a, b, tol=RTOL_F32, what=''):
    e = rel_err(a, b)
    assert e <= tol, '%s: rel err %.3e > %.1e' % (what, e, tol)
    return e


# ---- per-plane fp32 error bound against the float64 oracle ---------------------------------------------------------
# For an output plane y of a DTCWT / ScatLayer level, computed in fp32 and, from the same fp32 inputs and taps widened
# exactly, in fp64 (y64):
#     |y - y64| <= K * U32 * G * s
#   s  max |input| over the input planes that feed the output plane (the (n, c) plane; for the inverses the low-pass
#      plane and the twelve band-pass planes of that (n, c));
#   G  product of the filters' l1 norms along the path (summed over the bands an inverse adds up), times sqrt(2) where
#      q2c / c2q mixes two bands: the largest |y| the inputs allow;
#   K  a constant per output kind.  Counting every rounding (n per n-tap FMA chain) gives a bound that always holds
#      but sits 10-40x above what fp32 does, because G * s already assumes every product has the largest magnitude;
#      such a bound cannot see a wrong border column in a small plane.  So K is set from measurement instead, between
#      the largest error the fp32 oracle and the emulated generic kernels reach (K >= 1.2x that) and the largest value
#      at which an error of 1e-6 of the scale in one element of the smallest plane still fails the bound.
#      tests/test_error_bound_cpu.py checks both ends at the shapes and scales of the GPU sweep and prints the ratios.
# The bound is per plane, so an error that lands in a plane scaled 1e-6 next to planes scaled 1e6 cannot hide.

U32 = 2.0 ** -24
SQRT2 = 2.0 ** 0.5


def l1(f):
    """l1 norm of fp32 taps (what the kernels multiply by)."""
    return float(np.abs(np.asarray(f, dtype=np.float64).astype(np.float32).astype(np.float64)).sum())


def l1_phase(f):
    """Largest l1 norm of one interpolation phase (even or odd taps) of a synthesis filter."""
    f = np.asarray(f, dtype=np.float64).ravel()
    return max(l1(f[0::2]), l1(f[1::2]))


def bound_fwd_j1(h0, h1):
    """(G, K) of the level-1 forward outputs: low-pass, band-pass (q2c: x * (1/sqrt2), then a sum)."""
    g = max(l1(h0), l1(h1))
    return {'ll': (l1(h0) ** 2, 4.0), 'highs': (g * g * SQRT2, 3.0)}


def bound_fwd_j2plus(h0a, h1a, h0b, h1b):
    lo = max(l1(h0a), l1(h0b))
    g = max(lo, l1(h1a), l1(h1b))
    return {'ll': (lo * lo, 3.3), 'highs': (g * g * SQRT2, 2.0)}


def _inv_G(n0, n1, has_ll, has_hi):
    # y = C1(R1(hh) + R0(lh)) + C0(R1(hl) + R0(ll)); the band samples come from c2q ((p +- q) * (1/sqrt2))
    return (n1 * n1 + n1 * n0 + n0 * n1) * SQRT2 * has_hi + n0 * n0 * has_ll


def bound_inv_j1(g0, g1, has_ll=True, has_hi=True):
    # (low-pass only: two filter passes and a G of one band, like the forward low-pass)
    return _inv_G(l1(g0), l1(g1), has_ll, has_hi), (1.2 if has_hi else 4.0)


def bound_inv_j2plus(g0a, g1a, g0b, g1b, has_ll=True, has_hi=True):
    n0, n1 = max(l1_phase(g0a), l1_phase(g0b)), max(l1_phase(g1a), l1_phase(g1b))
    return _inv_G(n0, n1, has_ll, has_hi), (2.2 if has_hi else 4.0)


def bound_scat(h0, h1, magbias):
    """(G, K, additive scale) of the ScatLayer outputs.  z[0] is the 2x2 mean of the low-pass (three sums, an exact
    * 0.25); a magnitude sqrt(re^2 + im^2 + b^2) - b is 1-Lipschitz in (re, im) and adds squares, two sums, a root and
    a difference, whose rounding scales with r <= |w| + b: its bound gets magbias as an additive scale."""
    hG, hK = bound_fwd_j1(h0, h1)['highs']
    return {'avg': (l1(h0) ** 2, 3.0, 0.0), 'mag': (hG * SQRT2, 2.5, float(magbias)), 'band': (hG, hK)}


def bound_sfb2d(gh_lo, gh_hi, gw_lo, gw_hi, has_hi=True):
    """(G, K) of one DWT synthesis level (sfb2d).  An output sample is one interpolation phase of each filter along H
    and along W, summed over the bands present: G = (sum of the per-phase l1 norms along H) x (the same along W).
    The generic kernel / oracle run H then W, the streaming kernels W then H, each with a final add per pass.
    K: 2.5 for 2 taps (every tap is 1/sqrt2, so G * s is reached and the roundings are a larger share of it), 1.5 for
    longer filters, 2.0 for the low-pass band alone."""
    nh = l1_phase(gh_lo) + (l1_phase(gh_hi) if has_hi else 0.0)
    nw = l1_phase(gw_lo) + (l1_phase(gw_hi) if has_hi else 0.0)
    if not has_hi:
        return nh * nw, 2.0
    return nh * nw, (2.5 if max(np.size(gh_lo), np.size(gw_lo)) <= 2 else 1.5)


def planes_err_ratio(y, y64, s, G, K, add=0.0):
    """Per (n, c) plane: max|y - y64| / (K * U32 * (G * s + add)).  y, y64: (N, C, ...) arrays, s: (N, C).
    NaN (an unwritten output) gives inf."""
    y = np.asarray(y, dtype=np.float64)
    y64 = np.asarray(y64, dtype=np.float64)
    assert y.shape == y64.shape, (y.shape, y64.shape)
    N, C = y.shape[:2]
    err = np.abs(y - y64).reshape(N, C, -1)
    err = np.where(np.isnan(err), np.inf, err).max(axis=2)
    bnd = K * U32 * (G * np.asarray(s, dtype=np.float64) + add)
    return err / np.maximum(bnd, 1e-300)


def assert_plane_bound(y, y64, s, G, K, add=0.0, what=''):
    """Every (n, c) plane of y within its own bound; returns the worst error / bound ratio."""
    r = planes_err_ratio(y, y64, s, G, K, add)
    worst = float(r.max()) if r.size else 0.0
    if worst > 1.0:
        n, c = np.unravel_index(int(np.argmax(r)), r.shape)
        raise AssertionError('%s: plane (n=%d, c=%d) error %.3g x its bound (s = %.3g)'
                             % (what, n, c, worst, float(np.asarray(s)[n, c])))
    return worst


def assert_ratio_bound(q, q64, band_err, r64, what=''):
    """re/r and im/r elementwise: |q - q64| <= (1 + sqrt2) * band_err / r64 + 4 u.  (re/r moves by at most
    (|d re| + |d r|) / r, and |d r| <= sqrt2 * band_err.)"""
    q = np.asarray(q, dtype=np.float64)
    q64 = np.asarray(q64, dtype=np.float64)
    bnd = (1 + SQRT2) * band_err / np.asarray(r64, dtype=np.float64) + 4 * U32
    bad = ~(np.abs(q - q64) <= bnd)
    assert not bad.any(), '%s: %d elements outside the bound, first at %s' % (
        what, int(bad.sum()), tuple(int(i) for i in np.argwhere(bad)[0]))


def plane_scales(N, C, rng, lo=-6, hi=6):
    """One power of ten per (n, c) plane, spread over 10^lo .. 10^hi (both ends present)."""
    e = np.linspace(lo, hi, N * C) if N * C > 1 else np.array([0.0])
    e = np.round(e).astype(np.int64)
    rng.shuffle(e)
    return (10.0 ** e).reshape(N, C)


def scaled_uniform(shape, rng, lo=-6, hi=6, scales=None):
    """float32 uniform in [-1, 1) times one power of ten per (n, c) plane (so max|x| of a plane is about its scale);
    returns (x, scales).  `scales` (N, C) reuses the scales of another tensor of the same planes."""
    sc = plane_scales(shape[0], shape[1], rng, lo, hi) if scales is None else scales
    x = rng.uniform(-1.0, 1.0, shape) * sc.reshape(sc.shape + (1,) * (len(shape) - 2))
    return x.astype(np.float32), sc


def plane_max(*arrs):
    """max |.| per (n, c) plane over several (N, C, ...) arrays (None entries are skipped)."""
    out = None
    for a in arrs:
        if a is None:
            continue
        a = np.abs(np.asarray(a, dtype=np.float64))
        m = a.reshape(a.shape[0], a.shape[1], -1).max(axis=2)
        out = m if out is None else np.maximum(out, m)
    return out
