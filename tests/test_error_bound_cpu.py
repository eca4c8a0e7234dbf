"""The per-plane fp32 error bound of tests/util.py, checked on the CPU at the shapes and scales of
tests/test_gpu_dtcwt_stream_sweep.py and tests/test_gpu_dwt_stream_sweep.py:
  soundness  the oracle's fp32 form and the host emulation of the shipped generic kernels (tests/emu) pass it against
             the float64 oracle evaluated on the same fp32 operands;
  tightness  one element of the smallest-scale plane moved by 1e-6 of that plane's scale fails it;
  report     the worst error / bound ratio per family is printed (-s); a bound far above what fp32 does (ratio below
             ~1/50) would be too loose to be useful."""
import numpy as np
import pytest

from oracle import oracle as orc
from pytorch_wavelets_b200.dtcwt._tables import TABLES
from pytorch_wavelets_b200.wavelets import Wavelet
from tests import util
from tests.emu import emu_backend as emu

IMPLS = {'oracle_f32': orc, 'emu_generic': emu}


def _rev(name, key):
    return np.array(TABLES[name][key])[::-1].copy()


def _f32(a):
    return np.asarray(a, dtype=np.float64).astype(np.float32)


def scaled_input(shape, seed, lo=-6, hi=6):
    return util.scaled_uniform(shape, np.random.default_rng(seed), lo, hi)


smax = util.plane_max


def z_nc_first(z):
    """ScatLayer (N, 7|6, C, h, w) -> (N, C, 7|6, h, w)."""
    return np.swapaxes(z, 1, 2)


# ---- the families: inputs, taps, and a function computing (outputs, bounds) with a given implementation ------------

def case_fwd_j1(biort, mode, shape=(2, 6, 38, 132), seed=1):
    x, sc = scaled_input(shape, seed)
    h0, h1 = _rev(biort, 'h0o'), _rev(biort, 'h1o')
    b = util.bound_fwd_j1(h0, h1)
    s = smax(x)

    def run(impl, dt):
        ll, hi = impl.dtcwt_fwd_j1(x.astype(dt), _f32(h0).astype(dt), _f32(h1).astype(dt), False, 2, -1, mode)
        return {'ll': ll, 'highs': hi}
    return run, {'ll': b['ll'] + (0.0,), 'highs': b['highs'] + (0.0,)}, s, sc


def case_fwd_j2plus(qshift, shape=(2, 6, 36, 136), seed=2):
    x, sc = scaled_input(shape, seed)
    f = [_rev(qshift, k) for k in ('h0a', 'h1a', 'h0b', 'h1b')]
    b = util.bound_fwd_j2plus(*f)
    s = smax(x)

    def run(impl, dt):
        ll, hi = impl.dtcwt_fwd_j2plus(x.astype(dt), *[_f32(t).astype(dt) for t in f], False, 2, -1)
        return {'ll': ll, 'highs': hi}
    return run, {'ll': b['ll'] + (0.0,), 'highs': b['highs'] + (0.0,)}, s, sc


def _inv_inputs(N, C, H, W, seed):
    rng = np.random.default_rng(seed)
    ll, sc = util.scaled_uniform((N, C, H, W), rng)
    hi, _ = util.scaled_uniform((N, C, 6, H // 2, W // 2, 2), rng, scales=sc)
    return ll, hi, sc


def case_inv_j1(biort, mode, has_ll=True, has_hi=True, shape=(2, 6, 36, 136), seed=3):
    ll, hi, sc = _inv_inputs(*shape, seed)
    ll, hi = (ll if has_ll else None), (hi if has_hi else None)
    g0, g1 = _rev(biort, 'g0o'), _rev(biort, 'g1o')
    s = smax(ll, hi)

    def run(impl, dt):
        return {'y': impl.dtcwt_inv_j1(None if ll is None else ll.astype(dt), None if hi is None else hi.astype(dt),
                                       _f32(g0).astype(dt), _f32(g1).astype(dt), 2, -1, mode)}
    return run, {'y': util.bound_inv_j1(g0, g1, has_ll, has_hi) + (0.0,)}, s, sc


def case_inv_j2plus(qshift, has_ll=True, has_hi=True, shape=(2, 6, 36, 136), seed=4):
    ll, hi, sc = _inv_inputs(*shape, seed)
    ll, hi = (ll if has_ll else None), (hi if has_hi else None)
    g = [_rev(qshift, k) for k in ('g0a', 'g1a', 'g0b', 'g1b')]
    s = smax(ll, hi)

    def run(impl, dt):
        return {'y': impl.dtcwt_inv_j2plus(None if ll is None else ll.astype(dt), None if hi is None else hi.astype(dt),
                                           *[_f32(t).astype(dt) for t in g])}
    return run, {'y': util.bound_inv_j2plus(*g, has_ll=has_ll, has_hi=has_hi) + (0.0,)}, s, sc


def case_scat(biort, mode, magbias, shape=(2, 6, 38, 132), seed=5):
    x, sc = scaled_input(shape, seed)
    h0, h1 = _rev(biort, 'h0o'), _rev(biort, 'h1o')
    b = util.bound_scat(h0, h1, magbias)
    s = smax(x)

    def run(impl, dt):
        z = impl.scat_j1(x.astype(dt), _f32(h0).astype(dt), _f32(h1).astype(dt), mode, magbias)
        z = z_nc_first(z)
        return {'avg': z[:, :, :1], 'mag': z[:, :, 1:]}
    return run, {'avg': b['avg'], 'mag': b['mag']}, s, sc


def case_dwt_sfb2d(L, mode, has_hi=True, shape=(2, 6, 19, 37), seed=6):
    """One DWT synthesis level with the dbL/2 synthesis filters (the filter lengths of the DWT stream sweep)."""
    rng = np.random.default_rng(seed + L)
    ll, sc = util.scaled_uniform(shape, rng)
    hi, _ = util.scaled_uniform(shape[:2] + (3,) + shape[2:], rng, scales=sc)
    hi = hi if has_hi else None
    w = Wavelet('db%d' % (L // 2))
    g0, g1 = _f32(w.rec_lo).astype(np.float64), _f32(w.rec_hi).astype(np.float64)
    s = smax(ll, hi)

    def run(impl, dt):
        return {'y': impl.dwt_sfb2d(ll.astype(dt), None if hi is None else hi.astype(dt), *[g.astype(dt) for g in
                                                                                             (g0, g1, g0, g1)], mode)}
    return run, {'y': util.bound_sfb2d(g0, g1, g0, g1, has_hi) + (0.0,)}, s, sc


INV_INPUTS = [(True, True), (False, True), (True, False)]   # (low-pass present, band-pass present)
DWT_MODES = ('zero', 'symmetric', 'reflect', 'periodic', 'periodization')
FAMILIES = {
    'fwd_j1': [lambda b=b, m=m: case_fwd_j1(b, m) for b in ('near_sym_a', 'near_sym_b', 'antonini', 'legall')
               for m in ('symmetric', 'zero')],
    'fwd_j2plus': [lambda q=q: case_fwd_j2plus(q) for q in ('qshift_a', 'qshift_b', 'qshift_c', 'qshift_d')],
    'inv_j1': [lambda b=b, m=m, p=p: case_inv_j1(b, m, *p) for b in ('near_sym_a', 'near_sym_b', 'antonini', 'legall')
               for m in ('symmetric', 'zero') for p in INV_INPUTS],
    'inv_j2plus': [lambda q=q, p=p: case_inv_j2plus(q, *p) for q in ('qshift_a', 'qshift_b', 'qshift_c', 'qshift_d')
                   for p in INV_INPUTS],
    'scat_j1': [lambda b=b, m=m, mb=mb: case_scat(b, m, mb) for b in ('near_sym_a', 'near_sym_b', 'antonini')
                for m in ('symmetric', 'zero') for mb in (1e-2, 0.0)],
    'dwt_sfb2d': [lambda L=L, m=m, h=h: case_dwt_sfb2d(L, m, h) for L in range(2, 21, 2) for m in DWT_MODES
                  for h in (True, False)],
}

_WORST = {}


@pytest.mark.parametrize('impl', sorted(IMPLS))
@pytest.mark.parametrize('family', sorted(FAMILIES))
def test_bound_is_sound(family, impl):
    worst = 0.0
    for make in FAMILIES[family]:
        run, bounds, s, _ = make()
        ref = run(orc, np.float64)
        got = run(IMPLS[impl], np.float32)
        for k, (G, K, add) in bounds.items():
            worst = max(worst, util.assert_plane_bound(got[k], ref[k], s, G, K, add, '%s %s %s' % (family, impl, k)))
    _WORST[(family, impl)] = worst
    print('\n%-11s %-11s worst error / bound = %.3f' % (family, impl, worst))
    # far below 1 everywhere would mean K is too large to notice small errors (see the tightness test)
    assert worst > 1.0 / 50, 'bound more than 50x above what fp32 does: lower K'


@pytest.mark.parametrize('family', sorted(FAMILIES))
def test_bound_is_tight(family):
    """An error of 1e-6 of the scale of the smallest-scale plane, in any one of its elements, breaks the bound (for every
    output of every case; the ScatLayer magnitudes only where magbias = 0, since a bias of 1e-2 puts the fp32 rounding
    of the root far above such a plane)."""
    for make in FAMILIES[family]:
        run, bounds, s, sc = make()
        ref = run(orc, np.float64)
        got = run(orc, np.float32)
        n, c = np.unravel_index(int(np.argmin(sc)), sc.shape)
        for k, (G, K, add) in bounds.items():
            if add > 0:
                continue
            y = np.array(got[k], dtype=np.float32)
            plane = y[n, c].reshape(-1)
            rng = np.random.default_rng(len(plane))
            for idx in (0, len(plane) - 1, int(rng.integers(len(plane)))):
                y2 = y.copy()
                y2[n, c].reshape(-1)[idx] += np.float32(1e-6 * sc[n, c])
                assert y2[n, c].reshape(-1)[idx] != y[n, c].reshape(-1)[idx]
                r = util.planes_err_ratio(y2, ref[k], s, G, K, add)
                assert r[n, c] > 1.0, '%s %s: an error of 1e-6 of the scale passes (ratio %.3f)' % (family, k, r[n, c])


def test_bound_flags_unwritten_outputs():
    run, bounds, s, _ = FAMILIES['fwd_j1'][0]()
    ref = run(orc, np.float64)
    y = np.array(run(orc, np.float32)['ll'])
    y[1, 2, 5, 7] = np.nan
    G, K, add = bounds['ll']
    with pytest.raises(AssertionError):
        util.assert_plane_bound(y, ref['ll'], s, G, K, add)
