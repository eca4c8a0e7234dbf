"""The shipped generic kernel source (tile_kernels.h + launch_params.h), compiled for the host as
a CTA/thread-loop emulation, against the oracle.  CPU only: validates index arithmetic, tiling,
boundary handling and argument checks of the code that nvcc compiles for sm_90a.  Every test takes the element type as
a parameter (float32 by default) and has a `_f64` twin over the same cases that runs the double-precision kernels
(behind the `_f64` entry points) against the oracle in double precision."""
import numpy as np
import pytest

from oracle import oracle as orc
from pytorch_wavelets_b200.dtcwt._tables import TABLES
from pytorch_wavelets_b200.wavelets import Wavelet
from tests import util
from tests.emu import emu_backend as emu

DWT_MODES = ['zero', 'symmetric', 'reflect', 'periodic', 'periodization']
AFB_CASES = [('db4', (2, 2, 64, 64)), ('db1', (1, 2, 33, 70)), ('db3', (1, 1, 37, 50)), ('db8', (1, 1, 96, 41)),
             ('db2', (1, 1, 5, 130)), ('db20', (1, 1, 70, 45))]
SFB_CASES = [('db4', (2, 2, 35, 35)), ('db1', (1, 2, 17, 40)), ('db3', (1, 1, 21, 27)), ('db8', (1, 1, 55, 28)),
             ('db20', (1, 1, 60, 41))]


def _afilt(wave):
    w = Wavelet(wave)
    return np.array(w.dec_lo[::-1]), np.array(w.dec_hi[::-1])


def _sfilt(wave):
    w = Wavelet(wave)
    return np.array(w.rec_lo), np.array(w.rec_hi)


def _rev(name, key):
    return np.array(TABLES[name][key])[::-1].copy()


def _eq(a, b, tol=0.0, what=''):
    assert a.shape == b.shape, (what, a.shape, b.shape)
    assert not np.isnan(a).any(), what + ': unwritten outputs'
    if tol == 0.0:
        assert np.array_equal(a, b), '%s: rel err %.3e' % (what, util.rel_err(a, b))
    else:
        util.assert_close(a, b, tol, what)


@pytest.mark.parametrize('mode', DWT_MODES)
@pytest.mark.parametrize('wave,shape', AFB_CASES)
def test_afb2d(mode, wave, shape, dtype=np.float32):
    rng = np.random.default_rng(hash((mode, wave)) % 1000)
    x = rng.standard_normal(shape).astype(dtype)
    f0, f1 = _afilt(wave)
    if mode == 'reflect' and min(shape[2:]) <= len(f0):
        pytest.skip('reflect pad larger than the signal (torch rejects it too)')
    ll, hi = emu.dwt_afb2d(x, f0, f1, f0, f1, mode)
    oll, ohi = orc.dwt_afb2d(x, f0, f1, f0, f1, mode)
    _eq(ll, oll, what='ll')
    _eq(hi, ohi, what='highs')


@pytest.mark.parametrize('mode', DWT_MODES)
@pytest.mark.parametrize('wave,shape', AFB_CASES)
def test_afb2d_f64(mode, wave, shape):
    test_afb2d(mode, wave, shape, np.float64)


def test_afb2d_distinct_row_col_filters(dtype=np.float32):
    rng = np.random.default_rng(3)
    x = rng.standard_normal((1, 2, 32, 48)).astype(dtype)
    a0, a1 = _afilt('db4')
    b0, b1 = _afilt('db2')
    for mode in DWT_MODES:
        ll, hi = emu.dwt_afb2d(x, a0, a1, b0, b1, mode)
        oll, ohi = orc.dwt_afb2d(x, a0, a1, b0, b1, mode)
        _eq(ll, oll)
        _eq(hi, ohi)


def test_afb2d_distinct_row_col_filters_f64():
    test_afb2d_distinct_row_col_filters(np.float64)


@pytest.mark.parametrize('mode', DWT_MODES)
@pytest.mark.parametrize('wave,shape', SFB_CASES)
def test_sfb2d(mode, wave, shape, dtype=np.float32):
    rng = np.random.default_rng(hash((mode, wave)) % 1000 + 7)
    ll = rng.standard_normal(shape).astype(dtype)
    hi = rng.standard_normal(shape[:2] + (3,) + shape[2:]).astype(dtype)
    g0, g1 = _sfilt(wave)
    _eq(emu.dwt_sfb2d(ll, hi, g0, g1, g0, g1, mode), orc.dwt_sfb2d(ll, hi, g0, g1, g0, g1, mode), what='y')
    _eq(emu.dwt_sfb2d(ll, None, g0, g1, g0, g1, mode), orc.dwt_sfb2d(ll, None, g0, g1, g0, g1, mode), what='y(None)')
    # cropped output (AFB2D.backward)
    full = orc.dwt_sfb2d(ll, hi, g0, g1, g0, g1, mode)
    crop = (full.shape[2] - 1, full.shape[3] - 1)
    _eq(emu.dwt_sfb2d(ll, hi, g0, g1, g0, g1, mode, out_hw=crop), full[:, :, :crop[0], :crop[1]], what='crop')


@pytest.mark.parametrize('mode', DWT_MODES)
@pytest.mark.parametrize('wave,shape', SFB_CASES)
def test_sfb2d_f64(mode, wave, shape):
    test_sfb2d(mode, wave, shape, np.float64)


BIORTS = ['near_sym_a', 'near_sym_b', 'antonini', 'legall']
QSHIFTS = ['qshift_a', 'qshift_b', 'qshift_c', 'qshift_d', 'qshift_06']
LAYOUTS = [(2, -1), (1, 2), (4, 5), (3, 1), (5, 2), (2, 3), (1, -1)]
Q2C_TOL = 3e-7  # x*(1/sqrt2) in the kernels vs x/sqrt2 in the oracle: 1 ulp


@pytest.mark.parametrize('biort', BIORTS)
@pytest.mark.parametrize('mode', ['symmetric', 'zero'])
def test_fwd_j1(biort, mode, dtype=np.float32):
    rng = np.random.default_rng(11)
    x = (100 * rng.standard_normal((2, 3, 38, 70))).astype(dtype)
    h0, h1 = _rev(biort, 'h0o'), _rev(biort, 'h1o')
    for (o, r) in (LAYOUTS if biort == 'near_sym_a' else LAYOUTS[:1]):
        ll, hi = emu.dtcwt_fwd_j1(x, h0, h1, False, o, r, mode)
        oll, ohi = orc.dtcwt_fwd_j1(x, h0, h1, False, o, r, mode)
        _eq(ll, oll, what='ll')
        _eq(hi, ohi, Q2C_TOL, 'highs o%d r%d' % (o, r))
    ll, hi = emu.dtcwt_fwd_j1(x, h0, h1, True, 2, -1, mode)
    assert hi is None
    _eq(ll, oll, what='ll skip')


@pytest.mark.parametrize('biort', BIORTS)
@pytest.mark.parametrize('mode', ['symmetric', 'zero'])
def test_fwd_j1_f64(biort, mode):
    test_fwd_j1(biort, mode, np.float64)


@pytest.mark.parametrize('qshift', QSHIFTS)
def test_fwd_j2plus(qshift, dtype=np.float32):
    rng = np.random.default_rng(12)
    x = (100 * rng.standard_normal((2, 2, 40, 72))).astype(dtype)
    f = [_rev(qshift, k) for k in ('h0a', 'h1a', 'h0b', 'h1b')]
    for (o, r) in (LAYOUTS if qshift == 'qshift_a' else LAYOUTS[:1]):
        ll, hi = emu.dtcwt_fwd_j2plus(x, *f, False, o, r)
        oll, ohi = orc.dtcwt_fwd_j2plus(x, *f, False, o, r)
        _eq(ll, oll, what='ll')
        _eq(hi, ohi, Q2C_TOL, 'highs')
    ll, hi = emu.dtcwt_fwd_j2plus(x, *f, True)
    assert hi is None
    _eq(ll, oll)
    with pytest.raises(ValueError):
        emu.dtcwt_fwd_j2plus(x[:, :, :38], *f)


@pytest.mark.parametrize('qshift', QSHIFTS)
def test_fwd_j2plus_f64(qshift):
    test_fwd_j2plus(qshift, np.float64)


@pytest.mark.parametrize('biort', BIORTS)
@pytest.mark.parametrize('mode', ['symmetric', 'zero'])
def test_inv_j1(biort, mode, dtype=np.float32):
    rng = np.random.default_rng(13)
    g0, g1 = _rev(biort, 'g0o'), _rev(biort, 'g1o')
    N, C, H, W = 2, 2, 36, 68
    ll = rng.standard_normal((N, C, H, W)).astype(dtype)
    for (o, r) in (LAYOUTS if biort == 'near_sym_a' else LAYOUTS[:1]):
        shape, _ = orc.highs_shape_strides(N, C, H // 2, W // 2, o, r)
        hi = rng.standard_normal(shape).astype(dtype)
        _eq(emu.dtcwt_inv_j1(ll, hi, g0, g1, o, r, mode), orc.dtcwt_inv_j1(ll, hi, g0, g1, o, r, mode), 5e-7, 'full')
        _eq(emu.dtcwt_inv_j1(None, hi, g0, g1, o, r, mode), orc.dtcwt_inv_j1(None, hi, g0, g1, o, r, mode), 5e-7, 'no ll')
    _eq(emu.dtcwt_inv_j1(ll, None, g0, g1, 2, -1, mode), orc.dtcwt_inv_j1(ll, None, g0, g1, 2, -1, mode), 0.0, 'no highs')
    # ll two rows/cols larger than 2x highs: inv_j1 trims it (transform_funcs.py:170-176)
    shape, _ = orc.highs_shape_strides(N, C, H // 2 - 1, W // 2 - 1, 2, -1)
    hi = rng.standard_normal(shape).astype(dtype)
    _eq(emu.dtcwt_inv_j1(ll, hi, g0, g1, 2, -1, mode), orc.dtcwt_inv_j1(ll, hi, g0, g1, 2, -1, mode), 5e-7, 'trim')


@pytest.mark.parametrize('biort', BIORTS)
@pytest.mark.parametrize('mode', ['symmetric', 'zero'])
def test_inv_j1_f64(biort, mode):
    test_inv_j1(biort, mode, np.float64)


@pytest.mark.parametrize('qshift', QSHIFTS)
def test_inv_j2plus(qshift, dtype=np.float32):
    rng = np.random.default_rng(14)
    g = [_rev(qshift, k) for k in ('g0a', 'g1a', 'g0b', 'g1b')]
    N, C, H, W = 2, 2, 20, 36
    ll = rng.standard_normal((N, C, H, W)).astype(dtype)
    for (o, r) in (LAYOUTS if qshift == 'qshift_a' else LAYOUTS[:1]):
        shape, _ = orc.highs_shape_strides(N, C, H // 2, W // 2, o, r)
        hi = rng.standard_normal(shape).astype(dtype)
        _eq(emu.dtcwt_inv_j2plus(ll, hi, *g, o, r), orc.dtcwt_inv_j2plus(ll, hi, *g, o, r), 5e-7, 'full')
        _eq(emu.dtcwt_inv_j2plus(None, hi, *g, o, r), orc.dtcwt_inv_j2plus(None, hi, *g, o, r), 5e-7, 'no ll')
    _eq(emu.dtcwt_inv_j2plus(ll, None, *g), orc.dtcwt_inv_j2plus(ll, None, *g), 0.0, 'no highs')


@pytest.mark.parametrize('qshift', QSHIFTS)
def test_inv_j2plus_f64(qshift):
    test_inv_j2plus(qshift, np.float64)


@pytest.mark.parametrize('biort', ['near_sym_a', 'near_sym_b'])
@pytest.mark.parametrize('mode', ['symmetric', 'zero'])
def test_scat_j1(biort, mode, dtype=np.float32):
    rng = np.random.default_rng(15)
    x = rng.standard_normal((2, 3, 34, 66)).astype(dtype)
    h0, h1 = _rev(biort, 'h0o'), _rev(biort, 'h1o')
    z, dre, dim = emu.scat_j1(x, h0, h1, mode, 1e-2, True)
    oz, odre, odim = orc.scat_j1(x, h0, h1, mode, 1e-2, True)
    _eq(z, oz, 5e-7, 'z')
    _eq(dre, odre, 2e-5, 'dre')  # re/r: relative error amplified where r ~ bias
    _eq(dim, odim, 2e-5, 'dim')
    _eq(emu.scat_j1(x, h0, h1, mode, 1e-2), oz, 5e-7, 'z (no aux)')



@pytest.mark.parametrize('biort', ['near_sym_a', 'near_sym_b'])
@pytest.mark.parametrize('mode', ['symmetric', 'zero'])
def test_scat_j1_f64(biort, mode):
    test_scat_j1(biort, mode, np.float64)