"""CPU: the 3-D DWT's C ABI validation, host API, and the oracle composition it is tested against (no GPU)."""
import ctypes

import numpy as np
import pytest
import torch

import pytorch_wavelets_b200 as pw
from pytorch_wavelets_b200 import _build, _ffi, wavelets
from oracle import oracle as orc
from tests import oracle3d as o3
from tests import util

MODES = ['zero', 'symmetric', 'reflect', 'periodic', 'periodization']
MODE_INT = {'zero': 0, 'symmetric': 1, 'periodization': 2, 'reflect': 4, 'periodic': 6}


@pytest.fixture(scope='module')
def lib():
    _build.build()
    return _ffi.lib()


def _filters(name):
    w = wavelets.Wavelet(name)
    return (np.array(w.dec_lo[::-1]), np.array(w.dec_hi[::-1])), (np.array(w.rec_lo), np.array(w.rec_hi))


# ---- C ABI -------------------------------------------------------------------------------------------------------------

def test_abi_validates_without_gpu(lib):
    f = (ctypes.c_float * 8)(*([0.5] * 8))
    fp = ctypes.cast(f, ctypes.c_void_p)
    d = (ctypes.c_double * 8)(*([0.5] * 8))
    dp = ctypes.cast(d, ctypes.c_void_p)
    buf = ctypes.c_void_p(16)   # never dereferenced: validation fails first
    for v, taps in (('', fp), ('_generic', fp), ('_f64', dp)):
        afb = getattr(lib, 'b200w_dwt_afb3d' + v)
        sfb = getattr(lib, 'b200w_dwt_sfb3d' + v)
        assert afb(buf, 512, buf, buf, 1, 8, 8, 8, taps, taps, 8, 3, None, 0, None) == -1      # 'constant'
        assert afb(buf, 512, buf, buf, 1, 8, 8, 8, taps, taps, 8, 99, None, 0, None) == -1
        assert afb(None, 512, buf, buf, 1, 8, 8, 8, taps, taps, 8, 1, None, 0, None) == -3
        assert afb(buf, 512, buf, None, 1, 8, 8, 8, taps, taps, 8, 1, None, 0, None) == -3
        assert afb(buf, 512, buf, buf, 1, 8, 8, 8, None, taps, 8, 1, None, 0, None) == -3
        assert afb(buf, 512, buf, buf, 1, 8, 8, 8, taps, taps, 1, 1, None, 0, None) == -4     # L < 2
        assert afb(buf, 511, buf, buf, 1, 8, 8, 8, taps, taps, 8, 1, None, 0, None) == -3     # volume stride < D*H*W
        assert sfb(buf, 64, buf, buf, 1, 4, 4, 4, 2, 2, 2, taps, taps, 8, 5, None, 0, None) == -1
        assert sfb(None, 64, buf, buf, 1, 4, 4, 4, 2, 2, 2, taps, taps, 8, 1, None, 0, None) == -3
        assert sfb(buf, 64, buf, None, 1, 4, 4, 4, 2, 2, 2, taps, taps, 8, 1, None, 0, None) == -3
        assert sfb(buf, 64, buf, buf, 1, 4, 4, 4, 2, 2, 2, taps, taps, 1, 1, None, 0, None) == -4
        assert sfb(buf, 64, buf, buf, 1, 4, 4, 4, 3, 2, 2, taps, taps, 8, 1, None, 0, None) == -2  # Do > rec_len = 2
    # the two-step route needs its workspace: a missing one is an argument error, found before any launch
    assert lib.b200w_dwt_afb3d_generic(buf, 512, buf, buf, 1, 8, 8, 8, fp, fp, 8, 1, None, 0, None) == -3
    assert lib.b200w_dwt_sfb3d_f64(buf, 64, None, buf, 1, 4, 4, 4, 2, 2, 2, dp, dp, 8, 1, None, 0, None) == -3
    # no volumes: nothing to do
    assert lib.b200w_dwt_afb3d(buf, 512, buf, buf, 0, 8, 8, 8, fp, fp, 8, 1, None, 0, None) == 0


def test_workspace_queries(lib):
    """0 where the fused float32 kernel applies (L = 2 ... 8), else the two-step layout: the 2-D level's ll and three
    band-pass planes for every (volume, slice), each part rounded up to 256 bytes."""
    def two_step(elems, esz):
        return (elems * esz + 255) // 256 * 256 + (3 * elems * esz + 255) // 256 * 256
    vols, D, H, W = 3, 9, 20, 17
    for L in (2, 4, 6, 8, 10, 16):
        for m in MODE_INT.values():
            Ho, Wo = (lib.b200w_dwt_coeff_len(n, L, m) for n in (H, W))
            want = two_step(vols * D * Ho * Wo, 4)
            got = lib.b200w_dwt_afb3d_workspace(None, D * H * W, vols, D, H, W, L, m)
            assert got == (0 if L <= 8 else want)
            assert lib.b200w_dwt_afb3d_workspace_generic(None, D * H * W, vols, D, H, W, L, m) == want
            assert lib.b200w_dwt_afb3d_workspace_f64(None, D * H * W, vols, D, H, W, L, m) == two_step(
                vols * D * Ho * Wo, 8)
            Dc, Hc, Wc = 12, 13, 14
            Do = lib.b200w_dwt_rec_len(Dc, L, m) - 1
            Ho, Wo = lib.b200w_dwt_rec_len(Hc, L, m), lib.b200w_dwt_rec_len(Wc, L, m)
            want = two_step(vols * Do * Hc * Wc, 4)
            assert lib.b200w_dwt_sfb3d_workspace(vols, Dc, Hc, Wc, Do, Ho, Wo, L, m) == (0 if L <= 8 else want)
            assert lib.b200w_dwt_sfb3d_workspace_generic(vols, Dc, Hc, Wc, Do, Ho, Wo, L, m) == want
            assert lib.b200w_dwt_sfb3d_workspace_f64(vols, Dc, Hc, Wc, Do, Ho, Wo, L, m) == two_step(
                vols * Do * Hc * Wc, 8)
    assert lib.b200w_dwt_afb3d_workspace(None, 512, 1, 8, 8, 8, 8, 3) == -1
    assert lib.b200w_dwt_afb3d_workspace(None, 512, 1, 8, 8, 8, 1, 1) == -4
    assert lib.b200w_dwt_sfb3d_workspace(1, 4, 4, 4, 9, 4, 4, 4, 1) == -2


# ---- host API ----------------------------------------------------------------------------------------------------------

def test_modules_buffers_and_exports():
    assert pw.DWT3D is pw.DWT3DForward and pw.IDWT3D is pw.DWT3DInverse
    for name in ('DWT3DForward', 'DWT3DInverse', 'DWT3D', 'IDWT3D'):
        assert name in pw.__all__
    (h0, h1), (g0, g1) = _filters('db4')
    f = pw.DWT3DForward(J=2, wave='db4', mode='symmetric')
    assert sorted(n for n, _ in f.named_buffers()) == ['h0', 'h1']
    assert tuple(f.h0.shape) == (1, 1, 8) and tuple(f.h1.shape) == (1, 1, 8)
    np.testing.assert_array_equal(f.h0.numpy().ravel(), h0.astype(np.float32))   # stored reversed
    np.testing.assert_array_equal(f.h1.numpy().ravel(), h1.astype(np.float32))
    i = pw.DWT3DInverse(wave='db4', mode='symmetric')
    assert sorted(n for n, _ in i.named_buffers()) == ['g0', 'g1']
    np.testing.assert_array_equal(i.g0.numpy().ravel(), g0.astype(np.float32))
    np.testing.assert_array_equal(i.g1.numpy().ravel(), g1.astype(np.float32))
    w = wavelets.Wavelet('db2')
    t = pw.DWT3DForward(wave=(w.dec_lo, w.dec_hi))
    np.testing.assert_array_equal(t.h0.numpy().ravel(), np.array(w.dec_lo[::-1], np.float32))
    o = pw.DWT3DForward(wave=w)
    np.testing.assert_array_equal(o.h1.numpy().ravel(), np.array(w.dec_hi[::-1], np.float32))


def test_modules_raise_like_the_2d_shells():
    x = torch.randn(1, 1, 4, 8, 8)
    with pytest.raises(NotImplementedError):
        pw.DWT3DForward(J=1, wave='db2')(x)                                  # CPU tensor
    with pytest.raises(NotImplementedError):
        pw.DWT3DForward(J=1, wave='db2').double()(x.double())
    with pytest.raises(NotImplementedError):
        pw.DWT3DForward(J=1, wave='db2')(x.half())
    with pytest.raises(NotImplementedError):
        pw.DWT3DInverse(wave='db2')((torch.randn(1, 1, 3, 5, 5), [torch.randn(1, 1, 7, 3, 5, 5)]))
    with pytest.raises(ValueError):
        pw.DWT3DForward(J=1)(torch.randn(1, 8, 8, 8))                        # not 5-D
    with pytest.raises(ValueError):
        pw.DWT3DInverse()((torch.randn(1, 8, 8, 8), []))
    for bad in ('constant', 'replicate', 'nope'):
        with pytest.raises(ValueError, match='Unkown pad type'):
            pw.DWT3DForward(J=1, mode=bad)(x)
        with pytest.raises(ValueError, match='Unkown pad type'):
            pw.DWT3DInverse(mode=bad)((x, []))


def test_j0_returns_the_input():
    x = torch.randn(2, 1, 4, 8, 8)
    yl, yh = pw.DWT3DForward(J=0)(x)
    assert yl is x and yh == []


# ---- the oracle composition -----------------------------------------------------------------------------------------------

@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('wave', ['haar', 'db4', 'sym3', 'db8'])
def test_oracle_perfect_reconstruction_f64(mode, wave):
    (h0, h1), (g0, g1) = _filters(wave)
    rng = np.random.default_rng(3)
    x = rng.standard_normal((2, 2, 9, 12, 11))
    J = 1 if wave == 'db8' else 2
    yl, yh = o3.dwt3d_forward(x, (h0, h1), J, mode)
    assert yh[0].shape[2] == 7
    y = o3.dwt3d_inverse(yl, yh, (g0, g1), mode)
    assert np.abs(y[:, :, :9, :12, :11] - x).max() <= 1e-12 * np.abs(x).max()


@pytest.mark.parametrize('mode', ['symmetric', 'reflect', 'periodic', 'periodization'])
def test_oracle_d_constant_identity(mode):
    """An input constant along D: yl and bands 1, 3, 5 are sum(h0) times the 2-D transform of one slice, bands 0, 2, 4,
    6 are zero (the extension of a constant is that constant in these modes)."""
    (h0, h1), _ = _filters('db3')
    rng = np.random.default_rng(4)
    s = rng.standard_normal((2, 3, 1, 14, 13))
    x = np.repeat(s, 10, axis=2)
    yl, yh = o3.dwt_afb3d(x, h0, h1, mode)
    ll2, hi2 = orc.dwt_afb2d(s[:, :, 0], h0, h1, h0, h1, mode)
    k = h0.sum()
    np.testing.assert_allclose(yl, np.broadcast_to(k * ll2[:, :, None], yl.shape), atol=1e-12)
    for v in range(3):
        want = np.broadcast_to(k * hi2[:, :, v][:, :, None], yl.shape)
        np.testing.assert_allclose(yh[:, :, 2 * v + 1], want, atol=1e-12)
    for b in (0, 2, 4, 6):
        assert np.abs(yh[:, :, b]).max() < 1e-12


def test_synthesis_bound_holds_and_detects():
    """K of bound_sfb3d: the fp32 oracle in both pass orders (D first, as the two-step route; in-plane first, as the
    fused kernel) stays within the per-volume bound with margin, and an error of 1e-6 of the scale in one element of
    the smallest volume breaks it, for every fused filter length and all five modes."""
    rng = np.random.default_rng(1)
    worst, caught = 0.0, np.inf
    for wave in ('haar', 'db2', 'db3', 'db4', 'sym4', 'coif1'):
        _, (g0, g1) = _filters(wave)
        for mode in MODES:
            for has_hi in (True, False):
                yl, sc = util.scaled_uniform((2, 3, 9, 10, 11), rng)
                hi = util.scaled_uniform((2, 3, 7, 9, 10, 11), rng, scales=sc)[0] if has_hi else None
                s = util.plane_max(yl, None if hi is None else hi.reshape(2, 3, -1))
                y64 = o3.dwt_sfb3d(yl.astype(np.float64), None if hi is None else hi.astype(np.float64), g0, g1, mode)
                G, K = o3.bound_sfb3d(g0, g1, has_hi)
                for fn in (o3.dwt_sfb3d, o3.dwt_sfb3d_plane_first):
                    worst = max(worst, util.planes_err_ratio(fn(yl, hi, g0, g1, mode), y64, s, G, K).max())
                n, c = np.unravel_index(np.argmin(s), s.shape)
                y = o3.dwt_sfb3d(yl, hi, g0, g1, mode).copy()
                y[n, c, 0, 0, 0] += 1e-6 * s[n, c]
                caught = min(caught, util.planes_err_ratio(y, y64, s, G, K)[n, c])
    print('sfb3d bound: worst error / bound %.2f, smallest injected error / bound %.2f' % (worst, caught))
    assert worst <= 0.8
    assert caught > 1.0
