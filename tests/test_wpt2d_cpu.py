"""CPU: the 2-D wavelet packet transform's C ABI validation, host API, and the oracle composition it is tested against
(no GPU)."""
import ctypes

import numpy as np
import pytest
import torch

import pytorch_wavelets_b200 as pw
from pytorch_wavelets_b200 import _build, _ffi, wavelets
from oracle import oracle as orc
from tests import oracle_wpt2d as ow

MODES = ['zero', 'symmetric', 'reflect', 'periodic', 'periodization']


@pytest.fixture(scope='module')
def lib():
    _build.build()
    return _ffi.lib()


def _filts(wave, analysis, dtype=np.float64):
    m = pw.DWTForward(wave=wave) if analysis else pw.DWTInverse(wave=wave)
    names = ('h0_col', 'h1_col', 'h0_row', 'h1_row') if analysis else ('g0_col', 'g1_col', 'g0_row', 'g1_row')
    if isinstance(wave, str):
        w = wavelets.Wavelet(wave)
        lo, hi = (w.dec_lo[::-1], w.dec_hi[::-1]) if analysis else (w.rec_lo, w.rec_hi)
        return tuple(np.array(f, dtype) for f in (lo, hi, lo, hi))
    return tuple(getattr(m, n).double().numpy().ravel().astype(dtype) for n in names)


# ---- C ABI -------------------------------------------------------------------------------------------------------------

def test_abi_validates_without_gpu(lib):
    f = (ctypes.c_float * 8)(*([0.5] * 8))
    fp = ctypes.cast(f, ctypes.c_void_p)
    d = (ctypes.c_double * 8)(*([0.5] * 8))
    dp = ctypes.cast(d, ctypes.c_void_p)
    buf = ctypes.c_void_p(16)   # never dereferenced: validation fails first
    # 16 x 16 planes, db4 (8 taps), symmetric: Ho = Wo = 11
    for v, t in (('', fp), ('_generic', fp), ('_f64', dp)):
        afb = getattr(lib, 'b200w_wpt_afb2d' + v)
        sfb = getattr(lib, 'b200w_wpt_sfb2d' + v)
        ok = (buf, 256, 16, buf, 121, 11, 2, 16, 16, t, t, 8, t, t, 8, 1, None)

        def a(**kw):
            args = list(ok)
            for k, val in kw.items():
                args[int(k[1:])] = val
            return afb(*args)
        assert a(a15=3) == -1 and a(a15=99) == -1                       # 'constant', unknown
        assert a(a0=None) == -3 and a(a3=None) == -3 and a(a9=None) == -3
        assert a(a2=15) == -3                                              # x pitch below W
        assert a(a5=10) == -3                                              # y pitch below Wo
        assert a(a4=120) == -3                                             # node stride below Ho * pitch
        assert a(a6=-1) == -2 and a(a7=0) == -2 and a(a8=0) == -2          # sizes
        assert a(a11=1) == -4 and a(a14=1) == -4 and a(a11=41) == -4     # lengths outside 2 .. 40
        assert a(a6=0) == 0                                                # no planes: nothing to do
        # Lw != Lh is allowed: with Lw = 4, Wo = 9 and the call validates (zero planes, no launch)
        assert a(a11=4, a6=0) == 0
        sok = (buf, buf, 256, 16, 2, 11, 11, 16, 16, t, t, 8, t, t, 8, 1, None)

        def s(**kw):
            args = list(sok)
            for k, val in kw.items():
                args[int(k[1:])] = val
            return sfb(*args)
        assert s(a15=5) == -1
        assert s(a0=None) == -3 and s(a1=None) == -3 and s(a9=None) == -3
        assert s(a3=15) == -3                                              # y pitch below Wo
        assert s(a2=255) == -3                                             # plane stride below Ho * pitch
        assert s(a7=17) == -2 and s(a8=0) == -2 and s(a5=0) == -2 and s(a4=-1) == -2   # Ho > rec_len, sizes
        assert s(a11=1) == -4 and s(a14=42) == -4
        assert s(a4=0) == 0


def test_abi_rejects_a_grid_that_is_too_large(lib):
    f = (ctypes.c_float * 2)(0.5, 0.5)
    fp = ctypes.cast(f, ctypes.c_void_p)
    buf = ctypes.c_void_p(16)
    # 2^31 - 1 planes of 4096 x 4096 coefficients: far more tiles than a 1-D grid holds
    n = 2 ** 31 - 1
    assert lib.b200w_wpt_afb2d_generic(buf, 8192 * 8192, 8192, buf, 4096 * 4096, 4096, n, 8192, 8192,
                                       fp, fp, 2, fp, fp, 2, 2, None) == -2
    assert lib.b200w_wpt_sfb2d_generic(buf, buf, 8192 * 8192, 8192, n, 4096, 4096, 8192, 8192,
                                       fp, fp, 2, fp, fp, 2, 2, None) == -2


# ---- host API ----------------------------------------------------------------------------------------------------------

def test_modules_buffers_state_dict_and_exports():
    assert pw.WPT2D is pw.WPT2DForward and pw.IWPT2D is pw.WPT2DInverse
    for name in ('WPT2DForward', 'WPT2DInverse', 'WPT2D', 'IWPT2D'):
        assert name in pw.__all__
    w = wavelets.Wavelet('db3')
    for wave in ('db4', w, (w.dec_lo, w.dec_hi), (w.dec_lo, w.dec_hi, wavelets.Wavelet('db2').dec_lo,
                                                  wavelets.Wavelet('db2').dec_hi)):
        f, d = pw.WPT2DForward(J=2, wave=wave, mode='symmetric'), pw.DWTForward(J=2, wave=wave, mode='symmetric')
        assert list(f.state_dict()) == list(d.state_dict())
        for k, v in d.state_dict().items():
            assert torch.equal(f.state_dict()[k], v)
    inv_wave = (w.rec_lo, w.rec_hi)
    for wave in ('db4', w, inv_wave):
        i, d = pw.WPT2DInverse(wave=wave, mode='zero'), pw.DWTInverse(wave=wave, mode='zero')
        assert list(i.state_dict()) == list(d.state_dict())
        for k, v in d.state_dict().items():
            assert torch.equal(i.state_dict()[k], v)
    f = pw.WPT2DForward(J=1, wave='db2')
    d = pw.DWTForward(J=1, wave='db2')
    d.h0_col.mul_(2)
    f.load_state_dict(d.state_dict())
    assert torch.equal(f.h0_col, d.h0_col)


def test_modules_raise():
    x = torch.randn(1, 2, 16, 16)
    for J in (0, 2):
        with pytest.raises(NotImplementedError):
            pw.WPT2DForward(J=J, wave='db2')(x)                            # CPU tensor
        with pytest.raises(NotImplementedError):
            pw.WPT2DForward(J=J, wave='db2')(x.half())
    y = torch.randn(1, 2, 16, 5, 5)
    with pytest.raises(NotImplementedError):
        pw.WPT2DInverse(wave='db2')(y)
    with pytest.raises(NotImplementedError):
        pw.WPT2DInverse(wave='db2')(y.half())
    with pytest.raises(ValueError):
        pw.WPT2DForward(J=1, mode='constant')(x)
    with pytest.raises(ValueError):
        pw.WPT2DInverse(mode='replicate')(y)
    # checked before the device: a node count that is not a power of 4, a size that does not lead to (Hc, Wc)
    for n in (2, 3, 5, 8, 15):
        with pytest.raises(ValueError):
            pw.WPT2DInverse(wave='db2')(torch.randn(1, 2, n, 5, 5))
    inv = pw.WPT2DInverse(wave='db2', mode='symmetric')
    for size in ((6, 6), (12, 16), (16, 12)):                     # 6 -> 4 -> 3, 12 -> 7 -> 5
        with pytest.raises(ValueError):
            inv(torch.randn(1, 2, 16, 6, 6), size=size)
    with pytest.raises(NotImplementedError):                      # 16 -> 9 -> 6: consistent, then the device check
        inv(torch.randn(1, 2, 16, 6, 6), size=(16, 16))


# ---- the oracle composition ------------------------------------------------------------------------------------------

@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('wave,shape,J', [('haar', (2, 2, 16, 24), 3), ('db2', (1, 2, 19, 23), 4),
                                          ('db4', (2, 1, 37, 29), 2), ('db3', (1, 1, 9, 7), 1)])
def test_oracle_composition_reconstructs_in_float64(wave, shape, J, mode):
    rng = np.random.default_rng(J)
    x = rng.standard_normal(shape)
    y = ow.wpt2d_forward(x, _filts(wave, True), J, mode)
    assert y.shape[:3] == shape[:2] + (4 ** J,)
    Lf = len(wavelets.Wavelet(wave).dec_lo)
    sizes = ow.forward_sizes(shape[2], shape[3], J, Lf, Lf, mode)
    assert y.shape[-2:] == sizes[-1]
    xr = ow.wpt2d_inverse(y, _filts(wave, False), mode, sizes=sizes[:-1])
    assert xr.shape == x.shape
    assert np.abs(xr - x).max() <= 1e-12 * np.abs(x).max()
    if mode == 'periodization' and any(h % 2 or w % 2 for h, w in sizes[:-1]):
        return   # an odd level size: the natural (even) rec_len sizes do not rebuild the cropped levels' signals
    # natural sizes: the rebuilt signal starts with x (each level's rec_len is at least its input size)
    xn = ow.wpt2d_inverse(y, _filts(wave, False), mode)
    np.testing.assert_allclose(xn[..., :shape[2], :shape[3]], x, rtol=0, atol=1e-12 * np.abs(x).max())


@pytest.mark.parametrize('mode', MODES)
def test_oracle_composition_node0_is_the_dwt_lowpass(mode):
    rng = np.random.default_rng(7)
    x = rng.standard_normal((2, 3, 45, 38)).astype(np.float32)
    filts = _filts('db2', True, np.float32)
    y = ow.wpt2d_forward(x, filts, 3, mode)
    yl, yh = orc.dwt_forward(x, filts, 3, mode)
    assert np.array_equal(y[:, :, 0], yl)
    # J = 1 is the DWT level's four bands, stacked
    y1 = ow.wpt2d_forward(x, filts, 1, mode)
    yl1, yh1 = orc.dwt_forward(x, filts, 1, mode)
    assert np.array_equal(y1, np.concatenate([yl1[:, :, None], yh1[0]], 2))


def test_oracle_composition_natural_order():
    """Node 4p + b of level j + 1 is band b of node p of level j: the base-4 digits, first level most significant."""
    rng = np.random.default_rng(3)
    x = rng.standard_normal((1, 1, 20, 20))
    f = _filts('haar', True)
    y2 = ow.wpt2d_forward(x, f, 2, 'zero')
    y1 = ow.wpt2d_forward(x, f, 1, 'zero')
    for p in range(4):
        ll, hi = orc.dwt_afb2d(y1[:, :, p], *f, 'zero')
        bands = np.concatenate([ll[:, :, None], hi], 2)
        for b in range(4):
            assert np.array_equal(y2[:, :, 4 * p + b], bands[:, :, b])
