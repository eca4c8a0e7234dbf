"""CPU: the operators behind the DWT's double backward, pinned as dense matrices of the oracle, and the new C entries'
argument validation (no GPU).

Autograd differentiates each first-order backward pass B into its transpose B^T:
  AFB:  B = crop . S          B^T = S^T . pad = the zero-mode analysis (periodization: of the signal padded to even n)
  SFB:  B = A_m               B^T = A_m^T, the transposed analysis with the boundary extension folded back
"""
import ctypes

import numpy as np
import pytest

from oracle import oracle as orc
from tests import oracle_dwt_adjoint as oa
from pytorch_wavelets_b200 import _build, _ffi

LENGTHS = list(range(2, 21))


def taps(L, seed):
    r = np.random.default_rng(seed)
    return r.standard_normal(L), r.standard_normal(L)


def sizes(L):
    return sorted({1, 2, 3, L - 1, L, L + 1, 2 * L + 3, 2 * L + 4} - {0})


@pytest.mark.parametrize('mode', oa.MODES)
@pytest.mark.parametrize('L', LENGTHS)
def test_crop_synthesis_transpose_is_zero_mode_analysis(mode, L):
    if mode == 'periodization' and L % 2:
        pytest.skip('odd-length periodization synthesis is offset from the analysis (L/2 - 1 vs L - 1 - L/2)')
    f0, f1 = taps(L, L)
    for n in sizes(L):
        K = orc.coeff_len(n, L, mode)
        S = oa.dense_sfb1d(f0, f1, K, mode, n)                   # AFB1D.backward: crop_n . S
        if mode == 'periodization':
            npad = n + (n & 1)
            A = oa.dense_afb1d(f0, f1, npad, mode)[:, :n]         # analysis of the zero-padded signal
        else:
            A = oa.dense_afb1d(f0, f1, n, 'zero')
        assert A.shape == S.T.shape
        np.testing.assert_allclose(S.T, A, rtol=0, atol=1e-13, err_msg='n=%d' % n)


@pytest.mark.parametrize('mode', oa.MODES)
@pytest.mark.parametrize('L', LENGTHS)
def test_restated_adjoint_is_transposed_analysis(mode, L):
    f0, f1 = taps(L, 100 + L)
    for n in sizes(L):
        A = oa.dense_afb1d(f0, f1, n, mode)
        T = np.concatenate([oa.adjoint_matrix_1d(f0, n, mode), oa.adjoint_matrix_1d(f1, n, mode)], axis=1)
        np.testing.assert_allclose(T, A.T, rtol=0, atol=1e-13, err_msg='n=%d' % n)


@pytest.mark.parametrize('mode', oa.MODES)
@pytest.mark.parametrize('L', LENGTHS)
def test_adjoint_differs_from_crop_synthesis_only_at_the_border(mode, L):
    """The kernel's route: the cropped synthesis everywhere, then the outputs within L of an edge rewritten (the whole
    axis in periodization with odd L).  Outside that border the two agree."""
    f0, f1 = taps(L, 200 + L)
    for n in sizes(L):
        K = orc.coeff_len(n, L, mode)
        S = oa.dense_sfb1d(f0, f1, K, mode, n)
        T = np.concatenate([oa.adjoint_matrix_1d(f0, n, mode), oa.adjoint_matrix_1d(f1, n, mode)], axis=1)
        depth = n if (mode == 'periodization' and L % 2) else L
        inner = slice(depth, max(depth, n - depth))
        np.testing.assert_allclose(S[inner], T[inner], rtol=0, atol=1e-13, err_msg='n=%d' % n)
        exact = mode == 'zero' or (mode == 'periodization' and n % 2 == 0 and L % 2 == 0)
        if exact:   # the C entry launches only the synthesis here
            np.testing.assert_allclose(S, T, rtol=0, atol=1e-13, err_msg='n=%d' % n)


@pytest.mark.parametrize('mode', oa.MODES)
@pytest.mark.parametrize('H,W,Lh,Lw', [(7, 6, 4, 6), (3, 9, 8, 2), (10, 5, 6, 6), (1, 4, 4, 4)])
def test_adjoint_2d_composition_order(mode, H, W, Lh, Lw):
    """A = A_H . A_W (W first), so A^T = A_W^T . A_H^T: the 2-D restatement against the oracle's dense matrix."""
    r = np.random.default_rng(H * 100 + W)
    fw_lo, fw_hi, fh_lo, fh_hi = r.standard_normal(Lw), r.standard_normal(Lw), r.standard_normal(Lh), r.standard_normal(Lh)
    A = oa.dense_afb2d(fw_lo, fw_hi, fh_lo, fh_hi, H, W, mode)
    Hc, Wc = orc.coeff_len(H, Lh, mode), orc.coeff_len(W, Lw, mode)
    c = r.standard_normal((2, 4, Hc, Wc))
    y = oa.afb2d_adjoint(c[:, 0], c[:, 1:], fh_lo, fh_hi, fw_lo, fw_hi, mode, H, W)
    ref = c.reshape(2, -1) @ A
    np.testing.assert_allclose(y.reshape(2, -1), ref, rtol=0, atol=1e-12)
    # and the cropped synthesis is the transpose of the zero-mode (padded periodization) analysis in 2-D too
    S = oa.dense_sfb2d(fh_lo, fh_hi, fw_lo, fw_hi, Hc, Wc, mode, out_hw=(H, W))
    if mode == 'periodization':
        Hp, Wp = H + H % 2, W + W % 2
        Z = oa.dense_afb2d(fw_lo, fw_hi, fh_lo, fh_hi, Hp, Wp, mode).reshape(-1, Hp, Wp)[:, :H, :W].reshape(-1, H * W)
    else:
        Z = oa.dense_afb2d(fw_lo, fw_hi, fh_lo, fh_hi, H, W, 'zero')
    np.testing.assert_allclose(S.T, Z, rtol=0, atol=1e-12)


# ---- the C entries validate their arguments before any CUDA call ---------------------------------------------------

@pytest.fixture(scope='module')
def lib():
    _build.build()
    return _ffi.lib()


def test_adjoint_symbols_exported(lib):
    for s in ('b200w_dwt_afb2d_adjoint', 'b200w_dwt_afb2d_adjoint_f64', 'b200w_dwt_afb1d_adjoint',
              'b200w_dwt_afb1d_adjoint_f64'):
        assert hasattr(lib, s) and s in _ffi.SYMBOLS


@pytest.mark.parametrize('sfx,ct', [('', ctypes.c_float), ('_f64', ctypes.c_double)])
def test_adjoint_2d_validation(lib, sfx, ct):
    f = (ct * 41)(*([0.5] * 41))
    fp = ctypes.cast(f, ctypes.c_void_p)
    buf = ctypes.c_void_p(16)    # never dereferenced: validation fails first
    fn = getattr(lib, 'b200w_dwt_afb2d_adjoint' + sfx)
    # 8x8 input, L = 8, symmetric: Hc = Wc = 7
    ok = dict(ll=buf, lps=49, lp=7, hs=buf, y=buf, yps=64, yp=8, planes=1, Hc=7, Wc=7, H=8, W=8, L=8, mode=1)

    def call(**kw):
        a = dict(ok, **kw)
        return fn(a['ll'], a['lps'], a['lp'], a['hs'], a['y'], a['yps'], a['yp'], a['planes'], a['Hc'], a['Wc'],
                  a['H'], a['W'], fp, fp, a['L'], fp, fp, a['L'], a['mode'], None)
    assert call(mode=3) == -1 and call(mode=99) == -1
    assert call(ll=None) == -3 and call(y=None) == -3
    assert call(lp=6) == -3 and call(yp=7) == -3
    assert call(Hc=6) == -2 and call(Wc=8) == -2 and call(H=0) == -2 and call(planes=-1) == -2
    assert call(L=1) == -4 and call(L=41) == -4


@pytest.mark.parametrize('sfx,ct', [('', ctypes.c_float), ('_f64', ctypes.c_double)])
def test_adjoint_1d_validation(lib, sfx, ct):
    f = (ct * 41)(*([0.5] * 41))
    fp = ctypes.cast(f, ctypes.c_void_p)
    buf = ctypes.c_void_p(16)
    fn = getattr(lib, 'b200w_dwt_afb1d_adjoint' + sfx)
    # n = 21, L = 6, reflect: K = 13
    assert fn(buf, buf, 1, 13, buf, 21, fp, fp, 6, 3, None) == -1
    assert fn(None, buf, 1, 13, buf, 21, fp, fp, 6, 4, None) == -3
    assert fn(buf, buf, 1, 13, None, 21, fp, fp, 6, 4, None) == -3
    assert fn(buf, buf, 1, 12, buf, 21, fp, fp, 6, 4, None) == -2
    assert fn(buf, buf, -1, 13, buf, 21, fp, fp, 6, 4, None) == -2
    assert fn(buf, buf, 1, 13, buf, 0, fp, fp, 6, 4, None) == -2
    assert fn(buf, buf, 1, 13, buf, 21, fp, fp, 1, 4, None) == -4
    assert fn(buf, buf, 1, 13, buf, 21, fp, fp, 41, 4, None) == -4
