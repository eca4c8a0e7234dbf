"""CPU: the 1-D DTCWT's C ABI validation, module buffers and exports, and the oracle composition it is tested against
(perfect reconstruction and the transpose identities that define the backward passes).  No GPU."""
import ctypes

import numpy as np
import pytest
import torch

import pytorch_wavelets_b200 as pw
from pytorch_wavelets_b200 import _build, _ffi
from tests import oracle_dtcwt1d as o1

BIORTS = ['antonini', 'legall', 'near_sym_a', 'near_sym_b']
QSHIFTS = ['qshift_06', 'qshift_a', 'qshift_b', 'qshift_c', 'qshift_d', 'qshift_32']


@pytest.fixture(scope='module')
def lib():
    _build.build()
    return _ffi.lib()


def _np(t):
    return t.detach().cpu().numpy().ravel()


def _banks(biort, qshift, dtype=torch.float64):
    prev = torch.get_default_dtype()
    torch.set_default_dtype(dtype)
    try:
        f = pw.DTCWT1DForward(biort=biort, qshift=qshift)
        i = pw.DTCWT1DInverse(biort=biort, qshift=qshift)
    finally:
        torch.set_default_dtype(prev)
    fwd = ((_np(f.h0o), _np(f.h1o)), tuple(_np(getattr(f, k)) for k in ('h0a', 'h0b', 'h1a', 'h1b')))
    inv = ((_np(i.g0o), _np(i.g1o)), tuple(_np(getattr(i, k)) for k in ('g0a', 'g0b', 'g1a', 'g1b')))
    return fwd, inv


# ---- C ABI -------------------------------------------------------------------------------------------------------------

def test_abi_validates_without_gpu(lib):
    f = (ctypes.c_float * 40)(*([0.25] * 40))
    fp = ctypes.cast(f, ctypes.c_void_p)
    d = (ctypes.c_double * 40)(*([0.25] * 40))
    dp = ctypes.cast(d, ctypes.c_void_p)
    buf = ctypes.c_void_p(16)   # never dereferenced: validation fails first, or there is nothing to do
    for v, t in (('', fp), ('_f64', dp)):
        fj1 = getattr(lib, 'b200w_dtcwt1d_fwd_j1' + v)
        fj2 = getattr(lib, 'b200w_dtcwt1d_fwd_j2plus' + v)
        ij1 = getattr(lib, 'b200w_dtcwt1d_inv_j1' + v)
        ij2 = getattr(lib, 'b200w_dtcwt1d_inv_j2plus' + v)
        # level 1 forward
        assert fj1(buf, 16, 2, 16, buf, buf, t, 5, t, 7, 2, None) == -1           # periodization
        assert fj1(None, 16, 2, 16, buf, buf, t, 5, t, 7, 1, None) == -3
        assert fj1(buf, 16, 2, 16, None, buf, t, 5, t, 7, 1, None) == -3          # lo is required
        assert fj1(buf, 16, 2, 16, buf, buf, None, 5, t, 7, 1, None) == -3
        assert fj1(buf, 16, 2, 15, buf, buf, t, 5, t, 7, 1, None) == -2           # n odd
        assert fj1(buf, 15, 2, 16, buf, buf, t, 5, t, 7, 1, None) == -3           # pitch < n
        assert fj1(buf, 16, 2, 16, buf, buf, t, 4, t, 7, 1, None) == -4           # even level-1 filter
        assert fj1(buf, 16, 2, 16, buf, buf, t, 5, t, 41, 1, None) == -4          # longer than B200W_MAX_TAPS
        assert fj1(buf, 16, 0, 16, buf, None, t, 5, t, 7, 0, None) == 0           # empty batch
        # level >= 2 forward
        assert fj2(None, 16, 2, 16, buf, buf, t, t, t, t, 10, None) == -3
        assert fj2(buf, 16, 2, 16, buf, buf, t, t, None, t, 10, None) == -3
        assert fj2(buf, 18, 2, 18, buf, buf, t, t, t, t, 10, None) == -2          # n % 4 != 0
        assert fj2(buf, 16, 2, 16, buf, buf, t, t, t, t, 9, None) == -4           # odd q-shift length
        assert fj2(buf, 16, 2, 16, buf, buf, t, t, t, t, 42, None) == -4
        assert fj2(buf, 16, 0, 16, buf, None, t, t, t, t, 10, None) == 0
        # level 1 inverse
        assert ij1(buf, 16, buf, 2, 16, buf, t, 7, t, 5, 3, None) == -1
        assert ij1(buf, 16, buf, 2, 16, None, t, 7, t, 5, 1, None) == -3          # y is required
        assert ij1(buf, 16, buf, 2, 16, buf, t, 7, None, 5, 1, None) == -3
        assert ij1(buf, 16, buf, 2, 13, buf, t, 7, t, 5, 1, None) == -2
        assert ij1(buf, 8, buf, 2, 16, buf, t, 7, t, 5, 1, None) == -3
        assert ij1(buf, 16, buf, 2, 16, buf, t, 6, t, 5, 1, None) == -4
        assert ij1(None, 0, None, 0, 16, buf, t, 7, t, 5, 1, None) == 0
        # level >= 2 inverse (n = output length)
        assert ij2(buf, 8, buf, 2, 16, None, t, t, t, t, 10, None) == -3
        assert ij2(buf, 8, buf, 2, 16, buf, None, t, t, t, 10, None) == -3
        assert ij2(buf, 7, buf, 2, 14, buf, t, t, t, t, 10, None) == -2
        assert ij2(buf, 7, buf, 2, 16, buf, t, t, t, t, 10, None) == -3           # lo pitch < n / 2
        assert ij2(buf, 8, buf, 2, 16, buf, t, t, t, t, 11, None) == -4
        assert ij2(buf, 8, buf, 0, 16, buf, t, t, t, t, 10, None) == 0


# ---- modules -------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('biort', BIORTS)
@pytest.mark.parametrize('qshift', QSHIFTS)
def test_buffers_match_dtcwt2d(biort, qshift):
    f1, f2 = pw.DTCWT1DForward(biort=biort, qshift=qshift), pw.DTCWTForward(biort=biort, qshift=qshift)
    i1, i2 = pw.DTCWT1DInverse(biort=biort, qshift=qshift), pw.DTCWTInverse(biort=biort, qshift=qshift)
    for a, b in ((f1, f2), (i1, i2)):
        sa, sb = a.state_dict(), b.state_dict()
        assert list(sa) == list(sb)
        for k in sa:
            assert sa[k].shape == sb[k].shape and sa[k].dtype == sb[k].dtype
            assert torch.equal(sa[k], sb[k]), k


def test_filter_tuples_match_named_tables():
    t = pw.DTCWTForward()
    f = pw.DTCWT1DForward(biort=(_np(t.h0o)[::-1], _np(t.h1o)[::-1]),
                          qshift=tuple(_np(getattr(t, k))[::-1] for k in ('h0a', 'h0b', 'h1a', 'h1b')))
    for k, v in pw.DTCWT1DForward().state_dict().items():
        assert torch.equal(f.state_dict()[k], v), k


def test_exports_and_aliases():
    assert pw.DTCWT1D is pw.DTCWT1DForward and pw.IDTCWT1D is pw.DTCWT1DInverse
    for name in ('DTCWT1DForward', 'DTCWT1DInverse', 'DTCWT1D', 'IDTCWT1D'):
        assert name in pw.__all__


def test_j0_returns_input():
    x = torch.randn(2, 3, 17)
    yl, yh = pw.DTCWT1DForward(J=0)(x)
    assert yl is x and yh is None


def test_cpu_and_half_inputs_raise():
    with pytest.raises(NotImplementedError):
        pw.DTCWT1DForward(J=2)(torch.randn(2, 3, 32))
    with pytest.raises(NotImplementedError):
        pw.DTCWT1DForward(J=2)(torch.randn(2, 3, 32).half())
    with pytest.raises(NotImplementedError):
        pw.DTCWT1DInverse()((torch.randn(2, 3, 32), [torch.randn(2, 3, 16, 2)]))


# ---- oracle composition ----------------------------------------------------------------------------------------------

@pytest.mark.parametrize('biort', BIORTS)
@pytest.mark.parametrize('qshift', QSHIFTS)
def test_oracle_perfect_reconstruction_f64(biort, qshift):
    """Symmetric mode reconstructs for every table pair: n odd, n = 2 (mod 4), n shorter than the filters."""
    (l1, qs), (il1, iqs) = _banks(biort, qshift)
    tol = 1e-8 if qshift == 'qshift_32' else 1e-12
    rs = np.random.RandomState(7)
    for n in (2, 4, 6, 13, 22, 37, 64, 101):
        for J in (1, 2, 3, 5):
            x = rs.randn(2, 3, n)
            yl, yh = o1.dtcwt1d_forward(x, l1, qs, J)
            assert len(yh) == J and all(h.shape[-1] == 2 for h in yh)
            y = o1.dtcwt1d_inverse(yl, yh, il1, iqs)[:, :, :n]
            assert np.abs(y - x).max() <= tol * np.abs(x).max(), (n, J)


def _matrix(fn, n):
    """Dense matrix of a linear map on length-n signals, built from unit vectors."""
    return np.stack([fn(np.eye(n)[k].reshape(1, 1, n)).ravel() for k in range(n)], axis=1)


@pytest.mark.parametrize('qshift', QSHIFTS)
def test_oracle_transposes_define_backward(qshift):
    """D(., h0b, h0a)^T = I(., h0a, h0b) (and the high-pass pair): the backward of a forward level is the inverse
    level kernel with the analysis taps, trees swapped, and vice versa.  Exact wherever no two taps fold onto one
    sample (n >= m); below that the two sides sum the folded products in different orders and may differ by an ulp."""
    (l1, (h0a, h0b, h1a, h1b)), _ = _banks('near_sym_a', qshift)
    for n in (4, 8, 12, 16, 20, 32):
        tol = 0.0 if n >= len(h0a) else 1e-15
        D0 = _matrix(lambda e: o1.D(e, h0b, h0a, False), n)
        D1 = _matrix(lambda e: o1.D(e, h1b, h1a, True), n)
        # inverse level with the analysis taps, trees swapped: (g0a, g1a, g0b, g1b) = (h0b, h1b, h0a, h1a)
        I0 = _matrix(lambda e: o1.inv_j2plus(e, None, h0b, h1b, h0a, h1a), n // 2)
        I1 = _matrix(lambda e: o1.inv_j2plus(None, e, h0b, h1b, h0a, h1a), n // 2)
        assert np.abs(D0.T - I0).max() <= tol
        assert np.abs(D1.T - I1).max() <= tol


@pytest.mark.parametrize('biort', BIORTS)
@pytest.mark.parametrize('mode', ['symmetric', 'zero'])
def test_oracle_level1_filters_are_symmetric_matrices(biort, mode):
    """F(., h) is its own transpose, so each level-1 backward is the other direction's kernel with the same taps.
    Exact for palindromic taps where no two taps fold onto one sample (n > L / 2); the antonini table is palindromic
    only to ~4e-15 in float64 and symmetric-mode folding regroups products, so those cases agree to 1e-14."""
    (l1, _), (il1, _) = _banks(biort, 'qshift_a')
    for n in (2, 4, 6, 10, 16):
        for h in l1 + il1:
            M = _matrix(lambda e: o1.F(e, h, mode == 'symmetric'), n)
            exact = np.array_equal(h, h[::-1]) and (mode == 'zero' or n > len(h) // 2)
            assert np.abs(M - M.T).max() <= (0.0 if exact else 1e-14), (n, len(h))
