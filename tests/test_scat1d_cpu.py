"""CPU: the 1-D scattering layers' C ABI validation, module buffers, exports, exceptions and padding, and the dense-matrix
adjoint identities that define their backward passes (on the oracle composition, float64).  No GPU."""
import ctypes

import numpy as np
import pytest
import torch

import pytorch_wavelets_b200 as pw
from pytorch_wavelets_b200 import _build, _ffi
from pytorch_wavelets_b200.scatternet import scat1d, variants
from tests import oracle_dtcwt1d as o1
from tests import oracle_scat1d as os1

BIORTS = ['antonini', 'legall', 'near_sym_a', 'near_sym_b']
QSHIFTS = ['qshift_06', 'qshift_a', 'qshift_b', 'qshift_c', 'qshift_d', 'qshift_32']


@pytest.fixture(scope='module')
def lib():
    _build.build()
    return _ffi.lib()


def _np(t):
    return t.detach().cpu().numpy().ravel()


def _taps(m):
    return ((_np(m.h0o), _np(m.h1o)), tuple(_np(getattr(m, k)) for k in ('h0a', 'h0b', 'h1a', 'h1b')))


# ---- C ABI -------------------------------------------------------------------------------------------------------------

def test_abi_validates_without_gpu(lib):
    f = (ctypes.c_float * 40)(*([0.25] * 40))
    fp = ctypes.cast(f, ctypes.c_void_p)
    d = (ctypes.c_double * 40)(*([0.25] * 40))
    dp = ctypes.cast(d, ctypes.c_void_p)
    b = ctypes.c_void_p(16)   # never dereferenced: validation fails first, or there is nothing to do
    for v, t in (('', fp), ('_f64', dp)):
        j1 = getattr(lib, 'b200w_scat1d_j1' + v)
        j2 = getattr(lib, 'b200w_scat1d_j2plus' + v)

        def c1(x=b, pitch=16, N=2, C=3, n=16, lo=b, bs_lo=24, pool=1, mag=b, bs_mag=24, dre=b, bs_dre=24, dim=b,
               bs_dim=24, h0=t, L0=5, h1=t, L1=7, mode=1):
            return j1(x, pitch, N, C, n, lo, bs_lo, pool, mag, bs_mag, dre, bs_dre, dim, bs_dim, h0, L0, h1, L1, mode,
                      1e-2, None)

        def c2(x=b, pitch=16, N=2, C=3, n=16, lo=b, bs_lo=12, mag=b, bs_mag=12, dre=b, bs_dre=12, dim=b, bs_dim=12,
               h=(t, t, t, t), m=10):
            return j2(x, pitch, N, C, n, lo, bs_lo, mag, bs_mag, dre, bs_dre, dim, bs_dim, *h, m, 1e-2, None)

        # level 1
        assert c1(mode=2) == -1                       # periodization
        for k in ('x', 'lo', 'mag', 'h0', 'h1'):
            assert c1(**{k: None}) == -3, k           # required pointers
        assert c1(dre=None) == -3 and c1(dim=None) == -3   # dre / dim come together
        assert c1(n=15) == -2 and c1(n=0) == -2       # n odd, too short
        assert c1(N=-1) == -2 and c1(C=-1) == -2
        assert c1(N=1 << 16, C=1 << 16) == -2         # N * C above INT_MAX
        assert c1(pitch=15) == -3                     # pitch < n
        assert c1(bs_lo=23) == -3 and c1(pool=0, bs_lo=24) == -3 and c1(bs_mag=23) == -3 and c1(bs_dim=23) == -3
        assert c1(L0=4) == -4 and c1(L1=41) == -4     # even, longer than B200W_MAX_TAPS
        assert c1(N=0) == 0 and c1(C=0, bs_lo=0, bs_mag=0, bs_dre=0, bs_dim=0) == 0   # empty batch
        assert c1(N=0, dre=None, dim=None, mode=0) == 0
        # level >= 2
        for k in ('x', 'lo', 'mag'):
            assert c2(**{k: None}) == -3, k
        assert c2(h=(t, t, None, t)) == -3
        assert c2(dim=None) == -3
        assert c2(n=18, pitch=18) == -2 and c2(n=14) == -2   # n % 4 != 0
        assert c2(pitch=12) == -3 and c2(bs_lo=11) == -3 and c2(bs_dre=11) == -3
        assert c2(m=9) == -4 and c2(m=42) == -4        # odd, too long q-shift
        assert c2(N=0) == 0


# ---- modules -------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('biort', BIORTS)
def test_buffers_match_scatlayer(biort):
    for a, b in ((pw.ScatLayer1D(biort=biort), pw.ScatLayer(biort=biort)),
                 (pw.ScatLayer1Dj2(biort=biort), pw.ScatLayerj2(biort=biort))):
        sa, sb = a.state_dict(), b.state_dict()
        assert list(sa) == list(sb)
        for k in sa:
            assert sa[k].dtype == sb[k].dtype and torch.equal(sa[k], sb[k]), k
        for p in a.parameters():
            assert isinstance(p, torch.nn.Parameter) and not p.requires_grad
        assert a.extra_repr() == b.extra_repr()


@pytest.mark.parametrize('qshift', QSHIFTS)
def test_qshift_buffers_match_dtcwt1d(qshift):
    s, f = pw.ScatLayer1Dj2(qshift=qshift), pw.DTCWT1DForward(qshift=qshift)
    for k in ('h0o', 'h1o', 'h0a', 'h0b', 'h1a', 'h1b'):
        assert torch.equal(getattr(s, k), getattr(f, k)), k


def test_filter_tuples_match_named_tables():
    t = pw.DTCWT1DForward()
    l1 = (_np(t.h0o)[::-1], _np(t.h1o)[::-1])
    qs = tuple(_np(getattr(t, k))[::-1] for k in ('h0a', 'h0b', 'h1a', 'h1b'))
    for a, b in ((pw.ScatLayer1D(biort=l1), pw.ScatLayer1D()),
                 (pw.ScatLayer1Dj2(biort=l1, qshift=qs), pw.ScatLayer1Dj2())):
        for k, v in b.state_dict().items():
            assert torch.equal(a.state_dict()[k], v), k


def test_extra_repr():
    assert pw.ScatLayer1D(mode='zero', magbias=0.5).extra_repr() == "biort='near_sym_a', mode='zero', magbias=0.5"
    assert pw.ScatLayer1Dj2(biort='near_sym_b').extra_repr() == "biort='near_sym_b', mode='symmetric', magbias=0.01"


def test_exports():
    from pytorch_wavelets_b200 import scatternet
    for name in ('ScatLayer1D', 'ScatLayer1Dj2'):
        assert name in pw.__all__
        assert getattr(pw, name) is getattr(scatternet, name) is getattr(scat1d, name)


def test_cpu_half_and_zero_mode_raise():
    for m in (pw.ScatLayer1D(), pw.ScatLayer1Dj2()):
        with pytest.raises(NotImplementedError):
            m(torch.randn(2, 3, 32))
        with pytest.raises(NotImplementedError):
            m(torch.randn(2, 3, 32).half())
    with pytest.raises(NotImplementedError):
        pw.ScatLayer1Dj2(mode='zero')(torch.randn(2, 3, 32))


def _captured(module, x, monkeypatch, name):
    """The input the module hands its autograd Function (the device checks skipped)."""
    seen = []

    class Fake(object):
        @staticmethod
        def apply(x, *args):
            seen.append(x)
            N, C, n = x.shape
            S = 2 if name == 'ScatLayer1Dj1_f' else 4
            return x.new_zeros((N, S, C, n // S))
    monkeypatch.setattr(scat1d, '_check3', lambda t, n: t.dtype)
    monkeypatch.setattr(scat1d, name, Fake)
    out = module(x)
    return seen[0], out


def test_padding_rules(monkeypatch):
    for n in range(1, 26):
        x = torch.arange(2 * 3 * n, dtype=torch.float64).reshape(2, 3, n)
        p1, z1 = _captured(pw.ScatLayer1D(), x, monkeypatch, 'ScatLayer1Dj1_f')
        assert np.array_equal(p1.numpy(), os1.pad_j1(x.numpy()))
        assert z1.shape == (2, 6, (n + 1) // 2)
        p2, z2 = _captured(pw.ScatLayer1Dj2(), x, monkeypatch, 'ScatLayer1Dj2_f')
        assert np.array_equal(p2.numpy(), os1.pad_j2(x.numpy()))
        assert z2.shape == (2, 12, p2.shape[-1] // 4)
        assert p2.shape[-1] % 8 == 0 or n < 4      # (the rule repeats at most 4 samples at an end)
        # the 2-D layer extends its columns by the same rule
        seen = []
        monkeypatch.setattr(variants, 'scat_j2', lambda ops, x4, *a: seen.append(x4) or x4.new_zeros(
            (x4.shape[0], 49, x4.shape[1], x4.shape[2] // 4, x4.shape[3] // 4)))
        pw.ScatLayerj2()(x[:, :, None, :].expand(2, 3, 8, n))
        assert torch.equal(seen[0][:, :, 0], p2)


# ---- adjoints of the oracle composition ---------------------------------------------------------------------------------

def _matrix(fn, n):
    """Dense matrix of a map on (1, 1, n) signals, built from unit vectors."""
    return np.stack([np.asarray(fn(np.eye(n)[k].reshape(1, 1, n))).ravel() for k in range(n)], axis=1)


def _jacobian_fd(fn, x, eps=1e-6):
    cols = []
    for k in range(x.size):
        e = np.zeros_like(x)
        e.flat[k] = eps
        cols.append((fn(x + e) - fn(x - e)).ravel() / (2 * eps))
    return np.stack(cols, axis=1)


def _ders_matrix(dre, dim):
    """Jacobian of mag at a point: row q has dre[q], dim[q] at columns 2q, 2q + 1."""
    m = dre.size
    M = np.zeros((m, 2 * m))
    M[np.arange(m), 2 * np.arange(m)] = dre.ravel()
    M[np.arange(m), 2 * np.arange(m) + 1] = dim.ravel()
    return M


@pytest.mark.parametrize('biort', BIORTS)
@pytest.mark.parametrize('mode', ['symmetric', 'zero'])
def test_j1_backward_is_the_adjoint(biort, mode):
    (l1, _) = _taps(pw.ScatLayer1Dj2(biort=biort).double())
    h0, h1 = l1
    rs = np.random.RandomState(1)
    for n in (2, 6, 16, 30):
        x = rs.randn(1, 1, n)
        Z, dre, dim = os1.scat1d_j1(x, l1, mode)
        m = n // 2
        P = _matrix(os1.pool, n)
        F0 = _matrix(lambda e: o1.F(e, h0, mode == 'symmetric'), n)
        F1 = _matrix(lambda e: o1.F(e, h1, mode == 'symmetric'), n)
        J = np.concatenate((P @ F0, _ders_matrix(dre, dim) @ F1))
        # the chain rule matches the forward map itself
        assert np.abs(J - _jacobian_fd(lambda v: os1.scat1d_j1(v, l1, mode)[0], x)).max() < 1e-6
        B = _matrix(lambda e: os1.backward_j1(e.reshape(1, 2, 1, m), dre, dim, l1, mode), 2 * m)
        assert np.abs(B - J.T).max() <= 1e-14, n


@pytest.mark.parametrize('biort,qshift', [('near_sym_a', 'qshift_a'), ('near_sym_b', 'qshift_b'),
                                          ('antonini', 'qshift_c'), ('legall', 'qshift_d'),
                                          ('near_sym_a', 'qshift_06'), ('near_sym_a', 'qshift_32')])
def test_j2_backward_is_the_adjoint(biort, qshift):
    l1, qs = _taps(pw.ScatLayer1Dj2(biort=biort, qshift=qshift).double())
    h0, h1 = l1
    h0a, h0b, h1a, h1b = qs
    rs = np.random.RandomState(2)
    for n in (8, 16, 40):
        x = rs.randn(1, 1, n)
        Z, ders = os1.scat1d_j2(x, l1, qs)
        (dre1, dim1), (dre2, dim2), (dre3, dim3) = ders
        m = n // 4
        F0n, F1n = (_matrix(lambda e: o1.F(e, h, True), n) for h in (h0, h1))
        F0h, F1h = (_matrix(lambda e: o1.F(e, h, True), n // 2) for h in (h0, h1))
        D0 = _matrix(lambda e: o1.D(e, h0b, h0a, False), n)
        D1 = _matrix(lambda e: o1.D(e, h1b, h1a, True), n)
        P = _matrix(os1.pool, n // 2)
        M1 = _ders_matrix(dre1, dim1) @ F1n                      # dU1 / dx
        J = np.concatenate((
            P @ D0 @ F0n,                                         # s0 = pool(lo2)
            P @ F0h @ M1,                                         # s1_j1 = pool(u)
            _ders_matrix(dre2, dim2) @ D1 @ F0n,                  # s1_j2 = mag(hi2)
            _ders_matrix(dre3, dim3) @ F1h @ M1))                 # s2 = mag(hu)
        assert np.abs(J - _jacobian_fd(lambda v: os1.scat1d_j2(v, l1, qs)[0], x)).max() < 1e-6
        B = _matrix(lambda e: os1.backward_j2(e.reshape(1, 4, 1, m), ders, l1, qs), 4 * m)
        assert np.abs(B - J.T).max() <= 1e-13, n
