"""CPU oracle of the 1-D DTCWT: numpy compositions of the pinned oracle primitives ``orc.filter1d`` / ``dfilt1d`` /
``ifilt1d`` along the last axis (oracle/oracle.py; pinned to the reference by tests/golden/prims_24x28.npz).

TEST INFRASTRUCTURE, NOT PRODUCT.  Signals are the rows of x (N, C, n); taps are the stored (reversed) module buffers
as 1-D arrays.  The level definitions are those of pytorch_wavelets_b200/dtcwt/transform1d.py; each inverse level is
the sum of two separately rounded branches.  fp32 and fp64 alike (the dtype of x).
"""
import numpy as np

from oracle import oracle as orc


def _r(v):
    return v[:, :, None, :]        # (N, C, n) -> (N, C, 1, n): filter along W


def _u(v):
    return v[:, :, 0, :]


def F(v, h, symmetric=True):
    return _u(orc.filter1d(_r(v), h, symmetric, along_w=True))


def D(v, ha, hb, highpass=False):
    return _u(orc.dfilt1d(_r(v), ha, hb, highpass, along_w=True))


def I(v, ha, hb, highpass=False):  # noqa: E741,E743
    return _u(orc.ifilt1d(_r(v), ha, hb, highpass, along_w=True))


def _cast(taps, dt):
    return [np.asarray(t, np.float64).ravel().astype(dt) for t in taps]


def fwd_j1(x, h0o, h1o, mode='symmetric'):
    sym = mode == 'symmetric'
    return F(x, h0o, sym), F(x, h1o, sym)


def fwd_j2plus(x, h0a, h1a, h0b, h1b):
    return D(x, h0b, h0a, False), D(x, h1b, h1a, True)


def inv_j1(lo, hi, g0o, g1o, mode='symmetric'):
    sym = mode == 'symmetric'
    a = None if lo is None else F(lo, g0o, sym)
    b = None if hi is None else F(hi, g1o, sym)
    return a if b is None else (b if a is None else a + b)


def inv_j2plus(lo, hi, g0a, g1a, g0b, g1b):
    a = None if lo is None else I(lo, g0b, g0a, False)
    b = None if hi is None else I(hi, g1b, g1a, True)
    return a if b is None else (b if a is None else a + b)


def dtcwt1d_forward(x, level1, qshift, J=3, mode='symmetric', skip_hps=False, include_scale=False):
    """DTCWT1DForward.forward.  level1 = (h0o, h1o), qshift = (h0a, h0b, h1a, h1b), stored taps.  Returns
    (yl or the list of low-passes, [yh_j (N, C, m_j, 2) or None for a skipped level])."""
    x = np.ascontiguousarray(x)
    if J == 0:
        return x, None
    h0o, h1o = _cast(level1, x.dtype)
    h0a, h0b, h1a, h1b = _cast(qshift, x.dtype)
    skip = skip_hps if isinstance(skip_hps, (list, tuple)) else [skip_hps] * J
    scl = include_scale if isinstance(include_scale, (list, tuple)) else [include_scale] * J
    if x.shape[-1] % 2:
        x = np.concatenate((x, x[:, :, -1:]), axis=2)
    lo, hi = fwd_j1(x, h0o, h1o, mode)
    yh, scales = [None if skip[0] else _c(hi)], [lo if scl[0] else None]
    for j in range(1, J):
        if lo.shape[-1] % 4:
            lo = np.concatenate((lo[:, :, :1], lo, lo[:, :, -1:]), axis=2)
        lo, hi = fwd_j2plus(lo, h0a, h1a, h0b, h1b)
        yh.append(None if skip[j] else _c(hi))
        scales.append(lo if scl[j] else None)
    if True in scl:
        return scales, yh
    return lo, yh


def dtcwt1d_inverse(yl, yh, level1, qshift, mode='symmetric'):
    """DTCWT1DInverse.forward.  level1 = (g0o, g1o), qshift = (g0a, g0b, g1a, g1b); None band-passes are zeros."""
    lo = np.ascontiguousarray(yl)
    g0o, g1o = _cast(level1, lo.dtype)
    g0a, g0b, g1a, g1b = _cast(qshift, lo.dtype)
    for j in range(len(yh) - 1, 0, -1):
        lo = _trim(lo, yh[j])
        lo = inv_j2plus(lo, _q(yh[j]), g0a, g1a, g0b, g1b)
    lo = _trim(lo, yh[0])
    return inv_j1(lo, _q(yh[0]), g0o, g1o, mode)


def _c(hi):
    return hi.reshape(hi.shape[0], hi.shape[1], -1, 2)


def _q(h):
    return None if h is None else np.ascontiguousarray(h).reshape(h.shape[0], h.shape[1], -1)


def _trim(lo, h):
    if h is not None and lo.shape[-1] != 2 * h.shape[-2]:
        lo = lo[:, :, 1:-1]
    return np.ascontiguousarray(lo)
