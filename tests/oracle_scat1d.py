"""CPU oracle of the 1-D scattering layers (ScatLayer1D / ScatLayer1Dj2): numpy compositions of the 1-D DTCWT oracle
levels (tests/oracle_dtcwt1d.py) and the pointwise definitions of pytorch_wavelets_b200/scatternet/scat1d.py, every
operation rounded in the dtype of x (float32 or float64).

TEST INFRASTRUCTURE, NOT PRODUCT.  Taps are the stored (reversed) module buffers as 1-D arrays.
"""
import numpy as np

from tests import oracle_dtcwt1d as o1


def pool(v):
    """(v[2i] + v[2i+1]) * 0.5 along the last axis."""
    return (v[..., 0::2] + v[..., 1::2]) * v.dtype.type(0.5)


def mag(h, bias):
    """(sqrt((re re + im im) + T(b b)) - T(b), re / r, im / r) of the band-pass h (..., 2m), (re, im) interleaved."""
    dt = h.dtype.type
    re, im = h[..., 0::2], h[..., 1::2]
    r = np.sqrt((re * re + im * im) + dt(float(bias) * float(bias)))
    with np.errstate(invalid='ignore', divide='ignore'):
        return r - dt(bias), re / r, im / r


def pad_j1(x):
    """ScatLayer1D: an odd length repeats the last sample."""
    return np.concatenate((x, x[:, :, -1:]), axis=2) if x.shape[-1] % 2 else x


def pad_j2(x):
    """ScatLayer1Dj2: extend to a multiple of 8 by repeating the first / last samples (ScatLayerj2's per-axis rule)."""
    rem = x.shape[-1] % 8
    if rem:
        after, before = (9 - rem) // 2, (8 - rem) // 2
        x = np.concatenate((x[:, :, :before], x, x[:, :, -after:]), axis=2)
    return x


def scat1d_j1(x, level1, mode='symmetric', bias=1e-2):
    """ScatLayer1Dj1_f on x (N, C, n), n even: (Z (N, 2, C, n/2), dre, dim (N, C, n/2))."""
    x = np.ascontiguousarray(x)
    h0o, h1o = o1._cast(level1, x.dtype)
    lo, hi = o1.fwd_j1(x, h0o, h1o, mode)
    m, dre, dim = mag(hi, bias)
    return np.stack((pool(lo), m), axis=1), dre, dim


def scat1d_j2(x, level1, qshift, bias=1e-2):
    """ScatLayer1Dj2_f on x (N, C, n), n % 8 == 0: (Z (N, 4, C, n/4), [(dre, dim) of level 1, level 2, the second
    order pass])."""
    x = np.ascontiguousarray(x)
    h0o, h1o = o1._cast(level1, x.dtype)
    h0a, h0b, h1a, h1b = o1._cast(qshift, x.dtype)
    lo1, hi1 = o1.fwd_j1(x, h0o, h1o)
    U1, dre1, dim1 = mag(hi1, bias)
    lo2, hi2 = o1.fwd_j2plus(lo1, h0a, h1a, h0b, h1b)
    s1_j2, dre2, dim2 = mag(hi2, bias)
    u, hu = o1.fwd_j1(U1, h0o, h1o)
    s2, dre3, dim3 = mag(hu, bias)
    return np.stack((pool(lo2), pool(u), s1_j2, s2), axis=1), [(dre1, dim1), (dre2, dim2), (dre3, dim3)]


def up2_half(d):
    """Adjoint of pool."""
    return np.repeat(d * d.dtype.type(0.5), 2, axis=-1)


def band(d, dre, dim):
    """Adjoint of mag: (d dre, d dim) interleaved."""
    return np.stack((d * dre, d * dim), axis=-1).reshape(d.shape[:-1] + (-1,))


def backward_j1(dZ, dre, dim, level1, mode='symmetric'):
    """dx of ScatLayer1Dj1_f for dZ (N, 2, C, m): inv_j1 with the analysis taps."""
    h0o, h1o = o1._cast(level1, dZ.dtype)
    return o1.inv_j1(up2_half(dZ[:, 0]), band(dZ[:, 1], dre, dim), h0o, h1o, mode)


def backward_j2(dZ, ders, level1, qshift):
    """dx of ScatLayer1Dj2_f for dZ (N, 4, C, m), ders as returned by scat1d_j2."""
    h0o, h1o = o1._cast(level1, dZ.dtype)
    h0a, h0b, h1a, h1b = o1._cast(qshift, dZ.dtype)
    (dre1, dim1), (dre2, dim2), (dre3, dim3) = ders
    dU1 = o1.inv_j1(up2_half(dZ[:, 1]), band(dZ[:, 3], dre3, dim3), h0o, h1o)
    dlo1 = o1.inv_j2plus(up2_half(dZ[:, 0]), band(dZ[:, 2], dre2, dim2), h0b, h1b, h0a, h1a)
    return o1.inv_j1(dlo1, band(dU1, dre1, dim1), h0o, h1o)


def scat_layer1d(x, level1, mode='symmetric', bias=1e-2):
    """ScatLayer1D.forward: (N, 2C, ceil(n / 2))."""
    Z = scat1d_j1(pad_j1(x), level1, mode, bias)[0]
    return Z.reshape(Z.shape[0], -1, Z.shape[-1])


def scat_layer1d_j2(x, level1, qshift, bias=1e-2):
    """ScatLayer1Dj2.forward: (N, 4C, n' / 4)."""
    Z = scat1d_j2(pad_j2(x), level1, qshift, bias)[0]
    return Z.reshape(Z.shape[0], -1, Z.shape[-1])
