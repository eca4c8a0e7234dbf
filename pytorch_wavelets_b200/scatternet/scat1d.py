"""``ScatLayer1D`` / ``ScatLayer1Dj2``: DTCWT scattering layers for the rows of an (N, C, n) tensor, the 1-D
counterparts of ``ScatLayer`` / ``ScatLayerj2``.  Each launch is a 1-D DTCWT forward level (``csrc/dtcwt1d.cu``) with
the scattering epilogue, writing straight into its slot of the output.

Definition, with ``F`` / ``D`` the level functions of ``dtcwt/transform1d.py`` and T the element type (every operation
rounded in T):
  pool(v)[i] = (v[2i] + v[2i+1]) * 0.5                                         (== F.avg_pool1d(v, 2))
  mag(h)[q]  = sqrt((h[2q] h[2q] + h[2q+1] h[2q+1]) + T(b * b)) - T(b)         (== torch.sqrt(re**2 + im**2 + b**2) - b)
  j1: lo, hi = F(x, h0o), F(x, h1o);  Z = (pool(lo), mag(hi))                   (N, 2, C, n/2) -> (N, 2C, n/2)
  j2: lo1, hi1 = F(x, ...);  U1 = mag(hi1);  lo2, hi2 = D(lo1, q-shift);  u, hu = F(U1, ...)
      Z = (pool(lo2), pool(u), mag(hi2), mag(hu))                               (N, 4, C, n/4) -> (N, 4C, n/4)
The backward passes are the exact adjoints: the derivatives re / r, im / r of each magnitude (written by the forward
kernels when the input needs a gradient) times the incoming gradient, interleaved into a band-pass, and the 1-D
inverse level kernels with the analysis taps (trees swapped at level 2).
"""
import torch
import torch.nn as nn
from torch.autograd import Function

from pytorch_wavelets_b200 import _ffi
from pytorch_wavelets_b200.dtcwt.coeffs import biort as _biort
from pytorch_wavelets_b200.dtcwt.coeffs import qshift as _qshift
from pytorch_wavelets_b200.dtcwt.lowlevel import prep_filt
from pytorch_wavelets_b200.dtcwt.transform1d import _call, _check3, _rows_view, inv_j1, inv_j2plus
from pytorch_wavelets_b200.dwt.lowlevel import mode_to_int


# ---- level functions: one kernel launch each ---------------------------------------------------------------------

def _dest(t):
    """(pointer, batch stride) of an (N, C, m) output whose (C, m) block is dense, e.g. one slot of (N, S, C, m)."""
    N, C, m = t.shape
    assert (C == 1 or t.stride(1) == m) and (m == 1 or t.stride(2) == 1), 'scattering outputs need dense (C, m) blocks'
    return t.data_ptr(), (t.stride(0) if N > 1 else C * m)


def _derivatives(x, m, der):
    if not der:
        return None, None, (None, 0), (None, 0)
    dre = x.new_empty((x.shape[0], x.shape[1], m))
    dim = torch.empty_like(dre)
    return dre, dim, _dest(dre), _dest(dim)


def fwd_j1(x, h0, h1, mode, bias, lo, mag, der):
    """Level 1 of x (N, C, n), n even: writes pool(lo) into ``lo`` when it is (N, C, n/2), else the full low-pass into
    ``lo`` (N, C, n); mag(hi) into ``mag`` (N, C, n/2).  Returns (dre, dim) (N, C, n/2) when ``der``, else Nones."""
    dt = _check3(x, 'x')
    N, C, n = x.shape
    if n % 2:
        raise ValueError('level-1 ScatLayer1D input must have an even length, got {}'.format(tuple(x.shape)))
    h0, h1 = _ffi.host_taps(h0), _ffi.host_taps(h1)
    pool = lo.shape[-1] != n
    dre, dim, pre, pim = _derivatives(x, n // 2, der)
    if N * C > 0:
        x, pitch = _rows_view(x)
        nout = (n // 2 if pool else n) + n // 2 * (3 if der else 1)
        with _ffi.span('scat1d_j1 %d' % n, x.element_size() * N * C * (n + nout)):
            _call('b200w_scat1d_j1', dt, x, x.data_ptr(), pitch, N, C, n, *_dest(lo), int(pool), *_dest(mag), *pre,
                  *pim, h0.p(dt), h0.n, h1.p(dt), h1.n, int(mode), float(bias))
    return dre, dim


def fwd_j2plus(x, h0a, h1a, h0b, h1b, bias, lo, mag, der):
    """Level >= 2 of x (N, C, n), n % 4 == 0: writes pool(lo) into ``lo`` and mag(hi) into ``mag``, each (N, C, n/4).
    Returns (dre, dim) (N, C, n/4) when ``der``, else Nones."""
    dt = _check3(x, 'x')
    N, C, n = x.shape
    if n % 4:
        raise ValueError('No. of samples in X must be a multiple of 4\nX was {}'.format(x.shape))
    f = [_ffi.host_taps(t) for t in (h0a, h1a, h0b, h1b)]
    dre, dim, pre, pim = _derivatives(x, n // 4, der)
    if N * C > 0:
        x, pitch = _rows_view(x)
        with _ffi.span('scat1d_j2plus %d' % n, x.element_size() * N * C * (n + n // 4 * (4 if der else 2))):
            _call('b200w_scat1d_j2plus', dt, x, x.data_ptr(), pitch, N, C, n, *_dest(lo), *_dest(mag), *pre, *pim,
                  *[t.p(dt) for t in f], f[0].n, float(bias))
    return dre, dim


def _up2_half(d):
    """Adjoint of pool: each gradient sample times 0.5, repeated twice."""
    return (d * 0.5).repeat_interleave(2, dim=-1)


def _band(d, dre, dim):
    """Adjoint of mag: (d re / r, d im / r) interleaved into the (N, C, 2m) band-pass layout."""
    return torch.stack((d * dre, d * dim), dim=-1).flatten(-2)


# ---- autograd Functions --------------------------------------------------------------------------------------------

class ScatLayer1Dj1_f(Function):
    """``apply(x, h0o, h1o, mode, bias)`` -> Z of shape (N, 2, C, n/2); n even."""

    @staticmethod
    def forward(ctx, x, h0o, h1o, mode, bias):
        _check3(x, 'x')
        ctx.mode = int(mode)
        ctx.taps = (_ffi.host_taps(h0o), _ffi.host_taps(h1o))
        N, C, n = x.shape
        der = bool(ctx.needs_input_grad[0])
        Z = x.new_empty((N, 2, C, n // 2))
        dre, dim = fwd_j1(x, ctx.taps[0], ctx.taps[1], ctx.mode, bias, Z[:, 0], Z[:, 1], der)
        if der:
            ctx.save_for_backward(dre, dim)
        return Z

    @staticmethod
    def backward(ctx, dZ):
        dx = None
        if ctx.needs_input_grad[0]:
            dre, dim = ctx.saved_tensors
            dx = inv_j1(_up2_half(dZ[:, 0]), _band(dZ[:, 1], dre, dim), ctx.taps[0], ctx.taps[1], ctx.mode)
        return dx, None, None, None, None


class ScatLayer1Dj2_f(Function):
    """``apply(x, h0o, h1o, h0a, h0b, h1a, h1b, mode, bias)`` -> Z of shape (N, 4, C, n/4); n % 8 == 0.  Three
    launches: level 1 on x (low-pass and U1 to workspaces), level 2 on the low-pass (slots 0 and 2), and level 1 on U1
    with the pooled low-pass (slots 1 and 3)."""

    @staticmethod
    def forward(ctx, x, h0o, h1o, h0a, h0b, h1a, h1b, mode, bias):
        _check3(x, 'x')
        ctx.mode = int(mode)
        ctx.taps = tuple(_ffi.host_taps(f) for f in (h0o, h1o, h0a, h0b, h1a, h1b))
        h0o, h1o, h0a, h0b, h1a, h1b = ctx.taps
        N, C, n = x.shape
        if n % 8:
            raise ValueError('ScatLayer1Dj2 input length must be a multiple of 8, got {}'.format(n))
        der = bool(ctx.needs_input_grad[0])
        Z = x.new_empty((N, 4, C, n // 4))
        lo1 = x.new_empty((N, C, n))
        U1 = x.new_empty((N, C, n // 2))
        d1 = fwd_j1(x, h0o, h1o, ctx.mode, bias, lo1, U1, der)
        d2 = fwd_j2plus(lo1, h0a, h1a, h0b, h1b, bias, Z[:, 0], Z[:, 2], der)
        del lo1
        d3 = fwd_j1(U1, h0o, h1o, ctx.mode, bias, Z[:, 1], Z[:, 3], der)
        if der:
            ctx.save_for_backward(*d1, *d2, *d3)
        return Z

    @staticmethod
    def backward(ctx, dZ):
        dx = None
        if ctx.needs_input_grad[0]:
            h0o, h1o, h0a, h0b, h1a, h1b = ctx.taps
            dre1, dim1, dre2, dim2, dre3, dim3 = ctx.saved_tensors
            ds0, ds1_j1, ds1_j2, ds2 = dZ[:, 0], dZ[:, 1], dZ[:, 2], dZ[:, 3]
            # second order: U1's gradient through the level-1 pass on U1
            dU1 = inv_j1(_up2_half(ds1_j1), _band(ds2, dre3, dim3), h0o, h1o, ctx.mode)
            # level 2 on the level-1 low-pass: inverse level with the analysis taps, trees swapped
            dlo1 = inv_j2plus(_up2_half(ds0), _band(ds1_j2, dre2, dim2), h0b, h1b, h0a, h1a)
            # level 1
            dx = inv_j1(dlo1, _band(dU1, dre1, dim1), h0o, h1o, ctx.mode)
        return (dx,) + (None,) * 8


# ---- modules -------------------------------------------------------------------------------------------------------

def _grad_mode(x):
    """x, detached under ``torch.no_grad()``: the Functions write the derivatives only for an input that needs a
    gradient, and inside ``Function.forward`` the caller's grad mode is no longer visible."""
    return x if torch.is_grad_enabled() else x.detach()


def _level1_filters(biort):
    if isinstance(biort, str):
        h0o, _, h1o, _ = _biort(biort)[:4]
    else:
        h0o, h1o = biort[0], biort[1]
    return h0o, h1o


class ScatLayer1D(nn.Module):
    """First-order 1-D scattering layer: level-1 DTCWT of each row, smoothed complex magnitude (``magbias``) of the
    band-pass and a 2-sample average of the low-pass, stacked on the channel dimension.

    Args:
        biort (str | (h0o, h1o)): level-1 biorthogonal filters: 'antonini', 'legall', 'near_sym_a', 'near_sym_b'.
        mode (str): 'symmetric' or 'zero' extension.
        magbias (float): b in sqrt(re^2 + im^2 + b^2) - b.

    Input (N, C, n) -> output (N, 2C, ceil(n / 2)): the first C channels are the low-pass, the next C the magnitudes.
    An odd n repeats the last sample.
    """

    def __init__(self, biort='near_sym_a', mode='symmetric', magbias=1e-2):
        super().__init__()
        self.biort = biort
        self.mode_str = mode
        self.mode = mode_to_int(mode)
        self.magbias = magbias
        h0o, h1o = _level1_filters(biort)
        self.h0o = nn.Parameter(prep_filt(h0o, 1), False)
        self.h1o = nn.Parameter(prep_filt(h1o, 1), False)

    def forward(self, x):
        _check3(x, 'x')
        if x.shape[-1] % 2 != 0:
            x = torch.cat((x, x[:, :, -1:]), dim=2)
        Z = ScatLayer1Dj1_f.apply(_grad_mode(x), self.h0o, self.h1o, self.mode, self.magbias)
        b, _, c, m = Z.shape
        return Z.reshape(b, 2 * c, m)

    def extra_repr(self):
        return "biort='{}', mode='{}', magbias={}".format(self.biort, self.mode_str, self.magbias)


class ScatLayer1Dj2(nn.Module):
    """Second-order 1-D scattering over two scales, with the level-1 biorthogonal and level-2 q-shift filters.

    Args:
        biort (str | (h0o, h1o)): level-1 filters, as for ``ScatLayer1D``.
        qshift (str | (h0a, h0b, h1a, h1b)): level-2 filters: 'qshift_06', 'qshift_a' .. 'qshift_d', 'qshift_32'.
        mode (str): only 'symmetric' (the q-shift level is defined for symmetric extension).
        magbias (float): b in sqrt(re^2 + im^2 + b^2) - b.

    Input (N, C, n) -> output (N, 4C, n' / 4), n' = n extended to a multiple of 8 by repeating the first / last
    samples as ``ScatLayerj2`` does per axis.  Channel blocks of C: the level-2 low-pass, the low-pass of the
    second-order pass, the level-2 magnitudes, the second-order magnitudes.
    """

    def __init__(self, biort='near_sym_a', qshift='qshift_a', mode='symmetric', magbias=1e-2):
        super().__init__()
        self.biort = biort
        self.qshift = qshift
        self.mode_str = mode
        self.mode = mode_to_int(mode)
        self.magbias = magbias
        h0o, h1o = _level1_filters(biort)
        if isinstance(qshift, str):
            h0a, h0b, _, _, h1a, h1b, _, _ = _qshift(qshift)[:8]
        else:
            h0a, h0b, h1a, h1b = qshift[:4]
        for name, arr in (('h0o', h0o), ('h1o', h1o), ('h0a', h0a), ('h0b', h0b), ('h1a', h1a), ('h1b', h1b)):
            setattr(self, name, nn.Parameter(prep_filt(arr, 1), False))

    def forward(self, x):
        _check3(x, 'x')
        rem = x.shape[-1] % 8
        if rem != 0:
            after, before = (9 - rem) // 2, (8 - rem) // 2
            x = torch.cat((x[:, :, :before], x, x[:, :, -after:]), dim=2)
        if self.mode_str != 'symmetric':
            raise NotImplementedError('ScatLayer1Dj2 supports symmetric extension only')
        Z = ScatLayer1Dj2_f.apply(_grad_mode(x), self.h0o, self.h1o, self.h0a, self.h0b, self.h1a, self.h1b, self.mode,
                                  self.magbias)
        b, _, c, m = Z.shape
        return Z.reshape(b, 4 * c, m)

    def extra_repr(self):
        return "biort='{}', mode='{}', magbias={}".format(self.biort, self.mode_str, self.magbias)
