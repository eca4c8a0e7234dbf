"""``DTCWT1DForward`` / ``DTCWT1DInverse``: the 1-D dual-tree complex wavelet transform of the rows of an (N, C, n)
tensor, with the filter tables, buffers, return structure and padding / trimming rules of ``DTCWTForward`` /
``DTCWTInverse`` applied to one axis.  Each level is one CUDA kernel (``csrc/dtcwt1d.cu``) that filters both trees.

Definition, with ``F`` / ``D`` / ``I`` the standalone ``colfilter`` / ``coldfilt`` / ``colifilt`` along the row and the
stored (reversed) taps of the module buffers:
  level 1:      lo = F(x, h0o), hi = F(x, h1o)                        (symmetric extension or zero padding)
  levels >= 2:  hi = D(lo, h1b, h1a, highpass), lo = D(lo, h0b, h0a)  (symmetric)
The band-pass ``yh[j]`` is hi viewed as (N, C, len / 2, 2): (re, im) = (hi[2q], hi[2q + 1]), no 1/sqrt(2) factor.
The inverse sums two separately rounded branches per level: I(lo, g0b, g0a) + I(hi, g1b, g1a, highpass) and
F(lo, g0o) + F(hi, g1o).  Each Function's backward pass is the opposite direction's kernel with the same stored
filters (a / b trees swapped at levels >= 2), the exact transpose in 1-D.
"""
import torch
import torch.nn as nn
from numpy import ndarray
from torch.autograd import Function

from pytorch_wavelets_b200 import _ffi
from pytorch_wavelets_b200.dtcwt.coeffs import biort as _biort
from pytorch_wavelets_b200.dtcwt.coeffs import qshift as _qshift
from pytorch_wavelets_b200.dtcwt.lowlevel import prep_filt
from pytorch_wavelets_b200.dwt.lowlevel import mode_to_int


def _is_empty(t):
    return t is None or t.shape == torch.Size([])


def _rows_view(t):
    """(tensor, row pitch) for an (N, C, n) tensor whose rows are unit-stride and whose (N, C) dims collapse to one row
    index; copies to contiguous only when the layout does not allow it."""
    N, C, n = t.shape
    s = t.stride()
    ok = t.numel() > 0 and (n == 1 or s[2] == 1)
    pitch = s[1] if C > 1 else (s[0] if N > 1 else n)
    if ok and N > 1 and C > 1:
        ok = s[0] == C * s[1]
    if not ok or pitch < n:
        t = t.contiguous()
        pitch = n
    return t, int(pitch)


def _check3(t, name):
    dt = _ffi.require_cuda_real(t, name)
    if t.dim() != 3:
        raise ValueError('{} must be a 3-D (N, C, n) tensor, got shape {}'.format(name, tuple(t.shape)))
    return dt


def _call(name, dt, x, *args):
    fn = getattr(_ffi.lib(), name + ('_f64' if dt == torch.float64 else ''))
    with torch.cuda.device(x.device):
        rc = fn(*args, _ffi.stream_of(x))
    _ffi.check(rc, name)


# ---- level functions: one kernel launch each ---------------------------------------------------------------------

def fwd_j1(x, h0, h1, skip_hps, mode):
    """Level 1: (lo, hi) of x (N, C, n), n even, each (N, C, n); hi is None when skipped."""
    dt = _check3(x, 'x')
    N, C, n = x.shape
    if n % 2:
        raise ValueError('level-1 DTCWT1D input must have an even length, got {}'.format(tuple(x.shape)))
    h0, h1 = _ffi.host_taps(h0), _ffi.host_taps(h1)
    lo = x.new_empty((N, C, n))
    hi = None if skip_hps else x.new_empty((N, C, n))
    if N * C > 0:
        x, pitch = _rows_view(x)
        with _ffi.span('dtcwt1d_fwd_j1 %d' % n, x.element_size() * N * C * n * (2 if skip_hps else 3)):
            _call('b200w_dtcwt1d_fwd_j1', dt, x, x.data_ptr(), pitch, N * C, n, lo.data_ptr(),
                  None if hi is None else hi.data_ptr(), h0.p(dt), h0.n, h1.p(dt), h1.n, int(mode))
    return lo, hi


def fwd_j2plus(x, h0a, h1a, h0b, h1b, skip_hps):
    """Level >= 2: (lo, hi) of x (N, C, n), n % 4 == 0, each (N, C, n / 2); hi is None when skipped."""
    dt = _check3(x, 'x')
    N, C, n = x.shape
    if n % 4:
        raise ValueError('No. of samples in X must be a multiple of 4\nX was {}'.format(x.shape))
    f = [_ffi.host_taps(t) for t in (h0a, h1a, h0b, h1b)]
    lo = x.new_empty((N, C, n // 2))
    hi = None if skip_hps else x.new_empty((N, C, n // 2))
    if N * C > 0:
        x, pitch = _rows_view(x)
        with _ffi.span('dtcwt1d_fwd_j2plus %d' % n, x.element_size() * N * C * n * (3 if skip_hps else 4) // 2):
            _call('b200w_dtcwt1d_fwd_j2plus', dt, x, x.data_ptr(), pitch, N * C, n, lo.data_ptr(),
                  None if hi is None else hi.data_ptr(), *[t.p(dt) for t in f], f[0].n)
    return lo, hi


def _inv_inputs(lo, hi):
    """Validated (lo, lo pitch, hi contiguous, N, C, k, dtype, device tensor) of an inverse level; k = input length."""
    ref = lo if lo is not None else hi
    if ref is None:
        raise ValueError('an inverse DTCWT1D level needs a low-pass or a band-pass input')
    dt = _check3(ref, 'lo' if lo is not None else 'hi')
    N, C, k = ref.shape
    if hi is not None:
        _ffi.require_cuda_real(hi, 'hi', dt)
        if tuple(hi.shape) != (N, C, k):
            raise ValueError('band-pass of shape {} does not match the low-pass {}'.format(
                tuple(hi.shape), (N, C, k)))
        hi = hi.contiguous()
    pitch = 0
    if lo is not None:
        _ffi.require_cuda_real(lo, 'lo', dt)
        lo, pitch = _rows_view(lo)
    return lo, pitch, hi, N, C, k, dt, ref


def inv_j1(lo, hi, g0, g1, mode):
    """Level 1: y = F(lo, g0) + F(hi, g1); lo, hi (N, C, n) real layout or None (zeros), n even."""
    lo, pitch, hi, N, C, n, dt, ref = _inv_inputs(lo, hi)
    if n % 2:
        raise ValueError('level-1 DTCWT1D inputs must have an even length, got {}'.format(n))
    g0, g1 = _ffi.host_taps(g0), _ffi.host_taps(g1)
    y = ref.new_empty((N, C, n))
    if N * C > 0:
        nin = (lo is not None) + (hi is not None)
        with _ffi.span('dtcwt1d_inv_j1 %d' % n, y.element_size() * N * C * n * (1 + nin)):
            _call('b200w_dtcwt1d_inv_j1', dt, ref, None if lo is None else lo.data_ptr(), pitch,
                  None if hi is None else hi.data_ptr(), N * C, n, y.data_ptr(), g0.p(dt), g0.n, g1.p(dt), g1.n,
                  int(mode))
    return y


def inv_j2plus(lo, hi, g0a, g1a, g0b, g1b):
    """Level >= 2: y (N, C, 2k) = I(lo, g0b, g0a) + I(hi, g1b, g1a, highpass); lo, hi (N, C, k) or None, k even."""
    lo, pitch, hi, N, C, k, dt, ref = _inv_inputs(lo, hi)
    if k % 2:
        raise ValueError('No. of samples in X must be a multiple of 2\nX was {}'.format((N, C, k)))
    f = [_ffi.host_taps(t) for t in (g0a, g1a, g0b, g1b)]
    y = ref.new_empty((N, C, 2 * k))
    if N * C > 0:
        nin = (lo is not None) + (hi is not None)
        with _ffi.span('dtcwt1d_inv_j2plus %d' % (2 * k), y.element_size() * N * C * k * (2 + nin)):
            _call('b200w_dtcwt1d_inv_j2plus', dt, ref, None if lo is None else lo.data_ptr(), pitch,
                  None if hi is None else hi.data_ptr(), N * C, 2 * k, y.data_ptr(), *[t.p(dt) for t in f], f[0].n)
    return y


def _c(hi):
    """Real band-pass (N, C, n) -> complex view (N, C, n / 2, 2)."""
    return hi.view(hi.shape[0], hi.shape[1], -1, 2)


def _q(h):
    """Complex band-pass (N, C, m, 2) -> real layout (N, C, 2m), or None for a missing band."""
    if _is_empty(h):
        return None
    if h.dim() != 4 or h.shape[-1] != 2:
        raise ValueError('DTCWT1D band-pass must have shape (N, C, m, 2), got {}'.format(tuple(h.shape)))
    return h.reshape(h.shape[0], h.shape[1], -1)


# ---- autograd Functions --------------------------------------------------------------------------------------------

class FWD1D_J1(Function):
    """Differentiable level-1 forward: ``apply(x, h0o, h1o, skip_hps, mode)`` -> (lo, yh) with yh (N, C, n/2, 2)."""

    @staticmethod
    def forward(ctx, x, h0, h1, skip_hps, mode):
        ctx.mode = int(mode)
        ctx.taps = (_ffi.host_taps(h0), _ffi.host_taps(h1))
        lo, hi = fwd_j1(x, ctx.taps[0], ctx.taps[1], bool(skip_hps), ctx.mode)
        return lo, (lo.new_zeros([]) if hi is None else _c(hi))

    @staticmethod
    def backward(ctx, dl, dh):
        dx = None
        if ctx.needs_input_grad[0]:
            dx = inv_j1(dl, _q(dh), ctx.taps[0], ctx.taps[1], ctx.mode)
        return dx, None, None, None, None


class FWD1D_J2PLUS(Function):
    """Differentiable level >= 2 forward: ``apply(x, h0a, h1a, h0b, h1b, skip_hps)`` -> (lo, yh)."""

    @staticmethod
    def forward(ctx, x, h0a, h1a, h0b, h1b, skip_hps):
        ctx.taps = tuple(_ffi.host_taps(f) for f in (h0a, h1a, h0b, h1b))
        lo, hi = fwd_j2plus(x, *ctx.taps, bool(skip_hps))
        return lo, (lo.new_zeros([]) if hi is None else _c(hi))

    @staticmethod
    def backward(ctx, dl, dh):
        h0a, h1a, h0b, h1b = ctx.taps
        dx = None
        if ctx.needs_input_grad[0]:
            dx = inv_j2plus(dl, _q(dh), h0b, h1b, h0a, h1a)   # trees swap
        return dx, None, None, None, None, None


class INV1D_J1(Function):
    """Differentiable level-1 inverse: ``apply(lo, yh, g0o, g1o, mode)``; lo / yh may be None or 0-dim (zeros)."""

    @staticmethod
    def forward(ctx, lo, yh, g0, g1, mode):
        ctx.mode = int(mode)
        ctx.taps = (_ffi.host_taps(g0), _ffi.host_taps(g1))
        ctx.has = (not _is_empty(lo), not _is_empty(yh))
        return inv_j1(lo if ctx.has[0] else None, _q(yh), ctx.taps[0], ctx.taps[1], ctx.mode)

    @staticmethod
    def backward(ctx, dy):
        need_l = ctx.needs_input_grad[0] and ctx.has[0]
        need_h = ctx.needs_input_grad[1] and ctx.has[1]
        dl = dh = None
        if need_l or need_h:
            dl, dh = fwd_j1(dy, ctx.taps[0], ctx.taps[1], not need_h, ctx.mode)
            dl = dl if need_l else None
            dh = None if dh is None else _c(dh)
        return dl, dh, None, None, None


class INV1D_J2PLUS(Function):
    """Differentiable level >= 2 inverse: ``apply(lo, yh, g0a, g1a, g0b, g1b)``; lo / yh may be None or 0-dim."""

    @staticmethod
    def forward(ctx, lo, yh, g0a, g1a, g0b, g1b):
        ctx.taps = tuple(_ffi.host_taps(f) for f in (g0a, g1a, g0b, g1b))
        ctx.has = (not _is_empty(lo), not _is_empty(yh))
        return inv_j2plus(lo if ctx.has[0] else None, _q(yh), *ctx.taps)

    @staticmethod
    def backward(ctx, dy):
        g0a, g1a, g0b, g1b = ctx.taps
        need_l = ctx.needs_input_grad[0] and ctx.has[0]
        need_h = ctx.needs_input_grad[1] and ctx.has[1]
        dl = dh = None
        if need_l or need_h:
            dl, dh = fwd_j2plus(dy, g0b, g1b, g0a, g1a, not need_h)   # trees swap
            dl = dl if need_l else None
            dh = None if dh is None else _c(dh)
        return dl, dh, None, None, None, None


# ---- modules -------------------------------------------------------------------------------------------------------

class DTCWT1DForward(nn.Module):
    """1-D DTCWT forward decomposition of the rows of an (N, C, n) tensor.

    Args:
        biort (str | (h0o, h1o)): level-1 biorthogonal filters: 'antonini', 'legall', 'near_sym_a', 'near_sym_b'.
        qshift (str | (h0a, h0b, h1a, h1b)): level >= 2 quarter-shift filters: 'qshift_06', 'qshift_a' .. 'qshift_d',
            'qshift_32'.
        J (int): number of levels.
        skip_hps (bool | list[bool]): skip the band-pass outputs of a level (0-dim tensor returned instead).
        include_scale (bool | list[bool]): return the low-passes of all levels instead of the last one.
        mode (str): 'symmetric' or 'zero' extension at level 1 (levels >= 2 are always symmetric).

    ``forward(x)`` returns ``(yl, yh)``; ``yh[j]`` has shape (N, C, n_j / 2, 2), real and imaginary parts last.
    An odd n repeats the last sample; a level >= 2 input whose length is not a multiple of 4 is padded by one
    replicated sample at each end.
    """

    def __init__(self, biort='near_sym_a', qshift='qshift_a', J=3, skip_hps=False, include_scale=False,
                 mode='symmetric'):
        super().__init__()
        self.biort = biort
        self.qshift = qshift
        self.J = J
        self.mode = mode
        if isinstance(biort, str):
            h0o, _, h1o, _ = _biort(biort)[:4]
        else:
            h0o, h1o = biort[0], biort[1]
        self.register_buffer('h0o', prep_filt(h0o, 1))
        self.register_buffer('h1o', prep_filt(h1o, 1))
        if isinstance(qshift, str):
            h0a, h0b, _, _, h1a, h1b, _, _ = _qshift(qshift)[:8]
        else:
            h0a, h0b, h1a, h1b = qshift[:4]
        self.register_buffer('h0a', prep_filt(h0a, 1))
        self.register_buffer('h0b', prep_filt(h0b, 1))
        self.register_buffer('h1a', prep_filt(h1a, 1))
        self.register_buffer('h1b', prep_filt(h1b, 1))
        if isinstance(skip_hps, (list, tuple, ndarray)):
            self.skip_hps = skip_hps
        else:
            self.skip_hps = [skip_hps, ] * self.J
        if isinstance(include_scale, (list, tuple, ndarray)):
            self.include_scale = include_scale
        else:
            self.include_scale = [include_scale, ] * self.J

    def forward(self, x):
        if self.J == 0:
            return x, None
        _check3(x, 'x')
        mode = mode_to_int(self.mode)
        scales = [x.new_zeros([]), ] * self.J
        highs = [x.new_zeros([]), ] * self.J
        if x.shape[-1] % 2 != 0:
            x = torch.cat((x, x[:, :, -1:]), dim=2)
        low, h = FWD1D_J1.apply(x, self.h0o, self.h1o, self.skip_hps[0], mode)
        highs[0] = h
        if self.include_scale[0]:
            scales[0] = low
        for j in range(1, self.J):
            if low.shape[-1] % 4 != 0:
                low = torch.cat((low[:, :, 0:1], low, low[:, :, -1:]), dim=2)
            low, h = FWD1D_J2PLUS.apply(low, self.h0a, self.h1a, self.h0b, self.h1b, self.skip_hps[j])
            highs[j] = h
            if self.include_scale[j]:
                scales[j] = low
        if True in self.include_scale:
            return scales, highs
        return low, highs


class DTCWT1DInverse(nn.Module):
    """1-D DTCWT inverse.  ``forward((yl, yh))`` accepts ``None`` / 0-dim tensors for any band-pass level (zeros).
    A low-pass one sample longer at each end than twice its band's complex length (the forward's replicate padding)
    is trimmed first."""

    def __init__(self, biort='near_sym_a', qshift='qshift_a', mode='symmetric'):
        super().__init__()
        self.biort = biort
        self.qshift = qshift
        self.mode = mode
        if isinstance(biort, str):
            _, g0o, _, g1o = _biort(biort)[:4]
        else:
            g0o, g1o = biort[0], biort[1]
        self.register_buffer('g0o', prep_filt(g0o, 1))
        self.register_buffer('g1o', prep_filt(g1o, 1))
        if isinstance(qshift, str):
            _, _, g0a, g0b, _, _, g1a, g1b = _qshift(qshift)[:8]
        else:
            g0a, g0b, g1a, g1b = qshift[:4]
        self.register_buffer('g0a', prep_filt(g0a, 1))
        self.register_buffer('g0b', prep_filt(g0b, 1))
        self.register_buffer('g1a', prep_filt(g1a, 1))
        self.register_buffer('g1b', prep_filt(g1b, 1))

    @staticmethod
    def _trim(low, s):
        if not _is_empty(s) and low.shape[-1] != 2 * s.shape[-2]:
            low = low[:, :, 1:-1]
        return low

    def forward(self, coeffs):
        low, highs = coeffs
        mode = mode_to_int(self.mode)
        for j in range(len(highs) - 1, 0, -1):
            low = self._trim(low, highs[j])
            low = INV1D_J2PLUS.apply(low, highs[j], self.g0a, self.g1a, self.g0b, self.g1b)
        low = self._trim(low, highs[0])
        return INV1D_J1.apply(low, highs[0], self.g0o, self.g1o, mode)
