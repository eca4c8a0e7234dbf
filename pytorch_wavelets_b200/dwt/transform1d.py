"""``DWT1DForward`` / ``DWT1DInverse`` with the reference's constructor signatures, buffer names and return structure
(reference ``pytorch_wavelets/dwt/transform1d.py:7-115``), each level one CUDA kernel behind the C ABI
(``b200w_dwt_afb1d`` / ``b200w_dwt_sfb1d``)."""
import torch
import torch.nn as nn
from torch.autograd import Function

from pytorch_wavelets_b200 import _ffi, wavelets
from pytorch_wavelets_b200.dwt import lowlevel


def afb1d_level(x, h0, h1, mode):
    """x (N, C, L) -> lo, hi (N, C, K); stored (reversed) analysis taps."""
    dt = _ffi.require_cuda_real(x, 'x')
    lowlevel._check_bank_mode(mode)
    L = _ffi.lib()
    h0, h1 = _ffi.host_taps(h0), _ffi.host_taps(h1)
    if h0.n != h1.n:
        raise ValueError('low-pass and high-pass filters must have equal length')
    x = x.contiguous()
    N, C, n = x.shape
    K = L.b200w_dwt_coeff_len(n, h0.n, mode)
    lo, hi = x.new_empty((N, C, K)), x.new_empty((N, C, K))
    if N * C > 0:
        with torch.cuda.device(x.device), _ffi.span('dwt_afb1d %d L%d' % (n, h0.n), 4 * N * C * (n + 2 * K)):
            rc = (L.b200w_dwt_afb1d_f64 if dt == torch.float64 else L.b200w_dwt_afb1d)(x.data_ptr(), n, N * C, n, lo.data_ptr(), hi.data_ptr(), h0.p(dt), h1.p(dt), h0.n, mode,
                                   _ffi.stream_of(x))
        _ffi.check(rc, 'b200w_dwt_afb1d')
    return lo, hi


def sfb1d_level(lo, hi, g0, g1, mode, out_len=None):
    """lo, hi (N, C, K) (hi may be None) -> y (N, C, rec_len) or cropped to ``out_len``; stored synthesis taps."""
    dt = _ffi.require_cuda_real(lo, 'low')
    lowlevel._check_bank_mode(mode)
    L = _ffi.lib()
    g0, g1 = _ffi.host_taps(g0), _ffi.host_taps(g1)
    lo = lo.contiguous()
    N, C, K = lo.shape
    if hi is not None:
        _ffi.require_cuda_real(hi, 'high', dt)
        if tuple(hi.shape) != tuple(lo.shape):
            raise ValueError('high shape {} does not match low shape {}'.format(tuple(hi.shape), tuple(lo.shape)))
        hi = hi.contiguous()
    n = L.b200w_dwt_rec_len(K, g0.n, mode)
    if out_len is not None:
        n = min(n, int(out_len))
    if n < 1:
        raise ValueError('coefficient array of length {} too small for a {}-tap synthesis filter'.format(K, g0.n))
    y = lo.new_empty((N, C, n))
    if N * C > 0:
        with torch.cuda.device(lo.device), _ffi.span('dwt_sfb1d %d L%d' % (K, g0.n), 4 * N * C * (2 * K + n)):
            rc = (L.b200w_dwt_sfb1d_f64 if dt == torch.float64 else L.b200w_dwt_sfb1d)(lo.data_ptr(), None if hi is None else hi.data_ptr(), N * C, K, y.data_ptr(), n,
                                   g0.p(dt), g1.p(dt), g0.n, mode, _ffi.stream_of(lo))
        _ffi.check(rc, 'b200w_dwt_sfb1d')
    return y


def afb1d_adjoint_level(lo, hi, f0, f1, mode, n):
    """The transpose of ``afb1d_level`` in mode ``mode`` (``b200w_dwt_afb1d_adjoint``): lo, hi (N, C, K) (hi may be
    None) -> (N, C, n), n the analysis input length; stored analysis taps.  Equals ``sfb1d_level(..., out_len=n)`` in
    zero mode and even-size periodization (the C entry then launches only the synthesis kernel)."""
    dt = _ffi.require_cuda_real(lo, 'low')
    lowlevel._check_bank_mode(mode)
    L = _ffi.lib()
    f0, f1 = lowlevel._taps_pair(f0, f1)
    lo = lo.contiguous()
    N, C, K = lo.shape
    n = int(n)
    if K != L.b200w_dwt_coeff_len(n, f0.n, mode):
        raise ValueError('{} coefficients are not the analysis of a length-{} signal'.format(K, n))
    if hi is not None:
        _ffi.require_cuda_real(hi, 'high', dt)
        if tuple(hi.shape) != tuple(lo.shape):
            raise ValueError('high shape {} does not match low shape {}'.format(tuple(hi.shape), tuple(lo.shape)))
        hi = hi.contiguous()
    y = lo.new_empty((N, C, n))
    if N * C > 0:
        with torch.cuda.device(lo.device), _ffi.span('dwt_afb1d_adjoint %d L%d' % (K, f0.n),
                                                     lo.element_size() * N * C * (2 * K + n)):
            rc = _ffi.entry('b200w_dwt_afb1d_adjoint', dt)(lo.data_ptr(), None if hi is None else hi.data_ptr(),
                                                           N * C, K, y.data_ptr(), n, f0.p(dt), f1.p(dt), f0.n, mode,
                                                           _ffi.stream_of(lo))
        _ffi.check(rc, 'b200w_dwt_afb1d_adjoint')
    return y


# The backward passes as autograd Functions, each the other's transpose (see dwt/lowlevel.py, SynthesisCrop2D):
#   SynthesisCrop1D  crop_n . S  <->  SynthesisCrop1DT  zero-mode analysis (periodization: of the signal padded to even n)
#   Analysis1D       A_m         <->  Analysis1DT       A_m^T (b200w_dwt_afb1d_adjoint)

class SynthesisCrop1D(Function):
    """``apply(lo, hi, f0, f1, mode, n)``: the synthesis cropped to n (``AFB1D``'s backward pass)."""

    @staticmethod
    def forward(ctx, lo, hi, f0, f1, mode, n):
        ctx.taps, ctx.mode, ctx.has_hi = (f0, f1), mode, hi is not None
        return sfb1d_level(lo, hi, f0, f1, mode, out_len=n)

    @staticmethod
    def backward(ctx, dy):
        dlo = dhi = None
        if ctx.needs_input_grad[0] or (ctx.has_hi and ctx.needs_input_grad[1]):
            dlo, dhi = SynthesisCrop1DT.apply(dy, *ctx.taps, ctx.mode)
            if not ctx.has_hi:
                dhi = None
        return dlo, dhi, None, None, None, None


class SynthesisCrop1DT(Function):
    """``apply(y, f0, f1, mode) -> (lo, hi)``: the transpose of ``SynthesisCrop1D`` for a length-n y."""

    @staticmethod
    def forward(ctx, y, f0, f1, mode):
        ctx.taps, ctx.mode, ctx.n = (f0, f1), mode, y.shape[-1]
        if mode == lowlevel._MODES['periodization']:
            y = lowlevel._pad_odd(y, (-1,))
        else:
            mode = lowlevel._MODES['zero']
        return afb1d_level(y, f0, f1, mode)

    @staticmethod
    def backward(ctx, dlo, dhi):
        dy = None
        if ctx.needs_input_grad[0]:
            dy = SynthesisCrop1D.apply(dlo, dhi, *ctx.taps, ctx.mode, ctx.n)
        return dy, None, None, None


class Analysis1D(Function):
    """``apply(x, f0, f1, mode) -> (lo, hi)``: the analysis in mode ``mode`` (``SFB1D``'s backward pass)."""

    @staticmethod
    def forward(ctx, x, f0, f1, mode):
        ctx.taps, ctx.mode, ctx.n = (f0, f1), mode, x.shape[-1]
        return afb1d_level(x, f0, f1, mode)

    @staticmethod
    def backward(ctx, dlo, dhi):
        dx = None
        if ctx.needs_input_grad[0]:
            dx = Analysis1DT.apply(dlo, dhi, *ctx.taps, ctx.mode, ctx.n)
        return dx, None, None, None


class Analysis1DT(Function):
    """``apply(lo, hi, f0, f1, mode, n) -> y``: the transpose of ``Analysis1D`` for a length-n input."""

    @staticmethod
    def forward(ctx, lo, hi, f0, f1, mode, n):
        ctx.taps, ctx.mode = (f0, f1), mode
        return afb1d_adjoint_level(lo, hi, f0, f1, mode, n)

    @staticmethod
    def backward(ctx, dy):
        dlo = dhi = None
        if ctx.needs_input_grad[0] or ctx.needs_input_grad[1]:
            dlo, dhi = Analysis1D.apply(dy.contiguous(), *ctx.taps, ctx.mode)
        return dlo, dhi, None, None, None, None


class AFB1D(Function):
    """Single-level 1-D analysis; drop-in for the reference ``AFB1D`` (dwt/lowlevel.py:368-424):
    ``apply(x, h0, h1, mode) -> (x0, x1)``; backward = synthesis with the same filters, cropped to the input length
    (``SynthesisCrop1D``, differentiable to any order)."""

    @staticmethod
    def forward(ctx, x, h0, h1, mode):
        mode = int(mode)
        lowlevel.int_to_mode(mode)
        ctx.mode, ctx.n = mode, x.shape[-1]
        ctx.taps = (_ffi.host_taps(h0), _ffi.host_taps(h1))
        return afb1d_level(x, ctx.taps[0], ctx.taps[1], mode)

    @staticmethod
    def backward(ctx, dx0, dx1):
        dx = None
        if ctx.needs_input_grad[0]:
            dx = SynthesisCrop1D.apply(dx0, dx1, ctx.taps[0], ctx.taps[1], ctx.mode, ctx.n)
        return dx, None, None, None


class SFB1D(Function):
    """Single-level 1-D synthesis; drop-in for the reference ``SFB1D`` (dwt/lowlevel.py:697-743).  Backward = the
    analysis with the same filters (``Analysis1D``, differentiable to any order)."""

    @staticmethod
    def forward(ctx, low, high, g0, g1, mode):
        mode = int(mode)
        lowlevel.int_to_mode(mode)
        ctx.mode = mode
        ctx.taps = (_ffi.host_taps(g0), _ffi.host_taps(g1))
        return sfb1d_level(low, high, ctx.taps[0], ctx.taps[1], mode)

    @staticmethod
    def backward(ctx, dy):
        dlow = dhigh = None
        if ctx.needs_input_grad[0] or ctx.needs_input_grad[1]:
            dlow, dhigh = Analysis1D.apply(dy.contiguous(), ctx.taps[0], ctx.taps[1], ctx.mode)
        return dlow, dhigh, None, None, None


def _wave_pair(wave, analysis):
    if isinstance(wave, str):
        wave = wavelets.Wavelet(wave)
    if hasattr(wave, 'dec_lo') and hasattr(wave, 'rec_lo'):
        return (wave.dec_lo, wave.dec_hi) if analysis else (wave.rec_lo, wave.rec_hi)
    assert len(wave) == 2
    return wave[0], wave[1]


class DWT1DForward(nn.Module):
    """1-D DWT of a batch of signals (drop-in for the reference ``DWT1DForward``).  ``forward(x)`` with x (N, C, L)
    float32 on a CUDA device returns ``(yl, yh)``: the final low-pass and the list of J band-passes, finest first."""

    def __init__(self, J=1, wave='db1', mode='zero'):
        super().__init__()
        h0, h1 = _wave_pair(wave, True)
        filts = lowlevel.prep_filt_afb1d(h0, h1)
        self.register_buffer('h0', filts[0])
        self.register_buffer('h1', filts[1])
        self.J = J
        self.mode = mode

    def forward(self, x):
        assert x.ndim == 3, "Can only handle 3d inputs (N, C, L)"
        highs = []
        x0 = x
        mode = lowlevel.mode_to_int(self.mode)
        for _ in range(self.J):
            x0, x1 = AFB1D.apply(x0, self.h0, self.h1, mode)
            highs.append(x1)
        return x0, highs


class DWT1DInverse(nn.Module):
    """1-D inverse DWT (drop-in for the reference ``DWT1DInverse``); ``None`` band-passes count as zeros."""

    def __init__(self, wave='db1', mode='zero'):
        super().__init__()
        g0, g1 = _wave_pair(wave, False)
        filts = lowlevel.prep_filt_sfb1d(g0, g1)
        self.register_buffer('g0', filts[0])
        self.register_buffer('g1', filts[1])
        self.mode = mode

    def forward(self, coeffs):
        x0, highs = coeffs
        assert x0.ndim == 3, "Can only handle 3d inputs (N, C, L)"
        mode = lowlevel.mode_to_int(self.mode)
        for x1 in highs[::-1]:
            if x1 is not None and x0.shape[-1] > x1.shape[-1]:
                x0 = x0[..., :-1]          # 'unpad' (reference :111-112)
            x0 = SFB1D.apply(x0, x1, self.g0, self.g1, mode)
        return x0
