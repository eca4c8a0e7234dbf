"""Single-level 2-D DWT analysis / synthesis on the H100 engine.

Mirrors the reference's Function layer (``pytorch_wavelets/dwt/lowlevel.py``: ``AFB2D`` :312-365,
``SFB2D`` :647-694, ``prep_filt_afb2d`` :925-953, ``prep_filt_sfb2d`` :870-899, ``mode_to_int`` :274-290)
-- same names, argument order (including the row/col naming quirk), return structure and error
behaviour -- but every level is ONE fused CUDA kernel behind the C ABI (``b200w_dwt_afb2d`` /
``b200w_dwt_sfb2d``) instead of a sequence of ATen convolutions, gathers and copies.
"""
import ctypes

import numpy as np
import torch
from torch.autograd import Function

from pytorch_wavelets_b200 import _ffi

_MODES = {'zero': 0, 'symmetric': 1, 'per': 2, 'periodization': 2, 'constant': 3, 'reflect': 4,
          'replicate': 5, 'periodic': 6}
_MODE_NAMES = {0: 'zero', 1: 'symmetric', 2: 'periodization', 3: 'constant', 4: 'reflect', 5: 'replicate',
               6: 'periodic'}
# padding modes the filter banks implement (reference afb1d :134-170 / sfb1d :252-269)
_BANK_MODES = (0, 1, 2, 4, 6)


def mode_to_int(mode):
    """Reference ``mode_to_int`` (dwt/lowlevel.py:274-290)."""
    try:
        return _MODES[mode]
    except (KeyError, TypeError):
        raise ValueError("Unkown pad type: {}".format(mode))


def int_to_mode(mode):
    """Reference ``int_to_mode`` (dwt/lowlevel.py:293-309)."""
    try:
        return _MODE_NAMES[mode]
    except (KeyError, TypeError):
        raise ValueError("Unkown pad type: {}".format(mode))


def _check_bank_mode(mode):
    if mode not in _BANK_MODES:
        raise ValueError("Unkown pad type: {}".format(_MODE_NAMES.get(mode, mode)))


def prep_filt_afb1d(h0, h1, device=None):
    """Analysis filters -> time-reversed (1,1,L) tensors (reference :956-975)."""
    h0 = np.array(h0[::-1]).ravel()
    h1 = np.array(h1[::-1]).ravel()
    t = torch.get_default_dtype()
    h0 = torch.tensor(h0, device=device, dtype=t).reshape((1, 1, -1))
    h1 = torch.tensor(h1, device=device, dtype=t).reshape((1, 1, -1))
    return h0, h1


def prep_filt_sfb1d(g0, g1, device=None):
    """Synthesis filters -> (1,1,L) tensors, not reversed (reference :902-922)."""
    g0 = np.array(g0).ravel()
    g1 = np.array(g1).ravel()
    t = torch.get_default_dtype()
    g0 = torch.tensor(g0, device=device, dtype=t).reshape((1, 1, -1))
    g1 = torch.tensor(g1, device=device, dtype=t).reshape((1, 1, -1))
    return g0, g1


def prep_filt_afb2d(h0_col, h1_col, h0_row=None, h1_row=None, device=None):
    """Reference ``prep_filt_afb2d`` (:925-953): (1,1,L,1) column and (1,1,1,L) row filters, reversed."""
    h0_col, h1_col = prep_filt_afb1d(h0_col, h1_col, device)
    if h0_row is None:
        h0_row, h1_row = h0_col, h1_col
    else:
        h0_row, h1_row = prep_filt_afb1d(h0_row, h1_row, device)
    h0_col = h0_col.reshape((1, 1, -1, 1))
    h1_col = h1_col.reshape((1, 1, -1, 1))
    h0_row = h0_row.reshape((1, 1, 1, -1))
    h1_row = h1_row.reshape((1, 1, 1, -1))
    return h0_col, h1_col, h0_row, h1_row


def prep_filt_sfb2d(g0_col, g1_col, g0_row=None, g1_row=None, device=None):
    """Reference ``prep_filt_sfb2d`` (:870-899)."""
    g0_col, g1_col = prep_filt_sfb1d(g0_col, g1_col, device)
    if g0_row is None:
        g0_row, g1_row = g0_col, g1_col
    else:
        g0_row, g1_row = prep_filt_sfb1d(g0_row, g1_row, device)
    g0_col = g0_col.reshape((1, 1, -1, 1))
    g1_col = g1_col.reshape((1, 1, -1, 1))
    g0_row = g0_row.reshape((1, 1, 1, -1))
    g1_row = g1_row.reshape((1, 1, 1, -1))
    return g0_col, g1_col, g0_row, g1_row


# ---- raw kernel calls -----------------------------------------------------------------------------------

def afb2d_level(x, fw_lo, fw_hi, fh_lo, fh_hi, mode, pad_ll=False):
    """One analysis level on the GPU.  ``fw_*`` filter along W, ``fh_*`` along H (stored/reversed taps).
    Returns (ll (N,C,Ho,Wo), highs (N,C,3,Ho,Wo)); highs is contiguous, ll is contiguous unless ``pad_ll``:
    then its row pitch is rounded up to a 128-byte line (an internal hand-off between levels: this level
    writes it, and the next level stages it, as whole aligned lines)."""
    dt = _ffi.require_cuda_real(x, 'x')
    _check_bank_mode(mode)
    if x.dim() != 4:
        raise ValueError('expected a 4-D (N,C,H,W) input, got shape {}'.format(tuple(x.shape)))
    L = _ffi.lib()
    fw_lo, fw_hi, fh_lo, fh_hi = [_ffi.host_taps(f) for f in (fw_lo, fw_hi, fh_lo, fh_hi)]
    if fw_lo.n != fw_hi.n or fh_lo.n != fh_hi.n:
        raise ValueError('low-pass and high-pass filters must have equal length')
    N, C, H, W = x.shape
    Ho = L.b200w_dwt_coeff_len(H, fh_lo.n, mode)
    Wo = L.b200w_dwt_coeff_len(W, fw_lo.n, mode)
    x, xps, xpitch = _ffi.planes_view(x)
    Wp = (Wo + 31) // 32 * 32 if pad_ll else Wo
    ll = x.new_empty((N, C, Ho, Wp))
    if Wp != Wo:
        ll = ll[..., :Wo]
    highs = x.new_empty((N, C, 3, Ho, Wo))
    if N * C > 0:
        with torch.cuda.device(x.device), _ffi.span('dwt_afb2d %dx%d L%d' % (H, W, fw_lo.n),
                                                    x.element_size() * N * C * (H * W + 4 * Ho * Wo)):
            rc = _ffi.entry('b200w_dwt_afb2d', dt)(x.data_ptr(), xps, xpitch, ll.data_ptr(), Ho * Wp, Wp, highs.data_ptr(),
                                   N * C, H, W, fw_lo.p(dt), fw_hi.p(dt), fw_lo.n, fh_lo.p(dt), fh_hi.p(dt), fh_lo.n,
                                   mode, _ffi.stream_of(x))
        _ffi.check(rc, 'b200w_dwt_afb2d')
    return ll, highs


def sfb2d_level(ll, highs, gh_lo, gh_hi, gw_lo, gw_hi, mode, out_hw=None):
    """One synthesis level on the GPU.  ``gh_*`` act along H (first pass), ``gw_*`` along W.
    ``highs`` may be None (zeros).  ``out_hw`` crops the output (AFB2D.backward)."""
    dt = _ffi.require_cuda_real(ll, 'low')
    _check_bank_mode(mode)
    L = _ffi.lib()
    gh_lo, gh_hi, gw_lo, gw_hi = [_ffi.host_taps(f) for f in (gh_lo, gh_hi, gw_lo, gw_hi)]
    N, C, Hc, Wc = ll.shape
    if highs is not None:
        _ffi.require_cuda_real(highs, 'highs', dt)
        if tuple(highs.shape) != (N, C, 3, Hc, Wc):
            raise ValueError('highs shape {} does not match low shape {}'.format(tuple(highs.shape), tuple(ll.shape)))
        highs = highs.contiguous()
    Ho = L.b200w_dwt_rec_len(Hc, gh_lo.n, mode)
    Wo = L.b200w_dwt_rec_len(Wc, gw_lo.n, mode)
    if out_hw is not None:
        Ho, Wo = min(Ho, int(out_hw[0])), min(Wo, int(out_hw[1]))
    if Ho < 1 or Wo < 1:
        raise ValueError('coefficient array {}x{} too small for a {}-tap synthesis filter'.format(Hc, Wc, gh_lo.n))
    ll, llps, llpitch = _ffi.planes_view(ll)
    y = ll.new_empty((N, C, Ho, Wo))
    if N * C > 0:
        with torch.cuda.device(ll.device), _ffi.span('dwt_sfb2d %dx%d L%d' % (Hc, Wc, gh_lo.n),
                                                     ll.element_size() * N * C * ((1 if highs is None else 4) * Hc * Wc + Ho * Wo)):
            rc = _ffi.entry('b200w_dwt_sfb2d', dt)(ll.data_ptr(), llps, llpitch, None if highs is None else highs.data_ptr(),
                                   y.data_ptr(), Ho * Wo, Wo, N * C, Hc, Wc, Ho, Wo,
                                   gh_lo.p(dt), gh_hi.p(dt), gh_lo.n, gw_lo.p(dt), gw_hi.p(dt), gw_lo.n, mode,
                                   _ffi.stream_of(ll))
        _ffi.check(rc, 'b200w_dwt_sfb2d')
    return y


def afb2d_adjoint_level(ll, highs, fh_lo, fh_hi, fw_lo, fw_hi, mode, out_hw):
    """The transpose of ``afb2d_level`` in mode ``mode`` (``b200w_dwt_afb2d_adjoint``): ll (N,C,Hc,Wc) and highs
    (N,C,3,Hc,Wc) -> (N,C,H,W) with ``(H, W) = out_hw``, the analysis input size.  ``fh_*`` / ``fw_*``: the stored
    analysis taps along H / W.  Equals ``sfb2d_level(..., out_hw=out_hw)`` in zero mode and even-size
    periodization (the C entry then launches only the synthesis kernel); elsewhere the boundary extension is folded
    back onto the samples it copies."""
    dt = _ffi.require_cuda_real(ll, 'low')
    _check_bank_mode(mode)
    L = _ffi.lib()
    fh_lo, fh_hi = _taps_pair(fh_lo, fh_hi)
    fw_lo, fw_hi = _taps_pair(fw_lo, fw_hi)
    N, C, Hc, Wc = ll.shape
    H, W = int(out_hw[0]), int(out_hw[1])
    if Hc != L.b200w_dwt_coeff_len(H, fh_lo.n, mode) or Wc != L.b200w_dwt_coeff_len(W, fw_lo.n, mode):
        raise ValueError('coefficients {}x{} are not the analysis of a {}x{} input'.format(Hc, Wc, H, W))
    if highs is not None:
        _ffi.require_cuda_real(highs, 'highs', dt)
        if tuple(highs.shape) != (N, C, 3, Hc, Wc):
            raise ValueError('highs shape {} does not match low shape {}'.format(tuple(highs.shape), tuple(ll.shape)))
        highs = highs.contiguous()
    ll, llps, llpitch = _ffi.planes_view(ll)
    y = ll.new_empty((N, C, H, W))
    if N * C > 0:
        with torch.cuda.device(ll.device), _ffi.span('dwt_afb2d_adjoint %dx%d L%d' % (Hc, Wc, fh_lo.n),
                                                     ll.element_size() * N * C * ((1 if highs is None else 4) * Hc * Wc + H * W)):
            rc = _ffi.entry('b200w_dwt_afb2d_adjoint', dt)(
                ll.data_ptr(), llps, llpitch, None if highs is None else highs.data_ptr(), y.data_ptr(), H * W, W,
                N * C, Hc, Wc, H, W, fh_lo.p(dt), fh_hi.p(dt), fh_lo.n, fw_lo.p(dt), fw_hi.p(dt), fw_lo.n, mode,
                _ffi.stream_of(ll))
        _ffi.check(rc, 'b200w_dwt_afb2d_adjoint')
    return y


def _pad_odd(x, dims):
    """x with one zero appended along each dimension of ``dims`` whose size is odd (the periodization analysis of an
    odd-size signal is the analysis of the signal padded to even size)."""
    for d in dims:
        if x.shape[d] % 2:
            shape = list(x.shape)
            shape[d] = 1
            x = torch.cat([x, x.new_zeros(shape)], dim=d)
    return x


def dwt_forward_levels(x, fw_lo, fw_hi, fh_lo, fh_hi, mode, J):
    """All J analysis levels through ONE C-ABI call (``b200w_dwt_forward``): a single fused kernel launch when the
    pyramid kernel applies (no inter-level low-pass in device memory), one launch per level otherwise.
    Returns ``(yl (N,C,H_J,W_J), [yh_1 .. yh_J])`` -- contiguous, the reference's return layout."""
    dt = _ffi.require_cuda_real(x, 'x')
    _check_bank_mode(mode)
    if x.dim() != 4:
        raise ValueError('expected a 4-D (N,C,H,W) input, got shape {}'.format(tuple(x.shape)))
    L = _ffi.lib()
    fw_lo, fw_hi, fh_lo, fh_hi = [_ffi.host_taps(f) for f in (fw_lo, fw_hi, fh_lo, fh_hi)]
    if fw_lo.n != fw_hi.n or fh_lo.n != fh_hi.n:
        raise ValueError('low-pass and high-pass filters must have equal length')
    if dt == torch.float64:   # double precision: one generic-kernel launch per level (b200w_dwt_forward is float32-only)
        ll, yh = x, []
        for _ in range(J):
            ll, h = afb2d_level(ll, fw_lo, fw_hi, fh_lo, fh_hi, mode)
            yh.append(h)
        return ll, yh
    N, C, H, W = x.shape
    x, xps, xpitch = _ffi.planes_view(x)
    sizes = []
    h, w = H, W
    for _ in range(J):
        h, w = L.b200w_dwt_coeff_len(h, fh_lo.n, mode), L.b200w_dwt_coeff_len(w, fw_lo.n, mode)
        sizes.append((h, w))
    yh = [x.new_empty((N, C, 3, hh, ww)) for hh, ww in sizes]
    yl = x.new_empty((N, C) + sizes[-1])
    if N * C > 0:
        with torch.cuda.device(x.device):
            wsb = L.b200w_dwt_forward_workspace(x.data_ptr(), xps, xpitch, N * C, H, W, J, fw_lo.n, fh_lo.n, mode)
            if wsb < 0:
                _ffi.check(int(wsb), 'b200w_dwt_forward_workspace')
            ws = x.new_empty(((wsb + 3) // 4,)) if wsb > 0 else None
            ptrs = (ctypes.c_void_p * J)(*[t.data_ptr() for t in yh])
            alg = 4 * N * C * (H * W + 3 * sum(a * b for a, b in sizes) + sizes[-1][0] * sizes[-1][1])
            tag = ('dwt_pyramid' if wsb == 0 else 'dwt_levels') + ' %dx%d L%d J%d' % (H, W, fw_lo.n, J)
            with _ffi.span(tag, alg):
                rc = _ffi.entry('b200w_dwt_forward')(x.data_ptr(), xps, xpitch, N * C, H, W, J, yl.data_ptr(), ptrs,
                                                     fw_lo.p(dt), fw_hi.p(dt), fw_lo.n, fh_lo.p(dt), fh_hi.p(dt), fh_lo.n,
                                                     mode, None if ws is None else ws.data_ptr(), wsb,
                                                     _ffi.stream_of(x))
        _ffi.check(rc, 'b200w_dwt_forward')
    return yl, yh


def _taps_pair(f0, f1):
    f0, f1 = _ffi.host_taps(f0), _ffi.host_taps(f1)
    if f0.n != f1.n:
        raise ValueError('low-pass and high-pass filters must have equal length')
    return f0, f1


def _workspace(like, nbytes, what):
    if nbytes < 0:
        _ffi.check(int(nbytes), what)
    return like.new_empty(((nbytes + like.element_size() - 1) // like.element_size(),)) if nbytes > 0 else None


def afb3d_level(x, h0, h1, mode):
    """One 3-D analysis level on the GPU (``b200w_dwt_afb3d``): x (N,C,D,H,W) -> (yl (N,C,Do,Ho,Wo),
    highs (N,C,7,Do,Ho,Wo)), both contiguous.  ``h0, h1``: stored (reversed) taps, applied along W, H and D.
    Band b = 4*aW + 2*aH + aD - 1 (aX = 1: high-pass along X).  Honours ``_ffi.generic_kernels()``."""
    if x.dim() != 5:
        raise ValueError('expected a 5-D (N,C,D,H,W) input, got shape {}'.format(tuple(x.shape)))
    dt = _ffi.require_cuda_real(x, 'x')
    _check_bank_mode(mode)
    L = _ffi.lib()
    h0, h1 = _taps_pair(h0, h1)
    N, C, D, H, W = x.shape
    Do, Ho, Wo = [L.b200w_dwt_coeff_len(n, h0.n, mode) for n in (D, H, W)]
    yl = x.new_empty((N, C, Do, Ho, Wo))
    highs = x.new_empty((N, C, 7, Do, Ho, Wo))
    if N * C > 0:
        x, xvs = _ffi.volumes_view(x)
        with torch.cuda.device(x.device):
            wsb = _ffi.entry('b200w_dwt_afb3d_workspace', dt)(x.data_ptr(), xvs, N * C, D, H, W, h0.n, mode)
            ws = _workspace(x, wsb, 'b200w_dwt_afb3d_workspace')
            with _ffi.span('dwt_afb3d %dx%dx%d L%d' % (D, H, W, h0.n),
                           x.element_size() * N * C * (D * H * W + 8 * Do * Ho * Wo)):
                rc = _ffi.entry('b200w_dwt_afb3d', dt)(x.data_ptr(), xvs, yl.data_ptr(), highs.data_ptr(), N * C, D, H, W,
                                                       h0.p(dt), h1.p(dt), h0.n, mode,
                                                       None if ws is None else ws.data_ptr(), max(int(wsb), 0),
                                                       _ffi.stream_of(x))
        _ffi.check(rc, 'b200w_dwt_afb3d')
    return yl, highs


def sfb3d_level(yl, highs, g0, g1, mode, out_dhw=None):
    """One 3-D synthesis level on the GPU (``b200w_dwt_sfb3d``): yl (N,C,Dc,Hc,Wc) and highs (N,C,7,Dc,Hc,Wc) or None
    (zeros) -> y (N,C,Do,Ho,Wo).  ``out_dhw`` crops the output (the analysis backward pass)."""
    if yl.dim() != 5:
        raise ValueError('expected a 5-D (N,C,D,H,W) low-pass, got shape {}'.format(tuple(yl.shape)))
    dt = _ffi.require_cuda_real(yl, 'low')
    _check_bank_mode(mode)
    L = _ffi.lib()
    g0, g1 = _taps_pair(g0, g1)
    N, C, Dc, Hc, Wc = yl.shape
    if highs is not None:
        _ffi.require_cuda_real(highs, 'highs', dt)
        if tuple(highs.shape) != (N, C, 7, Dc, Hc, Wc):
            raise ValueError('highs shape {} does not match low shape {}'.format(tuple(highs.shape), tuple(yl.shape)))
        highs = highs.contiguous()
    out = [L.b200w_dwt_rec_len(n, g0.n, mode) for n in (Dc, Hc, Wc)]
    if out_dhw is not None:
        out = [min(a, int(b)) for a, b in zip(out, out_dhw)]
    if min(out) < 1:
        raise ValueError('coefficient array {}x{}x{} too small for a {}-tap synthesis filter'.format(Dc, Hc, Wc, g0.n))
    Do, Ho, Wo = out
    y = yl.new_empty((N, C, Do, Ho, Wo))
    if N * C > 0:
        yl, ylvs = _ffi.volumes_view(yl)
        with torch.cuda.device(yl.device):
            wsb = _ffi.entry('b200w_dwt_sfb3d_workspace', dt)(N * C, Dc, Hc, Wc, Do, Ho, Wo, g0.n, mode)
            ws = _workspace(yl, wsb, 'b200w_dwt_sfb3d_workspace')
            with _ffi.span('dwt_sfb3d %dx%dx%d L%d' % (Dc, Hc, Wc, g0.n),
                           yl.element_size() * N * C * ((1 if highs is None else 8) * Dc * Hc * Wc + Do * Ho * Wo)):
                rc = _ffi.entry('b200w_dwt_sfb3d', dt)(yl.data_ptr(), ylvs, None if highs is None else highs.data_ptr(),
                                                       y.data_ptr(), N * C, Dc, Hc, Wc, Do, Ho, Wo, g0.p(dt), g1.p(dt),
                                                       g0.n, mode, None if ws is None else ws.data_ptr(),
                                                       max(int(wsb), 0), _ffi.stream_of(yl))
        _ffi.check(rc, 'b200w_dwt_sfb3d')
    return y


# ---- autograd Functions (the reference's drop-in boundary) ------------------------------------------------

class AFB2D(Function):
    """Single-level 2-D analysis filter bank; drop-in for the reference ``AFB2D`` (dwt/lowlevel.py:312-365).

    ``forward(ctx, x, h0_row, h1_row, h0_col, h1_col, mode)``: the ``*_row`` filters act along W
    (dim 3) and the ``*_col`` filters along H (dim 2), exactly as in the reference (:341-342).
    Returns ``(low (N,C,H',W'), highs (N,C,3,H',W'))``.  The backward pass is the synthesis kernel
    with the same stored filters, cropped to the input size (:350-365), as the differentiable ``SynthesisCrop2D``.
    """

    @staticmethod
    def forward(ctx, x, h0_row, h1_row, h0_col, h1_col, mode, pad_ll=False):
        ctx.taps = tuple(_ffi.host_taps(f) for f in (h0_row, h1_row, h0_col, h1_col))
        ctx.shape = x.shape[-2:]
        mode = int(mode)
        int_to_mode(mode)
        ctx.mode = mode
        low, highs = afb2d_level(x, *ctx.taps, mode, pad_ll=bool(pad_ll))
        return low, highs

    @staticmethod
    def backward(ctx, low, highs):
        dx = None
        if ctx.needs_input_grad[0]:
            h0_row, h1_row, h0_col, h1_col = ctx.taps
            dx = SynthesisCrop2D.apply(low, highs, h0_col, h1_col, h0_row, h1_row, ctx.mode, ctx.shape)
        return dx, None, None, None, None, None, None


class SFB2D(Function):
    """Single-level 2-D synthesis filter bank; drop-in for the reference ``SFB2D`` (dwt/lowlevel.py:647-694).

    ``forward(ctx, low, highs, g0_row, g1_row, g0_col, g1_col, mode)``: ``*_col`` filters act along H
    first (:677-678), then ``*_row`` along W (:679).  ``highs`` may be None (treated as zeros).  The backward pass
    is the analysis with the same filters in the same mode (:683-694), as the differentiable ``Analysis2D``.
    """

    @staticmethod
    def forward(ctx, low, highs, g0_row, g1_row, g0_col, g1_col, mode):
        mode = int(mode)
        int_to_mode(mode)
        ctx.mode = mode
        ctx.has_highs = highs is not None
        ctx.taps = tuple(_ffi.host_taps(f) for f in (g0_row, g1_row, g0_col, g1_col))
        g0_row, g1_row, g0_col, g1_col = ctx.taps
        return sfb2d_level(low, highs, g0_col, g1_col, g0_row, g1_row, mode)

    @staticmethod
    def backward(ctx, dy):
        dlow, dhigh = None, None
        if ctx.needs_input_grad[0] or (ctx.has_highs and ctx.needs_input_grad[1]):
            g0_row, g1_row, g0_col, g1_col = ctx.taps
            dlow, dhigh = Analysis2D.apply(dy.contiguous(), g0_col, g1_col, g0_row, g1_row, ctx.mode)
            if not ctx.has_highs:
                dhigh = None
        return dlow, dhigh, None, None, None, None, None


class DWTPyramid(Function):
    """All J levels of ``DWTForward.forward`` (reference dwt/transform2d.py:68-74) as one differentiable op:
    ``apply(x, h0_row, h1_row, h0_col, h1_col, mode, J) -> (yl, yh_1, ..., yh_J)`` with the filter arguments of
    ``AFB2D`` (``*_row`` along W, ``*_col`` along H).  Forward = one fused kernel launch where the pyramid kernel
    applies; backward = the reference's chain of ``AFB2D.backward`` (synthesis with the stored analysis filters,
    cropped to each level's input size, dwt/lowlevel.py:350-365), one ``SynthesisCrop2D`` per level."""

    @staticmethod
    def forward(ctx, x, h0_row, h1_row, h0_col, h1_col, mode, J):
        ctx.taps = tuple(_ffi.host_taps(f) for f in (h0_row, h1_row, h0_col, h1_col))
        mode = int(mode)
        int_to_mode(mode)
        ctx.mode = mode
        yl, yh = dwt_forward_levels(x, *ctx.taps, mode, int(J))
        ctx.in_shapes = [tuple(x.shape[-2:])] + [tuple(h.shape[-2:]) for h in yh[:-1]]
        return (yl,) + tuple(yh)

    @staticmethod
    def backward(ctx, dyl, *dyh):
        dx = None
        if ctx.needs_input_grad[0]:
            h0_row, h1_row, h0_col, h1_col = ctx.taps
            low = dyl
            for j in range(len(dyh) - 1, -1, -1):
                sh = ctx.in_shapes[j]
                if low is None:
                    low = dyh[j].new_zeros(dyh[j].shape[:2] + dyh[j].shape[-2:])
                low = SynthesisCrop2D.apply(low.contiguous(), dyh[j], h0_col, h1_col, h0_row, h1_row, ctx.mode, sh)
            dx = low
        return dx, None, None, None, None, None, None


# ---- the backward passes as autograd Functions (double backward) ------------------------------------------
# Each first-order backward above is one of the four operators below, and each operator's backward is its exact
# transpose, which is again one of them.  So a graph built with create_graph=True differentiates to any order, as the
# reference's torch-op backward passes do.  With grad mode off (a plain .backward()) ``apply`` runs only the forward:
# the same kernel call, with the same arguments, as before these Functions existed.
#   SynthesisCrop2D   crop_(H,W) . S       <->  SynthesisCrop2DT  S^T . pad = zero-mode analysis (periodization: on the
#                                                                 input zero-padded to even size)
#   Analysis2D        A_m                  <->  Analysis2DT       A_m^T (b200w_dwt_afb2d_adjoint)
# Taps are HostTaps in the synthesis argument order: fh_* along H, fw_* along W.  They stay constants.

class SynthesisCrop2D(Function):
    """``apply(low, highs, fh_lo, fh_hi, fw_lo, fw_hi, mode, out_hw)``: the synthesis level cropped to ``out_hw``
    (``AFB2D``'s backward pass).  Its backward pass is ``SynthesisCrop2DT``."""

    @staticmethod
    def forward(ctx, low, highs, fh_lo, fh_hi, fw_lo, fw_hi, mode, out_hw):
        ctx.taps, ctx.mode, ctx.out_hw = (fh_lo, fh_hi, fw_lo, fw_hi), mode, tuple(out_hw)
        ctx.has_highs = highs is not None
        return sfb2d_level(low, highs, fh_lo, fh_hi, fw_lo, fw_hi, mode, out_hw=out_hw)

    @staticmethod
    def backward(ctx, dy):
        dlow = dhigh = None
        if ctx.needs_input_grad[0] or (ctx.has_highs and ctx.needs_input_grad[1]):
            dlow, dhigh = SynthesisCrop2DT.apply(dy, *ctx.taps, ctx.mode)
            if not ctx.has_highs:
                dhigh = None
        return dlow, dhigh, None, None, None, None, None, None


class SynthesisCrop2DT(Function):
    """``apply(y, fh_lo, fh_hi, fw_lo, fw_hi, mode) -> (low, highs)``: the transpose of ``SynthesisCrop2D`` for an
    (H, W) input.  The cropped synthesis does not depend on the mode outside periodization, so this is the zero-mode
    analysis there; in periodization it is the periodization analysis of y zero-padded to even size."""

    @staticmethod
    def forward(ctx, y, fh_lo, fh_hi, fw_lo, fw_hi, mode):
        ctx.taps, ctx.mode, ctx.shape = (fh_lo, fh_hi, fw_lo, fw_hi), mode, tuple(y.shape[-2:])
        if mode == _MODES['periodization']:
            y = _pad_odd(y, (-2, -1))
        else:
            mode = _MODES['zero']
        return afb2d_level(y.contiguous(), fw_lo, fw_hi, fh_lo, fh_hi, mode)

    @staticmethod
    def backward(ctx, dlow, dhighs):
        dy = None
        if ctx.needs_input_grad[0]:
            dy = SynthesisCrop2D.apply(dlow, dhighs, *ctx.taps, ctx.mode, ctx.shape)
        return dy, None, None, None, None, None


class Analysis2D(Function):
    """``apply(x, fh_lo, fh_hi, fw_lo, fw_hi, mode) -> (low, highs)``: the analysis level in mode ``mode``
    (``SFB2D``'s backward pass).  Its backward pass is ``Analysis2DT``."""

    @staticmethod
    def forward(ctx, x, fh_lo, fh_hi, fw_lo, fw_hi, mode):
        ctx.taps, ctx.mode, ctx.shape = (fh_lo, fh_hi, fw_lo, fw_hi), mode, tuple(x.shape[-2:])
        return afb2d_level(x, fw_lo, fw_hi, fh_lo, fh_hi, mode)

    @staticmethod
    def backward(ctx, dlow, dhighs):
        dx = None
        if ctx.needs_input_grad[0]:
            dx = Analysis2DT.apply(dlow, dhighs, *ctx.taps, ctx.mode, ctx.shape)
        return dx, None, None, None, None, None


class Analysis2DT(Function):
    """``apply(low, highs, fh_lo, fh_hi, fw_lo, fw_hi, mode, out_hw) -> y``: the transpose of ``Analysis2D`` for an
    ``out_hw`` input (``afb2d_adjoint_level``).  Its backward pass is ``Analysis2D``."""

    @staticmethod
    def forward(ctx, low, highs, fh_lo, fh_hi, fw_lo, fw_hi, mode, out_hw):
        ctx.taps, ctx.mode = (fh_lo, fh_hi, fw_lo, fw_hi), mode
        return afb2d_adjoint_level(low, highs, fh_lo, fh_hi, fw_lo, fw_hi, mode, out_hw)

    @staticmethod
    def backward(ctx, dy):
        dlow = dhigh = None
        if ctx.needs_input_grad[0] or ctx.needs_input_grad[1]:
            dlow, dhigh = Analysis2D.apply(dy.contiguous(), *ctx.taps, ctx.mode)
        return dlow, dhigh, None, None, None, None, None, None


class AFB3D(Function):
    """Single-level 3-D analysis: ``apply(x, h0, h1, mode) -> (yl, highs)`` with the stored (reversed) analysis taps
    along all three axes.  The backward pass is the synthesis with the same stored taps, cropped to the input size
    (as ``AFB2D.backward``)."""

    @staticmethod
    def forward(ctx, x, h0, h1, mode):
        mode = int(mode)
        int_to_mode(mode)
        ctx.mode, ctx.shape = mode, tuple(x.shape[-3:])
        ctx.taps = (_ffi.host_taps(h0), _ffi.host_taps(h1))
        return afb3d_level(x, ctx.taps[0], ctx.taps[1], mode)

    @staticmethod
    def backward(ctx, dyl, dhighs):
        dx = None
        if ctx.needs_input_grad[0]:
            dx = sfb3d_level(dyl.contiguous(), dhighs, ctx.taps[0], ctx.taps[1], ctx.mode, out_dhw=ctx.shape)
        return dx, None, None, None


class SFB3D(Function):
    """Single-level 3-D synthesis: ``apply(yl, highs, g0, g1, mode) -> y``; ``highs`` may be None (zeros).  The
    backward pass is the analysis with the synthesis taps (as ``SFB2D.backward``)."""

    @staticmethod
    def forward(ctx, yl, highs, g0, g1, mode):
        mode = int(mode)
        int_to_mode(mode)
        ctx.mode, ctx.has_highs = mode, highs is not None
        ctx.taps = (_ffi.host_taps(g0), _ffi.host_taps(g1))
        return sfb3d_level(yl, highs, ctx.taps[0], ctx.taps[1], mode)

    @staticmethod
    def backward(ctx, dy):
        dyl = dhighs = None
        if ctx.needs_input_grad[0] or (ctx.has_highs and ctx.needs_input_grad[1]):
            dyl, dhighs = afb3d_level(dy.contiguous(), ctx.taps[0], ctx.taps[1], ctx.mode)
            if not ctx.has_highs:
                dhighs = None
        return dyl, dhighs, None, None, None
