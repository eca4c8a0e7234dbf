"""2-D wavelet packet transform: ``WPT2DForward`` / ``WPT2DInverse``.

In a packet transform every band is split again at every level, not only the low-pass.  Level j+1 applies one DWT
analysis level (``AFB2D``'s arithmetic) to every node of level j; the children of node p are nodes 4p .. 4p+3 in
``DWTForward``'s band order (ll, lh, hl, hh).  That is the *natural* order: node index written in base 4 as
b_1 ... b_J, b_1 the band taken at level 1 and the most significant digit.  Each level is one launch of a kernel that
writes all four children of every plane straight into that layout (``b200w_wpt_afb2d``, csrc/wpt2d.cu), so the
(P, 4, Ho, Wo) output of a level is the next level's list of 4P planes with no copy in between.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.autograd import Function

from pytorch_wavelets_b200 import _ffi
from pytorch_wavelets_b200.dwt import lowlevel
from pytorch_wavelets_b200.dwt.transform2d import _resolve_wave


def _taps4(*fs):
    fs = [_ffi.host_taps(f) for f in fs]
    if fs[0].n != fs[1].n or fs[2].n != fs[3].n:
        raise ValueError('low-pass and high-pass filters must have equal length')
    return fs


def wpt_afb2d_level(x, fw_lo, fw_hi, fh_lo, fh_hi, mode, pad=False):
    """One packet analysis level on the GPU.  ``x``: (B, P, H, W), any layout whose rows are unit-stride and whose
    (B, P) planes have one plane stride (else it is copied).  ``fw_*`` filter along W, ``fh_*`` along H (stored taps).
    Returns y (B, 4P, Ho, Wo), node 4p + b = band b of plane p.  ``pad``: the row pitch of y is rounded up to 32
    elements (an internal hand-off between levels, so that odd sizes still give aligned rows to the next level)."""
    dt = _ffi.require_cuda_real(x, 'x')
    lowlevel._check_bank_mode(mode)
    if x.dim() != 4:
        raise ValueError('expected a 4-D (B,P,H,W) input, got shape {}'.format(tuple(x.shape)))
    L = _ffi.lib()
    fw_lo, fw_hi, fh_lo, fh_hi = _taps4(fw_lo, fw_hi, fh_lo, fh_hi)
    B, P, H, W = x.shape
    Ho = L.b200w_dwt_coeff_len(H, fh_lo.n, mode)
    Wo = L.b200w_dwt_coeff_len(W, fw_lo.n, mode)
    x, xps, xpitch = _ffi.planes_view(x)
    Wp = (Wo + 31) // 32 * 32 if pad else Wo
    y = x.new_empty((B, 4 * P, Ho, Wp))
    if Wp != Wo:
        y = y[..., :Wo]
    if B * P > 0:
        with torch.cuda.device(x.device), _ffi.span('wpt_afb2d %dx%d L%d' % (H, W, fw_lo.n),
                                                    x.element_size() * B * P * (H * W + 4 * Ho * Wo)):
            rc = _ffi.entry('b200w_wpt_afb2d', dt)(x.data_ptr(), xps, xpitch, y.data_ptr(), Ho * Wp, Wp, B * P, H, W,
                                                   fw_lo.p(dt), fw_hi.p(dt), fw_lo.n, fh_lo.p(dt), fh_hi.p(dt),
                                                   fh_lo.n, mode, _ffi.stream_of(x))
        _ffi.check(rc, 'b200w_wpt_afb2d')
    return y


def wpt_sfb2d_level(c, gh_lo, gh_hi, gw_lo, gw_hi, mode, out_hw=None):
    """One packet synthesis level on the GPU: c (B, 4P, Hc, Wc) -> y (B, P, Ho, Wo), plane p rebuilt from nodes
    4p .. 4p+3.  ``gh_*`` act along H (first pass), ``gw_*`` along W.  ``out_hw`` crops the output."""
    dt = _ffi.require_cuda_real(c, 'coefficients')
    lowlevel._check_bank_mode(mode)
    if c.dim() != 4 or c.shape[1] % 4:
        raise ValueError('expected a (B, 4P, H, W) coefficient tensor, got shape {}'.format(tuple(c.shape)))
    L = _ffi.lib()
    gh_lo, gh_hi, gw_lo, gw_hi = _taps4(gh_lo, gh_hi, gw_lo, gw_hi)
    B, P4, Hc, Wc = c.shape
    Ho = L.b200w_dwt_rec_len(Hc, gh_lo.n, mode)
    Wo = L.b200w_dwt_rec_len(Wc, gw_lo.n, mode)
    if out_hw is not None:
        Ho, Wo = min(Ho, int(out_hw[0])), min(Wo, int(out_hw[1]))
    if Ho < 1 or Wo < 1:
        raise ValueError('coefficient array {}x{} too small for a {}-tap synthesis filter'.format(Hc, Wc, gh_lo.n))
    c = c.contiguous()
    y = c.new_empty((B, P4 // 4, Ho, Wo))
    if B * P4 > 0:
        with torch.cuda.device(c.device), _ffi.span('wpt_sfb2d %dx%d L%d' % (Hc, Wc, gh_lo.n),
                                                    c.element_size() * B * P4 // 4 * (4 * Hc * Wc + Ho * Wo)):
            rc = _ffi.entry('b200w_wpt_sfb2d', dt)(c.data_ptr(), y.data_ptr(), Ho * Wo, Wo, B * P4 // 4, Hc, Wc, Ho, Wo,
                                                   gh_lo.p(dt), gh_hi.p(dt), gh_lo.n, gw_lo.p(dt), gw_hi.p(dt),
                                                   gw_lo.n, mode, _ffi.stream_of(c))
        _ffi.check(rc, 'b200w_wpt_sfb2d')
    return y


def packet_sizes(H, W, J, Lh, Lw, mode):
    """[(H_0, W_0), ..., (H_J, W_J)] under the forward length rule (``b200w_dwt_coeff_len``)."""
    L = _ffi.lib()
    sizes = [(int(H), int(W))]
    for _ in range(J):
        h, w = sizes[-1]
        sizes.append((L.b200w_dwt_coeff_len(h, Lh, mode), L.b200w_dwt_coeff_len(w, Lw, mode)))
    return sizes


class WPT2DAnalysis(Function):
    """All J packet analysis levels as one differentiable op: ``apply(x, h0_row, h1_row, h0_col, h1_col, mode, J)``
    -> (N, C, 4^J, H_J, W_J), with ``AFB2D``'s filter arguments (``*_row`` along W, ``*_col`` along H).  No
    intermediate level is saved.  The backward pass follows ``AFB2D.backward``: packet synthesis with the stored
    analysis taps, each level cropped to its input size (the exact gradient in zero mode and even-size
    periodization only, like the DWT's)."""

    @staticmethod
    def forward(ctx, x, h0_row, h1_row, h0_col, h1_col, mode, J):
        ctx.taps = tuple(_ffi.host_taps(f) for f in (h0_row, h1_row, h0_col, h1_col))
        mode = int(mode)
        lowlevel.int_to_mode(mode)
        ctx.mode = mode
        N, C = x.shape[:2]
        y = x
        ctx.in_shapes = []
        for j in range(J):
            ctx.in_shapes.append(tuple(y.shape[-2:]))
            y = wpt_afb2d_level(y, *ctx.taps, mode, pad=(j + 1 < J))
        return y.reshape(N, C, 4 ** J, y.shape[-2], y.shape[-1])

    @staticmethod
    def backward(ctx, dy):
        dx = None
        if ctx.needs_input_grad[0]:
            h0_row, h1_row, h0_col, h1_col = ctx.taps
            N, C = dy.shape[:2]
            g = dy.reshape(N, C * dy.shape[2], dy.shape[3], dy.shape[4])
            for sh in ctx.in_shapes[::-1]:
                g = wpt_sfb2d_level(g, h0_col, h1_col, h0_row, h1_row, ctx.mode, out_hw=sh)
            dx = g
        return dx, None, None, None, None, None, None


class WPT2DSynthesis(Function):
    """All packet synthesis levels as one differentiable op: ``apply(y, g0_row, g1_row, g0_col, g1_col, mode, sizes)``
    with ``SFB2D``'s filter arguments; ``sizes`` = [(H_0, W_0), ..., (H_{J-1}, W_{J-1})] the output size of each level
    (finest first), or None entries for the natural ``rec_len`` size.  The backward pass follows ``SFB2D.backward``:
    packet analysis with the synthesis taps, of each level's gradient zero-padded from its crop to its ``rec_len``
    size (the backward of ``SFB2D`` followed by a slice)."""

    @staticmethod
    def forward(ctx, y, g0_row, g1_row, g0_col, g1_col, mode, sizes):
        mode = int(mode)
        lowlevel.int_to_mode(mode)
        ctx.mode = mode
        ctx.taps = tuple(_ffi.host_taps(f) for f in (g0_row, g1_row, g0_col, g1_col))
        g0_row, g1_row, g0_col, g1_col = ctx.taps
        N, C, P = y.shape[:3]
        c = y.reshape(N, C * P, y.shape[3], y.shape[4])
        L = _ffi.lib()
        ctx.natural = []   # each level's uncropped output size, in the order the levels run
        for sh in sizes[::-1]:
            ctx.natural.append((L.b200w_dwt_rec_len(c.shape[-2], g0_col.n, mode),
                                L.b200w_dwt_rec_len(c.shape[-1], g0_row.n, mode)))
            c = wpt_sfb2d_level(c, g0_col, g1_col, g0_row, g1_row, mode, out_hw=sh)
        return c

    @staticmethod
    def backward(ctx, dx):
        dy = None
        if ctx.needs_input_grad[0]:
            g0_row, g1_row, g0_col, g1_col = ctx.taps
            N, C = dx.shape[:2]
            g = dx
            for h, w in ctx.natural[::-1]:
                # a cropped level: its gradient is zero outside the crop, as SFB2D's output sliced to the crop
                if g.shape[-2:] != (h, w):
                    g = F.pad(g, (0, w - g.shape[-1], 0, h - g.shape[-2]))
                g = wpt_afb2d_level(g, g0_row, g1_row, g0_col, g1_col, ctx.mode)
            J = len(ctx.natural)
            dy = g.reshape(N, C, 4 ** J, g.shape[-2], g.shape[-1])
        return dy, None, None, None, None, None, None


class WPT2DForward(nn.Module):
    """2-D wavelet packet decomposition.  Same constructor, buffers and ``state_dict`` keys as :class:`DWTForward`.

    ``forward(x)`` with x (N, C, H, W) float32 or float64 on a CUDA device returns ONE tensor (N, C, 4^J, H_J, W_J),
    H_j = ``b200w_dwt_coeff_len(H_{j-1}, L, mode)``.  Node order is natural: node n = sum_j b_j 4^(J-j), b_j the band
    (0 ll, 1 lh, 2 hl, 3 hh) taken at level j, so node 0 is ``DWTForward(J)``'s ``yl`` bit for bit, and with J = 1 the
    output is ``torch.cat([yl[:, :, None], yh[0]], 2)``.  J = 0 returns ``x[:, :, None]``.

    The gradient follows the DWT's convention (synthesis with the analysis taps); it is the exact gradient only in
    zero mode and in periodization with even sizes at every level.
    """

    def __init__(self, J=1, wave='db1', mode='zero'):
        super().__init__()
        h0_col, h1_col, h0_row, h1_row = _resolve_wave(wave, analysis=True)
        filts = lowlevel.prep_filt_afb2d(h0_col, h1_col, h0_row, h1_row)
        self.register_buffer('h0_col', filts[0])
        self.register_buffer('h1_col', filts[1])
        self.register_buffer('h0_row', filts[2])
        self.register_buffer('h1_row', filts[3])
        self.J = J
        self.mode = mode

    def forward(self, x):
        mode = lowlevel.mode_to_int(self.mode)
        lowlevel._check_bank_mode(mode)
        _ffi.require_cuda_real(x, 'x')
        if x.dim() != 4:
            raise ValueError('expected a 4-D (N,C,H,W) input, got shape {}'.format(tuple(x.shape)))
        if self.J < 1:
            return x[:, :, None]
        # the *_col buffers filter along W and the *_row buffers along H, as in DWTForward
        return WPT2DAnalysis.apply(x, self.h0_col, self.h1_col, self.h0_row, self.h1_row, mode, self.J)


class WPT2DInverse(nn.Module):
    """2-D wavelet packet reconstruction.  Same constructor, buffers and ``state_dict`` keys as :class:`DWTInverse`.

    ``forward(y, size=None)``: y (N, C, 4^J, Hc, Wc); J is read from the node count (a count that is not a power of 4
    raises ``ValueError``).  Each level rebuilds every group of four children into their parent with one DWT
    synthesis level.  ``size=(H, W)``: the size of the signal to rebuild; each level is cropped to the size the
    forward length rule gives for it, and a ``size`` from which that rule does not lead to (Hc, Wc) raises
    ``ValueError``.  ``size=None`` keeps each level's natural ``rec_len`` size.
    """

    def __init__(self, wave='db1', mode='zero'):
        super().__init__()
        g0_col, g1_col, g0_row, g1_row = _resolve_wave(wave, analysis=False)
        filts = lowlevel.prep_filt_sfb2d(g0_col, g1_col, g0_row, g1_row)
        self.register_buffer('g0_col', filts[0])
        self.register_buffer('g1_col', filts[1])
        self.register_buffer('g0_row', filts[2])
        self.register_buffer('g1_row', filts[3])
        self.mode = mode

    def forward(self, y, size=None):
        mode = lowlevel.mode_to_int(self.mode)
        lowlevel._check_bank_mode(mode)
        if y.dim() != 5:
            raise ValueError('expected a 5-D (N,C,4^J,H,W) input, got shape {}'.format(tuple(y.shape)))
        nodes = y.shape[2]
        J = 0
        while 4 ** J < nodes:
            J += 1
        if nodes < 1 or 4 ** J != nodes:
            raise ValueError('the node count {} is not a power of 4'.format(nodes))
        if J == 0:
            _ffi.require_cuda_real(y, 'y')
            return y[:, :, 0]
        Hc, Wc = y.shape[-2:]
        if size is None:
            sizes = [None] * J
        else:
            # the *_row buffers act along H here (SFB2D's first pass takes the *_col arguments = the *_row buffers)
            chain = packet_sizes(size[0], size[1], J, self.g0_row.numel(), self.g0_col.numel(), mode)
            if chain[-1] != (Hc, Wc):
                raise ValueError('size {} does not lead to {}x{} coefficients in {} levels (it leads to {}x{})'.format(
                    tuple(size), Hc, Wc, J, chain[-1][0], chain[-1][1]))
            sizes = chain[:-1]
        _ffi.require_cuda_real(y, 'y')
        return WPT2DSynthesis.apply(y, self.g0_col, self.g1_col, self.g0_row, self.g1_row, mode, sizes)
