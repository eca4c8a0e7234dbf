"""Single-level DTCWT autograd Functions on the H100 engine.

Drop-in for the reference's Function layer (``pytorch_wavelets/dtcwt/transform_funcs.py``):
``FWD_J1`` :343-374, ``FWD_J2PLUS`` :377-413, ``INV_J1`` :416-449, ``INV_J2PLUS`` :452-488 and the
dimension helpers ``get_dimensions5/6`` :10-58 -- same ``apply`` signatures, same return structure
(0-dim tensors for skipped band-passes), same backward definitions (each backward is the opposite
direction's kernel with the same stored filters, a/b trees swapped for the q-shift levels).
Each forward is one fused CUDA kernel (row + column filters, decimation / interpolation, symmetric
extension and the q2c / c2q packing) behind the C ABI.
"""
import torch
from torch.autograd import Function

from pytorch_wavelets_b200 import _ffi
from pytorch_wavelets_b200.dwt.lowlevel import int_to_mode


def get_dimensions5(o_dim, ri_dim):
    """Orientation / height / width dims once the real-imag dim is popped (reference :10-29)."""
    o_dim = (o_dim % 6)
    ri_dim = (ri_dim % 6)
    if ri_dim < o_dim:
        o_dim -= 1
    if o_dim == 4:
        h_dim, w_dim = 2, 3
    elif o_dim == 3:
        h_dim, w_dim = 2, 4
    else:
        h_dim, w_dim = 3, 4
    return o_dim, ri_dim, h_dim, w_dim


def get_dimensions6(o_dim, ri_dim):
    """Orientation, real/imag, height and width dims of the full 6-D tensor (reference :32-58)."""
    o_dim = (o_dim % 6)
    ri_dim = (ri_dim % 6)
    if ri_dim < o_dim:
        o_dim -= 1
    if o_dim >= 3 and ri_dim >= 3:
        h_dim = 2
    elif o_dim >= 4 or ri_dim >= 4:
        h_dim = 3
    else:
        h_dim = 4
    if o_dim >= 4 and ri_dim >= 4:
        w_dim = 3
    elif o_dim >= 4 or ri_dim >= 4:
        w_dim = 4
    else:
        w_dim = 5
    return o_dim, ri_dim, h_dim, w_dim


def _layout(o5, ri):
    """Dim names of the 6-D band-pass tensor: the 4-D bands are stacked at o5 (5-D index, i.e. after
    get_dimensions5), then real/imag at ri (reference highs_to_orientations :61-72 + stack :355)."""
    d = ['n', 'c', 'h', 'w']
    d.insert(o5, 'o')
    d.insert(ri, 'r')
    return d


def highs_shape_strides(N, C, h, w, o5, ri):
    names = _layout(o5, ri)
    size = {'n': N, 'c': C, 'o': 6, 'h': h, 'w': w, 'r': 2}
    shape = tuple(size[k] for k in names)
    strides, acc = {}, 1
    for k in reversed(names):
        strides[k] = acc
        acc *= size[k]
    return shape, [strides[k] for k in ('n', 'c', 'o', 'h', 'w', 'r')]


def _highs_dims(highs, o5, ri):
    names = _layout(o5, ri)
    if highs.dim() != 6:
        raise ValueError('band-pass tensor must have 6 dimensions, got shape {}'.format(tuple(highs.shape)))
    sz = dict(zip(names, highs.shape))
    if sz['o'] != 6 or sz['r'] != 2:
        raise ValueError('band-pass tensor of shape {} does not have 6 orientations / 2 real-imag entries at '
                         'o_dim / ri_dim'.format(tuple(highs.shape)))
    return sz


def _is_empty(t):
    return t is None or t.shape == torch.Size([])


# ---- raw kernel calls -------------------------------------------------------------------------------------

def fwd_j1(x, h0, h1, skip_hps, o5, ri, mode):
    """ll, highs (None when skipped) for one level-1 transform; o5/ri as returned by get_dimensions5."""
    dt = _ffi.require_cuda_real(x, 'x')
    L = _ffi.lib()
    h0, h1 = _ffi.host_taps(h0), _ffi.host_taps(h1)
    N, C, H, W = x.shape
    if H % 2 or W % 2:
        raise ValueError('level-1 DTCWT input must have even height and width, got {}'.format(tuple(x.shape)))
    x, xps, xpitch = _ffi.planes_view(x)
    ll = x.new_empty((N, C, H, W))
    highs, hs = None, [0] * 6
    if not skip_hps:
        shape, hs = highs_shape_strides(N, C, H // 2, W // 2, o5, ri)
        highs = x.new_empty(shape)
    if N * C > 0:
        with torch.cuda.device(x.device), _ffi.span('dtcwt_fwd_j1 %dx%d' % (H, W),
                                                    4 * N * C * H * W * (2 if skip_hps else 5)):
            rc = _ffi.entry('b200w_dtcwt_fwd_j1', dt)(x.data_ptr(), xps, xpitch, ll.data_ptr(), H * W, W,
                                      None if highs is None else highs.data_ptr(), _ffi.hs_array(hs),
                                      N, C, H, W, h0.p(dt), h0.n, h1.p(dt), h1.n, mode, _ffi.stream_of(x))
        _ffi.check(rc, 'b200w_dtcwt_fwd_j1')
    return ll, highs


def fwd_j2plus(x, h0a, h1a, h0b, h1b, skip_hps, o5, ri):
    dt = _ffi.require_cuda_real(x, 'x')
    L = _ffi.lib()
    N, C, H, W = x.shape
    if H % 4 != 0:
        raise ValueError('No. of rows in X must be a multiple of 4\nX was {}'.format(x.shape))
    if W % 4 != 0:
        raise ValueError('No. of cols in X must be a multiple of 4\nX was {}'.format(x.shape))
    f = [_ffi.host_taps(t) for t in (h0a, h1a, h0b, h1b)]
    x, xps, xpitch = _ffi.planes_view(x)
    ll = x.new_empty((N, C, H // 2, W // 2))
    highs, hs = None, [0] * 6
    if not skip_hps:
        shape, hs = highs_shape_strides(N, C, H // 4, W // 4, o5, ri)
        highs = x.new_empty(shape)
    if N * C > 0:
        with torch.cuda.device(x.device), _ffi.span('dtcwt_fwd_j2plus %dx%d' % (H, W),
                                                    N * C * H * W * (5 if skip_hps else 8)):
            rc = _ffi.entry('b200w_dtcwt_fwd_j2plus', dt)(x.data_ptr(), xps, xpitch, ll.data_ptr(), (H // 2) * (W // 2), W // 2,
                                          None if highs is None else highs.data_ptr(), _ffi.hs_array(hs),
                                          N, C, H, W, f[0].p(dt), f[1].p(dt), f[2].p(dt), f[3].p(dt), f[0].n,
                                          _ffi.stream_of(x))
        _ffi.check(rc, 'b200w_dtcwt_fwd_j2plus')
    return ll, highs


def fwd_j12(x, h0o, h1o, h0a, h1a, h0b, h1b, skip_hps1, o5, ri, mode):
    """Levels 1 and 2 in one call (float32, H % 4 == W % 4 == 0, level-1 band-pass kept): ll2, highs0, highs1 (None
    when skipped), equal bit for bit to fwd_j1 followed by fwd_j2plus on its low-pass."""
    if x.dtype != torch.float32:
        raise NotImplementedError('the fused DTCWT levels 1 + 2 run in float32 only, got %s' % x.dtype)
    _ffi.require_cuda_real(x, 'x')
    L = _ffi.lib()
    f = [_ffi.host_taps(t) for t in (h0o, h1o, h0a, h1a, h0b, h1b)]
    N, C, H, W = x.shape
    if H % 4 or W % 4:
        raise ValueError('the fused DTCWT levels 1 + 2 need a height and width divisible by 4, got {}'.format(tuple(x.shape)))
    x, xps, xpitch = _ffi.planes_view(x)
    ll = x.new_empty((N, C, H // 2, W // 2))
    shape0, hs0 = highs_shape_strides(N, C, H // 2, W // 2, o5, ri)
    highs0 = x.new_empty(shape0)
    highs1, hs1 = None, [0] * 6
    if not skip_hps1:
        shape1, hs1 = highs_shape_strides(N, C, H // 4, W // 4, o5, ri)
        highs1 = x.new_empty(shape1)
    if N * C > 0:
        if _ffi._USE_GENERIC:
            ws_bytes = 4 * N * C * H * W
        else:
            ws_bytes = L.b200w_dtcwt_fwd_j12_workspace(x.data_ptr(), xps, xpitch, highs0.data_ptr(), N, C, H, W,
                                                       f[0].n, f[1].n, f[2].n)
            _ffi.check(ws_bytes if ws_bytes < 0 else 0, 'b200w_dtcwt_fwd_j12_workspace')
        ws = x.new_empty((ws_bytes // 4,)) if ws_bytes > 0 else None
        with torch.cuda.device(x.device), _ffi.span('dtcwt_fwd_j12 %dx%d' % (H, W),
                                                    N * C * H * W * (17 if skip_hps1 else 20)):
            rc = _ffi.entry('b200w_dtcwt_fwd_j12')(
                x.data_ptr(), xps, xpitch, ll.data_ptr(), (H // 2) * (W // 2), W // 2,
                highs0.data_ptr(), _ffi.hs_array(hs0), None if highs1 is None else highs1.data_ptr(), _ffi.hs_array(hs1),
                N, C, H, W, f[0].p(torch.float32), f[0].n, f[1].p(torch.float32), f[1].n,
                f[2].p(torch.float32), f[3].p(torch.float32), f[4].p(torch.float32), f[5].p(torch.float32), f[2].n,
                mode, None if ws is None else ws.data_ptr(), ws_bytes, _ffi.stream_of(x))
        _ffi.check(rc, 'b200w_dtcwt_fwd_j12')
    return ll, highs0, highs1


def _inv_prepare(ll, highs, o5, ri, what):
    if _is_empty(ll):
        ll = None
    if _is_empty(highs):
        highs = None
    if ll is None and highs is None:
        raise ValueError('%s needs a low-pass or a band-pass input' % what)
    sz = None
    dt = None
    if highs is not None:
        dt = _ffi.require_cuda_real(highs, 'highs')
        highs = highs.contiguous()
        sz = _highs_dims(highs, o5, ri)
    if ll is not None:
        dt = _ffi.require_cuda_real(ll, 'lows', dt)
    return ll, highs, sz, dt


def inv_j1(ll, highs, g0, g1, o5, ri, mode):
    """Level-1 synthesis.  ``ll`` (N,C,H,W) or None, ``highs`` 6-D or None."""
    L = _ffi.lib()
    ll, highs, sz, dt = _inv_prepare(ll, highs, o5, ri, 'inv_j1')
    g0, g1 = _ffi.host_taps(g0), _ffi.host_taps(g1)
    hs = [0] * 6
    if highs is not None:
        if ll is not None:
            # "possibly cut back some rows to make the ll match the highs" (reference :170-176) -- a view
            if ll.shape[2] != 2 * sz['h']:
                ll = ll[:, :, 1:-1]
            if ll.shape[3] != 2 * sz['w']:
                ll = ll[:, :, :, 1:-1]
            if ll.shape[2] != 2 * sz['h'] or ll.shape[3] != 2 * sz['w']:
                raise ValueError('low-pass {} does not match band-pass {}'.format(tuple(ll.shape), tuple(highs.shape)))
            N, C, H, W = ll.shape
            if sz['n'] != N or sz['c'] != C:   # the kernel strides the band-pass with ll's N, C
                raise ValueError('low-pass {} does not match band-pass {}'.format(tuple(ll.shape), tuple(highs.shape)))
        else:
            N, C, H, W = sz['n'], sz['c'], 2 * sz['h'], 2 * sz['w']
        _, hs = highs_shape_strides(N, C, H // 2, W // 2, o5, ri)
    else:
        N, C, H, W = ll.shape
        # reference quirk: the low-pass-only path calls rowfilter(colfilter(ll, g0), g0) without `mode`,
        # i.e. always with the default symmetric extension (transform_funcs.py:158-159)
        mode = 1
    if H % 2 or W % 2:
        raise ValueError('level-1 DTCWT low-pass must have even height and width')
    ref = ll if ll is not None else highs
    llps = llpitch = 0
    if ll is not None:
        ll, llps, llpitch = _ffi.planes_view(ll)
    y = ref.new_empty((N, C, H, W))
    if N * C > 0:
        with torch.cuda.device(ref.device), _ffi.span('dtcwt_inv_j1 %dx%d' % (H, W),
                                                      4 * N * C * H * W * (1 + (ll is not None) + 3 * (highs is not None))):
            rc = _ffi.entry('b200w_dtcwt_inv_j1', dt)(None if ll is None else ll.data_ptr(), llps, llpitch,
                                      None if highs is None else highs.data_ptr(), _ffi.hs_array(hs),
                                      y.data_ptr(), H * W, W, N, C, H, W, g0.p(dt), g0.n, g1.p(dt), g1.n, mode,
                                      _ffi.stream_of(ref))
        _ffi.check(rc, 'b200w_dtcwt_inv_j1')
    return y


def inv_j2plus(ll, highs, g0a, g1a, g0b, g1b, o5, ri):
    """Level>=2 synthesis: ``ll`` (N,C,H,W) or None, ``highs`` at (H/2,W/2) or None -> (N,C,2H,2W)."""
    L = _ffi.lib()
    ll, highs, sz, dt = _inv_prepare(ll, highs, o5, ri, 'inv_j2plus')
    f = [_ffi.host_taps(t) for t in (g0a, g1a, g0b, g1b)]
    hs = [0] * 6
    if ll is not None:
        N, C, H, W = ll.shape
    else:
        N, C, H, W = sz['n'], sz['c'], 2 * sz['h'], 2 * sz['w']
    if highs is not None:
        if ll is not None and (H != 2 * sz['h'] or W != 2 * sz['w'] or sz['n'] != N or sz['c'] != C):
            raise ValueError('low-pass {} does not match band-pass {}'.format(tuple(ll.shape), tuple(highs.shape)))
        _, hs = highs_shape_strides(N, C, H // 2, W // 2, o5, ri)
    if H % 2 != 0:
        raise ValueError('No. of rows in X must be a multiple of 2.\nX was {}'.format((N, C, H, W)))
    if W % 2 != 0:
        raise ValueError('No. of cols in X must be a multiple of 2.\nX was {}'.format((N, C, H, W)))
    ref = ll if ll is not None else highs
    llps = llpitch = 0
    if ll is not None:
        ll, llps, llpitch = _ffi.planes_view(ll)
    y = ref.new_empty((N, C, 2 * H, 2 * W))
    if N * C > 0:
        with torch.cuda.device(ref.device), _ffi.span('dtcwt_inv_j2plus %dx%d' % (H, W),
                                                      4 * N * C * H * W * (4 + (ll is not None) + 3 * (highs is not None))):
            rc = _ffi.entry('b200w_dtcwt_inv_j2plus', dt)(None if ll is None else ll.data_ptr(), llps, llpitch,
                                          None if highs is None else highs.data_ptr(), _ffi.hs_array(hs),
                                          y.data_ptr(), 4 * H * W, 2 * W, N, C, H, W,
                                          f[0].p(dt), f[1].p(dt), f[2].p(dt), f[3].p(dt), f[0].n, _ffi.stream_of(ref))
        _ffi.check(rc, 'b200w_dtcwt_inv_j2plus')
    return y


# ---- autograd Functions ----------------------------------------------------------------------------------

def _mode_int(mode):
    mode = int(mode)
    int_to_mode(mode)
    return mode


class FWD_J1(Function):
    """Differentiable level-1 forward DTCWT: ``apply(x, h0, h1, skip_hps, o_dim, ri_dim, mode)``."""

    @staticmethod
    def forward(ctx, x, h0, h1, skip_hps, o_dim, ri_dim, mode):
        mode = _mode_int(mode)
        ctx.mode = mode
        ctx.taps = (_ffi.host_taps(h0), _ffi.host_taps(h1))
        ctx.dims = get_dimensions5(o_dim, ri_dim)
        o5, ri = ctx.dims[0], ctx.dims[1]
        ll, highs = fwd_j1(x, ctx.taps[0], ctx.taps[1], bool(skip_hps), o5, ri, mode)
        if highs is None:
            highs = ll.new_zeros([])
        return ll, highs

    @staticmethod
    def backward(ctx, dl, dh):
        h0, h1 = ctx.taps
        dx = None
        if ctx.needs_input_grad[0]:
            o5, ri = ctx.dims[0], ctx.dims[1]
            dx = inv_j1(dl, None if _is_empty(dh) else dh, h0, h1, o5, ri, ctx.mode)
        return dx, None, None, None, None, None, None


class FWD_J2PLUS(Function):
    """Differentiable level>=2 forward DTCWT:
    ``apply(x, h0a, h1a, h0b, h1b, skip_hps, o_dim, ri_dim, mode)`` (mode is ignored: always symmetric)."""

    @staticmethod
    def forward(ctx, x, h0a, h1a, h0b, h1b, skip_hps, o_dim, ri_dim, mode):
        ctx.taps = tuple(_ffi.host_taps(f) for f in (h0a, h1a, h0b, h1b))
        ctx.dims = get_dimensions5(o_dim, ri_dim)
        o5, ri = ctx.dims[0], ctx.dims[1]
        ll, highs = fwd_j2plus(x, *ctx.taps, bool(skip_hps), o5, ri)
        if highs is None:
            highs = ll.new_zeros([])
        return ll, highs

    @staticmethod
    def backward(ctx, dl, dh):
        h0a, h1a, h0b, h1b = ctx.taps
        dx = None
        if ctx.needs_input_grad[0]:
            o5, ri = ctx.dims[0], ctx.dims[1]
            # the interpolating filters correlate, so the trees swap (reference :398-401)
            dx = inv_j2plus(dl, None if _is_empty(dh) else dh, h0b, h1b, h0a, h1a, o5, ri)
        return dx, None, None, None, None, None, None, None, None


class FWD_J12(Function):
    """Differentiable levels 1 and 2 of the forward DTCWT in one call, without the level-1 low-pass:
    ``apply(x, h0o, h1o, h0a, h1a, h0b, h1b, skip_hps1, o_dim, ri_dim, mode)`` -> (ll2, highs0, highs1).
    Forward and backward equal FWD_J1 followed by FWD_J2PLUS bit for bit (the backward runs the same kernels in the
    same order: FWD_J2PLUS's backward, then FWD_J1's)."""

    @staticmethod
    def forward(ctx, x, h0o, h1o, h0a, h1a, h0b, h1b, skip_hps1, o_dim, ri_dim, mode):
        mode = _mode_int(mode)
        ctx.mode = mode
        ctx.taps = tuple(_ffi.host_taps(f) for f in (h0o, h1o, h0a, h1a, h0b, h1b))
        ctx.dims = get_dimensions5(o_dim, ri_dim)
        o5, ri = ctx.dims[0], ctx.dims[1]
        ll, highs0, highs1 = fwd_j12(x, *ctx.taps, bool(skip_hps1), o5, ri, mode)
        if highs1 is None:
            highs1 = ll.new_zeros([])
        return ll, highs0, highs1

    @staticmethod
    def backward(ctx, dl, dh0, dh1):
        h0o, h1o, h0a, h1a, h0b, h1b = ctx.taps
        dx = None
        if ctx.needs_input_grad[0]:
            o5, ri = ctx.dims[0], ctx.dims[1]
            dll1 = inv_j2plus(dl, None if _is_empty(dh1) else dh1, h0b, h1b, h0a, h1a, o5, ri)
            dx = inv_j1(dll1, None if _is_empty(dh0) else dh0, h0o, h1o, o5, ri, ctx.mode)
        return dx, None, None, None, None, None, None, None, None, None, None


class INV_J1(Function):
    """Differentiable level-1 inverse DTCWT: ``apply(lows, highs, g0, g1, o_dim, ri_dim, mode)``."""

    @staticmethod
    def forward(ctx, lows, highs, g0, g1, o_dim, ri_dim, mode):
        mode = _mode_int(mode)
        ctx.mode = mode
        ctx.taps = (_ffi.host_taps(g0), _ffi.host_taps(g1))
        ctx.dims = get_dimensions5(o_dim, ri_dim)
        ctx.has = (not _is_empty(lows), not _is_empty(highs))
        o5, ri = ctx.dims[0], ctx.dims[1]
        return inv_j1(lows, highs, ctx.taps[0], ctx.taps[1], o5, ri, mode)

    @staticmethod
    def backward(ctx, dy):
        g0, g1 = ctx.taps
        o5, ri = ctx.dims[0], ctx.dims[1]
        need_l = ctx.needs_input_grad[0] and ctx.has[0]
        need_h = ctx.needs_input_grad[1] and ctx.has[1]
        dl = dh = None
        if need_l or need_h:
            dl, dh = fwd_j1(dy.contiguous(), g0, g1, not need_h, o5, ri, ctx.mode)
            if not need_l:
                dl = None
        return dl, dh, None, None, None, None, None


class INV_J2PLUS(Function):
    """Differentiable level>=2 inverse DTCWT:
    ``apply(lows, highs, g0a, g1a, g0b, g1b, o_dim, ri_dim, mode)`` (always symmetric)."""

    @staticmethod
    def forward(ctx, lows, highs, g0a, g1a, g0b, g1b, o_dim, ri_dim, mode):
        ctx.taps = tuple(_ffi.host_taps(f) for f in (g0a, g1a, g0b, g1b))
        ctx.dims = get_dimensions5(o_dim, ri_dim)
        ctx.has = (not _is_empty(lows), not _is_empty(highs))
        o5, ri = ctx.dims[0], ctx.dims[1]
        return inv_j2plus(lows, highs, *ctx.taps, o5, ri)

    @staticmethod
    def backward(ctx, dy):
        g0a, g1a, g0b, g1b = ctx.taps
        o5, ri = ctx.dims[0], ctx.dims[1]
        need_l = ctx.needs_input_grad[0] and ctx.has[0]
        need_h = ctx.needs_input_grad[1] and ctx.has[1]
        dl = dh = None
        if need_l or need_h:
            # trees swap (reference :473-474)
            dl, dh = fwd_j2plus(dy.contiguous(), g0b, g1b, g0a, g1a, not need_h, o5, ri)
            if not need_l:
                dl = None
        return dl, dh, None, None, None, None, None, None, None
