"""GPU: the 2-D wavelet packet levels and modules against the DWT levels and the oracle composition
(tests/oracle_wpt2d.py).

``wpt_afb2d_level`` / ``wpt_sfb2d_level`` are called directly.  The entry points route each level (csrc/wpt2d.cu): the
streaming kernel where it applies (float32, equal filter lengths, aligned analysis input) except synthesis levels of at
most 8 coefficient columns, which take the packed small-plane kernel; otherwise the packed kernel up to 40 output
(analysis) or coefficient (synthesis) columns and the tile kernel above; ``_ffi.generic_kernels()`` selects the tile
kernel.  The sizes below sit below, at and past both thresholds, include odd sizes and planes smaller than the filter;
odd widths give unaligned analysis inputs, and the unequal-length pair never takes the streaming kernel.  Every
(n, c) plane carries its own power of ten (tests/util.py), so a wrong border in a small plane cannot hide behind a large
one.
  * analysis: bit-identical to ``afb2d_level`` on the same planes (rearranged) and to the fp32 oracle, on every route;
  * synthesis: bit-identical to ``sfb2d_level`` when both take the same kernel, the packed kernel bit-identical to the
    tile kernel, every plane within bound_sfb2d of the float64 oracle;
  * canaries, a child-process profiler trace of the route of each level, the modules, float64, gradients.
"""
import json
import os
import subprocess
import sys
import zlib

import numpy as np
import pytest
import torch

import pytorch_wavelets_b200 as pw
from pytorch_wavelets_b200 import _ffi, wavelets
from pytorch_wavelets_b200.dwt import lowlevel, packet2d as pk
from oracle import oracle as orc
from tests import oracle_wpt2d as ow
from tests import sweep_util, util

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = 'cuda'
MODES = ['zero', 'symmetric', 'reflect', 'periodic', 'periodization']
MI = {'zero': 0, 'symmetric': 1, 'periodization': 2, 'reflect': 4, 'periodic': 6}
WAVES = ['haar', 'db2', 'db4', 'db8', 'tuple']
PACKED_FIRST_W = 8   # csrc/wpt2d.cu kWptPackedFirstW
PACKED_MAX_W = 40    # csrc/wpt2d.cu kWptPackedMaxW


def _taps(wave):
    """(analysis fw_lo, fw_hi, fh_lo, fh_hi), (synthesis gh_lo, gh_hi, gw_lo, gw_hi): stored taps.  'tuple': db2 along W,
    db4 along H (unequal lengths)."""
    if wave == 'tuple':
        a, b = wavelets.Wavelet('db2'), wavelets.Wavelet('db4')
    else:
        a = b = wavelets.Wavelet(wave)
    an = tuple(np.array(f) for f in (a.dec_lo[::-1], a.dec_hi[::-1], b.dec_lo[::-1], b.dec_hi[::-1]))
    sy = tuple(np.array(f) for f in (b.rec_lo, b.rec_hi, a.rec_lo, a.rec_hi))
    return an, sy


def _in_for(wo, L, mode):
    """an input length whose analysis output has wo samples"""
    return 2 * wo if mode == 'periodization' else 2 * wo - L + 1


def _afb_sizes(wave, mode):
    an, _ = _taps(wave)
    Lw, Lh = len(an[0]), len(an[2])
    w = lambda wo: max(1, _in_for(wo, Lw, mode))   # noqa: E731
    h = lambda ho: max(1, _in_for(ho, Lh, mode))   # noqa: E731
    return {
        'small': (h(9), w(13)),
        'below': (h(21), w(PACKED_MAX_W - 1)),
        'at': (h(33), w(PACKED_MAX_W)),
        'past': (h(17), w(PACKED_MAX_W + 1)),
        'wide': (h(20), w(150)),
        'odd': (37, 91),
        'tiny': (3, 5),            # smaller than the filter
    }


def _x(shape, seed, dtype=torch.float32):
    rng = np.random.default_rng(seed)
    x, sc = util.scaled_uniform(shape, rng, -4, 4)
    return torch.from_numpy(x).to(DEV, dtype), sc


def _np(t):
    return t.detach().cpu().numpy()


def _stack_dwt(ll, highs):
    B, P, Ho, Wo = ll.shape
    return torch.cat([ll[:, :, None], highs], 2).reshape(B, 4 * P, Ho, Wo)


# ---- analysis ----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('generic', [False, True])
@pytest.mark.parametrize('size', ['small', 'below', 'at', 'past', 'wide', 'odd', 'tiny'])
@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('wave', WAVES)
def test_afb_level_matches_dwt_level_and_oracle(wave, mode, size, generic):
    an, _ = _taps(wave)
    H, W = _afb_sizes(wave, mode)[size]
    x, _ = _x((2, 3, H, W), zlib.crc32(('%s %s %s' % (wave, mode, size)).encode()) % 1000)

    def run():
        y = pk.wpt_afb2d_level(x, *an, MI[mode])
        ll, hi = lowlevel.afb2d_level(x, *an, MI[mode])
        return y, _stack_dwt(ll, hi)
    if generic:
        with _ffi.generic_kernels():
            y, d = run()
    else:
        y, d = run()
    assert torch.equal(y, d)
    oll, ohi = orc.dwt_afb2d(_np(x), *an, mode)
    assert np.array_equal(_np(y), _np(_stack_dwt(torch.from_numpy(oll), torch.from_numpy(ohi))))


@pytest.mark.parametrize('layout', ['channel_slice', 'strided', 'single_plane', 'many_planes'])
@pytest.mark.parametrize('wave,mode', [('db4', 'symmetric'), ('haar', 'periodization'), ('tuple', 'reflect')])
def test_afb_level_input_layouts(layout, wave, mode):
    an, _ = _taps(wave)
    if layout == 'channel_slice':
        x = _x((2, 7, 30, 44), 1)[0][:, 2:5]
    elif layout == 'strided':
        x = _x((2, 3, 30, 88), 2)[0][..., ::2]
    elif layout == 'single_plane':
        x = _x((1, 1, 70, 130), 3)[0]
    else:
        x = _x((5, 400, 12, 20), 4)[0]
    y = pk.wpt_afb2d_level(x, *an, MI[mode])
    ll, hi = lowlevel.afb2d_level(x.contiguous(), *an, MI[mode])
    assert torch.equal(y, _stack_dwt(ll, hi))


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('wave', ['haar', 'db4', 'tuple'])
def test_pitched_hand_off_between_levels(wave, mode):
    """pad=True rounds the row pitch of an intermediate level up to 32: odd sizes (e.g. 259, 133, 70 for db4
    symmetric on 512) then still reach the next level with aligned rows; the values are those of the dense hand-off."""
    an, _ = _taps(wave)
    x, _ = _x((1, 2, 259, 133), 5)
    a = pk.wpt_afb2d_level(x, *an, MI[mode], pad=True)
    assert a.stride(2) % 32 == 0 or a.shape[-1] % 32 == 0
    b = pk.wpt_afb2d_level(x, *an, MI[mode])
    assert torch.equal(a, b)
    assert torch.equal(pk.wpt_afb2d_level(a, *an, MI[mode]), pk.wpt_afb2d_level(b, *an, MI[mode]))


# ---- synthesis ---------------------------------------------------------------------------------------------------------

def _sfb_sizes():
    return {'narrow': (13, PACKED_FIRST_W), 'small': (7, PACKED_FIRST_W + 1), 'below': (12, PACKED_MAX_W - 1),
            'at': (21, PACKED_MAX_W), 'past': (9, PACKED_MAX_W + 1), 'wide': (10, 133), 'tiny': (1, 2)}


@pytest.mark.parametrize('crop', [False, True])
@pytest.mark.parametrize('size', ['narrow', 'small', 'below', 'at', 'past', 'wide', 'tiny'])
@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('wave', WAVES)
def test_sfb_level_routes_and_bound(wave, mode, size, crop):
    _, sy = _taps(wave)
    Hc, Wc = _sfb_sizes()[size]
    Lh, Lw = len(sy[0]), len(sy[2])
    Ho, Wo = orc.rec_len(Hc, Lh, mode), orc.rec_len(Wc, Lw, mode)
    if Ho < 1 or Wo < 1:
        pytest.skip('coefficients too small for this filter')
    out_hw = (max(1, Ho - 1), max(1, Wo - 3)) if crop else None
    c, _ = _x((2, 12, Hc, Wc), zlib.crc32(('%s %s %s' % (wave, mode, size)).encode()) % 1000)
    y = pk.wpt_sfb2d_level(c, *sy, MI[mode], out_hw=out_hw)
    with _ffi.generic_kernels():
        yg = pk.wpt_sfb2d_level(c, *sy, MI[mode], out_hw=out_hw)
        q = c.reshape(2, 3, 4, Hc, Wc)
        dg = lowlevel.sfb2d_level(q[:, :, 0], q[:, :, 1:], *sy, MI[mode], out_hw=out_hw)
    assert torch.equal(yg, dg)                           # tile kernel, both layouts
    route = _sfb_route(Wc, Ho if out_hw is None else out_hw[0], Wo if out_hw is None else out_hw[1], Lh, Lw, mode,
                       torch.float32)
    if route == 'wpt_sfb2d_packed':
        assert torch.equal(y, yg)                        # packed kernel == tile kernel
    else:
        d = lowlevel.sfb2d_level(q[:, :, 0], q[:, :, 1:], *sy, MI[mode], out_hw=out_hw)
        assert torch.equal(y, d)                         # the DWT level on the same kernel
    c64 = _np(c).astype(np.float64).reshape(2, 3, 4, Hc, Wc)
    o64 = orc.dwt_sfb2d(c64[:, :, 0], c64[:, :, 1:], *sy, mode, out_hw=out_hw)
    s = util.plane_max(c64.reshape(2, 3, -1))
    G, K = util.bound_sfb2d(*sy)
    util.assert_plane_bound(_np(y), o64, s, G, K, what='wpt sfb %s %s %s' % (wave, mode, size))


# ---- every element written, nothing outside ---------------------------------------------------------------------------

@pytest.mark.parametrize('route', ['packed', 'stream', 'tile'])
@pytest.mark.parametrize('mode', ['symmetric', 'periodization'])
def test_outputs_are_all_written_and_nothing_else(route, mode):
    an, sy = _taps('db4')
    H, W = {'packed': (9, 9), 'stream': (45, 172), 'tile': (45, 172)}[route]
    x, _ = _x((2, 3, H, W), 9)
    lib = _ffi.lib()
    m = MI[mode]
    Ho, Wo = orc.coeff_len(H, 8, mode), orc.coeff_len(W, 8, mode)
    y = sweep_util.Canaried((6 * 4, Ho, Wo))
    t = [_ffi.host_taps(f) for f in an]
    fn = lib.b200w_wpt_afb2d_generic if route == 'tile' else lib.b200w_wpt_afb2d
    assert fn(x.data_ptr(), H * W, W, y.ptr(), Ho * Wo, Wo, 6, H, W, t[0].ptr, t[1].ptr, 8, t[2].ptr, t[3].ptr, 8, m,
              _ffi.stream_of(x)) == 0
    torch.cuda.synchronize()
    y.check('wpt afb ' + route)
    s = [_ffi.host_taps(f) for f in sy]
    Hr, Wr = orc.rec_len(Ho, 8, mode) - 1, orc.rec_len(Wo, 8, mode) - 1
    z = sweep_util.Canaried((6, Hr, Wr))
    fn = lib.b200w_wpt_sfb2d_generic if route == 'tile' else lib.b200w_wpt_sfb2d
    assert fn(y.ptr(), z.ptr(), Hr * Wr, Wr, 6, Ho, Wo, Hr, Wr, s[0].ptr, s[1].ptr, 8, s[2].ptr, s[3].ptr, 8, m,
              _ffi.stream_of(x)) == 0
    torch.cuda.synchronize()
    z.check('wpt sfb ' + route)


# ---- which kernels run ------------------------------------------------------------------------------------------------

def _short(name):
    for k in ('wpt_afb2d_packed', 'wpt_sfb2d_packed', 'wpt_afb2d_stream', 'wpt_sfb2d_stream4', 'wpt_sfb2d_stream',
              'k_wpt_afb2d_tile', 'k_wpt_sfb2d_tile'):
        if k in name:
            return k
    return None


def _fits(floats, dt):
    return floats * (4 if dt == torch.float32 else 8) <= 64 * 1024   # csrc/wpt2d.cu kWptPlaneMaxBytes


def _afb_floats(Ho, Wo, L):
    IW, IH = 2 * Wo + L - 2, 2 * Ho + L - 2
    return IH * (IW | 1) + 2 * IH * Wo


def _sfb_floats(Ho, Wo, Lh, Lw, mode):
    def span(n, L):
        off = L // 2 - 1 if mode == 'periodization' else L - 2
        k0 = (off - L + 2) // 2
        return (n - 1 + off) // 2 - k0 + 1
    return 4 * span(Ho, Lh) * span(Wo, Lw) + 2 * Ho * span(Wo, Lw)


def _sfb_route(wc, ho, wo, Lh, Lw, mode, dt):
    """The kernel csrc/wpt2d.cu picks for a synthesis level of wc coefficient columns and an ho x wo output."""
    fits = _fits(_sfb_floats(ho, wo, Lh, Lw, mode), dt)
    if wc <= PACKED_FIRST_W and fits:
        return 'wpt_sfb2d_packed'
    if dt == torch.float32 and Lh == Lw <= 20:
        wide = Lw <= 8 and mode != 'periodization' and (wo + 1) // 2 > 64
        return 'wpt_sfb2d_stream4' if wide else 'wpt_sfb2d_stream'
    return 'wpt_sfb2d_packed' if wc <= PACKED_MAX_W and fits else 'k_wpt_sfb2d_tile'


def predicted_routes(H, W, J, L, mode, dt):
    """The kernel csrc/wpt2d.cu picks for each level of a J-level forward of contiguous (H, W) planes (Lw == Lh == L),
    then for each level of the inverse back to (H, W)."""
    sizes = ow.forward_sizes(H, W, J, L, L, mode)
    f32 = dt == torch.float32
    out = []
    for j in range(1, J + 1):
        (h, w), (ho, wo) = sizes[j - 1], sizes[j]
        aligned = j > 1 or (w % 4 == 0 and h * w % 4 == 0)
        if f32 and L <= 20 and aligned:
            out.append('wpt_afb2d_stream')
        elif wo <= PACKED_MAX_W and _fits(_afb_floats(ho, wo, L), dt):
            out.append('wpt_afb2d_packed')
        else:
            out.append('k_wpt_afb2d_tile')
    for j in range(J, 0, -1):
        (hc, wc), (ho, wo) = sizes[j], sizes[j - 1]
        out.append(_sfb_route(wc, ho, wo, L, L, mode, dt))
    return out


def trace_in_this_process(dtype_name, wave, mode, n):
    """(kernels traced, kernels predicted) for a J = 3 forward and inverse of 2 x 3 x n x n planes."""
    dt = getattr(torch, dtype_name)
    n = int(n)
    x = torch.randn(2, 3, n, n, device=DEV, dtype=dt)
    f = pw.WPT2DForward(J=3, wave=wave, mode=mode).to(DEV, dt)
    i = pw.WPT2DInverse(wave=wave, mode=mode).to(DEV, dt)
    y = f(x)
    want = predicted_routes(n, n, 3, len(wavelets.Wavelet(wave).dec_lo), mode, dt)

    def run():
        f(x)
        i(y, size=(n, n))
    return sweep_util.traced_kernels(run, _short), want


@pytest.mark.parametrize('dtype,wave,mode,n', [('float32', 'db4', 'symmetric', 152), ('float32', 'haar', 'periodization', 60),
                                               ('float32', 'db2', 'reflect', 61), ('float64', 'db2', 'zero', 152)])
def test_trace_shows_the_predicted_route_of_each_level(dtype, wave, mode, n):
    """The profiler session runs in a child process, so it leaves the CUDA activity tracing of this test process as the
    other trace tests expect it."""
    code = ('import json, sys; from tests import test_gpu_wpt2d as t; '
            'print(json.dumps(t.trace_in_this_process(*sys.argv[1:])))')
    r = subprocess.run([sys.executable, '-c', code, dtype, wave, mode, str(n)], cwd=ROOT, capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    ks, want = json.loads(r.stdout.strip().splitlines()[-1])
    if ks is None:
        pytest.skip('no CUDA activity trace on this machine')
    assert ks == want
    assert len(set(want)) >= 2    # the case covers several routes


# ---- modules ----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('wave', ['haar', 'db2', 'db4', 'tuple'])
def test_modules_match_dwt_and_reconstruct(wave, mode):
    if wave == 'tuple':
        a, b = wavelets.Wavelet('db2'), wavelets.Wavelet('db4')
        fw, iw = (a.dec_lo, a.dec_hi, b.dec_lo, b.dec_hi), (a.rec_lo, a.rec_hi, b.rec_lo, b.rec_hi)
    else:
        fw = iw = wave
    x, _ = _x((2, 3, 67, 90), 11)
    for J in range(5):
        f = pw.WPT2DForward(J=J, wave=fw, mode=mode).to(DEV)
        y = f(x)
        if J == 0:
            assert torch.equal(y, x[:, :, None])
            continue
        yl, yh = pw.DWTForward(J=J, wave=fw, mode=mode).to(DEV)(x)
        assert y.shape[:3] == (2, 3, 4 ** J)
        assert torch.equal(y[:, :, 0], yl)
        if J == 1:
            assert torch.equal(y, torch.cat([yl[:, :, None], yh[0]], 2))
        if J <= 2:
            filts = [_np(getattr(f, k)).ravel() for k in ('h0_col', 'h1_col', 'h0_row', 'h1_row')]
            assert np.array_equal(_np(y), ow.wpt2d_forward(_np(x), filts, J, mode))
        i = pw.WPT2DInverse(wave=iw, mode=mode).to(DEV)
        xr = i(y, size=(67, 90))
        assert xr.shape == x.shape
        err = (xr - x).abs().amax(dim=(2, 3)) / x.abs().amax(dim=(2, 3))
        assert err.max().item() < 1e-5, (J, err.max().item())
        xn = i(y)
        if mode != 'periodization':
            assert xn.shape[-2] >= 67 and xn.shape[-1] >= 90


def _f64_modules(wave, mode):
    """forward and inverse modules whose filters are built in float64 (as under torch's float64 default dtype)"""
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        return pw.WPT2DForward(J=3, wave=wave, mode=mode).to(DEV), pw.WPT2DInverse(wave=wave, mode=mode).to(DEV)
    finally:
        torch.set_default_dtype(prev)


@pytest.mark.parametrize('mode', MODES)
def test_float64_matches_oracle_and_reconstructs(mode):
    x = torch.from_numpy(np.random.default_rng(12).standard_normal((1, 2, 45, 52))).to(DEV)
    f, i = _f64_modules('db3', mode)
    assert f.h0_col.dtype == torch.float64
    y = f(x)
    filts = [_np(getattr(f, k)).ravel() for k in ('h0_col', 'h1_col', 'h0_row', 'h1_row')]
    o = ow.wpt2d_forward(_np(x), filts, 3, mode)
    assert np.abs(_np(y) - o).max() <= 1e-12 * np.abs(o).max()
    xr = i(y, size=(45, 52))
    assert (xr - x).abs().max().item() < 1e-10 * x.abs().max().item()


def test_inverse_node_count_and_size_errors():
    i = pw.WPT2DInverse(wave='db2', mode='symmetric').to(DEV)
    with pytest.raises(ValueError):
        i(torch.randn(1, 1, 8, 6, 6, device=DEV))
    with pytest.raises(ValueError):
        i(torch.randn(1, 1, 16, 6, 6, device=DEV), size=(12, 16))
    y = torch.randn(1, 1, 1, 6, 6, device=DEV)
    assert torch.equal(i(y), y[:, :, 0])


# ---- gradients ----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('mode,shape', [('zero', (1, 2, 11, 9)), ('periodization', (1, 1, 16, 8))])
@pytest.mark.parametrize('wave', ['haar', 'db2'])
def test_gradcheck_float64(wave, mode, shape):
    f = pw.WPT2DForward(J=2, wave=wave, mode=mode).to(DEV, torch.float64)
    i = pw.WPT2DInverse(wave=wave, mode=mode).to(DEV, torch.float64)
    x = torch.randn(*shape, device=DEV, dtype=torch.float64, requires_grad=True)
    assert torch.autograd.gradcheck(f, (x,))
    y = f(x).detach().requires_grad_(True)
    assert torch.autograd.gradcheck(lambda t: i(t, size=shape[-2:]), (y,))


def _level_composition_forward(x, f, J):
    """The packet forward as autograd-traced AFB2D levels and torch.cat (the hand-built composition)."""
    mode = lowlevel.mode_to_int(f.mode)
    N, C = x.shape[:2]
    y = x
    for _ in range(J):
        B, P, H, W = y.shape
        ll, hi = lowlevel.AFB2D.apply(y, f.h0_col, f.h1_col, f.h0_row, f.h1_row, mode)
        y = torch.cat([ll[:, :, None], hi], 2).reshape(B, 4 * P, ll.shape[-2], ll.shape[-1])
    return y.reshape(N, C, 4 ** J, y.shape[-2], y.shape[-1])


@pytest.mark.parametrize('mode', MODES)
def test_backward_equals_the_level_composition(mode):
    f = pw.WPT2DForward(J=3, wave='db2', mode=mode).to(DEV, torch.float64)
    i = pw.WPT2DInverse(wave='db2', mode=mode).to(DEV, torch.float64)
    x = torch.randn(2, 2, 29, 34, device=DEV, dtype=torch.float64, requires_grad=True)
    y = f(x)
    g = torch.randn_like(y)
    (gx,) = torch.autograd.grad(y, x, g)
    (gc,) = torch.autograd.grad(_level_composition_forward(x, f, 3), x, g)
    assert torch.allclose(gx, gc, rtol=0, atol=1e-12 * gc.abs().max().item())
    # synthesis: the level-by-level SFB2D composition, cropped as the inverse crops
    yd = y.detach().requires_grad_(True)
    xr = i(yd, size=(29, 34))
    h = torch.randn_like(xr)
    (gy,) = torch.autograd.grad(xr, yd, h)
    sizes = pk.packet_sizes(29, 34, 3, 4, 4, lowlevel.mode_to_int(mode))
    c = yd.reshape(2, 2 * 64, yd.shape[-2], yd.shape[-1])
    for sh in sizes[-2::-1]:
        B, P4, Hc, Wc = c.shape
        q = c.reshape(B, P4 // 4, 4, Hc, Wc)
        c = lowlevel.SFB2D.apply(q[:, :, 0], q[:, :, 1:], i.g0_col, i.g1_col, i.g0_row, i.g1_row,
                                 lowlevel.mode_to_int(mode))[..., :sh[0], :sh[1]]
    (gz,) = torch.autograd.grad(c, yd, h)
    assert torch.allclose(gy, gz, rtol=0, atol=1e-12 * gz.abs().max().item())
