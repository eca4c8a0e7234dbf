"""GPU: the 3-D DWT levels and modules against the oracle composition (tests/oracle3d.py).

``afb3d_level`` / ``sfb3d_level`` are called directly, so no policy can reroute a case: the float32 entry points run
the fused kernels for L = 2 ... 8, and ``_ffi.generic_kernels()`` selects the two-step route (2-D level plus a pass
along D).  Every (n, c) volume carries its own power of ten (tests/util.py), so a wrong border in a small volume cannot
hide behind a large one.
  * analysis: yl and all seven bands bit-identical to the fp32 oracle and to the two-step route;
  * synthesis: every volume within bound_sfb3d of the float64 oracle, on both routes;
  * canaries (once per fused instantiation), a profiler trace of the kernels launched, the modules, float64.
"""
import numpy as np
import pytest
import torch

import pytorch_wavelets_b200 as pw
from pytorch_wavelets_b200 import _ffi, wavelets
from pytorch_wavelets_b200.dwt.lowlevel import AFB3D, afb3d_level, mode_to_int, sfb3d_level
from oracle import oracle as orc
from tests import oracle3d as o3
from tests import sweep_util, util

pytestmark = pytest.mark.gpu

MODES = ['zero', 'symmetric', 'reflect', 'periodic', 'periodization']
FUSED = {2: 'haar', 4: 'db2', 6: 'db3', 8: 'db4'}
DEV = 'cuda'


def _filters(name):
    w = wavelets.Wavelet(name)
    return (np.array(w.dec_lo[::-1]), np.array(w.dec_hi[::-1])), (np.array(w.rec_lo), np.array(w.rec_hi))


def _np(t):
    return t.detach().cpu().numpy()


# analysis shapes (N, C, D, H, W), named by the boundary they exercise.  The fused analysis tile is 16 x 32 output
# positions; D chunks come from the march count (few big volumes: many chunks; many small volumes: one chunk).
AFB_SHAPES = {
    'below_one_tile': (1, 2, 5, 20, 30),
    'one_tile_and_past': (2, 1, 7, 33, 66),
    'several_tiles_partial': (1, 1, 6, 70, 140),
    'odd_all': (1, 3, 9, 35, 69),
    'd_below_L': (1, 2, 3, 18, 40),
    'd1': (2, 1, 1, 19, 37),
    'long_d_many_chunks': (1, 2, 75, 34, 66),
    'many_volumes_one_chunk': (4, 150, 12, 10, 12),
}


def _input(shape, seed, layout='contiguous'):
    rng = np.random.default_rng(seed)
    x, sc = util.scaled_uniform(shape, rng)
    if layout == 'contiguous':
        return torch.from_numpy(x).to(DEV), x
    N, C, D, H, W = shape
    if layout == 'channel_slice':      # x[:, 1:2] of a 3-channel tensor: volume stride 3*D*H*W
        big = torch.zeros((N, 3, D, H, W), device=DEV)
        big[:, 1:2] = torch.from_numpy(x).to(DEV)
        return big[:, 1:2], x
    # volume stride larger than D*H*W
    vs = D * H * W + 37
    buf = torch.zeros((N * C * vs,), device=DEV)
    t = buf.as_strided((N, C, D, H, W), (C * vs, vs, H * W, W, 1))
    t.copy_(torch.from_numpy(x).to(DEV))
    return t, x


def _afb_case(L, mode, shape, layout='contiguous'):
    (h0, h1), _ = _filters(FUSED[L])
    m = mode_to_int(mode)
    xt, x = _input(shape, 11 * L + m, layout)
    oyl, oyh = o3.dwt_afb3d(x, h0, h1, mode)
    yl, yh = afb3d_level(xt, h0, h1, m)
    with _ffi.generic_kernels():
        gyl, gyh = afb3d_level(xt, h0, h1, m)
    for what, a, b in (('yl', yl, oyl), ('highs', yh, oyh)):
        assert np.array_equal(_np(a), b), '%s differs from the oracle (L=%d %s %s)' % (what, L, mode, shape)
    assert torch.equal(yl, gyl) and torch.equal(yh, gyh), 'fused and two-step routes differ'


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('L', sorted(FUSED))
@pytest.mark.parametrize('case', sorted(AFB_SHAPES))
def test_afb3d_matches_oracle_and_two_step(case, L, mode):
    _afb_case(L, mode, AFB_SHAPES[case])


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('L', sorted(FUSED))
@pytest.mark.parametrize('layout', ['channel_slice', 'volume_stride'])
def test_afb3d_strided_views(layout, L, mode):
    _afb_case(L, mode, (2, 1, 7, 21, 45), layout)


# synthesis: coefficient shapes (N, C, Dc, Hc, Wc); the fused synthesis tile is 32 x 64 output positions
SFB_SHAPES = {
    'below_one_tile': (1, 2, 4, 10, 20),
    'one_tile_and_past': (2, 1, 5, 17, 33),
    'several_tiles_partial': (1, 1, 4, 40, 75),
    'odd_all': (1, 3, 7, 19, 35),
    'dc_below_L': (1, 2, 3, 12, 22),   # (non-periodization modes need L/2 coefficients: raised to L/2 there)
    'dc1': (2, 1, 1, 9, 17),
    'long_d_many_chunks': (1, 2, 40, 18, 34),
    'many_volumes_one_chunk': (4, 150, 8, 6, 7),
}


def _coeffs(shape, seed, has_hi=True):
    rng = np.random.default_rng(seed)
    yl, sc = util.scaled_uniform(shape, rng)
    hi = util.scaled_uniform(shape[:2] + (7,) + shape[2:], rng, scales=sc)[0] if has_hi else None
    return yl, hi


def _sfb_case(L, mode, shape, has_hi=True, crop=False, wave=None):
    _, (g0, g1) = _filters(wave or FUSED[L])
    m = mode_to_int(mode)
    if mode != 'periodization':
        shape = shape[:2] + tuple(max(n, L // 2) for n in shape[2:])
    yl, hi = _coeffs(shape, 7 * L + m + 100 * has_hi, has_hi)
    out = None
    if crop:
        out = [max(1, orc.rec_len(n, L, mode) - 3) for n in shape[2:]]
    y64 = o3.dwt_sfb3d(yl.astype(np.float64), None if hi is None else hi.astype(np.float64), g0, g1, mode, out)
    s = util.plane_max(yl, None if hi is None else hi.reshape(shape[0], shape[1], -1))
    G, K = o3.bound_sfb3d(g0, g1, has_hi)
    ylt = torch.from_numpy(yl).to(DEV)
    hit = None if hi is None else torch.from_numpy(hi).to(DEV)
    y = sfb3d_level(ylt, hit, g0, g1, m, out_dhw=out)
    with _ffi.generic_kernels():
        gy = sfb3d_level(ylt, hit, g0, g1, m, out_dhw=out)
    for what, a in (('fused', y), ('two-step', gy)):
        util.assert_plane_bound(_np(a), y64, s, G, K, what='%s L=%d %s %s' % (what, L, mode, shape))


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('L', sorted(FUSED))
@pytest.mark.parametrize('case', sorted(SFB_SHAPES))
def test_sfb3d_within_bound_both_routes(case, L, mode):
    _sfb_case(L, mode, SFB_SHAPES[case])


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('L', sorted(FUSED))
@pytest.mark.parametrize('variant', ['no_highs', 'crop', 'no_highs_crop'])
def test_sfb3d_no_highs_and_crop(variant, L, mode):
    _sfb_case(L, mode, (2, 1, 6, 21, 37), has_hi='no_highs' not in variant, crop='crop' in variant)


def test_sfb3d_low_pass_view_with_volume_stride():
    """A low-pass with a volume stride (a channel slice) is read in place and gives the contiguous result."""
    _, (g0, g1) = _filters('db4')
    yl, hi = _coeffs((2, 1, 5, 12, 20), 5)
    big = torch.zeros((2, 3, 5, 12, 20), device=DEV)
    big[:, 2:3] = torch.from_numpy(yl).to(DEV)
    hit = torch.from_numpy(hi).to(DEV)
    a = sfb3d_level(big[:, 2:3], hit, g0, g1, 1)
    b = sfb3d_level(torch.from_numpy(yl).to(DEV), hit, g0, g1, 1)
    assert torch.equal(a, b)


# ---- every element written, nothing outside ---------------------------------------------------------------------------

@pytest.mark.parametrize('L', sorted(FUSED))
def test_fused_kernels_write_every_output_and_nothing_else(L):
    (h0, h1), (g0, g1) = _filters(FUSED[L])
    N, C, D, H, W = 1, 3, 11, 37, 71
    hf0, hf1, sg0, sg1 = [_ffi.host_taps(f) for f in (h0, h1, g0, g1)]
    lib = _ffi.lib()
    x = torch.randn(N, C, D, H, W, device=DEV)
    Do, Ho, Wo = [orc.coeff_len(n, L, 'symmetric') for n in (D, H, W)]
    yl = sweep_util.Canaried((N, C, Do, Ho, Wo))
    hi = sweep_util.Canaried((N, C, 7, Do, Ho, Wo))
    assert lib.b200w_dwt_afb3d_workspace(x.data_ptr(), D * H * W, N * C, D, H, W, L, 1) == 0
    rc = lib.b200w_dwt_afb3d(x.data_ptr(), D * H * W, yl.ptr(), hi.ptr(), N * C, D, H, W, hf0.ptr, hf1.ptr, L, 1,
                             None, 0, _ffi.stream_of(x))
    assert rc == 0
    torch.cuda.synchronize()
    yl.check('afb3d yl')
    hi.check('afb3d highs')
    Dr, Hr, Wr = [orc.rec_len(n, L, 'symmetric') - 1 for n in (Do, Ho, Wo)]   # a crop
    y = sweep_util.Canaried((N, C, Dr, Hr, Wr))
    rc = lib.b200w_dwt_sfb3d(yl.ptr(), Do * Ho * Wo, hi.ptr(), y.ptr(), N * C, Do, Ho, Wo, Dr, Hr, Wr, sg0.ptr, sg1.ptr,
                             L, 1, None, 0, _ffi.stream_of(x))
    assert rc == 0
    torch.cuda.synchronize()
    y.check('sfb3d y')


# ---- which kernels run ------------------------------------------------------------------------------------------------

def _kernels(run):
    def short(name):
        for k in ('afb3d_stream', 'sfb3d_stream', 'afb1d_strided', 'sfb1d_strided', 'afb2d_stream', 'sfb2d_stream',
                  'k_afb2d_tile', 'k_sfb2d_tile'):
            if k in name:
                return k
        return None
    return sweep_util.traced_kernels(run, short)


@pytest.mark.parametrize('wave,generic,dtype', [('haar', False, torch.float32), ('db4', False, torch.float32),
                                                ('db4', True, torch.float32), ('db8', False, torch.float32),
                                                ('db4', False, torch.float64)])
def test_trace_shows_the_predicted_route(wave, generic, dtype):
    (h0, h1), (g0, g1) = _filters(wave)
    L = len(h0)
    x = torch.randn(2, 2, 9, 40, 70, device=DEV, dtype=dtype)
    fused = (not generic) and dtype == torch.float32 and L <= 8

    def run(fn):
        if generic:
            with _ffi.generic_kernels():
                return _kernels(fn)
        return _kernels(fn)
    yl, yh = afb3d_level(x, h0, h1, 1)
    ka = run(lambda: afb3d_level(x, h0, h1, 1))
    ks = run(lambda: sfb3d_level(yl, yh, g0, g1, 1))
    if ka is None:
        pytest.skip('no CUDA activity trace on this machine')
    if fused:
        assert ka == ['afb3d_stream'] and ks == ['sfb3d_stream']
    else:
        assert ka[-1] == 'afb1d_strided' and ka[0] in ('afb2d_stream', 'k_afb2d_tile') and 'afb3d_stream' not in ka
        assert ks[0] == 'sfb1d_strided' and ks[-1] in ('sfb2d_stream', 'k_sfb2d_tile') and 'sfb3d_stream' not in ks


# ---- modules --------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('wave', ['haar', 'db4', 'sym4', 'bior2.2', 'db8', 'tuple'])
def test_modules_match_oracle_and_reconstruct(wave, mode):
    if wave == 'tuple':
        w = wavelets.Wavelet('db3')
        fwd, inv = (w.dec_lo, w.dec_hi), (w.rec_lo, w.rec_hi)
    else:
        fwd = inv = wave
    f = pw.DWT3DForward(J=3 if wave != 'db8' else 1, wave=fwd, mode=mode).to(DEV)
    i = pw.DWT3DInverse(wave=inv, mode=mode).to(DEV)
    rng = np.random.default_rng(21)
    x = rng.standard_normal((2, 2, 19, 24, 29)).astype(np.float32)
    xt = torch.from_numpy(x).to(DEV)
    for J in range(1, f.J + 1):
        f.J = J
        yl, yh = f(xt)
        oyl, oyh = o3.dwt3d_forward(x, (_np(f.h0).ravel(), _np(f.h1).ravel()), J, mode)
        assert np.array_equal(_np(yl), oyl) and all(np.array_equal(_np(a), b) for a, b in zip(yh, oyh))
        y = i((yl, yh))
        assert (y[:, :, :19, :24, :29] - xt).abs().max().item() <= 1e-5 * np.abs(x).max()
    # float64: modules built under a float64 default dtype hold double-precision taps
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        f = pw.DWT3DForward(J=f.J, wave=fwd, mode=mode).to(DEV)
        i = pw.DWT3DInverse(wave=inv, mode=mode).to(DEV)
    finally:
        torch.set_default_dtype(prev)
    xd = xt.double()
    y = i(f(xd))
    assert (y[:, :, :19, :24, :29] - xd).abs().max().item() <= 1e-10 * np.abs(x).max()


def test_inverse_none_bands_and_trimmed_low_pass():
    f = pw.DWT3DForward(J=2, wave='db4', mode='symmetric').to(DEV)
    i = pw.DWT3DInverse(wave='db4', mode='symmetric').to(DEV)
    x = torch.randn(1, 2, 17, 20, 23, device=DEV)
    yl, yh = f(x)
    _, (g0, g1) = _filters('db4')
    y = i((yl, [None, yh[1]]))
    low = o3.dwt3d_inverse(_np(yl).astype(np.float64), [None, _np(yh[1]).astype(np.float64)], (g0, g1), 'symmetric')
    assert util.rel_err(_np(y), low) < 1e-5
    y = i((yl, [None, None]))
    low = o3.dwt3d_inverse(_np(yl).astype(np.float64), [None, None], (g0, g1), 'symmetric')
    assert util.rel_err(_np(y), low) < 1e-5
    # a low-pass one longer than the band-pass along one axis, or all three: its last sample is dropped first
    ref = i((yl, yh))
    for axes in ((2,), (3,), (4,), (2, 3, 4)):
        big = yl
        for ax in axes:
            big = torch.cat([big, torch.randn_like(big.narrow(ax, 0, 1))], dim=ax)
        assert torch.equal(i((big, yh)), ref)


@pytest.mark.parametrize('mode', ['symmetric', 'reflect', 'periodic', 'periodization'])
def test_d_constant_identity(mode):
    """Constant along D: yl and bands 1, 3, 5 are sum(h0) times DWTForward's yl and lh, hl, hh of one slice; bands 0,
    2, 4, 6 vanish.  Independent of the oracle."""
    s = torch.randn(2, 3, 1, 36, 70, device=DEV)
    x = s.expand(2, 3, 12, 36, 70).contiguous()
    f3 = pw.DWT3DForward(J=1, wave='db4', mode=mode).to(DEV)
    f2 = pw.DWTForward(J=1, wave='db4', mode=mode).to(DEV)
    yl, yh = f3(x)
    l2, h2 = f2(s[:, :, 0])
    k = float(f3.h0.sum())
    tol = 1e-5 * float(s.abs().max())
    assert (yl - k * l2[:, :, None]).abs().max().item() < tol
    for v in range(3):
        assert (yh[0][:, :, 2 * v + 1] - k * h2[0][:, :, v][:, :, None]).abs().max().item() < tol
    for b in (0, 2, 4, 6):
        assert yh[0][:, :, b].abs().max().item() < tol


# ---- float64 --------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('mode', MODES)
def test_f64_matches_oracle_and_backward_is_the_synthesis(mode):
    (h0, h1), _ = _filters('db3')
    m = mode_to_int(mode)
    rng = np.random.default_rng(8)
    x = rng.standard_normal((1, 2, 9, 13, 18))
    xt = torch.from_numpy(x).to(DEV).requires_grad_(True)
    yl, yh = AFB3D.apply(xt, h0, h1, m)
    oyl, oyh = o3.dwt_afb3d(x, h0, h1, mode)
    assert util.rel_err(_np(yl), oyl) < 1e-12 and util.rel_err(_np(yh), oyh) < 1e-12
    gl, gh = torch.randn_like(yl), torch.randn_like(yh)
    torch.autograd.backward((yl, yh), (gl, gh))
    want = sfb3d_level(gl, gh, h0, h1, m, out_dhw=x.shape[2:])
    assert torch.equal(xt.grad, want)


def test_gradcheck_f64_zero_mode():
    f = pw.DWT3DForward(J=1, wave='db2', mode='zero').to(DEV).double()
    i = pw.DWT3DInverse(wave='db2', mode='zero').to(DEV).double()
    x = torch.randn(1, 1, 5, 6, 7, device=DEV, dtype=torch.float64, requires_grad=True)
    assert torch.autograd.gradcheck(lambda t: tuple([f(t)[0]] + f(t)[1]), (x,))
    yl, yh = f(x.detach())
    yl = yl.clone().requires_grad_(True)
    h = yh[0].clone().requires_grad_(True)
    assert torch.autograd.gradcheck(lambda a, b: i((a, [b])), (yl, h))
