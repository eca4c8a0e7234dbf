"""GPU parity tests (-m gpu): the CUDA path through the public nn.Module API / C ABI against
  (1) the committed golden vectors produced by the reference itself (tests/golden),
  (2) the CPU oracle on seeded random inputs over the reference's case matrix (odd sizes, all modes,
      o_dim/ri_dim, skip_hps, None highs),
  (3) size-independent properties at larger sizes (perfect reconstruction, linearity, adjoint identity).
fp32 tolerance: RTOL_F32 (1e-5 of max|ref|), stated in tests/util.py; the DWT analysis path is
additionally required to be bit-identical to the oracle (same FMA order)."""
import numpy as np
import pytest
import torch

import pytorch_wavelets_b200 as pw
from oracle import oracle as orc
from pytorch_wavelets_b200 import _ffi
from tests import util

pytestmark = pytest.mark.gpu
DEV = 'cuda'
TOL = util.RTOL_F32


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _n(t):
    return t.detach().cpu().numpy()


@pytest.fixture(scope='module', autouse=True)
def _native_library_is_loaded():
    """The CUDA extension must be the thing that runs: it has to load, and there is no fallback."""
    assert torch.cuda.is_available()
    lib = _ffi.lib()
    assert lib.b200w_version() >= 100
    yield


# ---------------------------------------------------------------- golden vectors (reference outputs)

@pytest.mark.parametrize('name', util.fixtures('dwt_'))
def test_dwt_golden(name):
    g = util.load(name)
    J, mode, wave = int(g['J']), str(g['mode']), str(g['wave'])
    f = pw.DWTForward(J=J, wave=wave, mode=mode).to(DEV)
    i = pw.DWTInverse(wave=wave, mode=mode).to(DEV)
    x = _t(g['x'])
    yl, yh = f(x)
    assert yl.is_contiguous() and all(h.is_contiguous() for h in yh)
    util.assert_close(_n(yl), g['yl'], TOL, 'yl')
    for j in range(J):
        util.assert_close(_n(yh[j]), g['yh%d' % j], TOL, 'yh%d' % j)
    y = i((_t(g['yl']), [_t(g['yh%d' % j]) for j in range(J)]))
    util.assert_close(_n(y), g['y'], TOL, 'inverse')
    yh_drop = [_t(g['yh%d' % j]) for j in range(J)]
    if J > 1:
        yh_drop[0] = None
    util.assert_close(_n(i((_t(g['yl']), yh_drop))), g['y_drop0'], TOL, 'inverse None')


def test_config1_bit_check():
    """BASELINE.json configs[0]: DWTForward J=1 db4 zero on randn(4,3,64,64): max abs err <= 2e-6 and
    the bit-equal fraction vs the reference's own CPU output is reported (expected 1.0)."""
    g = util.load('dwt_c1_db4_zero_J1')
    yl, yh = pw.DWTForward(J=1, wave='db4', mode='zero').to(DEV)(_t(g['x']))
    assert np.abs(_n(yl) - g['yl']).max() <= 2e-6
    assert np.abs(_n(yh[0]) - g['yh0']).max() <= 2e-6
    frac = min(util.bit_equal_fraction(_n(yl), g['yl']), util.bit_equal_fraction(_n(yh[0]), g['yh0']))
    print('config-1 bit-equal fraction vs reference CPU output: %.6f' % frac)
    assert frac > 0.999


@pytest.mark.parametrize('name', util.fixtures('dtcwt_'))
def test_dtcwt_golden(name):
    g = util.load(name)
    J, mode = int(g['J']), str(g['mode'])
    o_dim, ri_dim = int(g['o_dim']), int(g['ri_dim'])
    skip = [bool(s) for s in g['skip']]
    kw = dict(biort=str(g['biort']), qshift=str(g['qshift']), o_dim=o_dim, ri_dim=ri_dim, mode=mode)
    f = pw.DTCWTForward(J=J, skip_hps=skip, **kw).to(DEV)
    i = pw.DTCWTInverse(**kw).to(DEV)
    yl, yh = f(_t(g['x']))
    util.assert_close(_n(yl), g['yl'], TOL, 'yl')
    for j in range(J):
        if skip[j]:
            assert yh[j].shape == torch.Size([])
        else:
            assert tuple(yh[j].shape) == g['yh%d' % j].shape
            util.assert_close(_n(yh[j]), g['yh%d' % j], TOL, 'yh%d' % j)
    yh_in = [None if skip[j] else _t(g['yh%d' % j]) for j in range(J)]
    util.assert_close(_n(i((_t(g['yl']), yh_in))), g['y'], TOL, 'inverse')


@pytest.mark.parametrize('name', util.fixtures('scat_'))
def test_scat_golden(name):
    g = util.load(name)
    kw = dict(biort=str(g['biort']), mode=str(g['mode']), magbias=float(g['magbias']))
    s = pw.ScatLayer(**kw).to(DEV)
    z = s(_t(g['x']))
    util.assert_close(_n(z), g['z'], TOL, 'z')
    s2 = torch.nn.Sequential(pw.ScatLayer(**kw), pw.ScatLayer(**kw)).to(DEV)
    util.assert_close(_n(s2(_t(g['x']))), g['z2'], TOL, 'z2')


# ---------------------------------------------------------------- oracle on seeded random inputs

DWT_MODES = ['zero', 'symmetric', 'reflect', 'periodic', 'periodization']


@pytest.mark.parametrize('mode', DWT_MODES)
@pytest.mark.parametrize('wave,J,shape', [('db4', 3, (3, 5, 128, 128)), ('db1', 3, (2, 3, 127, 126)),
                                          ('db3', 2, (2, 2, 100, 99)), ('db8', 2, (1, 3, 190, 256)),
                                          ('db2', 4, (1, 1, 201, 77)), ('db12', 1, (1, 2, 97, 64))])
def test_dwt_vs_oracle(mode, wave, J, shape):
    torch.manual_seed(1)
    x = torch.randn(*shape)
    f = pw.DWTForward(J=J, wave=wave, mode=mode)
    i = pw.DWTInverse(wave=wave, mode=mode)
    L = f.h0_col.numel()
    if mode == 'reflect' and min(shape[2:]) // (2 ** (J - 1)) <= L:
        pytest.skip('reflect pad would exceed the signal')
    hf = [b.numpy() for b in (f.h0_col, f.h1_col, f.h0_row, f.h1_row)]
    gf = [b.numpy() for b in (i.g0_col, i.g1_col, i.g0_row, i.g1_row)]
    oyl, oyh = orc.dwt_forward(x.numpy(), hf, J, mode)
    f, i = f.to(DEV), i.to(DEV)
    yl, yh = f(x.to(DEV))
    # same FMA order as the oracle: bit-identical (== ignores the sign of zero)
    assert np.array_equal(_n(yl), oyl), util.rel_err(_n(yl), oyl)
    for j in range(J):
        assert np.array_equal(_n(yh[j]), oyh[j]), util.rel_err(_n(yh[j]), oyh[j])
    oy = orc.dwt_inverse(oyl, oyh, gf, mode)
    y = i((yl, yh))
    # synthesis: the streaming kernel runs the W pass before the H pass (they commute; fp32 rounding differs)
    util.assert_close(_n(y), oy, TOL, 'inverse')
    # perfect reconstruction on the original extent
    H, W = shape[2:]
    assert np.abs(_n(y)[:, :, :H, :W] - x.numpy()).max() < 2e-5


@pytest.mark.parametrize('mode', ['zero', 'symmetric', 'periodization'])
@pytest.mark.parametrize('wave', ['bior2.4', 'bior1.3', 'bior4.4', 'rbio3.3', 'sym4', 'sym5', 'coif1'])
def test_dwt_other_families_vs_oracle(wave, mode):
    """Wavelet families beyond dbN (the reference's tests use 'bior2.4', tests/test_dwt.py:37): zero-padded biorthogonal
    banks, symlets, coif1 through the public modules against the oracle with the same taps."""
    torch.manual_seed(2)
    shape, J = (2, 3, 96, 120), 2
    x = torch.randn(*shape)
    f = pw.DWTForward(J=J, wave=wave, mode=mode)
    i = pw.DWTInverse(wave=wave, mode=mode)
    hf = [b.numpy() for b in (f.h0_col, f.h1_col, f.h0_row, f.h1_row)]
    gf = [b.numpy() for b in (i.g0_col, i.g1_col, i.g0_row, i.g1_row)]
    oyl, oyh = orc.dwt_forward(x.numpy(), hf, J, mode)
    f, i = f.to(DEV), i.to(DEV)
    yl, yh = f(x.to(DEV))
    assert np.array_equal(_n(yl), oyl), util.rel_err(_n(yl), oyl)
    for j in range(J):
        assert np.array_equal(_n(yh[j]), oyh[j]), util.rel_err(_n(yh[j]), oyh[j])
    y = i((yl, yh))
    util.assert_close(_n(y), orc.dwt_inverse(oyl, oyh, gf, mode), TOL, 'inverse')
    assert np.abs(_n(y) - x.numpy()).max() < 2e-5


def test_dwt_distinct_row_col_filters_quirk():
    """4-tuple wave: the *_col filters act along W and *_row along H (SURVEY 8(a) A0)."""
    torch.manual_seed(2)
    x = torch.randn(2, 2, 32, 48)
    wa, wb = pw.wavelets.Wavelet('db4'), pw.wavelets.Wavelet('db2')
    f = pw.DWTForward(J=1, wave=(wa.dec_lo, wa.dec_hi, wb.dec_lo, wb.dec_hi), mode='symmetric')
    hf = [b.numpy() for b in (f.h0_col, f.h1_col, f.h0_row, f.h1_row)]
    oyl, oyh = orc.dwt_forward(x.numpy(), hf, 1, 'symmetric')
    yl, yh = f.to(DEV)(x.to(DEV))
    assert tuple(yl.shape) == (2, 2, 17, 27)
    assert np.array_equal(_n(yl), oyl) and np.array_equal(_n(yh[0]), oyh[0])


def test_noncontiguous_and_offset_inputs():
    torch.manual_seed(3)
    big = torch.randn(2, 3, 70, 90, device=DEV)
    x = big[:, :, 3:67, 5:85]  # strided view, pitch 90
    f = pw.DWTForward(J=2, wave='db3', mode='symmetric').to(DEV)
    a = f(x)
    b = f(x.contiguous())
    assert torch.equal(a[0], b[0]) and all(torch.equal(p, q) for p, q in zip(a[1], b[1]))
    xt = big.transpose(2, 3)  # rows not unit-stride -> copied internally
    a = f(xt)
    b = f(xt.contiguous())
    assert torch.equal(a[0], b[0])


LAYOUTS = [(2, -1), (1, 2), (4, 5), (3, 1), (5, 2), (2, 3)]


@pytest.mark.parametrize('biort,qshift', [('near_sym_a', 'qshift_a'), ('near_sym_b', 'qshift_b'),
                                          ('antonini', 'qshift_c'), ('legall', 'qshift_d'),
                                          ('near_sym_a', 'qshift_06')])
@pytest.mark.parametrize('shape', [(2, 3, 128, 128), (1, 2, 100, 100), (1, 2, 99, 100), (1, 1, 104, 101)])
def test_dtcwt_vs_oracle(biort, qshift, shape):
    torch.manual_seed(4)
    J = 3
    x = 100 * torch.randn(*shape)
    f = pw.DTCWTForward(biort=biort, qshift=qshift, J=J)
    i = pw.DTCWTInverse(biort=biort, qshift=qshift)
    l1 = (f.h0o.numpy(), f.h1o.numpy())
    qs = (f.h0a.numpy(), f.h0b.numpy(), f.h1a.numpy(), f.h1b.numpy())
    oyl, oyh = orc.dtcwt_forward(x.numpy(), l1, qs, J)
    f, i = f.to(DEV), i.to(DEV)
    yl, yh = f(x.to(DEV))
    util.assert_close(_n(yl), oyl, TOL, 'yl')
    for j in range(J):
        util.assert_close(_n(yh[j]), oyh[j], TOL, 'yh%d' % j)
    gl1 = (_n(i.g0o), _n(i.g1o))
    gqs = (_n(i.g0a), _n(i.g0b), _n(i.g1a), _n(i.g1b))
    oy = orc.dtcwt_inverse(oyl, oyh, gl1, gqs)
    y = i((yl, yh))
    util.assert_close(_n(y), oy, TOL, 'inverse')
    H, W = shape[2:]
    assert np.abs(_n(y)[:, :, :H, :W] - x.numpy()).max() < 2e-5 * 100 * 5  # perfect reconstruction
    # None band-passes
    for drop in (0, 1):
        yh2 = list(yh)
        yh2[drop] = None
        oyh2 = list(oyh)
        oyh2[drop] = None
        util.assert_close(_n(i((yl, yh2))), orc.dtcwt_inverse(oyl, oyh2, gl1, gqs), TOL, 'inverse None %d' % drop)


@pytest.mark.parametrize('o_dim,ri_dim', LAYOUTS)
@pytest.mark.parametrize('mode', ['symmetric', 'zero'])
def test_dtcwt_layouts_and_modes(o_dim, ri_dim, mode):
    torch.manual_seed(5)
    x = 100 * torch.randn(2, 3, 72, 88)
    f = pw.DTCWTForward(J=2, o_dim=o_dim, ri_dim=ri_dim, mode=mode)
    i = pw.DTCWTInverse(o_dim=o_dim, ri_dim=ri_dim, mode=mode)
    l1 = (f.h0o.numpy(), f.h1o.numpy())
    qs = (f.h0a.numpy(), f.h0b.numpy(), f.h1a.numpy(), f.h1b.numpy())
    oyl, oyh = orc.dtcwt_forward(x.numpy(), l1, qs, 2, o_dim=o_dim, ri_dim=ri_dim, mode=mode)
    gl1 = (i.g0o.numpy(), i.g1o.numpy())
    gqs = (i.g0a.numpy(), i.g0b.numpy(), i.g1a.numpy(), i.g1b.numpy())
    f, i = f.to(DEV), i.to(DEV)
    yl, yh = f(x.to(DEV))
    util.assert_close(_n(yl), oyl, TOL)
    for j in range(2):
        assert tuple(yh[j].shape) == oyh[j].shape
        util.assert_close(_n(yh[j]), oyh[j], TOL)
    util.assert_close(_n(i((yl, yh))), orc.dtcwt_inverse(oyl, oyh, gl1, gqs, o_dim, ri_dim, mode), TOL)


def test_dtcwt_skip_hps_include_scale_and_j0():
    torch.manual_seed(6)
    x = torch.randn(1, 2, 64, 64, device=DEV)
    f = pw.DTCWTForward(J=3, skip_hps=[True, False, True], include_scale=[False, True, True]).to(DEV)
    scales, yh = f(x)
    assert isinstance(scales, list) and scales[0].shape == torch.Size([])
    assert tuple(scales[1].shape) == (1, 2, 32, 32) and tuple(scales[2].shape) == (1, 2, 16, 16)
    assert yh[0].shape == torch.Size([]) and yh[2].shape == torch.Size([])
    assert tuple(yh[1].shape) == (1, 2, 6, 16, 16, 2)
    full = pw.DTCWTForward(J=3).to(DEV)(x)
    assert torch.equal(scales[2], full[0]) and torch.equal(yh[1], full[1][1])
    y0 = pw.DTCWTForward(J=0).to(DEV)(x)
    assert y0[0] is x and y0[1] is None


def test_dtcwt_inverse_asserts_like_reference():
    i = pw.DTCWTInverse().to(DEV)
    yl = torch.zeros(1, 1, 8, 8, device=DEV)
    with pytest.raises(AssertionError):
        i((yl, [torch.zeros(1, 1, 6, 8, 8, 2, device=DEV), torch.zeros(1, 1, 5, 4, 4, 2, device=DEV)]))


@pytest.mark.parametrize('biort', ['near_sym_a', 'near_sym_b', 'antonini'])
@pytest.mark.parametrize('shape', [(4, 3, 64, 64), (2, 1, 31, 29), (1, 2, 30, 32)])
@pytest.mark.parametrize('mode', ['symmetric', 'zero'])
def test_scat_vs_oracle(biort, shape, mode):
    torch.manual_seed(7)
    x = torch.randn(*shape)
    s = pw.ScatLayer(biort=biort, mode=mode)
    oz = orc.scat_layer(x.numpy(), (s.h0o.data.numpy(), s.h1o.data.numpy()), mode, 1e-2)
    z = s.to(DEV)(x.to(DEV))
    util.assert_close(_n(z), oz, TOL)


@pytest.mark.parametrize('magbias', [0.0, 1e-20, 1e-2, 3.0])
def test_scat_magbias_range_and_zero_input(magbias):
    """The ScatLayer epilogue has two square-root paths: the plain one when magbias^2 >= 1e-30 and one that rescales tiny
    arguments and returns 0 for 0 (magbias = 0, where the reference computes sqrt(0) - 0 on flat regions).  Both against
    the oracle, on an image with an all-zero plane, a constant plane and tiny values."""
    torch.manual_seed(9)
    x = torch.randn(2, 3, 32, 64)
    x[0, 1] = 0.0
    x[1, 0] = 2.5
    x[1, 2] *= 1e-18
    s = pw.ScatLayer(magbias=magbias)
    oz = orc.scat_layer(x.numpy(), (s.h0o.data.numpy(), s.h1o.data.numpy()), 'symmetric', magbias)
    z = _n(s.to(DEV)(x.to(DEV)))
    assert np.isfinite(z).all()
    util.assert_close(z, oz, TOL)
    if magbias == 0.0:
        zero_plane = z[0].reshape(7, 3, 16, 32)[1:, 1]             # magnitudes of the all-zero input plane
        assert np.array_equal(zero_plane, np.zeros_like(zero_plane))


# ---------------------------------------------------------------- autograd (adjoint identities)

def _dot(a, b):
    return float((a.double() * b.double()).sum())


def _flat_dot(ya, yb):
    return sum(_dot(p, q) for p, q in zip(ya, yb))


@pytest.mark.parametrize('mode,shape', [('zero', (2, 2, 45, 64)), ('periodization', (2, 2, 48, 64))])
def test_dwt_backward_is_adjoint(mode, shape):
    """<A x, y> == <x, A^T y> with A^T computed by autograd.  Holds where the reference's backward is the
    true adjoint: zero padding, and periodization of even-sized inputs (for the other extensions the
    reference's backward ignores the fold-back of the padding; see test_dwt_gradient_identities)."""
    torch.manual_seed(8)
    f = pw.DWTForward(J=2, wave='db3', mode=mode).to(DEV)
    x = torch.randn(*shape, device=DEV, requires_grad=True)
    yl, yh = f(x)
    outs = [yl] + yh
    ws = [torch.randn_like(o) for o in outs]
    loss = sum((o * w).sum() for o, w in zip(outs, ws))
    loss.backward()
    x2 = torch.randn_like(x)
    with torch.no_grad():
        yl2, yh2 = f(x2)
    lhs = _flat_dot([yl2] + yh2, ws)
    rhs = _dot(x2, x.grad)
    assert abs(lhs - rhs) <= 1e-4 * max(1.0, abs(lhs)), (lhs, rhs)
    i = pw.DWTInverse(wave='db3', mode=mode).to(DEV)
    cl = yl.detach().clone().requires_grad_(True)
    ch = [h.detach().clone().requires_grad_(True) for h in yh]
    y = i((cl, ch))
    w = torch.randn_like(y)
    (y * w).sum().backward()
    dl = torch.randn_like(cl)
    dh = [torch.randn_like(h) for h in ch]
    with torch.no_grad():
        y2 = i((dl, dh))
    lhs = _dot(y2, w)
    rhs = _dot(dl, cl.grad) + sum(_dot(a, b.grad) for a, b in zip(dh, ch))
    assert abs(lhs - rhs) <= 1e-4 * max(1.0, abs(lhs)), (lhs, rhs)


@pytest.mark.parametrize('wave,J,mode', [('db1', 1, 'zero'), ('db1', 3, 'zero'), ('db3', 1, 'symmetric'),
                                         ('db3', 2, 'reflect'), ('db2', 3, 'periodization'), ('db4', 2, 'zero'),
                                         ('db3', 2, 'periodic')])
def test_dwt_gradient_identities(wave, J, mode):
    """The reference's own gradient tests (tests/test_dwt.py:215-299): the gradient of the forward transform is
    the inverse transform with the (time-reversed) analysis filters, and vice versa."""
    torch.manual_seed(14)
    w = pw.wavelets.Wavelet(wave)
    fwd_filts = (w.dec_lo, w.dec_hi)
    inv_filts = (w.dec_lo[::-1], w.dec_hi[::-1])
    dwt = pw.DWTForward(J=J, wave=fwd_filts, mode=mode).to(DEV)
    iwt = pw.DWTInverse(wave=inv_filts, mode=mode).to(DEV)
    x = torch.randn(3, 2, 128, 128, device=DEV, requires_grad=True)
    yl, yh = dwt(x)
    ylg = torch.randn_like(yl)
    yl.backward(ylg, retain_graph=True)
    zeros = [torch.zeros_like(h) for h in yh]
    ref = iwt((ylg, zeros))
    assert (x.grad - ref).abs().max() < 1e-4
    for j, y in enumerate(yh):
        x.grad.zero_()
        g = torch.randn_like(y)
        y.backward(g, retain_graph=True)
        hps = list(zeros)
        hps[j] = g
        ref = iwt((torch.zeros_like(yl), hps))
        assert (x.grad - ref).abs().max() < 1e-4
    # gradient of the inverse == forward with swapped filters
    with torch.no_grad():
        l, h = dwt(torch.zeros(3, 2, 128, 128, device=DEV))
    cl = torch.randn_like(l).requires_grad_(True)
    ch = [torch.randn_like(t).requires_grad_(True) for t in h]
    y = iwt((cl, ch))
    yg = torch.randn_like(y)
    y.backward(yg)
    with torch.no_grad():
        dyl, dyh = dwt(yg)
    assert (cl.grad - dyl).abs().max() < 1e-4
    for a, b in zip(ch, dyh):
        assert (a.grad - b).abs().max() < 1e-4


@pytest.mark.parametrize('biort,qshift', [('near_sym_a', 'qshift_a'), ('near_sym_b', 'qshift_b'),
                                          ('antonini', 'qshift_c'), ('legall', 'qshift_d')])
@pytest.mark.parametrize('o_dim,ri_dim', [(2, -1), (1, 2)])
def test_dtcwt_backward_is_adjoint(o_dim, ri_dim, biort, qshift):
    """Backward passes run the opposite transform's kernels with the stored filters (every filter pair has its own
    streaming instantiation for the default layout; other layouts take the generic kernels)."""
    torch.manual_seed(9)
    f = pw.DTCWTForward(J=3, o_dim=o_dim, ri_dim=ri_dim, biort=biort, qshift=qshift).to(DEV)
    x = torch.randn(2, 2, 64, 96, device=DEV, requires_grad=True)
    yl, yh = f(x)
    outs = [yl] + yh
    ws = [torch.randn_like(o) for o in outs]
    sum((o * w).sum() for o, w in zip(outs, ws)).backward()
    x2 = torch.randn_like(x)
    with torch.no_grad():
        yl2, yh2 = f(x2)
    lhs = _flat_dot([yl2] + yh2, ws)
    rhs = _dot(x2, x.grad)
    assert abs(lhs - rhs) <= 1e-4 * max(1.0, abs(lhs)), (lhs, rhs)
    i = pw.DTCWTInverse(o_dim=o_dim, ri_dim=ri_dim, biort=biort, qshift=qshift).to(DEV)
    cl = yl.detach().clone().requires_grad_(True)
    ch = [h.detach().clone().requires_grad_(True) for h in yh]
    y = i((cl, ch))
    w = torch.randn_like(y)
    (y * w).sum().backward()
    dl = torch.randn_like(cl)
    dh = [torch.randn_like(h) for h in ch]
    with torch.no_grad():
        y2 = i((dl, dh))
    lhs = _dot(y2, w)
    rhs = _dot(dl, cl.grad) + sum(_dot(a, b.grad) for a, b in zip(dh, ch))
    assert abs(lhs - rhs) <= 1e-4 * max(1.0, abs(lhs)), (lhs, rhs)


def test_scat_backward_matches_finite_difference():
    torch.manual_seed(10)
    s = pw.ScatLayer().to(DEV)
    x = torch.randn(1, 2, 16, 16, device=DEV, requires_grad=True)
    z = s(x)
    w = torch.randn_like(z)
    (z * w).sum().backward()
    d = torch.randn_like(x)
    eps = 1e-2
    with torch.no_grad():
        fd = (((s(x + eps * d) - s(x - eps * d)) * w).sum() / (2 * eps)).item()
    an = _dot(d, x.grad)
    assert abs(fd - an) <= 2e-2 * max(1.0, abs(an)), (fd, an)


# ---------------------------------------------------------------- properties at larger sizes

def test_dwt_linearity_and_pr_large():
    torch.manual_seed(11)
    f = pw.DWTForward(J=3, wave='db4', mode='symmetric').to(DEV)
    i = pw.DWTInverse(wave='db4', mode='symmetric').to(DEV)
    a = torch.randn(8, 32, 512, 512, device=DEV)
    b = torch.randn(8, 32, 512, 512, device=DEV)
    ya, yb, yab = f(a), f(b), f(2 * a - 3 * b)
    assert tuple(ya[0].shape) == (8, 32, 70, 70)
    assert [tuple(h.shape[-2:]) for h in ya[1]] == [(259, 259), (133, 133), (70, 70)]
    assert (yab[0] - (2 * ya[0] - 3 * yb[0])).abs().max() < 1e-3
    for p, q, r in zip(ya[1], yb[1], yab[1]):
        assert (r - (2 * p - 3 * q)).abs().max() < 1e-4
    assert (i(ya) - a).abs().max() < 2e-5
    # level-by-level consistency: J=3 equals three J=1 applications
    f1 = pw.DWTForward(J=1, wave='db4', mode='symmetric').to(DEV)
    l1, h1 = f1(a)
    l2, h2 = f1(l1)
    l3, h3 = f1(l2)
    assert torch.equal(l3, ya[0]) and torch.equal(h1[0], ya[1][0]) and torch.equal(h3[0], ya[1][2])


def test_config5_shape_db8_j4_zero():
    """BASELINE.json configs[4] per-GPU shard shape (db8, J=4, mode zero, 2048x2048), reduced batch: bit-identity
    with the oracle on one plane, pyramid shapes of SURVEY appendix A, perfect reconstruction."""
    torch.manual_seed(15)
    f = pw.DWTForward(J=4, wave='db8', mode='zero').to(DEV)
    i = pw.DWTInverse(wave='db8', mode='zero').to(DEV)
    x = torch.randn(2, 3, 2048, 2048, device=DEV)
    yl, yh = f(x)
    assert tuple(yl.shape) == (2, 3, 142, 142)
    assert [tuple(h.shape[-2:]) for h in yh] == [(1031, 1031), (523, 523), (269, 269), (142, 142)]
    hf = [_n(b) for b in (f.h0_col, f.h1_col, f.h0_row, f.h1_row)]
    oyl, oyh = orc.dwt_forward(_n(x[:1, :1]), hf, 4, 'zero')
    assert np.array_equal(_n(yl[:1, :1]), oyl)
    for a, b in zip(yh, oyh):
        assert np.array_equal(_n(a[:1, :1]), b)
    assert (i((yl, yh)) - x).abs().max() < 5e-5


@pytest.mark.parametrize('shape', [(2, 2, 256, 256), (1, 3, 255, 130)])
def test_periodization_roundtrip_and_oracle(shape):
    torch.manual_seed(16)
    x = torch.randn(*shape)
    f = pw.DWTForward(J=3, wave='db4', mode='periodization')
    hf = [b.numpy() for b in (f.h0_col, f.h1_col, f.h0_row, f.h1_row)]
    oyl, oyh = orc.dwt_forward(x.numpy(), hf, 3, 'periodization')
    yl, yh = f.to(DEV)(x.to(DEV))
    assert np.array_equal(_n(yl), oyl)
    y = pw.DWTInverse(wave='db4', mode='periodization').to(DEV)((yl, yh))
    H, W = shape[2:]
    assert (y[:, :, :H, :W].cpu() - x).abs().max() < 2e-5


def test_dtcwt_pr_and_energy_large():
    torch.manual_seed(12)
    f = pw.DTCWTForward(J=3).to(DEV)
    i = pw.DTCWTInverse().to(DEV)
    x = torch.randn(8, 3, 1024, 1024, device=DEV)
    yl, yh = f(x)
    assert tuple(yl.shape) == (8, 3, 256, 256)
    assert [tuple(h.shape) for h in yh] == [(8, 3, 6, 512, 512, 2), (8, 3, 6, 256, 256, 2), (8, 3, 6, 128, 128, 2)]
    assert (i((yl, yh)) - x).abs().max() < 3e-5
    # near-tight frame: energy of the coefficients ~ energy of the input (Kingsbury's DTCWT)
    e_in = float((x.double() ** 2).sum())
    e_out = float((yl.double() ** 2).sum()) + sum(float((h.double() ** 2).sum()) for h in yh)
    assert abs(e_out / e_in - 1.0) < 0.05


def test_generic_and_auto_paths_agree():
    """Whatever kernel the dispatcher picks (specialised streaming or generic tile), results are identical."""
    torch.manual_seed(13)
    lib = _ffi.lib()
    x = torch.randn(3, 4, 200, 264, device=DEV)
    f = pw.DWTForward(J=3, wave='db4', mode='symmetric').to(DEV)
    d = pw.DTCWTForward(J=3).to(DEV)
    with _ffi.generic_kernels():
        a, b = f(x), d(x)
        inv = pw.DWTInverse(wave='db4', mode='symmetric').to(DEV)
        ya = inv(a)
    a2, b2 = f(x), d(x)
    assert torch.equal(a[0], a2[0]) and all(torch.equal(p, q) for p, q in zip(a[1], a2[1]))
    assert torch.equal(b[0], b2[0]) and all(torch.equal(p, q) for p, q in zip(b[1], b2[1]))
    ya2 = inv(a2)
    assert (ya - ya2).abs().max().item() <= 1e-5 * ya.abs().max().item()


@pytest.mark.parametrize('mode', ['symmetric', 'zero', 'periodization'])
@pytest.mark.parametrize('wave', ['db5', 'db6', 'db7', 'db8', 'db9', 'db10'])
def test_dwt_long_filters_match_generic(wave, mode):
    """Filter lengths 10..20 have their own streaming instantiations (analysis and synthesis): forward bit-identical
    to the generic tile kernel, inverse within the fp32 tolerance (pass order differs), perfect reconstruction."""
    torch.manual_seed(37)
    lib = _ffi.lib()
    f = pw.DWTForward(J=2, wave=wave, mode=mode).to(DEV)
    g = pw.DWTInverse(wave=wave, mode=mode).to(DEV)
    x = torch.randn(2, 3, 150, 264, device=DEV)
    with _ffi.generic_kernels():
        a = f(x)
        ya = g(a)
    b = f(x)
    assert torch.equal(a[0], b[0]) and all(torch.equal(p, q) for p, q in zip(a[1], b[1]))
    yb = g(b)
    assert (ya - yb).abs().max().item() <= 1e-5 * ya.abs().max().item()
    assert (yb[..., :150, :264] - x).abs().max().item() < 1e-4


@pytest.mark.parametrize('wave', ['db1', 'db2', 'db3', 'db4'])
@pytest.mark.parametrize('shape', [(2, 2, 64, 96), (1, 3, 37, 130), (2, 1, 6, 10), (1, 2, 200, 259)])
def test_periodization_inverse_streaming_matches_generic_and_oracle(wave, shape):
    """Periodization synthesis on the streaming kernel (rotated stores, wrapped staging): odd sizes (cropped outputs),
    planes smaller than the filter, several strips; against the generic tile kernel and the oracle."""
    torch.manual_seed(41)
    lib = _ffi.lib()
    f = pw.DWTForward(J=2, wave=wave, mode='periodization').to(DEV)
    g = pw.DWTInverse(wave=wave, mode='periodization').to(DEV)
    x = torch.randn(*shape, device=DEV)
    c = f(x)
    with _ffi.generic_kernels():
        ya = g(c)
    yb = g(c)
    assert ya.shape == yb.shape
    assert (ya - yb).abs().max().item() <= 1e-5 * max(1.0, ya.abs().max().item())
    H, W = shape[2:]
    assert (yb[..., :H, :W] - x).abs().max().item() < 1e-4
    gf = [_n(b) for b in (g.g0_col, g.g1_col, g.g0_row, g.g1_row)]
    oy = orc.dwt_inverse(_n(c[0]), [_n(h) for h in c[1]], gf, 'periodization')
    util.assert_close(_n(yb), oy, TOL, 'vs oracle')


@pytest.mark.parametrize('mode', ['symmetric', 'zero'])
def test_wide_dtcwt_level1_inverse_matches_generic_and_oracle(mode):
    """DTCWT level-1 synthesis on planes several strips wide: widths around the strip boundaries, both extension modes, a
    missing low-pass / band-pass input, and the backward pass of FWD_J1 (the (5,7) instantiation) -- streaming kernel
    against the generic tile kernel (same arithmetic: 1e-6) and the oracle."""
    torch.manual_seed(47)
    i = pw.DTCWTInverse(biort='near_sym_a', qshift='qshift_a', mode=mode).to(DEV)
    f = pw.DTCWTForward(J=1, biort='near_sym_a', qshift='qshift_a', mode=mode).to(DEV)
    g0o, g1o = _n(i.g0o), _n(i.g1o)
    for k, W in enumerate([128, 132, 136, 192, 252, 256, 260, 388]):
        H = [16, 18, 30, 44][k % 4]
        yl = torch.randn(2, 2, H, W, device=DEV)
        yh = [torch.randn(2, 2, 6, H // 2, W // 2, 2, device=DEV)]
        with _ffi.generic_kernels():
            ya = i((yl, yh))
        yb = i((yl, yh))
        assert ya.shape == yb.shape == (2, 2, H, W)
        assert (ya - yb).abs().max().item() <= 1e-6 * max(1.0, ya.abs().max().item()), W
        util.assert_close(_n(yb), orc.dtcwt_inv_j1(_n(yl), _n(yh[0]), g0o, g1o, mode=mode), TOL, 'oracle W=%d' % W)
        for lo, hi in ((yl, [None]), (torch.zeros_like(yl), yh)):
            with _ffi.generic_kernels():
                ya = i((lo, hi))
            yb = i((lo, hi))
            assert (ya - yb).abs().max().item() <= 1e-6 * max(1.0, ya.abs().max().item()), W
        # FWD_J1.backward = the level-1 inverse with the analysis filters
        x = torch.randn(1, 2, H, W, device=DEV, requires_grad=True)
        gl, gh = torch.randn(1, 2, H, W, device=DEV), torch.randn(1, 2, 6, H // 2, W // 2, 2, device=DEV)
        grads = []
        for generic in (True, False):
            x.grad = None
            if generic:
                with _ffi.generic_kernels():
                    yl_, yh_ = f(x)
                    (yl_ * gl).sum().add((yh_[0] * gh).sum()).backward()
            else:
                yl_, yh_ = f(x)
                (yl_ * gl).sum().add((yh_[0] * gh).sum()).backward()
            grads.append(x.grad.clone())
        assert (grads[0] - grads[1]).abs().max().item() <= 1e-5 * max(1.0, grads[0].abs().max().item()), W


@pytest.mark.parametrize('mode', ['zero', 'symmetric', 'reflect', 'periodic'])
@pytest.mark.parametrize('wave', ['db1', 'db2', 'db3', 'db4'])
def test_wide_synthesis_kernel_every_width_matches_generic_and_oracle(wave, mode):
    """The wide synthesis kernel (sfb2d_stream4: 4 coefficient columns per lane, 128-column strips; taken when a plane has
    more than 64 coefficient column pairs): every output width around the strip / vector boundaries, odd heights, cropped
    outputs (AFB2D.backward), a missing band-pass tensor -- against the generic tile kernel (tolerance: the passes run in
    the other order) and the oracle."""
    torch.manual_seed(43)
    g = pw.DWTInverse(wave=wave, mode=mode).to(DEV)
    L = g.g0_col.numel()
    gf = [_n(b) for b in (g.g0_col, g.g1_col, g.g0_row, g.g1_row)]
    widths = list(range(65, 75)) + list(range(125, 135)) + [192, 193, 255, 256, 257, 259, 300]
    for k, wc in enumerate(widths):
        hc = 9 + (k % 5)
        yl = torch.randn(2, 2, hc, wc, device=DEV)
        yh = [torch.randn(2, 2, 3, hc, wc, device=DEV)]
        with _ffi.generic_kernels():
            ya = g((yl, yh))
        yb = g((yl, yh))
        assert ya.shape == yb.shape, (wc, ya.shape, yb.shape)
        assert (ya - yb).abs().max().item() <= 1e-5 * max(1.0, ya.abs().max().item()), wc
        if k % 6 == 0:
            util.assert_close(_n(yb), orc.dwt_inverse(_n(yl), [_n(yh[0])], gf, mode), TOL, 'vs oracle, Wc=%d' % wc)
    # band-pass absent (zeros), and a cropped output as AFB2D.backward requests it
    from pytorch_wavelets_b200.dwt import lowlevel
    m = lowlevel.mode_to_int(mode)
    yl = torch.randn(1, 3, 20, 131, device=DEV)
    hi = torch.randn(1, 3, 3, 20, 131, device=DEV)
    for highs, out_hw in ((None, None), (hi, (2 * 20 - L + 1, 2 * 131 - L - 1))):
        with _ffi.generic_kernels():
            ya = lowlevel.sfb2d_level(yl, highs, g.g0_row, g.g1_row, g.g0_col, g.g1_col, m, out_hw=out_hw)
        yb = lowlevel.sfb2d_level(yl, highs, g.g0_row, g.g1_row, g.g0_col, g.g1_col, m, out_hw=out_hw)
        assert ya.shape == yb.shape
        assert (ya - yb).abs().max().item() <= 1e-5 * max(1.0, ya.abs().max().item())


@pytest.mark.parametrize('mode', ['zero', 'symmetric'])
@pytest.mark.parametrize('wave', ['db1', 'db4', 'db6'])
def test_synthesis_streaming_kernels_multi_chunk(wave, mode):
    """Tall coefficient planes and few of them: the chunk cost model then splits every (plane, strip) march into many
    row chunks (16-row-pair chunks here), so the first rows of many chunks and the chunk seams are checked.  db1 / db4
    take the wide kernel, db6 (12 taps) the 2-column kernel; 1-strip and 3-strip widths, odd heights.  Against the
    generic tile kernel and the oracle."""
    torch.manual_seed(47)
    g = pw.DWTInverse(wave=wave, mode=mode).to(DEV)
    gf = [_n(b) for b in (g.g0_col, g.g1_col, g.g0_row, g.g1_row)]
    for hc, wc in ((203, 131), (157, 300)):
        yl = torch.randn(1, 2, hc, wc, device=DEV)
        yh = [torch.randn(1, 2, 3, hc, wc, device=DEV)]
        with _ffi.generic_kernels():
            ya = g((yl, yh))
        yb = g((yl, yh))
        assert ya.shape == yb.shape
        assert (ya - yb).abs().max().item() <= 1e-5 * max(1.0, ya.abs().max().item()), (hc, wc)
        util.assert_close(_n(yb), orc.dwt_inverse(_n(yl), [_n(yh[0])], gf, mode), TOL, 'vs oracle %dx%d' % (hc, wc))


@pytest.mark.parametrize('wave,size',[('db4', 16), ('db4', 32), ('db8', 32), ('db8', 48), ('db2', 8)])
def test_periodization_full_depth_pyramid_down_to_1x1(wave, size):
    """ADVICE r1 (medium): planes smaller than the filter at the deep levels -- the rotation L/2-1 of the
    periodization stores exceeds the plane size, which needs a true modulo.  J = log2(size) for power-of-two
    sizes (down to 1x1 coefficient planes), J = 4 for 48.  The output is pre-filled with NaN by poisoning
    the allocator's block, so a row that is never written cannot pass by luck."""
    torch.manual_seed(43)
    J = int(np.log2(size)) if size & (size - 1) == 0 else 4
    f = pw.DWTForward(J=J, wave=wave, mode='periodization').to(DEV)
    g = pw.DWTInverse(wave=wave, mode='periodization').to(DEV)
    x = torch.randn(2, 3, size, size, device=DEV)
    yl, yh = f(x)
    hf = [_n(b) for b in (f.h0_col, f.h1_col, f.h0_row, f.h1_row)]
    oyl, oyh = orc.dwt_forward(_n(x), hf, J, 'periodization')
    assert np.array_equal(_n(yl), oyl)
    for a, b in zip(yh, oyh):
        assert np.array_equal(_n(a), b)
    for _ in range(3):   # poison recently freed blocks so unwritten outputs show up as NaN
        junk = torch.full((2, 3, size, size), float('nan'), device=DEV)
        del junk
    y = g((yl, yh))
    assert torch.isfinite(y).all(), 'periodization synthesis left output rows / columns unwritten'
    gf = [_n(b) for b in (g.g0_col, g.g1_col, g.g0_row, g.g1_row)]
    oy = orc.dwt_inverse(oyl, oyh, gf, 'periodization')
    util.assert_close(_n(y), oy, TOL, 'vs oracle')
    assert (y - x).abs().max().item() < 1e-4
