"""float64 on the GPU: the reference computes in torch's default dtype (dwt/lowlevel.py:972, dtcwt/lowlevel.py:67; its
tests run both precisions, tests/test_dwt.py:143-160, tests/test_dtcwt.py:116-135).  Here double-precision modules take
the generic kernels instantiated for double (csrc/b200wave.cu, csrc/dwt1d.cu); they are compared with the float64 oracle at 1e-12."""
import numpy as np
import pytest
import torch

import pytorch_wavelets_b200 as pw
from oracle import oracle as orc
from tests import util

pytestmark = pytest.mark.gpu
DEV = 'cuda'
TOL64 = 1e-12


def _n(t):
    return t.detach().cpu().numpy()


class f64_default(object):
    """Build modules the way the reference's double-precision tests do: with torch's default dtype set to float64, so the
    filter buffers hold double-precision taps (``.double()`` on a float32 module would keep float32-rounded taps)."""

    def __enter__(self):
        self.prev = torch.get_default_dtype()
        torch.set_default_dtype(torch.float64)

    def __exit__(self, *exc):
        torch.set_default_dtype(self.prev)
        return False


@pytest.mark.parametrize('mode', ['zero', 'symmetric', 'reflect', 'periodic', 'periodization'])
@pytest.mark.parametrize('wave,J,shape', [('db4', 3, (2, 3, 128, 96)), ('db2', 2, (1, 2, 63, 50)), ('bior2.4', 2, (1, 2, 80, 72))])
def test_dwt_f64_vs_oracle(wave, J, shape, mode):
    torch.manual_seed(5)
    x = torch.randn(*shape, dtype=torch.float64)
    with f64_default():
        f = pw.DWTForward(J=J, wave=wave, mode=mode)
        i = pw.DWTInverse(wave=wave, mode=mode)
    assert f.h0_col.dtype == torch.float64
    hf = [b.numpy() for b in (f.h0_col, f.h1_col, f.h0_row, f.h1_row)]
    gf = [b.numpy() for b in (i.g0_col, i.g1_col, i.g0_row, i.g1_row)]
    oyl, oyh = orc.dwt_forward(x.numpy(), hf, J, mode)
    f, i = f.to(DEV), i.to(DEV)
    yl, yh = f(x.to(DEV))
    assert yl.dtype == torch.float64 and all(h.dtype == torch.float64 for h in yh)
    util.assert_close(_n(yl), oyl, TOL64, 'yl')
    for j in range(J):
        util.assert_close(_n(yh[j]), oyh[j], TOL64, 'yh%d' % j)
    y = i((yl, yh))
    assert y.dtype == torch.float64
    util.assert_close(_n(y), orc.dwt_inverse(oyl, oyh, gf, mode), TOL64, 'inverse')
    H, W = shape[2:]
    assert np.abs(_n(y)[:, :, :H, :W] - x.numpy()).max() < 1e-10   # double-precision perfect reconstruction


@pytest.mark.parametrize('biort,qshift', [('near_sym_a', 'qshift_a'), ('near_sym_b', 'qshift_b')])
@pytest.mark.parametrize('shape', [(2, 3, 64, 64), (1, 2, 50, 36)])
def test_dtcwt_f64_roundtrip_and_f32_agreement(biort, qshift, shape):
    torch.manual_seed(6)
    x = torch.randn(*shape, dtype=torch.float64, device=DEV)
    with f64_default():
        f64 = pw.DTCWTForward(J=3, biort=biort, qshift=qshift).to(DEV)
        i64 = pw.DTCWTInverse(biort=biort, qshift=qshift).to(DEV)
    yl, yh = f64(x)
    assert yl.dtype == torch.float64 and all(h.dtype == torch.float64 for h in yh)
    y = i64((yl, yh))
    H, W = shape[2:]
    assert float((y[:, :, :H, :W] - x).abs().max()) < 1e-10        # the reference's double-precision PR check
    # the float32 engine (streaming kernels) computes the same transform
    f32 = pw.DTCWTForward(J=3, biort=biort, qshift=qshift).to(DEV)
    zl, zh = f32(x.float())
    util.assert_close(_n(zl), _n(yl), 1e-5, 'yl f32 vs f64')
    for a, b in zip(zh, yh):
        util.assert_close(_n(a), _n(b), 1e-5, 'yh f32 vs f64')


def test_dtcwt_f64_vs_oracle():
    torch.manual_seed(7)
    x = torch.randn(1, 2, 48, 64, dtype=torch.float64)
    with f64_default():
        f = pw.DTCWTForward(J=2)
    lv1 = [b.numpy().ravel() for b in (f.h0o, f.h1o)]
    qs = [b.numpy().ravel() for b in (f.h0a, f.h0b, f.h1a, f.h1b)]   # the oracle's order
    oyl, oyh = orc.dtcwt_forward(x.numpy(), lv1, qs, J=2)
    yl, yh = f.to(DEV)(x.to(DEV))
    util.assert_close(_n(yl), oyl, TOL64, 'yl')
    for j in range(2):
        util.assert_close(_n(yh[j]), oyh[j], TOL64, 'yh%d' % j)


def test_dwt1d_and_scat_f64():
    torch.manual_seed(8)
    x = torch.randn(2, 3, 257, dtype=torch.float64, device=DEV)
    with f64_default():
        f = pw.DWT1DForward(J=3, wave='db4', mode='symmetric').to(DEV)
        i = pw.DWT1DInverse(wave='db4', mode='symmetric').to(DEV)
    yl, yh = f(x)
    assert yl.dtype == torch.float64
    y = i((yl, yh))
    assert float((y[..., :257] - x).abs().max()) < 1e-10
    s = pw.ScatLayer().double().to(DEV)
    xi = torch.randn(2, 3, 32, 32, dtype=torch.float64, device=DEV)
    z = s(xi)
    assert z.dtype == torch.float64
    z32 = pw.ScatLayer().to(DEV)(xi.float())
    util.assert_close(_n(z32), _n(z), 1e-5, 'scat f32 vs f64')


def test_dwt_f64_gradcheck():
    """Autograd through the float64 kernels: torch.autograd.gradcheck (the reference does this for its Functions,
    tests/test_dwt.py:215-299)."""
    f = pw.DWTForward(J=1, wave='db2', mode='zero').double().to(DEV)
    x = torch.randn(1, 1, 8, 10, dtype=torch.float64, device=DEV, requires_grad=True)
    assert torch.autograd.gradcheck(lambda t: f(t)[0], (x,), eps=1e-6, atol=1e-8)
    assert torch.autograd.gradcheck(lambda t: f(t)[1][0], (x,), eps=1e-6, atol=1e-8)
