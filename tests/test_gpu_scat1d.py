"""GPU: the 1-D scattering levels (the scattering epilogue of csrc/dtcwt1d.cu, k_scat1d) and ScatLayer1D /
ScatLayer1Dj2.

  * every epilogue instantiation (and a runtime-length tuple), both level-1 modes, the pooled and the full-length
    level-1 low-pass, with and without derivatives, float32 and float64, across segment boundaries, n below the filter
    length, both CTA shapes and the switch point between them, written into slots of a larger output: bit-identical to
    the GPU composition (the 1-D level kernels and torch pointwise ops) and to the oracle composition;
  * a row pitch larger than n and channel-slice views; magbias 0 (NaN from 0 / 0) and denormal squares;
  * canaries and a profiler trace (in a child process) once per instantiation;
  * the modules against the oracle for every table pair, the j1 gradient against the hand-built adjoint, gradcheck.
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import pytorch_wavelets_b200 as pw
from pytorch_wavelets_b200.dtcwt import transform1d as t1
from pytorch_wavelets_b200.scatternet import scat1d as s1
from tests import oracle_scat1d as os1
from tests import sweep_util, util
from tests.test_gpu_dtcwt1d import J1_PAIRS, J2_LENGTHS, J2_SETS, L1_SETS, N_FWD2, N_J1, _banks

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIORTS = ['near_sym_a', 'antonini', 'legall', 'near_sym_b']
QSHIFTS = ['qshift_06', 'qshift_a', 'qshift_b', 'qshift_c', 'qshift_d', 'qshift_32']
FWD1, FWD2 = 0, 1


def predicted_kernel(kind, n, L0, L1, dtype, der):
    """Name of the kernel the scattering dispatch launches (csrc/dtcwt1d.cu launch_kind with the epilogue)."""
    esz = 8 if dtype == torch.float64 else 4
    vec = 16 // esz
    ipu = 2 if kind == FWD1 else 4
    units = n // ipu
    halo = max(L0, L1) // 2 if kind == FWD1 else L0
    srow = (units * ipu + 2 * halo + 2 * vec - 1) // vec * vec
    packed = min((2048 // ipu) // units, 48 * 1024 // (srow * esz)) >= 2
    if kind == FWD1:
        la, lb = (L0, L1) if (L0, L1) in J1_PAIRS else (0, 0)
    else:
        la, lb = (L0 if L0 in J2_LENGTHS else 0), 0
    return 'k_scat1d<%s, %d, %d, %d, %s, %d>' % ('double' if esz == 8 else 'float', kind, la, lb,
                                                 'true' if packed else 'false', 2 if der else 1)


def _rows(n, rows, dtype, seed, scale=None):
    """(N, C, n), one power of ten per row (or all rows times `scale`), as CUDA tensor and numpy of that dtype."""
    rng = np.random.RandomState(seed)
    N, C = (rows, 1) if rows < 4 else (2, rows // 2)
    if scale is None:
        x, _ = util.scaled_uniform((N, C, n), rng)
        x = x.astype(np.float64 if dtype == torch.float64 else np.float32)
    else:
        x = (rng.uniform(-1, 1, (N, C, n)) * scale).astype(np.float64 if dtype == torch.float64 else np.float32)
    return torch.from_numpy(x).to(DEV), x


def _rowcount(n):
    return 4096 if n <= 16 else (64 if n <= 1100 else 3)


def torch_mag(hi, bias):
    """The torch composition the epilogue replaces: (sqrt(re**2 + im**2 + b**2) - b, re / r, im / r)."""
    re, im = hi[..., 0::2], hi[..., 1::2]
    r = torch.sqrt(re ** 2 + im ** 2 + bias ** 2)
    return r - bias, re / r, im / r


def _same(a, b):
    """Bit-identical (NaNs equal); b a tensor or a numpy array."""
    a = a.detach().cpu().numpy()
    b = b.detach().cpu().numpy() if isinstance(b, torch.Tensor) else b
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a, b, equal_nan=True)


def _check_j1(x, xn, h0, h1, mode, bias, pool, der, S=3):
    """One level-1 epilogue call into slots 2 and 0 of a NaN-filled (N, S, C, m) output, against both compositions."""
    N, C, n = x.shape
    m = 1 if mode == 'symmetric' else 0
    Z = torch.full((N, S, C, n // 2), float('nan'), device=DEV, dtype=x.dtype)
    lo = Z[:, 2] if pool else torch.full((N, C, n), float('nan'), device=DEV, dtype=x.dtype)
    dre, dim = s1.fwd_j1(x, h0, h1, m, bias, lo, Z[:, 0], der)
    assert torch.isnan(Z[:, 1]).all()
    glo, ghi = t1.fwd_j1(x, h0, h1, False, m)
    gm, gre, gim = torch_mag(ghi, bias)
    assert _same(lo, F.avg_pool1d(glo, 2) if pool else glo) and _same(Z[:, 0], gm)
    npdt = xn.dtype
    olo, ohi = os1.o1.fwd_j1(xn, h0.astype(npdt), h1.astype(npdt), mode)
    om, ore, oim = os1.mag(ohi, bias)
    assert _same(lo, os1.pool(olo) if pool else olo) and _same(Z[:, 0], om)
    if der:
        assert _same(dre, gre) and _same(dim, gim) and _same(dre, ore) and _same(dim, oim)
    else:
        assert dre is None and dim is None


def _check_j2(x, xn, qs, bias, der, S=3):
    N, C, n = x.shape
    h0a, h0b, h1a, h1b = qs
    Z = torch.full((N, S, C, n // 4), float('nan'), device=DEV, dtype=x.dtype)
    dre, dim = s1.fwd_j2plus(x, h0a, h1a, h0b, h1b, bias, Z[:, 0], Z[:, 2], der)
    assert torch.isnan(Z[:, 1]).all()
    glo, ghi = t1.fwd_j2plus(x, h0a, h1a, h0b, h1b, False)
    gm, gre, gim = torch_mag(ghi, bias)
    assert _same(Z[:, 0], F.avg_pool1d(glo, 2)) and _same(Z[:, 2], gm)
    c = [t.astype(xn.dtype) for t in (h0a, h1a, h0b, h1b)]
    olo, ohi = os1.o1.fwd_j2plus(xn, *c)
    om, ore, oim = os1.mag(ohi, bias)
    assert _same(Z[:, 0], os1.pool(olo)) and _same(Z[:, 2], om)
    if der:
        assert _same(dre, gre) and _same(dim, gim) and _same(dre, ore) and _same(dim, oim)


# ---- level 1 ------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('mode', ['symmetric', 'zero'])
@pytest.mark.parametrize('name,taps', L1_SETS, ids=[s[0] for s in L1_SETS])
def test_level1_bit_identical(name, taps, mode, dtype):
    h0, h1 = taps
    for n in N_J1:
        x, xn = _rows(n, _rowcount(n), dtype, n)
        for pool, der in ((True, False), (True, True), (False, True), (False, False)):
            _check_j1(x, xn, h0, h1, mode, 1e-2, pool, der)


# ---- level 2 ------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('name,qs,iqs', J2_SETS, ids=[s[0] for s in J2_SETS])
def test_level2_bit_identical(name, qs, iqs, dtype):
    for n in N_FWD2:
        x, xn = _rows(n, _rowcount(n), dtype, n)
        for der in (False, True):
            _check_j2(x, xn, qs, 1e-2, der)


# ---- layouts, magbias 0, denormal squares -------------------------------------------------------------------------------

def test_strided_inputs():
    l1, qs, _, _ = _banks()
    base = torch.randn(3, 5, 300, device=DEV)
    for x in (base[:, :, 7:7 + 256], base[:, 1:4, :256], base[1:2, 1:4, 10:266]):
        xn = x.cpu().numpy()
        _check_j1(x, xn, *l1, 'symmetric', 1e-2, True, True)
        _check_j1(x, xn, *l1, 'zero', 1e-2, False, True)
        _check_j2(x, xn, qs, 1e-2, True)


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
def test_zero_bias_and_denormal_squares(dtype):
    """magbias 0 gives 0 / 0 = NaN derivatives at zero band-pass pairs (all-zero rows); inputs near the square root
    of the smallest normal make the squares denormal."""
    l1, qs, _, _ = _banks()
    tiny = 1e-21 if dtype == torch.float32 else 1e-158
    for scale in (tiny, 1.0):
        for n in (64, 2050):
            x, xn = _rows(n, 6, dtype, n, scale=scale)
            x[:, 0] = 0
            xn[:, 0] = 0
            for bias in (0.0, 1e-2, tiny):
                _check_j1(x, xn, *l1, 'symmetric', bias, True, True)
                if n % 4 == 0:
                    _check_j2(x, xn, qs, bias, True)
    x = torch.zeros(1, 1, 16, device=DEV, dtype=dtype)
    dre, _ = s1.fwd_j1(x, *l1, 1, 0.0, torch.empty(1, 1, 8, device=DEV, dtype=dtype),
                       torch.empty(1, 1, 8, device=DEV, dtype=dtype), True)
    assert torch.isnan(dre).all()


# ---- canaries and traces, once per instantiation ------------------------------------------------------------------------

def _nan_like(shape, dtype):
    full = torch.full((int(np.prod(shape)) + 64,), float('nan'), device=DEV, dtype=dtype)
    return full, full[:int(np.prod(shape))].view(shape)


def _abi_calls(dtype):
    """Every epilogue instantiation once, packed and long rows, with and without derivatives, as C-ABI calls into
    NaN-filled canaried buffers: [(call, predicted kernel, [(full buffer, output view)])] and inputs to keep alive."""
    from pytorch_wavelets_b200 import _ffi
    lib = _ffi.lib()
    sfx = '_f64' if dtype == torch.float64 else ''
    stream = _ffi.stream_of(torch.empty(1, device=DEV))
    N, C = 2, 3
    calls, keep = [], []

    def outputs(m_lo, m, der):
        bufs = [_nan_like((N, C, m_lo), dtype), _nan_like((N, C, m), dtype)]
        bufs += [_nan_like((N, C, m), dtype) for _ in range(2)] if der else []
        args = []
        for k in range(4):
            args += [bufs[k][1].data_ptr(), C * (m_lo if k == 0 else m)] if k < len(bufs) else [None, 0]
        return bufs, args

    for n in (64, 2050):
        x = torch.randn(N, C, n, device=DEV, dtype=dtype)
        keep.append(x)
        for _, (h0, h1) in L1_SETS:
            f0, f1 = _ffi.host_taps(h0), _ffi.host_taps(h1)
            for der in (False, True):
                pool = der                       # both low-pass forms across the set
                bufs, a = outputs(n // 2 if pool else n, n // 2, der)
                args = [x.data_ptr(), n, N, C, n] + a[:2] + [int(pool)] + a[2:] + [
                    f0.p(dtype), f0.n, f1.p(dtype), f1.n, 1, 1e-2, stream]
                fn = getattr(lib, 'b200w_scat1d_j1' + sfx)
                calls.append(((lambda fn=fn, args=args: _ffi.check(fn(*args), 'scat1d_j1')),
                              predicted_kernel(FWD1, n, f0.n, f1.n, dtype, der), bufs))
    for n in (1024, 4100):
        x = torch.randn(N, C, n, device=DEV, dtype=dtype)
        keep.append(x)
        for _, qs, _ in J2_SETS:
            f = [_ffi.host_taps(t) for t in qs]       # (h0a, h0b, h1a, h1b)
            for der in (False, True):
                bufs, a = outputs(n // 4, n // 4, der)
                args = [x.data_ptr(), n, N, C, n] + a + [f[0].p(dtype), f[2].p(dtype), f[1].p(dtype), f[3].p(dtype),
                                                         f[0].n, 1e-2, stream]
                fn = getattr(lib, 'b200w_scat1d_j2plus' + sfx)
                calls.append(((lambda fn=fn, args=args: _ffi.check(fn(*args), 'scat1d_j2plus')),
                              predicted_kernel(FWD2, n, f[0].n, f[0].n, dtype, der), bufs))
    return calls, keep


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
def test_canaries(dtype):
    """Each call wrote every element of each output it was given and nothing past it."""
    calls, _ = _abi_calls(dtype)
    for c, _, _ in calls:
        c()
    torch.cuda.synchronize()
    for _, want, bufs in calls:
        for full, out in bufs:
            assert torch.isnan(full[out.numel():]).all(), want
            assert not torch.isnan(out).any(), want


def trace_in_this_process(dtype_name):
    """(kernels traced, kernels predicted) for _abi_calls and for a no-grad and a grad module forward."""
    calls, _ = _abi_calls(getattr(torch, dtype_name))
    x = torch.randn(2, 3, 256, device=DEV, dtype=getattr(torch, dtype_name))
    m1, m2 = pw.ScatLayer1D().to(DEV, x.dtype), pw.ScatLayer1Dj2().to(DEV, x.dtype)
    xg = x.clone().requires_grad_(True)

    def run():
        for c, _, _ in calls:
            c()
        m1(x)
        m2(x)
        with torch.no_grad():
            m1(xg)
        m1(xg)
        m2(xg)
    ks = sweep_util.traced_kernels(run, lambda name: name[name.index('k_scat1d<'):name.index('>') + 1]
                                   if 'k_scat1d<' in name else None)
    dt = x.dtype
    j1 = lambda n, der: predicted_kernel(FWD1, n, 5, 7, dt, der)   # noqa: E731
    j2 = lambda n, der: predicted_kernel(FWD2, n, 10, 10, dt, der)   # noqa: E731
    want = [w for _, w, _ in calls] + [j1(256, False), j1(256, False), j2(256, False), j1(128, False),
                                       j1(256, False), j1(256, True), j1(256, True), j2(256, True), j1(128, True)]
    return ks, want


@pytest.mark.parametrize('dtype', ['float32', 'float64'])
def test_trace_shows_the_predicted_kernels(dtype):
    """Each call launched the kernel the dispatch predicts; forwards without a gradient run the derivative-free
    instantiation.  The profiler session runs in a child process, so it leaves the CUDA activity tracing of this test
    process as the other trace tests expect it."""
    code = ('import json, sys; from tests import test_gpu_scat1d as t; '
            'print(json.dumps(t.trace_in_this_process(sys.argv[1])))')
    r = subprocess.run([sys.executable, '-c', code, dtype], cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    ks, want = json.loads(r.stdout.strip().splitlines()[-1])
    if ks is None:
        pytest.skip('no CUDA activity trace on this machine')
    assert ks == want


# ---- modules ------------------------------------------------------------------------------------------------------------

def _taps(m):
    n = lambda t: t.detach().cpu().numpy().ravel()   # noqa: E731
    return (n(m.h0o), n(m.h1o)), tuple(n(getattr(m, k)) for k in ('h0a', 'h0b', 'h1a', 'h1b'))


@pytest.mark.parametrize('biort', BIORTS)
@pytest.mark.parametrize('qshift', QSHIFTS)
def test_modules_match_oracle(biort, qshift):
    for dtype in (torch.float32, torch.float64):
        m1 = pw.ScatLayer1D(biort=biort).to(DEV, dtype)
        m2 = pw.ScatLayer1Dj2(biort=biort, qshift=qshift).to(DEV, dtype)
        l1, qs = _taps(m2)
        for n in (8, 13, 30, 203, 1000, 2101):
            x = torch.randn(2, 3, n, device=DEV, dtype=dtype)
            xn = x.cpu().numpy()
            assert _same(m1(x), os1.scat_layer1d(xn, l1))
            assert _same(m2(x), os1.scat_layer1d_j2(xn, l1, qs))
            # the GPU composition of ScatLayer1Dj2 from the level functions and torch ops
            xp = torch.from_numpy(os1.pad_j2(xn)).to(DEV)
            lo1, hi1 = t1.fwd_j1(xp, m2.h0o, m2.h1o, False, 1)
            U1 = torch_mag(hi1, 1e-2)[0]
            lo2, hi2 = t1.fwd_j2plus(lo1, m2.h0a, m2.h1a, m2.h0b, m2.h1b, False)
            u, hu = t1.fwd_j1(U1, m2.h0o, m2.h1o, False, 1)
            Z = torch.stack((F.avg_pool1d(lo2, 2), F.avg_pool1d(u, 2), torch_mag(hi2, 1e-2)[0],
                             torch_mag(hu, 1e-2)[0]), dim=1)
            assert _same(m2(x), Z.reshape(2, 12, -1))
    assert _same(pw.ScatLayer1D(biort=biort, mode='zero').to(DEV)(x.float()),
                 os1.scat_layer1d(x.float().cpu().numpy(), l1, 'zero'))


def test_j1_gradient_is_the_adjoint_kernel():
    for mode in ('symmetric', 'zero'):
        m = pw.ScatLayer1D(mode=mode).to(DEV)
        x = torch.randn(2, 3, 200, device=DEV, requires_grad=True)
        Z = m(x)
        dZ = torch.randn_like(Z)
        (dx,) = torch.autograd.grad(Z, (x,), dZ)
        mi = 1 if mode == 'symmetric' else 0
        _, hi = t1.fwd_j1(x.detach(), m.h0o, m.h1o, False, mi)
        _, dre, dim = torch_mag(hi, 1e-2)
        d = dZ.view(2, 2, 3, 100)
        lo = (d[:, 0] * 0.5).repeat_interleave(2, dim=-1)
        band = torch.stack((d[:, 1] * dre, d[:, 1] * dim), dim=-1).reshape(2, 3, 200)
        assert torch.equal(dx, t1.inv_j1(lo, band, m.h0o, m.h1o, mi))


def test_j2_gradient_matches_oracle():
    m = pw.ScatLayer1Dj2().to(DEV, torch.float64)
    l1, qs = _taps(m)
    x = torch.randn(2, 3, 96, device=DEV, dtype=torch.float64, requires_grad=True)
    Z = m(x)
    dZ = torch.randn_like(Z)
    (dx,) = torch.autograd.grad(Z, (x,), dZ)
    _, ders = os1.scat1d_j2(x.detach().cpu().numpy(), l1, qs)
    want = os1.backward_j2(dZ.view(2, 4, 3, 24).cpu().numpy(), ders, l1, qs)
    assert np.abs(dx.cpu().numpy() - want).max() <= 1e-13 * np.abs(want).max()


@pytest.mark.parametrize('mode', ['symmetric', 'zero'])
def test_gradcheck(mode):
    m1 = pw.ScatLayer1D(mode=mode).to(DEV, torch.float64)
    x = torch.randn(1, 2, 22, device=DEV, dtype=torch.float64, requires_grad=True)
    assert torch.autograd.gradcheck(m1, (x,))
    if mode == 'symmetric':
        m2 = pw.ScatLayer1Dj2(magbias=0.1).to(DEV, torch.float64)
        x = torch.randn(1, 2, 40, device=DEV, dtype=torch.float64, requires_grad=True)
        assert torch.autograd.gradcheck(m2, (x,))


def test_no_grad_forward_saves_nothing():
    m = pw.ScatLayer1Dj2().to(DEV)
    x = torch.randn(2, 3, 64, device=DEV, requires_grad=True)
    with torch.no_grad():
        z0 = m(x)
    assert not z0.requires_grad
    assert torch.equal(z0, m(x).detach())
