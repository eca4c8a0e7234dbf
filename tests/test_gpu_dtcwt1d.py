"""GPU: the 1-D DTCWT level kernels (csrc/dtcwt1d.cu) and modules.

  * every kernel instantiation (and a runtime-length tuple), both level-1 modes, through the level functions, across
    segment boundaries, n below the filter length, both CTA shapes and the switch point between them, a row pitch
    larger than n and a channel-slice view: bit-identical to the oracle composition (float32 and float64) and to the
    GPU-primitive composition;
  * the inverses with a missing low-pass or band-pass; canaries and a profiler trace (in a child process) once per
    instantiation;
  * the modules (J = 1 ... 5, skip_hps, include_scale, odd n, trimming), perfect reconstruction, and gradcheck.
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import pytorch_wavelets_b200 as pw
from pytorch_wavelets_b200.dtcwt import lowlevel as ll
from pytorch_wavelets_b200.dtcwt import transform1d as t1
from tests import oracle_dtcwt1d as o1
from tests import sweep_util, util

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIORTS = ['near_sym_a', 'antonini', 'legall', 'near_sym_b']
QSHIFTS = ['qshift_a', 'qshift_b', 'qshift_c', 'qshift_d', 'qshift_32']
FWD1, FWD2, INV1, INV2 = 0, 1, 2, 3
IPU = {FWD1: 1, FWD2: 4, INV1: 1, INV2: 2}
NIN = {FWD1: 1, FWD2: 1, INV1: 2, INV2: 2}
J1_PAIRS = {(5, 7), (7, 5), (9, 7), (7, 9), (5, 3), (3, 5), (13, 19), (19, 13)}
J2_LENGTHS = {10, 14, 16, 18, 32}
# level-1 / inverse-level-1 lengths n (one unit = one sample, 2048 units per long-row segment, packed up to 1024)
N_J1 = [2, 4, 6, 10, 64, 1022, 1024, 1026, 2048, 2050, 3 * 2048 + 100]
# forward j >= 2 input lengths (one unit = 4 samples, 512 units per segment, packed up to n = 1024)
N_FWD2 = [4, 8, 12, 16, 256, 1024, 1028, 2048, 2052, 3 * 2048 + 400]
# inverse j >= 2 output lengths (one unit = 4 outputs, 1024 units per segment, packed up to n = 2048)
N_INV2 = [4, 8, 12, 16, 256, 2048, 2052, 4096, 4100, 3 * 4096 + 400]


def _np(t):
    return t.detach().cpu().numpy().ravel()


def _banks(biort='near_sym_a', qshift='qshift_a'):
    f = pw.DTCWT1DForward(biort=biort, qshift=qshift)
    i = pw.DTCWT1DInverse(biort=biort, qshift=qshift)
    return ((_np(f.h0o), _np(f.h1o)), tuple(_np(getattr(f, k)) for k in ('h0a', 'h0b', 'h1a', 'h1b')),
            (_np(i.g0o), _np(i.g1o)), tuple(_np(getattr(i, k)) for k in ('g0a', 'g0b', 'g1a', 'g1b')))


def predicted_kernel(kind, n, L0, L1, dtype):
    """Name of the kernel the dispatch launches (csrc/dtcwt1d.cu launch_kind / dispatch_j1 / dispatch_j2)."""
    esz = 8 if dtype == torch.float64 else 4
    vec = 16 // esz
    units = n if kind in (FWD1, INV1) else n // 4
    halo = max(L0, L1) // 2 if kind in (FWD1, INV1) else (L0 if kind == FWD2 else L0 // 2 + 2)
    seg = 2048 // IPU[kind]
    srow = (units * IPU[kind] + 2 * halo + 2 * vec - 1) // vec * vec
    packed = min(seg // units, 48 * 1024 // (NIN[kind] * srow * esz)) >= 2
    if kind in (FWD1, INV1):
        la, lb = (L0, L1) if (L0, L1) in J1_PAIRS else (0, 0)
    else:
        la, lb = (L0 if L0 in J2_LENGTHS else 0), 0
    return 'k_dt1d<%s, %d, %d, %d, %s>' % ('double' if esz == 8 else 'float', kind, la, lb,
                                           'true' if packed else 'false')


def _traced(fn):
    return sweep_util.traced_kernels(fn, lambda name: name[name.index('k_dt1d<'):name.index('>') + 1]
                                     if 'k_dt1d<' in name else None)


def _rows(n, rows, dtype, seed):
    """(N, C, n) with one power of ten per row, as a CUDA tensor of the given dtype and as numpy of that dtype."""
    rng = np.random.RandomState(seed)
    N, C = (rows, 1) if rows < 4 else (2, rows // 2)
    x, _ = util.scaled_uniform((N, C, n), rng)
    x = x.astype(np.float64 if dtype == torch.float64 else np.float32)
    return torch.from_numpy(x).to(DEV), x


def _rowcount(n):
    return 4096 if n <= 16 else (64 if n <= 1100 else 3)


def _nan_like(shape, dtype):
    """NaN-filled buffer with a NaN canary region after it; returns (full, view of shape)."""
    full = torch.full((int(np.prod(shape)) + 64,), float('nan'), device=DEV, dtype=dtype)
    return full, full[:int(np.prod(shape))].view(shape)


def _l1_sets():
    """(name, forward-role taps) for every level-1 instantiation plus a runtime-length tuple."""
    out = []
    for b in BIORTS:
        l1, _, il1, _ = _banks(b)
        out += [(b + '-analysis', l1), (b + '-synthesis', il1)]
    rng = np.random.RandomState(3)
    out.append(('runtime-11-9', (rng.randn(11), rng.randn(9))))
    return out


def _j2_sets():
    out = []
    for q in QSHIFTS:
        _, qs, _, iqs = _banks('near_sym_a', q)
        out.append((q, qs, iqs))
    rng = np.random.RandomState(4)
    r = tuple(rng.randn(12) for _ in range(4))
    out.append(('runtime-12', r, r))
    return out


L1_SETS = _l1_sets()
J2_SETS = _j2_sets()


# ---- level 1 ------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('mode', ['symmetric', 'zero'])
@pytest.mark.parametrize('name,taps', L1_SETS, ids=[s[0] for s in L1_SETS])
def test_level1_bit_identical(name, taps, mode, dtype):
    h0, h1 = taps
    m = 1 if mode == 'symmetric' else 0
    npdt = np.float64 if dtype == torch.float64 else np.float32
    h0c, h1c = h0.astype(npdt), h1.astype(npdt)
    for n in N_J1:
        x, xn = _rows(n, _rowcount(n), dtype, n)
        lo, hi = t1.fwd_j1(x, h0, h1, False, m)
        olo, ohi = o1.fwd_j1(xn, h0c, h1c, mode)
        assert np.array_equal(lo.cpu().numpy(), olo) and np.array_equal(hi.cpu().numpy(), ohi), n
        y = t1.inv_j1(lo, hi, h0, h1, m)
        oy = o1.inv_j1(olo, ohi, h0c, h1c, mode)
        assert np.array_equal(y.cpu().numpy(), oy), n
        assert np.array_equal(t1.inv_j1(None, hi, h0, h1, m).cpu().numpy(), o1.inv_j1(None, ohi, h0c, h1c, mode))
        assert np.array_equal(t1.inv_j1(lo, None, h0, h1, m).cpu().numpy(), o1.inv_j1(olo, None, h0c, h1c, mode))
        if dtype == torch.float32:    # the GPU-primitive composition
            x4 = x[:, :, None, :]
            assert torch.equal(lo, ll.rowfilter(x4, h0, mode)[:, :, 0]) and torch.equal(hi, ll.rowfilter(x4, h1, mode)[:, :, 0])
            py = ll.rowfilter(lo[:, :, None], h0, mode) + ll.rowfilter(hi[:, :, None], h1, mode)
            assert torch.equal(y, py[:, :, 0])
        # skipped band-pass: the low-pass alone
        lo2, hi2 = t1.fwd_j1(x, h0, h1, True, m)
        assert hi2 is None and torch.equal(lo2, lo)


# ---- levels >= 2 --------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('name,qs,iqs', J2_SETS, ids=[s[0] for s in J2_SETS])
def test_level2plus_bit_identical(name, qs, iqs, dtype):
    h0a, h0b, h1a, h1b = qs
    g0a, g0b, g1a, g1b = iqs
    npdt = np.float64 if dtype == torch.float64 else np.float32
    c = [t.astype(npdt) for t in (h0a, h1a, h0b, h1b, g0a, g1a, g0b, g1b)]
    for n in N_FWD2:
        x, xn = _rows(n, _rowcount(n), dtype, n)
        lo, hi = t1.fwd_j2plus(x, h0a, h1a, h0b, h1b, False)
        olo, ohi = o1.fwd_j2plus(xn, *c[:4])
        assert np.array_equal(lo.cpu().numpy(), olo) and np.array_equal(hi.cpu().numpy(), ohi), n
        if dtype == torch.float32:
            x4 = x[:, :, None, :]
            assert torch.equal(lo, ll.rowdfilt(x4, h0b, h0a)[:, :, 0])
            assert torch.equal(hi, ll.rowdfilt(x4, h1b, h1a, highpass=True)[:, :, 0])
    for n in N_INV2:
        k = n // 2
        lo, lon = _rows(k, _rowcount(n), dtype, n + 1)
        hi, hin = _rows(k, _rowcount(n), dtype, n + 2)
        y = t1.inv_j2plus(lo, hi, g0a, g1a, g0b, g1b)
        assert np.array_equal(y.cpu().numpy(), o1.inv_j2plus(lon, hin, *c[4:])), n
        assert np.array_equal(t1.inv_j2plus(None, hi, g0a, g1a, g0b, g1b).cpu().numpy(),
                              o1.inv_j2plus(None, hin, *c[4:]))
        assert np.array_equal(t1.inv_j2plus(lo, None, g0a, g1a, g0b, g1b).cpu().numpy(),
                              o1.inv_j2plus(lon, None, *c[4:]))
        if dtype == torch.float32:
            py = ll.rowifilt(lo[:, :, None], g0b, g0a) + ll.rowifilt(hi[:, :, None], g1b, g1a, highpass=True)
            assert torch.equal(y, py[:, :, 0])


# ---- layouts: a row pitch larger than n, a channel slice ----------------------------------------------------------------

def test_strided_inputs():
    l1, qs, il1, iqs = _banks()
    h0a, h0b, h1a, h1b = qs
    base = torch.randn(3, 5, 300, device=DEV)
    for x in (base[:, :, 7:7 + 256], base[:, 1:4, :256], base[1:2, 1:4, 10:266]):
        xc = x.contiguous()
        for a, b in zip(t1.fwd_j1(x, *l1, False, 1), t1.fwd_j1(xc, *l1, False, 1)):
            assert torch.equal(a, b)
        for a, b in zip(t1.fwd_j2plus(x, h0a, h1a, h0b, h1b, False), t1.fwd_j2plus(xc, h0a, h1a, h0b, h1b, False)):
            assert torch.equal(a, b)
        hi = torch.randn(xc.shape, device=DEV)
        assert torch.equal(t1.inv_j1(x, hi, *il1, 1), t1.inv_j1(xc, hi, *il1, 1))
        assert torch.equal(t1.inv_j2plus(x, hi, *iqs), t1.inv_j2plus(xc, hi, *iqs))


# ---- canaries and traces, once per instantiation ------------------------------------------------------------------------

def _abi_calls(dtype):
    """Every instantiation once, packed and long rows, as C-ABI calls into NaN-filled canaried buffers:
    [(call, predicted kernel, [(full buffer, output view, written)])] and the inputs to keep alive."""
    from pytorch_wavelets_b200 import _ffi
    lib = _ffi.lib()
    sfx = '_f64' if dtype == torch.float64 else ''
    stream = _ffi.stream_of(torch.empty(1, device=DEV))
    rows = 6
    calls, keep = [], []

    def add(fn, args, want, nout, two_outputs):
        full0, out0 = _nan_like((rows, nout), dtype)
        full1, out1 = _nan_like((rows, nout), dtype)
        a = [out0.data_ptr() if v == 'out0' else (out1.data_ptr() if v == 'out1' else v) for v in args]
        calls.append((lambda: _ffi.check(fn(*a), 'dtcwt1d'), want, [(full0, out0, True), (full1, out1, two_outputs)]))

    for n in (64, 2050):                         # packed and long rows
        x = torch.randn(rows, n, device=DEV, dtype=dtype)
        keep.append(x)
        for _, (h0, h1) in L1_SETS:
            f0, f1 = _ffi.host_taps(h0), _ffi.host_taps(h1)
            t = [f0.p(dtype), f0.n, f1.p(dtype), f1.n, 1, stream]
            add(getattr(lib, 'b200w_dtcwt1d_fwd_j1' + sfx), [x.data_ptr(), n, rows, n, 'out0', 'out1'] + t,
                predicted_kernel(FWD1, n, f0.n, f1.n, dtype), n, True)
            add(getattr(lib, 'b200w_dtcwt1d_inv_j1' + sfx), [x.data_ptr(), n, x.data_ptr(), rows, n, 'out0'] + t,
                predicted_kernel(INV1, n, f0.n, f1.n, dtype), n, False)
    for n in (1024, 4100):                       # packed and long rows
        x = torch.randn(rows, n, device=DEV, dtype=dtype)
        h = torch.randn(rows, n // 2, device=DEV, dtype=dtype)
        keep += [x, h]
        for _, qs, _ in J2_SETS:
            f = [_ffi.host_taps(t) for t in qs]
            t = [v.p(dtype) for v in f] + [f[0].n, stream]
            add(getattr(lib, 'b200w_dtcwt1d_fwd_j2plus' + sfx), [x.data_ptr(), n, rows, n, 'out0', 'out1'] + t,
                predicted_kernel(FWD2, n, f[0].n, f[0].n, dtype), n // 2, True)
            add(getattr(lib, 'b200w_dtcwt1d_inv_j2plus' + sfx),
                [h.data_ptr(), n // 2, h.data_ptr(), rows, n, 'out0'] + t,
                predicted_kernel(INV2, n, f[0].n, f[0].n, dtype), n, False)
    assert len(calls) == 2 * 2 * len(L1_SETS) + 2 * 2 * len(J2_SETS)
    return calls, keep


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
def test_canaries(dtype):
    """Each call wrote every output it owns and nothing past it (the inverses leave the second buffer untouched)."""
    calls, _ = _abi_calls(dtype)
    for c, _, _ in calls:
        c()
    torch.cuda.synchronize()
    for _, want, bufs in calls:
        for full, out, written in bufs:
            assert torch.isnan(full[out.numel():]).all(), want
            assert (not torch.isnan(out).any()) if written else torch.isnan(out).all(), want


def trace_in_this_process(dtype_name):
    """(kernels traced, kernels predicted) for every call of _abi_calls, under one torch.profiler session."""
    calls, _ = _abi_calls(getattr(torch, dtype_name))
    ks = _traced(lambda: [c() for c, _, _ in calls])
    return ks, [w for _, w, _ in calls]


@pytest.mark.parametrize('dtype', ['float32', 'float64'])
def test_trace_shows_the_predicted_kernels(dtype):
    """Each call launched the kernel the dispatch predicts.  The profiler session runs in a child process, so it leaves
    the CUDA activity tracing of this test process exactly as the other trace tests expect it."""
    code = ('import json, sys; from tests import test_gpu_dtcwt1d as t; '
            'print(json.dumps(t.trace_in_this_process(sys.argv[1])))')
    r = subprocess.run([sys.executable, '-c', code, dtype], cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    ks, want = json.loads(r.stdout.strip().splitlines()[-1])
    if ks is None:
        pytest.skip('no CUDA activity trace on this machine')
    assert ks == want


# ---- modules ------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('biort,qshift', [('near_sym_a', 'qshift_a'), ('near_sym_b', 'qshift_b'),
                                          ('antonini', 'qshift_c'), ('legall', 'qshift_d'),
                                          ('near_sym_a', 'qshift_32')])
@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
def test_modules_match_oracle_and_reconstruct(biort, qshift, dtype):
    prev = torch.get_default_dtype()
    torch.set_default_dtype(dtype)      # float64 modules hold float64 taps
    try:
        l1, qs, il1, iqs = _banks(biort, qshift)
        fs = {J: pw.DTCWT1DForward(biort=biort, qshift=qshift, J=J).to(DEV) for J in range(1, 6)}
        i = pw.DTCWT1DInverse(biort=biort, qshift=qshift).to(DEV)
    finally:
        torch.set_default_dtype(prev)
    tol = (1e-8 if qshift == 'qshift_32' else 1e-10) if dtype == torch.float64 else 1e-5
    for n, J in ((64, 1), (129, 2), (250, 3), (333, 4), (1001, 5), (30, 5)):
        x = torch.randn(2, 3, n, device=DEV, dtype=dtype)
        yl, yh = fs[J](x)
        oyl, oyh = o1.dtcwt1d_forward(x.cpu().numpy(), l1, qs, J)
        assert np.array_equal(yl.cpu().numpy(), oyl)
        for a, b in zip(yh, oyh):
            assert a.shape == b.shape and np.array_equal(a.cpu().numpy(), b)
        y = i((yl, yh))
        assert np.array_equal(y.cpu().numpy(), o1.dtcwt1d_inverse(oyl, oyh, il1, iqs))
        assert (y[:, :, :n] - x).abs().max().item() <= tol * x.abs().max().item(), (n, J)


def test_module_options():
    x = torch.randn(2, 2, 200, device=DEV)
    f = pw.DTCWT1D(J=3, skip_hps=[False, True, False]).to(DEV)
    yl, yh = f(x)
    assert yh[1].shape == torch.Size([]) and yh[0].shape == (2, 2, 100, 2) and yh[2].shape[-1] == 2
    scales, yh2 = pw.DTCWT1D(J=3, include_scale=True).to(DEV)(x)
    assert len(scales) == 3 and torch.equal(scales[-1], yl)
    assert [s.shape[-1] for s in scales] == [200, 100, 50]
    # a skipped level reconstructs as if its band-pass were zeros
    i = pw.IDTCWT1D().to(DEV)
    full = pw.DTCWT1D(J=3).to(DEV)(x)
    zeroed = (full[0], [full[1][0], torch.zeros_like(full[1][1]), full[1][2]])
    assert torch.equal(i((yl, yh)), i(zeroed))
    assert torch.equal(i((yl, [None, None, yh[2]])), i((yl, [torch.zeros_like(full[1][0]), None, yh[2]])))


# ---- autograd -----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('mode', ['symmetric', 'zero'])
def test_gradcheck(mode):
    f = pw.DTCWT1DForward(J=2, mode=mode).to(DEV, torch.float64)
    i = pw.DTCWT1DInverse(mode=mode).to(DEV, torch.float64)
    x = torch.randn(1, 2, 22, device=DEV, dtype=torch.float64, requires_grad=True)

    def fwd(x):
        yl, yh = f(x)
        return (yl,) + tuple(yh)
    assert torch.autograd.gradcheck(fwd, (x,))
    yl, yh = f(x.detach())
    args = (yl.clone().requires_grad_(True), yh[0].clone().requires_grad_(True), yh[1].clone().requires_grad_(True))
    assert torch.autograd.gradcheck(lambda a, b, c: i((a, [b, c])), args)


def test_forward_backward_is_the_inverse_kernel():
    l1, qs, _, _ = _banks()
    h0a, h0b, h1a, h1b = qs
    x = torch.randn(2, 3, 64, device=DEV, requires_grad=True)
    lo, yh = t1.FWD1D_J2PLUS.apply(x, h0a, h1a, h0b, h1b, False)
    dl, dh = torch.randn_like(lo), torch.randn_like(yh)
    (dx,) = torch.autograd.grad((lo, yh), (x,), (dl, dh))
    assert torch.equal(dx, t1.inv_j2plus(dl, dh.reshape(2, 3, -1), h0b, h1b, h0a, h1a))
    lo, yh = t1.FWD1D_J1.apply(x, l1[0], l1[1], False, 1)
    dl, dh = torch.randn_like(lo), torch.randn_like(yh)
    (dx,) = torch.autograd.grad((lo, yh), (x,), (dl, dh))
    assert torch.equal(dx, t1.inv_j1(dl, dh.reshape(2, 3, -1), l1[0], l1[1], 1))
