"""GPU: the DWT's double backward.

* the reference's own second-order values (tests/golden/grad2_*.npz, from tests/golden/make_golden_grad2.py);
* ``gradgradcheck`` of AFB1D / SFB1D / AFB2D / SFB2D / DWTPyramid and of the four modules, every mode, odd sizes,
  planes smaller than the filter;
* the transposed-analysis kernel (b200w_dwt_afb2d_adjoint / _afb1d_adjoint) against the dense restatement in
  tests/oracle_dwt_adjoint.py, float64 and float32, per-plane scales and error bounds, NaN canaries;
* child-process profiler traces: which kernels each route launches, and that a plain first-order ``.backward()``
  launches the raw level calls it always made, bit for bit;
* an R1 gradient-penalty step through DWTForward / DWTInverse against the same graph written as torch ops.
"""
import ctypes
import glob
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import pytorch_wavelets_b200 as pw
from pytorch_wavelets_b200 import _ffi
from pytorch_wavelets_b200.dwt import lowlevel as ll2
from pytorch_wavelets_b200.dwt import transform1d as t1
from tests import oracle_dwt_adjoint as oa
from tests import sweep_util, util

pytestmark = pytest.mark.gpu
DEV = 'cuda'
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODES = oa.MODES


def _unit(dtype):
    return 2.0 ** -24 if dtype == 'float32' else 2.0 ** -53


def _wave_taps(wave):
    w = pw.wavelets.Wavelet(wave) if isinstance(wave, str) else wave
    return np.asarray(w.dec_lo[::-1], np.float64), np.asarray(w.dec_hi[::-1], np.float64), \
        np.asarray(w.rec_lo, np.float64), np.asarray(w.rec_hi, np.float64)


# ---- golden values of the reference -----------------------------------------------------------------------------------

def _module(kind, wave, mode, dtype):
    """The module with its filter buffers built in ``dtype`` (as the reference builds them in the default dtype)."""
    prev = torch.get_default_dtype()
    torch.set_default_dtype(dtype)
    try:
        return _module_in_default_dtype(kind, wave, mode, dtype)
    finally:
        torch.set_default_dtype(prev)


def _module_in_dtype(cls, dtype, **kw):
    prev = torch.get_default_dtype()
    torch.set_default_dtype(dtype)
    try:
        return cls(**kw).to(DEV)
    finally:
        torch.set_default_dtype(prev)


def _module_in_default_dtype(kind, wave, mode, dtype):
    if kind == 'dwt2':
        m = pw.DWTForward(J=2, wave=wave, mode=mode).to(DEV, dtype)
        return lambda xs: (lambda r: [r[0]] + list(r[1]))(m(xs[0]))
    if kind == 'idwt2':
        m = pw.DWTInverse(wave=wave, mode=mode).to(DEV, dtype)
        return lambda xs: [m((xs[0], list(xs[1:])))]
    if kind == 'dwt1':
        m = pw.DWT1DForward(J=2, wave=wave, mode=mode).to(DEV, dtype)
        return lambda xs: (lambda r: [r[0]] + list(r[1]))(m(xs[0]))
    m = pw.DWT1DInverse(wave=wave, mode=mode).to(DEV, dtype)
    return lambda xs: [m((xs[0], list(xs[1:])))]


GOLDEN = sorted(glob.glob(os.path.join(ROOT, 'tests', 'golden', 'grad2_*.npz')))


@pytest.mark.parametrize('dtype,tol', [(torch.float64, 1e-10), (torch.float32, 1e-5)])
@pytest.mark.parametrize('path', GOLDEN, ids=[os.path.basename(p)[6:-4] for p in GOLDEN])
def test_reference_second_order_values(path, dtype, tol):
    d = np.load(path)
    kind, wave, mode = str(d['kind']), str(d['wave']), str(d['mode'])
    nin, nout = int(d['n_in']), int(d['n_out'])
    f = _module(kind, wave, mode, dtype)
    t = lambda a: torch.tensor(a, device=DEV, dtype=dtype)   # noqa: E731
    xs = [t(d['in%d' % i]).requires_grad_(True) for i in range(nin)]
    us = [t(d['u%d' % i]).requires_grad_(True) for i in range(nout)]
    ws = [t(d['w%d' % i]) for i in range(nin)]
    gx = torch.autograd.grad(f(xs), xs, us, create_graph=True)
    ggu = torch.autograd.grad(gx, us, ws)
    s = sum((y ** 2).sum() for y in f(xs))
    g = torch.autograd.grad(s, xs, create_graph=True)
    x2 = torch.autograd.grad(sum((a ** 2).sum() for a in g), xs)
    for name, got in (('gx', gx), ('ggu', ggu), ('x2_', x2)):
        for i, a in enumerate(got):
            ref = d['%s%d' % (name, i)]
            err = np.abs(a.detach().cpu().double().numpy() - ref).max() / max(np.abs(ref).max(), 1e-300)
            assert err < tol, '%s%d: %g' % (name, i, err)


# ---- gradgradcheck ----------------------------------------------------------------------------------------------------

SIZES2 = [(5, 7), (3, 4), (9, 6)]   # odd sizes; 3x4 is smaller than every filter below but db1


def _r(shape, seed):
    g = torch.Generator(device='cpu').manual_seed(seed)
    return torch.randn(*shape, generator=g, dtype=torch.float64).to(DEV)


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('wave', ['db1', 'db3', 'db4'])
def test_gradgradcheck_functions_2d(mode, wave):
    m = ll2.mode_to_int(mode)
    h0, h1, g0, g1 = [torch.tensor(a, dtype=torch.float64) for a in _wave_taps(wave)]
    for k, (H, W) in enumerate(SIZES2):
        x = _r((1, 2, H, W), k).requires_grad_(True)
        assert torch.autograd.gradgradcheck(lambda x: ll2.AFB2D.apply(x, h0, h1, h0, h1, m), (x,))
        assert torch.autograd.gradgradcheck(lambda x: ll2.DWTPyramid.apply(x, h0, h1, h0, h1, m, 2), (x,))
        lo, hi = ll2.afb2d_level(x.detach(), h0, h1, h0, h1, m)
        lo, hi = lo.clone().requires_grad_(True), hi.clone().requires_grad_(True)
        assert torch.autograd.gradgradcheck(lambda a, b: ll2.SFB2D.apply(a, b, g0, g1, g0, g1, m), (lo, hi))
        assert torch.autograd.gradgradcheck(lambda a: ll2.SFB2D.apply(a, None, g0, g1, g0, g1, m), (lo,))


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('wave', ['db1', 'db3', 'db4'])
def test_gradgradcheck_functions_1d(mode, wave):
    m = ll2.mode_to_int(mode)
    h0, h1, g0, g1 = [torch.tensor(a, dtype=torch.float64) for a in _wave_taps(wave)]
    for k, n in enumerate((3, 7, 12, 21)):
        x = _r((2, 1, n), k).requires_grad_(True)
        assert torch.autograd.gradgradcheck(lambda x: t1.AFB1D.apply(x, h0, h1, m), (x,))
        lo, hi = t1.afb1d_level(x.detach(), h0, h1, m)
        lo, hi = lo.clone().requires_grad_(True), hi.clone().requires_grad_(True)
        assert torch.autograd.gradgradcheck(lambda a, b: t1.SFB1D.apply(a, b, g0, g1, m), (lo, hi))


@pytest.mark.parametrize('mode', MODES)
def test_gradgradcheck_modules(mode):
    for k, wave in enumerate(('db2', 'db3')):
        x = _r((1, 1, 7, 9), k).requires_grad_(True)
        f2 = pw.DWTForward(J=2, wave=wave, mode=mode).to(DEV, torch.float64)
        i2 = pw.DWTInverse(wave=wave, mode=mode).to(DEV, torch.float64)
        assert torch.autograd.gradgradcheck(lambda x: (lambda r: (r[0],) + tuple(r[1]))(f2(x)), (x,))
        yl, yh = f2(x.detach())
        cs = [c.clone().requires_grad_(True) for c in [yl] + yh]
        assert torch.autograd.gradgradcheck(lambda *c: i2((c[0], list(c[1:]))), cs)
        s = _r((1, 2, 11), k).requires_grad_(True)
        f1 = pw.DWT1DForward(J=2, wave=wave, mode=mode).to(DEV, torch.float64)
        i1 = pw.DWT1DInverse(wave=wave, mode=mode).to(DEV, torch.float64)
        assert torch.autograd.gradgradcheck(lambda s: (lambda r: (r[0],) + tuple(r[1]))(f1(s)), (s,))
        yl, yh = f1(s.detach())
        cs = [c.clone().requires_grad_(True) for c in [yl] + yh]
        assert torch.autograd.gradgradcheck(lambda *c: i1((c[0], list(c[1:]))), cs)


# ---- the transposed-analysis kernel against the dense restatement ----------------------------------------------------

def _coeffs(N, C, Hc, Wc, rng, dtype):
    """(ll, highs) with each (n, c) plane at its own power of ten, and the plane scales."""
    s = util.plane_scales(N, C, rng)
    c = rng.uniform(-1, 1, (N, C, 4, Hc, Wc)) * s[:, :, None, None, None]
    return c.astype(dtype), s


def _abs_adjoint_2d(c, fh_lo, fh_hi, fw_lo, fw_hi, mode, H, W):
    Thl, Thh = [np.abs(oa.adjoint_matrix_1d(f, H, mode)) for f in (fh_lo, fh_hi)]
    Twl, Twh = [np.abs(oa.adjoint_matrix_1d(f, W, mode)) for f in (fw_lo, fw_hi)]
    a = np.abs(c).astype(np.float64)
    lo = Thl @ a[:, :, 0] + Thh @ a[:, :, 1]
    hi = Thl @ a[:, :, 2] + Thh @ a[:, :, 3]
    return lo @ Twl.T + hi @ Twh.T


def _max_images(n, L, mode):
    pl = oa.ext_pl(L, mode)
    K = oa.orc.coeff_len(n, L, mode)
    return max(len(oa.images(i, n, mode, -pl, 2 * K - 3 + L - pl)) for i in range(n))


CASES2 = [(37, 41, 8), (64, 129, 8), (30, 256, 4), (13, 300, 20), (5, 3, 12), (50, 50, 2), (21, 128, 6), (7, 130, 16)]


@pytest.mark.parametrize('dtype', ['float64', 'float32'])
@pytest.mark.parametrize('mode', MODES)
def test_adjoint_2d_kernel_matches_dense_restatement(mode, dtype):
    """Widths below, at and past one synthesis strip (128 coefficient columns), L = 2 ... 20, a channel slice of the
    coefficients (pitched planes)."""
    rng = np.random.default_rng(7)
    tdt = getattr(torch, dtype)
    for (H, W, L) in CASES2 + [(H, 2 * L + 5, L) for L in range(2, 21, 3) for H in (L + 1,)]:
        fh_lo, fh_hi, fw_lo, fw_hi = [rng.standard_normal(L) for _ in range(4)]
        Hc, Wc = oa.orc.coeff_len(H, L, mode), oa.orc.coeff_len(W, L, mode)
        c, s = _coeffs(2, 5, Hc, Wc, rng, np.float64)
        ref = oa.afb2d_adjoint(c[:, :, 0], c[:, :, 1:], fh_lo, fh_hi, fw_lo, fw_hi, mode, H, W)
        full = torch.tensor(c, device=DEV).to(tdt)
        cs = full[:, 1:4]                               # a channel slice: pitched planes, not contiguous
        y = ll2.afb2d_adjoint_level(cs[:, :, 0], cs[:, :, 1:], fh_lo, fh_hi, fw_lo, fw_hi, ll2.mode_to_int(mode), (H, W))
        y = y.cpu().double().numpy()
        r = ref[:, 1:4]
        # per plane: the longest accumulation chain x unit roundoff x the largest sum of |terms|; rounding the float64
        # coefficients to float32 is one more relative error per term
        mag = _abs_adjoint_2d(c[:, 1:4], fh_lo, fh_hi, fw_lo, fw_hi, mode, H, W)
        depth = _max_images(H, L, mode) * L + _max_images(W, L, mode) * L + 4
        bnd = (depth + 1) * _unit(dtype) * mag.reshape(2, 3, -1).max(axis=2)
        err = np.abs(y - r).reshape(2, 3, -1).max(axis=2)
        assert (err <= bnd).all(), (H, W, L, (err / bnd).max())


@pytest.mark.parametrize('dtype', ['float64', 'float32'])
@pytest.mark.parametrize('mode', MODES)
def test_adjoint_1d_kernel_matches_dense_restatement(mode, dtype):
    rng = np.random.default_rng(11)
    tdt = getattr(torch, dtype)
    for L in range(2, 21):
        f0, f1 = rng.standard_normal(L), rng.standard_normal(L)
        for n in sorted({1, 2, L - 1, L, L + 3, 2 * L + 1, 300, 513} - {0}):
            K = oa.orc.coeff_len(n, L, mode)
            s = util.plane_scales(3, 2, rng)
            lo = rng.uniform(-1, 1, (3, 2, K)) * s[..., None]
            hi = rng.uniform(-1, 1, (3, 2, K)) * s[..., None]
            ref = oa.afb1d_adjoint(lo, hi, f0, f1, mode, n)
            y = t1.afb1d_adjoint_level(torch.tensor(lo, device=DEV).to(tdt), torch.tensor(hi, device=DEV).to(tdt),
                                       f0, f1, ll2.mode_to_int(mode), n).cpu().double().numpy()
            mag = np.abs(lo) @ np.abs(oa.adjoint_matrix_1d(f0, n, mode)).T + \
                np.abs(hi) @ np.abs(oa.adjoint_matrix_1d(f1, n, mode)).T
            depth = 2 * _max_images(n, L, mode) * L + 4
            bnd = (depth + 1) * _unit(dtype) * mag.max(axis=2)
            assert (np.abs(y - ref).max(axis=2) <= bnd).all(), (L, n)


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
def test_adjoint_canaries(dtype):
    """NaN-filled outputs with a wider row pitch / longer rows: every output written, no padding touched."""
    ct = ctypes.c_float if dtype == torch.float32 else ctypes.c_double
    sfx = '' if dtype == torch.float32 else '_f64'
    L, mode = 8, ll2.mode_to_int('symmetric')
    f = (ct * L)(*np.random.default_rng(0).standard_normal(L))
    fp = ctypes.cast(f, ctypes.c_void_p)
    lib = _ffi.lib()
    H, W, pitch = 37, 45, 64
    Hc, Wc = lib.b200w_dwt_coeff_len(H, L, mode), lib.b200w_dwt_coeff_len(W, L, mode)
    c = torch.randn(3, 4, Hc, Wc, device=DEV, dtype=dtype)
    y = torch.full((3, H + 2, pitch), float('nan'), device=DEV, dtype=dtype)
    rc = getattr(lib, 'b200w_dwt_afb2d_adjoint' + sfx)(c.data_ptr(), 4 * Hc * Wc, Wc, c[:, 1:].contiguous().data_ptr(),
                                                      y.data_ptr(), (H + 2) * pitch, pitch, 3, Hc, Wc, H, W, fp, fp, L,
                                                      fp, fp, L, mode, None)
    torch.cuda.synchronize()
    assert rc == 0
    assert torch.isfinite(y[:, :H, :W]).all()
    assert torch.isnan(y[:, :H, W:]).all() and torch.isnan(y[:, H:]).all()
    n = 77
    K = lib.b200w_dwt_coeff_len(n, L, mode)
    lo, hi = torch.randn(4, K, device=DEV, dtype=dtype), torch.randn(4, K, device=DEV, dtype=dtype)
    y1 = torch.full((4 * n + 16,), float('nan'), device=DEV, dtype=dtype)
    rc = getattr(lib, 'b200w_dwt_afb1d_adjoint' + sfx)(lo.data_ptr(), hi.data_ptr(), 4, K, y1.data_ptr(), n, fp, fp, L,
                                                      mode, None)
    torch.cuda.synchronize()
    assert rc == 0
    assert torch.isfinite(y1[:4 * n]).all() and torch.isnan(y1[4 * n:]).all()


# ---- routes (child-process profiler traces) ---------------------------------------------------------------------------

def _short(name):
    for k in ('adjoint_border', 'afb2d', 'sfb2d', 'afb1d', 'sfb1d', 'pyramid'):
        if k in name:
            return k
    return None


def trace_in_this_process(mode):
    """Kernel traces of (a) a plain first-order backward through every module, (b) the raw level calls the backward
    passes made before they became autograd Functions, (c) one double backward of each 2-D / 1-D synthesis."""
    torch.manual_seed(0)
    m = ll2.mode_to_int(mode)
    x = torch.randn(2, 3, 70, 90, device=DEV, requires_grad=True)
    f = pw.DWTForward(J=2, wave='db4', mode=mode).to(DEV)
    i = pw.DWTInverse(wave='db4', mode=mode).to(DEV)
    s = torch.randn(2, 3, 301, device=DEV, requires_grad=True)
    f1 = pw.DWT1DForward(J=1, wave='db4', mode=mode).to(DEV)
    i1 = pw.DWT1DInverse(wave='db4', mode=mode).to(DEV)
    yl, yh = f(x)
    c = [yl.detach().requires_grad_(True)] + [h.detach().requires_grad_(True) for h in yh]
    y = i((c[0], c[1:]))
    l1, h1 = f1(s)
    c1 = [l1.detach().requires_grad_(True), h1[0].detach().requires_grad_(True)]
    y1 = i1((c1[0], [c1[1]]))
    gs = [torch.randn_like(t) for t in (yl, yh[0], yh[1], y, l1, h1[0], y1)]

    def plain():
        torch.autograd.backward([yl, yh[0], yh[1], y, l1, h1[0], y1], gs, retain_graph=True)
    h0c, h1c, h0r, h1r = [_ffi.host_taps(b) for b in (f.h0_col, f.h1_col, f.h0_row, f.h1_row)]
    g0c, g1c, g0r, g1r = [_ffi.host_taps(b) for b in (i.g0_col, i.g1_col, i.g0_row, i.g1_row)]
    outs = {}

    def raw():   # the parent implementation's calls, in autograd's order
        # DWTForward passes its *_col buffers as the Function's W filters (transform2d.py)
        low = ll2.sfb2d_level(gs[0].contiguous(), gs[2], h0r, h1r, h0c, h1c, m, out_hw=tuple(yh[0].shape[-2:]))
        outs['x'] = ll2.sfb2d_level(low.contiguous(), gs[1], h0r, h1r, h0c, h1c, m, out_hw=(70, 90))
        d = ll2.afb2d_level(gs[3].contiguous(), g0c, g1c, g0r, g1r, m)
        d = ll2.afb2d_level(d[0].contiguous(), g0c, g1c, g0r, g1r, m)
        outs['s'] = t1.sfb1d_level(gs[4], gs[5], f1.h0, f1.h1, m, out_len=301)
        t1.afb1d_level(gs[6].contiguous(), i1.g0, i1.g1, m)
    ks_plain = sweep_util.traced_kernels(plain, _short)
    ks_raw = sweep_util.traced_kernels(raw, _short)
    same = bool(torch.equal(x.grad, outs['x']) and torch.equal(s.grad, outs['s']))

    def double():
        u = torch.randn_like(y, requires_grad=True)
        g = torch.autograd.grad(y, c[0], u, create_graph=True)[0]
        torch.autograd.grad(g, u, torch.randn_like(g))
        u1 = torch.randn_like(y1, requires_grad=True)
        g1 = torch.autograd.grad(y1, c1[0], u1, create_graph=True)[0]
        torch.autograd.grad(g1, u1, torch.randn_like(g1))
    ks_double = sweep_util.traced_kernels(double, _short)
    return ks_plain, ks_raw, same, ks_double


@pytest.mark.parametrize('mode', MODES)
def test_trace_first_order_is_unchanged_and_double_routes(mode):
    code = ('import json, sys; from tests import test_gpu_dwt_grad2 as t; '
            'print(json.dumps(t.trace_in_this_process(sys.argv[1])))')
    r = subprocess.run([sys.executable, '-c', code, mode], cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    ks_plain, ks_raw, same, ks_double = json.loads(r.stdout.strip().splitlines()[-1])
    assert same, 'the first-order gradients differ from the raw level calls'
    if ks_plain is None:
        pytest.skip('no CUDA activity trace on this machine')
    assert sorted(ks_plain) == sorted(ks_raw), (ks_plain, ks_raw)
    assert 'adjoint_border' not in ks_plain
    # double backward: each SFB's backward (an analysis) differentiates into A_m^T = synthesis (+ border kernel)
    # (two SFB2D levels of DWTInverse and one SFB1D lie on the differentiated paths; the even sizes of periodization
    # need no border kernel)
    n_border = ks_double.count('adjoint_border')
    assert n_border == (0 if mode in ('zero', 'periodization') else 3), ks_double
    assert 'sfb2d' in ks_double and 'sfb1d' in ks_double


# ---- R1 penalty through a wavelet discriminator, against torch ops ---------------------------------------------------

def _ext(n, npad_l, total, mode):
    """Source index of each extended position (reference mypad / pywt extension), -1 = zero."""
    idx = []
    for q in range(total):
        p = q - npad_l
        if 0 <= p < n:
            idx.append(p)
        elif mode == 'zero':
            idx.append(-1)
        elif mode == 'symmetric':
            r = p % (2 * n)
            idx.append(r if r < n else 2 * n - 1 - r)
        elif mode == 'reflect':
            r = p % (2 * n - 2)
            idx.append(r if r < n else 2 * n - 2 - r)
        elif mode == 'periodic':
            idx.append(p % n)
        else:
            r = p % (n + n % 2)
            idx.append(r if r < n else n - 1)
    return idx


def afb1d_torch(x, f0, f1, mode, dim):
    """The analysis along ``dim`` (-1 or -2) of x as torch ops: extension gather + stride-2 conv (reference afb1d)."""
    n = x.shape[dim]
    L = f0.numel()
    K = oa.orc.coeff_len(n, L, mode)
    pl = oa.ext_pl(L, mode)
    idx = _ext(n, pl, 2 * K - 2 + L, mode)
    src = torch.tensor([max(i, 0) for i in idx], device=x.device)
    mask = torch.tensor([i >= 0 for i in idx], device=x.device, dtype=x.dtype)
    xe = x.index_select(dim, src) * (mask if dim == -1 else mask[:, None])
    N, C = x.shape[:2]
    w = torch.stack([f0, f1]).to(x)[:, None]                  # (2, 1, L)
    if dim == -1:
        y = F.conv2d(xe.reshape(-1, 1, xe.shape[-2], xe.shape[-1]), w[:, :, None, :], stride=(1, 2))
    else:
        y = F.conv2d(xe.reshape(-1, 1, xe.shape[-2], xe.shape[-1]), w[:, :, :, None], stride=(2, 1))
    y = y.reshape(N, C, 2, y.shape[-2], y.shape[-1])
    return y[:, :, 0], y[:, :, 1]


def sfb1d_torch(lo, hi, g0, g1, mode, dim, n):
    """The synthesis along ``dim`` cropped to n as torch ops: stride-2 transposed conv, offset L - 2 (reference
    sfb1d, zero / symmetric / reflect / periodic)."""
    L = g0.numel()
    N, C = lo.shape[:2]
    w = torch.stack([g0, g1]).to(lo)[:, None]                 # (2, 1, L)
    z = torch.stack([lo, hi], 2).reshape(-1, 2, lo.shape[-2], lo.shape[-1])
    if dim == -1:
        y = F.conv_transpose2d(z, w[:, :, None, :], stride=(1, 2))[..., L - 2:L - 2 + n]
    else:
        y = F.conv_transpose2d(z, w[:, :, :, None], stride=(2, 1))[..., L - 2:L - 2 + n, :]
    return y.reshape(N, C, y.shape[-2], y.shape[-1])


class _AFB2DOps(torch.autograd.Function):
    """The reference's AFB2D as torch ops: forward = the analysis along W then H; backward = the synthesis with the
    same taps cropped to the input, written in differentiable torch ops (reference dwt/lowlevel.py:341-365), so a
    second backward differentiates it as the reference's autograd does."""

    @staticmethod
    def forward(ctx, x, h0, h1, mode):
        ctx.h, ctx.mode, ctx.shape = (h0, h1), mode, x.shape[-2:]
        return _analysis_ops(x, h0, h1, mode)

    @staticmethod
    def backward(ctx, dll, dhs):
        (h0, h1), mode, (H, W) = ctx.h, ctx.mode, ctx.shape
        lo = sfb1d_torch(dll, dhs[:, :, 0], h0, h1, mode, -2, H)
        hi = sfb1d_torch(dhs[:, :, 1], dhs[:, :, 2], h0, h1, mode, -2, H)
        return sfb1d_torch(lo, hi, h0, h1, mode, -1, W), None, None, None


class _SFB2DOps(torch.autograd.Function):
    """The reference's SFB2D as torch ops: forward = the synthesis along H then W; backward = the analysis with the
    same taps in the same mode, in differentiable torch ops (reference dwt/lowlevel.py:671-694)."""

    @staticmethod
    def forward(ctx, ll, hs, g0, g1, mode):
        ctx.g, ctx.mode = (g0, g1), mode
        L = g0.numel()
        Ho, Wo = 2 * ll.shape[-2] - L + 2, 2 * ll.shape[-1] - L + 2
        lo = sfb1d_torch(ll, hs[:, :, 0], g0, g1, mode, -2, Ho)
        hi = sfb1d_torch(hs[:, :, 1], hs[:, :, 2], g0, g1, mode, -2, Ho)
        return sfb1d_torch(lo, hi, g0, g1, mode, -1, Wo)

    @staticmethod
    def backward(ctx, dy):
        (g0, g1), mode = ctx.g, ctx.mode
        return _analysis_ops(dy, g0, g1, mode) + (None, None, None)


def _analysis_ops(x, h0, h1, mode):
    lo, hi = afb1d_torch(x, h0, h1, mode, -1)
    ll, lh = afb1d_torch(lo, h0, h1, mode, -2)
    hl, hh = afb1d_torch(hi, h0, h1, mode, -2)
    return ll, torch.stack([lh, hl, hh], 2)


def dwt_torch(x, h0, h1, mode, J):
    """DWTForward as the reference's Function graph in torch ops (symmetric / zero / reflect / periodic)."""
    yh = []
    for _ in range(J):
        x, h = _AFB2DOps.apply(x, h0, h1, mode)
        yh.append(h)
    return x, yh


def idwt_torch(yl, yh, g0, g1, mode):
    """DWTInverse as the reference's Function graph in torch ops."""
    ll = yl
    for h in yh[::-1]:
        ll = ll[..., :h.shape[-2], :h.shape[-1]]
        ll = _SFB2DOps.apply(ll, h, g0, g1, mode)
    return ll


def r1_step(features, x_leaves, lin):
    """One R1 step: logit = lin(features), loss = softplus(logit); penalty = |d loss / d x|^2; returns the weight
    gradient of loss + penalty."""
    lin.zero_grad()
    feats = features(*x_leaves)
    logit = lin(torch.cat([t.flatten(1) for t in feats], 1))
    loss = F.softplus(logit).sum()
    g = torch.autograd.grad(loss, x_leaves, create_graph=True)
    pen = sum((t ** 2).sum() for t in g)
    (loss + pen).backward()
    return lin.weight.grad.clone()


@pytest.mark.parametrize('case', ['forward', 'inverse'])
def test_r1_step_matches_torch_ops(case):
    """float64: the weight gradient of an R1 step is badly conditioned (in float32 the torch-op graph alone moves by
    tens of percent against its own float64 result at this size), so both graphs run in double precision."""
    torch.manual_seed(3)
    mode, wave, J = 'symmetric', 'db4', 3
    f = _module_in_dtype(pw.DWTForward, torch.float64, J=J, wave=wave, mode=mode)
    i = _module_in_dtype(pw.DWTInverse, torch.float64, wave=wave, mode=mode)
    h0, h1 = f.h0_col.flatten(), f.h1_col.flatten()
    g0, g1 = i.g0_col.flatten(), i.g1_col.flatten()
    x = torch.randn(2, 3, 512, 512, device=DEV, dtype=torch.float64)
    if case == 'forward':
        ours = lambda x: (lambda r: [r[0]] + r[1])(f(x))            # noqa: E731
        ops = lambda x: (lambda r: [r[0]] + r[1])(dwt_torch(x, h0, h1, mode, J))   # noqa: E731
        leaves = [x]
    else:
        yl, yh = f(x)
        ours = lambda *c: [i((c[0], list(c[1:])))]                  # noqa: E731
        ops = lambda *c: [idwt_torch(c[0], list(c[1:]), g0, g1, mode)]   # noqa: E731
        leaves = [yl] + yh
    nfeat = sum(t.numel() // t.shape[0] for t in ours(*leaves))
    lin = torch.nn.Linear(nfeat, 1).to(DEV, torch.float64)
    torch.nn.init.normal_(lin.weight, std=nfeat ** -0.5)
    a = r1_step(ours, [t.detach().clone().requires_grad_(True) for t in leaves], lin)
    b = r1_step(ops, [t.detach().clone().requires_grad_(True) for t in leaves], lin)
    err = (a - b).abs().max().item() / b.abs().max().item()
    assert err < 1e-10, err
