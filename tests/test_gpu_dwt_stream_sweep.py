"""Boundary sweep of the DWT streaming and fused kernels (-m gpu): every instantiation of afb2d_stream, sfb2d_stream,
sfb2d_stream4 and dwt_pyramid, called through the level entry points (dwt.lowlevel.afb2d_level, sfb2d_level,
dwt_forward_levels) at widths / heights / plane counts / layouts around each kernel's strip, chunk and plan boundaries.
The case matrix and the dispatch rules live in tests/dwt_sweep_cases.py (checked on the CPU by
tests/test_dwt_sweep_matrix.py).

Every (n, c) plane is scaled by its own power of ten (10^-6 .. 10^6).  Per case:
  analysis   ll and highs bit-identical to the generic tile kernel and to the fp32 oracle;
  synthesis  every output plane within its own bound K u G s of the float64 oracle (tests/util.py bound_sfb2d), for the
             streaming and the generic kernel, and the two within 2 K of each other;
  pyramid    yl and every yh[j] bit-identical to the fp32 oracle and to the generic kernel run level by level;
and, once per instantiation, NaN-filled outputs inside canaried buffers through the C ABI (the kPyramidFirst workspace:
canaries only, its pad columns are never written), and (one test) the kernels each case launches, read from a
torch.profiler CUDA trace, are the ones the dispatch rules predict."""
import ctypes
import zlib

import numpy as np
import pytest
import torch

from oracle import oracle as orc
from pytorch_wavelets_b200 import _ffi
from pytorch_wavelets_b200.dwt import lowlevel
from pytorch_wavelets_b200.wavelets import Wavelet
from tests import dwt_sweep_cases as dc
from tests import sweep_util, util
from tests.sweep_util import Canaried

pytestmark = pytest.mark.gpu
DEV = 'cuda'
CASES = dc.CASES


def _f32(a):
    return np.asarray(a, dtype=np.float64).astype(np.float32)


def analysis_taps(L):
    """dbL/2 analysis filters in stored (time-reversed) order, fp32: (lo, hi)."""
    w = Wavelet('db%d' % (L // 2))
    return _f32(w.dec_lo[::-1].copy()), _f32(w.dec_hi[::-1].copy())


def synthesis_taps(L):
    w = Wavelet('db%d' % (L // 2))
    return _f32(w.rec_lo), _f32(w.rec_hi)


def _np(t):
    return None if t is None else t.detach().cpu().numpy()


class Prepared(object):
    """Inputs (host fp32 + device tensors in the case's layout), taps, and runners."""

    def __init__(self, c):
        self.c = c
        fam, L, mode = c['family'], c['L'], c['mode']
        self.m = lowlevel.mode_to_int(mode)
        rng = np.random.default_rng(zlib.crc32(c['id'].encode()))
        N, C, H, W = c['shape']
        if fam in ('afb', 'pyr'):
            self.x, self.sc = util.scaled_uniform((N, C, H, W), rng)
            lo, hi = analysis_taps(L)
            self.fw = analysis_taps(c['lw']) if c['lw'] else (lo, hi)
            self.fh = (lo, hi)
            self.xt = self._device_input()
        else:
            self.ll, self.sc = util.scaled_uniform((N, C, H, W), rng)
            hi, _ = util.scaled_uniform((N, C, 3, H, W), rng, scales=self.sc)
            self.hi = hi if c['has_hi'] else None
            self.gh = synthesis_taps(L)
            self.gw = synthesis_taps(c['lw']) if c['lw'] else self.gh
            if c['ll_trim']:
                big = (rng.uniform(-1, 1, (N, C, H + 1, W + 1)) * 1e6).astype(np.float32)   # row H, column W: dropped
                big[:, :, :H, :W] = self.ll
                self.llt = torch.from_numpy(big).to(DEV)[:, :, :H, :W]
            else:
                self.llt = torch.from_numpy(self.ll).to(DEV)
            self.hit = None if self.hi is None else torch.from_numpy(self.hi).to(DEV)

    def _device_input(self):
        c = self.c
        N, C, H, W = c['shape']
        ps, pitch, off = dc.layout(c)
        if c['offset'] and c['offset'] == H * W and N == 1:          # a channel slice of a wider tensor
            big = torch.full((1, C + 1, H, W), float('nan'), device=DEV)
            big[0, 1:] = torch.from_numpy(self.x[0]).to(DEV)
            return big[:, 1:]
        n = (N * C - 1) * ps + (H - 1) * pitch + W
        flat = torch.full((n + off,), float('nan'), device=DEV)
        xt = flat[off:].as_strided((N, C, H, W), (C * ps, ps, pitch, 1))
        xt.copy_(torch.from_numpy(self.x).to(DEV))
        got = _ffi.planes_view(xt)
        assert got[0].data_ptr() == xt.data_ptr() and got[1:] == (ps, pitch), (c['id'], got[1:])
        return xt

    # -- the level entry points (auto dispatch, or the generic kernels) --
    def run(self, generic=False):
        c, fam = self.c, self.c['family']
        with (_ffi.generic_kernels() if generic else _Null()):
            if fam == 'afb':
                ll, hi = lowlevel.afb2d_level(self.xt, *self.fw, *self.fh, self.m)
                return {'ll': ll, 'highs': hi}
            if fam == 'sfb':
                return {'y': lowlevel.sfb2d_level(self.llt, self.hit, *self.gh, *self.gw, self.m, out_hw=c['crop'])}
            if not generic:
                yl, yh = lowlevel.dwt_forward_levels(self.xt, *self.fw, *self.fh, self.m, c['J'])
            else:   # the generic level chain
                ll, yh = self.xt, []
                for _ in range(c['J']):
                    ll, h = lowlevel.afb2d_level(ll, *self.fw, *self.fh, self.m)
                    yh.append(h)
                yl = ll
            out = {'yl': yl}
            out.update(('yh%d' % j, h) for j, h in enumerate(yh))
            return out

    def oracle(self, dtype):
        c, fam = self.c, self.c['family']
        if fam == 'afb':
            ll, hi = orc.dwt_afb2d(self.x.astype(dtype), *[t.astype(dtype) for t in self.fw + self.fh], c['mode'])
            return {'ll': ll, 'highs': hi}
        if fam == 'sfb':
            return {'y': orc.dwt_sfb2d(self.ll.astype(dtype), None if self.hi is None else self.hi.astype(dtype),
                                       *[t.astype(dtype) for t in self.gh + self.gw], c['mode'], out_hw=c['crop'])}
        ll, out = self.x.astype(dtype), {}
        for j in range(c['J']):
            ll, out['yh%d' % j] = orc.dwt_afb2d(ll, *[t.astype(dtype) for t in self.fw + self.fh], c['mode'])
        out['yl'] = ll
        return out


class _Null(object):
    def __enter__(self):
        return self

    def __exit__(self, *exc):
        return False


def check_case(c):
    P = Prepared(c)
    got = {k: _np(v) for k, v in P.run().items()}
    gen = {k: _np(v) for k, v in P.run(generic=True).items()}
    what = c['id']
    if c['family'] in ('afb', 'pyr'):
        o32 = P.oracle(np.float32)
        assert sorted(got) == sorted(o32)
        for k in sorted(o32):
            assert np.array_equal(got[k], gen[k]), '%s: %s differs from the generic kernel' % (what, k)
            assert np.array_equal(got[k], o32[k]), '%s: %s differs from the fp32 oracle' % (what, k)
        return
    o64 = P.oracle(np.float64)['y']
    s = util.plane_max(P.ll, P.hi)
    G, K = util.bound_sfb2d(*P.gh, *P.gw, has_hi=c['has_hi'])
    util.assert_plane_bound(got['y'], o64, s, G, K, what=what + ' stream vs float64')
    util.assert_plane_bound(gen['y'], o64, s, G, K, what=what + ' generic vs float64')
    util.assert_plane_bound(got['y'], gen['y'], s, G, 2 * K, what=what + ' stream vs generic')


@pytest.fixture(scope='module', autouse=True)
def _native_library_is_loaded():
    assert torch.cuda.is_available()
    assert _ffi.lib().b200w_version() >= 100
    yield


@pytest.mark.parametrize('c', CASES, ids=[c['id'] for c in CASES])
def test_dwt_stream_sweep(c):
    check_case(c)


# ---- unwritten outputs and stray writes, through the C ABI ---------------------------------------------------------------

@pytest.mark.parametrize('c', [c for c in CASES if c['canary']], ids=[c['id'] for c in CASES if c['canary']])
def test_canaries_and_unwritten_outputs(c):
    P = Prepared(c)
    L = _ffi.lib()
    fam, (N, C, H, W) = c['family'], c['shape']
    st = _ffi.stream_of(P.xt if fam != 'sfb' else P.llt)
    ws = None
    if fam == 'afb':
        x, xps, xpitch = _ffi.planes_view(P.xt)
        fw = [_ffi.host_taps(t) for t in P.fw]
        fh = [_ffi.host_taps(t) for t in P.fh]
        Ho, Wo = orc.coeff_len(H, fh[0].n, c['mode']), orc.coeff_len(W, fw[0].n, c['mode'])
        outs = [Canaried((N, C, Ho, Wo)), Canaried((N, C, 3, Ho, Wo))]
        rc = L.b200w_dwt_afb2d(x.data_ptr(), xps, xpitch, outs[0].ptr(), Ho * Wo, Wo, outs[1].ptr(), N * C, H, W,
                               fw[0].ptr, fw[1].ptr, fw[0].n, fh[0].ptr, fh[1].ptr, fh[0].n, P.m, st)
    elif fam == 'sfb':
        ll, llps, llpitch = _ffi.planes_view(P.llt)
        gh = [_ffi.host_taps(t) for t in P.gh]
        gw = [_ffi.host_taps(t) for t in P.gw]
        Ho, Wo = orc.rec_len(H, gh[0].n, c['mode']), orc.rec_len(W, gw[0].n, c['mode'])
        if c['crop']:
            Ho, Wo = min(Ho, c['crop'][0]), min(Wo, c['crop'][1])
        outs = [Canaried((N, C, Ho, Wo))]
        rc = L.b200w_dwt_sfb2d(ll.data_ptr(), llps, llpitch, None if P.hit is None else P.hit.data_ptr(), outs[0].ptr(),
                               Ho * Wo, Wo, N * C, H, W, Ho, Wo, gh[0].ptr, gh[1].ptr, gh[0].n, gw[0].ptr, gw[1].ptr,
                               gw[0].n, P.m, st)
    else:
        x, xps, xpitch = _ffi.planes_view(P.xt)
        taps = [_ffi.host_taps(t) for t in P.fw + P.fh]
        Lf = taps[0].n
        sizes, h, w = [], H, W
        for _ in range(c['J']):
            h, w = orc.coeff_len(h, Lf, c['mode']), orc.coeff_len(w, Lf, c['mode'])
            sizes.append((h, w))
        outs = [Canaried((N, C) + sizes[-1])] + [Canaried((N, C, 3) + s) for s in sizes]
        wsb = L.b200w_dwt_forward_workspace(x.data_ptr(), xps, xpitch, N * C, H, W, c['J'], Lf, Lf, P.m)
        assert wsb >= 0, wsb
        assert (wsb == 0) == (dc.dwt_policy(c)[0] == 'all'), (c['id'], wsb)
        if wsb:
            ws = Canaried(((wsb + 3) // 4,))
        ptrs = (ctypes.c_void_p * c['J'])(*[o.ptr() for o in outs[1:]])
        rc = L.b200w_dwt_forward(x.data_ptr(), xps, xpitch, N * C, H, W, c['J'], outs[0].ptr(), ptrs,
                                 taps[0].ptr, taps[1].ptr, Lf, taps[2].ptr, taps[3].ptr, Lf, P.m,
                                 None if ws is None else ws.ptr(), wsb, st)
    assert rc == 0, rc
    torch.cuda.synchronize()
    for k, o in enumerate(outs):
        o.check('%s output %d' % (c['id'], k))
    if ws is not None:
        ws.check_canaries(c['id'] + ' workspace')
    ref = [v for v in P.run().values()]
    assert len(ref) == len(outs)
    for k, (o, r) in enumerate(zip(outs, ref)):
        assert torch.equal(o.t, r.contiguous()), '%s: output %d of the C ABI call and the level function differ' % (
            c['id'], k)


# ---- which kernels each case launched --------------------------------------------------------------------------------

_short = sweep_util.kernel_namer(['afb2d_stream', 'sfb2d_stream4', 'sfb2d_stream', 'dwt_pyramid'], ['afb2d', 'sfb2d'])


def test_dispatch_launches_the_expected_kernels():
    """One auto-dispatch call per case under a torch.profiler CUDA trace: the engine kernels it launched are the
    instantiations the dispatch rules and the shipped pyramid plan predict (the generic tile kernel for the fallback
    cases), and the streaming / fused kernels seen are every instantiation but the unreachable one."""
    prepared = [Prepared(c) for c in CASES]
    seen = sweep_util.traced_kernels(lambda: [P.run() for P in prepared], _short)
    if seen is None:
        pytest.skip('CUDA activity tracing is unavailable or recorded no kernels')
    want = [dc.expected_kernels(c) for c in CASES]
    assert len(seen) == sum(len(w) for w in want), (len(seen), sum(len(w) for w in want))
    wrong, i = [], 0
    for c, w in zip(CASES, want):
        if seen[i:i + len(w)] != w:
            wrong.append((c['id'], w, seen[i:i + len(w)]))
        i += len(w)
    assert not wrong, wrong[:10]
    assert sorted(set(s for s in seen if not s.endswith('_tile'))) == sorted(set(dc.ALL_KERNELS) - set(dc.UNREACHABLE))
