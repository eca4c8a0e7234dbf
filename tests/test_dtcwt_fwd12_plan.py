"""CPU tests of the fused DTCWT forward levels 1 + 2 (no GPU):

  * the shipped plan (pytorch_wavelets_b200/csrc/dtcwt_fwd12_plan.h, compiled with g++ into a small test library):
    shared-memory layout within the device limit, and the LL ring depth replayed against level 2's group schedule for
    every band of many (H, band height) pairs, the bands at the plane's top and bottom edges included;
  * the route predicate and the argument validation of b200w_dtcwt_fwd_j12 through the built library (neither touches
    the device)."""
import ctypes
import os
import subprocess

import pytest

from pytorch_wavelets_b200 import _build, _ffi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'pytorch_wavelets_b200', 'csrc')
MAX_SMEM = 227 * 1024

SHIM = r'''
#include "dtcwt_fwd12_plan.h"
using namespace b200w;
extern "C" int plan(int H, int W, int L0, int L1, int MQ, int* out) {
  Fwd12Plan p;
  const int rc = fwd12_plan(p, H, W, L0, L1, MQ);
  out[0] = p.threads; out[1] = p.sw1; out[2] = p.sw2; out[3] = p.ring; out[4] = p.ll_off; out[5] = p.smem_bytes;
  out[6] = kF12InStages;
  return rc;
}
extern "C" void band(int b, int CH, int Hq, int nmg, int* out) {
  const Fwd12Band v = fwd12_band(b, CH, Hq, nmg);
  out[0] = v.qy0; out[1] = v.qy1; out[2] = v.g0; out[3] = v.n2; out[4] = v.a0; out[5] = v.a1; out[6] = v.lag;
}
extern "C" int slot(int v, int ring) { return fwd12_slot(v, ring); }
'''


@pytest.fixture(scope='module')
def shim(tmp_path_factory):
    d = tmp_path_factory.mktemp('fwd12_plan')
    src, so = str(d / 'shim.cpp'), str(d / 'libshim.so')
    with open(src, 'w') as f:
        f.write(SHIM)
    subprocess.check_call(['g++', '-O1', '-fPIC', '-std=c++17', '-shared', '-I', CSRC, '-o', so, src])
    return ctypes.CDLL(so)


def _plan(shim, H, W, L0=5, L1=7, MQ=10):
    out = (ctypes.c_int * 7)()
    rc = shim.plan(H, W, L0, L1, MQ, out)
    keys = ('threads', 'sw1', 'sw2', 'ring', 'll_off', 'smem_bytes', 'in_stages')
    return None if rc else dict(zip(keys, out))


def _band(shim, b, CH, Hq, nmg):
    out = (ctypes.c_int * 7)()
    shim.band(b, CH, Hq, nmg, out)
    return dict(zip(('qy0', 'qy1', 'g0', 'n2', 'a0', 'a1', 'lag'), out))


def test_layout_fits_the_device(shim):
    for W in range(8, 1025, 4):
        p = _plan(shim, 64, W)
        assert p is not None, W
        assert p['threads'] % 32 == 0 and p['threads'] <= 256 and 4 * p['threads'] >= W
        assert p['sw1'] == W + 8 and p['sw2'] == W + 16 and p['sw1'] % 4 == 0 and p['sw2'] % 4 == 0
        assert p['ll_off'] == p['in_stages'] * 2 * p['sw1']                     # input ring first, then the LL ring
        assert p['smem_bytes'] == 4 * (p['ll_off'] + p['ring'] * 4 * p['sw2']) <= MAX_SMEM
    assert _plan(shim, 64, 1024)['threads'] == 256


def test_predicate(shim):
    assert _plan(shim, 64, 1024) is not None
    assert _plan(shim, 64, 1028) is None           # wider than 256 threads hold
    assert _plan(shim, 64, 4) is None              # the level-2 mirror needs 8 columns
    assert _plan(shim, 20, 1024) is None           # ... and 24 rows (three times the mirrored groups, for the ring)
    assert _plan(shim, 24, 1024) is not None
    assert _plan(shim, 62, 1024) is None and _plan(shim, 64, 1022) is None
    assert _plan(shim, 64, 1024, 7, 5) is None     # filter pairs that are not compiled
    assert _plan(shim, 64, 1024, 5, 7, 14) is None


def _mirror(v, Hq):
    """The real group a virtual group of LL1 rows copies (symmetric extension, one reflection)."""
    if v < 0:
        return -1 - v
    if v >= Hq:
        return 2 * Hq - 1 - v
    return v


@pytest.mark.parametrize('MQ', [10])
def test_ring_depth_covers_the_level2_schedule(shim, MQ):
    """Replay the kernel's step schedule for every band: level 1 produces real group a0 + s in phase A of step s and
    writes it (and its in-band mirrors) into slot v mod ring; level 2 reads virtual group g0 + s - lag in phase B.  Every
    group a stage reads must have been written, and no other write may land in its slot in between."""
    nmg = (MQ - 2) // 4
    ring = _plan(shim, 64, 1024, 5, 7, MQ)['ring']
    assert _plan(shim, 12 * nmg - 4, 1024, 5, 7, MQ) is None and _plan(shim, 12 * nmg, 1024, 5, 7, MQ) is not None
    for H in list(range(12 * nmg, 161, 4)) + [512, 1024]:
        Hq = H // 4
        for CH in sorted({2 * nmg, 2 * nmg + 1, 5, 8, 13, 64, Hq}):
            if CH < 1:
                continue
            for bi in range((Hq + CH - 1) // CH):
                b = _band(shim, bi, CH, Hq, nmg)
                assert b['qy1'] > b['qy0']
                lo, hi = b['g0'], b['g0'] + b['n2']
                assert b['a0'] <= max(0, lo) and b['a1'] >= min(Hq, hi)
                writes = {}   # virtual group -> step it is written (phase A)
                for g in range(b['a0'], b['a1']):
                    s = g - b['a0']
                    for v in {g, -1 - g, 2 * Hq - 1 - g}:
                        if lo <= v < hi and _mirror(v, Hq) == g:
                            writes[v] = s
                by_slot = {}
                for u, wu in writes.items():
                    by_slot.setdefault(shim.slot(u, ring), []).append((u, wu))
                for v in range(lo, hi):
                    read = v - lo + b['lag']
                    assert v in writes and writes[v] <= read, ('unwritten', H, CH, bi, v)
                    sv = shim.slot(v, ring)
                    assert sv == v % ring
                    for u, wu in by_slot[sv]:
                        if u != v:
                            assert not (writes[v] <= wu <= read), ('overwritten', H, CH, bi, v, u)
                # the kernel runs lag + n2 steps; level 1 is done by then
                assert b['a1'] - b['a0'] <= b['lag'] + b['n2']


@pytest.fixture(scope='module')
def lib():
    _build.build()
    return _ffi.lib()


def test_route_predicate_of_the_entry(lib):
    ws = lib.b200w_dtcwt_fwd_j12_workspace
    a = 1 << 20     # a 16-byte aligned (never dereferenced) address
    full = 4 * 2 * 3 * 64 * 1024
    assert ws(a, 64 * 1024, 1024, 16, 2, 3, 64, 1024, 5, 7, 10) == 0                 # fused: no workspace
    assert ws(a + 4, 64 * 1024, 1024, 16, 2, 3, 64, 1024, 5, 7, 10) == full          # unaligned base
    assert ws(a, 64 * 1026, 1026, 16, 2, 3, 64, 1024, 5, 7, 10) == full              # row pitch not a 16-byte multiple
    assert ws(a, 64 * 1024, 1024, None, 2, 3, 64, 1024, 5, 7, 10) == full            # level-1 band-pass skipped
    assert ws(a, 64 * 1024, 1024, 16, 2, 3, 64, 1024, 13, 19, 10) == full            # near_sym_b: not compiled
    assert ws(a, 64 * 1024, 1024, 16, 2, 3, 64, 1024, 5, 7, 14) == full              # qshift_b: not compiled
    assert ws(a, 64 * 2048, 2048, 16, 2, 3, 64, 2048, 5, 7, 10) == 2 * full          # wider than the kernel holds
    assert ws(a, 64 * 1024, 1024, 16, 2, 3, 62, 1024, 5, 7, 10) == -2                # H % 4 != 0
    assert ws(a, 64 * 1024, 1024, 16, 2, 3, 64, 1022, 5, 7, 10) == -2                # W % 4 != 0


def test_argument_validation_without_a_gpu(lib):
    fn = lib.b200w_dtcwt_fwd_j12
    buf = ctypes.c_void_p(1 << 20)
    t = (ctypes.c_float * 64)(*([0.1] * 64))
    hs = _ffi.hs_array([1] * 6)

    def call(x=buf, ll2=buf, h0=buf, hs0=hs, h1=buf, hs1=hs, N=1, C=1, H=16, W=16, xpitch=16, llpitch=8, L0=5, L1=7,
             m=10, taps=t):
        return fn(x, H * xpitch, xpitch, ll2, (H // 2) * llpitch, llpitch, h0, hs0, h1, hs1, N, C, H, W, taps, L0, taps,
                  L1, taps, taps, taps, taps, m, 1, None, 0, None)
    assert call(N=0) == 0                                   # empty batch: no launch, no CUDA call
    assert call(x=None, N=0) == -3
    assert call(ll2=None, N=0) == -3
    assert call(hs0=None, N=0) == -3 and call(hs1=None, N=0) == -3
    assert call(H=18, N=0) == -2 and call(W=18, xpitch=18, N=0) == -2 and call(W=2, xpitch=2, llpitch=1, N=0) == -2
    assert call(C=0) == -2
    assert call(L0=4, N=0) == -4 and call(m=9, N=0) == -4 and call(m=42, N=0) == -4
    assert call(taps=None, N=0) == -3
    assert call(xpitch=12, N=0) == -3 and call(llpitch=6, N=0) == -3
