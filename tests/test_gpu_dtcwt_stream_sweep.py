"""Boundary sweep of the DTCWT / ScatLayer streaming kernels (-m gpu): every instantiation that
fwd_j1_stream, fwd_j2plus_stream, inv_j1_stream and inv_j2plus_stream dispatch to, called through the level functions
(dtcwt.transform_funcs, scatternet.lowlevel.scat_j1) at widths / heights / plane counts around each kernel's own strip and
chunk boundaries, plus one filter pair per family that no instantiation covers (the generic fallback).

Every (n, c) plane is scaled by its own power of ten (10^-6 .. 10^6; the inverses use one scale for the low-pass and
band-pass planes of an (n, c)), and every output plane is held to its own fp32 error bound against the float64 oracle
(tests/util.py), so an error confined to a small plane, or one that reads a neighbour plane, cannot hide under the
largest plane.  Per case:
  (a) forward DTCWT levels bit-identical to the generic tile kernel (same FMA order); inverses and ScatLayer within twice
      the bound of (c) of it (both are held to (c));
  (b) forward low-pass bit-identical to the fp32 oracle;
  (c) every output plane within its bound of the float64 oracle run on the same fp32 operands;
and, once per instantiation, (d) NaN-filled outputs inside canaried buffers through the C ABI, and (e, one test) the kernel
each case launches, read from a torch.profiler CUDA trace, is the one the dispatch rules predict."""
import contextlib
import zlib

import numpy as np
import pytest
import torch

from oracle import oracle as orc
from pytorch_wavelets_b200 import _ffi
from pytorch_wavelets_b200.dtcwt import transform_funcs as tf
from pytorch_wavelets_b200.dtcwt._tables import TABLES
from pytorch_wavelets_b200.scatternet.lowlevel import scat_j1
from tests import sweep_util, util

pytestmark = pytest.mark.gpu
DEV = 'cuda'
SYM, ZERO = 1, 0
MODE_NAME = {SYM: 'symmetric', ZERO: 'zero'}


def _rev(name, key):
    return np.array(TABLES[name][key], dtype=np.float64)[::-1].copy()


def _f32(a):
    return np.asarray(a, dtype=np.float64).astype(np.float32)


# ---- the instantiations (dtcwt_fwd_stream.cuh try_launch_j1_any / try_launch_fwd_j2plus, dtcwt_inv_stream.cuh
#      try_launch_inv_j1 / try_launch_inv_j2plus) and the stored taps that reach them --------------------------------
PAIR_TAPS = {(5, 7): ('near_sym_a', 'h'), (7, 5): ('near_sym_a', 'g'), (9, 7): ('antonini', 'h'),
             (5, 3): ('legall', 'h'), (13, 19): ('near_sym_b', 'h'), (7, 9): ('antonini', 'g'),
             (3, 5): ('legall', 'g'), (19, 13): ('near_sym_b', 'g')}
SCAT_PAIRS = [(5, 7), (7, 5), (9, 7), (5, 3), (13, 19)]
QSHIFTS = {10: 'qshift_a', 14: 'qshift_b', 16: 'qshift_c', 18: 'qshift_d'}
ODD_PAIR = (11, 9)            # no instantiation: the generic kernel
ODD_QSHIFT = 'qshift_32'      # 32 taps: no instantiation


def pair_taps(pair):
    if pair == ODD_PAIR:
        rng = np.random.default_rng(77)
        return rng.uniform(-0.5, 0.5, 11), rng.uniform(-0.5, 0.5, 9)
    name, kind = PAIR_TAPS[pair]
    return _rev(name, kind + '0o'), _rev(name, kind + '1o')


def q_taps(name, kind):
    return [_rev(name, kind + s) for s in ('0a', '1a', '0b', '1b')]


def hla_j1(pair):
    m = max(pair) // 2
    return (m + 3) // 4 * 4


def hla_i2(mq):
    m2 = mq // 2
    omin, omax = (0, 3) if m2 % 2 == 0 else (1, 2)
    h = max(m2 - omin, m2 + omax - 3)
    return (h + 3) // 4 * 4


def chunk_counts(case):
    """(min, max) chunk count over every possible occupancy, from the kernel's own strip / chunk parameters."""
    N, C, H, W = case['shape']
    fam = case['family']
    if fam in ('fwd_j1', 'scat'):
        items, rows, unit, pro = (W + 63) // 64, H // 2, 8, 4
    elif fam == 'fwd_j2plus':
        items, rows, unit, pro = ((W // 4) + 31) // 32, H // 4, 4, 3
    else:
        items, rows, unit, pro = (W + 63) // 64, H // 2, 8, 8
    return sweep_util.chunk_range(N * C * items, rows, unit, pro)


# ---- case matrices ---------------------------------------------------------------------------------------------------
# fwd_j1 / ScatLayer: strips of 64 input columns, chunks of 8 quad rows (16 image rows); H = 38 leaves a short last
# chunk (19 quad rows).  fwd_j2plus: strips of 128 input columns, chunks of 4 quad rows (16 rows); H = 36 (9 quad rows).
# Inverses: strips of 64 low-pass columns, chunks of 8 complex rows (16 low-pass rows); H = 38 (19 complex rows).
J1_WIDTHS = [40, 64, 68, 256, 292]          # < 1 strip, 1 strip, 1 strip + 4 columns, 4 strips, partial 5th strip
J2_WIDTHS = [96, 128, 132, 384, 424]
INV_WIDTHS = [40, 64, 68, 192, 228]
SWEEP_NC = (2, 3)
MANY_CHUNKS, ONE_CHUNK = sweep_util.MANY_CHUNKS, sweep_util.ONE_CHUNK


_DEFAULTS = dict(mode=SYM, layout=(2, -1), pad=0, has_ll=True, has_hi=True, ll_trim=False, aux=False, magbias=1e-2,
                 regime=None)


def _case(family, key, shape, **kw):
    c = dict(_DEFAULTS, family=family, key=key, shape=shape, lo=-6, hi=6, canary=False)
    c.update(kw)
    c['id'] = '%s-%s-%s' % (family, '_'.join(map(str, key)) if isinstance(key, tuple) else key,
                            'x'.join(map(str, shape)))
    for k, v in _DEFAULTS.items():
        if c[k] != v:
            c['id'] += '-%s=%s' % (k, str(c[k]).replace(' ', ''))
    return c


def fwd_j1_cases():
    out = []
    for pair in PAIR_TAPS:
        for k, W in enumerate(J1_WIDTHS):
            out.append(_case('fwd_j1', pair, SWEEP_NC + (38, W), canary=(k == 4)))
    p = (5, 7)
    out += [
        _case('fwd_j1', p, (2, 3, 38, 66)),                              # W = 2 mod 4: rows not 16-byte aligned
        _case('fwd_j1', p, (2, 3, 38, 292), mode=ZERO),
        _case('fwd_j1', p, (1, 2, 214, 388), regime=MANY_CHUNKS),        # 107 quad rows
        _case('fwd_j1', p, (1000, 2, 14, 68), regime=ONE_CHUNK),          # 7 quad rows: a short single chunk
        _case('fwd_j1', p, (2, 3, 38, 292), layout=(1, 2)),
        _case('fwd_j1', p, (2, 3, 38, 292), layout=(3, 1)),
        _case('fwd_j1', p, (2, 3, 38, 256), pad=4),                      # row pitch W + 4: aligned, fast path
        _case('fwd_j1', p, (2, 3, 38, 256), pad=2),                      # row pitch W + 2: generic kernel
        _case('fwd_j1', ODD_PAIR, (2, 3, 38, 292), canary=True),
    ]
    return out


def fwd_j2_cases():
    out = []
    for mq in QSHIFTS:
        for k, W in enumerate(J2_WIDTHS):
            out.append(_case('fwd_j2plus', mq, SWEEP_NC + (36, W), canary=(k == 4)))
    m = 14
    out += [
        _case('fwd_j2plus', m, (1, 2, 212, 424), regime=MANY_CHUNKS),    # 53 quad rows
        _case('fwd_j2plus', m, (1000, 2, 12, 132), regime=ONE_CHUNK),    # 3 quad rows
        _case('fwd_j2plus', m, (2, 3, 36, 424), layout=(1, 2)),
        _case('fwd_j2plus', m, (2, 3, 36, 424), layout=(3, 1)),
        _case('fwd_j2plus', m, (2, 3, 36, 384), pad=4),
        _case('fwd_j2plus', m, (2, 3, 36, 384), pad=2),
        _case('fwd_j2plus', ODD_QSHIFT, (2, 3, 36, 424), canary=True),
    ]
    return out


def inv_j1_cases():
    out = []
    for pair in PAIR_TAPS:
        for k, W in enumerate(INV_WIDTHS):
            out.append(_case('inv_j1', pair, SWEEP_NC + (38, W), canary=(k == 4)))
    p = (7, 5)
    out += [
        _case('inv_j1', p, (2, 3, 38, 4)),                               # W < 2 HLA: generic kernel
        _case('inv_j1', (19, 13), (2, 3, 38, 20)),                       # W < 2 HLA = 24
        _case('inv_j1', p, (2, 3, 38, 228), mode=ZERO),
        _case('inv_j1', p, (2, 3, 38, 228), has_ll=False),
        _case('inv_j1', p, (2, 3, 38, 228), has_ll=False, mode=ZERO),
        _case('inv_j1', p, (2, 3, 38, 228), has_hi=False, mode=ZERO),   # low-pass only: always symmetric
        _case('inv_j1', p, (1, 2, 214, 388), regime=MANY_CHUNKS),
        _case('inv_j1', p, (1000, 2, 14, 68), regime=ONE_CHUNK),
        _case('inv_j1', p, (2, 3, 38, 228), layout=(1, 5)),              # ScatLayer backward: (n, o, c, h, w, re/im)
        _case('inv_j1', (5, 7), (2, 3, 38, 228), layout=(1, 5), mode=ZERO),
        _case('inv_j1', p, (2, 3, 38, 228), ll_trim=True),               # low-pass 2 rows taller: a view one row in
        _case('inv_j1', ODD_PAIR, (2, 3, 38, 228), canary=True),
    ]
    return out


def inv_j2_cases():
    out = []
    for mq in QSHIFTS:
        for k, W in enumerate(INV_WIDTHS):
            out.append(_case('inv_j2plus', mq, SWEEP_NC + (38, W), canary=(k == 4)))
    m = 18
    out += [
        _case('inv_j2plus', m, (2, 3, 38, 12)),                          # W < 2 HLA = 16: generic kernel
        _case('inv_j2plus', m, (2, 3, 38, 228), has_ll=False),
        _case('inv_j2plus', m, (2, 3, 38, 228), has_hi=False),
        _case('inv_j2plus', m, (1, 2, 214, 228), regime=MANY_CHUNKS),
        _case('inv_j2plus', m, (1000, 2, 14, 68), regime=ONE_CHUNK),
        _case('inv_j2plus', m, (2, 3, 38, 228), ll_trim=True),           # DTCWTInverse's row trim: a view one row in
        _case('inv_j2plus', ODD_QSHIFT, (2, 3, 38, 228), canary=True),
    ]
    return out


def scat_cases():
    out = []
    for pair in SCAT_PAIRS:
        for aux in (False, True):
            for k, W in enumerate(J1_WIDTHS):
                out.append(_case('scat', pair, SWEEP_NC + (38, W), aux=aux, canary=(k == 4)))
    p = (5, 7)
    for aux in (False, True):
        out += [
            _case('scat', p, (2, 3, 38, 292), aux=aux, mode=ZERO),
            # magbias 0 and planes down to 1e-18: the rescaled square root (sum of squares below 1e-30)
            _case('scat', p, (2, 3, 38, 292), aux=aux, magbias=0.0, lo=-18, hi=0),
            _case('scat', p, (2, 3, 38, 66), aux=aux),                   # W = 2 mod 4: generic kernel
            _case('scat', ODD_PAIR, (2, 3, 38, 292), aux=aux, canary=True),
        ]
    out += [
        _case('scat', p, (1, 2, 214, 388), aux=True, regime=MANY_CHUNKS),
        _case('scat', p, (1000, 2, 14, 68), aux=True, regime=ONE_CHUNK),
    ]
    return out


CASES = fwd_j1_cases() + fwd_j2_cases() + inv_j1_cases() + inv_j2_cases() + scat_cases()


def expected_kernel(c):
    """The kernel the dispatch rules pick: '<family>_stream<args>' or '<family>_tile'."""
    fam, key, (N, C, H, W) = c['family'], c['key'], c['shape']
    if fam in ('fwd_j1', 'scat'):
        pitch = W + c['pad']
        ok = key in (PAIR_TAPS if fam == 'fwd_j1' else SCAT_PAIRS) and pitch % 4 == 0
        if fam == 'scat':
            return 'fwd_j1_stream<%d,%d,%d>' % (key + (2 if c['aux'] else 1,)) if ok else 'scat_j1_tile'
        return 'fwd_j1_stream<%d,%d,0>' % key if ok else 'fwd_j1_tile'
    if fam == 'fwd_j2plus':
        ok = key in QSHIFTS and (W + c['pad']) % 4 == 0
        return 'fwd_j2plus_stream<%d>' % key if ok else 'fwd_j2plus_tile'
    if fam == 'inv_j1':
        ok = key in PAIR_TAPS and W % 4 == 0 and W >= 2 * hla_j1(key)
        return 'inv_j1_stream<%d,%d>' % key if ok else 'inv_j1_tile'
    ok = key in QSHIFTS and W % 4 == 0 and W >= 2 * hla_i2(key)
    return 'inv_j2plus_stream<%d>' % key if ok else 'inv_j2plus_tile'


ALL_STREAM_KERNELS = (['fwd_j1_stream<%d,%d,0>' % p for p in PAIR_TAPS] +
                      ['fwd_j1_stream<%d,%d,%d>' % (p + (s,)) for p in SCAT_PAIRS for s in (1, 2)] +
                      ['fwd_j2plus_stream<%d>' % m for m in QSHIFTS] +
                      ['inv_j1_stream<%d,%d>' % p for p in PAIR_TAPS] +
                      ['inv_j2plus_stream<%d>' % m for m in QSHIFTS])


# ---- running a case ----------------------------------------------------------------------------------------------------

def _permute_nc_first(a, names):
    order = [names.index(k) for k in ('n', 'c', 'o', 'h', 'w', 'r')]
    return np.transpose(np.asarray(a), order)


class Prepared(object):
    """Inputs (host fp32 + device tensors in the case's layout), taps, and the float64 / fp32 oracle outputs."""

    def __init__(self, c):
        self.c = c
        fam, key, (N, C, H, W) = c['family'], c['key'], c['shape']
        rng = np.random.default_rng(zlib.crc32(c['id'].encode()))
        if fam in ('fwd_j1', 'scat', 'fwd_j2plus'):
            self.x, self.sc = util.scaled_uniform((N, C, H, W), rng, c['lo'], c['hi'])
            self.s = util.plane_max(self.x)
            big = np.zeros((N, C, H, W + c['pad']), np.float32)
            big[..., :W] = self.x
            self.xt = torch.from_numpy(big).to(DEV)[..., :W]
            if fam == 'fwd_j2plus':
                self.taps = q_taps(key if isinstance(key, str) else QSHIFTS[key], 'h')
            else:
                self.taps = list(pair_taps(key))
        else:
            h2, w2 = H // 2, W // 2
            ll, self.sc = util.scaled_uniform((N, C, H, W), rng, c['lo'], c['hi'])
            hi, _ = util.scaled_uniform((N, C, 6, h2, w2, 2), rng, scales=self.sc)
            self.ll = ll if c['has_ll'] else None
            self.hi = hi if c['has_hi'] else None
            self.s = util.plane_max(self.ll, self.hi)
            o_dim, ri_dim = c['layout']
            self.names = orc._dim_names(o_dim, ri_dim)
            self.hi_layout = None
            if self.hi is not None:
                inv = [('n', 'c', 'o', 'h', 'w', 'r').index(k) for k in self.names]
                self.hi_layout = np.ascontiguousarray(np.transpose(self.hi, inv))
            self.llt = self.hit = None
            if self.ll is not None:
                if c['ll_trim']:
                    big = rng.uniform(-1, 1, (N, C, H + 2, W)).astype(np.float32) * 1e6   # rows 0, H+1 are dropped
                    big[:, :, 1:-1] = self.ll
                    self.llt = torch.from_numpy(big).to(DEV)
                    if fam == 'inv_j2plus':
                        self.llt = self.llt[:, :, 1:-1]
                else:
                    self.llt = torch.from_numpy(self.ll).to(DEV)
            if self.hi is not None:
                self.hit = torch.from_numpy(self.hi_layout).to(DEV)
            self.taps = (q_taps(key if isinstance(key, str) else QSHIFTS[key], 'g') if fam == 'inv_j2plus'
                         else list(pair_taps(key)))
        self.t64 = [_f32(t).astype(np.float64) for t in self.taps]

    # -- the level functions (auto dispatch, or the generic kernel) --
    def run(self, generic=False):
        c, fam = self.c, self.c['family']
        ctx = _ffi.generic_kernels() if generic else contextlib.nullcontext()
        with ctx:
            if fam == 'fwd_j1':
                o5, ri = tf.get_dimensions5(*c['layout'])[:2]
                ll, hi = tf.fwd_j1(self.xt, *self.taps, False, o5, ri, c['mode'])
                return {'ll': ll, 'highs': hi}
            if fam == 'fwd_j2plus':
                o5, ri = tf.get_dimensions5(*c['layout'])[:2]
                ll, hi = tf.fwd_j2plus(self.xt, *self.taps, False, o5, ri)
                return {'ll': ll, 'highs': hi}
            if fam == 'scat':
                z, dre, dim = scat_j1(self.xt, *self.taps, c['mode'], c['magbias'], c['aux'])
                return {'z': z, 'dre': dre, 'dim': dim}
            o5, ri = tf.get_dimensions5(*c['layout'])[:2]
            if fam == 'inv_j1':
                return {'y': tf.inv_j1(self.llt, self.hit, *self.taps, o5, ri, c['mode'])}
            return {'y': tf.inv_j2plus(self.llt, self.hit, *self.taps, o5, ri)}

    def oracle(self, dtype):
        c, fam = self.c, self.c['family']
        t = [a.astype(dtype) for a in self.t64]
        o_dim, ri_dim = c['layout']
        m = MODE_NAME[c['mode']]
        if fam == 'fwd_j1':
            ll, hi = orc.dtcwt_fwd_j1(self.x.astype(dtype), *t, False, o_dim, ri_dim, m)
            return {'ll': ll, 'highs': hi}
        if fam == 'fwd_j2plus':
            ll, hi = orc.dtcwt_fwd_j2plus(self.x.astype(dtype), *t, False, o_dim, ri_dim)
            return {'ll': ll, 'highs': hi}
        if fam == 'scat':
            z, dre, dim = orc.scat_j1(self.x.astype(dtype), *t, m, c['magbias'], True)
            return {'z': z, 'dre': dre, 'dim': dim}
        ll = None if self.ll is None else self.ll.astype(dtype)
        hi = None if self.hi is None else self.hi_layout.astype(dtype)
        if fam == 'inv_j1':
            return {'y': orc.dtcwt_inv_j1(ll, hi, *t, o_dim, ri_dim, m)}
        return {'y': orc.dtcwt_inv_j2plus(ll, hi, *t, o_dim, ri_dim)}


def _np(t):
    return None if t is None else t.detach().cpu().numpy()


def check_case(c):
    P = Prepared(c)
    fam = c['family']
    got = {k: _np(v) for k, v in P.run().items()}
    gen = {k: _np(v) for k, v in P.run(generic=True).items()}
    o64 = P.oracle(np.float64)
    what = c['id']
    if fam in ('fwd_j1', 'fwd_j2plus'):
        names = orc._dim_names(*c['layout'])
        bounds = (util.bound_fwd_j1 if fam == 'fwd_j1' else util.bound_fwd_j2plus)(*P.t64)
        # (a) bit-identical to the generic kernel
        assert np.array_equal(got['ll'], gen['ll']), what + ': low-pass differs from the generic kernel'
        assert np.array_equal(got['highs'], gen['highs']), what + ': band-pass differs from the generic kernel'
        # (b) low-pass bit-identical to the fp32 oracle
        o32 = P.oracle(np.float32)
        assert np.array_equal(got['ll'], o32['ll']), what + ': low-pass differs from the fp32 oracle'
        # (c) per-plane bound against the float64 oracle
        G, K = bounds['ll']
        util.assert_plane_bound(got['ll'], o64['ll'], P.s, G, K, what=what + ' ll')
        G, K = bounds['highs']
        util.assert_plane_bound(_permute_nc_first(got['highs'], names), _permute_nc_first(o64['highs'], names),
                                P.s, G, K, what=what + ' highs')
        return
    if fam == 'scat':
        b = util.bound_scat(*P.t64, c['magbias'])
        sw = lambda a: np.swapaxes(a, 1, 2)  # noqa: E731  (N, 7|6, C, h, w) -> (N, C, 7|6, h, w)
        for name, y in (('stream', got), ('generic', gen)):
            for part, sl in (('avg', slice(0, 1)), ('mag', slice(1, 7))):
                G, K, add = b[part]
                util.assert_plane_bound(sw(y['z'])[:, :, sl], sw(o64['z'])[:, :, sl], P.s, G, K, add,
                                        '%s %s %s' % (what, name, part))
        for part, sl in (('avg', slice(0, 1)), ('mag', slice(1, 7))):
            G, K, add = b[part]
            util.assert_plane_bound(sw(got['z'])[:, :, sl], sw(gen['z'])[:, :, sl], P.s, G, 2 * K, add,
                                    what + ' stream vs generic ' + part)
        if c['aux']:
            G, K = b['band']
            band_err = (K * util.U32 * G * P.s)[:, None, :, None, None]
            r64 = o64['z'][:, 1:] + c['magbias']
            for k in ('dre', 'dim'):
                util.assert_ratio_bound(got[k], o64[k], band_err, r64, '%s %s' % (what, k))
                util.assert_ratio_bound(gen[k], o64[k], band_err, r64, '%s generic %s' % (what, k))
        else:
            assert got['dre'] is None and got['dim'] is None
        return
    G, K = (util.bound_inv_j1 if fam == 'inv_j1' else util.bound_inv_j2plus)(*P.t64, has_ll=c['has_ll'],
                                                                          has_hi=c['has_hi'])
    util.assert_plane_bound(got['y'], o64['y'], P.s, G, K, what=what + ' stream vs float64')
    util.assert_plane_bound(gen['y'], o64['y'], P.s, G, K, what=what + ' generic vs float64')
    # two fp32 results, each within K of the float64 value, are within 2 K of each other
    util.assert_plane_bound(got['y'], gen['y'], P.s, G, 2 * K, what=what + ' stream vs generic')


@pytest.fixture(scope='module', autouse=True)
def _native_library_is_loaded():
    assert torch.cuda.is_available()
    assert _ffi.lib().b200w_version() >= 100
    yield


@pytest.mark.parametrize('c', CASES, ids=[c['id'] for c in CASES])
def test_stream_sweep(c):
    check_case(c)


def test_case_matrix_covers_the_kernels_and_both_chunk_regimes():
    """The matrix reaches every streaming instantiation, and the cases labelled with a chunk regime are in it for every
    occupancy the kernel could have."""
    assert sorted(set(expected_kernel(c) for c in CASES if '_stream' in expected_kernel(c))) == sorted(ALL_STREAM_KERNELS)
    assert len(ALL_STREAM_KERNELS) == 34
    for c in CASES:
        if c['regime'] == MANY_CHUNKS:
            assert chunk_counts(c)[0] >= 4, c['id']
        elif c['regime'] == ONE_CHUNK:
            assert chunk_counts(c) == (1, 1), c['id']


# ---- (d) unwritten outputs and stray writes, through the C ABI ---------------------------------------------------------

Canaried = sweep_util.Canaried


@pytest.mark.parametrize('c', [c for c in CASES if c['canary']], ids=[c['id'] for c in CASES if c['canary']])
def test_canaries_and_unwritten_outputs(c):
    P = Prepared(c)
    L = _ffi.lib()
    fam, (N, C, H, W) = c['family'], c['shape']
    taps = [_ffi.host_taps(t) for t in P.taps]
    x = P.xt.contiguous() if fam in ('fwd_j1', 'fwd_j2plus', 'scat') else None
    st = _ffi.stream_of(x if x is not None else P.hit)
    if fam == 'fwd_j1':
        shape, hs = tf.highs_shape_strides(N, C, H // 2, W // 2, 2, 5)
        outs = [Canaried((N, C, H, W)), Canaried(shape)]
        rc = L.b200w_dtcwt_fwd_j1(x.data_ptr(), H * W, W, outs[0].ptr(), H * W, W, outs[1].ptr(), _ffi.hs_array(hs),
                                  N, C, H, W, taps[0].ptr, taps[0].n, taps[1].ptr, taps[1].n, c['mode'], st)
    elif fam == 'fwd_j2plus':
        shape, hs = tf.highs_shape_strides(N, C, H // 4, W // 4, 2, 5)
        outs = [Canaried((N, C, H // 2, W // 2)), Canaried(shape)]
        rc = L.b200w_dtcwt_fwd_j2plus(x.data_ptr(), H * W, W, outs[0].ptr(), (H // 2) * (W // 2), W // 2,
                                      outs[1].ptr(), _ffi.hs_array(hs), N, C, H, W,
                                      *[t.ptr for t in taps], taps[0].n, st)
    elif fam == 'scat':
        outs = [Canaried((N, 7, C, H // 2, W // 2))]
        if c['aux']:
            outs += [Canaried((N, 6, C, H // 2, W // 2)), Canaried((N, 6, C, H // 2, W // 2))]
        rc = L.b200w_scat_j1(x.data_ptr(), outs[0].ptr(), outs[1].ptr() if c['aux'] else None,
                             outs[2].ptr() if c['aux'] else None, N, C, H, W, taps[0].ptr, taps[0].n, taps[1].ptr,
                             taps[1].n, c['mode'], c['magbias'], st)
    else:
        ll = P.llt.contiguous()
        _, hs = tf.highs_shape_strides(N, C, H // 2, W // 2, 2, 5)
        if fam == 'inv_j1':
            outs = [Canaried((N, C, H, W))]
            rc = L.b200w_dtcwt_inv_j1(ll.data_ptr(), H * W, W, P.hit.data_ptr(), _ffi.hs_array(hs), outs[0].ptr(),
                                      H * W, W, N, C, H, W, taps[0].ptr, taps[0].n, taps[1].ptr, taps[1].n, c['mode'],
                                      st)
        else:
            outs = [Canaried((N, C, 2 * H, 2 * W))]
            rc = L.b200w_dtcwt_inv_j2plus(ll.data_ptr(), H * W, W, P.hit.data_ptr(), _ffi.hs_array(hs),
                                          outs[0].ptr(), 4 * H * W, 2 * W, N, C, H, W, *[t.ptr for t in taps],
                                          taps[0].n, st)
    assert rc == 0, rc
    torch.cuda.synchronize()
    for k, o in enumerate(outs):
        o.check('%s output %d' % (c['id'], k))
    ref = P.run()
    ref = [v for v in ref.values() if v is not None]
    for o, r in zip(outs, ref):
        assert torch.equal(o.t, r), c['id'] + ': C ABI call and level function differ'


# ---- (e) which kernel each case launched -------------------------------------------------------------------------------

_short = sweep_util.kernel_namer(['fwd_j1_stream', 'fwd_j2plus_stream', 'inv_j1_stream', 'inv_j2plus_stream'],
                                 ['fwd_j1', 'fwd_j2plus', 'inv_j1', 'inv_j2plus', 'scat_j1'])


def test_dispatch_launches_the_expected_kernel():
    """One auto-dispatch call per case under a torch.profiler CUDA trace: the engine kernel it launched is the streaming
    instantiation the dispatch rules predict, or the generic tile kernel for the fallback cases -- so a width that
    silently fell back cannot turn test_stream_sweep's comparison with the generic kernel into a self-comparison."""
    prepared = [Prepared(c) for c in CASES]
    seen = sweep_util.traced_kernels(lambda: [P.run() for P in prepared], _short)
    if seen is None:
        pytest.skip('CUDA activity tracing is unavailable or recorded no kernels')
    want = [expected_kernel(c) for c in CASES]
    assert len(seen) == len(want), (len(seen), len(want))
    wrong = [(c['id'], w, s) for c, w, s in zip(CASES, want, seen) if w != s]
    assert not wrong, wrong[:10]
    assert sorted(set(s for s in seen if '_stream' in s)) == sorted(ALL_STREAM_KERNELS)
