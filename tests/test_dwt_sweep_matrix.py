"""CPU checks of the DWT boundary sweep's case matrix (tests/dwt_sweep_cases.py): with the shipped pyramid plan and the
dispatch rules, the cases reach every streaming / fused DWT kernel instantiation that a 227 KB device can run, the one
that it cannot run is unreachable for every shape, and the cases labelled with a row-chunk regime are in it at every
occupancy."""
import collections

from tests import dwt_sweep_cases as dc
from tests.emu import emu_backend as eb
from tests.sweep_util import MANY_CHUNKS, ONE_CHUNK


def test_case_ids_are_unique():
    ids = [c['id'] for c in dc.CASES]
    assert len(ids) == len(set(ids)), [k for k, v in collections.Counter(ids).items() if v > 1]


def test_matrix_reaches_every_instantiation():
    assert len(dc.ALL_KERNELS) == len(set(dc.ALL_KERNELS)) == 72
    seen = set(k for c in dc.CASES for k in dc.expected_kernels(c) if not k.endswith('_tile'))
    assert seen <= set(dc.ALL_KERNELS), sorted(seen - set(dc.ALL_KERNELS))
    assert sorted(set(dc.ALL_KERNELS) - seen) == sorted(dc.UNREACHABLE)
    # ... and every one of them runs once into canaried NaN-filled outputs
    canaried = set(k for c in dc.CASES if c['canary'] for k in dc.expected_kernels(c) if not k.endswith('_tile'))
    assert canaried == seen, sorted(seen - canaried)
    # the fallback / rejected-plan cases are labelled as such and take the kernels the rules say
    for c in dc.CASES:
        ks = dc.expected_kernels(c)
        if c['label'] == 'fallback':
            assert ks == [c['family'] + '2d_tile'], (c['id'], ks)
        elif c['family'] in ('afb', 'sfb'):
            assert not ks[0].endswith('_tile'), (c['id'], ks)


def test_pyramid_routes_and_edges():
    routes = collections.Counter()
    for c in dc.CASES:
        if c['family'] != 'pyr':
            continue
        pol, _ = dc.dwt_policy(c)
        routes[(pol, c['J'])] += 1
        if c['label'] == 'edge':
            assert pol != 'all', c['id']       # the plan rejects the whole pyramid: level 1 only, or level kernels
    assert routes[('all', 4)] >= 5 and routes[('first', 2)] >= 6 and routes[('first', 3)] >= 6
    assert routes[('levels', 1)] >= 1 and routes[('levels', 3)] >= 1


def test_pyramid_with_ten_taps_never_needs_512_threads():
    """dwt_pyramid<10, 512, 1, 1> is unreachable on a 227 KB device: of the plans the policy asks for (one level at any
    width, several levels from 512 columns), every one for 10 taps that would need more than 256 threads exceeds the
    shared memory per block, whatever the height.  (Narrower multi-level plans can fit, but only level 1 of those is ever
    fused.)"""
    for J in (1, 2, 3, 4):
        for W in range(12 if J == 1 else 512, 2400, 4):
            for H in (28, 64, 130):
                d = eb.plan_pyramid(2, H, W, J, 10, 'symmetric')
                assert d is None or d['threads'] <= 256, (J, H, W)


def test_analysis_widths_cover_the_strip_boundaries():
    for L in dc.LS:
        for mode in ('symmetric', 'zero', 'reflect', 'periodic', 'periodization'):
            cs = [c for c in dc.CASES if c['family'] == 'afb' and c['L'] == L and c['mode'] == mode]
            wo = set(dc.orc.coeff_len(c['shape'][3], L, mode) for c in cs)
            assert set(dc.AFB_WO) <= wo, (L, mode, wo)
            win = set(c['shape'][3] % 4 for c in cs)
            assert {1, 2} <= win or {3, 2} <= win or {1, 3} <= win, (L, mode, win)


def test_chunk_regimes():
    regimes = collections.Counter()
    for c in dc.CASES:
        if c['regime'] == MANY_CHUNKS:
            assert dc.chunk_counts(c)[0] >= 4, c['id']
        elif c['regime'] == ONE_CHUNK:
            assert dc.chunk_counts(c) == (1, 1), c['id']
        regimes[(c['family'], c['regime'])] += 1
    for fam in ('afb', 'sfb'):
        assert regimes[(fam, MANY_CHUNKS)] >= 2 and regimes[(fam, ONE_CHUNK)] >= 2
