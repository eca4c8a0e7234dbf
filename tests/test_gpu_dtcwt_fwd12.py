"""GPU: DTCWT forward levels 1 and 2 in one call (csrc/dtcwt_fwd12.cuh, b200w_dtcwt_fwd_j12, FWD_J12).

  * the fused kernel (or, where its plan rejects the call, the two level kernels behind the same entry) is bit-identical
    to the per-level route (fwd_j1, then fwd_j2plus on its low-pass) and its LL2 to the float32 oracle composition:
    widths at the mirror corner cases, the bench width and just past the kernel's width limit, heights in the
    one-band and many-band regimes with a short last band, both level-1 modes, every o_dim / ri_dim layout, skipped
    level-2 band-passes, a row pitch larger than W, a channel slice and a base address that is not 16-byte aligned;
  * NaN-filled outputs between canaries through the C ABI, and a profiler trace (in a child process) of the kernels
    each call launches;
  * DTCWTForward routes levels 1 + 2 through FWD_J12 exactly when it may, and its gradients are the two-Function
    path's bit for bit; one run at the bench shape.
"""
import itertools
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import pytorch_wavelets_b200 as pw
from oracle import oracle as orc
from pytorch_wavelets_b200 import _ffi
from pytorch_wavelets_b200.dtcwt import transform_funcs as tf
from pytorch_wavelets_b200.dwt.lowlevel import mode_to_int
from tests import sweep_util

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FUSED = 'dtcwt_fwd12_band<5,7,10>'
LEVELS = ['fwd_j1_stream<5,7,0>', 'fwd_j2plus_stream<10>']
MAX_W = 1024          # widest plane the fused kernel holds (4 columns per thread, 256 threads)


def _taps():
    m = pw.DTCWTForward(biort='near_sym_a', qshift='qshift_a')
    return [getattr(m, k).detach().cpu().numpy().ravel().copy() for k in ('h0o', 'h1o', 'h0a', 'h1a', 'h0b', 'h1b')]


TAPS = _taps()


def _input(N, C, H, W, seed=0, pitch=None):
    """Standard normal planes scaled by per-plane powers of ten (a plane mix-up cannot go unnoticed)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, C, H, pitch or W, generator=g)
    x *= (10.0 ** (torch.arange(N * C, dtype=torch.float32) % 7 - 3)).view(N, C, 1, 1)
    return x.cuda()[..., :W]


def _per_level(x, skip1, o5, ri, mode):
    ll1, h0 = tf.fwd_j1(x, TAPS[0], TAPS[1], False, o5, ri, mode)
    ll2, h1 = tf.fwd_j2plus(ll1, *TAPS[2:], skip1, o5, ri)
    return ll2, h0, h1


def _check_equal(x, skip1=False, o_dim=2, ri_dim=-1, mode=1, oracle=True):
    o5, ri = tf.get_dimensions5(o_dim, ri_dim)[:2]
    got = tf.fwd_j12(x, *TAPS, skip1, o5, ri, mode)
    want = _per_level(x, skip1, o5, ri, mode)
    for name, a, b in zip(('ll2', 'yh0', 'yh1'), got, want):
        if b is None:
            assert a is None, name
            continue
        assert a.shape == b.shape, name
        assert torch.equal(a, b), '%s differs from the per-level route, %s' % (name, tuple(x.shape))
    if oracle:
        xn = x.cpu().numpy()
        oll1, _ = orc.dtcwt_fwd_j1(xn, TAPS[0], TAPS[1], True, o_dim, ri_dim, 'symmetric' if mode == 1 else 'zero')
        oll2, _ = orc.dtcwt_fwd_j2plus(oll1, *TAPS[2:], True, o_dim, ri_dim)
        assert np.array_equal(got[0].cpu().numpy(), oll2), 'll2 differs from the oracle, %s' % (tuple(x.shape),)


# widths: the mirror corner cases (W = 4 falls back), odd multiples of 4, the bench width, just past the width limit
@pytest.mark.parametrize('W', [4, 8, 12, 64, 100, 512, 1024, MAX_W + 4])
@pytest.mark.parametrize('mode', [1, 0])
def test_widths_match_the_per_level_route(W, mode):
    _check_equal(_input(1, 2, 24, W, seed=W), mode=mode, oracle=W <= 512)


# heights: one band per plane (many planes), many bands per plane (one tall plane), a short last band, tiny planes
@pytest.mark.parametrize('N,C,H,W', [(40, 50, 64, 64), (1, 1, 512, 64), (1, 1, 520, 64), (1, 1, 20, 512),
                                     (1, 1, 24, 64), (1, 1, 28, 512), (1, 2, 1028, 128), (2, 3, 200, 1024)])
def test_band_regimes_match_the_per_level_route(N, C, H, W):
    _check_equal(_input(N, C, H, W, seed=H), oracle=N * C * H * W <= (1 << 20))


@pytest.mark.parametrize('o_dim,ri_dim', [(o, r) for o, r in itertools.product(range(1, 6), [1, 2, 3, 4, 5, -1])
                                          if o != r % 6])
def test_every_layout_matches_the_per_level_route(o_dim, ri_dim):
    _check_equal(_input(2, 2, 24, 28, seed=o_dim * 7 + ri_dim), o_dim=o_dim, ri_dim=ri_dim)


@pytest.mark.parametrize('mode', [1, 0])
def test_skipped_level2_band_pass(mode):
    _check_equal(_input(2, 3, 72, 96, seed=3), skip1=True, mode=mode)


def test_pitched_sliced_and_unaligned_inputs():
    _check_equal(_input(2, 3, 40, 96, seed=4, pitch=104))                # row pitch > W
    _check_equal(_input(2, 5, 40, 96, seed=5)[:, 1:4])                   # channel slice
    flat = _input(1, 1, 1, 2 * 48 * 64 + 1, seed=6).reshape(-1)
    _check_equal(flat[1:].view(1, 2, 48, 64))                            # base address not 16-byte aligned


def _abi_call(x, ll2, yh0, yh1, hs0, hs1, ws=None, ws_bytes=0, generic=False):
    N, C, H, W = x.shape
    x, xps, xpitch = _ffi.planes_view(x)
    f = [_ffi.host_taps(t) for t in TAPS]
    fn = getattr(_ffi.lib(), 'b200w_dtcwt_fwd_j12' + ('_generic' if generic else ''))
    return fn(x.data_ptr(), xps, xpitch, ll2, (H // 2) * (W // 2), W // 2, yh0, _ffi.hs_array(hs0), yh1,
              _ffi.hs_array(hs1), N, C, H, W, f[0].ptr, f[0].n, f[1].ptr, f[1].n, f[2].ptr, f[3].ptr, f[4].ptr,
              f[5].ptr, f[2].n, 1, ws, ws_bytes, _ffi.stream_of(x))


def test_canaried_outputs_of_the_fused_kernel():
    """Every output element written once, nothing written outside the outputs (the one instantiation, on a plane the
    plan accepts, with several bands)."""
    N, C, H, W = 1, 3, 136, 520
    x = _input(N, C, H, W, seed=9)
    assert _ffi.lib().b200w_dtcwt_fwd_j12_workspace(x.data_ptr(), H * W, W, 16, N, C, H, W, 5, 7, 10) == 0
    sh0, hs0 = tf.highs_shape_strides(N, C, H // 2, W // 2, 2, 5)
    sh1, hs1 = tf.highs_shape_strides(N, C, H // 4, W // 4, 2, 5)
    ll2, yh0, yh1 = (sweep_util.Canaried(s) for s in ((N, C, H // 2, W // 2), sh0, sh1))
    assert _abi_call(x, ll2.ptr(), yh0.ptr(), yh1.ptr(), hs0, hs1) == 0
    torch.cuda.synchronize()
    for name, buf in (('ll2', ll2), ('yh0', yh0), ('yh1', yh1)):
        buf.check(name)
    want = _per_level(x, False, 2, 5, 1)
    for a, b in zip((ll2.t, yh0.t, yh1.t), want):
        assert torch.equal(a, b)


def test_generic_entry_and_workspace_rule():
    N, C, H, W = 2, 2, 32, 48
    x = _input(N, C, H, W, seed=10)
    sh0, hs0 = tf.highs_shape_strides(N, C, H // 2, W // 2, 2, 5)
    sh1, hs1 = tf.highs_shape_strides(N, C, H // 4, W // 4, 2, 5)
    ll2, yh0, yh1 = x.new_empty((N, C, H // 2, W // 2)), x.new_empty(sh0), x.new_empty(sh1)
    ws = x.new_empty((N * C * H * W,))
    assert _abi_call(x, ll2.data_ptr(), yh0.data_ptr(), yh1.data_ptr(), hs0, hs1, generic=True) == -3   # no workspace
    assert _abi_call(x, ll2.data_ptr(), yh0.data_ptr(), yh1.data_ptr(), hs0, hs1, ws.data_ptr(), 4 * ws.numel() - 4,
                     generic=True) == -3
    assert _abi_call(x, ll2.data_ptr(), yh0.data_ptr(), yh1.data_ptr(), hs0, hs1, ws.data_ptr(), 4 * ws.numel(),
                     generic=True) == 0
    want = _per_level(x, False, 2, 5, 1)
    for a, b in zip((ll2, yh0, yh1), want):
        assert torch.equal(a, b)
    # level 1 without its band-pass: the two level kernels through the workspace
    assert _ffi.lib().b200w_dtcwt_fwd_j12_workspace(x.data_ptr(), H * W, W, None, N, C, H, W, 5, 7, 10) == 4 * N * C * H * W


# ---- which kernels run: one profiler session in a child process --------------------------------------------------------

def _calls():
    """(call, predicted kernels) pairs covering the fused route and every fallback class."""
    def fused(x):
        return lambda: tf.fwd_j12(x, *TAPS, False, 2, 5, 1)
    flat = _input(1, 1, 1, 64 * 64 + 1, seed=6).reshape(-1)
    m3 = pw.DTCWTForward(J=3).cuda()
    m_scale = pw.DTCWTForward(J=3, include_scale=[True, False, False]).cuda()
    m_skip = pw.DTCWTForward(J=2, skip_hps=[True, False]).cuda()
    m1 = pw.DTCWTForward(J=1).cuda()
    return [
        (fused(_input(1, 3, 64, 1024)), [FUSED]),
        (fused(_input(1, 3, 64, 8)), [FUSED]),
        (fused(_input(1, 3, 64, 4)), LEVELS),                           # narrower than the mirror rule
        (fused(_input(1, 3, 64, MAX_W + 4)), LEVELS),                   # wider than the kernel holds
        (fused(flat[1:].view(1, 1, 64, 64)), ['fwd_j1_tile', 'fwd_j2plus_stream<10>']),   # unaligned base
        (lambda: m3(_input(1, 3, 64, 64)), [FUSED, 'fwd_j2plus_stream<10>']),
        (lambda: m3(_input(1, 3, 63, 63)), [FUSED, 'fwd_j2plus_stream<10>']),     # odd sizes pad to 64 x 64
        (lambda: m3(_input(1, 3, 62, 64)), LEVELS + ['fwd_j2plus_stream<10>']),   # 62 % 4 != 0
        (lambda: m_scale(_input(1, 3, 64, 64)), LEVELS + ['fwd_j2plus_stream<10>']),
        (lambda: m_skip(_input(1, 3, 64, 64)), ['fwd_j1_tile', 'fwd_j2plus_stream<10>']),
        (lambda: m1(_input(1, 3, 64, 64)), LEVELS[:1]),
    ]


def trace_in_this_process():
    namer = sweep_util.kernel_namer(['dtcwt_fwd12_band', 'fwd_j1_stream', 'fwd_j2plus_stream'],
                                    ['fwd_j1', 'fwd_j2plus'])
    calls = _calls()
    got = []
    for c, _ in calls:
        ks = sweep_util.traced_kernels(c, namer)
        if ks is None:
            return None, None
        got.append(ks)
    return got, [w for _, w in calls]


def test_trace_shows_the_predicted_kernels():
    code = ('import json; from tests import test_gpu_dtcwt_fwd12 as t; '
            'print(json.dumps(t.trace_in_this_process()))')
    r = subprocess.run([sys.executable, '-c', code], cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    got, want = json.loads(r.stdout.strip().splitlines()[-1])
    if got is None:
        pytest.skip('no CUDA activity trace on this machine')
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, (i, g, w)


# ---- the module ---------------------------------------------------------------------------------------------------------

def _two_function_forward(m, x):
    """DTCWTForward.forward with every level on its own Function (the route before FWD_J12)."""
    mode = mode_to_int(m.mode)
    low, h = tf.FWD_J1.apply(x, m.h0o, m.h1o, m.skip_hps[0], m.o_dim, m.ri_dim, mode)
    highs = [h]
    for j in range(1, m.J):
        low, h = tf.FWD_J2PLUS.apply(low, m.h0a, m.h1a, m.h0b, m.h1b, m.skip_hps[j], m.o_dim, m.ri_dim, mode)
        highs.append(h)
    return low, highs


@pytest.mark.parametrize('J,skip1,mode', [(2, False, 'symmetric'), (3, False, 'zero'), (3, True, 'symmetric')])
def test_module_forward_and_gradients_match_the_two_function_path(J, skip1, mode):
    m = pw.DTCWTForward(J=J, skip_hps=[False, skip1] + [False] * (J - 2), mode=mode).cuda()
    x0 = _input(2, 3, 96, 128, seed=J)
    outs, grads = [], []
    for fwd in (m, lambda x: _two_function_forward(m, x)):
        x = x0.clone().requires_grad_(True)
        low, highs = fwd(x)
        g = torch.Generator(device='cuda').manual_seed(5)
        loss = (low * torch.randn(low.shape, generator=g, device='cuda')).sum()
        for h in highs:
            if h.dim():
                loss = loss + (h * torch.randn(h.shape, generator=g, device='cuda')).sum()
        loss.backward()
        outs.append([low.detach()] + [h.detach() for h in highs])
        grads.append(x.grad)
    for a, b in zip(*outs):
        assert a.shape == b.shape and torch.equal(a, b)
    assert torch.equal(grads[0], grads[1])


def test_bench_shape():
    """64 x 3 x 1024^2, J = 3: the module (fused levels 1 + 2) against the two-Function path."""
    m = pw.DTCWTForward(J=3, biort='near_sym_a', qshift='qshift_a').cuda()
    x = torch.randn(64, 3, 1024, 1024, device='cuda', generator=torch.Generator(device='cuda').manual_seed(11))
    with torch.no_grad():
        low, highs = m(x)
        low2, highs2 = _two_function_forward(m, x)
    same = torch.equal(low, low2) and all(torch.equal(a, b) for a, b in zip(highs, highs2))
    del x, low, highs, low2, highs2
    torch.cuda.empty_cache()     # (about 8 GB: hand it back to the tests that follow)
    assert same
