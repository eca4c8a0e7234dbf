"""numpy wrappers over the host emulation of the shipped tile kernels (tests/emu/emu.cpp).
TEST ONLY -- same per-level call signatures as oracle/oracle.py so tests can swap them; like the oracle, the
precision follows the input arrays (float32, or float64 for the `_f64` kernels)."""
import ctypes
import os
import subprocess

import numpy as np

from oracle import oracle as orc

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, 'libb200wave_emu.so')
        srcs = [os.path.join(_HERE, 'emu.cpp')] + [
            os.path.join(_ROOT, 'pytorch_wavelets_b200', 'csrc', f)
            for f in ('common.h', 'tile_kernels.h', 'launch_params.h', 'pyramid_plan.h')]
        if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
            subprocess.check_call(['g++', '-O2', '-fPIC', '-fopenmp', '-ffp-contract=off', '-std=c++17',
                                   '-Wno-unknown-pragmas', '-shared', '-o', so, srcs[0]])
        _LIB = ctypes.CDLL(so)
    return _LIB


def _p(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def _fn(name, dtype):
    """The float32 or float64 emulation of one entry point."""
    sfx = {np.dtype(np.float32): '', np.dtype(np.float64): '_f64'}[np.dtype(dtype)]
    return getattr(lib(), name + sfx)


def _t(f, dtype):
    return np.ascontiguousarray(np.asarray(f, dtype=np.float64).ravel().astype(dtype))


def _dtype(a):
    return a.dtype if a.dtype == np.float64 else np.dtype(np.float32)


LL = ctypes.c_longlong


def dwt_afb2d(x, fw_lo, fw_hi, fh_lo, fh_hi, mode):
    dt = _dtype(x)
    x = np.ascontiguousarray(x, dt)
    N, C, H, W = x.shape
    m = orc.mode_int(mode)
    fw_lo, fw_hi, fh_lo, fh_hi = [_t(f, dt) for f in (fw_lo, fw_hi, fh_lo, fh_hi)]
    Ho, Wo = orc.coeff_len(H, fh_lo.size, m), orc.coeff_len(W, fw_lo.size, m)
    ll = np.full((N, C, Ho, Wo), np.nan, dt)
    highs = np.full((N, C, 3, Ho, Wo), np.nan, dt)
    rc = _fn('emu_dwt_afb2d', dt)(_p(x), LL(H * W), W, _p(ll), LL(Ho * Wo), Wo, _p(highs), N * C, H, W,
                             _p(fw_lo), _p(fw_hi), fw_lo.size, _p(fh_lo), _p(fh_hi), fh_lo.size, m)
    assert rc == 0, rc
    return ll, highs


def dwt_sfb2d(ll, highs, gh_lo, gh_hi, gw_lo, gw_hi, mode, out_hw=None):
    dt = _dtype(ll)
    ll = np.ascontiguousarray(ll, dt)
    N, C, Hc, Wc = ll.shape
    m = orc.mode_int(mode)
    if highs is not None:
        highs = np.ascontiguousarray(highs, dt)
    gh_lo, gh_hi, gw_lo, gw_hi = [_t(f, dt) for f in (gh_lo, gh_hi, gw_lo, gw_hi)]
    Ho, Wo = orc.rec_len(Hc, gh_lo.size, m), orc.rec_len(Wc, gw_lo.size, m)
    if out_hw is not None:
        Ho, Wo = min(Ho, out_hw[0]), min(Wo, out_hw[1])
    y = np.full((N, C, Ho, Wo), np.nan, dt)
    rc = _fn('emu_dwt_sfb2d', dt)(_p(ll), LL(Hc * Wc), Wc, _p(highs), _p(y), LL(Ho * Wo), Wo, N * C, Hc, Wc, Ho, Wo,
                             _p(gh_lo), _p(gh_hi), gh_lo.size, _p(gw_lo), _p(gw_hi), gw_lo.size, m)
    assert rc == 0, rc
    return y


def dtcwt_fwd_j1(x, h0, h1, skip_hps=False, o_dim=2, ri_dim=-1, mode='symmetric'):
    dt = _dtype(x)
    x = np.ascontiguousarray(x, dt)
    N, C, H, W = x.shape
    h0, h1 = _t(h0, dt), _t(h1, dt)
    ll = np.full((N, C, H, W), np.nan, dt)
    shape, hs = orc.highs_shape_strides(N, C, H // 2, W // 2, o_dim, ri_dim)
    highs = None if skip_hps else np.full(shape, np.nan, dt)
    rc = _fn('emu_dtcwt_fwd_j1', dt)(_p(x), LL(H * W), W, _p(ll), LL(H * W), W, _p(highs), orc._hs(hs), N, C, H, W,
                                _p(h0), h0.size, _p(h1), h1.size, orc.mode_int(mode))
    assert rc == 0, rc
    return ll, highs


def dtcwt_fwd_j2plus(x, h0a, h1a, h0b, h1b, skip_hps=False, o_dim=2, ri_dim=-1):
    dt = _dtype(x)
    x = np.ascontiguousarray(x, dt)
    N, C, H, W = x.shape
    h0a, h1a, h0b, h1b = [_t(f, dt) for f in (h0a, h1a, h0b, h1b)]
    ll = np.full((N, C, H // 2, W // 2), np.nan, dt)
    shape, hs = orc.highs_shape_strides(N, C, H // 4, W // 4, o_dim, ri_dim)
    highs = None if skip_hps else np.full(shape, np.nan, dt)
    rc = _fn('emu_dtcwt_fwd_j2plus', dt)(_p(x), LL(H * W), W, _p(ll), LL((H // 2) * (W // 2)), W // 2, _p(highs),
                                    orc._hs(hs), N, C, H, W, _p(h0a), _p(h1a), _p(h0b), _p(h1b), h0a.size)
    if rc == -2:
        raise ValueError('size')
    assert rc == 0, rc
    return ll, highs


def _inv_dims(ll, highs, o_dim, ri_dim):
    names = orc._dim_names(o_dim, ri_dim)
    if highs is not None:
        sz = dict(zip(names, highs.shape))
    if ll is not None:
        N, C, H, W = ll.shape
    else:
        N, C, H, W = sz['n'], sz['c'], 2 * sz['h'], 2 * sz['w']
    return N, C, H, W


def dtcwt_inv_j1(ll, highs, g0, g1, o_dim=2, ri_dim=-1, mode='symmetric'):
    if highs is not None and ll is not None:
        names = orc._dim_names(o_dim, ri_dim)
        sz = dict(zip(names, highs.shape))
        if ll.shape[2] != 2 * sz['h']:
            ll = ll[:, :, 1:-1]
        if ll.shape[3] != 2 * sz['w']:
            ll = ll[:, :, :, 1:-1]
    dt = _dtype(ll if ll is not None else highs)
    if ll is not None:
        ll = np.ascontiguousarray(ll, dt)
    if highs is not None:
        highs = np.ascontiguousarray(highs, dt)
    N, C, H, W = _inv_dims(ll, highs, o_dim, ri_dim)
    _, hs = orc.highs_shape_strides(N, C, H // 2, W // 2, o_dim, ri_dim)
    g0, g1 = _t(g0, dt), _t(g1, dt)
    y = np.full((N, C, H, W), np.nan, dt)
    rc = _fn('emu_dtcwt_inv_j1', dt)(_p(ll), LL(H * W), W, _p(highs), orc._hs(hs), _p(y), LL(H * W), W, N, C, H, W,
                                _p(g0), g0.size, _p(g1), g1.size, orc.mode_int(mode))
    assert rc == 0, rc
    return y


def dtcwt_inv_j2plus(ll, highs, g0a, g1a, g0b, g1b, o_dim=2, ri_dim=-1):
    dt = _dtype(ll if ll is not None else highs)
    if ll is not None:
        ll = np.ascontiguousarray(ll, dt)
    if highs is not None:
        highs = np.ascontiguousarray(highs, dt)
    N, C, H, W = _inv_dims(ll, highs, o_dim, ri_dim)
    _, hs = orc.highs_shape_strides(N, C, H // 2, W // 2, o_dim, ri_dim)
    g0a, g1a, g0b, g1b = [_t(f, dt) for f in (g0a, g1a, g0b, g1b)]
    y = np.full((N, C, 2 * H, 2 * W), np.nan, dt)
    rc = _fn('emu_dtcwt_inv_j2plus', dt)(_p(ll), LL(H * W), W, _p(highs), orc._hs(hs), _p(y), LL(4 * H * W), 2 * W,
                                    N, C, H, W, _p(g0a), _p(g1a), _p(g0b), _p(g1b), g0a.size)
    assert rc == 0, rc
    return y


def scat_j1(x, h0, h1, mode='symmetric', magbias=1e-2, want_grad_aux=False):
    dt = _dtype(x)
    x = np.ascontiguousarray(x, dt)
    N, C, H, W = x.shape
    h0, h1 = _t(h0, dt), _t(h1, dt)
    z = np.full((N, 7, C, H // 2, W // 2), np.nan, dt)
    dre = dim = None
    if want_grad_aux:
        dre = np.full((N, 6, C, H // 2, W // 2), np.nan, dt)
        dim = np.full_like(dre, np.nan)
    rc = _fn('emu_scat_j1', dt)(_p(x), _p(z), _p(dre), _p(dim), N, C, H, W, _p(h0), h0.size, _p(h1), h1.size,
                           orc.mode_int(mode), (ctypes.c_double if dt == np.float64 else ctypes.c_float)(magbias))
    assert rc == 0, rc
    return (z, dre, dim) if want_grad_aux else z


PLAN_FIELDS = ('H', 'W', 'Ho', 'Wo', 'n_stage', 'warp0', 'nwarps', 'in_off', 'in_pitch', 'in_rows', 'n_in', 'bar_in',
               'st_off', 'st_cap', 'nbands', 'bar_out')


def plan_pyramid(planes, H, W, J, L, mode, xpitch=None, max_smem=227 * 1024, ll_pitch=0):
    """The shipped plan of the fused DWT pyramid kernel (pyramid_plan.h) as a dict, or None when it does not apply."""
    out = (ctypes.c_int * (8 + 16 * 4))()
    rc = lib().emu_plan_pyramid(planes, H, W, J, L, orc.mode_int(mode), W if xpitch is None else xpitch, max_smem,
                                ll_pitch, out)
    if rc:
        return None
    d = {'smem_bytes': out[1], 'threads': out[2], 'n_bars': out[3], 'zero_off': out[4], 'nslot': out[69],
         'split': out[70], 'll_pitch': out[71], 'levels': []}
    for l in range(J):
        d['levels'].append(dict(zip(PLAN_FIELDS, out[5 + 16 * l: 5 + 16 * (l + 1)])))
    return d
