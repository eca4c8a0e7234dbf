"""CPU oracle of the 3-D DWT: numpy compositions of the pinned 1-D and 2-D oracle entries (oracle/oracle.py).

TEST INFRASTRUCTURE, NOT PRODUCT.  A 3-D analysis level is ``dwt_afb2d`` on every (n, c, d) slice (along W, then H),
then ``dwt_afb1d`` along D, each pass rounded to the element type; synthesis is ``dwt_sfb1d`` along D, then
``dwt_sfb2d`` (H, then W).  Band b = 4*aW + 2*aH + aD - 1 (aX = 1: high-pass along X).  Filters are in stored form
(analysis taps reversed), one pair for all three axes.  fp32 and fp64 alike.
"""
import numpy as np

from oracle import oracle as orc


def _rows(a):
    """(N, C, D, H, W) -> (N*C, H*W, D): signals along D, the layout of the 1-D oracle entries."""
    N, C, D, H, W = a.shape
    return np.ascontiguousarray(np.moveaxis(a, 2, -1)).reshape(N * C, H * W, D)


def _unrows(o, N, C, H, W):
    return np.ascontiguousarray(np.moveaxis(o.reshape(N, C, H, W, o.shape[-1]), -1, 2))


def dwt_afb3d(x, h0, h1, mode):
    """x (N,C,D,H,W) -> yl (N,C,Do,Ho,Wo), highs (N,C,7,Do,Ho,Wo)."""
    x = np.ascontiguousarray(x)
    N, C, D, H, W = x.shape
    ll2, hi2 = orc.dwt_afb2d(x.reshape(N, C * D, H, W), h0, h1, h0, h1, mode)
    Ho, Wo = ll2.shape[-2:]
    groups = [ll2.reshape(N, C, D, Ho, Wo)] + [hi2[:, :, k].reshape(N, C, D, Ho, Wo) for k in range(3)]
    yl = None
    highs = [None] * 7
    for v, g in enumerate(groups):
        lo, hi = [_unrows(o, N, C, Ho, Wo) for o in orc.dwt_afb1d(_rows(g), h0, h1, mode)]
        if v == 0:
            yl = lo
        else:
            highs[2 * v - 1] = lo
        highs[2 * v] = hi
    return yl, np.stack(highs, axis=2)


def dwt_sfb3d(yl, highs, g0, g1, mode, out_dhw=None):
    """yl (N,C,Dc,Hc,Wc), highs (N,C,7,Dc,Hc,Wc) or None -> y (N,C,Do,Ho,Wo), cropped to ``out_dhw``."""
    yl = np.ascontiguousarray(yl)
    N, C, Dc, Hc, Wc = yl.shape
    Do = orc.rec_len(Dc, np.size(g0), mode)
    if out_dhw is not None:
        Do = min(Do, out_dhw[0])
    groups = []
    for v in range(4 if highs is not None else 1):
        lo = yl if v == 0 else highs[:, :, 2 * v - 1]
        hi = None if highs is None else highs[:, :, 2 * v]
        y = orc.dwt_sfb1d(_rows(lo), None if hi is None else _rows(hi), g0, g1, mode, out_len=Do)
        groups.append(_unrows(y, N, C, Hc, Wc))
    ll2 = groups[0].reshape(N, C * Do, Hc, Wc)
    hi2 = None if highs is None else np.stack([g.reshape(N, C * Do, Hc, Wc) for g in groups[1:]], axis=2)
    y = orc.dwt_sfb2d(ll2, hi2, g0, g1, g0, g1, mode, out_hw=None if out_dhw is None else out_dhw[1:])
    return y.reshape((N, C, Do) + y.shape[-2:])


def dwt3d_forward(x, filts, J, mode):
    """DWT3DForward.forward; filts = stored (h0, h1)."""
    ll, yh = x, []
    for _ in range(J):
        ll, h = dwt_afb3d(ll, filts[0], filts[1], mode)
        yh.append(h)
    return ll, yh


def dwt3d_inverse(yl, yh, filts, mode):
    """DWT3DInverse.forward; filts = (g0, g1).  None band-passes are zeros; along each axis the low-pass loses its last
    sample when it is one longer than the band-pass."""
    ll = yl
    for h in yh[::-1]:
        if h is not None:
            for ax in (2, 3, 4):
                if ll.shape[ax] > h.shape[ax + 1]:
                    ll = np.take(ll, np.arange(ll.shape[ax] - 1), axis=ax)
        ll = dwt_sfb3d(ll, h, filts[0], filts[1], mode)
    return ll


def dwt_sfb3d_plane_first(yl, highs, g0, g1, mode, out_dhw=None):
    """The same synthesis with the passes in the fused kernel's order: the 2-D synthesis of the D-low bands
    (yl, 1, 3, 5) and of the D-high bands (0, 2, 4, 6) on every coefficient slice, then the synthesis along D."""
    yl = np.ascontiguousarray(yl)
    N, C, Dc, Hc, Wc = yl.shape
    Do = orc.rec_len(Dc, np.size(g0), mode)
    if out_dhw is not None:
        Do = min(Do, out_dhw[0])
    hw = None if out_dhw is None else out_dhw[1:]
    planes = []
    for d in range(2 if highs is not None else 1):
        ll = yl if d == 0 else highs[:, :, 0]
        hi = None if highs is None else np.stack([highs[:, :, 1 + d], highs[:, :, 3 + d], highs[:, :, 5 + d]], axis=3)
        y = orc.dwt_sfb2d(np.ascontiguousarray(ll).reshape(N, C * Dc, Hc, Wc),
                          None if hi is None else hi.reshape(N, C * Dc, 3, Hc, Wc), g0, g1, g0, g1, mode, out_hw=hw)
        planes.append(y.reshape((N, C, Dc) + y.shape[-2:]))
    Ho, Wo = planes[0].shape[-2:]
    y = orc.dwt_sfb1d(_rows(planes[0]), None if highs is None else _rows(planes[1]), g0, g1, mode, out_len=Do)
    return _unrows(y, N, C, Ho, Wo)


def bound_sfb3d(g0, g1, has_hi=True):
    """(G, K) of one 3-D synthesis level for tests/util.py's per-plane bound: util.bound_sfb2d's G (per-phase l1 norms
    along H times along W) times the same factor along D.  K: 3.5 for 2 taps, 1.5 for 4 to 8 taps, 5.0 for the low-pass
    band alone -- about 1.3x the largest error / (u G s) the fp32 oracle reaches in either pass order on the small volumes
    of tests/test_dwt3d_cpu.py, since larger volumes reach further into the tail (a 1 x 8 x 80 x 150 haar volume of the
    GPU sweep reached 2.7), and still small enough that 1e-6 of the scale in one element breaks the bound."""
    from tests import util
    n = util.l1_phase(g0) + (util.l1_phase(g1) if has_hi else 0.0)
    if not has_hi:
        return n ** 3, 5.0
    return n ** 3, (3.5 if np.size(g0) <= 2 else 1.5)
