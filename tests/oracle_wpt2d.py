"""The 2-D wavelet packet transform composed from the pinned oracle levels (``oracle.dwt_afb2d`` / ``dwt_sfb2d``):
every node split by one DWT level, children 4p .. 4p+3 of node p in ``DWTForward``'s band order (ll, lh, hl, hh)."""
import numpy as np

from oracle import oracle as orc


def wpt2d_forward(x, filts, J, mode):
    """x (N, C, H, W) -> (N, C, 4^J, H_J, W_J).  filts = the stored (h0_col, h1_col, h0_row, h1_row) buffers of
    ``DWTForward``: the *_col pair filters along W and the *_row pair along H (``oracle.dwt_forward``'s orientation)."""
    h0_col, h1_col, h0_row, h1_row = filts
    N, C, H, W = x.shape
    y = np.asarray(x)[:, :, None]
    for _ in range(J):
        P, H, W = y.shape[2:]
        ll, hi = orc.dwt_afb2d(y.reshape(N, C * P, H, W), h0_col, h1_col, h0_row, h1_row, mode)
        Ho, Wo = ll.shape[-2:]
        y = np.concatenate([ll[:, :, None], hi], axis=2).reshape(N, C, 4 * P, Ho, Wo)
    return y


def wpt2d_inverse(y, filts, mode, sizes=None):
    """y (N, C, 4^J, Hc, Wc) -> (N, C, H, W).  filts = the stored (g0_col, g1_col, g0_row, g1_row) buffers of
    ``DWTInverse`` (the *_row pair along H, the *_col pair along W, ``oracle.dwt_inverse``'s orientation).  ``sizes``:
    the output size of each level, finest first (J entries), or None for the natural ``rec_len`` sizes."""
    g0_col, g1_col, g0_row, g1_row = filts
    N, C, P = y.shape[:3]
    J = int(round(np.log(P) / np.log(4)))
    assert 4 ** J == P
    sizes = sizes if sizes is not None else [None] * J
    c = np.asarray(y)
    for j in range(J - 1, -1, -1):
        P, Hc, Wc = c.shape[2:]
        q = c.reshape(N, C * P // 4, 4, Hc, Wc)
        out = orc.dwt_sfb2d(q[:, :, 0], q[:, :, 1:], g0_row, g1_row, g0_col, g1_col, mode, out_hw=sizes[j])
        c = out.reshape(N, C, P // 4, out.shape[-2], out.shape[-1])
    return c[:, :, 0]


def forward_sizes(H, W, J, Lh, Lw, mode):
    """[(H_0, W_0), ..., (H_J, W_J)] under the forward length rule."""
    sizes = [(H, W)]
    for _ in range(J):
        h, w = sizes[-1]
        sizes.append((orc.coeff_len(h, Lh, mode), orc.coeff_len(w, Lw, mode)))
    return sizes
