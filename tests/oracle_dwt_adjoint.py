"""Dense-matrix restatement of the DWT banks and of the transposed analysis bank A_m^T (csrc/dwt_adjoint.cu).

TEST INFRASTRUCTURE.  Matrices are built column by column from the CPU oracle (oracle/oracle.py) on unit inputs, so
they are the reference's per-level arithmetic.  ``adjoint_matrix_1d`` restates the kernel's index arithmetic (the
images of each output under the boundary extension), and ``afb2d_adjoint`` / ``afb1d_adjoint`` apply it to arrays.
Filters are stored (reversed) analysis taps, as the module buffers hold them.
"""
import numpy as np

from oracle import oracle as orc

MODES = ('zero', 'symmetric', 'reflect', 'periodic', 'periodization')


def ext_pl(L, mode):
    return L - 1 - L // 2 if mode == 'periodization' else L - 2


def images(i, n, mode, plo, phi):
    """Every extended position p in [plo, phi] with ext_index(p, n, mode) == i (csrc/common.h, inverted)."""
    bases, per = [i], None
    if mode == 'symmetric':
        per, bases = 2 * n, [i, 2 * n - 1 - i]
    elif mode == 'reflect':
        if n == 1:
            per = 1
        else:
            per = 2 * n - 2
            if 0 < i < n - 1:
                bases.append(2 * n - 2 - i)
    elif mode == 'periodic':
        per = n
    elif mode == 'periodization':
        per = n + (n & 1)
        if n & 1 and i == n - 1:
            bases.append(n)
    else:
        return [i] if plo <= i <= phi else []
    out = []
    for b in bases:
        p = plo + (b - plo) % per
        while p <= phi:
            out.append(p)
            p += per
    return sorted(out)


def adjoint_matrix_1d(f, n, mode):
    """T (n, K): T[i, k] = sum over the images p of i of f[p + pl - 2k] -- one band of A_m^T."""
    f = np.asarray(f, np.float64).ravel()
    L = f.size
    K = orc.coeff_len(n, L, mode)
    pl = ext_pl(L, mode)
    T = np.zeros((n, K))
    for i in range(n):
        for p in images(i, n, mode, -pl, 2 * K - 3 + L - pl):
            for k in range(K):
                t = p + pl - 2 * k
                if 0 <= t < L:
                    T[i, k] += f[t]
    return T


def afb1d_adjoint(lo, hi, f0, f1, mode, n):
    """A_m^T of the 1-D analysis: lo, hi (..., K) -> (..., n)."""
    return lo @ adjoint_matrix_1d(f0, n, mode).T + hi @ adjoint_matrix_1d(f1, n, mode).T


def afb2d_adjoint(ll, highs, fh_lo, fh_hi, fw_lo, fw_hi, mode, H, W):
    """A_m^T of the 2-D analysis, H first then W: ll (..., Hc, Wc), highs (..., 3, Hc, Wc) -> (..., H, W).  Bands:
    highs[0] = H high / W low, highs[1] = H low / W high, highs[2] = both high."""
    Thl, Thh = adjoint_matrix_1d(fh_lo, H, mode), adjoint_matrix_1d(fh_hi, H, mode)
    Twl, Twh = adjoint_matrix_1d(fw_lo, W, mode), adjoint_matrix_1d(fw_hi, W, mode)
    lo = Thl @ ll + Thh @ highs[..., 0, :, :]
    hi = Thl @ highs[..., 1, :, :] + Thh @ highs[..., 2, :, :]
    return lo @ Twl.T + hi @ Twh.T


def dense_afb1d(f0, f1, n, mode):
    """(2K, n) matrix of the oracle's dwt_afb1d: rows [lo; hi]."""
    lo, hi = orc.dwt_afb1d(np.eye(n).reshape(n, 1, n), f0, f1, mode)
    return np.concatenate([lo[:, 0, :], hi[:, 0, :]], axis=1).T


def dense_sfb1d(g0, g1, K, mode, n=None):
    """(n, 2K) matrix of the oracle's dwt_sfb1d (cropped to n when given): columns [lo | hi]."""
    e = np.eye(2 * K).reshape(2 * K, 1, 2 * K)
    y = orc.dwt_sfb1d(np.ascontiguousarray(e[..., :K]), np.ascontiguousarray(e[..., K:]), g0, g1, mode, out_len=n)
    return y[:, 0, :].T


def dense_afb2d(fw_lo, fw_hi, fh_lo, fh_hi, H, W, mode):
    """(4 Hc Wc, H W) matrix of the oracle's dwt_afb2d: rows [ll; highs[0]; highs[1]; highs[2]], each row-major."""
    ll, hs = orc.dwt_afb2d(np.eye(H * W).reshape(H * W, 1, H, W), fw_lo, fw_hi, fh_lo, fh_hi, mode)
    n = H * W
    return np.concatenate([ll.reshape(n, -1), hs.reshape(n, 3, -1).reshape(n, -1)], axis=1).T


def dense_sfb2d(gh_lo, gh_hi, gw_lo, gw_hi, Hc, Wc, mode, out_hw=None):
    """(Ho Wo, 4 Hc Wc) matrix of the oracle's dwt_sfb2d (cropped to out_hw when given)."""
    m = 4 * Hc * Wc
    e = np.eye(m).reshape(m, 1, 4, Hc, Wc)
    y = orc.dwt_sfb2d(np.ascontiguousarray(e[:, :, 0]), np.ascontiguousarray(e[:, :, 1:]), gh_lo, gh_hi, gw_lo, gw_hi,
                      mode, out_hw=out_hw)
    return y.reshape(m, -1).T
