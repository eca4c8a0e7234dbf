"""``DWT3DForward`` / ``DWT3DInverse``: the separable 3-D DWT of volumes (N, C, D, H, W), an addition beyond the
reference (which has 1-D and 2-D DWTs only).  One filter pair acts along W, H and D; each level is one C-ABI call
(``b200w_dwt_afb3d`` / ``b200w_dwt_sfb3d``), one fused kernel launch where the fused kernels apply."""
import torch.nn as nn

from pytorch_wavelets_b200.dwt import lowlevel
from pytorch_wavelets_b200.dwt.transform1d import _wave_pair


class DWT3DForward(nn.Module):
    """3-D DWT forward decomposition.

    Args:
        J (int): number of levels.
        wave (str | Wavelet | tuple(ndarray)): wavelet name, an object with ``dec_lo/dec_hi/rec_lo/rec_hi``, or the
            analysis filter arrays ``(h0, h1)``.  The same pair filters all three axes.
        mode (str): 'zero', 'symmetric', 'reflect', 'periodic' or 'periodization'.

    ``forward(x)`` with x (N, C, D, H, W) float32 or float64 on a CUDA device returns ``(yl, yh)``: ``yl`` the final
    low-pass (N, C, D_J, H_J, W_J) and ``yh`` a list of J tensors (N, C, 7, D_j, H_j, W_j), finest first.  Band
    b = 4*aW + 2*aH + aD - 1 (aX = 1: high-pass along X): bands 1, 3, 5 are the 2-D lh, hl, hh low-passed along D,
    bands 0, 2, 4, 6 are high-pass along D.
    """

    def __init__(self, J=1, wave='db1', mode='zero'):
        super().__init__()
        h0, h1 = _wave_pair(wave, True)
        filts = lowlevel.prep_filt_afb1d(h0, h1)
        self.register_buffer('h0', filts[0])
        self.register_buffer('h1', filts[1])
        self.J = J
        self.mode = mode

    def forward(self, x):
        if x.dim() != 5:
            raise ValueError('expected a 5-D (N,C,D,H,W) input, got shape {}'.format(tuple(x.shape)))
        mode = lowlevel.mode_to_int(self.mode)
        lowlevel._check_bank_mode(mode)
        if self.J < 1:
            return x, []
        yh = []
        ll = x
        for _ in range(self.J):
            ll, high = lowlevel.AFB3D.apply(ll, self.h0, self.h1, mode)
            yh.append(high)
        return ll, yh


class DWT3DInverse(nn.Module):
    """3-D DWT inverse reconstruction.  ``forward((yl, yh))`` takes the output format of :class:`DWT3DForward`; any
    entry of ``yh`` may be ``None`` (zeros).  Along any axis where the low-pass is one longer than the band-pass, its
    last sample is dropped first (the 2-D rule, per axis); odd-sized axes come back one longer."""

    def __init__(self, wave='db1', mode='zero'):
        super().__init__()
        g0, g1 = _wave_pair(wave, False)
        filts = lowlevel.prep_filt_sfb1d(g0, g1)
        self.register_buffer('g0', filts[0])
        self.register_buffer('g1', filts[1])
        self.mode = mode

    def forward(self, coeffs):
        yl, yh = coeffs
        if yl.dim() != 5:
            raise ValueError('expected a 5-D (N,C,D,H,W) low-pass, got shape {}'.format(tuple(yl.shape)))
        mode = lowlevel.mode_to_int(self.mode)
        lowlevel._check_bank_mode(mode)
        ll = yl
        for h in yh[::-1]:
            if h is not None:
                for ax in (2, 3, 4):
                    if ll.shape[ax] > h.shape[ax + 1]:
                        ll = ll.narrow(ax, 0, ll.shape[ax] - 1)
            ll = lowlevel.SFB3D.apply(ll, h, self.g0, self.g1, mode)
        return ll
