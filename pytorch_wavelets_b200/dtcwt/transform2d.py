"""``DTCWTForward`` / ``DTCWTInverse`` with the reference's constructor signatures, buffer names, return
structures and error behaviour (reference ``pytorch_wavelets/dtcwt/transform2d.py:20-254``), running each
level as one fused kernel of the H100 engine."""
import torch
import torch.nn as nn
from numpy import ndarray

from pytorch_wavelets_b200.dtcwt.coeffs import biort as _biort
from pytorch_wavelets_b200.dtcwt.coeffs import qshift as _qshift
from pytorch_wavelets_b200.dtcwt.lowlevel import prep_filt
from pytorch_wavelets_b200.dtcwt.transform_funcs import (FWD_J1, FWD_J12, FWD_J2PLUS, INV_J1, INV_J2PLUS,
                                                         get_dimensions6)
from pytorch_wavelets_b200.dwt.lowlevel import mode_to_int


def _replicate_pad(low, rows, cols):
    """Pad one replicated row/col on BOTH sides (reference transform2d.py:131-135)."""
    if rows:
        low = torch.cat((low[:, :, 0:1], low, low[:, :, -1:]), dim=2)
    if cols:
        low = torch.cat((low[:, :, :, 0:1], low, low[:, :, :, -1:]), dim=3)
    return low


class DTCWTForward(nn.Module):
    """2-D DTCWT forward decomposition (drop-in for the reference ``DTCWTForward``).

    Args:
        biort (str | (h0o, h1o)): level-1 biorthogonal filters: 'antonini', 'legall', 'near_sym_a', 'near_sym_b'.
        qshift (str | (h0a, h0b, h1a, h1b)): level>=2 quarter-shift filters: 'qshift_06', 'qshift_a' .. 'qshift_d'.
        J (int): number of levels.
        skip_hps (bool | list[bool]): skip the band-pass outputs of a level (0-dim tensor returned instead).
        include_scale (bool | list[bool]): also return the low-pass of the marked levels.
        o_dim (int): dimension that holds the 6 orientations.  ri_dim (int): dimension of real/imag.
        mode (str): 'symmetric' or zero padding for level 1 (levels >= 2 are always symmetric).

    ``forward(x)`` returns ``(yl, yh)``; ``yh[j]`` has shape (N, C, 6, H_j, W_j, 2) for the default dims.
    """

    def __init__(self, biort='near_sym_a', qshift='qshift_a', J=3, skip_hps=False, include_scale=False,
                 o_dim=2, ri_dim=-1, mode='symmetric'):
        super().__init__()
        if o_dim == ri_dim:
            raise ValueError("Orientations and real/imaginary parts must be in different dimensions.")
        self.biort = biort
        self.qshift = qshift
        self.J = J
        self.o_dim = o_dim
        self.ri_dim = ri_dim
        self.mode = mode
        if isinstance(biort, str):
            h0o, _, h1o, _ = _biort(biort)[:4]
            self.register_buffer('h0o', prep_filt(h0o, 1))
            self.register_buffer('h1o', prep_filt(h1o, 1))
        else:
            self.register_buffer('h0o', prep_filt(biort[0], 1))
            self.register_buffer('h1o', prep_filt(biort[1], 1))
        if isinstance(qshift, str):
            h0a, h0b, _, _, h1a, h1b, _, _ = _qshift(qshift)[:8]
            self.register_buffer('h0a', prep_filt(h0a, 1))
            self.register_buffer('h0b', prep_filt(h0b, 1))
            self.register_buffer('h1a', prep_filt(h1a, 1))
            self.register_buffer('h1b', prep_filt(h1b, 1))
        else:
            self.register_buffer('h0a', prep_filt(qshift[0], 1))
            self.register_buffer('h0b', prep_filt(qshift[1], 1))
            self.register_buffer('h1a', prep_filt(qshift[2], 1))
            self.register_buffer('h1b', prep_filt(qshift[3], 1))
        if isinstance(skip_hps, (list, tuple, ndarray)):
            self.skip_hps = skip_hps
        else:
            self.skip_hps = [skip_hps, ] * self.J
        if isinstance(include_scale, (list, tuple, ndarray)):
            self.include_scale = include_scale
        else:
            self.include_scale = [include_scale, ] * self.J

    def forward(self, x):
        scales = [x.new_zeros([]), ] * self.J
        highs = [x.new_zeros([]), ] * self.J
        mode = mode_to_int(self.mode)
        if self.J == 0:
            return x, None
        # odd height / width: repeat the last row / col (reference :116-120)
        r, c = x.shape[2:]
        if r % 2 != 0:
            x = torch.cat((x, x[:, :, -1:]), dim=2)
        if c % 2 != 0:
            x = torch.cat((x, x[:, :, :, -1:]), dim=3)
        j0 = 1
        if (self.J >= 2 and x.dtype == torch.float32 and not self.include_scale[0] and not self.skip_hps[0]
                and x.shape[2] % 4 == 0 and x.shape[3] % 4 == 0):
            # levels 1 and 2 in one call: the level-1 low-pass is neither returned nor padded between the levels
            low, highs[0], highs[1] = FWD_J12.apply(x, self.h0o, self.h1o, self.h0a, self.h1a, self.h0b, self.h1b,
                                                    self.skip_hps[1], self.o_dim, self.ri_dim, mode)
            if self.include_scale[1]:
                scales[1] = low
            j0 = 2
        else:
            low, h = FWD_J1.apply(x, self.h0o, self.h1o, self.skip_hps[0], self.o_dim, self.ri_dim, mode)
            highs[0] = h
            if self.include_scale[0]:
                scales[0] = low
        for j in range(j0, self.J):
            r, c = low.shape[2:]
            low = _replicate_pad(low, r % 4 != 0, c % 4 != 0)
            low, h = FWD_J2PLUS.apply(low, self.h0a, self.h1a, self.h0b, self.h1b, self.skip_hps[j],
                                      self.o_dim, self.ri_dim, mode)
            highs[j] = h
            if self.include_scale[j]:
                scales[j] = low
        if True in self.include_scale:
            return scales, highs
        return low, highs


class DTCWTInverse(nn.Module):
    """2-D DTCWT inverse (drop-in for the reference ``DTCWTInverse``).  ``forward((yl, yh))`` accepts
    ``None`` / 0-dim tensors for any band-pass level (treated as zeros)."""

    def __init__(self, biort='near_sym_a', qshift='qshift_a', o_dim=2, ri_dim=-1, mode='symmetric'):
        super().__init__()
        self.biort = biort
        self.qshift = qshift
        self.o_dim = o_dim
        self.ri_dim = ri_dim
        self.mode = mode
        if isinstance(biort, str):
            _, g0o, _, g1o = _biort(biort)[:4]
            self.register_buffer('g0o', prep_filt(g0o, 1))
            self.register_buffer('g1o', prep_filt(g1o, 1))
        else:
            self.register_buffer('g0o', prep_filt(biort[0], 1))
            self.register_buffer('g1o', prep_filt(biort[1], 1))
        if isinstance(qshift, str):
            _, _, g0a, g0b, _, _, g1a, g1b = _qshift(qshift)[:8]
            self.register_buffer('g0a', prep_filt(g0a, 1))
            self.register_buffer('g0b', prep_filt(g0b, 1))
            self.register_buffer('g1a', prep_filt(g1a, 1))
            self.register_buffer('g1b', prep_filt(g1b, 1))
        else:
            self.register_buffer('g0a', prep_filt(qshift[0], 1))
            self.register_buffer('g0b', prep_filt(qshift[1], 1))
            self.register_buffer('g1a', prep_filt(qshift[2], 1))
            self.register_buffer('g1b', prep_filt(qshift[3], 1))

    def forward(self, coeffs):
        low, highs = coeffs
        J = len(highs)
        mode = mode_to_int(self.mode)
        _, _, h_dim, w_dim = get_dimensions6(self.o_dim, self.ri_dim)
        for j, s in zip(range(J - 1, 0, -1), highs[1:][::-1]):
            if s is not None and s.shape != torch.Size([]):
                assert s.shape[self.o_dim] == 6, "Inverse transform must have input with 6 orientations"
                assert len(s.shape) == 6, "Bandpass inputs must have 6 dimensions"
                assert s.shape[self.ri_dim] == 2, "Inputs must be complex with real and imaginary parts in the ri dimension"
                # the low-pass was padded to a multiple of 4 on the way down: trim it (reference :233-238)
                r, c = low.shape[2:]
                r1, c1 = s.shape[h_dim], s.shape[w_dim]
                if r != r1 * 2:
                    low = low[:, :, 1:-1]
                if c != c1 * 2:
                    low = low[:, :, :, 1:-1]
            low = INV_J2PLUS.apply(low, s, self.g0a, self.g1a, self.g0b, self.g1b, self.o_dim, self.ri_dim, mode)
        if highs[0] is not None and highs[0].shape != torch.Size([]):
            r, c = low.shape[2:]
            r1, c1 = highs[0].shape[h_dim], highs[0].shape[w_dim]
            if r != r1 * 2:
                low = low[:, :, 1:-1]
            if c != c1 * 2:
                low = low[:, :, :, 1:-1]
        low = INV_J1.apply(low, highs[0], self.g0o, self.g1o, self.o_dim, self.ri_dim, mode)
        return low
