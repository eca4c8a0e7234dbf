"""pytorch_wavelets_b200 -- H100 (sm_90a) engine for the 2-D wavelet filterbank hot path of
fbcotter/pytorch_wavelets, behind the reference's nn.Module API.

The reference package's export list and aliases (``pytorch_wavelets/__init__.py:1-36``) for the classes on the
hot path and its direct callers (SURVEY.md section 8), plus the 3-D DWT (``DWT3DForward`` / ``DWT3DInverse``,
aliases ``DWT3D`` / ``IDWT3D``), the 1-D DTCWT (``DTCWT1DForward`` / ``DTCWT1DInverse``, aliases ``DTCWT1D`` /
``IDTCWT1D``), the 1-D scattering layers (``ScatLayer1D`` / ``ScatLayer1Dj2``) and the 2-D wavelet packet transform
(``WPT2DForward`` / ``WPT2DInverse``, aliases ``WPT2D`` / ``IWPT2D``), which the reference does not have.
Every transform runs in hand-written CUDA kernels through the C ABI of ``libb200wave.so``; there is no
CPU or eager fallback.
"""
__all__ = [
    '__version__',
    'DTCWTForward',
    'DTCWTInverse',
    'DTCWT1DForward',
    'DTCWT1DInverse',
    'DWTForward',
    'DWTInverse',
    'DTCWT',
    'IDTCWT',
    'DTCWT1D',
    'IDTCWT1D',
    'DWT',
    'IDWT',
    'DWT2D',
    'IDWT2D',
    'DWT1DForward',
    'DWT1DInverse',
    'DWT1D',
    'IDWT1D',
    'DWT3DForward',
    'DWT3DInverse',
    'DWT3D',
    'IDWT3D',
    'ScatLayer',
    'ScatLayerj2',
    'ScatLayer1D',
    'ScatLayer1Dj2',
    'WPT2DForward',
    'WPT2DInverse',
    'WPT2D',
    'IWPT2D',
]

from pytorch_wavelets_b200._version import __version__
from pytorch_wavelets_b200.dtcwt.transform1d import DTCWT1DForward, DTCWT1DInverse
from pytorch_wavelets_b200.dtcwt.transform2d import DTCWTForward, DTCWTInverse
from pytorch_wavelets_b200.dwt.transform1d import DWT1DForward, DWT1DInverse
from pytorch_wavelets_b200.dwt.transform2d import DWTForward, DWTInverse
from pytorch_wavelets_b200.dwt.transform3d import DWT3DForward, DWT3DInverse
from pytorch_wavelets_b200.dwt.packet2d import WPT2DForward, WPT2DInverse
from pytorch_wavelets_b200.scatternet import ScatLayer, ScatLayer1D, ScatLayer1Dj2, ScatLayerj2

# aliases, as in the reference
DTCWT = DTCWTForward
IDTCWT = DTCWTInverse
DTCWT1D = DTCWT1DForward
IDTCWT1D = DTCWT1DInverse
DWT = DWTForward
IDWT = DWTInverse
DWT2D = DWT
IDWT2D = IDWT
DWT1D = DWT1DForward
IDWT1D = DWT1DInverse
DWT3D = DWT3DForward
IDWT3D = DWT3DInverse
WPT2D = WPT2DForward
IWPT2D = WPT2DInverse
