from pytorch_wavelets_b200.scatternet.layers import ScatLayer, ScatLayerj2  # noqa: F401
from pytorch_wavelets_b200.scatternet.scat1d import ScatLayer1D, ScatLayer1Dj2  # noqa: F401
