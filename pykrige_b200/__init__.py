"""pykrige_b200 — H100-native ``backend='cuda'`` kriging ``execute()`` path.

Keeps the class API of GeoStat-Framework/PyKrige (OrdinaryKriging, UniversalKriging,
OrdinaryKriging3D, UniversalKriging3D) and its variogram_models plug-in surface; the
kriging system is assembled, factored and solved by hand-written sm_90a CUDA kernels
behind a C ABI (include/krige_b200.h, pykrige_b200/csrc). No CPU fallback.
"""
from . import variogram_models  # noqa: F401
from .ok import OrdinaryKriging  # noqa: F401
from .uk import UniversalKriging  # noqa: F401
from .ok3d import OrdinaryKriging3D  # noqa: F401
from .uk3d import UniversalKriging3D  # noqa: F401

__version__ = "0.1.0"
__all__ = ["OrdinaryKriging", "UniversalKriging", "OrdinaryKriging3D", "UniversalKriging3D", "variogram_models"]
