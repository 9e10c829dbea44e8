"""nerf2mesh_b200 -- H100-native (sm_90a) stage-0 ray-marching hot path behind nerf2mesh's
operator surface.

Sub-packages `raymarching`, `gridencoder`, `shencoder` mirror the reference's modules of the
same names; `install()` registers them under those top-level names so the reference's
`nerf/renderer.py`, `nerf/network.py` and `encoding.py` import them unmodified.
"""
import sys

__version__ = "0.1.0"


def install():
    """Make `import raymarching`, `import gridencoder`, `import shencoder` resolve to this package."""
    from . import gridencoder, raymarching, shencoder
    sys.modules["raymarching"] = raymarching
    sys.modules["gridencoder"] = gridencoder
    sys.modules["shencoder"] = shencoder
    return raymarching, gridencoder, shencoder
