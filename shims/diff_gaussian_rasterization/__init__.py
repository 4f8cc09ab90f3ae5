"""`import diff_gaussian_rasterization` drop-in (put <repo>/shims and <repo> on PYTHONPATH):
what gaussian_renderer/__init__.py:14-17 imports, served by libgsb200.so."""
from instantsplat_b200.rasterizer import (GaussianRasterizationSettings, GaussianRasterizer,  # noqa: F401
                                          rasterize_gaussians)
from . import _C  # noqa: F401,E402
