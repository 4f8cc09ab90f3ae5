"""instantsplat_b200 -- H100-native (sm_90a) replacement for the native code under InstantSplat's
training hot path: differentiable Gaussian rasterizer (+ fused camera-pose transform), fused
L1/SSIM loss and per-point Adam, behind the reference's own Python interfaces.

    from instantsplat_b200 import render, GaussianRasterizer, GaussianRasterizationSettings,
                                  fused_ssim, PerPointAdam, JointTrainer

The CUDA library (instantsplat_b200/lib/libgsb200.so, C ABI in include/gsb200.h) is mandatory:
nothing here falls back to PyTorch or the CPU.
"""
from ._lib import GsbError, build, lib  # noqa: F401
from .rasterizer import (GaussianRasterizationSettings, GaussianRasterizer, rasterize_fused,  # noqa: F401
                         rasterize_gaussians)
from .renderer import render  # noqa: F401
from .ssim import fused_ssim, fused_training_loss  # noqa: F401
from .per_point_adam import PerPointAdam  # noqa: F401
from .trainer import CHECKPOINT_KEY, JointTrainer, OptimConfig, read_checkpoint  # noqa: F401
from .model import GaussianModel, PipelineDefaults, SimpleGaussianModel, optimization_defaults  # noqa: F401
from .knn import distCUDA2  # noqa: F401
from .densify import cameras_extent, densify_plan  # noqa: F401
from .evaluation import image_metrics  # noqa: F401
