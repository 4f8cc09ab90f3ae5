"""`from fused_ssim import fused_ssim` drop-in (train.py:39-43)."""
from instantsplat_b200.ssim import fused_ssim  # noqa: F401
