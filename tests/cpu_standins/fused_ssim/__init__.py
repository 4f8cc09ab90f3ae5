"""CPU stand-in for `fused_ssim` (tests only): the oracle's restatement of utils/loss_utils.py:55-85."""
from oracle import gs_oracle as O


def fused_ssim(img1, img2, padding="same", train=True):
    assert padding == "same"
    return O.ssim(img1, img2)
