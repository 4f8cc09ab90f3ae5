"""Drop-in for `fused_ssim.fused_ssim` (boundary B3): train.py:39-43,172-173.
Semantics = the reference's PyTorch fallback utils/loss_utils.py:55-85
(11x11 sigma-1.5 window, zero 'same' padding, C1=1e-4, C2=9e-4, mean over all elements).
Also the fused L1+DSSIM training loss of train.py:171-176 (`fused_training_loss`)."""
from __future__ import annotations

import torch

from . import _lib
from ._lib import check, f32c


class _FusedSSIM(torch.autograd.Function):
    @staticmethod
    def forward(ctx, img1, img2, train):
        L = _lib.lib()
        a, b = f32c(img1), f32c(img2)
        if a.dim() != 4 or a.shape != b.shape:
            raise RuntimeError("fused_ssim expects two [B,C,H,W] tensors of the same shape")
        B, C, H, W = a.shape
        with torch.cuda.device(a.device):
            sums = torch.zeros(2, dtype=torch.float64, device=a.device)
            maps = torch.empty((3, B, C, H, W), dtype=torch.float32, device=a.device) if train else None
            check(L.gsb_ssim_forward(B * C, H, W, a.data_ptr(), b.data_ptr(), sums.data_ptr(),
                                     None if maps is None else maps.data_ptr(), _lib.stream_ptr()), "gsb_ssim_forward")
        ctx.save_for_backward(a, b, maps)
        ctx.n = B * C * H * W
        return (sums[1] / ctx.n).float()

    @staticmethod
    def backward(ctx, grad):
        a, b, maps = ctx.saved_tensors
        if maps is None:
            raise RuntimeError("fused_ssim(train=False) cannot be differentiated")
        B, C, H, W = a.shape
        with torch.cuda.device(a.device):
            out = torch.empty_like(a)
            g = f32c(grad).reshape(1)
            check(_lib.lib().gsb_ssim_backward(B * C, H, W, a.data_ptr(), b.data_ptr(), maps.data_ptr(),
                                               1.0 / ctx.n, g.data_ptr(), out.data_ptr(), _lib.stream_ptr()),
                  "gsb_ssim_backward")
        return out, None, None


def fused_ssim(img1, img2, padding="same", train=True):
    if padding != "same":
        raise NotImplementedError("only padding='same' (what train.py uses) is implemented")
    return _FusedSSIM.apply(img1, img2, train)


class _FusedLoss(torch.autograd.Function):
    """(1-l)*mean|I-G| + l*(1-mean ssim(I,G)) in two kernels (forward + backward)."""

    @staticmethod
    def forward(ctx, image, gt, lambda_dssim):
        L = _lib.lib()
        a, b = f32c(image), f32c(gt)
        C, H, W = a.shape
        with torch.cuda.device(a.device):
            sums = torch.zeros(2, dtype=torch.float64, device=a.device)
            maps = torch.empty((3, C, H, W), dtype=torch.float32, device=a.device)
            check(L.gsb_loss_forward(C, H, W, a.data_ptr(), b.data_ptr(), sums.data_ptr(), maps.data_ptr(),
                                     _lib.stream_ptr()), "gsb_loss_forward")
        ctx.save_for_backward(a, b, maps)
        ctx.lam = float(lambda_dssim)
        n = C * H * W
        return ((1.0 - ctx.lam) * sums[0] / n + ctx.lam * (1.0 - sums[1] / n)).float()

    @staticmethod
    def backward(ctx, grad):
        a, b, maps = ctx.saved_tensors
        C, H, W = a.shape
        with torch.cuda.device(a.device):
            out = torch.empty_like(a)
            check(_lib.lib().gsb_loss_backward(C, H, W, a.data_ptr(), b.data_ptr(), maps.data_ptr(), ctx.lam,
                                               out.data_ptr(), _lib.stream_ptr()), "gsb_loss_backward")
        return out * grad, None, None


def fused_training_loss(image, gt, lambda_dssim=0.2):
    return _FusedLoss.apply(image, gt, lambda_dssim)
