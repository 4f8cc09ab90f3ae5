"""Image quality of rendered views: the numbers train.py's training_report (train.py:256-290) and metrics.py
(metrics.py:55-84) report, from one batched, deterministic metrics kernel (gsb_image_metrics_batch, DESIGN.md
section 4.11).

Two conventions, both kept:
  * mode="clamp": render and target clamped to [0, 1], as training_report does.  It averages the per-channel PSNRs
    (utils/image_utils.py:17-19 on a [3, H, W] image): `psnr_channels.mean(1)`.
  * mode="png8": render and target through torchvision's save_image (8-bit, ties round up) and to_tensor (/255), as
    render.py -> metrics.py does.  metrics.py's PSNR is that of the whole image's MSE (a [1, 3, H, W] image): `psnr`.
SSIM is the training loss's (utils/loss_utils.py:55-85) on the transformed images.

NaN follows torch in both: the clamp keeps it (torch.clamp), so a render with a NaN pixel gets NaN l1, ssim and psnr,
and NaN psnr_channels in that pixel's channel (its other channels and the other views are unaffected); save_image's
quantisation makes it 0 (+inf 255, -inf 0), so png8 stays finite as render.py's PNG files do.
"""
from __future__ import annotations

from typing import Dict, Optional, Sequence

import torch

from . import _lib
from ._lib import check

MODES = {"clamp": 1, "png8": 2}     # GSB_METRIC_CLAMP, GSB_METRIC_PNG8


def metrics_from_sums(sums: torch.Tensor, H: int, W: int) -> Dict[str, torch.Tensor]:
    """The per-view metrics from the kernel's sums [V, 2 + C] (fp64: sum|a-b|, sum of the SSIM map, per-channel
    sum (a-b)^2).  Pure torch, on any device.  Identical images give an MSE of 0 and a PSNR of inf, as the reference."""
    C = sums.shape[1] - 2
    n = float(C * H * W)
    mse = sums[:, 2:] / float(H * W)
    whole = sums[:, 2:].sum(1) / n
    psnr = lambda m: 20.0 * torch.log10(1.0 / torch.sqrt(m))
    return dict(l1=sums[:, 0] / n, mse=mse, psnr_channels=psnr(mse), psnr=psnr(whole), ssim=sums[:, 1] / n)


def _mode(mode: str) -> int:
    if mode not in MODES:
        raise ValueError(f"unknown metrics mode {mode!r} (expected one of {sorted(MODES)})")
    return MODES[mode]


def _images(t, what: str, device=None) -> torch.Tensor:
    if not isinstance(t, torch.Tensor) or t.dim() != 4 or t.shape[1] != 3 or t.shape[2] < 1 or t.shape[3] < 1:
        raise ValueError(f"{what}: expected a [V, 3, H, W] tensor, got {tuple(getattr(t, 'shape', ()))}")
    if t.dtype != torch.float32:
        raise ValueError(f"{what}: expected float32, got {t.dtype}")
    if not t.is_cuda:
        raise ValueError(f"{what}: expected a CUDA tensor (there is no CPU path), got one on {t.device}")
    if device is not None and t.device != device:
        raise ValueError(f"{what}: tensor on {t.device}, expected {device}")
    return t.contiguous()


def _rows(rows, V: int, N: int, what: str):
    rows = list(range(V)) if rows is None else [int(r) for r in rows]
    if len(rows) != V:
        raise ValueError(f"{what}: {len(rows)} target rows for {V} images")
    if any(not 0 <= r < N for r in rows):
        raise ValueError(f"{what}: target rows {rows} out of range 0..{N - 1}")
    return rows


def metric_sums(imgs: torch.Tensor, gts: torch.Tensor, rows: Sequence[int], mode: int) -> torch.Tensor:
    """gsb_image_metrics_batch on checked inputs (imgs [V, 3, H, W], gts [N, 3, H, W], rows: V ints in 0..N-1, both
    contiguous fp32 on one device): the sums [V, 5] (fp64) on the device.  Two kernels, no host sync."""
    L = _lib.lib()
    V, C, H, W = imgs.shape
    dev = imgs.device
    with torch.cuda.device(dev):
        row_dev = torch.tensor(rows, dtype=torch.int32).pin_memory().to(dev, non_blocking=True)
        nbytes = L.gsb_image_metrics_scratch_bytes(V, C, H, W)
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        out = torch.empty(V, 2 + C, dtype=torch.float64, device=dev)
        check(L.gsb_image_metrics_batch(V, C, H, W, imgs.data_ptr(), gts.data_ptr(), row_dev.data_ptr(), mode,
                                        out.data_ptr(), scratch.data_ptr(), nbytes, _lib.stream_ptr()),
              "gsb_image_metrics_batch")
    return out


def image_metrics(imgs: torch.Tensor, gts: torch.Tensor, rows: Optional[Sequence[int]] = None,
                  mode: str = "clamp") -> Dict[str, torch.Tensor]:
    """Per-view metrics of imgs [V, 3, H, W] against gts [N, 3, H, W] (float32 CUDA tensors on one device): view v is
    compared with gts[rows[v]] (rows=None: gts[v], N = V).  mode: "clamp" (training_report) or "png8" (metrics.py).
    One library call; returns fp64 device tensors without waiting for the GPU:
      l1 [V] mean |a-b|; mse [V, 3] per-channel MSE; psnr_channels [V, 3] their PSNRs (training_report reports their
      mean); psnr [V] the PSNR of the whole image's MSE (metrics.py); ssim [V] mean SSIM.
    Each view's values are bit-identical from run to run and independent of the other views in the call."""
    m = _mode(mode)
    imgs = _images(imgs, "image_metrics: imgs")
    gts = _images(gts, "image_metrics: gts", imgs.device)
    if tuple(gts.shape[1:]) != tuple(imgs.shape[1:]):
        raise ValueError(f"image_metrics: gts {tuple(gts.shape)} and imgs {tuple(imgs.shape)} differ in frame size")
    V, _, H, W = imgs.shape
    if V == 0:
        raise ValueError("image_metrics: no images")
    rows = _rows(rows, V, gts.shape[0], "image_metrics")
    return metrics_from_sums(metric_sums(imgs, gts, rows, m), H, W)
