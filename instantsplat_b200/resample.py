"""Pillow's bicubic resize of 8-bit RGB images on the GPU (gsb_resample_u8_batch, DESIGN.md section 4.21): what
loadCam's PILtoTorch does with `pil_image.resize(resolution)` (Pillow's default BICUBIC, no reducing_gap) when `-r`
changes an image's size, opt-in with `--resample_images` on the train, render_views and freeview command lines.

Pillow (libImaging Resample.c, 8 bits per channel) resamples each axis with integer weights: `coefficients` builds
them in fp64 in Pillow's order, and the kernel adds the integer products, which any order adds exactly, so the bytes
are Pillow's.  There is no host path: Pillow is the test oracle, not a second runtime.
"""
from __future__ import annotations

import argparse
import functools
import math
from typing import Tuple

import numpy as np
import torch

from . import _lib
from ._lib import check

SUPPORT = 2.0          # the bicubic filter's support
PRECISION_BITS = 22    # Pillow's fixed-point weights: w * 2^22, rounded half away from zero


def _bicubic(x: float) -> float:
    """Pillow's bicubic_filter, a = -0.5, in its operation order."""
    a = -0.5
    if x < 0.0:
        x = -x
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * a
    return 0.0


@functools.lru_cache(maxsize=64)
def _tables(in_size: int, out_size: int) -> Tuple[np.ndarray, np.ndarray]:
    scale = in_size / out_size
    filterscale = max(scale, 1.0)
    support = SUPPORT * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    ss = 1.0 / filterscale
    bounds = np.zeros((out_size, 2), np.int32)
    coefs = np.zeros((out_size, ksize), np.int32)
    one = float(1 << PRECISION_BITS)
    for o in range(out_size):
        center = (o + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)                   # int(): truncation toward zero, as C's (int)
        n = min(int(center + support + 0.5), in_size) - xmin
        w = [_bicubic((x + xmin - center + 0.5) * ss) for x in range(n)]
        ww = 0.0
        for v in w:                                                  # in index order, as Pillow adds them
            ww += v
        if ww != 0.0:
            w = [v / ww for v in w]
        coefs[o, :n] = [int(-0.5 + v * one) if v < 0 else int(0.5 + v * one) for v in w]
        bounds[o] = (xmin, n)
    bounds.setflags(write=False)
    coefs.setflags(write=False)
    return bounds, coefs


def coefficients(in_size: int, out_size: int) -> Tuple[np.ndarray, np.ndarray]:
    """Pillow's precompute_coeffs and normalize_coeffs_8bpc for resizing an axis of in_size pixels to out_size:
    (bounds [out_size, 2] int32: the first source index and the tap count of each output index; coefs
    [out_size, ksize] int32: the weights times 2^22, zero past each tap count).  Built in Python fp64 in Pillow's
    order and cached per size pair; the arrays are read-only."""
    in_size, out_size = int(in_size), int(out_size)
    if in_size < 1 or out_size < 1:
        raise ValueError(f"resample.coefficients: sizes must be >= 1, got {in_size} -> {out_size}")
    return _tables(in_size, out_size)


def resize_u8(images: torch.Tensor, size: Tuple[int, int]) -> torch.Tensor:
    """Image.resize(size) (size = (width, height), BICUBIC) of every view of images, a contiguous uint8 CUDA
    [V, H, W, 3] tensor -> a new uint8 [V, height, width, 3] tensor on the same device, computed on the current
    stream.  Each view's bytes are what Pillow gives for it alone."""
    if not isinstance(images, torch.Tensor) or images.dim() != 4 or images.shape[3] != 3 \
            or images.dtype != torch.uint8 or not images.is_cuda or not images.is_contiguous():
        raise ValueError(f"resample.resize_u8: expected a contiguous uint8 CUDA [V, H, W, 3] tensor, got "
                         f"{tuple(getattr(images, 'shape', ()))} {getattr(images, 'dtype', type(images))} on "
                         f"{getattr(images, 'device', 'the host')}")
    Wo, Ho = int(size[0]), int(size[1])
    V, H, W, _ = images.shape
    if Wo < 1 or Ho < 1:
        raise ValueError(f"resample.resize_u8: the output size must be at least 1 x 1, got {Wo} x {Ho}")
    dev = images.device
    out = torch.empty(V, Ho, Wo, 3, dtype=torch.uint8, device=dev)
    if V == 0:
        return out

    def axis(n_in: int, n_out: int):
        if n_in == n_out:
            return None, None, 0
        b, c = coefficients(n_in, n_out)
        return torch.from_numpy(b.copy()).to(dev), torch.from_numpy(c.copy()).to(dev), c.shape[1]

    with torch.cuda.device(dev):
        xb, xc, xk = axis(W, Wo)
        yb, yc, yk = axis(H, Ho)
        scratch = torch.empty(V * H * Wo * 3 if (W != Wo and H != Ho) else 0, dtype=torch.uint8, device=dev)
        p = lambda t: None if t is None else t.data_ptr()
        check(_lib.lib().gsb_resample_u8_batch(V, H, W, Ho, Wo, images.data_ptr(), out.data_ptr(), p(xb), p(xc), xk,
                                               p(yb), p(yc), yk, p(scratch) if scratch.numel() else None,
                                               scratch.numel(), _lib.stream_ptr()),
              "gsb_resample_u8_batch")
    return out


def add_arg(ap: argparse.ArgumentParser) -> None:
    """--resample_images.  The namespace has no resample_images attribute unless the flag is given, so a command line
    without it parses to the namespace it parsed to before the flag existed; read it with requested(args)."""
    ap.add_argument("--resample_images", action="store_true", default=argparse.SUPPRESS,
                    help="resize the images to the size -r loads them at, on the GPU (Pillow's bicubic resize, byte "
                         "for byte); without it a -r that changes an image's size is refused")


def requested(args: argparse.Namespace) -> bool:
    """Whether --resample_images was given."""
    return bool(getattr(args, "resample_images", False))
