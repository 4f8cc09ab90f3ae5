"""Mip-Splatting on the stage command lines (DESIGN.md section 4.22): `--kernel_size K` on train, render_views, freeview
and pipeline.  K is the 2D Mip filter's kappa, the name render() uses (Mip-Splatting uses 0.1), and giving the flag
turns on both filters, as OptimConfig.mip_kernel_size does: train trains with them, so its ply carries filter_3D,
and the render stages build their tracker with kappa and the ply's filter_3D.

Without the flag nothing changes: the namespace has no kernel_size attribute (read it with kernel_size(args)), and a
ply that carries filter_3D renders without the filters, as render.py renders it.
"""
from __future__ import annotations

import argparse
import math
import os
from typing import List, Optional


def add_arg(ap: argparse.ArgumentParser) -> None:
    """--kernel_size K, left out of the namespace unless it is given, so a command line without it parses to the
    namespace it parsed to before the flag existed."""
    ap.add_argument("--kernel_size", type=float, metavar="K", default=argparse.SUPPRESS,
                    help="Mip-Splatting: the 2D Mip filter's kernel size (0.1 in Mip-Splatting), with the 3D smoothing "
                         "filter; render stages need a ply trained with it (its filter_3D property)")


def kernel_size(args: argparse.Namespace) -> Optional[float]:
    """The --kernel_size given, or None."""
    k = getattr(args, "kernel_size", None)
    return None if k is None else float(k)


def argv(k: Optional[float]) -> List[str]:
    """The flag as a stage's command line carries it: [] for None.  repr gives back the same float when parsed."""
    return [] if k is None else ["--kernel_size", repr(float(k))]


def kernel_refusal(k: Optional[float]) -> Optional[str]:
    """Why kappa cannot be used, or None: the 2D filter adds it to the screen-space covariance's diagonal, so it must
    be a finite number >= 0."""
    if k is None or (math.isfinite(k) and k >= 0):
        return None
    return f"--kernel_size {k}: the 2D Mip filter's kernel size must be a finite number >= 0"


def ply_refusal(k: Optional[float], ply: str) -> Optional[str]:
    """Why a render stage cannot apply the filters to ply, or None: with --kernel_size the ply must carry filter_3D (a
    model trained with the flag).  A missing ply is left to the loader, which names it."""
    if k is None or not os.path.isfile(ply):
        return None
    from .scene_io import ply_properties
    if "filter_3D" in ply_properties(ply):
        return None
    return (f"--kernel_size: {ply} has no filter_3D property, so there is no 3D filter to apply (train the model with "
            "--kernel_size)")
