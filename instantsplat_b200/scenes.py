"""Seeded synthetic scenes for the BASELINE.json configs (SURVEY.md section 8d).

Everything is generated on the CPU with a seeded ``torch.Generator`` (seed = 1000 + config index)
and moved to the device by the caller, so tests, the oracle and the CUDA path see identical inputs.

Shapes follow the reference's parameter tensors (scene/gaussian_model.py:146-172):
``xyz [P,3]``, ``f_dc [P,1,3]``, ``f_rest [P,15,3]``, ``opacity [P,1]`` (logit), ``scaling [P,3]``
(log), ``rotation [P,4]`` (raw quaternion, real first), pose table ``poses [n_views,7]`` =
[qw,qx,qy,qz,tx,ty,tz] of the world-to-camera transform
(scene/gaussian_model.py:126-136).
"""
from __future__ import annotations

import functools
import math
from dataclasses import dataclass, field
from typing import Dict, List

import torch


def _single_threaded(fn):
    """Run a generator on one CPU thread.  PyTorch splits large elementwise CPU ops into per-thread chunks, and a chunk's
    vectorised body and its tail round sin / cos / log / randn differently, so a multi-threaded generator's output
    depends on the core count.  Training amplifies such last-bit differences, so the same arguments would give different
    results on machines with different core counts.  On one thread the output is the same on every CPU with AVX2 or
    AVX-512."""
    @functools.wraps(fn)
    def run(*args, **kwargs):
        n = torch.get_num_threads()
        torch.set_num_threads(1)
        try:
            return fn(*args, **kwargs)
        finally:
            torch.set_num_threads(n)
    return run


@dataclass
class Scene:
    params: Dict[str, torch.Tensor]
    poses: torch.Tensor                 # [n_views, 7]
    width: int
    height: int
    fovx: float
    fovy: float
    sh_degree: int
    bg: torch.Tensor = field(default_factory=lambda: torch.zeros(3))
    per_point_lr: torch.Tensor | None = None
    name: str = ""

    @property
    def P(self) -> int:
        return self.params["xyz"].shape[0]

    @property
    def n_views(self) -> int:
        return self.poses.shape[0]


def _rotmat_to_quat(R: torch.Tensor) -> torch.Tensor:
    """Rotation matrix -> unit quaternion (real first); R is a proper rotation near identity."""
    w = math.sqrt(max(0.0, 1.0 + float(R[0, 0] + R[1, 1] + R[2, 2]))) / 2.0
    x = float(R[2, 1] - R[1, 2]) / (4.0 * w)
    y = float(R[0, 2] - R[2, 0]) / (4.0 * w)
    z = float(R[1, 0] - R[0, 1]) / (4.0 * w)
    return torch.tensor([w, x, y, z], dtype=torch.float32)


@_single_threaded
def random_scene(P: int = 10_000, width: int = 256, height: int = 256, seed: int = 1001,
                 sh_degree: int = 3, fovx_deg: float = 60.0) -> Scene:
    """cfg1: camera-frame random Gaussians, one perturbed-identity pose."""
    g = torch.Generator().manual_seed(seed)
    xyz = torch.rand(P, 3, generator=g)
    xyz[:, 0:2] = xyz[:, 0:2] * 3.0 - 1.5
    xyz[:, 2] = xyz[:, 2] * 4.0 + 2.0
    scaling = math.log(0.03) + 0.3 * torch.randn(P, 3, generator=g)
    rotation = torch.randn(P, 4, generator=g)
    opacity = 1.5 * torch.randn(P, 1, generator=g)
    f_dc = torch.randn(P, 1, 3, generator=g)
    f_rest = 0.1 * torch.randn(P, 15, 3, generator=g)
    pose = torch.tensor([1.0, 0, 0, 0, 0, 0, 0]) + 1e-2 * torch.randn(7, generator=g)
    fovx = math.radians(fovx_deg)
    fovy = 2.0 * math.atan(math.tan(fovx / 2) * height / width)
    return Scene(dict(xyz=xyz, f_dc=f_dc, f_rest=f_rest, opacity=opacity, scaling=scaling,
                      rotation=rotation), pose[None].clone(), width, height, fovx, fovy,
                 sh_degree, name=f"random{P}")


@_single_threaded
def surface_scene(P: int, n_views: int, width: int, height: int, seed: int, sh_degree: int = 3,
                  fovx_deg: float = 60.0, opacity_mode: str = "mid", sh_rest_std: float = 0.05
                  ) -> Scene:
    """cfg2-5: what init_geo.py produces -- per view, a regular pixel grid of P/n_views points
    unprojected with a smooth random depth in [2,6]; cameras on a small arc looking at the scene.
    Scale = log(grid spacing in world units) (the kNN init rule of
    scene/gaussian_model.py:156-160 for a regular grid); quat = (1,0,0,0);
    opacity 0.1 ("init") or logit ~ N(0,1.5^2) ("mid"); colours from a procedural texture.
    """
    g = torch.Generator().manual_seed(seed)
    fovx = math.radians(fovx_deg)
    tanx = math.tan(fovx / 2)
    tany = tanx * height / width
    fovy = 2.0 * math.atan(tany)
    per = P // n_views
    gw = max(1, int(round(math.sqrt(per * width / height))))
    gh = max(1, per // gw)
    centre = torch.tensor([0.0, 0.0, 4.0])
    xyz_all, scale_all, col_all = [], [], []
    poses = []
    for v in range(n_views):
        ang = (v - (n_views - 1) / 2.0) * (0.2 / max(1, n_views - 1)) * 2.0   # ~0.2*depth baseline
        # camera centre on an arc of radius 4 around `centre`, looking at it
        c = centre + torch.tensor([4.0 * math.sin(ang), 0.0, -4.0 * math.cos(ang)])
        fwd = (centre - c) / (centre - c).norm()
        up = torch.tensor([0.0, 1.0, 0.0])
        right = torch.linalg.cross(up, fwd)
        right = right / right.norm()
        up2 = torch.linalg.cross(fwd, right)
        Rwc = torch.stack([right, up2, fwd], dim=0)          # rows: camera axes in world
        t = -Rwc @ c
        poses.append(torch.cat([_rotmat_to_quat(Rwc), t]))
        n = gw * gh if v < n_views - 1 else P - (gw * gh) * (n_views - 1)
        ii = torch.arange(n)
        u = ((ii % gw).float() + 0.5) / gw * 2 - 1
        w_ = (torch.div(ii, gw, rounding_mode="floor").float() % gh + 0.5) / gh * 2 - 1
        ph = torch.rand(4, 3, generator=g) * 6.283
        fr = torch.rand(4, 2, generator=g) * 2.5 + 0.5
        d = torch.zeros(n)
        for k in range(4):
            d = d + torch.sin(fr[k, 0] * u * 3.0 + ph[k, 0]) * torch.cos(fr[k, 1] * w_ * 3.0 + ph[k, 1])
        d = 4.0 + d * 0.5                                     # in [2, 6]
        pc = torch.stack([u * tanx * d, w_ * tany * d, d], dim=-1)
        pw = (pc - t[None]) @ Rwc                             # R^T (p - t)
        spacing = d * (2.0 * tanx / gw)
        xyz_all.append(pw)
        scale_all.append(torch.log(spacing)[:, None].repeat(1, 3))
        tex = 0.5 + 0.5 * torch.stack([torch.sin(7 * pw[:, 0] + 1.0), torch.sin(5 * pw[:, 1] + 2.0),
                                       torch.sin(9 * pw[:, 0] * pw[:, 1] + 0.5)], dim=-1)
        col_all.append(tex)
    xyz = torch.cat(xyz_all)[:P]
    scaling = torch.cat(scale_all)[:P] + 0.05 * torch.randn(P, 3, generator=g)
    cols = torch.cat(col_all)[:P]
    f_dc = ((cols - 0.5) / 0.28209479177387814)[:, None, :].contiguous()
    f_rest = sh_rest_std * torch.randn(P, 15, 3, generator=g)
    rotation = torch.zeros(P, 4)
    rotation[:, 0] = 1.0
    if opacity_mode == "init":
        opacity = torch.full((P, 1), math.log(0.1 / 0.9))
    else:
        opacity = 1.5 * torch.randn(P, 1, generator=g)
    ppl = 1.0 + 99.0 * (1.0 - torch.sigmoid(torch.randn(P, 1, generator=g)))
    return Scene(dict(xyz=xyz.contiguous(), f_dc=f_dc, f_rest=f_rest, opacity=opacity,
                      scaling=scaling.contiguous(), rotation=rotation),
                 torch.stack(poses), width, height, fovx, fovy, sh_degree, per_point_lr=ppl,
                 name=f"surface{P}x{n_views}@{width}x{height}")


def make_config(idx: int, scale: float = 1.0) -> Scene:
    """BASELINE.json ``configs[idx]``.  ``scale`` < 1 shrinks P (tests only)."""
    if idx == 0:
        return random_scene(int(10_000 * scale), 256, 256, seed=1000)
    if idx == 1:
        return surface_scene(int(200_000 * scale), 3, 512, 512, seed=1001, sh_degree=0)
    if idx in (2, 3):
        return surface_scene(int(1_000_000 * scale), 12, 1920, 1080, seed=1002, sh_degree=3)
    if idx == 4:
        return surface_scene(int(4_000_000 * scale), 24, 3840, 2160, seed=1004, sh_degree=3)
    raise ValueError(idx)


@_single_threaded
def perturbed_copy(scene: Scene, seed: int = 7, sigma: float = 0.02) -> Dict[str, torch.Tensor]:
    """Parameters of a perturbed copy (used to render non-trivial ground-truth images)."""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for k, v in scene.params.items():
        out[k] = v + sigma * torch.randn(v.shape, generator=g) * (0.2 if k == "xyz" else 1.0)
    return out
