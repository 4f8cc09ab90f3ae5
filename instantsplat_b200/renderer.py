"""Drop-in for `gaussian_renderer.render` (boundary B1): gaussian_renderer/__init__.py:23-144.

Same signature and result dict.  With the default pipeline flags (no compute_cov3D_python /
convert_SHs_python / override_color) the whole body -- pose pre-transform (:81-89), activations,
feature cat, rasterizer -- is ONE fused call into libgsb200.so; the other branches go through the
generic GaussianRasterizer exactly like the reference does."""
from __future__ import annotations

import math

import torch

from .rasterizer import GaussianRasterizationSettings, GaussianRasterizer, rasterize_fused

# FUSED = True : the whole body (pose pre-transform, activations, feature cat, rasterizer) is ONE call into the library.
# FUSED = False: the reference's own body is restated op for op (PyTorch pose pre-transform -> GaussianRasterizer), i.e.
#                what an UNCHANGED gaussian_renderer/__init__.py does on top of the rasterizer shim;
#                bench.py times it as `dropin_unchanged`.  Env GSB_FUSED_RENDER=0 selects it process-wide.
import os as _os

FUSED = _os.environ.get("GSB_FUSED_RENDER", "1") != "0"
_RASTERIZER = (GaussianRasterizationSettings, GaussianRasterizer)    # replaceable by the CPU tests

_const_cache = {}


def _identity_consts(device):
    c = _const_cache.get(device)
    if c is None:
        c = (torch.eye(4, device=device), torch.zeros(3, device=device))
        _const_cache[device] = c
    return c


def get_camera_from_tensor(pose):
    """utils/pose_utils.py:57-84 (used only by the non-fused branches)."""
    q = pose[:4] / torch.sqrt((pose[:4] * pose[:4]).sum())
    r, x, y, z = q[0], q[1], q[2], q[3]
    R = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                     2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                     2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)]).reshape(3, 3)
    w2c = torch.eye(4, device=pose.device, dtype=pose.dtype)
    w2c = torch.cat([torch.cat([R, pose[4:7].reshape(3, 1)], 1), w2c[3:4]], 0)
    return w2c


def quadmultiply(q1, q2):
    """utils/pose_utils.py:86-104."""
    w1, x1, y1, z1 = q1.unbind(-1)
    w2, x2, y2, z2 = q2.unbind(-1)
    return torch.stack([w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2,
                        w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2, w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2], dim=-1)


def render(viewpoint_camera, pc, pipe, bg_color, scaling_modifier=1.0, override_color=None, camera_pose=None):
    """Render the scene.  Background tensor (bg_color) must be on GPU!"""
    xyz = pc.get_xyz
    screenspace_points = torch.zeros_like(xyz, dtype=xyz.dtype, requires_grad=True, device=xyz.device) + 0
    try:
        screenspace_points.retain_grad()
    except Exception:
        pass
    tanfovx = math.tan(viewpoint_camera.FoVx * 0.5)
    tanfovy = math.tan(viewpoint_camera.FoVy * 0.5)
    w2c, campos = _identity_consts(xyz.device)
    Settings, Rasterizer = _RASTERIZER
    # identity view: projmatrix = I @ P^T (reference :55-59)
    raster_settings = Settings(
        image_height=int(viewpoint_camera.image_height), image_width=int(viewpoint_camera.image_width),
        tanfovx=tanfovx, tanfovy=tanfovy, bg=bg_color, scale_modifier=scaling_modifier, viewmatrix=w2c,
        projmatrix=viewpoint_camera.projection_matrix, sh_degree=pc.active_sh_degree, campos=campos,
        prefiltered=False, debug=bool(getattr(pipe, "debug", False)))
    fused = (FUSED and override_color is None and not getattr(pipe, "compute_cov3D_python", False)
             and not getattr(pipe, "convert_SHs_python", False))
    if fused:
        rendered_image, radii = rasterize_fused(pc._xyz, pc._rotation, pc._scaling, pc._opacity,
                                                pc._features_dc, pc._features_rest, camera_pose,
                                                screenspace_points, raster_settings)
    else:
        rel_w2c = get_camera_from_tensor(camera_pose)
        gaussians_xyz, gaussians_rot = pc._xyz.clone(), pc._rotation.clone()            # reference :83-84
        homo = torch.cat((gaussians_xyz, torch.ones(xyz.shape[0], 1, device=xyz.device)), dim=1)
        means3D = (rel_w2c @ homo.T).T[:, :3]
        rots = quadmultiply(camera_pose[:4], gaussians_rot)
        scales = rotations = cov3D_precomp = shs = colors_precomp = None
        if getattr(pipe, "compute_cov3D_python", False):
            cov3D_precomp = pc.get_covariance(scaling_modifier)
        else:
            scales, rotations = pc.get_scaling, rots
        if override_color is None:
            if getattr(pipe, "convert_SHs_python", False):
                from .sh import eval_sh_python
                colors_precomp = eval_sh_python(pc, viewpoint_camera)
            else:
                shs = pc.get_features
        else:
            colors_precomp = override_color
        rasterizer = Rasterizer(raster_settings=raster_settings)
        rendered_image, radii = rasterizer(means3D=means3D, means2D=screenspace_points, shs=shs,
                                           colors_precomp=colors_precomp, opacities=pc.get_opacity,
                                           scales=scales, rotations=rotations, cov3D_precomp=cov3D_precomp)
    return {"render": rendered_image, "viewspace_points": screenspace_points,
            "visibility_filter": radii > 0, "radii": radii}
