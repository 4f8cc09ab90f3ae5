"""Host-side mirror of the part of the reference's `GaussianModel` that the training hot path touches
(scene/gaussian_model.py): parameter tensors and their activations (:101-121), the pose table
(:126-136), `oneupSHdegree` (:142-144), `create_from_pcd` (:146-172, with `distCUDA2` served by libgsb200.so),
`capture` / `restore` (:65-99), `training_setup` (:174-200), `training_setup_pp` (:203-232),
`update_learning_rate` (:234-243) and the optimizer-state surgery behind
densify / prune / opacity reset (:280-283, :328-478; SURVEY.md section 8 row f4).

Same attribute and method names, argument meaning and param-group layout as the reference, so that the body of
train.py:140-211 runs on it verbatim (tests/test_reference_loop.py, bench.py `dropin_*`).  The
reference tree is not a dependency, hence a mirror rather than an import; tests/test_reference_shims_cpu.py checks
the mirror on the CPU against what the REAL reference modules computed (tests/golden/ref_loop.npz).
"""
from __future__ import annotations

import math
from types import SimpleNamespace
from typing import Callable, Dict, Optional

import torch
from torch import nn

from .per_point_adam import PerPointAdam
from .trainer import ADAM_BETAS, ADAM_EPS, OptimConfig, group_lrs, lr_schedules

SH_C0 = 0.28209479177387814


def inverse_sigmoid(x):
    return torch.log(x / (1 - x))


def optimization_defaults(**over):
    """arguments/__init__.py:73-94 (OptimizationParams defaults, as in OptimConfig; InstantSplat's scripts pass
    --iterations 1000 --pp_optimizer --optim_pose)."""
    keys = ("iterations", "position_lr_init", "position_lr_final", "position_lr_delay_mult", "position_lr_max_steps",
            "feature_lr", "opacity_lr", "scaling_lr", "rotation_lr", "percent_dense", "lambda_dssim",
            "densification_interval", "opacity_reset_interval", "densify_from_iter", "densify_until_iter",
            "densify_grad_threshold", "pp_optimizer", "optim_pose")
    d = {k: getattr(OptimConfig, k) for k in keys}
    d["random_background"] = False
    d.update(over)
    return SimpleNamespace(**d)


class GaussianModel:
    _ATTR = dict(xyz="_xyz", f_dc="_features_dc", f_rest="_features_rest", opacity="_opacity", scaling="_scaling",
                 rotation="_rotation")

    def __init__(self, sh_degree: int, device="cuda"):
        self.active_sh_degree = 0
        self.max_sh_degree = sh_degree
        self.device = torch.device(device)
        e = torch.empty(0)
        self._xyz = self._features_dc = self._features_rest = self._scaling = self._rotation = self._opacity = e
        self.max_radii2D = self.xyz_gradient_accum = self.denom = e
        self.optimizer = None
        self.percent_dense = 0
        self.spatial_lr_scale = 0
        self.per_point_lr = None
        self.P = None
        self.filter_3D = None           # Mip-Splatting's 3D smoothing filter [P, 1] (DESIGN.md section 4.7), a constant
        self._filter_cams = None

    # ---- activations (reference :101-121) ----------------------------------------------------
    get_xyz = property(lambda s: s._xyz)
    get_scaling = property(lambda s: torch.exp(s._scaling))
    get_rotation = property(lambda s: torch.nn.functional.normalize(s._rotation))
    get_opacity = property(lambda s: torch.sigmoid(s._opacity))
    get_features = property(lambda s: torch.cat((s._features_dc, s._features_rest), dim=1))

    # ---- Mip-Splatting's 3D smoothing filter (same names as its gaussian_model.py) ------------
    @property
    def get_scaling_with_3D_filter(self):
        return torch.sqrt(torch.square(self.get_scaling) + torch.square(self.filter_3D))

    @property
    def get_opacity_with_3D_filter(self):
        s2 = torch.square(self.get_scaling)
        coef = torch.sqrt(s2.prod(dim=1) / (s2 + torch.square(self.filter_3D)).prod(dim=1))
        return self.get_opacity * coef[..., None]

    @torch.no_grad()
    def compute_3D_filter(self, cameras):
        """filter_3D from the training views' current poses (self.P, one row per camera) and their shared intrinsics
        (FoVx, FoVy, image_width, image_height), computed by gsb_mip_filter3d.  The cameras are remembered so that
        densification_postfix can recompute the filter for the new rows."""
        from .frame import mip_filter3d
        c0 = cameras[0]
        intr = lambda c: (int(c.image_width), int(c.image_height), float(c.FoVx), float(c.FoVy))
        if any(intr(c) != intr(c0) for c in cameras):
            raise ValueError("compute_3D_filter: the training views must share one intrinsics")
        W, H, fovx, fovy = intr(c0)
        f = mip_filter3d(self._xyz, self.P[:len(cameras)], W, H, math.tan(fovx * 0.5), math.tan(fovy * 0.5))
        self.filter_3D = f[:, None]
        self._filter_cams = list(cameras)
        return self.filter_3D

    def get_covariance(self, scaling_modifier=1):
        """Upper triangle of R S S^T R^T with the NORMALISED quaternion (reference :32-36, general_utils.py:64-110)."""
        q = torch.nn.functional.normalize(self._rotation)
        r, x, y, z = q.unbind(-1)
        R = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y), 2 * (x * y + r * z),
                         1 - 2 * (x * x + z * z), 2 * (y * z - r * x), 2 * (x * z - r * y), 2 * (y * z + r * x),
                         1 - 2 * (x * x + y * y)], -1).reshape(-1, 3, 3)
        M = R * (scaling_modifier * self.get_scaling)[:, None, :]
        S = M @ M.transpose(1, 2)
        return torch.stack([S[:, 0, 0], S[:, 0, 1], S[:, 0, 2], S[:, 1, 1], S[:, 1, 2], S[:, 2, 2]], -1)

    # ---- pose table (reference :126-136) -----------------------------------------------------
    def init_RT_seq(self, poses):
        """poses: [n_views, 7] = (qw,qx,qy,qz,tx,ty,tz) of the world-to-camera transforms, or a list of 4x4 W2C
        matrices (converted like utils/pose_utils.get_tensor_from_camera)."""
        if not torch.is_tensor(poses):
            poses = torch.stack([w2c_to_pose(torch.as_tensor(m, dtype=torch.float32)) for m in poses])
        self.P = poses.to(self.device).float().contiguous().requires_grad_(True)

    def get_RT(self, idx):
        return self.P[idx]

    def oneupSHdegree(self):
        if self.active_sh_degree < self.max_sh_degree:
            self.active_sh_degree += 1

    # ---- initialisation (reference :146-172) -------------------------------------------------
    def create_from_pcd(self, points, colors, spatial_lr_scale: float, scale_gaussian=None):
        """points [P,3], colors [P,3] in [0,1].  Scale = sqrt of the mean squared distance to the 3 nearest
        neighbours (simple_knn.distCUDA2 -> gsb_knn_mean_dist2), optionally capped by `scale_gaussian`."""
        from .knn import distCUDA2
        self.spatial_lr_scale = spatial_lr_scale
        dev = self.device
        xyz = torch.as_tensor(points).float().to(dev).contiguous()
        n = xyz.shape[0]
        M = (self.max_sh_degree + 1) ** 2
        f_dc = ((torch.as_tensor(colors).float().to(dev) - 0.5) / SH_C0)[:, None, :].contiguous()
        f_rest = torch.zeros(n, M - 1, 3, device=dev)
        dist2 = torch.clamp_min(distCUDA2(xyz), 0.0000001)
        if scale_gaussian is not None:
            # squared in its own dtype, then rounded to fp32, as the reference does (torch.from_numpy(sg ** 2).float())
            dist2 = torch.min((torch.as_tensor(scale_gaussian) ** 2).float().to(dev), dist2)
        scales = torch.log(torch.sqrt(dist2))[..., None].repeat(1, 3)
        rots = torch.zeros(n, 4, device=dev)
        rots[:, 0] = 1
        opac = inverse_sigmoid(0.1 * torch.ones(n, 1, device=dev))
        self._set_params(dict(xyz=xyz, f_dc=f_dc, f_rest=f_rest, opacity=opac, scaling=scales, rotation=rots))
        self.max_radii2D = torch.zeros(n, device=dev)

    def _set_params(self, tensors: Dict[str, torch.Tensor]):
        for g, t in tensors.items():
            setattr(self, self._ATTR[g], nn.Parameter(t.to(self.device).float().contiguous().requires_grad_(True)))

    @classmethod
    def from_scene(cls, scene, device="cuda", active_sh_degree: Optional[int] = None):
        """Bench / test helper: parameters and poses of a synthetic `Scene` (instantsplat_b200/scenes.py)."""
        m = cls(3, device)
        m._fill_from_scene(scene, active_sh_degree)
        return m

    def _fill_from_scene(self, scene, active_sh_degree: Optional[int]):
        self._set_params(scene.params)
        self.active_sh_degree = scene.sh_degree if active_sh_degree is None else active_sh_degree
        self.init_RT_seq(scene.poses)
        self.per_point_lr = None if scene.per_point_lr is None else scene.per_point_lr.to(self.device).float().reshape(-1, 1)
        self.max_radii2D = torch.zeros(scene.P, device=self.device)
        self.spatial_lr_scale = 1.0

    # ---- optimizer (reference :174-243) ------------------------------------------------------
    def training_setup_pp(self, training_args=None, confidence_lr=None):
        if confidence_lr is not None:
            self.per_point_lr = confidence_lr
        groups = self._setup_groups(training_args or optimization_defaults())
        groups[0]["per_point_lr"] = self.per_point_lr
        self.optimizer = PerPointAdam(groups, lr=0, betas=ADAM_BETAS, eps=ADAM_EPS, weight_decay=0.0)
        return self.optimizer

    def training_setup(self, training_args=None):
        """Reference :174-200: the groups and learning rates of training_setup_pp, without the per-point multiplier, on
        torch.optim.Adam."""
        self.optimizer = torch.optim.Adam(self._setup_groups(training_args or optimization_defaults()), lr=0.0,
                                          eps=ADAM_EPS)
        return self.optimizer

    def _setup_groups(self, a):
        """What both setups share: the densification statistics, the two schedules and the seven param groups."""
        n = self.get_xyz.shape[0]
        self.percent_dense = a.percent_dense
        self.xyz_gradient_accum = torch.zeros(n, 1, device=self.device)
        self.denom = torch.zeros(n, 1, device=self.device)
        self.xyz_scheduler_args, self.cam_scheduler_args = lr_schedules(a, self.spatial_lr_scale)
        return [{"params": [self.P if g == "pose" else getattr(self, self._ATTR[g])], "lr": lr, "name": g}
                for g, lr in group_lrs(a, self.spatial_lr_scale).items()]

    # ---- checkpoints (reference :65-99; train.py:103-105, :225-227) ---------------------------
    def capture(self):
        """The reference's 13-tuple, in its order: what train.py saves as chkpnt<N>.pth."""
        return (self.active_sh_degree, self._xyz, self._features_dc, self._features_rest, self._scaling, self._rotation,
                self._opacity, self.max_radii2D, self.xyz_gradient_accum, self.denom, self.optimizer.state_dict(),
                self.spatial_lr_scale, self.P)

    def restore(self, model_args, training_args=None):
        """Reference :82-99.  Like the reference, this calls training_setup, not training_setup_pp: a restored model
        continues on torch.optim.Adam without the per-point learning rate, even when the checkpoint was written by a
        PerPointAdam run (the saved groups, `per_point_lr` key included, replace the new ones; Adam ignores the key).
        A state dict with extra top-level keys (JointTrainer's checkpoints) loads the same way: load_state_dict reads
        only `state` and `param_groups`."""
        (self.active_sh_degree, self._xyz, self._features_dc, self._features_rest, self._scaling, self._rotation,
         self._opacity, self.max_radii2D, xyz_gradient_accum, denom, opt_dict, self.spatial_lr_scale,
         self.P) = model_args
        self.training_setup(training_args)
        self.xyz_gradient_accum = xyz_gradient_accum
        self.denom = denom
        self.optimizer.load_state_dict(opt_dict)

    def update_learning_rate(self, iteration):
        for group in self.optimizer.param_groups:
            if group["name"] == "pose":
                group["lr"] = self.cam_scheduler_args(iteration)
            elif group["name"] == "xyz":
                group["lr"] = self.xyz_scheduler_args(iteration)

    # ---- optimizer-state surgery (reference :280-283, :328-478; row f4) -----------------------
    def _rebuild_groups(self, edit: Callable[[str, torch.Tensor, Optional[dict]], tuple]):
        """For every Gaussian param group: (new_param_tensor, new_state_or_None) = edit(name, old_param, old_state);
        the group's Parameter object is replaced and the optimizer state re-keyed, like the reference's
        _prune_optimizer / cat_tensors_to_optimizer / replace_tensor_to_optimizer."""
        out = {}
        for group in self.optimizer.param_groups:
            name = group["name"]
            if name not in self._ATTR:
                continue
            old = group["params"][0]
            state = self.optimizer.state.get(old, None)
            res = edit(name, old, state)
            if res is None:
                continue
            new_t, new_state = res
            if state is not None:
                del self.optimizer.state[old]
            newp = nn.Parameter(new_t.requires_grad_(True))
            group["params"][0] = newp
            if new_state is not None:
                self.optimizer.state[newp] = new_state
            setattr(self, self._ATTR[name], newp)
            out[name] = newp
        return out

    def prune_points(self, mask):
        """Remove the Gaussians where `mask` is True (parameters, Adam moments, densification statistics)."""
        keep = ~mask

        def edit(name, p, st):
            if st is not None:
                st["exp_avg"], st["exp_avg_sq"] = st["exp_avg"][keep], st["exp_avg_sq"][keep]
            return p.detach()[keep], st

        self._rebuild_groups(edit)
        if self.filter_3D is not None:
            self.filter_3D = self.filter_3D[keep]
        self.xyz_gradient_accum = self.xyz_gradient_accum[keep]
        self.denom = self.denom[keep]
        self.max_radii2D = self.max_radii2D[keep]
        if self.per_point_lr is not None:
            self.per_point_lr = self.per_point_lr[keep]
            self.optimizer.param_groups[0]["per_point_lr"] = self.per_point_lr

    def densification_postfix(self, new_xyz, new_features_dc, new_features_rest, new_opacities, new_scaling,
                              new_rotation, new_per_point_lr=None):
        """Append Gaussians (zero Adam moments for the new rows) and reset the densification statistics."""
        ext = dict(xyz=new_xyz, f_dc=new_features_dc, f_rest=new_features_rest, opacity=new_opacities,
                   scaling=new_scaling, rotation=new_rotation)

        def edit(name, p, st):
            e = ext[name].to(p.device)
            if st is not None:
                st["exp_avg"] = torch.cat((st["exp_avg"], torch.zeros_like(e)), dim=0)
                st["exp_avg_sq"] = torch.cat((st["exp_avg_sq"], torch.zeros_like(e)), dim=0)
            return torch.cat((p.detach(), e), dim=0), st

        self._rebuild_groups(edit)
        n = self.get_xyz.shape[0]
        self.xyz_gradient_accum = torch.zeros(n, 1, device=self.device)
        self.denom = torch.zeros(n, 1, device=self.device)
        self.max_radii2D = torch.zeros(n, device=self.device)
        if self.per_point_lr is not None:
            add = new_per_point_lr if new_per_point_lr is not None else torch.ones(new_xyz.shape[0], 1, device=self.device)
            self.per_point_lr = torch.cat((self.per_point_lr, add.to(self.device)), dim=0)
            self.optimizer.param_groups[0]["per_point_lr"] = self.per_point_lr
        if self.filter_3D is not None:
            if self._filter_cams is not None:
                self.compute_3D_filter(self._filter_cams)
            else:
                # filter_3D was set directly (e.g. loaded from a PLY), so there are no cameras to recompute it from: the
                # new rows take the largest existing size, the rule for Gaussians no training view counts for
                fill = self.filter_3D.max() if self.filter_3D.numel() else torch.zeros((), device=self.device)
                add = fill.reshape(1, 1).expand(new_xyz.shape[0], 1).to(self.filter_3D)
                self.filter_3D = torch.cat((self.filter_3D, add), dim=0)

    def reset_opacity(self):
        """opacity <- min(opacity, 0.01) in logit space, Adam moments of the opacity tensor zeroed (reference :280-283)."""
        new = inverse_sigmoid(torch.min(self.get_opacity, torch.ones_like(self.get_opacity) * 0.01)).detach()

        def edit(name, p, st):
            if name != "opacity":
                return None
            if st is not None:
                st["exp_avg"], st["exp_avg_sq"] = torch.zeros_like(new), torch.zeros_like(new)
            return new, st

        self._rebuild_groups(edit)

    def densify_and_clone(self, grads, grad_threshold, scene_extent):
        sel = (torch.norm(grads, dim=-1) >= grad_threshold) & \
              (torch.max(self.get_scaling, dim=1).values <= self.percent_dense * scene_extent)
        self.densification_postfix(self._xyz[sel].detach(), self._features_dc[sel].detach(),
                                   self._features_rest[sel].detach(), self._opacity[sel].detach(),
                                   self._scaling[sel].detach(), self._rotation[sel].detach(),
                                   None if self.per_point_lr is None else self.per_point_lr[sel])

    def densify_and_split(self, grads, grad_threshold, scene_extent, N=2, generator=None):
        n0 = self.get_xyz.shape[0]
        padded = torch.zeros(n0, device=self.device)
        padded[:grads.shape[0]] = grads.squeeze()
        sel = (padded >= grad_threshold) & (torch.max(self.get_scaling, dim=1).values > self.percent_dense * scene_extent)
        stds = self.get_scaling[sel].repeat(N, 1)
        samples = torch.normal(mean=torch.zeros_like(stds), std=stds, generator=generator)
        q = torch.nn.functional.normalize(self._rotation[sel])
        r, x, y, z = q.unbind(-1)
        R = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y), 2 * (x * y + r * z),
                         1 - 2 * (x * x + z * z), 2 * (y * z - r * x), 2 * (x * z - r * y), 2 * (y * z + r * x),
                         1 - 2 * (x * x + y * y)], -1).reshape(-1, 3, 3).repeat(N, 1, 1)
        new_xyz = torch.bmm(R, samples.unsqueeze(-1)).squeeze(-1) + self.get_xyz[sel].repeat(N, 1)
        new_scaling = torch.log(self.get_scaling[sel].repeat(N, 1) / (0.8 * N))
        self.densification_postfix(new_xyz.detach(), self._features_dc[sel].repeat(N, 1, 1).detach(),
                                   self._features_rest[sel].repeat(N, 1, 1).detach(), self._opacity[sel].repeat(N, 1).detach(),
                                   new_scaling.detach(), self._rotation[sel].repeat(N, 1).detach(),
                                   None if self.per_point_lr is None else self.per_point_lr[sel].repeat(N, 1))
        self.prune_points(torch.cat((sel, torch.zeros(N * int(sel.sum()), device=self.device, dtype=torch.bool))))

    def densify_and_prune(self, max_grad, min_opacity, extent, max_screen_size, clone_and_split=False, generator=None):
        """Reference :455-474 (InstantSplat keeps clone / split commented out; `clone_and_split=True` enables the
        vanilla-3DGS behaviour, split samples drawn from `generator`).  The rows of densify_and_clone,
        densify_and_split and the prune come from one `densify_plan` (shared with JointTrainer) and are applied in one
        rebuild; the result is that of running the three in sequence."""
        from .densify import densify_plan
        plan = densify_plan(self._xyz.detach(), self._scaling.detach(), self._rotation.detach(), self._opacity.detach(),
                            self.xyz_gradient_accum, self.denom, self.max_radii2D, max_grad, min_opacity, extent,
                            max_screen_size, self.percent_dense, clone_and_split, generator)
        self.apply_densify_plan(plan)
        return plan

    def apply_densify_plan(self, plan):
        computed = dict(xyz=plan.split_xyz, scaling=plan.split_scaling)

        def edit(name, p, st):
            if st is not None:
                st["exp_avg"], st["exp_avg_sq"] = plan.moments(st["exp_avg"]), plan.moments(st["exp_avg_sq"])
            return plan.gather(p.detach(), computed.get(name)), st

        xyz_before_prune = plan.gather(self._xyz.detach(), plan.split_xyz, prune=False) if plan.reset_stats else None
        self._rebuild_groups(edit)
        if plan.reset_stats:     # densification_postfix ran
            n = plan.P
            self.xyz_gradient_accum = torch.zeros(n, 1, device=self.device)
            self.denom = torch.zeros(n, 1, device=self.device)
            self.max_radii2D = torch.zeros(n, device=self.device)
        else:
            self.xyz_gradient_accum = self.xyz_gradient_accum[plan.src]
            self.denom = self.denom[plan.src]
            self.max_radii2D = self.max_radii2D[plan.src]
        if self.per_point_lr is not None:
            self.per_point_lr = plan.gather(self.per_point_lr)
            self.optimizer.param_groups[0]["per_point_lr"] = self.per_point_lr
        if self.filter_3D is not None:
            if plan.reset_stats and self._filter_cams is not None:
                # postfix recomputes from the cameras over the rows before the prune, which then keeps its rows
                cams = self._filter_cams
                c0 = cams[0]
                f = mip_filter3d_of(xyz_before_prune, self.P[:len(cams)], c0)
                self.filter_3D = f[:, None][plan.keep]
            elif plan.reset_stats:
                # no cameras: new rows take the largest existing size (densification_postfix)
                fill = self.filter_3D.max() if self.filter_3D.numel() else torch.zeros((), device=self.device)
                f = self.filter_3D[plan.src2].clone()
                f[plan.new2] = fill.to(f)
                self.filter_3D = f[plan.keep]
            else:
                self.filter_3D = self.filter_3D[plan.src]

    def add_densification_stats(self, viewspace_point_tensor, update_filter):
        self.xyz_gradient_accum[update_filter] += torch.norm(viewspace_point_tensor.grad[update_filter, :2], dim=-1,
                                                              keepdim=True)
        self.denom[update_filter] += 1


def mip_filter3d_of(xyz, poses, cam):
    """gsb_mip_filter3d for camera-like intrinsics (FoVx, FoVy, image_width, image_height)."""
    from .frame import mip_filter3d
    return mip_filter3d(xyz, poses, int(cam.image_width), int(cam.image_height), math.tan(float(cam.FoVx) * 0.5),
                        math.tan(float(cam.FoVy) * 0.5))


def w2c_to_pose(RT: torch.Tensor) -> torch.Tensor:
    """4x4 world-to-camera -> (qw,qx,qy,qz,tx,ty,tz); rotation -> quaternion by the trace method
    (utils/pose_utils.py:183-240 get_tensor_from_camera / rotation2quad)."""
    R, t = RT[:3, :3].double(), RT[:3, 3]
    tr = float(R[0, 0] + R[1, 1] + R[2, 2])
    if tr > 0:
        s = math.sqrt(tr + 1.0) * 2
        q = [0.25 * s, float(R[2, 1] - R[1, 2]) / s, float(R[0, 2] - R[2, 0]) / s, float(R[1, 0] - R[0, 1]) / s]
    elif R[0, 0] > R[1, 1] and R[0, 0] > R[2, 2]:
        s = math.sqrt(1.0 + float(R[0, 0] - R[1, 1] - R[2, 2])) * 2
        q = [float(R[2, 1] - R[1, 2]) / s, 0.25 * s, float(R[0, 1] + R[1, 0]) / s, float(R[0, 2] + R[2, 0]) / s]
    elif R[1, 1] > R[2, 2]:
        s = math.sqrt(1.0 + float(R[1, 1] - R[0, 0] - R[2, 2])) * 2
        q = [float(R[0, 2] - R[2, 0]) / s, float(R[0, 1] + R[1, 0]) / s, 0.25 * s, float(R[1, 2] + R[2, 1]) / s]
    else:
        s = math.sqrt(1.0 + float(R[2, 2] - R[0, 0] - R[1, 1])) * 2
        q = [float(R[1, 0] - R[0, 1]) / s, float(R[0, 2] + R[2, 0]) / s, float(R[1, 2] + R[2, 1]) / s, 0.25 * s]
    return torch.cat([torch.tensor(q, dtype=torch.float32), t.float()])


class SimpleGaussianModel(GaussianModel):
    """Back-compat constructor: a `GaussianModel` filled from a synthetic `Scene`."""

    def __init__(self, scene, device="cuda", sh_degree=None):
        super().__init__(3, device)
        self._fill_from_scene(scene, sh_degree)


class PipelineDefaults:
    """arguments/__init__.py:66-71"""
    convert_SHs_python = False
    compute_cov3D_python = False
    debug = False
