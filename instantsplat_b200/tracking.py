"""Pose-only "tracking" mode (SURVEY.md section 8 row f2): the test-view pose optimisation of
render.py:99-170 as a device-resident loop.

Reference semantics, per test view:
  * Gaussians frozen (render.py:106-111); the 7 pose parameters start from the view's W2C (:115);
  * torch.optim.Adam, groups {T: lr 0.003, q: lr 0.001}, betas (0.9, 0.999), weight_decay 1e-4 (:119-125), with
    CosineAnnealingLR(T_max=num_iter, eta_min=1e-4) stepped once per iteration (:128, :156);
  * loss = l1_loss_mask(render, gt, mask = render > 0) (:136-139; utils/loss_utils.py:17-23);
  * the candidate pose is the one AFTER an optimizer step whose pre-step loss was the lowest so far (:146-151);
  * the result is that candidate (:158-161).

Here every iteration is: fused-pose preprocess -> binning -> blend -> masked-L1 (one pass: loss sums and dL/dimage)
-> blend backward specialised for this mode (8 accumulated values per Gaussian, no per-Gaussian gradient writes) ->
pose-gradient reduction -> gsb_track_step (normalisation, Adam, candidate bookkeeping on the device).  The host only
evaluates the cosine schedule; nothing waits for the GPU until the best pose is read back after the last iteration.

optimize_batch runs the loop for many test views at once (render.py:99 loops over them; they are independent and
share the frozen cloud and the intrinsics): every kernel above runs once per iteration for the whole batch, with a
view index, and each view's result is bit-identical to optimize() on that view alone (DESIGN.md section 4.6).
"""
from __future__ import annotations

import math
from typing import Optional

import torch

from . import _lib
from ._lib import GsbCamera, GsbGaussians, check
from .frame import ST_OVERFLOW, ST_WORDS, Frame, IdentityView, capacity, gaussians, mip_filter, read_R


def cosine_lr(base_lr: float, k: int, t_max: int, eta_min: float = 1e-4) -> float:
    """Closed form of torch.optim.lr_scheduler.CosineAnnealingLR after k scheduler steps."""
    return eta_min + (base_lr - eta_min) * (1.0 + math.cos(math.pi * k / t_max)) / 2.0


class PoseTracker:
    """Frozen Gaussians (raw parameter tensors, the layout of GaussianModel / JointTrainer) + scratch buffers.
    kernel_size / filter_3D: Mip-Splatting's 2D Mip filter and (frozen) 3D smoothing filter, DESIGN.md section 4.7."""

    def __init__(self, xyz, rotation, scaling, opacity, f_dc, f_rest, width, height, fovx, fovy, bg=None,
                 sh_degree: int = 3, device=None, kernel_size=None, filter_3D=None):
        self.dev = torch.device(device) if device is not None else xyz.device
        f = lambda t: t.detach().to(self.dev).float().contiguous()
        self.xyz, self.rotation, self.scaling = f(xyz), f(rotation), f(scaling)
        self.opacity, self.f_dc, self.f_rest = f(opacity).reshape(-1), f(f_dc).reshape(-1, 3), f(f_rest)
        self.P = self.xyz.shape[0]
        self.W, self.H = int(width), int(height)
        self.sh_degree = int(sh_degree)
        self.ident = IdentityView(self.W, self.H, fovx, fovy, torch.zeros(3) if bg is None else bg, self.dev)
        self.frame = Frame(self.dev, self.P, self.W, self.H, views=1)   # scratch of the last call's view count
        self.host_status = torch.zeros(ST_WORDS, dtype=torch.int32).pin_memory()
        self.headroom = 1.6            # the pose moves during tracking, and with it the instance count
        self.R_seen = 0
        self.filter_3D = None if filter_3D is None else f(filter_3D).reshape(-1)
        self.filt = mip_filter(kernel_size, self.filter_3D)

    @classmethod
    def from_model(cls, pc, camera, bg=None, device=None, kernel_size=None):
        """pc: a GaussianModel-like object (reference attribute names), camera: FoVx/FoVy/image_width/image_height."""
        return cls(pc._xyz, pc._rotation, pc._scaling, pc._opacity, pc._features_dc, pc._features_rest,
                   camera.image_width, camera.image_height, camera.FoVx, camera.FoVy, bg=bg,
                   sh_degree=pc.active_sh_degree, device=device, kernel_size=kernel_size,
                   filter_3D=getattr(pc, "filter_3D", None))

    # ------------------------------------------------------------------------------------------
    def _cam(self) -> GsbCamera:
        return self.ident.camera(self.sh_degree, 1 + self.f_rest.shape[1])

    def _gauss(self, pose: torch.Tensor) -> GsbGaussians:
        return gaussians(self.P, self.xyz, self.rotation, self.scaling, self.opacity, self.f_dc,
                         self.f_rest if self.f_rest.numel() else None, pose)

    def render(self, pose: torch.Tensor) -> torch.Tensor:
        """[3, H, W] at pose [7] (render_batch of one view)."""
        return self.render_batch(pose.reshape(1, 7))[0]

    def optimize(self, init_pose: torch.Tensor, gt: torch.Tensor, num_iter: int = 500, lr_T: float = 0.003,
                 lr_q: float = 0.001, weight_decay: float = 1e-4, eta_min: float = 1e-4,
                 threshold: float = 0.0, return_trace: bool = False):
        """render.py:113-161 for one view.  Returns (best_pose [7], best_loss) -- and the per-iteration losses if
        return_trace.  Raises if the instance count outgrew the binning buffer during the run.  This is the batched
        loop at V = 1 (same kernels, measured no slower than a separate single-view loop, DESIGN.md section 4.6)."""
        with torch.cuda.device(self.dev):
            pose = init_pose.detach().to(self.dev).float().reshape(1, 7).clone()
            gt = gt.detach().to(self.dev).float().reshape(1, 3, self.H, self.W).contiguous()
            out, trace = self._optimize_views(pose, gt, num_iter, lr_T, lr_q, weight_decay, eta_min, threshold,
                                              return_trace)
        if return_trace:
            return out[0, 1:].clone(), float(out[0, 0]), trace[0].clone()
        return out[0, 1:].clone(), float(out[0, 0])

    # ---- a batch of views ------------------------------------------------------------------------------------
    def _frame_batch(self, V: int) -> Frame:
        """The tracker's one scratch frame, reallocated for V views when the last call had another view count (the
        old buffers are released first, so scratch for one view count is held at a time)."""
        if self.frame.views != V:
            self.frame = None
            self.frame = Frame(self.dev, self.P, self.W, self.H, views=V)
        return self.frame

    def _poses(self, poses: torch.Tensor, what: str) -> torch.Tensor:
        if not isinstance(poses, torch.Tensor) or poses.dim() != 2 or poses.shape[1] != 7:
            raise ValueError(f"{what}: expected a [V, 7] pose tensor, got {tuple(getattr(poses, 'shape', ()))}")
        self._same_device(poses, what)
        return poses.detach().to(self.dev).float().contiguous()

    def _same_device(self, t: torch.Tensor, what: str) -> None:
        """Inputs may come from the host or from the tracker's own device, not from another device."""
        dev = self.dev if self.dev.index is not None else torch.device(self.dev.type, torch.cuda.current_device())
        if t.device.type != "cpu" and t.device != dev:
            raise ValueError(f"{what}: tensor on {t.device}, the tracker is on {dev}")

    def _forward_batch(self, fr: Frame, cam, g, poses, first: bool):
        fr.preprocess_batch(cam, g, poses, self.host_status if first else None, self.filt)
        if first:                      # size the binning buffer once, from the total count of all views
            torch.cuda.current_stream().synchronize()
            self.R_seen = R = read_R(self.host_status)
            if capacity(R, self.headroom) > fr.cap:
                fr.alloc_binning(capacity(R, self.headroom))
        fr.render_batch(cam)

    def render_batch(self, poses: torch.Tensor) -> torch.Tensor:
        """render() at each row of poses [V, 7] in one batched forward: [V, 3, H, W], view v bit-identical to
        render(poses[v])."""
        p = self._poses(poses, "render_batch")
        V = p.shape[0]
        if V == 0:
            return torch.empty(0, 3, self.H, self.W, device=self.dev)
        with torch.cuda.device(self.dev):
            fr = self._frame_batch(V)
            self._forward_batch(fr, self._cam(), self._gauss(p), p, True)
            return fr.color.clone()

    def optimize_batch(self, init_poses: torch.Tensor, gts: torch.Tensor, num_iter: int = 500, lr_T: float = 0.003,
                       lr_q: float = 0.001, weight_decay: float = 1e-4, eta_min: float = 1e-4, threshold: float = 0.0,
                       max_batch: Optional[int] = None, return_trace: bool = False):
        """render.py:99-170 for V test views at once: init_poses [V, 7], gts [V, 3, H, W].  Returns
        (best_poses [V, 7], best_losses [V]) -- and the per-iteration losses [V, num_iter] if return_trace -- where
        row v is bit-identical to optimize(init_poses[v], gts[v], ...).  Same schedule and candidate rule as optimize.

        max_batch: views per batched loop (None: all V at once).  The scratch of a loop over B views is about
        B * (150 * P + 44 * H * W + 28 * T) bytes (T = 16x16 tiles of a frame; per (view, Gaussian) the 145-byte
        record set, radii and pose partials; per pixel image buffers, colour, dL/dimage and the on-device copy of gts,
        which is skipped when gts already is a contiguous fp32 tensor on the device; per tile ranges and the per-tile
        arrays once B * T exceeds 65536), plus the binning buffer: 12 bytes per slot, headroom x the first forward's
        instance count of all B views + 65536 slots.  One set of scratch is held at a time; a last chunk of another
        size replaces it.  Raises GsbError if a loop's instance count outgrew its binning buffer."""
        init = self._poses(init_poses, "optimize_batch")
        V = init.shape[0]
        if not isinstance(gts, torch.Tensor) or tuple(gts.shape) != (V, 3, self.H, self.W):
            raise ValueError(f"optimize_batch: expected gts of shape {(V, 3, self.H, self.W)}, got "
                             f"{tuple(getattr(gts, 'shape', ()))}")
        self._same_device(gts, "optimize_batch")
        if max_batch is not None and int(max_batch) < 1:
            raise ValueError("optimize_batch: max_batch must be >= 1")
        gts = gts.detach().to(self.dev).float().contiguous()
        n = max(1, num_iter)
        best = torch.zeros(V, 8)
        trace = torch.zeros(V, n) if return_trace else None
        step = max(1, V) if max_batch is None else int(max_batch)
        for v0 in range(0, V, step):
            v1 = min(V, v0 + step)
            b, t = self._optimize_views(init[v0:v1].clone(), gts[v0:v1], num_iter, lr_T, lr_q, weight_decay, eta_min,
                                        threshold, return_trace)
            best[v0:v1] = b
            if return_trace:
                trace[v0:v1] = t
        if return_trace:
            return best[:, 1:].clone(), best[:, 0].clone(), trace
        return best[:, 1:].clone(), best[:, 0].clone()

    def evaluate_batch(self, poses: torch.Tensor, gts: torch.Tensor, mode: str = "png8",
                       max_batch: Optional[int] = None):
        """render.py -> metrics.py for V views: render each row of poses [V, 7] (render_batch) and measure it against
        gts [V, 3, H, W] (evaluation.image_metrics; mode "png8" is the 8-bit round trip of save_image and readImages).
        Same input checks as optimize_batch; max_batch: views per batched forward (None: all at once).  Returns
        image_metrics' dict (fp64 device tensors); view v's values are those of evaluate_batch on it alone."""
        from .evaluation import _mode, metric_sums, metrics_from_sums
        m = _mode(mode)
        p = self._poses(poses, "evaluate_batch")
        V = p.shape[0]
        if not isinstance(gts, torch.Tensor) or tuple(gts.shape) != (V, 3, self.H, self.W):
            raise ValueError(f"evaluate_batch: expected gts of shape {(V, 3, self.H, self.W)}, got "
                             f"{tuple(getattr(gts, 'shape', ()))}")
        self._same_device(gts, "evaluate_batch")
        if max_batch is not None and int(max_batch) < 1:
            raise ValueError("evaluate_batch: max_batch must be >= 1")
        if V == 0:
            raise ValueError("evaluate_batch: no views")
        step = V if max_batch is None else int(max_batch)
        with torch.cuda.device(self.dev):
            gts = gts.detach().to(self.dev).float().contiguous()
            cam = self._cam()
            sums, ovf = [], torch.zeros(1, dtype=torch.int32, device=self.dev)
            for v0 in range(0, V, step):
                v1 = min(V, v0 + step)
                fr = self._frame_batch(v1 - v0)
                self._forward_batch(fr, cam, self._gauss(p[v0:v1]), p[v0:v1], True)
                ovf |= fr.word(ST_OVERFLOW)
                sums.append(metric_sums(fr.color, gts[v0:v1], list(range(v1 - v0)), m))
            if int(ovf.item()):
                raise _lib.GsbError("evaluate_batch: a tile list outgrew the binning buffer")
            return metrics_from_sums(torch.cat(sums), self.H, self.W)

    def _optimize_views(self, poses, gts, num_iter, lr_T, lr_q, weight_decay, eta_min, threshold, return_trace):
        """One batched loop over poses.shape[0] views: (best [V, 8] on the host, trace [V, num_iter] or None)."""
        L = _lib.lib()
        V, dev = poses.shape[0], self.dev
        with torch.cuda.device(dev):
            st = _lib.stream_ptr()
            fr = self._frame_batch(V)
            dL = torch.empty_like(fr.color)
            m, v = torch.zeros(V, 7, device=dev), torch.zeros(V, 7, device=dev)
            dpose = torch.zeros(V, 7, device=dev)
            best = torch.zeros(V, 8, device=dev)
            best[:, 0] = 1e20
            best[:, 1:] = poses
            n = max(1, num_iter)
            sums = torch.zeros(n, V, 2, dtype=torch.float64, device=dev)
            trace = torch.zeros(V, n, device=dev) if return_trace else None
            cam, g = self._cam(), self._gauss(poses)
            ovf = torch.zeros(1, dtype=torch.int32, device=dev)
            ovf_word = fr.word(ST_OVERFLOW)
            for k in range(num_iter):
                self._forward_batch(fr, cam, g, poses, k == 0)
                ovf |= ovf_word                            # sticky overflow flag, checked once at the end
                check(L.gsb_l1_mask_fwd_bwd_batch(V, 3, self.H, self.W, fr.color.data_ptr(), gts.data_ptr(),
                                                  float(threshold), sums[k].data_ptr(), dL.data_ptr(), st),
                      "gsb_l1_mask_fwd_bwd_batch")
                fr.backward_pose_batch(cam, g, poses, dL, dpose, self.filt)
                check(L.gsb_track_step_batch(V, poses.data_ptr(), dpose.data_ptr(), sums[k].data_ptr(), m.data_ptr(),
                                             v.data_ptr(), best.data_ptr(),
                                             trace[:, k:].data_ptr() if return_trace else None, n, k + 1,
                                             cosine_lr(lr_q, k, num_iter, eta_min), cosine_lr(lr_T, k, num_iter, eta_min),
                                             0.9, 0.999, 1e-8, float(weight_decay), st), "gsb_track_step_batch")
            out = best.cpu()
            if int(ovf.item()):
                raise _lib.GsbError("tracking: the instance count outgrew the binning buffer; raise PoseTracker.headroom")
            return out, trace.cpu() if return_trace else None
