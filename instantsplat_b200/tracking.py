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
"""
from __future__ import annotations

import ctypes
import math
from typing import Optional

import torch

from . import _lib
from ._lib import GsbCamera, GsbGaussians, GsbGrads, check


def cosine_lr(base_lr: float, k: int, t_max: int, eta_min: float = 1e-4) -> float:
    """Closed form of torch.optim.lr_scheduler.CosineAnnealingLR after k scheduler steps."""
    return eta_min + (base_lr - eta_min) * (1.0 + math.cos(math.pi * k / t_max)) / 2.0


class PoseTracker:
    """Frozen Gaussians (raw parameter tensors, the layout of GaussianModel / JointTrainer) + scratch buffers."""

    def __init__(self, xyz, rotation, scaling, opacity, f_dc, f_rest, width, height, fovx, fovy, bg=None,
                 sh_degree: int = 3, device=None):
        self.dev = torch.device(device) if device is not None else xyz.device
        f = lambda t: t.detach().to(self.dev).float().contiguous()
        self.xyz, self.rotation, self.scaling = f(xyz), f(rotation), f(scaling)
        self.opacity, self.f_dc, self.f_rest = f(opacity).reshape(-1), f(f_dc).reshape(-1, 3), f(f_rest)
        self.P = self.xyz.shape[0]
        self.W, self.H = int(width), int(height)
        self.sh_degree = int(sh_degree)
        from .camera import projection_matrix
        self.tanfovx, self.tanfovy = math.tan(fovx * 0.5), math.tan(fovy * 0.5)
        self.viewmatrix = torch.eye(4, device=self.dev)
        self.projmatrix = projection_matrix(0.01, 100.0, fovx, fovy).t().contiguous().to(self.dev)
        self.campos = torch.zeros(3, device=self.dev)
        self.bg = (torch.zeros(3) if bg is None else bg).to(self.dev).float().contiguous()
        L = _lib.lib()
        self.geom_bytes = L.gsb_geom_bytes(self.P)
        self.geom = torch.empty(self.geom_bytes, dtype=torch.uint8, device=self.dev)
        self.image_buf = torch.empty(L.gsb_image_bytes(self.W, self.H), dtype=torch.uint8, device=self.dev)
        self.radii = torch.empty(self.P, dtype=torch.int32, device=self.dev)
        self.color = torch.empty(3, self.H, self.W, dtype=torch.float32, device=self.dev)
        self.dL = torch.empty_like(self.color)
        self.host_status = torch.zeros(8, dtype=torch.int32).pin_memory()
        self.cap, self.binning, self.bin_bytes = 0, None, 0
        self.headroom = 1.6            # the pose moves during tracking, and with it the instance count
        self.R_seen = 0

    @classmethod
    def from_model(cls, pc, camera, bg=None, device=None):
        """pc: a GaussianModel-like object (reference attribute names), camera: FoVx/FoVy/image_width/image_height."""
        return cls(pc._xyz, pc._rotation, pc._scaling, pc._opacity, pc._features_dc, pc._features_rest,
                   camera.image_width, camera.image_height, camera.FoVx, camera.FoVy, bg=bg,
                   sh_degree=pc.active_sh_degree, device=device)

    # ------------------------------------------------------------------------------------------
    def _cam(self) -> GsbCamera:
        cam = GsbCamera()
        cam.width, cam.height = self.W, self.H
        cam.tanfovx, cam.tanfovy, cam.scale_modifier = self.tanfovx, self.tanfovy, 1.0
        cam.sh_degree, cam.sh_coeffs, cam.exact_cull = self.sh_degree, 1 + self.f_rest.shape[1], 1
        cam.bg, cam.viewmatrix = self.bg.data_ptr(), self.viewmatrix.data_ptr()
        cam.projmatrix, cam.campos = self.projmatrix.data_ptr(), self.campos.data_ptr()
        return cam

    def _gauss(self, pose: torch.Tensor) -> GsbGaussians:
        g = GsbGaussians()
        g.P, g.sh_packed, g.raw_params = self.P, 0, 1
        g.means3D, g.scales, g.rotations = self.xyz.data_ptr(), self.scaling.data_ptr(), self.rotation.data_ptr()
        g.opacities, g.sh_dc = self.opacity.data_ptr(), self.f_dc.data_ptr()
        g.sh_rest = self.f_rest.data_ptr() if self.f_rest.numel() else None
        g.pose = pose.data_ptr()
        return g

    def _forward(self, cam, g, first: bool):
        L = _lib.lib()
        st = _lib.stream_ptr()
        check(L.gsb_preprocess(ctypes.byref(cam), ctypes.byref(g), self.geom.data_ptr(), self.geom_bytes,
                               self.radii.data_ptr(), self.host_status.data_ptr() if first else None, st), "gsb_preprocess")
        if first:                      # size the binning buffer once, from the real count at the initial pose
            torch.cuda.current_stream().synchronize()
            R = int(self.host_status[0]) & 0xFFFFFFFF
            self.R_seen = R
            if R * self.headroom + 65536 > self.cap:
                self.cap = int(R * self.headroom) + 65536
                self.bin_bytes = L.gsb_binning_bytes(self.cap, self.W, self.H)
                self.binning = torch.empty(self.bin_bytes, dtype=torch.uint8, device=self.dev)
        check(L.gsb_render(ctypes.byref(cam), self.P, self.geom.data_ptr(), self.binning.data_ptr(), self.bin_bytes,
                           self.cap, self.image_buf.data_ptr(), self.color.data_ptr(), None, st), "gsb_render")

    def render(self, pose: torch.Tensor) -> torch.Tensor:
        with torch.cuda.device(self.dev):
            p = pose.detach().to(self.dev).float().contiguous()
            self._forward(self._cam(), self._gauss(p), True)
            return self.color.clone()

    def optimize(self, init_pose: torch.Tensor, gt: torch.Tensor, num_iter: int = 500, lr_T: float = 0.003,
                 lr_q: float = 0.001, weight_decay: float = 1e-4, eta_min: float = 1e-4,
                 threshold: float = 0.0, return_trace: bool = False):
        """render.py:113-161 for one view.  Returns (best_pose [7], best_loss) -- and the per-iteration losses if
        return_trace.  Raises if the instance count outgrew the binning buffer during the run."""
        L = _lib.lib()
        with torch.cuda.device(self.dev):
            st = _lib.stream_ptr()
            pose = init_pose.detach().to(self.dev).float().contiguous().clone()
            gt = gt.detach().to(self.dev).float().contiguous()
            m, v = torch.zeros(7, device=self.dev), torch.zeros(7, device=self.dev)
            dpose = torch.zeros(7, device=self.dev)
            best = torch.zeros(8, device=self.dev)
            best[0] = 1e20
            best[1:] = pose
            sums = torch.zeros(max(1, num_iter), 2, dtype=torch.float64, device=self.dev)
            trace = torch.zeros(max(1, num_iter), device=self.dev) if return_trace else None
            cam, g = self._cam(), self._gauss(pose)
            gr = GsbGrads()
            gr.dL_dpose = dpose.data_ptr()
            status_dev = L.gsb_status_device(self.geom.data_ptr(), self.P)
            ovf = torch.zeros(1, dtype=torch.int32, device=self.dev)
            so = status_dev - self.geom.data_ptr()
            status_t = self.geom[so:so + 32].view(torch.int32)
            for k in range(num_iter):
                self._forward(cam, g, k == 0)
                ovf |= status_t[1:2]                       # sticky overflow flag, checked once at the end
                check(L.gsb_l1_mask_fwd_bwd(3, self.H, self.W, self.color.data_ptr(), gt.data_ptr(), float(threshold),
                                            sums[k].data_ptr(), self.dL.data_ptr(), st), "gsb_l1_mask_fwd_bwd")
                check(L.gsb_backward(ctypes.byref(cam), ctypes.byref(g), self.geom.data_ptr(), self.binning.data_ptr(),
                                     self.cap, self.image_buf.data_ptr(), self.dL.data_ptr(), ctypes.byref(gr), st),
                      "gsb_backward")
                check(L.gsb_track_step(pose.data_ptr(), dpose.data_ptr(), sums[k].data_ptr(), m.data_ptr(), v.data_ptr(),
                                       best.data_ptr(), trace[k:].data_ptr() if return_trace else None, k + 1,
                                       cosine_lr(lr_q, k, num_iter, eta_min), cosine_lr(lr_T, k, num_iter, eta_min),
                                       0.9, 0.999, 1e-8, float(weight_decay), st), "gsb_track_step")
            out = best.cpu()
            if int(ovf.item()):
                raise _lib.GsbError("tracking: the instance count outgrew the binning buffer; raise PoseTracker.headroom")
            if return_trace:
                return out[1:].clone(), float(out[0]), trace.cpu()
            return out[1:].clone(), float(out[0])
