"""Host side of one forward of libgsb200.so: the status-word format, the scratch buffers of a (device, P, W, H), the
binning-capacity rule and the camera / Gaussians descriptors.

The library protocol is gsb_preprocess -> (the caller may wait for the instance count R) -> size the binning buffer
-> gsb_render -> gsb_backward.  When to wait, how much headroom to give and when to grow the buffer is the caller's
policy (rasterizer.py, trainer.py, tracking.py); this module only owns the mechanism and the formats.
"""
from __future__ import annotations

import ctypes
import math

import torch

from . import _lib
from ._lib import FILTER_MIP2D, GsbCamera, GsbDensifyStats, GsbFilter, GsbGaussians, check

# the status words of a forward (kSt* of csrc/gs_internal.cuh); the library writes them as uint32
ST_R, ST_OVERFLOW, ST_MAX_LIST, ST_HUGE_TILES, ST_NLARGE, ST_NHUGE, ST_SEQ = range(7)
ST_WORDS = 8


def u32(word) -> int:
    """A status word (int32 in a torch tensor) as the unsigned value the device wrote."""
    return int(word) & 0xFFFFFFFF


def read_R(words) -> int:
    """Instance count R from a host or device copy of the status words."""
    return u32(words[ST_R])


def capacity(R: int, headroom: float) -> int:
    """Binning capacity (instances) for an expected count R: the headroom is the caller's, the floor keeps tiny
    frames from overflowing on small changes."""
    return int(R * headroom) + 65536


def _p(t):
    return None if t is None else t.data_ptr()


def camera(W, H, tanfovx, tanfovy, sh_degree, sh_coeffs, bg, viewmatrix, projmatrix, campos, scale_modifier=1.0,
           exact_cull=True) -> GsbCamera:
    """GsbCamera over contiguous fp32 device tensors; exact_cull: lossless alpha < 1/255 tile culling."""
    cam = GsbCamera()
    cam.width, cam.height = int(W), int(H)
    cam.tanfovx, cam.tanfovy, cam.scale_modifier = float(tanfovx), float(tanfovy), float(scale_modifier)
    cam.sh_degree, cam.sh_coeffs, cam.exact_cull = int(sh_degree), int(sh_coeffs), 1 if exact_cull else 0
    cam.bg, cam.viewmatrix, cam.projmatrix, cam.campos = _p(bg), _p(viewmatrix), _p(projmatrix), _p(campos)
    return cam


class IdentityView:
    """InstantSplat's camera (gaussian_renderer/__init__.py:55-59): identity view matrix, camera at the origin and
    the projection of (fovx, fovy); the camera pose moves the Gaussians instead.  Holds the tensors GsbCamera points to."""

    def __init__(self, W, H, fovx, fovy, bg, device):
        from .camera import projection_matrix
        self.W, self.H = int(W), int(H)
        self.tanfovx, self.tanfovy = math.tan(fovx * 0.5), math.tan(fovy * 0.5)
        self.viewmatrix = torch.eye(4, device=device)
        self.projmatrix = projection_matrix(0.01, 100.0, fovx, fovy).t().contiguous().to(device)
        self.campos = torch.zeros(3, device=device)
        self.bg = bg.to(device).float().contiguous()

    def camera(self, sh_degree, sh_coeffs, exact_cull=True) -> GsbCamera:
        return camera(self.W, self.H, self.tanfovx, self.tanfovy, sh_degree, sh_coeffs, self.bg, self.viewmatrix,
                      self.projmatrix, self.campos, exact_cull=exact_cull)


def gaussians(P, xyz, rotation, scaling, opacity, f_dc, f_rest, pose, raw_params=1, sh_packed=0, colors_precomp=None,
              cov3D_precomp=None) -> GsbGaussians:
    """GsbGaussians over contiguous fp32 device tensors (None: not given).  raw_params=1: the model's raw parameters
    (log scales, unnormalised quaternions, logit opacities) moved by `pose`; raw_params=0: activated values as the
    upstream rasterizer takes them, sh_packed=1 when all SH coefficients are in f_dc as [P, M, 3]."""
    g = GsbGaussians()
    g.P, g.sh_packed, g.raw_params = P, int(sh_packed), int(raw_params)
    g.means3D, g.rotations, g.scales, g.opacities = _p(xyz), _p(rotation), _p(scaling), _p(opacity)
    g.sh_dc, g.sh_rest, g.pose = _p(f_dc), _p(f_rest), _p(pose)
    g.colors_precomp, g.cov3D_precomp = _p(colors_precomp), _p(cov3D_precomp)
    return g


def mip_filter(kernel_size=None, filter3D=None):
    """GsbFilter of the Mip-Splatting filters (DESIGN.md section 4.7), or None (the reference path) when both are off.
    kernel_size: the 2D Mip filter's dilation (Mip-Splatting uses 0.1); filter3D: contiguous fp32 [P] device tensor of
    3D smoothing filter sizes (raw parameters only).  The tensor must stay alive while the filter is in use."""
    if kernel_size is None and filter3D is None:
        return None
    f = GsbFilter()
    if kernel_size is not None:
        f.kernel_size, f.flags = float(kernel_size), FILTER_MIP2D
    f.filter3D = _p(filter3D)
    return f


def mip_filter3d(xyz, poses7, W, H, tanfovx, tanfovy, out=None) -> torch.Tensor:
    """Size of the 3D smoothing filter [P] from world points xyz [P, 3] and the training views' pose table
    poses7 [V, 7] with one shared intrinsics (gsb_mip_filter3d); written into `out` when given."""
    xyz, poses7 = xyz.detach().float().contiguous(), poses7.detach().float().contiguous()
    if out is None:
        out = torch.empty(xyz.shape[0], dtype=torch.float32, device=xyz.device)
    check(_lib.lib().gsb_mip_filter3d(xyz.shape[0], xyz.data_ptr(), poses7.shape[0], poses7.data_ptr(), int(W), int(H),
                                      float(tanfovx), float(tanfovy), out.data_ptr(), _lib.stream_ptr()),
          "gsb_mip_filter3d")
    return out


def densify_stats(radii, grad_accum, denom, max_radii2D) -> GsbDensifyStats:
    """GsbDensifyStats over contiguous device tensors of P elements: radii int32 (the forward's), the other three fp32,
    updated in place by the backward (train.py:197-199).  The tensors must stay alive while the struct is in use."""
    s = GsbDensifyStats()
    s.radii, s.grad_accum, s.denom, s.max_radii2D = _p(radii), _p(grad_accum), _p(denom), _p(max_radii2D)
    return s


def _f(filt):
    return None if filt is None else ctypes.byref(filt)


def _bg_table(bg, views) -> None:
    """Refuse a per-view background table that is not a contiguous fp32 [views, 3] CUDA tensor."""
    if not (isinstance(bg, torch.Tensor) and bg.is_cuda and bg.dtype == torch.float32 and bg.is_contiguous() and
            tuple(bg.shape) == (views, 3)):
        raise _lib.GsbError(f"background table: expected a contiguous float32 [{views}, 3] CUDA tensor, got "
                            f"{getattr(bg, 'dtype', type(bg))} {tuple(getattr(bg, 'shape', ()))}")


class Frame:
    """Scratch of forwards at one (device, P, W, H): the geometry buffer (which holds the status words), radii, the
    image buffer, the rendered colour [3, H, W], and a binning buffer of `cap` instances (0: none yet).

    views: scratch of a batch of that many views of the same Gaussians and intrinsics (the *_batch methods,
    gsb_preprocess_batch and friends); radii is then [views, P] and color [views, 3, H, W].  None: one view.

    host_status arguments are the caller's pinned 8-word slots (or None): the library copies the status words there
    after the phase."""

    def __init__(self, device, P, W, H, views=None):
        L = _lib.lib()
        self.P, self.W, self.H, self.views = P, W, H, 1 if views is None else int(views)
        if views is None:
            geom_bytes, image_bytes = L.gsb_geom_bytes(P), L.gsb_image_bytes(W, H)
            self.radii = torch.empty(P, dtype=torch.int32, device=device)
            self.color = torch.empty(3, H, W, dtype=torch.float32, device=device)
        else:
            geom_bytes, image_bytes = L.gsb_geom_bytes_batch(P, views, W, H), L.gsb_image_bytes_batch(W, H, views)
            self.radii = torch.empty(views, P, dtype=torch.int32, device=device)
            self.color = torch.empty(views, 3, H, W, dtype=torch.float32, device=device)
        self.geom = torch.empty(geom_bytes, dtype=torch.uint8, device=device)
        self.image = torch.empty(image_bytes, dtype=torch.uint8, device=device)
        self._so = L.gsb_status_device_batch(self.geom.data_ptr(), P, self.views) - self.geom.data_ptr()
        self.binning, self.cap = None, 0

    @property
    def status(self) -> torch.Tensor:
        """Device view of the status words (int32)."""
        return self.geom[self._so:self._so + 4 * ST_WORDS].view(torch.int32)

    def word(self, i: int) -> torch.Tensor:
        """Device view of status word i (one int32); its data_ptr() is the word's device address."""
        return self.geom[self._so + 4 * i:self._so + 4 * i + 4].view(torch.int32)

    def alloc_binning(self, cap: int, round_to: int = 1) -> None:
        """A new binning buffer of `cap` instances, its byte size rounded up to a multiple of round_to."""
        nbytes = (_lib.lib().gsb_binning_bytes_batch(cap, self.W, self.H, self.views) + round_to - 1) // round_to * round_to
        self.binning = torch.empty(nbytes, dtype=torch.uint8, device=self.geom.device)
        self.cap = cap

    def preprocess(self, cam, g, host_status=None, filt=None) -> None:
        """filt: mip_filter(...) or None; pass the same one to the backward."""
        check(_lib.lib().gsb_preprocess_ex(ctypes.byref(cam), ctypes.byref(g), _f(filt), self.geom.data_ptr(),
                                           self.geom.numel(), self.radii.data_ptr(), _p(host_status),
                                           _lib.stream_ptr()), "gsb_preprocess")

    def render(self, cam, host_status=None) -> None:
        check(_lib.lib().gsb_render(ctypes.byref(cam), self.P, self.geom.data_ptr(), self.binning.data_ptr(),
                                    self.binning.numel(), self.cap, self.image.data_ptr(), self.color.data_ptr(),
                                    _p(host_status), _lib.stream_ptr()), "gsb_render")

    def backward(self, cam, g, dL_dimage, grads, filt=None, stats=None) -> None:
        """stats: densify_stats(...) over this frame's radii, or None; accumulated by the same launch."""
        if stats is None:
            check(_lib.lib().gsb_backward_ex(ctypes.byref(cam), ctypes.byref(g), _f(filt), self.geom.data_ptr(),
                                             self.binning.data_ptr(), self.cap, self.image.data_ptr(),
                                             dL_dimage.data_ptr(), ctypes.byref(grads), _lib.stream_ptr()), "gsb_backward")
        else:
            check(_lib.lib().gsb_backward_stats(ctypes.byref(cam), ctypes.byref(g), _f(filt), ctypes.byref(stats),
                                                self.geom.data_ptr(), self.binning.data_ptr(), self.cap,
                                                self.image.data_ptr(), dL_dimage.data_ptr(), ctypes.byref(grads),
                                                _lib.stream_ptr()), "gsb_backward_stats")

    def blend_stats(self, cam, dL_dimage, stats) -> None:
        check(_lib.lib().gsb_blend_stats(ctypes.byref(cam), self.P, self.geom.data_ptr(), self.binning.data_ptr(),
                                         self.cap, self.image.data_ptr(), self.color.data_ptr(), dL_dimage.data_ptr(),
                                         stats.data_ptr(), _lib.stream_ptr()), "gsb_blend_stats")

    # ---- a batch of views (views > 1; gsb200.h "batched tracking") ----------------------------------------------
    def preprocess_batch(self, cam, g, poses7, host_status=None, filt=None) -> None:
        """poses7: contiguous fp32 [views, 7] device tensor; g holds raw parameters (its pose is not used)."""
        check(_lib.lib().gsb_preprocess_batch(ctypes.byref(cam), ctypes.byref(g), _f(filt), self.views,
                                              poses7.data_ptr(), self.geom.data_ptr(), self.geom.numel(),
                                              self.radii.data_ptr(), _p(host_status), _lib.stream_ptr()),
              "gsb_preprocess_batch")

    def render_batch(self, cam, host_status=None, bg=None) -> None:
        """bg: contiguous fp32 [views, 3] device tensor, view v blended over row v (gsb_render_batch_bg); None: cam's
        background for every view."""
        if bg is None:
            check(_lib.lib().gsb_render_batch(ctypes.byref(cam), self.P, self.views, self.geom.data_ptr(),
                                              self.binning.data_ptr(), self.binning.numel(), self.cap,
                                              self.image.data_ptr(), self.color.data_ptr(), _p(host_status),
                                              _lib.stream_ptr()), "gsb_render_batch")
            return
        _bg_table(bg, self.views)
        check(_lib.lib().gsb_render_batch_bg(ctypes.byref(cam), self.P, self.views, bg.data_ptr(), self.geom.data_ptr(),
                                             self.binning.data_ptr(), self.binning.numel(), self.cap,
                                             self.image.data_ptr(), self.color.data_ptr(), _p(host_status),
                                             _lib.stream_ptr()), "gsb_render_batch_bg")

    def backward_pose_batch(self, cam, g, poses7, dL_dimage, dpose7, filt=None) -> None:
        """dL_dimage [views, 3, H, W] -> dpose7 [views, 7] (pose gradients only)."""
        check(_lib.lib().gsb_backward_pose_batch(ctypes.byref(cam), ctypes.byref(g), _f(filt), self.views,
                                                 poses7.data_ptr(), self.geom.data_ptr(), self.binning.data_ptr(),
                                                 self.cap, self.image.data_ptr(), dL_dimage.data_ptr(),
                                                 dpose7.data_ptr(), _lib.stream_ptr()), "gsb_backward_pose_batch")

    def backward_batch(self, cam, g, poses7, dL_dimage, grads, dpose7, filt=None, stats=None, n_stats=0,
                       bg=None) -> None:
        """dL_dimage [views, 3, H, W] -> every per-Gaussian gradient of `grads` summed over the views in view order
        (bit-identical to single-view backwards added in that order), and dpose7 [views, 7].  stats: densify_stats(...)
        over this frame's [views, P] radii, or None; the same launch accumulates the statistics of views 0..n_stats-1,
        bit-identical to single-view backwards with statistics made in view order.  bg: the [views, 3] table the
        forward was rendered over (render_batch), or None."""
        if bg is not None:
            _bg_table(bg, self.views)
            check(_lib.lib().gsb_backward_batch_stats_bg(
                ctypes.byref(cam), ctypes.byref(g), _f(filt), self.views, bg.data_ptr(), int(n_stats),
                None if stats is None else ctypes.byref(stats), poses7.data_ptr(), self.geom.data_ptr(),
                self.binning.data_ptr(), self.cap, self.image.data_ptr(), dL_dimage.data_ptr(), ctypes.byref(grads),
                dpose7.data_ptr(), _lib.stream_ptr()), "gsb_backward_batch_stats_bg")
            return
        check(_lib.lib().gsb_backward_batch_stats(ctypes.byref(cam), ctypes.byref(g), _f(filt), self.views, int(n_stats),
                                                  None if stats is None else ctypes.byref(stats), poses7.data_ptr(),
                                                  self.geom.data_ptr(), self.binning.data_ptr(), self.cap,
                                                  self.image.data_ptr(), dL_dimage.data_ptr(), ctypes.byref(grads),
                                                  dpose7.data_ptr(), _lib.stream_ptr()), "gsb_backward_batch_stats")
