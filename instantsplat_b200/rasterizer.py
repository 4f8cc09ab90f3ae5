"""Drop-in for the `diff_gaussian_rasterization` package (boundary B2 of SURVEY.md section 8b) on top
of libgsb200.so, plus the fused InstantSplat entry (`rasterize_fused`) used by `render()`.

Mirrors the interface the reference calls at gaussian_renderer/__init__.py:14-17,
60-78,126-135 (and the vanilla-3DGS form at gaussian_renderer/__init__3dgs.py:36-51,85-93):
same names, argument meaning and error behaviour.
"""
from __future__ import annotations

import ctypes
import warnings
import weakref
from typing import NamedTuple, Optional

import torch
import torch.nn as nn

from . import _lib
from ._lib import GsbCamera, GsbGaussians, GsbGrads, check, f32c, ptr

_vp = ctypes.c_void_p


class GaussianRasterizationSettings(NamedTuple):
    image_height: int
    image_width: int
    tanfovx: float
    tanfovy: float
    bg: torch.Tensor
    scale_modifier: float
    viewmatrix: torch.Tensor
    projmatrix: torch.Tensor
    sh_degree: int
    campos: torch.Tensor
    prefiltered: bool
    debug: bool


EXACT_CULL = True   # lossless alpha<1/255 tile culling (set False for the reference's rect-only binning)

# The instance count R (number of (Gaussian, tile) pairs) never has to reach the host BEFORE the render phase is
# launched: the kernels read it from device memory, the host only chooses the CAPACITY of the binning buffer.
# SYNC_FREE = True sizes it from the counts seen for the same (device, P, W, H) with 50 % headroom, enqueues binning
# and blend, and only then waits for the status words of the PREPROCESS phase (an event right behind the tile scan):
# while the host waits, the GPU has the whole render phase queued, so it never idles -- unlike the reference's
# blocking cudaMemcpy of num_rendered, which stalls the GPU until the host has sized its buffers and launched the
# rest.  If the capacity was exceeded (rare), the render phase is repeated with an exact buffer before the forward
# returns, so whatever the caller computes from the image is consistent.  LAZY_VERIFY = True postpones the check to
# the backward / the next forward instead (forward-only loops that never look at R); the very first call of a shape
# -- and every call when SYNC_FREE is False -- waits for R before launching the render phase and sizes it exactly.
SYNC_FREE = True
LAZY_VERIFY = False
HEADROOM = 1.5
_last_R = {}            # (device index, P, W, H) -> last verified instance count
_pending = {}           # same key -> _State whose capacity check has not been read yet


class _StatusRing:
    """Pinned 8-word status slots, recycled round-robin (a slot is long verified before it comes round again)."""

    def __init__(self, n=512):
        self.buf = torch.zeros(n, 8, dtype=torch.int32).pin_memory()
        self.n, self.i = n, 0

    def take(self) -> torch.Tensor:
        t = self.buf[self.i]
        self.i = (self.i + 1) % self.n
        return t


_ring = None


def _status_slot() -> torch.Tensor:
    global _ring
    if _ring is None:
        _ring = _StatusRing()
    return _ring.take()


class _State:
    """Everything the backward needs; keeps the torch buffers alive."""
    __slots__ = ("cam", "g", "geom", "binning", "image", "R", "keep", "P", "M", "packed", "has_pose",
                 "key", "status", "event", "checked", "color", "bin_bytes", "R_true", "__weakref__")


def _camera(settings: GaussianRasterizationSettings, sh_coeffs: int, keep: list) -> GsbCamera:
    bg, vm, pm, cp = (f32c(settings.bg), f32c(settings.viewmatrix), f32c(settings.projmatrix),
                      f32c(settings.campos))
    keep += [bg, vm, pm, cp]
    cam = GsbCamera()
    cam.width, cam.height = int(settings.image_width), int(settings.image_height)
    cam.tanfovx, cam.tanfovy = float(settings.tanfovx), float(settings.tanfovy)
    cam.scale_modifier = float(settings.scale_modifier)
    cam.sh_degree, cam.sh_coeffs = int(settings.sh_degree), int(sh_coeffs)
    cam.exact_cull = 1 if EXACT_CULL else 0
    cam.bg, cam.viewmatrix, cam.projmatrix, cam.campos = ptr(bg), ptr(vm), ptr(pm), ptr(cp)
    return cam


def _render_phase(st: _State, cap: int, dev):
    """Binning + blend into st.color with a binning buffer of `cap` instances (allocation rounded up to 32 MiB so
    the caching allocator can reuse the block of the previous call)."""
    L = _lib.lib()
    H, W = st.cam.height, st.cam.width
    bin_bytes = (L.gsb_binning_bytes(cap, W, H) + (1 << 25) - 1) >> 25 << 25
    st.binning = torch.empty(bin_bytes, dtype=torch.uint8, device=dev)
    st.bin_bytes, st.R = bin_bytes, cap
    check(L.gsb_render(ctypes.byref(st.cam), st.P, st.geom.data_ptr(), st.binning.data_ptr(), bin_bytes, cap,
                       st.image.data_ptr(), st.color.data_ptr(), None, _lib.stream_ptr()), "gsb_render")
    st.checked = False


def _note_R(key, R: int) -> None:
    """Capacity estimate = slowly decaying maximum of the counts seen (different views share a key)."""
    _last_R[key] = max(R, int(0.98 * _last_R.get(key, 0)))


def _verify(st: _State, dev) -> None:
    """Read the lazily copied status words of st's forward; if the binning buffer was too small, redo the render
    phase in place with an exactly sized one (image and scratch become exact before anybody differentiates)."""
    if st.checked:
        return
    st.event.synchronize()                 # recorded right behind the tile scan: early in the forward
    R_true = int(st.status[0]) & 0xFFFFFFFF
    overflow = R_true > st.R
    _note_R(st.key, R_true)
    st.checked, st.R_true = True, R_true
    _pending.pop(st.key, None)
    if overflow:
        warnings.warn(f"instantsplat_b200: instance count {R_true} exceeded the binning capacity {st.R}; "
                      "the render phase was repeated with an exact buffer", RuntimeWarning)
        with torch.cuda.device(dev):
            _render_phase(st, R_true, dev)
            st.checked = True


def _verify_pending(key, dev) -> None:
    """At the next forward of the same shape: settle the previous call's capacity check (its result has long
    arrived; the forward's state may already be gone if nobody differentiated it)."""
    rec = _pending.pop(key, None)
    if rec is None:
        return
    ref, status, event, cap = rec
    st = ref()
    if st is not None:
        _pending[key] = rec
        _verify(st, dev)
        return
    event.synchronize()
    _note_R(key, int(status[0]) & 0xFFFFFFFF)
    if (int(status[0]) & 0xFFFFFFFF) > cap:
        warnings.warn(f"instantsplat_b200: a forward-only call rendered with a truncated binning buffer "
                      f"({_last_R[key]} instances > capacity {cap}); the capacity has been raised", RuntimeWarning)


def _forward(settings, means3D, scales, rotations, opacities, sh_dc, sh_rest, sh_packed, M,
             colors_precomp, cov3D_precomp, pose, raw_params):
    L = _lib.lib()
    dev = means3D.device
    if means3D.dim() != 2 or means3D.shape[1] != 3:
        raise RuntimeError("means3D must have dimensions (num_points, 3)")
    P = means3D.shape[0]
    st = _State()
    st.keep = []
    st.cam = _camera(settings, M, st.keep)
    g = GsbGaussians()
    g.P, g.sh_packed, g.raw_params = P, int(sh_packed), int(raw_params)
    ts = dict(means3D=means3D, scales=scales, rotations=rotations, opacities=opacities, sh_dc=sh_dc,
              sh_rest=sh_rest, colors_precomp=colors_precomp, cov3D_precomp=cov3D_precomp, pose=pose)
    for k, v in ts.items():
        v = f32c(v)
        st.keep.append(v)
        setattr(g, k, ptr(v))
    st.g, st.P, st.M, st.packed, st.has_pose = g, P, M, bool(sh_packed), pose is not None
    H, W = st.cam.height, st.cam.width
    st.key = (dev.index, P, W, H)
    with torch.cuda.device(dev):
        _verify_pending(st.key, dev)   # long finished in practice: just reads the pinned words
        stream = _lib.stream_ptr()
        geom_bytes = L.gsb_geom_bytes(P)
        st.geom = torch.empty(geom_bytes, dtype=torch.uint8, device=dev)
        radii = torch.empty(P, dtype=torch.int32, device=dev)
        st.image = torch.empty(L.gsb_image_bytes(W, H), dtype=torch.uint8, device=dev)
        st.color = torch.empty(3, H, W, dtype=torch.float32, device=dev)
        est = _last_R.get(st.key) if (SYNC_FREE and not settings.debug) else None
        st.status = _status_slot()
        check(L.gsb_preprocess(ctypes.byref(st.cam), ctypes.byref(g), st.geom.data_ptr(), geom_bytes,
                               radii.data_ptr(), st.status.data_ptr(), stream), "gsb_preprocess")
        st.event = torch.cuda.Event()
        st.event.record()
        if est is None:
            st.event.synchronize()                         # exact sizing: wait for R once
            cap = int(st.status[0]) & 0xFFFFFFFF
        else:
            cap = int(est * HEADROOM) + 65536
        _render_phase(st, cap, dev)
        if est is None:
            _note_R(st.key, cap)
            st.checked, st.R_true = True, cap
        elif LAZY_VERIFY:
            _pending[st.key] = (weakref.ref(st), st.status, st.event, cap)
        else:
            _verify(st, dev)             # waits for the preprocess phase only; repeats the render phase on overflow
        if settings.debug:
            torch.cuda.synchronize()
    return st.color, radii, st


def _backward(st: _State, dL_dout, want, dev):
    """want: None (everything) or a set of names to compute; gradients that are not wanted are neither
    allocated nor written by the kernels (e.g. the pose-only test-view optimisation of
    render.py:99-170 passes {"pose"}).  Returns dict of dense grad tensors."""
    L = _lib.lib()
    P, M = st.P, st.M
    _verify(st, dev)
    dL = f32c(dL_dout)
    gr = GsbGrads()
    out = {}

    def alloc(name, shape, field):
        if want is not None and name not in want:
            return
        t = torch.empty(shape, dtype=torch.float32, device=dev)
        out[name] = t
        setattr(gr, field, t.data_ptr())

    alloc("means3D", (P, 3), "dL_dmeans3D")
    alloc("means2D", (P, 3), "dL_dmeans2D")
    alloc("opacities", (P,), "dL_dopacities")
    if st.g.scales:
        alloc("scales", (P, 3), "dL_dscales")
        alloc("rotations", (P, 4), "dL_drotations")
    if st.g.cov3D_precomp:
        alloc("cov3D", (P, 6), "dL_dcov3D")
    if st.g.colors_precomp:
        alloc("colors", (P, 3), "dL_dcolors")
    else:
        if st.packed:
            alloc("sh", (P, M, 3), "dL_dsh_dc")
        else:
            alloc("sh_dc", (P, 1, 3), "dL_dsh_dc")
            if M > 1:
                alloc("sh_rest", (P, M - 1, 3), "dL_dsh_rest")
    if st.has_pose:
        t = torch.empty(7, dtype=torch.float32, device=dev)     # always required by the ABI when pose is fused
        out["pose"] = t
        gr.dL_dpose = t.data_ptr()
    check(L.gsb_backward(ctypes.byref(st.cam), ctypes.byref(st.g), st.geom.data_ptr(), st.binning.data_ptr(),
                         st.R, st.image.data_ptr(), dL.data_ptr(), ctypes.byref(gr), _lib.stream_ptr()),
          "gsb_backward")
    return out


def _debug_snapshot(path: str, args) -> None:
    """Upstream's wrapper, in debug mode, saves the arguments of a failing call (snapshot_fw.dump / snapshot_bw.dump)
    before re-raising, so that the failure can be replayed."""
    try:
        torch.save(tuple(a.detach().cpu() if torch.is_tensor(a) else a for a in args), path)
        print(f"\nAn error occured in {'forward' if 'fw' in path else 'backward'}. Writing {path} for debugging.")
    except Exception as e:            # never mask the original error
        print(f"(could not write {path}: {e})")


class _RasterizeGaussians(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                raster_settings):
        has = lambda t: t is not None and t.numel() > 0
        M = sh.shape[1] if has(sh) else 1
        try:
            color, radii, st = _forward(
                raster_settings, means3D, scales if has(scales) else None,
                rotations if has(rotations) else None, opacities.reshape(-1) if opacities.dim() > 1 else opacities,
                sh if has(sh) else None, None, 1, M, colors_precomp if has(colors_precomp) else None,
                cov3Ds_precomp if has(cov3Ds_precomp) else None, None, 0)
        except Exception:
            if raster_settings.debug:
                _debug_snapshot("snapshot_fw.dump", (means3D, sh, colors_precomp, opacities, scales, rotations,
                                                     cov3Ds_precomp, tuple(raster_settings)))
            raise
        ctx.st = st
        # registered only so that autograd's version counters catch in-place edits between forward and backward
        # (the backward re-projects from the live input buffers)
        ctx.save_for_backward(*[t for t in (means3D, sh, colors_precomp, opacities, scales, rotations,
                                            cov3Ds_precomp) if torch.is_tensor(t)])
        ctx.shapes = (opacities.shape,)
        ctx.debug = raster_settings.debug
        ctx.mark_non_differentiable(radii)
        return color, radii

    @staticmethod
    def backward(ctx, grad_out_color, _grad_radii):
        st = ctx.st
        saved = ctx.saved_tensors
        try:
            g = _backward(st, grad_out_color, None, grad_out_color.device)
            if ctx.debug:
                torch.cuda.synchronize()
        except Exception:
            if ctx.debug:
                _debug_snapshot("snapshot_bw.dump", tuple(saved) + (grad_out_color,))
            raise
        return (g["means3D"], g["means2D"], g.get("sh"), g.get("colors"),
                g["opacities"].reshape(ctx.shapes[0]), g.get("scales"), g.get("rotations"), g.get("cov3D"),
                None)


def rasterize_gaussians(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                        raster_settings):
    return _RasterizeGaussians.apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                                     cov3Ds_precomp, raster_settings)


class _RasterizeFused(torch.autograd.Function):
    """InstantSplat path with everything fused: raw model tensors + camera pose in, image out.
    Replaces gaussian_renderer/__init__.py:81-135 and its autograd chain."""

    @staticmethod
    def forward(ctx, xyz, rotation, scaling, opacity, f_dc, f_rest, pose, means2D, raster_settings):
        M = 1 + (f_rest.shape[1] if f_rest is not None and f_rest.dim() == 3 else 0)
        color, radii, st = _forward(raster_settings, xyz, scaling, rotation, opacity.reshape(-1),
                                    f_dc.reshape(-1, 3), f_rest if M > 1 else None, 0, M, None, None, pose, 1)
        ctx.st = st
        ctx.save_for_backward(*[t for t in (xyz, rotation, scaling, opacity, f_dc, f_rest, pose) if torch.is_tensor(t)])
        ctx.shapes = (opacity.shape, f_dc.shape, None if f_rest is None else f_rest.shape)
        ctx.mark_non_differentiable(radii)
        return color, radii

    @staticmethod
    def backward(ctx, grad_out_color, _grad_radii):
        st = ctx.st
        _ = ctx.saved_tensors
        need = ctx.needs_input_grad      # xyz, rotation, scaling, opacity, f_dc, f_rest, pose, means2D, settings
        names = ("means3D", "rotations", "scales", "opacities", "sh_dc", "sh_rest", "pose", "means2D")
        want = {n for n, k in zip(names, need) if k}
        g = _backward(st, grad_out_color, want, grad_out_color.device)
        osh, dsh, rsh = ctx.shapes
        g_rest = g.get("sh_rest")
        if g_rest is None and rsh is not None and need[5]:
            g_rest = torch.zeros(rsh, dtype=torch.float32, device=grad_out_color.device)
        g_op = g.get("opacities")
        g_dc = g.get("sh_dc")
        return (g.get("means3D"), g.get("rotations"), g.get("scales"),
                None if g_op is None else g_op.reshape(osh), None if g_dc is None else g_dc.reshape(dsh), g_rest,
                g.get("pose") if need[6] else None, g.get("means2D"), None)


def rasterize_fused(xyz, rotation, scaling, opacity, f_dc, f_rest, pose, means2D, raster_settings):
    return _RasterizeFused.apply(xyz, rotation, scaling, opacity, f_dc, f_rest, pose, means2D, raster_settings)


class GaussianRasterizer(nn.Module):
    def __init__(self, raster_settings: GaussianRasterizationSettings):
        super().__init__()
        self.raster_settings = raster_settings

    def markVisible(self, positions):
        with torch.no_grad():
            rs = self.raster_settings
            pos = f32c(positions)
            vm, pm = f32c(rs.viewmatrix), f32c(rs.projmatrix)
            out = torch.empty(pos.shape[0], dtype=torch.uint8, device=pos.device)
            check(_lib.lib().gsb_mark_visible(pos.shape[0], ptr(pos), ptr(vm), ptr(pm), ptr(out),
                                              _lib.stream_ptr()), "gsb_mark_visible")
        return out.bool()

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                cov3D_precomp=None):
        rs = self.raster_settings
        if (shs is None and colors_precomp is None) or (shs is not None and colors_precomp is not None):
            raise Exception("Please provide excatly one of either SHs or precomputed colors!")
        if ((scales is None or rotations is None) and cov3D_precomp is None) or \
                ((scales is not None or rotations is not None) and cov3D_precomp is not None):
            raise Exception("Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!")
        e = torch.Tensor([]).to(means3D.device)
        return rasterize_gaussians(means3D, means2D, e if shs is None else shs,
                                   e if colors_precomp is None else colors_precomp, opacities,
                                   e if scales is None else scales, e if rotations is None else rotations,
                                   e if cov3D_precomp is None else cov3D_precomp, rs)
