"""Drop-in for the `diff_gaussian_rasterization` package (boundary B2 of SURVEY.md section 8b) on top
of libgsb200.so, plus the fused InstantSplat entry (`rasterize_fused`) used by `render()`.

Mirrors the interface the reference calls at gaussian_renderer/__init__.py:14-17,
60-78,126-135 (and the vanilla-3DGS form at gaussian_renderer/__init__3dgs.py:36-51,85-93):
same names, argument meaning and error behaviour.
"""
from __future__ import annotations

import warnings
from typing import NamedTuple, Optional

import torch
import torch.nn as nn

from . import _lib
from ._lib import GsbGrads, check, f32c, ptr
from .frame import ST_WORDS, Frame, camera, capacity, gaussians, mip_filter, read_R


class _Settings(NamedTuple):
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


class GaussianRasterizationSettings(_Settings):
    """The upstream settings tuple (its 12 fields, positional or keyword) plus Mip-Splatting's keyword `kernel_size`:
    the 2D Mip filter (0.1 in Mip-Splatting; 0.3 is the upstream rasterizer's later `antialiasing` mode), None for the
    reference's 0.3 px^2 dilation.  DESIGN.md section 4.7.  It is an attribute, not a tuple field, so the tuple
    stays the one upstream callers build and unpack."""

    def __new__(cls, *args, kernel_size: Optional[float] = None, **kw):
        self = super().__new__(cls, *args, **kw)
        self.kernel_size = None if kernel_size is None else float(kernel_size)
        return self

    # the namedtuple helpers, copy and pickle rebuild from the fields alone: carry kernel_size through them
    def _replace(self, **kw):
        ks = kw.pop("kernel_size", self.kernel_size)
        return type(self)(*_Settings._replace(self, **kw), kernel_size=ks)

    @classmethod
    def _make(cls, iterable, kernel_size: Optional[float] = None):
        return cls(*iterable, kernel_size=kernel_size)

    def __reduce__(self):
        return (_settings_with_kernel_size, (tuple(self), self.kernel_size))


def _settings_with_kernel_size(fields, kernel_size):
    return GaussianRasterizationSettings(*fields, kernel_size=kernel_size)


EXACT_CULL = True   # lossless alpha<1/255 tile culling (set False for the reference's rect-only binning)

# The instance count R (number of (Gaussian, tile) pairs) never has to reach the host BEFORE the render phase is
# launched: the kernels read it from device memory, the host only chooses the CAPACITY of the binning buffer.
# A forward sizes it from the counts seen for the same (device, P, W, H) with 50 % headroom, enqueues binning and
# blend, and only then waits for the status words of the PREPROCESS phase (an event right behind the tile scan):
# while the host waits, the GPU has the whole render phase queued, so it never idles -- unlike the reference's
# blocking cudaMemcpy of num_rendered, which stalls the GPU until the host has sized its buffers and launched the
# rest.  If the capacity was exceeded (rare), the render phase is repeated with an exact buffer before the forward
# returns, so whatever the caller computes from the image is consistent.  The first call of a shape, and every call
# in debug mode, waits for R before launching the render phase and sizes it exactly.
HEADROOM = 1.5
_last_R = {}            # (device index, P, W, H) -> last verified instance count


class _StatusRing:
    """Pinned 8-word status slots, recycled round-robin (a slot is long verified before it comes round again)."""

    def __init__(self, n=512):
        self.buf = torch.zeros(n, ST_WORDS, dtype=torch.int32).pin_memory()
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


class _State(Frame):
    """One forward: its scratch buffers and everything the backward needs (cam, g, and `keep`, the converted inputs
    they point to).  R_true: the forward's instance count."""

    @property
    def R(self) -> int:
        """The capacity the render phase ran with (the instance count it was sized for)."""
        return self.cap


_BIN_ROUND = 1 << 25    # binning allocations rounded up to 32 MiB so the caching allocator can reuse the last block


def _forward(settings, means3D, scales, rotations, opacities, sh_dc, sh_rest, sh_packed, M,
             colors_precomp, cov3D_precomp, pose, raw_params, filter3D=None):
    dev = means3D.device
    if means3D.dim() != 2 or means3D.shape[1] != 3:
        raise RuntimeError("means3D must have dimensions (num_points, 3)")
    P = means3D.shape[0]
    W, H = int(settings.image_width), int(settings.image_height)
    keep = [f32c(t) for t in (settings.bg, settings.viewmatrix, settings.projmatrix, settings.campos, means3D,
                              scales, rotations, opacities, sh_dc, sh_rest, colors_precomp, cov3D_precomp, pose,
                              filter3D)]
    bg, vm, pm, cp, xyz, sca, rot, op, dc, rest, cpre, cov, pos, f3d = keep
    cam = camera(W, H, settings.tanfovx, settings.tanfovy, settings.sh_degree, M, bg, vm, pm, cp,
                 settings.scale_modifier, EXACT_CULL)
    g = gaussians(P, xyz, rot, sca, op, dc, rest, pos, raw_params, sh_packed, cpre, cov)
    key = (dev.index, P, W, H)
    with torch.cuda.device(dev):
        st = _State(dev, P, W, H)
        st.cam, st.g, st.keep = cam, g, keep
        st.filt = mip_filter(getattr(settings, "kernel_size", None), f3d)
        st.M, st.packed, st.has_pose = M, bool(sh_packed), pose is not None
        est = None if settings.debug else _last_R.get(key)
        status = _status_slot()
        st.preprocess(cam, g, status, st.filt)
        event = torch.cuda.Event()
        event.record()
        if est is None:
            event.synchronize()                            # exact sizing: wait for R once
        st.alloc_binning(read_R(status) if est is None else capacity(est, HEADROOM), _BIN_ROUND)
        st.render(cam)
        event.synchronize()                                # recorded right behind the tile scan: early in the forward
        st.R_true = R = read_R(status)
        _last_R[key] = max(R, int(0.98 * _last_R.get(key, 0)))   # decaying maximum: different views share a key
        if R > st.cap:
            warnings.warn(f"instantsplat_b200: instance count {R} exceeded the binning capacity {st.cap}; "
                          "the render phase was repeated with an exact buffer", RuntimeWarning)
            st.alloc_binning(R, _BIN_ROUND)
            st.render(cam)
        if settings.debug:
            torch.cuda.synchronize()
    return st.color, st.radii, st


def _backward(st: _State, dL_dout, want, dev):
    """want: None (everything) or a set of names to compute; gradients that are not wanted are neither
    allocated nor written by the kernels (e.g. the pose-only test-view optimisation of
    render.py:99-170 passes {"pose"}).  Returns dict of dense grad tensors."""
    P, M = st.P, st.M
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
    st.backward(st.cam, st.g, dL, gr, st.filt)
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
    Replaces gaussian_renderer/__init__.py:81-135 and its autograd chain.  filter_3D: Mip-Splatting's 3D smoothing
    filter [P] (or [P, 1]), a constant."""

    @staticmethod
    def forward(ctx, xyz, rotation, scaling, opacity, f_dc, f_rest, pose, means2D, raster_settings, filter_3D=None):
        M = 1 + (f_rest.shape[1] if f_rest is not None and f_rest.dim() == 3 else 0)
        color, radii, st = _forward(raster_settings, xyz, scaling, rotation, opacity.reshape(-1),
                                    f_dc.reshape(-1, 3), f_rest if M > 1 else None, 0, M, None, None, pose, 1,
                                    None if filter_3D is None else filter_3D.detach().reshape(-1))
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
                g.get("pose") if need[6] else None, g.get("means2D"), None, None)


def rasterize_fused(xyz, rotation, scaling, opacity, f_dc, f_rest, pose, means2D, raster_settings, filter_3D=None):
    return _RasterizeFused.apply(xyz, rotation, scaling, opacity, f_dc, f_rest, pose, means2D, raster_settings,
                                 filter_3D)


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
