"""`diff_gaussian_rasterization._C` surface (SURVEY.md section 8b, boundary B2): the three functions the upstream
Python wrapper binds from its torch C++ extension, with the upstream argument order, served by libgsb200.so.

    rasterize_gaussians(bg, means3D, colors_precomp, opacities, scales, rotations, scale_modifier, cov3D_precomp,
                        viewmatrix, projmatrix, tanfovx, tanfovy, image_height, image_width, sh, degree, campos,
                        prefiltered, debug) -> (num_rendered, color, radii, geomBuffer, binningBuffer, imgBuffer)
    rasterize_gaussians_backward(bg, means3D, radii, colors_precomp, scales, rotations, scale_modifier, cov3D_precomp,
                        viewmatrix, projmatrix, tanfovx, tanfovy, dL_dout_color, sh, degree, campos, geomBuffer,
                        num_rendered, binningBuffer, imgBuffer, debug)
                        -> (dL_dmeans2D, dL_dcolors, dL_dopacity, dL_dmeans3D, dL_dcov3D, dL_dsh, dL_dscales, dL_drotations)
    mark_visible(means3D, viewmatrix, projmatrix) -> bool[P]

Empty tensors stand for "not provided", as upstream.  The scratch buffers are torch byte tensors owned by the caller.
"""
import weakref

import torch

from instantsplat_b200 import rasterizer as _R

_live = {}      # geomBuffer.data_ptr() -> state of the forward (the upstream backward signature carries no opacities)


def _forget(key, st):
    if _live.get(key) is st:
        del _live[key]


def _opt(t):
    return t if (t is not None and t.numel() > 0) else None


def rasterize_gaussians(bg, means3D, colors_precomp, opacities, scales, rotations, scale_modifier, cov3D_precomp,
                        viewmatrix, projmatrix, tanfovx, tanfovy, image_height, image_width, sh, degree, campos,
                        prefiltered, debug):
    if means3D.dim() != 2 or means3D.shape[1] != 3:
        raise RuntimeError("means3D must have dimensions (num_points, 3)")
    rs = _R.GaussianRasterizationSettings(int(image_height), int(image_width), float(tanfovx), float(tanfovy), bg,
                                          float(scale_modifier), viewmatrix, projmatrix, int(degree), campos,
                                          bool(prefiltered), bool(debug))
    sh_ = _opt(sh)
    M = sh_.shape[1] if sh_ is not None else 1
    color, radii, st = _R._forward(rs, means3D, _opt(scales), _opt(rotations), opacities.reshape(-1), sh_, None, 1, M,
                                   _opt(colors_precomp), _opt(cov3D_precomp), None, 0)
    geom, binning, image = st.geom, st.binning, st.image
    st.geom = st.binning = st.image = None          # the registry must not keep the scratch alive
    # upstream's signature has no room for a handle, so the call is keyed on the buffer's address; the entry dies
    # with the tensor (finalizer, only if it still belongs to this call) and a forward whose geomBuffer reuses
    # the address replaces it
    key = geom.data_ptr()
    _live[key] = st
    weakref.finalize(geom, _forget, key, st)         # forget the call when the caller drops geomBuffer
    return st.R_true, color, radii, geom, binning, image


def rasterize_gaussians_backward(bg, means3D, radii, colors_precomp, scales, rotations, scale_modifier, cov3D_precomp,
                                 viewmatrix, projmatrix, tanfovx, tanfovy, dL_dout_color, sh, degree, campos,
                                 geomBuffer, num_rendered, binningBuffer, imgBuffer, debug):
    st = _live.get(geomBuffer.data_ptr())
    if st is None or st.R_true != int(num_rendered):
        raise RuntimeError("rasterize_gaussians_backward: unknown geomBuffer (call rasterize_gaussians first)")
    st.geom, st.binning, st.image = geomBuffer, binningBuffer, imgBuffer
    try:
        g = _R._backward(st, dL_dout_color, None, dL_dout_color.device)
    finally:
        st.geom = st.binning = st.image = None
    e = torch.empty(0, device=dL_dout_color.device)
    P = st.P
    return (g["means2D"], g.get("colors", e), g["opacities"].reshape(P, 1), g["means3D"], g.get("cov3D", e),
            g.get("sh", e), g.get("scales", e), g.get("rotations", e))


def mark_visible(means3D, viewmatrix, projmatrix):
    rs = _R.GaussianRasterizationSettings(1, 1, 1.0, 1.0, torch.zeros(3, device=means3D.device), 1.0, viewmatrix,
                                          projmatrix, 0, torch.zeros(3, device=means3D.device), False, False)
    return _R.GaussianRasterizer(rs).markVisible(means3D)
