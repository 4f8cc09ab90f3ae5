"""fp64 restatement of the Mip-Splatting filters (DESIGN.md section 4.7) on top of the CPU oracle -- test code.

`project_mip` is `oracle.gs_oracle.project` with the 2D Mip filter: kernel_size * I replaces the 0.3 px^2 dilation and
the opacity is multiplied by h2 = sqrt(max(2.5e-5, det(cov2D) / det(cov2D + kernel_size I))), with no gradient
through h2 where the floor is active.  The upstream backward's 1/(det^2 + 1e-7) on the conic applies to the dilated
matrix, as in `O.project`; h2 takes the exact derivative.  With kernel_size None it returns `O.project` itself.
`filter3d_ref` restates the size of the 3D smoothing filter; `apply_filter3d` its effect on scales and opacities.
"""
import math

import torch

from oracle import gs_oracle as O

H2_MIN = 2.5e-5
MARGIN = 0.15
NEAR = 0.2


def apply_filter3d(scales, opacities, filter3D):
    """Activated scales [P,3] and opacities [P] -> the 3D-filtered ones (Mip-Splatting's get_*_with_3D_filter)."""
    f2 = (filter3D.reshape(-1, 1) ** 2).to(scales.dtype)
    s2 = scales * scales
    coef = torch.sqrt((s2 / (s2 + f2)).prod(dim=1))
    return torch.sqrt(s2 + f2), opacities.reshape(-1) * coef


def project_mip(means3D, scales, rotations, opacities, shs, cam, kernel_size=None, means2D=None,
                colors_precomp=None, cov3D_precomp=None):
    if kernel_size is None:
        return O.project(means3D, scales, rotations, opacities, shs, cam, means2D, colors_precomp, cov3D_precomp)
    dt = means3D.dtype
    P = means3D.shape[0]
    V, Pm = cam.viewmatrix.to(dt), cam.projmatrix.to(dt)
    W, H = cam.width, cam.height
    homo = torch.cat([means3D, torch.ones(P, 1, dtype=dt)], dim=1)
    p_view = (homo @ V)[:, :3]
    p_hom = homo @ Pm
    p_w = 1.0 / (p_hom[:, 3] + 1e-7)
    ndc = p_hom[:, :2] * p_w[:, None]
    if means2D is not None:
        ndc = ndc + means2D[:, :2]
    in_front = p_view[:, 2].detach() > NEAR
    if cov3D_precomp is None:
        r, x, y, z = rotations.unbind(-1)
        R = torch.stack([
            1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
            2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
            2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], dim=-1).reshape(P, 3, 3)
        M = R * (cam.scale_modifier * scales)[:, None, :]
        Sigma = M @ M.transpose(1, 2)
    else:
        c = cov3D_precomp
        Sigma = torch.stack([c[:, 0], c[:, 1], c[:, 2], c[:, 1], c[:, 3], c[:, 4],
                             c[:, 2], c[:, 4], c[:, 5]], dim=-1).reshape(P, 3, 3)
    fx = W / (2.0 * cam.tanfovx)
    fy = H / (2.0 * cam.tanfovy)
    tx, ty, tz = p_view.unbind(-1)
    tz_safe = torch.where(in_front, tz, torch.ones_like(tz))
    limx, limy = 1.3 * cam.tanfovx, 1.3 * cam.tanfovy
    txtz, tytz = tx / tz_safe, ty / tz_safe
    clx = (txtz.detach() < -limx) | (txtz.detach() > limx)
    cly = (tytz.detach() < -limy) | (tytz.detach() > limy)
    tx_c = torch.where(clx, (txtz.clamp(-limx, limx) * tz_safe).detach(), tx)
    ty_c = torch.where(cly, (tytz.clamp(-limy, limy) * tz_safe).detach(), ty)
    zero = torch.zeros_like(tz)
    J = torch.stack([fx / tz_safe, zero, -fx * tx_c / (tz_safe * tz_safe),
                     zero, fy / tz_safe, -fy * ty_c / (tz_safe * tz_safe)], dim=-1).reshape(P, 2, 3)
    T = J @ V[:3, :3].t()
    cov = T @ Sigma @ T.transpose(1, 2)
    a0, b0, c0 = cov[:, 0, 0], cov[:, 0, 1], cov[:, 1, 1]
    k = float(kernel_size)
    # compensation, exact derivative (no gradient where the floor is active)
    det0 = a0 * c0 - b0 * b0
    det1 = (a0 + k) * (c0 + k) - b0 * b0
    ratio = det0 / torch.where(det1.detach() != 0, det1, torch.ones_like(det1))
    clamp = ~(ratio.detach() > H2_MIN)
    h2 = torch.where(clamp, torch.full_like(ratio, math.sqrt(H2_MIN)), torch.sqrt(torch.where(clamp, torch.ones_like(ratio), ratio)))
    abc = torch.stack([a0 + k, b0, c0 + k], dim=-1)
    det_ng = (abc[:, 0] * abc[:, 2] - abc[:, 1] * abc[:, 1]).detach()
    abc = O._GradScale.apply(abc, (det_ng * det_ng / (det_ng * det_ng + 1e-7))[:, None])
    a, b, c_ = abc.unbind(-1)
    det = a * c_ - b * b
    det_ok = det.detach() != 0
    det_safe = torch.where(det_ok, det, torch.ones_like(det))
    conic = torch.stack([c_ / det_safe, -b / det_safe, a / det_safe], dim=-1)
    with torch.no_grad():
        mid = 0.5 * (a + c_)
        lam = mid + torch.sqrt(torch.clamp(mid * mid - det, min=0.1))
        radius = torch.ceil(3.0 * torch.sqrt(lam))
    pix = torch.stack([((ndc[:, 0] + 1.0) * W - 1.0) * 0.5, ((ndc[:, 1] + 1.0) * H - 1.0) * 0.5], dim=-1)
    gx, gy = (W + O.BLOCK - 1) // O.BLOCK, (H + O.BLOCK - 1) // O.BLOCK
    with torch.no_grad():
        def tr(v, hi):
            return torch.trunc(v.clamp(-1.0e8, 1.0e8)).clamp(0, hi).to(torch.int64)

        rx0 = tr((pix[:, 0] - radius) / O.BLOCK, gx)
        ry0 = tr((pix[:, 1] - radius) / O.BLOCK, gy)
        rx1 = tr((pix[:, 0] + radius + O.BLOCK - 1) / O.BLOCK, gx)
        ry1 = tr((pix[:, 1] + radius + O.BLOCK - 1) / O.BLOCK, gy)
        ntiles = (rx1 - rx0) * (ry1 - ry0)
        visible = in_front & det_ok & (ntiles > 0)
        ntiles = torch.where(visible, ntiles, torch.zeros_like(ntiles))
        radii = torch.where(visible, radius, torch.zeros_like(radius)).to(torch.int32)
    if colors_precomp is None:
        d = means3D - cam.campos.to(dt)[None]
        d = d / d.norm(dim=1, keepdim=True)
        raw = O.eval_sh(cam.sh_degree, shs, d) + 0.5
        clamped = raw.detach() < 0
        rgb = torch.where(clamped, torch.zeros_like(raw), raw)
    else:
        rgb = colors_precomp
        clamped = torch.zeros_like(rgb, dtype=torch.bool)
    return dict(xy=pix, depth=p_view[:, 2], conic=conic, opacity=opacities.reshape(P) * h2, h2=h2, h2_clamp=clamp,
                rgb=rgb, clamped=clamped, radii=radii, visible=visible,
                rect=torch.stack([rx0, ry0, rx1, ry1], dim=-1), ntiles=ntiles, cov2d=abc, grid=(gx, gy))


def render_mip(xyz, rotation, scaling, opacity, f_dc, f_rest, pose, cam, kernel_size=None, filter3D=None,
               means2D=None, return_aux=False, lists=None, **blend_kw):
    """`O.render_instantsplat` with the filters: the fused path on raw parameters."""
    means, rots = O.pose_pretransform(xyz, rotation, pose)
    s, o = torch.exp(scaling), torch.sigmoid(opacity).reshape(-1)
    if filter3D is not None:
        s, o = apply_filter3d(s, o, filter3D)
    proj = project_mip(means, s, rots, o, torch.cat([f_dc, f_rest], dim=1), cam, kernel_size, means2D)
    res = O.blend(proj, cam, return_aux=return_aux, lists=lists, **blend_kw)
    if return_aux:
        img, aux = res
        aux["proj"] = proj
        return img, proj["radii"], aux
    return res, proj["radii"]


def filter3d_ref(xyz, poses7, W, H, tanfovx, tanfovy, return_margin=False):
    """Size of the 3D smoothing filter in fp64.  return_margin: also the per-Gaussian distance (over all views) of the
    depth and frame-border tests from their thresholds, to flag decisions within fp32 rounding."""
    xyz = xyz.double()
    fx, fy = W / (2.0 * tanfovx), H / (2.0 * tanfovy)
    d = torch.full((xyz.shape[0],), math.inf, dtype=torch.float64)
    margin = torch.full((xyz.shape[0],), math.inf, dtype=torch.float64)
    for pose in poses7.double():
        Rm = O.quad2rotation(pose[:4])
        p = xyz @ Rm.t() + pose[4:7]
        z = p[:, 2]
        zs = torch.where(z > 0, z, torch.ones_like(z))
        u = p[:, 0] / zs * fx + W / 2
        v = p[:, 1] / zs * fy + H / 2
        ok = (z > NEAR) & (u >= -MARGIN * W) & (u <= (1 + MARGIN) * W) & (v >= -MARGIN * H) & (v <= (1 + MARGIN) * H)
        d = torch.where(ok, torch.minimum(d, z), d)
        m = torch.stack([(z - NEAR).abs() / NEAR, (u + MARGIN * W).abs() / W, (u - (1 + MARGIN) * W).abs() / W,
                         (v + MARGIN * H).abs() / H, (v - (1 + MARGIN) * H).abs() / H], 1).min(1)[0]
        margin = torch.minimum(margin, m)
    seen = torch.isfinite(d)
    fill = d[seen].max() if bool(seen.any()) else torch.tensor(0.0, dtype=torch.float64)
    d = torch.where(seen, d, fill)
    f = d / fx * math.sqrt(0.2)
    return (f, margin) if return_margin else f
