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

import _geom as GM

H2_MIN = 2.5e-5
MARGIN = 0.15
NEAR = 0.2


def apply_filter3d(scales, opacities, filter3D, h3_grad=True):
    """Activated scales [P,3] and opacities [P] -> the 3D-filtered ones (Mip-Splatting's get_*_with_3D_filter).
    h3_grad=False: a wrong variant for tests to tell apart, without the gradient through h3 (the dh3 f^2 / s~^2 term)."""
    f2 = (filter3D.reshape(-1, 1) ** 2).to(scales.dtype)
    s2 = scales * scales
    coef = torch.sqrt((s2 / (s2 + f2)).prod(dim=1))
    return torch.sqrt(s2 + f2), opacities.reshape(-1) * (coef if h3_grad else coef.detach())


def project_mip(means3D, scales, rotations, opacities, shs, cam, kernel_size=None, means2D=None,
                colors_precomp=None, cov3D_precomp=None, floor_grad=False):
    """floor_grad=True: a wrong variant for tests to tell apart, which keeps differentiating through sqrt(r) where h2
    sits at its floor (where r > 0)."""
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
    if floor_grad:
        sr = torch.sqrt(torch.where(ratio.detach() > 0, ratio, torch.ones_like(ratio)))
        h2 = torch.where(clamp & (ratio.detach() > 0), math.sqrt(H2_MIN) + (sr - sr.detach()), h2)
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
               means2D=None, return_aux=False, lists=None, h3_grad=True, floor_grad=False, **blend_kw):
    """`O.render_instantsplat` with the filters: the fused path on raw parameters.  h3_grad, floor_grad: the wrong
    variants of apply_filter3d and project_mip."""
    means, rots = O.pose_pretransform(xyz, rotation, pose)
    s, o = torch.exp(scaling), torch.sigmoid(opacity).reshape(-1)
    if filter3D is not None:
        s, o = apply_filter3d(s, o, filter3D, h3_grad)
    proj = project_mip(means, s, rots, o, torch.cat([f_dc, f_rest], dim=1), cam, kernel_size, means2D,
                       floor_grad=floor_grad)
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


def mip_records(params, pose, cam, kappa, f3d):
    """`_geom.oracle_records_fused` of the filtered projection (fp64): `project_mip` of the raw parameters moved by
    `pose`, with what `_geom.flags` needs.  cam: the fused path's camera (its scale_modifier and sh_degree are used)."""
    p = {k: v.detach().cpu().double() for k, v in params.items()}
    cam = cam.to(torch.float64)
    means, rots = O.pose_pretransform(p["xyz"], p["rotation"], pose.detach().cpu().double())
    s, o = torch.exp(p["scaling"]), torch.sigmoid(p["opacity"]).reshape(-1)
    if f3d is not None:
        s, o = apply_filter3d(s, o, f3d.detach().cpu().double())
    shs = torch.cat([p["f_dc"], p["f_rest"]], 1) if p["f_rest"].numel() else p["f_dc"]
    with torch.no_grad():
        proj = project_mip(means, s, rots, o, shs, cam, kappa)
        # the kernel stops before h2 for a Gaussian behind the near plane: its record keeps o3
        proj["opacity"] = torch.where(means[:, 2] > NEAR, proj["opacity"], o)
        proj["tview"] = means
        d = means / means.norm(dim=1, keepdim=True)
        proj["raw_rgb"] = O.eval_sh(cam.sh_degree, shs, d) + 0.5
        proj["limx"], proj["limy"] = 1.3 * cam.tanfovx, 1.3 * cam.tanfovy
        proj["W"], proj["H"], proj["mean_norm"] = cam.width, cam.height, means.norm(dim=1)
        proj["h3"] = torch.ones_like(o) if f3d is None else o / torch.sigmoid(p["opacity"]).reshape(-1)
    return proj


def mip_flags(o, kappa):
    """Gaussians whose fp32 result may legitimately differ from the fp64 one because of a filter, on top of
    `_geom.flags` (o: mip_records).  fp32 resolves det Sigma2 = a0 c0 - b^2 only to about (a0 c0 + b^2) * 1e-7, so r =
    det0 / det1 to E = 1e-6 (a0 c0 + b^2) / det1:

    * h2_floor: r within E of the floor, where the gradient through h2 may be cut in one arm and not in the other;
    * ill: the conditioning bound of the record check, 2e-7 (a0 c0 + b^2) / |det0| > 1e-5, on rows not surely below
      the floor (those have h2 = sqrt(2.5e-5) exactly, whatever fp32 makes of det0).

    -> dict of bool [P]: h2_floor, ill, sure_clamp, and r, cond (fp64) for the bounds."""
    vis = o["visible"]
    a, b, c = o["cov2d"].unbind(-1)
    k = float(kappa or 0.0)
    a0, c0 = a - k, c - k
    det0, det1 = a0 * c0 - b * b, a * c - b * b
    scale = (a0 * c0 + b * b).abs()
    r = det0 / torch.where(det1 != 0, det1, torch.ones_like(det1))
    err = 1e-6 * scale / det1.abs().clamp(min=1e-300)
    cond = scale / det0.abs().clamp(min=1e-300)
    on = kappa is not None
    sure = vis & (r + err < H2_MIN) & on
    return dict(h2_floor=vis & ((r - H2_MIN).abs() <= err) & on, ill=vis & (2e-7 * cond > 1e-5) & ~sure & on,
                sure_clamp=sure, r=r, cond=cond)


def row_errors(a, b, tau=1e-3):
    """Per-row error of `_parity.row_err` (max |a_i - b_i| / (max |b_i| + tau max |b|)) as a vector, with the rows
    where either arm is non-zero."""
    a, b = a.detach().cpu().double(), b.detach().cpu().double()
    a, b = a.reshape(a.shape[0], -1), b.reshape(b.shape[0], -1)
    e = (a - b).abs().amax(1) / (b.abs().amax(1) + tau * b.abs().max() + 1e-300)
    return e, (b.abs().amax(1) > 0) | (a.abs().amax(1) > 0)


# ---- edge populations (tests/test_mip_edges.py, tests/test_mip_edges_cpu.py) ---------------------------------------
# Each builder returns dict(sc, kappa, f3d (fp32 [P] or None), groups {name: index range}, smod (scale_modifier));
# the populations sit in front of the pose, with a layer of ordinary Gaussians behind them (tests/test_projection_edges).
EDGE_POSE = (math.cos(0.1), math.sin(0.1) / math.sqrt(5), 2 * math.sin(0.1) / math.sqrt(5), 0.0, 0.2, -0.1, 0.3)


def _pe():
    import test_projection_edges as PE
    return PE


def _unit_quats(n, g):
    q = torch.randn(n, 4, generator=g, dtype=torch.float64)
    return q / q.norm(dim=1, keepdim=True)


def _at_pixel_centres(n, W, H, z, g, jitter=0.1):
    """Camera-frame centres at depths z whose projections lie within `jitter` px of a pixel centre (so that a Gaussian
    whose footprint is the 2D filter's alone still reaches one)."""
    tx, ty = _pe().camera_of(W, H)[2:4]
    u = torch.randint(2, W - 2, (n,), generator=g).double() + jitter * (2 * torch.rand(n, generator=g, dtype=torch.float64) - 1)
    v = torch.randint(2, H - 2, (n,), generator=g).double() + jitter * (2 * torch.rand(n, generator=g, dtype=torch.float64) - 1)
    return torch.stack([((2 * u + 1) / W - 1) * z * tx, ((2 * v + 1) / H - 1) * z * ty, z], 1)


def scale_to_ratio(pc, sig, q, W, H, kappa, r):
    """Scale each Gaussian (camera-frame centre pc, world sigmas sig, unit quaternion q) by the factor that makes
    r = det Sigma2 / det(Sigma2 + kappa I) equal to `r` in fp64.  With u the squared factor, D = det Sigma2 and
    S = trace Sigma2 at factor 1: r = u^2 D / (u^2 D + kappa u S + kappa^2), a quadratic in u."""
    fovx, fovy = _pe().camera_of(W, H)[:2]
    cam = O.Camera.instantsplat(W, H, fovx, fovy, sh_degree=0, dtype=torch.float64)
    n = pc.shape[0]
    pr = project_mip(pc, sig, q, torch.ones(n, dtype=torch.float64), None, cam, 0.0,
                     colors_precomp=torch.zeros(n, 3, dtype=torch.float64))
    a0, b, c0 = pr["cov2d"].unbind(-1)
    D, S = a0 * c0 - b * b, a0 + c0
    u = (r * kappa * S + torch.sqrt((r * kappa * S) ** 2 + 4 * D * (1 - r) * r * kappa ** 2)) / (2 * D * (1 - r))
    return sig * torch.sqrt(u)[:, None]


def _assemble(parts, W, H, seed, names, deg=1, pose=EDGE_POSE):
    PE = _pe()
    groups, off = {}, 0
    for nm, p in zip(names, parts):
        groups[nm] = (off, off + p[0].shape[0])
        off += p[0].shape[0]
    # camera-frame rotations q: the fused path composes pose_q (x) rotation, so store conj(pose_q) (x) q
    w, x, y, z = torch.tensor(pose[:4], dtype=torch.float64)
    q = torch.cat([p[3] for p in parts])
    rot = torch.stack([w * q[:, 0] + x * q[:, 1] + y * q[:, 2] + z * q[:, 3],
                       w * q[:, 1] - x * q[:, 0] - y * q[:, 3] + z * q[:, 2],
                       w * q[:, 2] + x * q[:, 3] - y * q[:, 0] - z * q[:, 1],
                       w * q[:, 3] - x * q[:, 2] + y * q[:, 1] - z * q[:, 0]], 1)
    sc = PE.build_scene([p[:3] for p in parts], W, H, seed=seed, pose=pose, deg=deg, rot=rot)
    return sc, groups


def _bg(n, W, H, g):
    pc, sig, op = _pe().background(n, W, H, g)
    return pc, sig, op, _unit_quats(n, g)


def population_h2(seed=901):
    """kernel_size 0.1, 256 x 192 (192 tiles: frame-filling rects exceed kBigRect = 128).
    needles: one axis 0.5-1.5 px, two 1e-6-1e-4 px (r far below the floor; det0 <= 0 in fp32 for many);
    straddle: r = 2.5e-5 (1 +- 1 %); subpixel: h2 from 0.05 to 0.9; frame: sigma 15-2e4 px, h2 > 0.999.
    Needles and straddle rows sit within 0.1 px of a pixel centre and are nearly opaque, so that their floored
    o_eff = o3 sqrt(2.5e-5) still reaches alpha 1/255 there."""
    W, H, kappa = 256, 192, 0.1
    PE = _pe()
    g = torch.Generator().manual_seed(seed)
    fx = PE.camera_of(W, H)[4]
    parts = []
    n = 300
    z = 2.0 + 3.0 * torch.rand(n, generator=g, dtype=torch.float64)
    lo = lambda a, b, k=1: torch.exp(torch.empty(n, k, dtype=torch.float64).uniform_(math.log(a), math.log(b), generator=g))
    sig = torch.cat([0.5 + torch.rand(n, 1, generator=g, dtype=torch.float64), lo(1e-6, 1e-4, 2)], 1) * (z / fx)[:, None]
    parts.append((_at_pixel_centres(n, W, H, z, g), sig, 0.85 + 0.14 * torch.rand(n, generator=g, dtype=torch.float64),
                  _unit_quats(n, g)))
    z = 2.0 + 3.0 * torch.rand(n, generator=g, dtype=torch.float64)
    pc, q = _at_pixel_centres(n, W, H, z, g), _unit_quats(n, g)
    base = (0.7 + 0.6 * torch.rand(n, 3, generator=g, dtype=torch.float64)) * (z / fx)[:, None]
    r = H2_MIN * (1.0 + 0.01 * (2 * torch.rand(n, generator=g, dtype=torch.float64) - 1))
    parts.append((pc, scale_to_ratio(pc, base, q, W, H, kappa, r),
                  0.85 + 0.14 * torch.rand(n, generator=g, dtype=torch.float64), q))
    z = 2.0 + 3.0 * torch.rand(n, generator=g, dtype=torch.float64)
    pc, q = PE.on_screen(n, W, H, z, g), _unit_quats(n, g)
    base = (0.7 + 0.6 * torch.rand(n, 3, generator=g, dtype=torch.float64)) * (z / fx)[:, None]
    h2 = 0.05 + 0.85 * torch.rand(n, generator=g, dtype=torch.float64)
    parts.append((pc, scale_to_ratio(pc, base, q, W, H, kappa, h2 * h2), 0.3 + 0.6 * torch.rand(n, generator=g,
                                                                                                  dtype=torch.float64), q))
    m = 40
    z = 2.0 + 3.0 * torch.rand(m, generator=g, dtype=torch.float64)
    s_px = torch.exp(torch.empty(m, dtype=torch.float64).uniform_(math.log(15.0), math.log(2e4), generator=g))
    sig = (s_px * z / fx)[:, None] * (0.8 + 0.4 * torch.rand(m, 3, generator=g, dtype=torch.float64))
    parts.append((PE.on_screen(m, W, H, z, g, margin=60.0), sig, 0.01 + 0.03 * torch.rand(m, generator=g,
                                                                                            dtype=torch.float64),
                  _unit_quats(m, g)))
    parts.append(_bg(600, W, H, g))
    sc, groups = _assemble(parts, W, H, seed + 1, ("needles", "straddle", "subpixel", "frame", "background"))
    return dict(sc=sc, kappa=kappa, f3d=None, groups=groups, smod=1.0)


def population_mixed(seed=911):
    """One mixed population for the kernel sizes 0, 0.3 and 4.0: sigma 0.02-8 px (within a factor 1.3 per axis)."""
    W, H = 128, 96
    PE = _pe()
    g = torch.Generator().manual_seed(seed)
    fx = PE.camera_of(W, H)[4]
    n = 600
    z = 2.0 + 3.0 * torch.rand(n, generator=g, dtype=torch.float64)
    s_px = torch.exp(torch.empty(n, dtype=torch.float64).uniform_(math.log(0.02), math.log(8.0), generator=g))
    sig = (s_px * z / fx)[:, None] * (0.75 + 0.5 * torch.rand(n, 3, generator=g, dtype=torch.float64))
    parts = [(PE.on_screen(n, W, H, z, g), sig, 0.3 + 0.65 * torch.rand(n, generator=g, dtype=torch.float64),
              _unit_quats(n, g)), _bg(300, W, H, g)]
    sc, groups = _assemble(parts, W, H, seed + 1, ("mixed", "background"))
    return dict(sc=sc, kappa=None, f3d=None, groups=groups, smod=1.0)


def population_clamp(seed=921):
    """kernel_size 0.1 with the frustum clamp: centres at |x/z| (|y/z|) from 1 to 3 x limx (limy), sized so that
    they still reach into the frame."""
    W, H = 128, 96
    PE = _pe()
    g = torch.Generator().manual_seed(seed)
    _, _, tx, ty, fx = PE.camera_of(W, H)
    limx, limy = 1.3 * tx, 1.3 * ty
    n = 600
    z = 2.0 + 4.0 * torch.rand(n, generator=g, dtype=torch.float64)
    kx = (1.0 + 2.0 * torch.rand(n, generator=g, dtype=torch.float64)) * limx
    ky = (1.0 + 2.0 * torch.rand(n, generator=g, dtype=torch.float64)) * limy
    sx = torch.where(torch.rand(n, generator=g) < 0.5, -1.0, 1.0).double()
    sy = torch.where(torch.rand(n, generator=g) < 0.5, -1.0, 1.0).double()
    which = torch.randint(0, 3, (n,), generator=g)             # 0: x clamped, 1: y clamped, 2: both
    inner_x = (2 * torch.rand(n, generator=g, dtype=torch.float64) - 1) * tx * 0.8
    inner_y = (2 * torch.rand(n, generator=g, dtype=torch.float64) - 1) * ty * 0.8
    xz = torch.where(which == 1, inner_x, sx * kx)
    yz = torch.where(which == 0, inner_y, sy * ky)
    off = torch.maximum((xz.abs() / tx - 1) * W / 2, (yz.abs() / ty - 1) * H / 2).clamp(min=0)
    s_px = (off + 8 + 32 * torch.rand(n, generator=g, dtype=torch.float64)) / 2.5
    sig = (s_px * z / fx)[:, None] * (0.8 + 0.4 * torch.rand(n, 3, generator=g, dtype=torch.float64))
    parts = [(torch.stack([xz * z, yz * z, z], 1), sig, 0.3 + 0.5 * torch.rand(n, generator=g, dtype=torch.float64),
              _unit_quats(n, g)), _bg(400, W, H, g)]
    sc, groups = _assemble(parts, W, H, seed + 1, ("clamp", "background"))
    return dict(sc=sc, kappa=0.1, f3d=None, groups=groups, smod=1.0)


def population_near(seed=931):
    """kernel_size 0.1 at the near plane: tz from 0.199 to 0.25, translucent, sigma 3-4e3 px, some centred off
    screen; 256 x 192 so that the largest rects go to the k_big_rects queue."""
    W, H = 256, 192
    PE = _pe()
    g = torch.Generator().manual_seed(seed)
    fx = PE.camera_of(W, H)[4]
    n = 200
    z = 0.199 + 0.051 * torch.rand(n, generator=g, dtype=torch.float64)
    s_px = torch.exp(torch.empty(n, dtype=torch.float64).uniform_(math.log(3.0), math.log(4e3), generator=g))
    sig = (s_px * z / fx)[:, None] * (0.8 + 0.4 * torch.rand(n, 3, generator=g, dtype=torch.float64))
    parts = [(PE.on_screen(n, W, H, z, g, margin=60.0), sig, 0.01 + 0.04 * torch.rand(n, generator=g,
                                                                                      dtype=torch.float64),
              _unit_quats(n, g)), _bg(600, W, H, g)]
    sc, groups = _assemble(parts, W, H, seed + 1, ("near", "background"))
    return dict(sc=sc, kappa=0.1, f3d=None, groups=groups, smod=1.0)


LOG_TINY = (-45.0, -52.0, -60.0)


def population_3d(seed=941, smod=1.0):
    """kernel_size 0.1 with the 3D filter.  ratio_axes: f/s_k from 1e-3 to 1e3, different on each axis; ratio_all: one
    f/s for all three axes; tiny_f: log-scales -45, -52, -60 with f > 0 (h3 = 0: no tiles); tiny_f0 and plain_f0: the same
    log-scales and ordinary Gaussians with f = 0 (no filter: h3 = 1 exactly), near pixel centres and nearly opaque."""
    W, H = 128, 96
    PE = _pe()
    g = torch.Generator().manual_seed(seed)
    fx = PE.camera_of(W, H)[4]
    parts, fs = [], []
    n = 250
    for per_axis in (True, False):
        z = 2.0 + 3.0 * torch.rand(n, generator=g, dtype=torch.float64)
        f = (0.01 + 0.04 * torch.rand(n, generator=g, dtype=torch.float64)) * z / fx
        lr = torch.empty(n, 1, dtype=torch.float64).uniform_(math.log(1e-3), math.log(1e3), generator=g)
        if per_axis:         # within a factor 4.5 of each other: wider spreads make needles, the h2 tests' business
            lr = lr + torch.empty(n, 3, dtype=torch.float64).uniform_(-1.5, 1.5, generator=g)
        rho = torch.exp(lr).expand(n, 3)
        parts.append((PE.on_screen(n, W, H, z, g), f[:, None] / rho, 0.3 + 0.6 * torch.rand(n, generator=g,
                                                                                             dtype=torch.float64),
                      _unit_quats(n, g)))
        fs.append(f)
    for f0 in (False, True):
        m = 3 * len(LOG_TINY)
        z = 2.0 + 3.0 * torch.rand(m, generator=g, dtype=torch.float64)
        ls = torch.tensor(LOG_TINY, dtype=torch.float64).repeat_interleave(3)
        parts.append((_at_pixel_centres(m, W, H, z, g), torch.exp(ls)[:, None].expand(m, 3).contiguous(),
                      torch.full((m,), 0.95, dtype=torch.float64), _unit_quats(m, g)))
        fs.append(torch.zeros(m, dtype=torch.float64) if f0 else 0.5 * z / fx)
    m = 30
    z = 2.0 + 3.0 * torch.rand(m, generator=g, dtype=torch.float64)
    parts.append((PE.on_screen(m, W, H, z, g), (1.0 + 3.0 * torch.rand(m, 3, generator=g, dtype=torch.float64))
                  * (z / fx)[:, None], 0.3 + 0.6 * torch.rand(m, generator=g, dtype=torch.float64), _unit_quats(m, g)))
    fs.append(torch.zeros(m, dtype=torch.float64))
    bgp = _bg(300, W, H, g)
    parts.append(bgp)
    fs.append(0.3 * bgp[0][:, 2] / fx)
    sc, groups = _assemble(parts, W, H, seed + 1, ("ratio_axes", "ratio_all", "tiny_f", "tiny_f0", "plain_f0",
                                                   "background"))
    return dict(sc=sc, kappa=0.1, f3d=torch.cat(fs).float(), groups=groups, smod=smod)


def group_mask(pop, *names):
    m = torch.zeros(pop["sc"].P, dtype=torch.bool)
    for nm in names:
        a, b = pop["groups"][nm]
        m[a:b] = True
    return m


def camera_of_pop(pop, dtype=torch.float64):
    """The fused path's camera of a population (its scale_modifier, sh_degree 1)."""
    sc = pop["sc"]
    cam = O.Camera.instantsplat(sc.width, sc.height, sc.fovx, sc.fovy, bg=torch.tensor([0.1, 0.2, 0.3]),
                                sh_degree=sc.sh_degree, dtype=dtype)
    cam.scale_modifier = pop["smod"]
    return cam


def edge_flags(o, kappa):
    """Rows whose decision lies within fp32 rounding: mip_flags' h2_floor and ill, _geom's cutoff, frustum-clamp and
    visibility flags."""
    mf, gf = mip_flags(o, kappa), GM.flags(o)
    return mf["h2_floor"] | mf["ill"] | gf["cutoff"] | gf["clamp_x"] | gf["clamp_y"] | gf["visibility"]


def reached(name, pop, kappa, o):
    """Counts that show a population's regime was reached (fp64, and fp32 where the regime is an fp32 event); name:
    h2, mixed..., clamp, near or 3d...; o: mip_records."""
    vis, clamp = o["visible"], o["h2_clamp"] & o["visible"]
    gm = lambda *g: group_mask(pop, *g)
    tiles = o["ntiles"]
    o255 = o["opacity"] * 255.0
    if name == "h2":
        # det0 = a0 c0 - b^2 as fp32 forms it (the restatement run in fp32 without a dilation)
        sc = pop["sc"]
        p = {k: v.float() for k, v in sc.params.items()}
        means, rots = O.pose_pretransform(p["xyz"], p["rotation"], sc.poses[0])
        cam32 = camera_of_pop(pop, torch.float32)
        a, b, c = project_mip(means, torch.exp(p["scaling"]), rots, torch.sigmoid(p["opacity"]).reshape(-1),
                                  torch.cat([p["f_dc"], p["f_rest"]], 1), cam32, 0.0)["cov2d"].unbind(-1)
        det0_32 = a * c - b * b
        r = mip_flags(o, kappa)["r"]
        st = gm("straddle")
        return dict(needles_clamped=int((clamp & gm("needles")).sum()),
                    needles_det0_fp32_le_0=int((gm("needles") & (det0_32 <= 0)).sum()),
                    straddle_clamped=int((clamp & st).sum()), straddle_free=int((vis & ~clamp & st).sum()),
                    straddle_r_off=float(((r / H2_MIN - 1).abs())[st].max()),
                    subpixel_h2_min=float(o["h2"][gm("subpixel")].min()),
                    subpixel_h2_max=float(o["h2"][gm("subpixel")].max()),
                    frame_h2_gt_0_999=int((vis & gm("frame") & (o["h2"] > 0.999)).sum()),
                    frame_big_rects=int((gm("frame") & (tiles > 128)).sum()),
                    clamped_reaching_cutoff=int((clamp & (o255 >= 1.0)).sum()))
    if name.startswith("mixed"):
        return dict(r_is_1=int((vis & (o["h2"] == 1.0)).sum()), visible=int(vis.sum()), clamped=int(clamp.sum()))
    t = o["tview"]
    if name == "clamp":
        clx = vis & ((t[:, 0] / t[:, 2]).abs() > o["limx"])
        cly = vis & ((t[:, 1] / t[:, 2]).abs() > o["limy"])
        return dict(clamp_x=int(clx.sum()), clamp_y=int(cly.sum()), both=int((clx & cly).sum()))
    if name == "near":
        tz = t[:, 2]
        return dict(visible_below_0_25=int((vis & (tz < 0.25)).sum()), behind_near=int((gm("near") & ~vis).sum()),
                    big_rects=int((tiles > 128).sum()))
    f = pop["f3d"].double()
    s = torch.exp(pop["sc"].params["scaling"].double())
    rho = f[:, None] / s
    h3 = o["h3"]
    rg = gm("ratio_axes", "ratio_all")
    return dict(h3_below_cutoff=int((rg & (h3 < 1 / 255)).sum()),
                s_near_f=int((rg & ((rho > 0.5) & (rho < 2.0)).all(1)).sum()),
                s_far_above_f=int((rg & (rho < 1e-2).all(1)).sum()),
                rho_min=float(rho[rg].min()), rho_max=float(rho[rg].max()),
                per_axis_spread=float((rho.amax(1) / rho.amin(1))[gm("ratio_axes")].min()),
                tiny_f_no_tiles=int((gm("tiny_f") & (o255 < 0.999)).sum()),
                tiny_f0_h3_1=int((gm("tiny_f0") & (h3 == 1.0) & (o255 >= 1.0)).sum()),
                plain_f0_h3_1=int((gm("plain_f0") & (h3 == 1.0)).sum()))
