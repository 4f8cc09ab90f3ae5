"""CPU oracle for the InstantSplat hot path  --  TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s cpu_baseline / ``--impl reference``
legs may import this module.  The product path (``instantsplat_b200``) never imports it and
fails loudly when the CUDA library is missing.

What it restates (pure PyTorch, CPU, differentiable through autograd, fp32 or fp64):

* pose pre-transform              gaussian_renderer/__init__.py:81-92,
                                  utils/pose_utils.py:10-55,57-84,86-104
* projection matrix               utils/graphics_utils.py:71-91
* SH -> RGB                       utils/sh_utils.py:57-112 (+0.5 / clamp:
                                  gaussian_renderer/__init__.py:119)
* EWA projection, tile rect, (tile, depth) order, front-to-back blend and the analytic
  backward's deviations from naive autograd: SURVEY.md Appendix A.  The arithmetic lives in
  graphdeco-inria/diff-gaussian-rasterization @ 59f5f77e3ddbac3ed9db93ec2cfe99ed6c5d121d,
  which is an EMPTY submodule in the reference checkout, so this part is a restatement of the
  published algorithm anchored on the reference's call site
  (gaussian_renderer/__init__.py:60-78,126-135).
* L1 / SSIM loss                  utils/loss_utils.py:39-40,45-85 ;
                                  combine train.py:176
* per-point Adam                  scene/per_point_adam.py:34-98

PARITY PINNING STATUS
  pinned   : eval_sh, ssim, l1_loss, get_camera_from_tensor, quadmultiply, getProjectionMatrix,
             PerPointAdam -- checked against the reference's own Python modules imported from
             an InstantSplat checkout (oracle/make_golden.py; vectors in tests/golden/).
  unpinned : the rasterizer proper (EWA / binning / blend / backward).  The reference holds no
             source, tests or golden vectors for it ("parity unpinned" -- see DESIGN.md); it is
             cross-checked only by fp64 finite differences and internal consistency.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Optional

import torch
import torch.nn.functional as F

BLOCK = 16
ALPHA_MIN = 1.0 / 255.0
T_EPS = 1e-4

# utils/sh_utils.py:24-52
SH_C0 = 0.28209479177387814
SH_C1 = 0.4886025119029199
SH_C2 = (1.0925484305920792, -1.0925484305920792, 0.31539156525252005,
         -1.0925484305920792, 0.5462742152960396)
SH_C3 = (-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154,
         -0.4570457994644658, 1.445305721320277, -0.5900435899266435)


# ----------------------------------------------------------------------------------------------
# camera / pose helpers
# ----------------------------------------------------------------------------------------------
def projection_matrix(znear: float, zfar: float, fovx: float, fovy: float, dtype=torch.float32):
    """utils/graphics_utils.py:71-91 (returned NOT transposed)."""
    ty = math.tan(fovy / 2)
    tx = math.tan(fovx / 2)
    top, right = ty * znear, tx * znear
    bottom, left = -top, -right
    P = torch.zeros(4, 4, dtype=dtype)
    P[0, 0] = 2.0 * znear / (right - left)
    P[1, 1] = 2.0 * znear / (top - bottom)
    P[0, 2] = (right + left) / (right - left)
    P[1, 2] = (top + bottom) / (top - bottom)
    P[3, 2] = 1.0
    P[2, 2] = zfar / (zfar - znear)
    P[2, 3] = -(zfar * znear) / (zfar - znear)
    return P


@dataclass
class Camera:
    """Rasterizer settings, gaussian_renderer/__init__.py:60-76.

    ``viewmatrix`` / ``projmatrix`` are stored TRANSPOSED (row-vector convention,
    scene/cameras.py:54-56): p_view = [p,1] @ viewmatrix.
    """
    width: int
    height: int
    tanfovx: float
    tanfovy: float
    viewmatrix: torch.Tensor
    projmatrix: torch.Tensor
    campos: torch.Tensor
    bg: torch.Tensor
    sh_degree: int = 3
    scale_modifier: float = 1.0

    @staticmethod
    def instantsplat(width, height, fovx, fovy, bg=None, sh_degree=3, dtype=torch.float32,
                     znear=0.01, zfar=100.0):
        """Identity view, projmatrix = I @ P^T, campos = 0
        (gaussian_renderer/__init__.py:55-59)."""
        Pm = projection_matrix(znear, zfar, fovx, fovy, dtype).t().contiguous()
        if bg is None:
            bg = torch.zeros(3, dtype=dtype)
        return Camera(width, height, math.tan(fovx * 0.5), math.tan(fovy * 0.5),
                      torch.eye(4, dtype=dtype), Pm, torch.zeros(3, dtype=dtype),
                      bg.to(dtype), sh_degree)

    def to(self, dtype):
        return Camera(self.width, self.height, self.tanfovx, self.tanfovy,
                      self.viewmatrix.to(dtype), self.projmatrix.to(dtype),
                      self.campos.to(dtype), self.bg.to(dtype), self.sh_degree,
                      self.scale_modifier)


def quad2rotation(q: torch.Tensor) -> torch.Tensor:
    """utils/pose_utils.py:34-55 -- normalises q.  q: [4] -> [3,3]."""
    q = q / torch.sqrt((q * q).sum())
    r, x, y, z = q[0], q[1], q[2], q[3]
    return torch.stack([
        1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
        2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
        2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)]).reshape(3, 3)


def pose_to_w2c(pose: torch.Tensor) -> torch.Tensor:
    """utils/pose_utils.py:57-84.  pose = [qw,qx,qy,qz,tx,ty,tz] -> 4x4."""
    R = quad2rotation(pose[:4])
    top = torch.cat([R, pose[4:7].reshape(3, 1)], dim=1)
    bottom = torch.tensor([[0.0, 0.0, 0.0, 1.0]], dtype=pose.dtype, device=pose.device)
    return torch.cat([top, bottom], dim=0)


def quadmultiply(q1: torch.Tensor, q2: torch.Tensor) -> torch.Tensor:
    """utils/pose_utils.py:86-104 (Hamilton product, real first, no normalise)."""
    w1, x1, y1, z1 = q1.unbind(-1)
    w2, x2, y2, z2 = q2.unbind(-1)
    return torch.stack([
        w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2,
        w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2,
        w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2,
        w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2], dim=-1)


def pose_pretransform(xyz: torch.Tensor, rot: torch.Tensor, pose: torch.Tensor):
    """gaussian_renderer/__init__.py:81-89."""
    w2c = pose_to_w2c(pose)
    homo = torch.cat([xyz, torch.ones(xyz.shape[0], 1, dtype=xyz.dtype, device=xyz.device)], dim=1)
    means = (w2c @ homo.t()).t()[:, :3]
    rots = quadmultiply(pose[:4], rot)
    return means, rots


# ----------------------------------------------------------------------------------------------
# SH
# ----------------------------------------------------------------------------------------------
def eval_sh(deg: int, sh: torch.Tensor, dirs: torch.Tensor) -> torch.Tensor:
    """sh: [P, M, 3] (coefficient-major, the rasterizer's layout), dirs [P,3] unit -> [P,3].
    Polynomial of utils/sh_utils.py:57-112."""
    res = SH_C0 * sh[:, 0]
    if deg > 0:
        x, y, z = dirs[:, 0:1], dirs[:, 1:2], dirs[:, 2:3]
        res = res - SH_C1 * y * sh[:, 1] + SH_C1 * z * sh[:, 2] - SH_C1 * x * sh[:, 3]
        if deg > 1:
            xx, yy, zz = x * x, y * y, z * z
            xy, yz, xz = x * y, y * z, x * z
            res = (res + SH_C2[0] * xy * sh[:, 4] + SH_C2[1] * yz * sh[:, 5]
                   + SH_C2[2] * (2.0 * zz - xx - yy) * sh[:, 6]
                   + SH_C2[3] * xz * sh[:, 7] + SH_C2[4] * (xx - yy) * sh[:, 8])
            if deg > 2:
                res = (res + SH_C3[0] * y * (3 * xx - yy) * sh[:, 9]
                       + SH_C3[1] * xy * z * sh[:, 10]
                       + SH_C3[2] * y * (4 * zz - xx - yy) * sh[:, 11]
                       + SH_C3[3] * z * (2 * zz - 3 * xx - 3 * yy) * sh[:, 12]
                       + SH_C3[4] * x * (4 * zz - xx - yy) * sh[:, 13]
                       + SH_C3[5] * z * (xx - yy) * sh[:, 14]
                       + SH_C3[6] * x * (xx - 3 * yy) * sh[:, 15])
    return res


class _GradScale(torch.autograd.Function):
    """Identity in forward; multiplies the incoming gradient by ``factor`` (A.3: the conic
    backward uses 1/(det^2 + 1e-7) in place of 1/det^2)."""

    @staticmethod
    def forward(ctx, x, factor):
        ctx.save_for_backward(factor)
        return x.clone()

    @staticmethod
    def backward(ctx, g):
        (factor,) = ctx.saved_tensors
        return g * factor, None


# ----------------------------------------------------------------------------------------------
# per-Gaussian projection  (Appendix A.2 steps 1-8)
# ----------------------------------------------------------------------------------------------
def project(means3D, scales, rotations, opacities, shs, cam: Camera, means2D=None,
            colors_precomp=None, cov3D_precomp=None):
    """Returns a dict of per-Gaussian projected quantities.

    means3D [P,3] (already in the frame the rasterizer is given), scales [P,3] (activated),
    rotations [P,4] raw (never normalised), opacities [P] or [P,1] (activated),
    shs [P,M,3].  ``means2D`` is the dummy whose grad receives dL/d(ndc_xy) (A.3).
    """
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
    in_front = p_view[:, 2].detach() > 0.2                      # A.2.1

    if cov3D_precomp is None:
        r, x, y, z = rotations.unbind(-1)                       # A.2.2, un-normalised
        R = torch.stack([
            1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
            2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
            2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)],
            dim=-1).reshape(P, 3, 3)
        M = R * (cam.scale_modifier * scales)[:, None, :]
        Sigma = M @ M.transpose(1, 2)
    else:
        c = cov3D_precomp
        Sigma = torch.stack([c[:, 0], c[:, 1], c[:, 2], c[:, 1], c[:, 3], c[:, 4],
                             c[:, 2], c[:, 4], c[:, 5]], dim=-1).reshape(P, 3, 3)

    fx = W / (2.0 * cam.tanfovx)
    fy = H / (2.0 * cam.tanfovy)
    tx, ty, tz = p_view.unbind(-1)
    tz_safe = torch.where(in_front, tz, torch.ones_like(tz))    # avoid inf/nan in culled rows
    limx, limy = 1.3 * cam.tanfovx, 1.3 * cam.tanfovy
    txtz, tytz = tx / tz_safe, ty / tz_safe
    clx = (txtz.detach() < -limx) | (txtz.detach() > limx)
    cly = (tytz.detach() < -limy) | (tytz.detach() > limy)
    # A.3: the clamp is a constant when active (no grad to t_x, and none to t_z through it)
    tx_c = torch.where(clx, (txtz.clamp(-limx, limx) * tz_safe).detach(), tx)
    ty_c = torch.where(cly, (tytz.clamp(-limy, limy) * tz_safe).detach(), ty)
    zero = torch.zeros_like(tz)
    J = torch.stack([fx / tz_safe, zero, -fx * tx_c / (tz_safe * tz_safe),
                     zero, fy / tz_safe, -fy * ty_c / (tz_safe * tz_safe)],
                    dim=-1).reshape(P, 2, 3)
    Wr = V[:3, :3].t()                                          # true rotation of w2c
    T = J @ Wr
    cov = T @ Sigma @ T.transpose(1, 2)
    abc = torch.stack([cov[:, 0, 0] + 0.3, cov[:, 0, 1], cov[:, 1, 1] + 0.3], dim=-1)
    det_ng = (abc[:, 0] * abc[:, 2] - abc[:, 1] * abc[:, 1]).detach()
    abc = _GradScale.apply(abc, (det_ng * det_ng / (det_ng * det_ng + 1e-7))[:, None])
    a, b, c_ = abc.unbind(-1)
    det = a * c_ - b * b
    det_ok = det.detach() != 0
    det_safe = torch.where(det_ok, det, torch.ones_like(det))
    conic = torch.stack([c_ / det_safe, -b / det_safe, a / det_safe], dim=-1)
    with torch.no_grad():
        mid = 0.5 * (a + c_)
        lam = mid + torch.sqrt(torch.clamp(mid * mid - det, min=0.1))
        radius = torch.ceil(3.0 * torch.sqrt(lam))
    pix = torch.stack([((ndc[:, 0] + 1.0) * W - 1.0) * 0.5,
                       ((ndc[:, 1] + 1.0) * H - 1.0) * 0.5], dim=-1)
    gx, gy = (W + BLOCK - 1) // BLOCK, (H + BLOCK - 1) // BLOCK
    with torch.no_grad():
        big = 1.0e8

        def tr(v, hi):
            return torch.trunc(v.clamp(-big, big)).clamp(0, hi).to(torch.int64)

        rx0 = tr((pix[:, 0] - radius) / BLOCK, gx)
        ry0 = tr((pix[:, 1] - radius) / BLOCK, gy)
        rx1 = tr((pix[:, 0] + radius + BLOCK - 1) / BLOCK, gx)
        ry1 = tr((pix[:, 1] + radius + BLOCK - 1) / BLOCK, gy)
        ntiles = (rx1 - rx0) * (ry1 - ry0)
        visible = in_front & det_ok & (ntiles > 0)
        ntiles = torch.where(visible, ntiles, torch.zeros_like(ntiles))
        radii = torch.where(visible, radius, torch.zeros_like(radius)).to(torch.int32)

    if colors_precomp is None:
        d = means3D - cam.campos.to(dt)[None]
        d = d / d.norm(dim=1, keepdim=True)
        raw = eval_sh(cam.sh_degree, shs, d) + 0.5
        clamped = raw.detach() < 0
        rgb = torch.where(clamped, torch.zeros_like(raw), raw)
    else:
        rgb = colors_precomp
        clamped = torch.zeros_like(rgb, dtype=torch.bool)

    return dict(xy=pix, depth=p_view[:, 2], conic=conic, opacity=opacities.reshape(P),
                rgb=rgb, clamped=clamped, radii=radii, visible=visible,
                rect=torch.stack([rx0, ry0, rx1, ry1], dim=-1), ntiles=ntiles,
                cov2d=abc, grid=(gx, gy))


# ----------------------------------------------------------------------------------------------
# binning  (A.2 steps 7, 9)
# ----------------------------------------------------------------------------------------------
def build_tile_lists(proj):
    """Returns (sorted gaussian ids [R], ranges [T,2]) in (tile, depth, index) order."""
    gx, gy = proj["grid"]
    vis = proj["visible"]
    ids = torch.nonzero(vis).reshape(-1)
    depth = proj["depth"].detach()[ids].to(torch.float32)
    # depth compared as the uint32 bit pattern of a positive fp32; ties -> ascending index
    order = torch.argsort(depth.view(torch.int32).to(torch.int64), stable=True)
    ids = ids[order]
    rect = proj["rect"][ids]
    w = rect[:, 2] - rect[:, 0]
    h = rect[:, 3] - rect[:, 1]
    n = w * h
    R = int(n.sum())
    rank = torch.arange(ids.numel())
    rep = torch.repeat_interleave(rank, n)
    start = torch.cumsum(n, 0) - n
    local = torch.arange(R) - start[rep]
    wx = w[rep]
    txy = rect[rep, 0] + local % wx
    tyy = rect[rep, 1] + local // wx
    tile = tyy * gx + txy
    key = tile * (ids.numel() + 1) + rep
    o2 = torch.argsort(key, stable=True)
    tile_sorted = tile[o2]
    gids = ids[rep[o2]]
    T = gx * gy
    bounds = torch.searchsorted(tile_sorted, torch.arange(T + 1))
    ranges = torch.stack([bounds[:-1], bounds[1:]], dim=-1)
    return gids, ranges


# ----------------------------------------------------------------------------------------------
# blend  (A.2 step 10, A.3)
# ----------------------------------------------------------------------------------------------
def blend(proj, cam: Camera, tiles=None, return_aux=False, alpha_min=ALPHA_MIN, t_eps=T_EPS):
    """Front-to-back alpha blend per 16x16 tile.  ``tiles``: optional iterable of tile ids to
    render (others left at bg) -- used for bounded CPU timing samples."""
    dt = proj["xy"].dtype
    W, H = cam.width, cam.height
    gx, gy = proj["grid"]
    gids, ranges = build_tile_lists(proj)
    bg = cam.bg.to(dt)
    out = bg[:, None, None].expand(3, H, W).clone()
    final_T = torch.ones(H, W, dtype=dt)
    n_contrib = torch.zeros(H, W, dtype=torch.int32)
    ambiguous = torch.zeros(H, W, dtype=torch.bool)
    pieces = []
    tile_iter = range(gx * gy) if tiles is None else tiles
    for t in tile_iter:
        s, e = int(ranges[t, 0]), int(ranges[t, 1])
        if e <= s:
            continue
        ty_, tx_ = divmod(t, gx)
        x0, y0 = tx_ * BLOCK, ty_ * BLOCK
        x1, y1 = min(x0 + BLOCK, W), min(y0 + BLOCK, H)
        ys, xs = torch.meshgrid(torch.arange(y0, y1), torch.arange(x0, x1), indexing="ij")
        px = xs.reshape(-1).to(dt)
        py = ys.reshape(-1).to(dt)
        g = gids[s:e]
        xy = proj["xy"][g]
        con = proj["conic"][g]
        op = proj["opacity"][g]
        col = proj["rgb"][g]
        dx = xy[:, 0:1] - px[None]
        dy = xy[:, 1:2] - py[None]
        power = -0.5 * (con[:, 0:1] * dx * dx + con[:, 2:3] * dy * dy) - con[:, 1:2] * dx * dy
        G = torch.exp(torch.clamp(power, max=0.0))
        alpha_raw = op[:, None] * G
        # straight-through min(0.99, .)  (A.3)
        alpha = alpha_raw + (alpha_raw.clamp(max=0.99) - alpha_raw).detach()
        with torch.no_grad():
            valid = (power <= 0) & (alpha >= alpha_min)
            a0 = torch.where(valid, alpha, torch.zeros_like(alpha))
            Tincl = torch.cumprod(1 - a0, dim=0)
            stop = valid & (Tincl < t_eps)
            done = torch.cummax(stop.to(torch.int8), dim=0)[0].bool()
            live = valid & ~done
            if return_aux:
                amb = ((alpha * 255.0 - 1.0).abs() < 5e-4) | (valid & ((Tincl - T_EPS).abs() < 1e-7)) \
                      | ((power > -1e-7) & (power != 0) & (op[:, None] >= ALPHA_MIN))
                amb = amb & ~torch.cat([torch.zeros_like(done[:1]), done[:-1]], dim=0)
                ambiguous[y0:y1, x0:x1] = amb.any(0).reshape(y1 - y0, x1 - x0)
                idx = torch.arange(1, e - s + 1)[:, None] * live
                n_contrib[y0:y1, x0:x1] = idx.max(0)[0].reshape(y1 - y0, x1 - x0).to(torch.int32)
        a = torch.where(live, alpha, torch.zeros_like(alpha))
        one_m = 1 - a
        Tin = torch.cumprod(one_m, dim=0)
        Tex = torch.cat([torch.ones_like(Tin[:1]), Tin[:-1]], dim=0)
        wgt = a * Tex
        C = wgt.t() @ col                                       # [npix,3]
        Tf = Tin[-1]
        img = C.t() + Tf[None] * bg[:, None]
        pieces.append((t, img.reshape(3, y1 - y0, x1 - x0)))
        if return_aux:
            final_T[y0:y1, x0:x1] = Tf.detach().reshape(y1 - y0, x1 - x0)
    # assemble differentiably
    for t, img in pieces:
        ty_, tx_ = divmod(t, gx)
        x0, y0 = tx_ * BLOCK, ty_ * BLOCK
        out[:, y0:y0 + img.shape[1], x0:x0 + img.shape[2]] = img
    if return_aux:
        return out, dict(final_T=final_T, n_contrib=n_contrib, ambiguous=ambiguous,
                         gids=gids, ranges=ranges)
    return out


def rasterize(means3D, scales, rotations, opacities, shs, cam: Camera, means2D=None,
              colors_precomp=None, cov3D_precomp=None, tiles=None, return_aux=False, **blend_kw):
    """The ``GaussianRasterizer.forward`` boundary (B2): returns (color [3,H,W], radii [P])."""
    proj = project(means3D, scales, rotations, opacities, shs, cam, means2D,
                   colors_precomp, cov3D_precomp)
    res = blend(proj, cam, tiles=tiles, return_aux=return_aux, **blend_kw)
    if return_aux:
        img, aux = res
        aux["proj"] = proj
        return img, proj["radii"], aux
    return res, proj["radii"]


def render_instantsplat(xyz, rotation, scaling, opacity, f_dc, f_rest, pose, cam: Camera,
                        means2D=None, tiles=None, return_aux=False, **blend_kw):
    """The ``render()`` boundary (B1) on RAW parameters
    (gaussian_renderer/__init__.py:23-144 with the default pipe flags;
    activations scene/gaussian_model.py:101-121)."""
    means, rots = pose_pretransform(xyz, rotation, pose)
    shs = torch.cat([f_dc, f_rest], dim=1)
    return rasterize(means, torch.exp(scaling), rots, torch.sigmoid(opacity), shs, cam,
                     means2D=means2D, tiles=tiles, return_aux=return_aux, **blend_kw)


# ----------------------------------------------------------------------------------------------
# loss  (A.4)
# ----------------------------------------------------------------------------------------------
def l1_loss(a, b):
    """utils/loss_utils.py:39-40."""
    return (a - b).abs().mean()


def gaussian_window(window_size=11, sigma=1.5, dtype=torch.float32):
    """utils/loss_utils.py:45-47 (built in fp32 like the reference)."""
    g = torch.tensor([math.exp(-(x - window_size // 2) ** 2 / float(2 * sigma ** 2))
                      for x in range(window_size)], dtype=torch.float32)
    return (g / g.sum()).to(dtype)


def ssim_map(img1, img2, window_size=11):
    """utils/loss_utils.py:65-85; img [C,H,W] or [B,C,H,W]; zero 'same' padding."""
    squeeze = img1.dim() == 3
    if squeeze:
        img1, img2 = img1[None], img2[None]
    ch = img1.shape[1]
    g = gaussian_window(window_size, 1.5, img1.dtype).to(img1.device)
    w2 = (g[:, None] @ g[None, :])[None, None].expand(ch, 1, window_size, window_size).contiguous()
    pad = window_size // 2
    mu1 = F.conv2d(img1, w2, padding=pad, groups=ch)
    mu2 = F.conv2d(img2, w2, padding=pad, groups=ch)
    mu1_sq, mu2_sq, mu12 = mu1 * mu1, mu2 * mu2, mu1 * mu2
    s1 = F.conv2d(img1 * img1, w2, padding=pad, groups=ch) - mu1_sq
    s2 = F.conv2d(img2 * img2, w2, padding=pad, groups=ch) - mu2_sq
    s12 = F.conv2d(img1 * img2, w2, padding=pad, groups=ch) - mu12
    C1, C2 = 0.01 ** 2, 0.03 ** 2
    m = ((2 * mu12 + C1) * (2 * s12 + C2)) / ((mu1_sq + mu2_sq + C1) * (s1 + s2 + C2))
    return m[0] if squeeze else m


def ssim(img1, img2):
    return ssim_map(img1, img2).mean()


def training_loss(image, gt, lambda_dssim=0.2):
    """train.py:171-176."""
    return (1.0 - lambda_dssim) * l1_loss(image, gt) + lambda_dssim * (1.0 - ssim(image, gt))


# ----------------------------------------------------------------------------------------------
# per-point Adam  (scene/per_point_adam.py:34-98)
# ----------------------------------------------------------------------------------------------
def per_point_adam_step(p, grad, exp_avg, exp_avg_sq, step, lr, beta1=0.9, beta2=0.999,
                        eps=1e-15, weight_decay=0.0, per_point_lr=None):
    """One step on one tensor, in place on p/exp_avg/exp_avg_sq; ``step`` is the value AFTER
    the increment (state['step'] += 1 precedes its use, :59).  Old-style bias correction (:80-81);
    whole-tensor gate grad.norm() > 0 (:66-73); param updated even when the gate is false."""
    if weight_decay != 0:
        grad = grad.add(p, alpha=weight_decay)
    if bool(grad.norm() > 0):
        exp_avg.mul_(beta1).add_(grad, alpha=1 - beta1)
        exp_avg_sq.mul_(beta2).addcmul_(grad, grad, value=1 - beta2)
    bc1 = 1 - beta1 ** step
    bc2 = 1 - beta2 ** step
    denom = exp_avg_sq.sqrt().add_(eps)
    step_size = lr * (bc2 ** 0.5 / bc1)
    if per_point_lr is not None:
        p.add_(-(step_size * per_point_lr) * (exp_avg / denom))
    else:
        p.addcdiv_(exp_avg, denom, value=-step_size)
    return p
