"""Decode the camera-pose gradient chain of the per-Gaussian backward (gs_raster.cu) from the geometry buffer and
restate every stage of it in fp64.

After a backward with the pose fused in, the geometry buffer (`_geom.geom_layout`) holds, for each view v of a batch:

    pose_part [V, nb, 16] f32   CTA b's sum of its 128 Gaussians' contributions pa = [dqc_raw(4), dt(3), dRc(9)]
                                (k_preprocess_bwd / block_pose_partials: a 32-lane xor butterfly, then the 4 warps in
                                order), nb = ceil(P / 128)
    pose_acc  [V, 16]     f32   k_pose_reduce's column sums of pose_part[v]

and dL/dpose[v] = k_pose_finalize(pose_acc[v], pose[v]) (pose_grad_finalize in gs_math.cuh).

The fp64 side starts from the kernel's own decoded moments (`moments`: the 9 fixed-point slots of `dacc`, the 8-slot
tracking layout remapped) so that a difference is the pose chain's and not the blend's.  `pose_rows` maps them with
the constants k_preprocess_bwd applies (dL/dx = -(A Sx + B Sy), dL/dA = -Sxx / 2, ...) onto the outputs of the
oracle's fp64 projection, whose inputs are moved by the pose split into the three leaves the kernel differentiates
against -- the raw quaternion qc that quadmultiply takes, the translation t and the rotation Rc of the normalised
quaternion, one identical row per Gaussian -- so each autograd pass returns every Gaussian's 16-vector row.
`finalize_jacobian` is d[qc, t, Rc(qc / |qc|)] / dpose (autograd, [16, 7]); dL/dpose = acc @ J is linear in acc, so
every stage is compared in the 7-dim dpose space.

Error scales.  Each Gaussian's row is a sum of elementary terms, one per (moment, projected output): the moment times
its constant times d(output)/d(leaves).  `pose_rows` also returns each row's absolute scale, the same sum over the
absolute values of the terms, those through the conic and the pixel position (whose constants are the conic) weighted
by the conic's conditioning kappa = (a c + b^2) / (a c - b^2) of the 2-D covariance it inverts (as in
`_geom.check_records`): the kernel's fp32 det = a c - b^2 carries kappa roundings into every one of them.  A row
computed in fp32 differs from fp64 by a small multiple of eps times that scale.
`abs_jacobian` is the matching absolute map [16, 7] (the quaternion-normalisation projection's two terms counted
separately), so `scale @ abs_jacobian(pose)` bounds the 7-dim size of everything a stage adds up.
"""
import numpy as np
import torch

from oracle import gs_oracle as O

import _blend as BD
import _geom as GM

EPS32 = 2.0 ** -24
PT = GM.PT
# roundings on a term's way into its CTA partial: 5 butterfly levels, then the warps added in order to 0
CTA_DEPTH = 5 + PT // 32 - 1
# pose_grad_finalize in fp32 against finalize64, in units of |acc| @ abs_jacobian(pose): ~4x the largest H100
# measurement (3.7 eps, DESIGN.md section 2, "The pose gradient chain")
FINALIZE_TAU = 16 * EPS32


def gamma(n):
    """The classical bound on n roundings in a chain of fp32 additions: |error| <= gamma(n) * sum |terms|."""
    return n * EPS32 / (1.0 - n * EPS32)


def reduce_depth(nb):
    """Most roundings on any term's way through k_pose_reduce over nb partials: a thread's serial sum, the
    (v0 + v1) + (v2 + v3) combine and the 8 levels of the 256-wide tree."""
    return -(-nb // 256) + 2 + 8


# ---- the device side -----------------------------------------------------------------------------------------------
def decode(geom, P, V=1):
    """The pose chain's state in a geometry buffer (a uint8 device or host tensor) of P Gaussians and V views:
    dict(part [V, nb, 16] f32, acc [V, 16] f32, raw [V, P, 9] int64 (dacc), M [V] (the float dscale holds),
    extent [V, P] f64 (the records' fixed-point extent), tiles [V, P] int64)."""
    lay = GM.geom_layout(P, V)
    g = geom.detach().cpu()
    nb = (max(P, 1) + PT - 1) // PT

    def part(name, n, dt):
        off = lay[name][0]
        return g[off:off + n * torch.empty(0, dtype=dt).element_size()].view(dt)

    rec = part("rec", 12 * V * P, torch.float32).reshape(V, P, 3, 4)
    return dict(part=part("pose_part", V * nb * 16, torch.float32).reshape(V, nb, 16).clone(),
                acc=part("pose_acc", V * 16, torch.float32).reshape(V, 16).clone(),
                raw=part("dacc", V * P * 9, torch.int64).reshape(V, P, 9).clone(),
                M=[float(m) for m in part("dscale", V, torch.float32)],
                extent=rec[:, :, 2, 3].double(),
                tiles=part("tiles", V * P, torch.int32).reshape(V, P).long() & 0xFFFFFFFF)


def moments(dec, v, pose_only=False):
    """View v's decoded moments [P, 9] fp64 as k_preprocess_bwd reads them: zero for a Gaussian without tiles; the
    8-slot tracking layout (slot 5 = dL/db, no S w) moved back to [.., S w = 0, .., dL/db]."""
    val = dec["raw"][v].double() * BD.fix_unit(dec["extent"][v], dec["M"][v])
    val[dec["tiles"][v] == 0] = 0.0
    if pose_only:
        val[:, 8] = val[:, 5]
        val[:, 5] = 0.0
    return val


def reduce_exact(part):
    """k_pose_reduce restated in its exact fp32 order: part [nb, 16] (float32) -> the 16 column sums (float32).
    Thread t adds b = t, t + 1024, ... into v0..v3 (b, b + 256, b + 512, b + 768) while b + 768 < nb, then the rest
    into v0 with stride 256; s[t] = (v0 + v1) + (v2 + v3); a 256-wide tree halves it."""
    part = np.ascontiguousarray(np.asarray(part, dtype=np.float32))
    nb = part.shape[0]
    v = np.zeros((4, 256, 16), np.float32)
    b = np.arange(256)
    while True:
        on = b + 768 < nb
        if not on.any():
            break
        for k in range(4):
            v[k, on] = v[k, on] + part[b[on] + 256 * k]
        b = np.where(on, b + 1024, b)
    while True:
        on = b < nb
        if not on.any():
            break
        v[0, on] = v[0, on] + part[b[on]]
        b = np.where(on, b + 256, b)
    s = (v[0] + v[1]) + (v[2] + v[3])
    o = 128
    while o > 0:
        s[:o] = s[:o] + s[o:2 * o]
        o //= 2
    return s[0]


def cta_sums_fp32(rows):
    """The CTA partials of fp32 rows [P, 16] in k_preprocess_bwd's order (xor butterfly over each warp's 32 lanes,
    then warp 0, 1, 2, 3 added to 0): [nb, 16] float32.  Calibrates the summation's share of the partials' bound."""
    r = np.asarray(rows, dtype=np.float32)
    P = r.shape[0]
    nb = (P + PT - 1) // PT
    x = np.zeros((nb * PT, 16), np.float32)
    x[:P] = r
    x = x.reshape(nb, PT // 32, 32, 16)
    lane = np.arange(32)
    o = 16
    while o > 0:
        x = x + x[:, :, lane ^ o]
        o //= 2
    out = np.zeros((nb, 16), np.float32)
    for w in range(PT // 32):
        out = out + x[:, w, 0]
    return out


# ---- the fp64 side -------------------------------------------------------------------------------------------------
def _R_raw(q):
    """quat_to_R of gs_math.cuh: the rotation formula of a quaternion, without normalising it."""
    r, x, y, z = q.unbind(-1)
    return torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                        2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                        2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], -1)


def finalize_jacobian(pose):
    """J [16, 7] = d[qc, t, Rc(qc / |qc|)] / dpose in fp64: dL/dpose = acc @ J for acc = [dqc_raw(4), dt(3), dRc(9)]."""
    p = torch.as_tensor(pose, dtype=torch.float64).detach().cpu().reshape(7)
    f = lambda x: torch.cat([x[:4], x[4:], O.quad2rotation(x[:4]).reshape(9)])
    return torch.autograd.functional.jacobian(f, p)


def abs_jacobian(pose):
    """The absolute counterpart of finalize_jacobian [16, 7]: identity on qc and t; for Rc,
    (|dR/dqn| + |dR/dqn| |qn| |qn|^T) / |q| -- pose_grad_finalize's dqn and its projection -qn (qn . dqn), each
    counted in absolute value."""
    p = torch.as_tensor(pose, dtype=torch.float64).detach().cpu().reshape(7)
    n = float(p[:4].norm())
    qn = p[:4] / n
    JR = torch.autograd.functional.jacobian(_R_raw, qn).abs()        # [9, 4]
    Ja = torch.zeros(16, 7, dtype=torch.float64)
    Ja[:7, :7] = torch.eye(7, dtype=torch.float64)
    Ja[7:, :4] = (JR + (JR @ qn.abs())[:, None] * qn.abs()[None]) / n
    return Ja


def finalize64(pose, acc):
    """dL/dpose [.., 7] of acc [.., 16] in fp64."""
    return torch.as_tensor(acc).double() @ finalize_jacobian(pose)


def cotangents(val, conic, opacity):
    """k_preprocess_bwd's map of the moments val [P, 9] ([S w dx, S w dy, S w dx^2, S w dx dy, S w dy^2, S w, dL/drgb])
    onto the projected outputs (x, y, A, B, C, r, g, b), each with its absolute scale: -> (cot [P, 8], cot_abs [P, 8])
    and dL/dopacity (which no pose leaf reaches)."""
    Sx, Sy, Sxx, Sxy, Syy, Sw = val[:, :6].unbind(1)
    A, B, C = conic.unbind(1)
    cot = torch.stack([-(A * Sx + B * Sy), -(C * Sy + B * Sx), -0.5 * Sxx, -Sxy, -0.5 * Syy], 1)
    cab = torch.stack([(A * Sx).abs() + (B * Sy).abs(), (C * Sy).abs() + (B * Sx).abs(), 0.5 * Sxx.abs(), Sxy.abs(),
                       0.5 * Syy.abs()], 1)
    dop = torch.where(opacity > 0, Sw / opacity.clamp(min=1e-300), torch.zeros_like(Sw))
    return torch.cat([cot, val[:, 6:9]], 1), torch.cat([cab, val[:, 6:9].abs()], 1), dop


def pose_rows(params, pose, cam, val):
    """Each Gaussian's pose contribution in fp64 from its moments val [P, 9] (`moments`): -> dict(rows [P, 16],
    scale [P, 16] (the rows' absolute scale, see the module doc), has [P] (Gaussians with a moment), proj (the fp64
    projection, detached), flags (`_geom.flags` of the Gaussians whose fp32 branch may legitimately differ: near
    plane, frustum clamp, colour clamp), tview [P, 3]).  params: the scene's raw parameters; pose [7]; cam: the fp64
    identity-view camera (`_geom.camera64`)."""
    p = {k: v.detach().cpu().double() for k, v in params.items()}
    P = p["xyz"].shape[0]
    pose = torch.as_tensor(pose).detach().cpu().double().reshape(7)
    qc = pose[:4].expand(P, 4).clone().requires_grad_(True)
    t = pose[4:].expand(P, 3).clone().requires_grad_(True)
    Rc = O.quad2rotation(pose[:4]).expand(P, 3, 3).clone().requires_grad_(True)
    means = torch.einsum("pij,pj->pi", Rc, p["xyz"]) + t
    rots = O.quadmultiply(qc, p["rotation"])
    shs = torch.cat([p["f_dc"], p["f_rest"]], 1)
    proj = O.project(means, torch.exp(p["scaling"]), rots, torch.sigmoid(p["opacity"]).reshape(-1), shs, cam)
    outs = (proj["xy"][:, 0], proj["xy"][:, 1], proj["conic"][:, 0], proj["conic"][:, 1], proj["conic"][:, 2],
            proj["rgb"][:, 0], proj["rgb"][:, 1], proj["rgb"][:, 2])
    cot, cab, _ = cotangents(val, proj["conic"].detach(), proj["opacity"].detach())
    a, b, c = proj["cov2d"].detach().unbind(1)
    cab[:, :5] *= ((a * c + b * b) / (a * c - b * b).abs().clamp(min=1e-300))[:, None]   # conic conditioning
    has = (val != 0).any(1)
    rows = torch.zeros(P, 16, dtype=torch.float64)
    scale = torch.zeros(P, 16, dtype=torch.float64)
    for k, o in enumerate(outs):
        if not o.requires_grad or not bool((cot[:, k] != 0).any()):      # colour at SH degree 0: no pose leaf
            continue
        g = torch.autograd.grad(o.sum(), (qc, t, Rc), retain_graph=True, allow_unused=True)
        J = torch.cat([torch.zeros(P, s, dtype=torch.float64) if x is None else x.reshape(P, s)
                       for x, s in zip(g, (4, 3, 9))], 1)
        J = torch.where(has[:, None], J, torch.zeros_like(J))             # rows without moments: 0, never NaN
        rows += cot[:, k:k + 1] * J
        scale += cab[:, k:k + 1] * J.abs()
    with torch.no_grad():
        tview = means.detach()
        dirs = tview / tview.norm(dim=1, keepdim=True)
        o = dict({k: (v.detach() if torch.is_tensor(v) else v) for k, v in proj.items()}, tview=tview,
                 mean_norm=p["xyz"].norm(dim=1), raw_rgb=O.eval_sh(cam.sh_degree, shs, dirs) + 0.5,
                 limx=1.3 * cam.tanfovx, limy=1.3 * cam.tanfovy, W=cam.width, H=cam.height)
        f = GM.flags(o)
    flag = f["visibility"] | f["clamp_x"] | f["clamp_y"] | f["clamp_bit"].any(1)
    return dict(rows=rows, scale=scale, has=has, proj=o, flag=flag & has, tview=tview)


def cta_index(P):
    return torch.arange(P) // PT


def per_cta(x, nb):
    """Per-Gaussian rows [P, k] summed per CTA (fp64): [nb, k]."""
    return torch.zeros(nb, x.shape[1], dtype=torch.float64).index_add_(0, cta_index(x.shape[0]), x)
