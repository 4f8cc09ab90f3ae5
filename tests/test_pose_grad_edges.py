"""The camera-pose gradient chain of the per-Gaussian backward (gs_raster.cu), checked stage by stage against fp64 on
the kernel's own state (tests/_pose.py):

* per-CTA partials: finalize64(pose_part[v, b]) against the fp64 sum of CTA b's per-Gaussian rows, computed from the
  kernel's own decoded moments, within PART_TAU of the CTA's absolute scale; a CTA whose Gaussians have no moments
  holds exactly 0;
* reduction: pose_acc[v] bit for bit against `reduce_exact` (k_pose_reduce's order restated in numpy), and against
  the fp64 sum of the kernel's fp32 partials within gamma(reduce_depth(nb)) of their absolute sum;
* finalize: dL/dpose[v] against finalize64(pose_acc[v]) within FINALIZE_TAU of |acc| @ abs_jacobian;
* end to end: dL/dpose[v] against the fp64 total of the rows, within the bound the three stages compose to.

Every backward instance that feeds the chain is run: the single-view one (full backward, and tracking mode with the
8-slot moments), the view-batched one of training (kViews, one CTA per Gaussian slice for every view) and tracking's
batched pose-only one (grid y = view).  Each case asserts that it reached its regime and records its numbers.
"""
import math

import pytest
import torch

import _geom as GM
import _pose as PG
from _parity import DEV, REPORT
from oracle import gs_oracle as O
from test_projection_edges import POSES, build_scene, camera_of, on_screen, pose_vector

pytestmark = pytest.mark.gpu
# a CTA partial against the fp64 sum of its rows, in units of its absolute scale: the summation's share is at most
# gamma(CTA_DEPTH) (8 eps), the rest is each Gaussian's fp32 backward; ~3.5x the largest H100 measurement (36 eps,
# DESIGN.md section 2, "The pose gradient chain")
PART_TAU = 128 * PG.EPS32
NBLOCKS = (1, 2, 255, 256, 257, 768, 769, 1023, 1024, 1025, 4096 + 3)
RAGGED = 91                       # Gaussians in the last CTA of a boundary case


# ---- driving the library -------------------------------------------------------------------------------------------
def run(sc, poses, deg, mode, make_dL=None, bg=(0.0, 0.0, 0.0)):
    """One forward of sc's Gaussians at poses [V, 7] and (make_dL given: color [V, 3, H, W] -> dL/dimage) one backward.
    mode: "full" (V = 1, every gradient: the single-view k_preprocess_bwd), "pose_only" (V = 1, only dL/dpose: the
    8-slot tracking layout), "views" (gsb_backward_batch: the kViews instance) or "track" (gsb_backward_pose_batch:
    grid y = view).  -> dict(color, dpose [V, 7] and the decoded pose state of `_pose.decode`)."""
    from instantsplat_b200 import frame as F
    from instantsplat_b200._lib import GsbGrads
    V, P, W, H = poses.shape[0], sc.P, sc.width, sc.height
    batched = mode in ("views", "track")
    assert batched or V == 1
    f = lambda t: t.to(DEV).float().contiguous()
    xyz, rot, scl = f(sc.params["xyz"]), f(sc.params["rotation"]), f(sc.params["scaling"])
    opa, fdc, frest = f(sc.params["opacity"].reshape(-1)), f(sc.params["f_dc"].reshape(-1, 3)), f(sc.params["f_rest"])
    M = 1 + frest.shape[1]
    ident = F.IdentityView(W, H, sc.fovx, sc.fovy, torch.tensor(bg), DEV)
    cam = ident.camera(deg, M)
    p7 = f(poses)
    g = F.gaussians(P, xyz, rot, scl, opa, fdc, frest if frest.numel() else None, p7)
    hs = torch.zeros(F.ST_WORDS, dtype=torch.int32).pin_memory()
    fr = F.Frame(DEV, P, W, H, views=V if batched else None)
    fr.preprocess_batch(cam, g, p7, hs) if batched else fr.preprocess(cam, g, hs)
    torch.cuda.synchronize()
    fr.alloc_binning(F.capacity(F.read_R(hs), 1.0))
    fr.render_batch(cam) if batched else fr.render(cam)
    color = fr.color.reshape(V, 3, H, W)
    if make_dL is None:
        torch.cuda.synchronize()
        return dict(color=color.clone())
    dL = make_dL(color).float().contiguous()
    dpose = torch.zeros(V, 7, device=DEV)
    gr, keep = GsbGrads(), []
    if mode in ("full", "views"):
        for field, shape in (("dL_dmeans3D", (P, 3)), ("dL_dmeans2D", (P, 3)), ("dL_dscales", (P, 3)),
                             ("dL_drotations", (P, 4)), ("dL_dopacities", (P,)), ("dL_dsh_dc", (P, 3)),
                             ("dL_dsh_rest", (P, M - 1, 3))):
            keep.append(torch.zeros(shape, device=DEV))
            setattr(gr, field, keep[-1].data_ptr())
    if mode == "track":
        fr.backward_pose_batch(cam, g, p7, dL, dpose)
    elif mode == "views":
        fr.backward_batch(cam, g, p7, dL, gr, dpose)
    else:
        gr.dL_dpose = dpose.data_ptr()
        fr.backward(cam, g, dL[0], gr)
    torch.cuda.synchronize()
    assert F.u32(fr.status[F.ST_OVERFLOW]) == 0
    out = PG.decode(fr.geom, P, V)
    out.update(color=color.clone(), dpose=dpose.cpu())
    return out


def signed_dL(seed):
    def make(color):
        g = torch.Generator().manual_seed(seed)
        return (2 * torch.rand(*color.shape, generator=g) - 1).to(DEV)
    return make


# ---- the stage checks ----------------------------------------------------------------------------------------------
def check_chain(name, sc, deg, poses, mode, out, pose_only=False):
    """Every stage of every view of one run against fp64; asserts and records.  -> (record, per-view fp64 state)."""
    V, P = poses.shape[0], sc.P
    nb = (P + PG.PT - 1) // PG.PT
    cam = GM.camera64(sc, deg)
    rec = dict(case=f"pose chain: {name}", mode=mode, P=P, V=V, nblocks=nb, width=sc.width, height=sc.height,
               views=[])
    fp = []
    for v in range(V):
        val = PG.moments(out, v, pose_only)
        if pose_only:
            assert int(out["raw"][v][:, 8].count_nonzero()) == 0, "tracking mode did not use the 8-slot layout"
        r = PG.pose_rows(sc.params, poses[v], cam, val)
        J, Ja = PG.finalize_jacobian(poses[v]), PG.abs_jacobian(poses[v])
        part, acc, dpose = out["part"][v], out["acc"][v], out["dpose"][v].double()
        part64 = part.double()
        # per-CTA partials (CTAs holding a Gaussian whose fp32 branch may legitimately differ are not compared)
        ref = PG.per_cta(r["rows"], nb)
        s16 = PG.per_cta(r["scale"], nb)
        s7 = s16 @ Ja
        live = s16.abs().sum(1) > 0
        exempt = torch.zeros(nb, dtype=torch.bool).index_fill_(0, PG.cta_index(P)[r["flag"]].unique(), True) \
            if bool(r["flag"].any()) else torch.zeros(nb, dtype=torch.bool)
        e_part = ((part64 - ref) @ J).abs()
        sel = live & ~exempt
        ratio = e_part[sel] / s7[sel].clamp(min=1e-300)
        part_worst = float(ratio.max()) if ratio.numel() else 0.0
        dead = int(part[~live].count_nonzero())
        # reduction: exact order, and its fp64 bound
        exact = torch.from_numpy(PG.reduce_exact(part.numpy()))
        bits_equal = torch.equal(exact.view(torch.int32), acc.view(torch.int32))
        red_bound = PG.gamma(PG.reduce_depth(nb)) * part64.abs().sum(0)
        e_red = (acc.double() - part64.sum(0)).abs()
        red_worst = float((e_red / red_bound.clamp(min=1e-300)).max())
        # finalize
        s_fin = acc.double().abs() @ Ja
        e_fin = (dpose - acc.double() @ J).abs()
        fin_worst = float((e_fin / s_fin.clamp(min=1e-300)).max())
        # end to end
        t7 = r["rows"] @ J
        total = t7.sum(0)
        b_e2e = PART_TAU * (s16.sum(0) @ Ja) + red_bound @ Ja + PG.FINALIZE_TAU * s_fin \
            + 2.0 * (r["scale"][r["flag"]].sum(0) @ Ja)
        e_e2e = (dpose - total).abs()
        e2e_worst = float((e_e2e / b_e2e.clamp(min=1e-300)).max())
        cancel = (t7.abs().sum(0) / total.abs().clamp(min=1e-300))
        rv = dict(view=v, live_ctas=int(live.sum()), dead_ctas=int((~live).sum()), exempt_ctas=int(exempt.sum()),
                  flagged=int(r["flag"].sum()), with_moments=int(r["has"].sum()),
                  part_err_eps=part_worst / PG.EPS32, reduce_bits_equal=bits_equal, reduce_err_over_bound=red_worst,
                  finalize_err_eps=fin_worst / PG.EPS32, e2e_err_over_bound=e2e_worst,
                  e2e_rel=float((e_e2e / total.abs().clamp(min=1e-300)).max()),
                  cancellation=[float(c) for c in cancel], dpose=[float(x) for x in dpose])
        rv["_dead_nonzero"], rv["_acc"], rv["_exact"] = dead, acc.tolist(), exact.tolist()
        rec["views"].append(rv)
        fp.append(dict(rows=r, ref=ref, s7=s7, J=J, live=live, exempt=exempt, total=total, tview=r["tview"]))
    REPORT.append(rec)
    rec["part_err_eps_max"] = max(rv["part_err_eps"] for rv in rec["views"])
    for rv in rec["views"]:
        v, dead, acc, exact = rv["view"], rv.pop("_dead_nonzero"), rv.pop("_acc"), rv.pop("_exact")
        assert dead == 0, f"{name} view {v}: CTAs without moments hold a non-zero partial"
        assert rv["part_err_eps"] * PG.EPS32 <= PART_TAU, f"{name} view {v}: CTA partial over its bound: {rv}"
        assert rv["reduce_bits_equal"], f"{name} view {v}: pose_acc differs from k_pose_reduce's order: {acc} vs {exact}"
        assert rv["reduce_err_over_bound"] <= 1.0, f"{name} view {v}: reduction error over its bound: {rv}"
        assert rv["finalize_err_eps"] * PG.EPS32 <= PG.FINALIZE_TAU, f"{name} view {v}: finalize over its bound: {rv}"
        assert rv["e2e_err_over_bound"] <= 1.0, f"{name} view {v}: end-to-end error over the composed bound: {rv}"
    return rec, fp


# ---- scenes ----------------------------------------------------------------------------------------------------------
def cloud(n, W, H, g, z0=2.0, z1=6.0, s0=0.8, s1=3.0, margin=4.0, op0=0.2, op1=0.9):
    """n Gaussians over a W x H frame: z in [z0, z1], sigma s0-s1 px, opacity op0-op1."""
    fx = camera_of(W, H)[4]
    z = z0 + (z1 - z0) * torch.rand(n, generator=g, dtype=torch.float64)
    s_px = s0 + (s1 - s0) * torch.rand(n, generator=g, dtype=torch.float64)
    sig = (s_px * z / fx)[:, None] * (0.7 + 0.6 * torch.rand(n, 3, generator=g, dtype=torch.float64))
    return on_screen(n, W, H, z, g, margin=margin), sig, op0 + (op1 - op0) * torch.rand(n, generator=g, dtype=torch.float64)


def with_dead(part, g, frac=0.1, whole=()):
    """Move a fraction of a part's Gaussians, and every Gaussian of the index ranges in `whole`, behind the camera."""
    pc, sig, op = part
    pc = pc.clone()
    n = pc.shape[0]
    m = torch.rand(n, generator=g) < frac
    for a, b in whole:
        m[a:min(b, n)] = True
    pc[m, 2] = -1.0 - torch.rand(int(m.sum()), generator=g, dtype=torch.float64)
    return pc, sig, op


def pose_of(deg, t=(0.2, -0.1, 0.3), axis=(1, 2, 3)):
    return pose_vector(axis, deg, 1.0, t)


# ---- populations -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nb", NBLOCKS)
def test_reduction_loop_boundaries(nb):
    """P = (nb - 1) * 128 + 91 Gaussians (a ragged last CTA) over a 4:3 frame of about 2 pixels per Gaussian (at least
    256 x 192), translucent enough that most CTAs hold a contributing Gaussian; 10 % of them and every Gaussian of
    CTA 1 behind the camera: nblocks on both sides of k_pose_reduce's one stride (256), the first run of its
    4-way loop (768 / 769), one and two of its iterations (1024 / 1025) and 4099.  Single-view full backward."""
    P = (nb - 1) * PG.PT + RAGGED
    W = max(256, 16 * round(math.sqrt(8 / 3 * P) / 16))               # about two pixels per Gaussian
    H = W * 3 // 4
    g = torch.Generator().manual_seed(700 + nb)
    sc = build_scene([with_dead(cloud(P, W, H, g, op0=0.05, op1=0.4), g, whole=((PG.PT, 2 * PG.PT),))], W, H,
                     seed=701 + nb, pose=pose_of(20), deg=1)
    out = run(sc, sc.poses, 1, "full", signed_dL(nb))
    rec, fp = check_chain(f"nblocks {nb}", sc, 1, sc.poses, "full", out)
    rv = rec["views"][0]
    assert rec["nblocks"] == nb and P % PG.PT == RAGGED % PG.PT
    assert rv["live_ctas"] >= 0.9 * (nb - 1) and (nb < 3 or rv["dead_ctas"] >= 1), rv
    rec["reached"] = dict(unrolled_loop=nb > 768, two_unrolled_iterations=nb > 1792, tail_after_unrolled=nb % 1024)


def clamp_near_scene(W=192, H=128, seed=811):
    """600 faint frustum-clamped Gaussians (|x/z| or |y/z| 1-3 x the clamp limit, sized to reach into the frame),
    400 faint near-plane ones (tz 0.201-0.3, and 100 at 0.195 / 0.199 behind the plane) and a background layer with
    20 % of it, and all of CTAs 8 and 9, behind the camera, in front of a 181-degree pose."""
    g = torch.Generator().manual_seed(seed)
    _, _, tx, ty, fx = camera_of(W, H)
    r = lambda *s: torch.rand(*s, generator=g, dtype=torch.float64)
    n = 600
    z = 2.0 + 4.0 * r(n)
    which = torch.randint(0, 3, (n,), generator=g)
    sgn = lambda: torch.where(r(n) < 0.5, -1.0, 1.0).double()
    kx, ky = (1.0 + 2.0 * r(n)) * 1.3 * tx * sgn(), (1.0 + 2.0 * r(n)) * 1.3 * ty * sgn()
    xz = torch.where(which == 1, (2 * r(n) - 1) * 0.8 * tx, kx)
    yz = torch.where(which == 0, (2 * r(n) - 1) * 0.8 * ty, ky)
    off = torch.maximum((xz.abs() / tx - 1) * W / 2, (yz.abs() / ty - 1) * H / 2).clamp(min=0)
    clamp = (torch.stack([xz * z, yz * z, z], 1), ((off + 8 + 32 * r(n)) / 2.5 * z / fx)[:, None].expand(n, 3) * 1.0,
             0.02 + 0.04 * r(n))
    m = 400
    zn = torch.cat([torch.tensor([0.195, 0.199], dtype=torch.float64).repeat(50), 0.201 + 0.099 * r(m - 100)])
    near = (on_screen(m, W, H, zn, g, margin=20.0),
            (torch.exp(math.log(2.0) + (math.log(60.0) - math.log(2.0)) * r(m)) * zn / fx)[:, None].expand(m, 3) * 1.0,
            0.01 + 0.04 * r(m))
    parts = [clamp, near, with_dead(cloud(3000, W, H, g, z0=3.0, z1=8.0), g, frac=0.2, whole=((24, 280),))]
    return build_scene(parts, W, H, seed=seed + 1, pose=pose_vector((1, -1, 2), 181, 1.0, (-0.3, 0.2, 0.1)), deg=2)


def clamp_near_reached(tview, has, tanfovx, tanfovy):
    t = tview
    return dict(clamped_x=int((has & ((t[:, 0] / t[:, 2]).abs() > 1.3 * tanfovx)).sum()),
                clamped_y=int((has & ((t[:, 1] / t[:, 2]).abs() > 1.3 * tanfovy)).sum()),
                near_below_0_25=int((has & (t[:, 2] < 0.25)).sum()), behind_near_plane=int((t[:, 2] <= 0.2).sum()),
                no_moments=int((~has).sum()))


@pytest.mark.parametrize("mode", ["full", "pose_only"])
def test_clamp_and_near_plane(mode):
    """clamp_near_scene in the full backward and in tracking mode: the zeroed dtx / dty of the frustum clamp and the
    1 / tz^2 of the near plane in the Gaussians' rows, and exactly-zero partials where nothing contributes."""
    sc = clamp_near_scene()
    out = run(sc, sc.poses, 2, mode, signed_dL(813))
    rec, fp = check_chain(f"clamp and near plane ({mode})", sc, 2, sc.poses, mode, out, pose_only=mode == "pose_only")
    cam = GM.camera64(sc, 2)
    rec["reached"] = reached = dict(clamp_near_reached(fp[0]["tview"], fp[0]["rows"]["has"], cam.tanfovx,
                                                       cam.tanfovy), dead_ctas=rec["views"][0]["dead_ctas"])
    assert reached["clamped_x"] >= 100 and reached["clamped_y"] >= 100 and reached["near_below_0_25"] >= 100, reached
    assert reached["behind_near_plane"] >= 300 and reached["no_moments"] >= 1000 and reached["dead_ctas"] >= 2, reached


@pytest.mark.parametrize("mode", ["full", "pose_only"])
def test_cancellation_at_1m(mode):
    """1M Gaussians over a 1920 x 1080 frame (nblocks 7813).  The target is the kernel's own render at the true
    pose; the backward is of the L1 sign gradient at the pose rolled by 0.05 degrees about the optical axis, where
    the per-Gaussian terms are large, signed and nearly cancel: the records carry sum |t| / |sum t| per component,
    and every bound is relative to the absolute sums."""
    W, H, n = 1920, 1080, 1_000_000
    g = torch.Generator().manual_seed(901)
    pose = pose_vector((0.3, -0.2, 1.0), 15, 1.0, (0.1, -0.2, 0.4))
    sc = build_scene([cloud(n, W, H, g, z0=2.0, z1=10.0, s0=0.6, s1=4.0, margin=8.0, op0=0.05, op1=0.3)], W, H,
                     seed=902, pose=pose, deg=3)
    target = run(sc, sc.poses, 3, "full")["color"]
    roll = torch.tensor(pose_vector((0, 0, 1), 0.05, 1.0, (0.0, 0.0, 0.0)), dtype=torch.float64)
    q = O.quadmultiply(roll[:4], sc.poses[0].double()[:4])
    R = O.quad2rotation(roll[:4])
    moved = torch.cat([q, R @ sc.poses[0].double()[4:]]).float()[None]
    N = 3 * H * W
    out = run(sc, moved, 3, mode, lambda c: torch.sign(c - target) / N)
    rec, fp = check_chain(f"cancellation at 1M ({mode})", sc, 3, moved, mode, out, pose_only=mode == "pose_only")
    c = rec["views"][0]["cancellation"]
    rec["reached"] = dict(cancellation_max=max(c), pixels_moved=int((out["color"] != target).sum()))
    assert rec["nblocks"] == 7813 and max(c) >= 100, rec["views"][0]


def view_poses(V, seed):
    """V distinct poses a few degrees and centimetres apart around a 20-degree base pose."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for v in range(V):
        ax = tuple((torch.randn(3, generator=g)).tolist())
        out.append(pose_vector(ax, 20 + 4 * v, 1.0, tuple((0.05 * torch.randn(3, generator=g)).tolist())))
    return torch.tensor(out, dtype=torch.float32)


@pytest.mark.parametrize("mode", ["views", "track"])
@pytest.mark.parametrize("V", [3, 8])
def test_view_rows(mode, V):
    """V views of one cloud at distinct poses through gsb_backward_batch (the kViews instance: one CTA per Gaussian
    slice for all views, pose_part row (v, CTA) from block_pose_partials) and through tracking's gsb_backward_pose_batch
    (grid y = view, 8-slot moments): each view's partials match its own view's fp64 rows, and every other view's
    rows miss them by far more than the bound, so a row written to the wrong view cannot pass."""
    W, H = 160, 120
    g = torch.Generator().manual_seed(1000 + V)
    poses = view_poses(V, 1010 + V)
    P = 40 * PG.PT + 57
    sc = build_scene([with_dead(cloud(P, W, H, g, z0=2.5, z1=6.0), g, frac=0.05)], W, H, seed=1020 + V,
                     pose=tuple(poses[0].tolist()), deg=1)
    out = run(sc, poses, 1, mode, signed_dL(1030 + V))
    rec, fp = check_chain(f"view rows, V {V}", sc, 1, poses, mode, out, pose_only=mode == "track")
    cross = []
    for v in range(V):
        part64 = out["part"][v].double()
        for w in range(V):
            if w == v:
                continue
            s = fp[w]["live"] & fp[v]["live"]
            e = ((part64 - fp[w]["ref"]) @ fp[w]["J"]).abs()[s] / fp[w]["s7"][s].clamp(min=1e-300)
            cross.append(float(e.max()))
    rec["reached"] = dict(views=V, distinct_poses=int(torch.unique(poses, dim=0).shape[0]),
                          other_view_err_min_eps=min(cross) / PG.EPS32)
    assert rec["reached"]["distinct_poses"] == V >= 3
    assert min(cross) >= 100 * PART_TAU, rec["reached"]


def test_finalize_pose_table():
    """The pose-table poses of test_projection_edges (rotations of 30, 90, 180 and 181 degrees, quaternion norms
    0.25, 1 and 4, qw = 0 and qw < 0), 300 Gaussians each at 64 x 48: the finalize at every pose, and the whole chain."""
    W, H = 64, 48
    worst = 0.0
    for k, (axis, deg, norm, t) in enumerate(POSES):
        g = torch.Generator().manual_seed(1100 + k)
        n = 300
        pc, sig, op = cloud(n, W, H, g, s0=1.0, s1=5.0, margin=8.0)
        pose = pose_vector(axis, deg, norm, t)
        sc = build_scene([(pc, sig / max(1.0, norm * norm), op)], W, H, seed=1150 + k, pose=pose, deg=3)
        out = run(sc, sc.poses, 3, "full", signed_dL(1200 + k))
        rec, _ = check_chain(f"pose table: {deg} deg about {axis}, |q| {norm}", sc, 3, sc.poses, "full", out)
        worst = max(worst, rec["views"][0]["finalize_err_eps"])
    qw = [pose_vector(*p)[0] for p in POSES]
    assert 0.0 in qw and min(qw) < 0
    REPORT.append(dict(case="pose chain: pose table, finalize", finalize_err_eps_max=worst))
