"""The fp64 restatement of the camera-pose gradient chain (tests/_pose.py) pinned without a GPU: its per-Gaussian rows
add up to the oracle's fp64 autograd pose gradient, its finalize to the host build of pose_grad_finalize, its
k_pose_reduce order and CTA order to their error bounds, and its decoders to the library's layout."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

import _blend as BD
import _geom as GM
import _pose as PG
from oracle import gs_oracle as O
from test_projection_edges import POSES, background, build_scene, camera_of, on_screen, pose_vector

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NBLOCKS = (1, 2, 255, 256, 257, 768, 769, 1023, 1024, 1025, 4099)


def test_batch_layout_matches_library():
    """_geom.geom_layout(P, V, tiles) is gsb_geom_bytes_batch's layout: its total, and the status words where
    gsb_status_device_batch finds them."""
    import __graft_entry__ as G
    G.build()
    import instantsplat_b200 as I
    L = I.lib()
    base = 1 << 20
    for P in (1, 127, 129, 100_000):
        for V in (1, 3, 8):
            for W, H in ((64, 48), (1920, 1080), (4096, 4096)):
                nt = ((W + 15) // 16) * ((H + 15) // 16)
                lay = GM.geom_layout(P, V, nt)
                assert lay["total"] == L.gsb_geom_bytes_batch(P, V, W, H), (P, V, W, H)
                assert L.gsb_status_device_batch(base, P, V) - base == lay["status"][0], (P, V)


def test_tracking_layout_is_remapped():
    """In the 8-slot layout slot 5 carries dL/db: `moments` moves it to slot 8 and zeroes S w, and a Gaussian
    without tiles reads as zero whatever its accumulator holds, as in k_preprocess_bwd."""
    P = 5
    raw = torch.arange(1, 2 * P * 9 + 1, dtype=torch.int64).reshape(2, P, 9)
    dec = dict(raw=raw, M=[1.0, 2.0], extent=torch.full((2, P), 3.0, dtype=torch.float64),
               tiles=torch.tensor([[1, 0, 2, 3, 1], [1, 1, 1, 1, 0]]))
    full, track = PG.moments(dec, 1), PG.moments(dec, 1, pose_only=True)
    unit = BD.fix_unit(dec["extent"][1], 2.0)
    assert torch.equal(full[:4], raw[1, :4].double() * unit[:4]) and int(full[4].count_nonzero()) == 0
    assert torch.equal(track[:, 8], full[:, 5]) and int(track[:, 5].count_nonzero()) == 0
    assert torch.equal(track[:, [0, 1, 2, 3, 4, 6, 7]], full[:, [0, 1, 2, 3, 4, 6, 7]])
    assert int(PG.moments(dec, 0)[1].count_nonzero()) == 0


# ---- the restatement against the oracle's autograd -----------------------------------------------------------------
def cpu_scene(seed, pose, deg, W=80, H=56):
    """Ordinary Gaussians, frustum-clamped ones (|x/z| or |y/z| 1.05-2 x the clamp limit, large enough to reach into
    the frame), near-plane ones (tz 0.205-0.3), and no-tile ones (behind the camera, or far off screen), in front of
    `pose`.  The composed quaternion carries the pose quaternion's norm and R(q) grows like |q|^2, so the sizes are
    divided by it above 1."""
    g = torch.Generator().manual_seed(seed)
    _, _, tx, ty, fx = camera_of(W, H)
    r = lambda *s: torch.rand(*s, generator=g, dtype=torch.float64)
    n = 60
    z = 2.0 + 3.0 * r(n)
    which = torch.randint(0, 2, (n,), generator=g)
    k = (1.05 + 0.95 * r(n)) * torch.where(r(n) < 0.5, -1.0, 1.0).double()
    xz = torch.where(which == 0, k * 1.3 * tx, (2 * r(n) - 1) * 0.8 * tx)
    yz = torch.where(which == 1, k * 1.3 * ty, (2 * r(n) - 1) * 0.8 * ty)
    off = torch.maximum((xz.abs() / tx - 1) * W / 2, (yz.abs() / ty - 1) * H / 2).clamp(min=0)
    clamp = (torch.stack([xz * z, yz * z, z], 1), ((off + 6 + 20 * r(n)) / 2.5 * z / fx)[:, None].expand(n, 3) * 1.0,
             0.3 + 0.5 * r(n))
    zn = 0.205 + 0.095 * r(30)
    near = (on_screen(30, W, H, zn, g, margin=10.0), ((2.0 + 30 * r(30)) * zn / fx)[:, None].expand(30, 3) * 1.0,
            0.02 + 0.1 * r(30))
    dead = (torch.cat([torch.randn(20, 2, generator=g, dtype=torch.float64), -1.0 - r(20, 1)], 1),
            torch.full((20, 3), 0.05, dtype=torch.float64), torch.full((20,), 0.5, dtype=torch.float64))
    zf = torch.full((10,), 3.0, dtype=torch.float64)
    far = (torch.stack([zf * 8 * tx, zf * 0, zf], 1), torch.full((10, 3), 0.01, dtype=torch.float64),
           torch.full((10,), 0.5, dtype=torch.float64))
    shrink = max(1.0, sum(v * v for v in pose[:4]))
    parts = [(c, s / shrink, o) for c, s, o in (background(150, W, H, g), clamp, near, dead, far)]
    return build_scene(parts, W, H, seed=seed + 1, pose=pose, deg=deg)


def oracle_case(sc, deg, seed):
    """O.render_instantsplat in fp64 with the pose as the leaf, dL/dimage random; the restatement's moments on the
    oracle's own records and lists.  -> (pose.grad, moments [P, 9], fp64 camera)."""
    W, H = sc.width, sc.height
    bg = torch.tensor([0.1, 0.2, 0.3], dtype=torch.float64)
    cam = GM.camera64(sc, deg, bg=bg)
    p = {k: v.double() for k, v in sc.params.items()}
    pose = sc.poses[0].double().clone().requires_grad_(True)
    img, _, aux = O.render_instantsplat(p["xyz"], p["rotation"], p["scaling"], p["opacity"], p["f_dc"], p["f_rest"],
                                        pose, cam, return_aux=True)
    dL = torch.randn(3, H, W, generator=torch.Generator().manual_seed(seed), dtype=torch.float64)
    (img * dL).sum().backward()
    pr = aux["proj"]
    rec = dict(x=pr["xy"][:, 0].detach(), y=pr["xy"][:, 1].detach(), A=pr["conic"][:, 0].detach(),
               B=pr["conic"][:, 1].detach(), C=pr["conic"][:, 2].detach(), opacity=pr["opacity"].detach(),
               rgb=pr["rgb"].detach())
    ref = BD.restate(rec, BD.tile_groups((aux["gids"], aux["ranges"]), W, H), W, H, bg, dL, alpha_max=0.99)
    return pose.grad.clone(), ref["mom"], cam


@pytest.mark.parametrize("case", [(30, 1.0, 3), (181, 4.0, 1), (90, 0.25, 0)])
def test_rows_add_up_to_oracle_autograd(case):
    """The per-Gaussian rows of `pose_rows`, from the fp64 moments of the oracle's own blend, finalized with
    `finalize_jacobian`, sum to O.render_instantsplat's fp64 autograd pose gradient to 1e-10 of their absolute
    scale; a Gaussian without moments has a zero row.  The scenes hold frustum-clamped, near-plane and no-tile
    Gaussians and poses with quaternion norms 0.25, 1 and 4 and rotations of 30, 90 and 181 degrees."""
    deg_rot, norm, deg = case
    pose = pose_vector((1, 2, 3), deg_rot, norm, (0.3, -0.2, 0.5))
    sc = cpu_scene(500 + deg_rot, pose, deg)
    grad, mom, cam = oracle_case(sc, deg, 7)
    r = PG.pose_rows(sc.params, sc.poses[0], cam, mom)
    J, Ja = PG.finalize_jacobian(sc.poses[0]), PG.abs_jacobian(sc.poses[0])
    total = r["rows"].sum(0) @ J
    scale = r["scale"].sum(0) @ Ja
    err = (total - grad).abs()
    assert bool((err <= 1e-10 * scale).all()), (err / scale, total, grad)
    assert int(r["rows"][~r["has"]].count_nonzero()) == 0
    t, has = r["tview"], r["has"]
    limx, limy = 1.3 * cam.tanfovx, 1.3 * cam.tanfovy
    clamped = has & (((t[:, 0] / t[:, 2]).abs() > limx) | ((t[:, 1] / t[:, 2]).abs() > limy))
    reached = dict(clamped=int(clamped.sum()), near=int((has & (t[:, 2] < 0.3)).sum()), no_tile=int((~has).sum()),
                   flagged=int(r["flag"].sum()))
    assert reached["clamped"] >= 15 and reached["near"] >= 10 and reached["no_tile"] >= 30, reached


def test_finalize_matches_host_build(tmp_path):
    """pose_grad_finalize compiled for the host (g++, no FMA contraction) against `finalize64` at the pose-table
    quaternions (norms 0.25, 1 and 4; qw = 0 and qw < 0; 30 to 181 degrees), for accumulators with every part
    dominant in turn: within FINALIZE_TAU of the absolute scale |acc| @ abs_jacobian.  Dropping the projection
    -qn (qn . dqn) exceeds that bound a hundredfold."""
    so = str(tmp_path / "libhostmath.so")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-x", "c++", "-ffp-contract=off",
                           os.path.join(ROOT, "tests", "host_math.cpp"), "-o", so])
    lib = ctypes.CDLL(so)
    fp = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_float))
    g = np.random.default_rng(5)
    worst, mutant = 0.0, np.inf
    for pose in POSES:
        p32 = np.array(pose_vector(*pose), np.float32)
        p64 = torch.from_numpy(p32.astype(np.float64))
        J, Ja = PG.finalize_jacobian(p64), PG.abs_jacobian(p64)
        for k in range(12):
            acc = (g.standard_normal(16) * np.exp(g.uniform(-3, 3, 16))).astype(np.float32)
            acc[[0, 4, 7][k % 3]] *= 1e3
            out = np.zeros(7, np.float32)
            lib.host_pose_grad_finalize(fp(p32), fp(acc), fp(out))
            a64 = torch.from_numpy(acc.astype(np.float64))
            ref = a64 @ J
            s = a64.abs() @ Ja
            worst = max(worst, float(((torch.from_numpy(out).double() - ref).abs() / s).max()))
            n = p64[:4].norm()
            qn = p64[:4] / n
            dqn = torch.autograd.functional.jacobian(PG._R_raw, qn).t() @ a64[7:]
            bad = torch.cat([a64[:4] + dqn / n, a64[4:7]])
            mutant = min(mutant, float(((bad - ref).abs() / s).max()))
    assert worst <= PG.FINALIZE_TAU, worst / PG.EPS32
    assert mutant >= 100 * PG.FINALIZE_TAU, mutant / PG.EPS32


# ---- summation orders ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nb", NBLOCKS)
def test_reduce_order_restatement(nb):
    """reduce_exact adds every partial exactly once: integer-valued partials (exact in fp32) give the exact column
    sums; random ones stay within gamma(reduce_depth(nb)) of the fp64 sum of their absolute values."""
    g = np.random.default_rng(nb)
    ints = g.integers(-1024, 1025, (nb, 16)).astype(np.float32)
    assert np.array_equal(PG.reduce_exact(ints), ints.astype(np.float64).sum(0).astype(np.float32))
    x = (g.standard_normal((nb, 16)) * np.exp(g.uniform(-4, 4, (nb, 16)))).astype(np.float32)
    err = np.abs(PG.reduce_exact(x).astype(np.float64) - x.astype(np.float64).sum(0))
    assert (err <= PG.gamma(PG.reduce_depth(nb)) * np.abs(x.astype(np.float64)).sum(0)).all()


def test_cta_order_calibration():
    """The CTA partials of fp32-rounded fp64 rows, summed in k_preprocess_bwd's order by cta_sums_fp32, stay within
    gamma(CTA_DEPTH + 1) of the fp64 sums (the +1: rounding the rows to fp32) in absolute-scale units, and a sum over
    one warp fewer does not."""
    pose = pose_vector((0, 1, 0), 30, 1.0, (0.0, 0.0, 0.0))
    sc = cpu_scene(611, pose, 1)
    _, mom, cam = oracle_case(sc, 1, 3)
    r = PG.pose_rows(sc.params, sc.poses[0], cam, mom)
    nb = (sc.P + PG.PT - 1) // PG.PT
    rows32 = r["rows"].float().numpy()
    got = torch.from_numpy(PG.cta_sums_fp32(rows32)).double()
    ref = PG.per_cta(r["rows"], nb)
    s = PG.per_cta(r["rows"].abs(), nb)
    ratio = float(((got - ref).abs() / s.clamp(min=1e-300)).max())
    assert ratio <= PG.gamma(PG.CTA_DEPTH + 1), ratio / PG.EPS32
    short = torch.from_numpy(rows32.astype(np.float64))
    short[(torch.arange(sc.P) % PG.PT) >= PG.PT - 32] = 0.0
    assert float(((PG.per_cta(short, nb) - ref).abs() / s.clamp(min=1e-300)).max()) > 1e3 * PG.gamma(PG.CTA_DEPTH + 1)
