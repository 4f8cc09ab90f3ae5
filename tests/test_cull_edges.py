"""The lossless culls on the GPU, on scenes built from the populations of tests/test_cull_edges_cpu.py: long needles
at every angle (mask, cooperative and queued big-rect paths), near-plane Gaussians a few thousand pixels long that only
graze the frame, opacities at the 1/255 cutoff and centres just outside a frame with partial last tiles.

  - tile lists: every (Gaussian, tile) pair holding a pixel at which the blend's pair rule passes, evaluated on the
    kernel's own record in fp64 and fp32 (tests/_cull.py), is in the kernel's lists;
  - cull on vs off (rasterizer.EXACT_CULL): image, final_T, each pixel's last contributor, radii and every gradient
    bit for bit.  (The blend's sub-tile cull runs in both arms; tests/test_cull_edges_cpu.py checks it.)
"""
import math

import numpy as np
import pytest
import torch

import _binning as BL
import _blend as BD
import _cull as CU
import _geom as GM
from _parity import DEV, NAMES, REPORT, settings_for
from instantsplat_b200.scenes import Scene, _single_threaded

W, H = 80 * 16 - 3, 45 * 16 - 7                   # partial last tile row and column


@_single_threaded
def cull_scene(seed=5):
    """Camera-space Gaussians (identity pose, SH degree 0): (u, v) pixel centre, z depth, sigma_long / sigma_short in
    pixels, theta the long axis' angle on screen, o opacity."""
    rng = np.random.default_rng(seed)
    fovx = math.radians(60.0)
    fovy = 2.0 * math.atan(math.tan(fovx / 2) * H / W)
    tx_, ty_ = math.tan(fovx / 2), math.tan(fovy / 2)
    fx = W / (2 * tx_)
    near = (0.0, math.pi / 4, math.pi / 2, 3 * math.pi / 4)
    rows = []
    for i in range(240):                            # needles, 3 - 3000 px, every angle
        sl = math.exp(rng.uniform(math.log(3), math.log(3000)))
        th = rng.uniform(0, math.pi) if i % 3 else near[(i // 3) % 4] + rng.uniform(-1e-3, 1e-3)
        rows.append((rng.uniform(0, W), rng.uniform(0, H), rng.uniform(2, 8), sl,
                     sl * math.exp(rng.uniform(math.log(1e-4), math.log(1e-1))), th, rng.uniform(0.05, 1.0)))
    for i in range(24):                             # near-plane, sigma_long 300 - 30000 px along a frame edge, grazing
        off = rng.uniform(60, 180)
        side = i % 4
        u = W - 1 + off if side == 0 else (-off if side == 1 else rng.uniform(0, W))
        v = H - 1 + off if side == 2 else (-off if side == 3 else rng.uniform(0, H))
        th = math.pi / 2 if side < 2 else 0.0
        rows.append((u, v, rng.uniform(0.3, 1.0), math.exp(rng.uniform(math.log(300), math.log(30000))),
                     off / 3.3 * rng.uniform(0.9, 1.1), th + rng.uniform(-0.02, 0.02), rng.uniform(0.3, 1.0)))
    for i in range(80):                             # opacity at the cutoff
        sl = math.exp(rng.uniform(math.log(0.5), math.log(100)))
        rows.append((rng.uniform(0, W), rng.uniform(0, H), rng.uniform(2, 8), sl, sl * rng.uniform(0.01, 1.0),
                     rng.uniform(0, math.pi), rng.uniform(0.999, 1.02) / 255.0))
    for i in range(80):                             # centres just outside the frame
        sl = math.exp(rng.uniform(math.log(1), math.log(100)))
        off = rng.uniform(0.01, 2.0) * sl
        side = i % 4
        u = W - 1 + off if side == 0 else (-off if side == 1 else rng.uniform(0, W))
        v = H - 1 + off if side == 2 else (-off if side == 3 else rng.uniform(0, H))
        rows.append((u, v, rng.uniform(2, 8), sl, sl * rng.uniform(0.01, 1.0), rng.uniform(0, math.pi),
                     rng.uniform(0.05, 1.0)))
    a = np.array(rows, dtype=np.float64)
    u, v, z, sl, ss, th, op = a.T
    P = len(rows)
    xyz = np.stack([((2 * u + 1) / W - 1) * z * tx_, ((2 * v + 1) / H - 1) * z * ty_, z], 1)
    sig = np.stack([sl, np.maximum(ss, 1e-6), np.maximum(ss, 1e-6)], 1) * (z / fx)[:, None]
    rot = np.stack([np.cos(th / 2), 0 * th, 0 * th, np.sin(th / 2)], 1)
    t = lambda x: torch.tensor(x, dtype=torch.float32).contiguous()
    g = torch.Generator().manual_seed(seed)
    params = dict(xyz=t(xyz), f_dc=torch.rand(P, 1, 3, generator=g) - 0.5, f_rest=torch.zeros(P, 15, 3),
                  opacity=t(np.log(op / (1 - op))[:, None]), scaling=t(np.log(sig)), rotation=t(rot))
    return Scene(params, torch.tensor([[1.0, 0, 0, 0, 0, 0, 0]]), W, H, fovx, fovy, 0, name="cull edges")


def run(sc, cull, gt):
    """Forward and backward with the binning cull on or off -> (state, image, grads)."""
    import instantsplat_b200 as I
    import instantsplat_b200.rasterizer as R
    prm = {k: v.to(DEV).clone().requires_grad_(True) for k, v in sc.params.items()}
    pose = sc.poses[0].to(DEV).clone().requires_grad_(True)
    saved = R.EXACT_CULL
    try:
        R.EXACT_CULL = cull
        img, _ = I.rasterize_fused(prm["xyz"], prm["rotation"], prm["scaling"], prm["opacity"], prm["f_dc"],
                                   prm["f_rest"], pose, torch.zeros(sc.P, 3, device=DEV),
                                   settings_for(sc, 0, torch.tensor([0.1, 0.2, 0.3])))
        st = img.grad_fn.st
        (img * gt).sum().backward()
    finally:
        R.EXACT_CULL = saved
    grads = {k: prm[k].grad for k in NAMES}
    grads["pose"] = pose.grad
    return st, img.detach(), grads


def record_of(d, i):
    """The kernel's fp32 record of Gaussian i, in tests/_cull.py's form."""
    f = lambda v: np.float32(float(v))
    e0z, e0w, e1x = (f(d["A"][i] * (-0.5 * GM.LOG2E)), f(d["B"][i] * -GM.LOG2E), f(d["C"][i] * (-0.5 * GM.LOG2E)))
    return dict(A=-e0z, B=f(-0.5 * float(e0w)), C=-e1x, o=f(d["opacity"][i]), qthr=f(d["qthr"][i] * 0.5 * GM.LOG2E),
                e0z=e0z, e0w=e0w, e1x=e1x)


def ref_rect(x, y, rad, gx, gy):
    """project_geometry's tile rect (A.2.7, fp32, C truncation) of the reference."""
    f = np.float32
    c = lambda v, m: int(min(max(int(np.float32(v)), 0), m))
    return (c((f(x) - f(rad)) / f(16), gx), c((f(y) - f(rad)) / f(16), gy),
            c((f(x) + f(rad) + f(15)) / f(16), gx), c((f(y) + f(rad) + f(15)) / f(16), gy))


@pytest.mark.gpu
def test_cull_edges_lists_and_cull_on_off():
    sc = cull_scene()
    gt = torch.rand(3, H, W, generator=torch.Generator().manual_seed(9)).to(DEV)
    st, img, grads = run(sc, True, gt)
    d = GM.decode(st)
    lists = BL.decode(st)
    summ = BL.check_lists(lists)
    gx, gy = lists["gx"], lists["gy"]
    ntiles = gx * gy
    vis = (d["radii"] > 0) & (d["qthr"] >= 0)
    area = (d["rx1"] - d["rx0"]).clamp(min=0) * (d["ry1"] - d["ry0"]).clamp(min=0)
    paths = dict(mask=int((vis & (area > 0) & (area <= 24)).sum()), coop=int((vis & (area > 24) & (area <= 128)).sum()),
                 big=int((vis & (area > 128)).sum()))
    assert d["n_big"] == paths["big"], (d["n_big"], paths)
    for k in ("mask", "coop", "big"):
        assert paths[k] >= 10, paths
    # ---- every contributing (Gaussian, tile) pair is listed
    ids, rng = lists["ids"].cpu(), lists["ranges"].cpu()
    lens = rng[:, 1] - rng[:, 0]
    tile_of = torch.repeat_interleave(torch.arange(ntiles), lens)
    listed = set((ids[:int(lens.sum())] * ntiles + tile_of).tolist())
    must, missing, skipped, cancel = 0, [], 0, 0.0
    must_by_path = dict(mask=0, coop=0, big=0)
    for i in torch.nonzero(vis).reshape(-1).tolist():
        r = record_of(d, i)
        x, y = float(d["x"][i]), float(d["y"][i])
        if not (r["A"] > 0 and r["C"] > 0 and float(r["A"]) * float(r["C"]) > float(r["B"]) ** 2):
            skipped += 1
            continue
        px, py = CU.candidates(x, y, r, W, H)
        ok64, ok32, okf, s, q = CU.pair_rules(x, y, r, px, py)
        sel = ok64 | ok32 | okf
        px, py = px[sel], py[sel]
        if px.size:
            cancel = max(cancel, float((s[sel] / np.maximum(np.abs(q[sel]), 1.0)).max()))
        rx0, ry0, rx1, ry1 = ref_rect(x, y, int(d["radii"][i]), gx, gy)
        tx, ty = px // 16, py // 16
        inr = (tx >= rx0) & (tx < rx1) & (ty >= ry0) & (ty < ry1)
        tiles = np.unique(ty[inr] * gx + tx[inr])
        must += tiles.size
        a = int(area[i])
        must_by_path["mask" if a <= 24 else ("coop" if a <= 128 else "big")] += tiles.size
        missing += [(i, int(t)) for t in tiles if i * ntiles + int(t) not in listed]
    assert must > 2000 and cancel > 1e4, (must, cancel)
    assert all(v > 0 for v in must_by_path.values()), must_by_path
    assert not missing, f"{len(missing)} contributing (Gaussian, tile) pairs missing from the lists, e.g. {missing[:8]}"
    # ---- cull on vs off, bit for bit
    ft_on, nc_on = BD.decode_image(st)
    st_off, img_off, grads_off = run(sc, False, gt)
    ft_off, nc_off = BD.decode_image(st_off)
    lo = BL.decode(st_off)
    R_on, R_off = summ["R"], BL.check_lists(lo)["R"]
    assert torch.equal(img, img_off) and torch.equal(ft_on, ft_off)
    # n_contrib is a list position, which the extra entries of the cull-off lists move: compare whose position it is
    last_on = BD.last_contributor(ids, rng, nc_on, W)
    last_off = BD.last_contributor(lo["ids"].cpu(), lo["ranges"].cpu(), nc_off, W)
    assert torch.equal(last_on, last_off) and torch.equal(nc_on > 0, nc_off > 0)
    assert torch.equal(st.radii, st_off.radii)
    for k in grads:
        assert torch.equal(grads[k], grads_off[k]), k
    REPORT.append(dict(case="cull edges", paths=paths, must_tiles=must, must_by_path=must_by_path,
                       skipped_non_pd=skipped, max_cancel=cancel, R_cull_on=R_on, R_cull_off=R_off))
