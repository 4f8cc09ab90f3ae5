"""Mip-Splatting filters on the H100 (DESIGN.md section 4.7): the off path, full-frame parity with the fp64 restatement
of tests/_mip.py, the filter-size kernel, tracking mode and the trainer."""
import ctypes
import math

import pytest
import torch

from oracle import gs_oracle as O

import _mip as MIP
from _parity import DEV, GRAD_TOL, ROW_TOL, assert_image, image_stats, rel_err, row_err, settings_for

pytestmark = pytest.mark.gpu

NAMES = ("xyz", "rotation", "scaling", "opacity", "f_dc", "f_rest")


def _scene(P=3000, W=128, H=96, seed=61, log_s=math.log(0.03)):
    from instantsplat_b200.scenes import random_scene
    sc = random_scene(P, W, H, seed=seed, sh_degree=3)
    g = torch.Generator().manual_seed(seed + 1)
    sc.params["scaling"] = log_s + 0.8 * torch.randn(P, 3, generator=g)
    sc.params["scaling"][:100] = math.log(1e-4) + 0.1 * torch.randn(100, 3, generator=g)   # far below a pixel
    # poses of three views; the first one is rendered
    extra = torch.tensor([[0.99, 0.02, -0.05, 0.01, 0.1, -0.05, 0.3], [0.98, -0.04, 0.03, 0.02, -0.2, 0.1, -0.2]])
    sc.poses = torch.cat([sc.poses, extra])
    return sc


def _filter3d(sc):
    return MIP.filter3d_ref(sc.params["xyz"], sc.poses, sc.width, sc.height, math.tan(sc.fovx / 2),
                            math.tan(sc.fovy / 2)).float()


def test_off_path_ex_with_null_equals_old_entry_points():
    import instantsplat_b200 as I
    from instantsplat_b200 import _lib
    from instantsplat_b200.frame import Frame, IdentityView, gaussians
    sc = _scene(seed=62)
    L = I.lib()
    prm = {k: v.to(DEV).contiguous() for k, v in sc.params.items()}
    pose = sc.poses[0].to(DEV).contiguous()
    iv = IdentityView(sc.width, sc.height, sc.fovx, sc.fovy, torch.tensor([0.1, 0.2, 0.3]), DEV)
    cam = iv.camera(3, 16)
    g = gaussians(sc.P, prm["xyz"], prm["rotation"], prm["scaling"], prm["opacity"], prm["f_dc"], prm["f_rest"], pose)
    w = torch.rand(3, sc.height, sc.width, generator=torch.Generator().manual_seed(3)).to(DEV)
    out = []
    for old in (False, True):
        fr = Frame(DEV, sc.P, sc.width, sc.height)
        fr.alloc_binning(4_000_000)
        if old:
            _lib.check(L.gsb_preprocess(ctypes.byref(cam), ctypes.byref(g), fr.geom.data_ptr(), fr.geom.numel(),
                                        fr.radii.data_ptr(), None, _lib.stream_ptr()), "gsb_preprocess")
        else:
            fr.preprocess(cam, g, None, None)
        fr.render(cam)
        grads = {k: torch.zeros_like(v) for k, v in prm.items()}
        grads["pose"] = torch.zeros(7, device=DEV)
        gr = _lib.GsbGrads()
        for f, k in (("dL_dmeans3D", "xyz"), ("dL_dscales", "scaling"), ("dL_drotations", "rotation"),
                     ("dL_dopacities", "opacity"), ("dL_dsh_dc", "f_dc"), ("dL_dsh_rest", "f_rest"),
                     ("dL_dpose", "pose")):
            setattr(gr, f, grads[k].data_ptr())
        if old:
            _lib.check(L.gsb_backward(ctypes.byref(cam), ctypes.byref(g), fr.geom.data_ptr(), fr.binning.data_ptr(),
                                      fr.cap, fr.image.data_ptr(), w.data_ptr(), ctypes.byref(gr), _lib.stream_ptr()),
                       "gsb_backward")
        else:
            fr.backward(cam, g, w, gr, None)
        torch.cuda.synchronize()
        out.append((fr.color.clone(), fr.radii.clone(), grads))
    (ia, ra, ga), (ib, rb, gb) = out
    assert torch.equal(ia, ib) and torch.equal(ra, rb)
    for k in ga:
        assert torch.equal(ga[k], gb[k]), k


def _compare(name, sc, view, kappa, f3d, bg=torch.tensor([0.1, 0.2, 0.3]), seed=11):
    """rasterize_fused with the filters against render_mip in fp64, full frame, random weights."""
    import instantsplat_b200 as I
    cam64 = O.Camera.instantsplat(sc.width, sc.height, sc.fovx, sc.fovy, bg=bg, sh_degree=3, dtype=torch.float64)
    cam32 = O.Camera.instantsplat(sc.width, sc.height, sc.fovx, sc.fovy, bg=bg, sh_degree=3)
    with torch.no_grad():       # tile lists of the fp32 projection (rect bounds and depth order as an fp32 kernel bins)
        p = sc.params
        means, rots = O.pose_pretransform(p["xyz"], p["rotation"], sc.poses[view])
        s, o = torch.exp(p["scaling"]), torch.sigmoid(p["opacity"]).reshape(-1)
        if f3d is not None:
            s, o = MIP.apply_filter3d(s, o, f3d)
        pr32 = MIP.project_mip(means, s, rots, o, torch.cat([p["f_dc"], p["f_rest"]], 1), cam32, kappa)
        lists = O.build_tile_lists(pr32)
    po = {k: v.double().clone().requires_grad_(True) for k, v in sc.params.items()}
    pose_o = sc.poses[view].double().clone().requires_grad_(True)
    img_o, radii_o, aux = MIP.render_mip(po["xyz"], po["rotation"], po["scaling"], po["opacity"], po["f_dc"],
                                         po["f_rest"], pose_o, cam64, kappa, None if f3d is None else f3d.double(),
                                         return_aux=True, lists=lists)
    pc = {k: v.to(DEV).clone().requires_grad_(True) for k, v in sc.params.items()}
    pose_c = sc.poses[view].to(DEV).clone().requires_grad_(True)
    rs = settings_for(sc, 3, bg)
    rs = I.GaussianRasterizationSettings(*rs, kernel_size=kappa)
    img_c, radii_c = I.rasterize_fused(pc["xyz"], pc["rotation"], pc["scaling"], pc["opacity"], pc["f_dc"],
                                       pc["f_rest"], pose_c, torch.zeros(sc.P, 3, device=DEV), rs,
                                       None if f3d is None else f3d.to(DEV))
    amb = aux["ambiguous"]
    st = image_stats(img_c, img_o.detach(), amb)
    assert_image(st, name)
    assert float((radii_c.cpu() != radii_o).float().mean()) < 2e-3
    w = torch.rand(3, sc.height, sc.width, generator=torch.Generator().manual_seed(seed)) * (~amb)[None]
    (img_o * w.double()).sum().backward()
    (img_c * w.to(DEV)).sum().backward()
    g_o = {k: po[k].grad for k in po}
    g_c = {k: pc[k].grad for k in pc}
    g_o["pose"], g_c["pose"] = pose_o.grad, pose_c.grad
    ge = {k: rel_err(g_c[k], g_o[k]) for k in g_o}
    rows = {k: row_err(g_c[k], g_o[k])["p999"] for k in NAMES}
    assert max(ge.values()) < GRAD_TOL, (name, ge)
    assert max(rows.values()) <= ROW_TOL, (name, rows)
    return aux["proj"], st, ge, rows


def test_filters_full_frame_parity_populations():
    sc = _scene(P=3000, seed=63, log_s=math.log(0.004))          # many sub-pixel Gaussians, some large ones
    f3d = _filter3d(sc)
    s = torch.exp(sc.params["scaling"])
    # both sides of the 3D filter are populated: every scale below f, and some scale above it
    assert int((s < f3d[:, None]).all(1).sum()) > 100 and int((s > f3d[:, None]).any(1).sum()) > 100
    for view in range(3):
        proj, _, _, _ = _compare(f"mip view {view}", sc, view, 0.1, f3d)
        assert float(proj["h2"].detach()[proj["visible"]].min()) < 0.9
    # the 2D filter alone reaches the floor of h2 on the tiny Gaussians; the 3D filter alone; strength 0.3
    proj, _, _, _ = _compare("mip2d only", sc, 0, 0.1, None)
    vis = proj["visible"]
    assert int((proj["h2_clamp"] & vis).sum()) > 0 and int((~proj["h2_clamp"] & vis).sum()) > 100
    _compare("mip3d only", sc, 1, None, f3d)
    _compare("mip2d 0.3", sc, 2, 0.3, f3d)


def test_b2_boundary_kernel_size_packed_sh_and_precomputed():
    import instantsplat_b200 as I
    sc = _scene(P=2000, seed=64, log_s=math.log(0.006))
    bg = torch.tensor([0.2, 0.1, 0.0])
    p = sc.params
    means, rots = O.pose_pretransform(p["xyz"], p["rotation"], sc.poses[0])
    means, rots = means.contiguous(), rots.contiguous()
    s, o = torch.exp(p["scaling"]), torch.sigmoid(p["opacity"])
    shs = torch.cat([p["f_dc"], p["f_rest"]], 1)
    cam64 = O.Camera.instantsplat(sc.width, sc.height, sc.fovx, sc.fovy, bg=bg, sh_degree=3, dtype=torch.float64)
    cam32 = O.Camera.instantsplat(sc.width, sc.height, sc.fovx, sc.fovy, bg=bg, sh_degree=3)
    cols = torch.rand(sc.P, 3, generator=torch.Generator().manual_seed(2))
    r, x, y, z = rots.unbind(-1)
    R = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y), 2 * (x * y + r * z),
                     1 - 2 * (x * x + z * z), 2 * (y * z - r * x), 2 * (x * z - r * y), 2 * (y * z + r * x),
                     1 - 2 * (x * x + y * y)], -1).reshape(-1, 3, 3)
    M = R * s[:, None, :]
    S = M @ M.transpose(1, 2)
    cov6 = torch.stack([S[:, 0, 0], S[:, 0, 1], S[:, 0, 2], S[:, 1, 1], S[:, 1, 2], S[:, 2, 2]], -1)
    for case in ("sh", "precomp"):
        kw32 = dict(colors_precomp=cols, cov3D_precomp=cov6) if case == "precomp" else {}
        with torch.no_grad():
            lists = O.build_tile_lists(MIP.project_mip(means, s, rots, o, shs, cam32, 0.1, **kw32))
        leaves = [t.double().clone().requires_grad_(True) for t in (means, s, rots, o, shs, cols, cov6)]
        m_o, s_o, r_o, o_o, sh_o, c_o, v_o = leaves
        kw64 = dict(colors_precomp=c_o, cov3D_precomp=v_o) if case == "precomp" else {}
        pr = MIP.project_mip(m_o, s_o, r_o, o_o, sh_o, cam64, 0.1, **kw64)
        img_o, aux = O.blend(pr, cam64, return_aux=True, lists=lists)
        lc = [t.to(DEV).clone().requires_grad_(True) for t in (means, s, rots, o, shs, cols, cov6)]
        m_c, s_c, r_c, o_c, sh_c, c_c, v_c = lc
        rs = I.GaussianRasterizationSettings(*settings_for(sc, 3, bg), kernel_size=0.1)
        rast = I.GaussianRasterizer(rs)
        if case == "precomp":
            img_c, _ = rast(means3D=m_c, means2D=torch.zeros_like(m_c), opacities=o_c, colors_precomp=c_c,
                            cov3D_precomp=v_c)
        else:
            img_c, _ = rast(means3D=m_c, means2D=torch.zeros_like(m_c), opacities=o_c, shs=sh_c, scales=s_c,
                            rotations=r_c)
        amb = aux["ambiguous"]
        assert_image(image_stats(img_c, img_o.detach(), amb), f"b2 {case}")
        w = torch.rand(3, sc.height, sc.width, generator=torch.Generator().manual_seed(4)) * (~amb)[None]
        (img_o * w.double()).sum().backward()
        (img_c * w.to(DEV)).sum().backward()
        pairs = [(m_c, m_o), (o_c, o_o)] + ([(c_c, c_o), (v_c, v_o)] if case == "precomp" else
                                             [(s_c, s_o), (r_c, r_o), (sh_c, sh_o)])
        for a, b in pairs:
            assert rel_err(a.grad, b.grad) < GRAD_TOL, case


def test_filter3d_kernel_matches_restatement():
    from instantsplat_b200.frame import mip_filter3d
    g = torch.Generator().manual_seed(5)
    P, V, W, H = 200_000, 12, 1920, 1080
    xyz = torch.rand(P, 3, generator=g) * torch.tensor([8.0, 6.0, 10.0]) - torch.tensor([4.0, 3.0, 2.0])
    poses = torch.cat([torch.tensor([1.0, 0, 0, 0]) + 0.05 * torch.randn(V, 4, generator=g),
                       0.3 * torch.randn(V, 3, generator=g)], 1)
    t = math.tan(math.radians(60.0) / 2)
    ref, margin = MIP.filter3d_ref(xyz, poses, W, H, t, t * H / W, return_margin=True)
    out = mip_filter3d(xyz.to(DEV), poses.to(DEV), W, H, t, t * H / W).cpu().double()
    flip = margin < 1e-5                         # depth or border decision within fp32 rounding of its threshold
    ok = ~flip
    assert int(flip.sum()) < 1e-3 * P, int(flip.sum())
    assert float(((out - ref).abs() / ref)[ok].max()) < 2e-6
    # every branch was reached: unseen (filled with the max), seen
    unseen = torch.isclose(ref, ref.max())
    assert 0 < int(unseen.sum()) < P
    again = mip_filter3d(xyz.to(DEV), poses.to(DEV), W, H, t, t * H / W).cpu().double()
    assert torch.equal(again, out)


def test_tracking_mode_pose_gradient_with_mip2d_equals_full_backward():
    import instantsplat_b200 as I
    sc = _scene(P=3000, seed=65, log_s=math.log(0.004))
    f3d = _filter3d(sc).to(DEV)
    gt = torch.rand(3, sc.height, sc.width, generator=torch.Generator().manual_seed(1)).to(DEV)
    rs = I.GaussianRasterizationSettings(*settings_for(sc, 3, torch.zeros(3)), kernel_size=0.1)
    grads = []
    for full in (True, False):
        prm = {k: v.to(DEV).clone().requires_grad_(full) for k, v in sc.params.items()}
        pose = sc.poses[0].to(DEV).clone().requires_grad_(True)
        img, _ = I.rasterize_fused(prm["xyz"], prm["rotation"], prm["scaling"], prm["opacity"], prm["f_dc"],
                                   prm["f_rest"], pose, torch.zeros(sc.P, 3, device=DEV), rs, f3d)
        I.fused_training_loss(img, gt).backward()
        grads.append(pose.grad.clone())
    assert rel_err(grads[1], grads[0]) < 1e-5, (grads[1], grads[0])
    # PoseTracker with the filters: its first forward is the boundary's image
    from instantsplat_b200.tracking import PoseTracker
    tr = PoseTracker(sc.params["xyz"], sc.params["rotation"], sc.params["scaling"], sc.params["opacity"],
                       sc.params["f_dc"], sc.params["f_rest"], sc.width, sc.height, sc.fovx, sc.fovy, sh_degree=3,
                       device=DEV, kernel_size=0.1, filter_3D=f3d)
    prm = {k: v.to(DEV) for k, v in sc.params.items()}
    img, _ = I.rasterize_fused(prm["xyz"], prm["rotation"], prm["scaling"], prm["opacity"], prm["f_dc"],
                               prm["f_rest"], sc.poses[0].to(DEV), torch.zeros(sc.P, 3, device=DEV), rs, f3d)
    assert torch.equal(tr.render(sc.poses[0]), img)
    pose, loss, trace = tr.optimize(sc.poses[0] + 0.01, img.detach(), num_iter=30, return_trace=True)
    assert math.isfinite(loss) and loss <= float(trace[0]) and bool(torch.isfinite(pose).all())


def _trainer_run(sc, gts, use_graph, steps=12):
    import instantsplat_b200 as I
    from instantsplat_b200.trainer import OptimConfig
    cfg = OptimConfig()
    cfg.mip_kernel_size, cfg.mip_filter3d_interval, cfg.iterations = 0.1, 4, 120
    tr = I.JointTrainer(sc, DEV, gt_images=gts, cfg=cfg, use_graph=use_graph)
    for it in range(steps):
        tr.step(it % sc.n_views)
    torch.cuda.synchronize()
    return tr


def test_trainer_with_filters_is_deterministic_and_matches_boundary():
    import instantsplat_b200 as I
    from instantsplat_b200.scenes import surface_scene
    from instantsplat_b200.frame import mip_filter3d
    sc = surface_scene(20_000, 3, 160, 112, seed=43, sh_degree=3)
    gts = torch.rand(3, 3, sc.height, sc.width, generator=torch.Generator().manual_seed(8))
    # first step's gradients == the autograd boundary with the same filters
    from instantsplat_b200.trainer import OptimConfig
    cfg = OptimConfig()
    cfg.mip_kernel_size = 0.1
    tr = I.JointTrainer(sc, DEV, gt_images=gts, cfg=cfg)
    f3d = mip_filter3d(sc.params["xyz"].to(DEV), sc.poses.to(DEV), sc.width, sc.height, math.tan(sc.fovx / 2),
                       math.tan(sc.fovy / 2))
    assert torch.equal(tr.filter_3D, f3d)
    tr.render(1)
    tr.loss_and_backward(1, tr.gt[1])
    pc = {k: v.to(DEV).clone().requires_grad_(True) for k, v in sc.params.items()}
    pose = sc.poses[1].to(DEV).clone().requires_grad_(True)
    rs = I.GaussianRasterizationSettings(*settings_for(sc, tr.active_sh_degree, torch.zeros(3)), kernel_size=0.1)
    img, _ = I.rasterize_fused(pc["xyz"], pc["rotation"], pc["scaling"], pc["opacity"], pc["f_dc"], pc["f_rest"],
                               pose, torch.zeros(sc.P, 3, device=DEV), rs, f3d)
    assert torch.equal(img, tr.color)
    I.fused_training_loss(img, gts[1].to(DEV)).backward()
    for k in NAMES:
        assert rel_err(tr.view(tr.grads, k), pc[k].grad.reshape(sc.P, -1)) < 1e-4, k
    assert rel_err(tr.pose_grad[1], pose.grad) < 1e-4
    # eager == graph replay == eager again, bit for bit; the filter recomputes every 4 iterations
    a = _trainer_run(sc, gts, False)
    b = _trainer_run(sc, gts, True)
    c = _trainer_run(sc, gts, False)
    assert a.mip_recomputed_at == [4, 8, 12] == b.mip_recomputed_at
    for t in (b, c):
        assert torch.equal(a.params, t.params) and torch.equal(a.poses, t.poses) and torch.equal(a.filter_3D, t.filter_3D)
    # the recompute follows the current xyz and poses
    xyz = a.view(a.params, "xyz").clone()
    assert torch.equal(a.filter_3D, mip_filter3d(xyz, a.poses, sc.width, sc.height, a.ident.tanfovx, a.ident.tanfovy))
    # not in the last 100 iterations
    a.cfg.iterations = 116
    n = len(a.mip_recomputed_at)
    for it in range(4):
        a.step(it % 3)
    assert len(a.mip_recomputed_at) == n


# ---- records, cull, mass -------------------------------------------------------------------------------------------
def test_records_follow_the_filtered_opacity_and_cull_is_lossless():
    import instantsplat_b200 as I
    import instantsplat_b200.rasterizer as RZ
    import _geom as G
    sc = _scene(P=3000, seed=66, log_s=math.log(0.004))
    f3d = _filter3d(sc)
    for kappa, f in ((0.1, f3d), (0.1, None), (0.3, f3d)):
        rs = I.GaussianRasterizationSettings(*settings_for(sc, 3, torch.zeros(3)), kernel_size=kappa)
        prm = {k: v.to(DEV) for k, v in sc.params.items()}
        args = (prm["xyz"], prm["rotation"], prm["scaling"], prm["opacity"], prm["f_dc"], prm["f_rest"],
                sc.poses[0].to(DEV), torch.zeros(sc.P, 3, device=DEV), rs, None if f is None else f.to(DEV))
        x = [t.clone().requires_grad_(True) if k < 7 else t for k, t in enumerate(args)]
        img, _ = I.rasterize_fused(*x)
        cam = O.Camera.instantsplat(sc.width, sc.height, sc.fovx, sc.fovy, sh_degree=3)
        o = MIP.mip_records(sc.params, sc.poses[0], cam, kappa, f)
        d = G.decode(img.grad_fn.st)
        # h2 comes from det(Sigma2) = a0 c0 - b^2, resolved by fp32 to (a0 c0 + b^2) / det * 6e-8 relative: the record
        # opacity of an ill-conditioned Gaussian (a needle far below a pixel) is bounded on that scale, flagged and
        # counted, and its fp64 opacity replaced by the kernel's for the rest of the record check
        a_, b_, c_ = o["cov2d"].unbind(-1)
        det0 = (a_ - kappa) * (c_ - kappa) - b_ * b_
        cond = ((a_ - kappa) * (c_ - kappa) + b_ * b_).abs() / det0.abs().clamp(min=1e-300)
        ill = (2e-7 * cond > 1e-5) & o["visible"]
        rel = (d["opacity"] - o["opacity"]).abs() / o["opacity"].abs()
        assert bool((rel[ill] <= 2e-5 + 2e-7 * cond[ill]).all())
        # this population is mostly sub-pixel on purpose; the bulk is still checked at REC_TOL
        assert int(ill.sum()) < 0.1 * int(o["visible"].sum()), int(ill.sum())
        o["opacity"] = torch.where(ill, d["opacity"], o["opacity"])
        summary = G.check_records(d, o)
        assert summary["visible"] > 1000 and summary["below_cutoff"] > 0, summary
        # the record opacity is o_eff, not the unfiltered one
        raw = torch.sigmoid(sc.params["opacity"]).reshape(-1).double()
        assert float((o["opacity"] - raw).abs().max()) > 0.1
        saved = RZ.EXACT_CULL
        try:
            RZ.EXACT_CULL = False
            img_off, _ = I.rasterize_fused(*args)
        finally:
            RZ.EXACT_CULL = saved
        assert torch.equal(img.detach(), img_off), (kappa, f is None)


@pytest.mark.parametrize("kappa", [0.1, 0.3])
def test_mass_of_isolated_gaussians_is_the_compensated_mass(kappa):
    """Against the formula, not the restatement: the image of one Gaussian (background 0, colour c, o_eff < 0.99)
    sums to c * 2 pi (o3 sqrt(det S2) - sqrt(det S2') / 255) -- the compensated mass minus what lies below the 1/255
    cutoff (the integral of o G over {o G >= t} is 2 pi sqrt(det) (o - t)).  The pixel sum differs from the integral
    only along the cutoff contour, by at most 1/255 per pixel there: the tolerance is c (perimeter + 8) / 255."""
    import instantsplat_b200 as I
    W = H = 512
    fovx = math.radians(60.0)
    t = math.tan(fovx / 2)
    fx = W / (2 * t)
    g = torch.Generator().manual_seed(7)
    n = 7
    ij = torch.stack(torch.meshgrid(torch.arange(n), torch.arange(n), indexing="ij"), -1).reshape(-1, 2).double()
    P = ij.shape[0]
    z = 4.0 + torch.rand(P, generator=g, dtype=torch.float64)
    px = 40.0 + 72.0 * ij + torch.rand(P, 2, generator=g, dtype=torch.float64)   # pixel position of the mean
    x = (px[:, 0] + 0.5 - W / 2) / fx * z
    y = (px[:, 1] + 0.5 - H / 2) / fx * z
    means = torch.stack([x, y, z], 1)
    s = (0.01 + 0.03 * torch.rand(P, 3, generator=g, dtype=torch.float64)) * z[:, None] / 4.0
    cov = torch.stack([s[:, 0] ** 2, torch.zeros(P, dtype=torch.float64), torch.zeros(P, dtype=torch.float64),
                       s[:, 1] ** 2, torch.zeros(P, dtype=torch.float64), s[:, 2] ** 2], 1)
    o3 = 0.3 + 0.6 * torch.rand(P, generator=g, dtype=torch.float64)
    col = torch.tensor([0.5, 0.3, 0.8], dtype=torch.float64)
    # the 2-D covariance, straight from the EWA formula (identity view)
    J = torch.zeros(P, 2, 3, dtype=torch.float64)
    J[:, 0, 0], J[:, 0, 2] = fx / z, -fx * x / z ** 2
    J[:, 1, 1], J[:, 1, 2] = fx / z, -fx * y / z ** 2
    S3 = torch.diag_embed(s ** 2)
    S2 = J @ S3 @ J.transpose(1, 2)
    det0 = torch.linalg.det(S2)
    S2d = S2 + kappa * torch.eye(2, dtype=torch.float64)
    det1 = torch.linalg.det(S2d)
    h2 = torch.sqrt(det0 / det1)
    o_eff = o3 * h2
    assert float(o_eff.max()) < 0.99 and float(o_eff.min()) > 2.0 / 255
    lam = torch.linalg.eigvalsh(S2d)
    assert float(lam.min()) >= 1.0                          # sigma >= 1 px
    R = torch.sqrt(2.0 * torch.log(255.0 * o_eff))          # cutoff contour in Mahalanobis units
    a_, b_ = R * lam[:, 1].sqrt(), R * lam[:, 0].sqrt()
    perim = math.pi * (3 * (a_ + b_) - torch.sqrt((3 * a_ + b_) * (a_ + 3 * b_)))
    assert float((a_ + 2).max()) < 36                       # each Gaussian alone in its 72 px cell
    expect = 2 * math.pi * (o3 * det0.sqrt() - det1.sqrt() / 255.0)
    tol = (perim + 8.0) / 255.0
    # the check can tell: without the compensation the mass would be o3 2 pi sqrt(det S2') (less the cutoff part)
    uncompensated = 2 * math.pi * (o3 * det1.sqrt() - det1.sqrt() / (255.0 * h2))
    assert float(((uncompensated - expect).abs() > 2 * tol).float().mean()) > 0.25
    rs = I.GaussianRasterizationSettings(*settings_for(
        type("S", (), dict(width=W, height=H, fovx=fovx, fovy=fovx, sh_degree=0))(), 0, torch.zeros(3)),
        kernel_size=kappa)
    rast = I.GaussianRasterizer(rs)
    img, _ = rast(means3D=means.float().to(DEV), means2D=torch.zeros(P, 3, device=DEV),
                  opacities=o3.float()[:, None].to(DEV), colors_precomp=col.float().expand(P, 3).contiguous().to(DEV),
                  cov3D_precomp=cov.float().to(DEV))
    img = img.detach().cpu().double()
    for i in range(P):
        cx, cy = int(px[i, 0]), int(px[i, 1])
        blk = img[:, cy - 36:cy + 36, cx - 36:cx + 36].sum((1, 2))
        err = (blk - col * float(expect[i])).abs() / col
        assert float(err.max()) < float(tol[i]), (i, float(err.max()), float(tol[i]), float(expect[i]))


# ---- tracking against the CPU restatement --------------------------------------------------------------------------
def test_pose_tracker_with_filters_matches_cpu_restatement():
    from instantsplat_b200.scenes import surface_scene
    from instantsplat_b200.tracking import PoseTracker
    sc = surface_scene(6000, 3, 128, 96, seed=61, sh_degree=2)
    view, n_it, kappa = 1, 12, 0.1
    f3d = _filter3d(sc)
    cam = O.Camera.instantsplat(sc.width, sc.height, sc.fovx, sc.fovy, sh_degree=2)
    p = sc.params
    with torch.no_grad():
        gt, _ = MIP.render_mip(p["xyz"], p["rotation"], p["scaling"], p["opacity"], p["f_dc"], p["f_rest"],
                               sc.poses[view], cam, kappa, f3d)
    init = sc.poses[view] + torch.tensor([0.0, 0.004, -0.003, 0.002, 0.01, -0.008, 0.012])
    # render.py:113-161 on the restatement (as tests/test_tracking.py reference_tracking, with the filters)
    T = init[-3:].clone().requires_grad_()
    q = init[:4].clone().requires_grad_()
    opt = torch.optim.Adam([{"params": [T], "lr": 0.003}, {"params": [q], "lr": 0.001}], betas=(0.9, 0.999),
                           weight_decay=1e-4)
    sched = torch.optim.lr_scheduler.CosineAnnealingLR(opt, T_max=n_it, eta_min=0.0001)
    cand, best_ref, losses = torch.cat([q, T]).detach(), 1e20, []
    for _ in range(n_it):
        img, _ = MIP.render_mip(p["xyz"], p["rotation"], p["scaling"], p["opacity"], p["f_dc"], p["f_rest"],
                                torch.cat([q, T]), cam, kappa, f3d)
        mask = (img > 0.0).float()
        loss = ((img - gt).abs() * mask).sum() / mask.sum()
        loss.backward()
        with torch.no_grad():
            opt.step()
            opt.zero_grad(set_to_none=True)
            losses.append(float(loss))
            if float(loss) < best_ref:
                best_ref, cand = float(loss), torch.cat([q, T]).detach().clone()
        sched.step()
    tr = PoseTracker(p["xyz"], p["rotation"], p["scaling"], p["opacity"], p["f_dc"], p["f_rest"], sc.width, sc.height,
                     sc.fovx, sc.fovy, sh_degree=2, device=DEV, kernel_size=kappa, filter_3D=f3d)
    pose, best, trace = tr.optimize(init, gt, num_iter=n_it, return_trace=True)
    assert losses[-1] < losses[0]
    dl = max(abs(a - float(b)) for a, b in zip(losses, trace))
    assert dl < 2e-5, (dl, losses, trace.tolist())
    assert abs(best - best_ref) < 2e-5
    assert float((pose - cand).abs().max()) < 2e-4, (pose, cand)


# ---- trainer against the restatement, model mirror ----------------------------------------------------------------
def test_trainer_first_step_gradients_match_restatement():
    import instantsplat_b200 as I
    from instantsplat_b200.scenes import surface_scene
    from instantsplat_b200.trainer import OptimConfig
    sc = surface_scene(8000, 3, 128, 96, seed=45, sh_degree=3)
    gts = torch.rand(3, 3, sc.height, sc.width, generator=torch.Generator().manual_seed(8))
    cfg = OptimConfig()
    cfg.mip_kernel_size = 0.1
    tr = I.JointTrainer(sc, DEV, gt_images=gts, cfg=cfg)
    view = 1
    tr.render(view)
    tr.loss_and_backward(view, tr.gt[view])
    f3d = tr.filter_3D.cpu()
    cam32 = O.Camera.instantsplat(sc.width, sc.height, sc.fovx, sc.fovy, sh_degree=3)
    cam64 = O.Camera.instantsplat(sc.width, sc.height, sc.fovx, sc.fovy, sh_degree=3, dtype=torch.float64)
    p = sc.params
    with torch.no_grad():
        means, rots = O.pose_pretransform(p["xyz"], p["rotation"], sc.poses[view])
        s, o = MIP.apply_filter3d(torch.exp(p["scaling"]), torch.sigmoid(p["opacity"]).reshape(-1), f3d)
        lists = O.build_tile_lists(MIP.project_mip(means, s, rots, o, torch.cat([p["f_dc"], p["f_rest"]], 1), cam32,
                                                   0.1))
    po = {k: v.double().clone().requires_grad_(True) for k, v in p.items()}
    pose = sc.poses[view].double().clone().requires_grad_(True)
    img, _, aux = MIP.render_mip(po["xyz"], po["rotation"], po["scaling"], po["opacity"], po["f_dc"], po["f_rest"],
                                 pose, cam64, 0.1, f3d.double(), return_aux=True, lists=lists)
    assert_image(image_stats(tr.color, img.detach(), aux["ambiguous"]), "trainer forward")
    loss = O.training_loss(img, gts[view].double())
    assert abs(float(loss.detach()) - float(tr.loss_value())) < 2e-5
    loss.backward()
    for k in NAMES:
        e = rel_err(tr.view(tr.grads, k), po[k].grad.reshape(sc.P, -1))
        assert e < GRAD_TOL, (k, e)
    assert rel_err(tr.pose_grad[view], pose.grad) < GRAD_TOL


def test_model_mirror_filter_render_and_surgery():
    import instantsplat_b200 as I
    import instantsplat_b200.renderer as RD
    from instantsplat_b200.camera import SimpleCamera
    from instantsplat_b200.frame import mip_filter3d
    from instantsplat_b200.scenes import surface_scene
    from instantsplat_b200.tracking import PoseTracker
    sc = surface_scene(20_000, 3, 160, 112, seed=47, sh_degree=3)
    m = I.GaussianModel.from_scene(sc, DEV)
    m.training_setup_pp()
    cams = [SimpleCamera(sc.width, sc.height, sc.fovx, sc.fovy, device=DEV) for _ in range(sc.n_views)]
    f = m.compute_3D_filter(cams)
    ref, margin = MIP.filter3d_ref(sc.params["xyz"], sc.poses, sc.width, sc.height, math.tan(sc.fovx / 2),
                                   math.tan(sc.fovy / 2), return_margin=True)
    ok = margin >= 1e-5
    assert f.shape == (sc.P, 1) and float(((f.cpu().reshape(-1).double() - ref).abs() / ref)[ok].max()) < 2e-6
    # render(kernel_size=0.1): the fused body and the unfused one (getters + GaussianRasterizer) against the restatement
    bg = torch.tensor([0.1, 0.2, 0.3])
    cam64 = O.Camera.instantsplat(sc.width, sc.height, sc.fovx, sc.fovy, bg=bg, sh_degree=3, dtype=torch.float64)
    p = sc.params
    img_o, _, aux = MIP.render_mip(*(p[k].double() for k in ("xyz", "rotation", "scaling", "opacity", "f_dc",
                                                                "f_rest")), sc.poses[0].double(), cam64, 0.1,
                                   f.cpu().reshape(-1).double(), return_aux=True)
    out = {}
    saved = RD.FUSED
    try:
        for fused in (True, False):
            RD.FUSED = fused
            pkg = I.render(cams[0], m, I.PipelineDefaults(), bg.to(DEV), camera_pose=m.get_RT(0), kernel_size=0.1)
            out[fused] = pkg["render"].detach()
            assert_image(image_stats(pkg["render"], img_o.detach(), aux["ambiguous"]), f"render fused={fused}")
            pkg["render"].sum().backward()
            assert float(m._scaling.grad.abs().max()) > 0
            m.optimizer.zero_grad(set_to_none=True)
    finally:
        RD.FUSED = saved
    # prune keeps the surviving rows; densification_postfix recomputes from the remembered cameras
    keep = torch.rand(sc.P, generator=torch.Generator().manual_seed(1)) > 0.3
    f_before = m.filter_3D.clone()
    m.prune_points(~keep.to(DEV))
    assert torch.equal(m.filter_3D, f_before[keep.to(DEV)])
    n_new = 100
    m.densification_postfix(m._xyz[:n_new].detach() + 0.01, m._features_dc[:n_new].detach(),
                            m._features_rest[:n_new].detach(), m._opacity[:n_new].detach(),
                            m._scaling[:n_new].detach(), m._rotation[:n_new].detach())
    assert torch.equal(m.filter_3D.reshape(-1), mip_filter3d(m._xyz, m.P[:3], sc.width, sc.height,
                                                             math.tan(sc.fovx / 2), math.tan(sc.fovy / 2)))
    # a filter set directly (e.g. from a PLY) has no cameras: new rows take the largest size
    m.filter_3D, m._filter_cams = m.filter_3D.clone(), None
    m.densification_postfix(m._xyz[:n_new].detach(), m._features_dc[:n_new].detach(),
                            m._features_rest[:n_new].detach(), m._opacity[:n_new].detach(),
                            m._scaling[:n_new].detach(), m._rotation[:n_new].detach())
    assert m.filter_3D.shape[0] == m._xyz.shape[0]
    assert bool((m.filter_3D[-n_new:] == m.filter_3D[:-n_new].max()).all())
    # PoseTracker.from_model carries kernel_size and the model's filter
    tr = PoseTracker.from_model(m, cams[0], device=DEV, kernel_size=0.1)
    assert tr.filt is not None and tr.filt.flags == 1 and torch.equal(tr.filter_3D, m.filter_3D.reshape(-1))
    RD.FUSED = True
    try:
        img = I.render(cams[0], m, I.PipelineDefaults(), torch.zeros(3, device=DEV), camera_pose=m.get_RT(0),
                       kernel_size=0.1)["render"].detach()
    finally:
        RD.FUSED = saved
    assert torch.equal(tr.render(m.get_RT(0)), img)
