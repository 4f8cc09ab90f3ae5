"""GPU parity tests (-m gpu): the CUDA path, called through the C ABI (ctypes) and the reference-shaped
Python boundary, against the CPU oracle on the same seeded inputs.

Tolerances (BASELINE.json north_star): render <= 1e-4 max abs per pixel; gradients <= 1e-3 relative
(max |a-b| / max |b| per tensor) -- held for every case, see tests/_parity.py for the protocol (oracle-flagged
threshold-ambiguous pixels are counted, bounded, and given zero loss weight in BOTH arms).
"""
import math
import os

import numpy as np
import pytest
import torch

from oracle import gs_oracle as O
from instantsplat_b200.scenes import make_config, random_scene, surface_scene
from _parity import (DEV, GRAD_TOL, NAMES, REPORT, ROW_TOL, assert_image, compare_fused, image_stats, rel_err,
                     settings_for)

pytestmark = pytest.mark.gpu


def oracle_run(sc, deg, bg, gt, pose=None):
    cam = O.Camera.instantsplat(sc.width, sc.height, sc.fovx, sc.fovy, bg=bg, sh_degree=deg)
    prm = {k: v.clone().requires_grad_(True) for k, v in sc.params.items()}
    pose = (sc.poses[0] if pose is None else pose).clone().requires_grad_(True)
    m2d = torch.zeros(sc.P, 3, requires_grad=True)
    img, radii, aux = O.render_instantsplat(prm["xyz"], prm["rotation"], prm["scaling"], prm["opacity"],
                                            prm["f_dc"], prm["f_rest"], pose, cam, means2D=m2d, return_aux=True)
    loss = O.training_loss(img, gt)
    loss.backward()
    grads = {k: prm[k].grad for k in prm}
    grads["pose"] = pose.grad
    grads["means2D"] = m2d.grad
    return img.detach(), radii, aux, loss.detach(), grads


def cuda_run(sc, deg, bg, gt, fused_loss=True):
    import instantsplat_b200 as I
    prm = {k: v.to(DEV).clone().requires_grad_(True) for k, v in sc.params.items()}
    pose = sc.poses[0].to(DEV).clone().requires_grad_(True)
    m2d = torch.zeros(sc.P, 3, device=DEV, requires_grad=True)
    rs = settings_for(sc, deg, bg)
    img, radii = I.rasterize_fused(prm["xyz"], prm["rotation"], prm["scaling"], prm["opacity"], prm["f_dc"],
                                   prm["f_rest"], pose, m2d, rs)
    if fused_loss:
        loss = I.fused_training_loss(img, gt.to(DEV))
    else:
        loss = 0.8 * (img - gt.to(DEV)).abs().mean() + 0.2 * (1.0 - I.fused_ssim(img[None], gt.to(DEV)[None]))
    loss.backward()
    grads = {k: prm[k].grad for k in prm}
    grads["pose"] = pose.grad
    grads["means2D"] = m2d.grad
    torch.cuda.synchronize()
    return img.detach(), radii, loss.detach(), grads


def check_image(img_cuda, img_or, amb):
    st = image_stats(img_cuda, img_or, amb)
    assert_image(st)
    return st["n_over_tol"]


def masked_weights(shape, amb, seed):
    """Seeded random loss weights, zero on the oracle-flagged (threshold-ambiguous) pixels."""
    return torch.rand(*shape, generator=torch.Generator().manual_seed(seed)) * (~amb)[None]


# ----------------------------------------------------------------------------------------------
def test_library_loads_and_reports_device():
    import instantsplat_b200 as I
    assert I.lib().gsb_abi_version() == 2
    assert torch.cuda.get_device_capability() == (9, 0), "these kernels are built for sm_90a only"


@pytest.mark.parametrize("deg", [0, 3])
def test_tiny_scene_vs_oracle(deg):
    sc = random_scene(600, 80, 56, seed=21 + deg, sh_degree=deg)      # W,H not multiples of 16
    bg = torch.tensor([0.2, 0.4, 0.1])
    gt = torch.rand(3, sc.height, sc.width, generator=torch.Generator().manual_seed(5))
    compare_fused(f"tiny600_80x56_deg{deg}", sc, 0, deg, bg, gt=gt)


def test_golden_raster_tiny(golden_dir):
    """Committed fp64 oracle output (regression pin; the reference ships no rasterizer vectors)."""
    z = np.load(os.path.join(golden_dir, "raster_tiny.npz"))
    sc = random_scene(400, int(z["width"]), int(z["height"]), seed=77)
    for k in NAMES:
        assert np.array_equal(sc.params[k].numpy(), z["in_" + k])
    bg, gt = torch.from_numpy(z["bg"]), torch.from_numpy(z["gt"])
    img_c, radii_c, loss_c, g_c = cuda_run(sc, 3, bg, gt)
    n_flip = check_image(img_c, torch.from_numpy(z["image"]).float(), torch.from_numpy(z["ambiguous"]))
    assert abs(float(loss_c) - float(z["loss"])) < 2e-5
    if n_flip == 0:      # the stored gradients are those of the full training loss (no per-pixel weights to mask)
        g_o = {k: torch.from_numpy(z["g_" + k]) for k in NAMES}
        g_o["pose"], g_o["means2D"] = torch.from_numpy(z["g_pose"]), torch.from_numpy(z["g_means2D"])
        errs = {k: rel_err(g_c[k], g_o[k]) for k in g_o}
        assert max(errs.values()) < GRAD_TOL, errs


def test_config0_10k_random_256():
    """BASELINE.json configs[0]: 10k random Gaussians, one 256x256 camera (the CPU-runnable case)."""
    sc = make_config(0)
    gt = torch.rand(3, 256, 256, generator=torch.Generator().manual_seed(9))
    compare_fused("configs[0] 10k random 256x256", sc, 0, 3, torch.zeros(3), gt=gt)


def test_config1_surface_scene_scaled():
    """configs[1] shape (surface scene, 3 views, SH deg 0) at 1/10 scale, full frame, training-loss weights."""
    sc = surface_scene(20_000, 3, 160, 160, seed=1001, sh_degree=0)
    gt = torch.rand(3, 160, 160, generator=torch.Generator().manual_seed(4))
    for v in (0, 2):
        compare_fused(f"configs[1]/10 20k 160x160 view {v}", sc, v, 0, torch.zeros(3), gt=gt)


def stratified_tiles(gx, gy, n_interior, seed, extra=()):
    """Corner tiles, one tile per image edge, `n_interior` seeded random interior tiles and `extra`."""
    g = torch.Generator().manual_seed(seed)
    tiles = {0, gx - 1, (gy - 1) * gx, gy * gx - 1, gx // 2, (gy - 1) * gx + gx // 3, (gy // 2) * gx, (gy // 3) * gx + gx - 1}
    while len(tiles) < 8 + n_interior:
        tx = int(torch.randint(1, gx - 1, (1,), generator=g))
        ty = int(torch.randint(1, gy - 1, (1,), generator=g))
        tiles.add(ty * gx + tx)
    tiles.update(int(t) for t in extra)
    return sorted(tiles)


def enlarge_some(sc, n, factor, seed):
    """Blow up n seeded Gaussians so that their tile rects exceed the cooperative-emission threshold (> 24 tiles)."""
    g = torch.Generator().manual_seed(seed)
    idx = torch.randperm(sc.P, generator=g)[:n]
    sc.params["scaling"][idx] += math.log(factor)
    return idx


def tiles_under(sc, view, deg, idx):
    """Tile ids under the centres of Gaussians `idx` in `view` (oracle projection, no grad)."""
    with torch.no_grad():
        cam = O.Camera.instantsplat(sc.width, sc.height, sc.fovx, sc.fovy, sh_degree=deg)
        means, rots = O.pose_pretransform(sc.params["xyz"][idx], sc.params["rotation"][idx], sc.poses[view])
        shs = torch.cat([sc.params["f_dc"][idx], sc.params["f_rest"][idx]], dim=1)
        pr = O.project(means, torch.exp(sc.params["scaling"][idx]), rots, torch.sigmoid(sc.params["opacity"][idx]), shs, cam)
    gx, gy = pr["grid"]
    out = []
    for k in range(len(idx)):
        if bool(pr["visible"][k]) and int(pr["ntiles"][k]) > 24:
            tx, ty = int(pr["xy"][k, 0] // 16), int(pr["xy"][k, 1] // 16)
            if 0 <= tx < gx and 0 <= ty < gy:
                out.append(ty * gx + tx)
    return out


def test_config1_full_size_on_tile_subset():
    """BASELINE.json configs[1] at FULL size (200k Gaussians, 512x512, SH deg 0): 40 of 1024 tiles (3.9 %) incl.
    corners and edges, two views."""
    sc = make_config(1)
    for v, seed in ((1, 3), (2, 4)):
        compare_fused(f"configs[1] 200k 512x512 view {v}", sc, v, 0, torch.zeros(3),
                      tiles=stratified_tiles(32, 32, 12, seed))


def test_config2_full_size_on_tile_subsets_three_views():
    """BASELINE.json configs[2] at FULL size (1M Gaussians, 1920x1080, SH deg 3): >= 1 % of the 8160 tiles,
    stratified over three views, incl. image corners / edges and tiles under Gaussians whose rect spans more than
    24 tiles (the warp-cooperative counting / emission path)."""
    sc = make_config(2)
    big = enlarge_some(sc, 96, 6.0, seed=5)
    total = 0
    for v, seed in ((0, 21), (5, 22), (11, 23)):
        extra = tiles_under(sc, v, 3, big)[:6]
        assert len(extra) >= 2, "expected some > 24-tile Gaussians in view"
        tiles = stratified_tiles(120, 68, 16, seed, extra)
        total += len(tiles)
        compare_fused(f"configs[2] 1M 1920x1080 view {v}", sc, v, 3, torch.zeros(3), tiles=tiles, row_tol=ROW_TOL)
    assert total >= 82          # 1 % of 8160


def test_config4_4k_on_tile_subset():
    """BASELINE.json configs[4] geometry (4M Gaussians, 3840x2160 = 32 400 tiles, SH deg 3, R ~ 46 M), one view,
    tile subset incl. corners and edges."""
    sc = make_config(4)
    compare_fused("configs[4] 4M 3840x2160 view 13", sc, 13, 3, torch.zeros(3), tiles=stratified_tiles(240, 135, 24, 31),
                  row_tol=ROW_TOL)


def test_exact_cull_is_lossless():
    import instantsplat_b200.rasterizer as R
    sc = random_scene(5000, 200, 136, seed=3)
    bg = torch.tensor([0.0, 0.1, 0.0])
    gt = torch.rand(3, sc.height, sc.width)
    try:
        R.EXACT_CULL = True
        a_img, a_r, _, a_g = cuda_run(sc, 3, bg, gt)
        R.EXACT_CULL = False
        b_img, b_r, _, b_g = cuda_run(sc, 3, bg, gt)
    finally:
        R.EXACT_CULL = True
    assert torch.equal(a_r, b_r)
    assert float((a_img - b_img).abs().max()) <= 1e-6
    for k in NAMES + ("pose",):
        assert rel_err(a_g[k], b_g[k]) < 1e-4, k


def test_big_rects_flattened_path_vs_oracle():
    """Gaussians whose tile rect exceeds 128 tiles are not walked by their own warp: k_preprocess queues them and
    k_big_rects counts / emits them as (Gaussian, trip) work items spread over the grid (gs_bin.cu).  40 Gaussians
    blown up 12x (a few hundred tiles each) and 3 blown up 150x (the whole 640x400 frame = 1000 tiles) on a 20k scene:
    image and gradients vs the oracle on a tile subset that includes tiles under the big ones, the instance count is
    reproducible, and the lossless cull stays lossless on this path."""
    import instantsplat_b200.rasterizer as R
    sc = surface_scene(20_000, 3, 640, 400, seed=23, sh_degree=3)
    mid = enlarge_some(sc, 40, 12.0, seed=6)
    huge = enlarge_some(sc, 3, 150.0, seed=7)
    sc.params["opacity"][huge] = -2.0                 # keep the frame-filling ones translucent: everything behind still counts
    with torch.no_grad():
        cam = O.Camera.instantsplat(sc.width, sc.height, sc.fovx, sc.fovy, sh_degree=3)
        idx = torch.cat([mid, huge])
        means, rots = O.pose_pretransform(sc.params["xyz"][idx], sc.params["rotation"][idx], sc.poses[1])
        shs = torch.cat([sc.params["f_dc"][idx], sc.params["f_rest"][idx]], dim=1)
        pr = O.project(means, torch.exp(sc.params["scaling"][idx]), rots, torch.sigmoid(sc.params["opacity"][idx]), shs, cam)
    assert int((pr["ntiles"] > 128).sum()) >= 10 and int(pr["ntiles"].max()) >= 900, pr["ntiles"]
    extra = tiles_under(sc, 1, 3, idx)[:8]
    compare_fused("big rects (flattened count/emit), 20k 640x400 view 1", sc, 1, 3, torch.tensor([0.1, 0.2, 0.3]),
                  tiles=stratified_tiles(40, 25, 10, 41, extra))
    sc.poses = sc.poses[1:2]
    bg = torch.zeros(3)
    gt = torch.rand(3, sc.height, sc.width, generator=torch.Generator().manual_seed(4))
    try:
        R.EXACT_CULL = True
        a_img, a_r, _, a_g = cuda_run(sc, 3, bg, gt)
        a2_img = cuda_run(sc, 3, bg, gt)[0]
        R.EXACT_CULL = False
        b_img, b_r, _, b_g = cuda_run(sc, 3, bg, gt)
    finally:
        R.EXACT_CULL = True
    assert torch.equal(a_img, a2_img)                 # deterministic although the emission order is not
    assert torch.equal(a_r, b_r) and float((a_img - b_img).abs().max()) <= 1e-6
    for k in NAMES + ("pose",):
        assert rel_err(a_g[k], b_g[k]) < 1e-4, k


def test_sync_free_capacity_overflow_is_repaired():
    """The autograd boundary sizes the binning buffer from earlier counts and launches the render phase without waiting
    for the instance count.  With a (forced) far too small estimate the tile lists are truncated; the check at the end of
    the forward notices, repeats the render phase with an exact buffer (RuntimeWarning) and image, loss and gradients
    equal those of an exactly sized call."""
    import instantsplat_b200.rasterizer as R
    sc = random_scene(24000, 200, 136, seed=3)
    bg = torch.tensor([0.0, 0.1, 0.0])
    gt = torch.rand(3, sc.height, sc.width, generator=torch.Generator().manual_seed(2))
    a_img, a_r, a_loss, a_g = cuda_run(sc, 3, bg, gt)
    key = (torch.zeros(1, device=DEV).device.index, sc.P, sc.width, sc.height)
    assert R._last_R.get(key, 0) > 65536, "scene too small to overflow the minimum capacity"
    true_R, saved = None, R.HEADROOM
    try:
        R.HEADROOM = 0.0                     # capacity = 0 * estimate + 65536 instances
        R._last_R[key] = 1
        with pytest.warns(RuntimeWarning):
            b_img, b_r, b_loss, b_g = cuda_run(sc, 3, bg, gt)
        true_R = R._last_R[key]
    finally:
        R.HEADROOM = saved
    assert true_R > 65536
    assert torch.equal(a_r, b_r) and float((a_img - b_img).abs().max()) <= 1e-6
    assert abs(float(a_loss) - float(b_loss)) < 1e-6
    for k in NAMES + ("pose",):
        assert rel_err(b_g[k], a_g[k]) < 1e-4, k


def test_blend_kernel_versions_agree():
    """v1 (one pixel per lane) and v2 (two pixels per lane) blend kernels, with and without TMA bulk
    staging, on a scene whose image size is not a multiple of the tile size."""
    import instantsplat_b200 as I
    L = I.lib()
    sc = surface_scene(40_000, 3, 300, 200, seed=17, sh_degree=2)
    bg = torch.tensor([0.1, 0.0, 0.2])
    gt = torch.rand(3, sc.height, sc.width, generator=torch.Generator().manual_seed(3))
    res = {}
    try:
        for ver, bulk in ((1, 0), (2, 1), (2, 0)):
            assert L.gsb_set_option(b"blend_version", ver) == 0 and L.gsb_set_option(b"stage_bulk", bulk) == 0
            res[(ver, bulk)] = cuda_run(sc, 2, bg, gt)
    finally:
        L.gsb_set_option(b"blend_version", 2)
        L.gsb_set_option(b"stage_bulk", 1)
    assert L.gsb_set_option(b"blend_version", 7) != 0 and L.gsb_set_option(b"nope", 1) != 0
    a_img, a_r, a_loss, a_g = res[(1, 0)]
    for key, (b_img, b_r, b_loss, b_g) in res.items():
        assert torch.equal(a_r, b_r), key
        # the versions round alpha differently, so an occasional 1/255-threshold flip is legitimate
        d = (a_img - b_img).abs().max(0)[0]
        assert float((d > 1e-5).float().mean()) < 1e-4 and float(d.max()) < 5e-3, key
        for k in NAMES + ("pose", "means2D"):
            assert rel_err(b_g[k], a_g[k]) < 5e-3, (key, k)
    # bulk vs cooperative staging of the same version must agree exactly in the forward
    assert torch.equal(res[(2, 1)][0], res[(2, 0)][0])


def test_generic_boundary_b2_nonidentity_view_packed_sh():
    """GaussianRasterizer called the vanilla-3DGS way (real view matrix, activated inputs, packed SHs)."""
    import instantsplat_b200 as I
    sc = random_scene(3000, 128, 96, seed=8)
    pose = torch.tensor([0.98, 0.05, -0.1, 0.02, 0.1, -0.05, 0.3])
    w2c = O.pose_to_w2c(pose)
    from instantsplat_b200.camera import projection_matrix
    Pm = projection_matrix(0.01, 100.0, sc.fovx, sc.fovy)
    view_t = w2c.t().contiguous()
    full = (view_t @ Pm.t()).contiguous()
    campos = torch.linalg.inv(w2c)[:3, 3].contiguous()
    bg = torch.tensor([0.3, 0.3, 0.3])
    cam = O.Camera(sc.width, sc.height, math.tan(sc.fovx / 2), math.tan(sc.fovy / 2), view_t, full, campos, bg, 2, 1.3)
    base = dict(means=sc.params["xyz"], scales=torch.exp(sc.params["scaling"]), rots=sc.params["rotation"],
                opac=torch.sigmoid(sc.params["opacity"]), shs=torch.cat([sc.params["f_dc"], sc.params["f_rest"]], 1))
    po = {k: v.clone().requires_grad_(True) for k, v in base.items()}
    m2o = torch.zeros(sc.P, 3, requires_grad=True)
    img_o, radii_o, aux = O.rasterize(po["means"], po["scales"], po["rots"], po["opac"], po["shs"], cam,
                                      means2D=m2o, return_aux=True)
    w = masked_weights((3, sc.height, sc.width), aux["ambiguous"], 1)
    (img_o * w).sum().backward()
    pc = {k: v.to(DEV).clone().requires_grad_(True) for k, v in base.items()}
    m2c = torch.zeros(sc.P, 3, device=DEV, requires_grad=True)
    rs = I.GaussianRasterizationSettings(sc.height, sc.width, cam.tanfovx, cam.tanfovy, bg.to(DEV), 1.3,
                                         view_t.to(DEV), full.to(DEV), 2, campos.to(DEV), False, True)
    rast = I.GaussianRasterizer(rs)
    img_c, radii_c = rast(means3D=pc["means"], means2D=m2c, opacities=pc["opac"], shs=pc["shs"],
                          scales=pc["scales"], rotations=pc["rots"])
    (img_c * w.to(DEV)).sum().backward()
    st = image_stats(img_c, img_o, aux["ambiguous"])
    assert_image(st, "B2 non-identity view")
    ge = {k: rel_err(pc[k].grad, po[k].grad) for k in base}
    ge["means2D"] = rel_err(m2c.grad, m2o.grad)
    REPORT.append(dict(case="B2 GaussianRasterizer, non-identity view, packed SH deg 2, scale_modifier 1.3", P=sc.P,
                       width=sc.width, height=sc.height, **st, grad_rel_err=ge, grad_rel_err_max=max(ge.values())))
    assert max(ge.values()) < GRAD_TOL, ge
    vis = rast.markVisible(pc["means"].detach())
    assert vis.dtype == torch.bool and vis.shape == (sc.P,)
    # error behaviour of the reference wrapper
    with pytest.raises(Exception):
        rast(means3D=pc["means"], means2D=m2c, opacities=pc["opac"], scales=pc["scales"], rotations=pc["rots"])
    with pytest.raises(Exception):
        rast(means3D=pc["means"], means2D=m2c, opacities=pc["opac"], shs=pc["shs"])


def test_precomputed_colors_and_cov3d():
    import instantsplat_b200 as I
    sc = random_scene(2000, 96, 96, seed=12)
    cam = O.Camera.instantsplat(sc.width, sc.height, sc.fovx, sc.fovy, sh_degree=0)
    means = sc.params["xyz"].clone()
    scales, rots = torch.exp(sc.params["scaling"]), sc.params["rotation"]
    r, x, y, z = rots.unbind(-1)
    Rm = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y), 2 * (x * y + r * z),
                      1 - 2 * (x * x + z * z), 2 * (y * z - r * x), 2 * (x * z - r * y), 2 * (y * z + r * x),
                      1 - 2 * (x * x + y * y)], -1).reshape(-1, 3, 3)
    Mx = Rm * scales[:, None, :]
    S = Mx @ Mx.transpose(1, 2)
    cov6 = torch.stack([S[:, 0, 0], S[:, 0, 1], S[:, 0, 2], S[:, 1, 1], S[:, 1, 2], S[:, 2, 2]], -1).contiguous()
    colors = torch.rand(sc.P, 3, generator=torch.Generator().manual_seed(2))
    opac = torch.sigmoid(sc.params["opacity"])
    leaves_o = [t.clone().requires_grad_(True) for t in (means, cov6, colors, opac)]
    img_o, _, aux = O.rasterize(leaves_o[0], None, None, leaves_o[3], None, cam, colors_precomp=leaves_o[2],
                                cov3D_precomp=leaves_o[1], return_aux=True)
    w = masked_weights((3, sc.height, sc.width), aux["ambiguous"], 3)
    (img_o * w).sum().backward()
    leaves_c = [t.to(DEV).clone().requires_grad_(True) for t in (means, cov6, colors, opac)]
    rs = settings_for(sc, 0, torch.zeros(3))
    img_c, _ = I.GaussianRasterizer(rs)(means3D=leaves_c[0], means2D=torch.zeros(sc.P, 3, device=DEV),
                                        opacities=leaves_c[3], colors_precomp=leaves_c[2], cov3D_precomp=leaves_c[1])
    (img_c * w.to(DEV)).sum().backward()
    st = image_stats(img_c, img_o, aux["ambiguous"])
    assert_image(st, "precomputed colours / cov3D")
    ge = {name: rel_err(a.grad, b.grad) for a, b, name in zip(leaves_c, leaves_o, ("means", "cov3D", "colors", "opac"))}
    REPORT.append(dict(case="B2 colors_precomp + cov3D_precomp", P=sc.P, width=sc.width, height=sc.height, **st,
                       grad_rel_err=ge, grad_rel_err_max=max(ge.values())))
    assert max(ge.values()) < GRAD_TOL, ge


def test_edge_cases_empty_and_culled():
    import instantsplat_b200 as I
    sc = random_scene(64, 48, 32, seed=1)
    bg = torch.tensor([0.5, 0.25, 0.125])
    rs = settings_for(sc, 3, bg)
    # everything behind the camera -> background only, zero grads, radii 0
    prm = {k: v.to(DEV).clone().requires_grad_(True) for k, v in sc.params.items()}
    with torch.no_grad():
        prm["xyz"][:, 2] = -5.0
    pose = sc.poses[0].to(DEV).clone().requires_grad_(True)
    img, radii = I.rasterize_fused(prm["xyz"], prm["rotation"], prm["scaling"], prm["opacity"], prm["f_dc"],
                                   prm["f_rest"], pose, torch.zeros(64, 3, device=DEV, requires_grad=True), rs)
    img.sum().backward()
    assert int(radii.abs().sum()) == 0
    assert torch.allclose(img, bg.to(DEV)[:, None, None].expand_as(img))
    assert float(prm["xyz"].grad.abs().max()) == 0.0 and float(pose.grad.abs().max()) == 0.0
    # P == 0
    e = lambda *s: torch.zeros(*s, device=DEV)
    img0, radii0 = I.rasterize_fused(e(0, 3), e(0, 4), e(0, 3), e(0, 1), e(0, 1, 3), e(0, 15, 3), pose.detach(),
                                     e(0, 3), rs)
    assert radii0.numel() == 0 and torch.allclose(img0, bg.to(DEV)[:, None, None].expand_as(img0))
    # one huge opaque Gaussian covering the whole image (max tile count, early termination)
    one = dict(xyz=torch.tensor([[0.0, 0.0, 3.0]]), rotation=torch.tensor([[1.0, 0, 0, 0]]),
               scaling=torch.full((1, 3), math.log(5.0)), opacity=torch.tensor([[8.0]]),
               f_dc=torch.ones(1, 1, 3), f_rest=torch.zeros(1, 15, 3))
    sc1 = random_scene(1, 48, 32, seed=1)
    sc1.params = one
    sc1.poses = torch.tensor([[1.0, 0, 0, 0, 0, 0, 0]])
    img_o, _, aux, _, g_o = oracle_run(sc1, 3, bg, torch.zeros(3, 32, 48))
    img_c, radii_c, _, g_c = cuda_run(sc1, 3, bg, torch.zeros(3, 32, 48))
    check_image(img_c, img_o, aux["ambiguous"])
    assert int(radii_c[0]) > 48


# ----------------------------------------------------------------------------------------------
def test_fused_ssim_and_loss_vs_reference_golden(golden_dir):
    import instantsplat_b200 as I
    z = np.load(os.path.join(golden_dir, "loss.npz"))
    a = torch.from_numpy(z["img1"]).to(DEV).requires_grad_(True)
    b = torch.from_numpy(z["img2"]).to(DEV)
    s = I.fused_ssim(a[None], b[None])
    assert abs(float(s) - float(z["ssim"])) < 2e-6
    (g,) = torch.autograd.grad(s, a)
    assert rel_err(g, torch.from_numpy(z["ssim_grad"])) < 1e-4
    tot = I.fused_training_loss(a, b)
    assert abs(float(tot) - float(z["total"])) < 2e-6
    (g2,) = torch.autograd.grad(tot, a)
    assert rel_err(g2, torch.from_numpy(z["total_grad"])) < 1e-4
    # eval mode (train=False) gives the same value and refuses backward
    s2 = I.fused_ssim(a[None].detach(), b[None], train=False)
    assert abs(float(s2) - float(s)) < 1e-7


def test_fused_ssim_odd_sizes_vs_oracle():
    import instantsplat_b200 as I
    g = torch.Generator().manual_seed(0)
    for (B, C, H, W) in ((1, 3, 17, 33), (2, 1, 5, 7), (1, 3, 64, 48)):
        a = torch.rand(B, C, H, W, generator=g)
        b = torch.rand(B, C, H, W, generator=g)
        ao = a.clone().requires_grad_(True)
        so = O.ssim_map(ao, b).mean()
        so.backward()
        ac = a.to(DEV).requires_grad_(True)
        sc_ = I.fused_ssim(ac, b.to(DEV))
        sc_.backward()
        assert abs(float(sc_) - float(so)) < 2e-6
        assert rel_err(ac.grad, ao.grad) < 1e-4


def test_per_point_adam_vs_reference_golden(golden_dir):
    import instantsplat_b200 as I
    z = np.load(os.path.join(golden_dir, "per_point_adam.npz"))
    a = torch.nn.Parameter(torch.from_numpy(z["p_pp"]).to(DEV))
    b = torch.nn.Parameter(torch.from_numpy(z["p_pl"]).to(DEV))
    lr_pp = torch.from_numpy(z["lr_pp"]).to(DEV)
    opt = I.PerPointAdam([{"params": [a], "lr": 1.6e-4, "per_point_lr": lr_pp, "name": "xyz"},
                          {"params": [b], "lr": 2.5e-2, "name": "f_dc"}], lr=0.0, betas=(0.9, 0.999), eps=1e-15)
    for it in range(6):
        a.grad = torch.from_numpy(z[f"ga{it}"]).to(DEV)
        b.grad = torch.from_numpy(z[f"gb{it}"]).to(DEV)
        opt.step()
        for mine, ref in ((a, f"a{it}"), (opt.state[a]["exp_avg"], f"am{it}"), (opt.state[a]["exp_avg_sq"], f"av{it}"),
                          (b, f"b{it}"), (opt.state[b]["exp_avg"], f"bm{it}"), (opt.state[b]["exp_avg_sq"], f"bv{it}")):
            np.testing.assert_allclose(mine.detach().cpu().numpy(), z[ref], rtol=3e-6, atol=1e-7, err_msg=ref)
        assert opt.state[a]["step"] == it + 1
    # error behaviour mirrors the reference
    with pytest.raises(ValueError):
        I.PerPointAdam([a], lr=-1.0)
    with pytest.raises(ValueError):
        I.PerPointAdam([a], betas=(1.0, 0.9))
    bad = I.PerPointAdam([{"params": [a], "per_point_lr": torch.ones(3, device=DEV)}], lr=1e-3)
    a.grad = torch.ones_like(a)
    with pytest.raises(ValueError):
        bad.step()


def test_per_point_adam_large_unaligned():
    """Many-block tensors incl. a length that is not a multiple of the vector width, vs the oracle."""
    import instantsplat_b200 as I
    g = torch.Generator().manual_seed(2)
    shapes = [(70001, 3), (70001, 15, 3), (12, 7), (70001, 1)]
    ps = [torch.randn(*s, generator=g) for s in shapes]
    ppl = 1 + 99 * torch.rand(70001, 1, generator=g)
    params = [torch.nn.Parameter(p.to(DEV)) for p in ps]
    opt = I.PerPointAdam([{"params": [params[0]], "lr": 1e-3, "per_point_lr": ppl.to(DEV)},
                          {"params": params[1:], "lr": 2e-3}], lr=0.0, eps=1e-15)
    ref = [p.clone() for p in ps]
    ms = [torch.zeros_like(p) for p in ps]
    vs = [torch.zeros_like(p) for p in ps]
    for it in range(3):
        gr = [torch.randn(*s, generator=g) * 1e-2 for s in shapes]
        for p, gg in zip(params, gr):
            p.grad = gg.to(DEV)
        opt.step()
        for i in range(len(ps)):
            O.per_point_adam_step(ref[i], gr[i], ms[i], vs[i], it + 1, 1e-3 if i == 0 else 2e-3,
                                  per_point_lr=ppl if i == 0 else None)
    for i in range(len(ps)):
        np.testing.assert_allclose(params[i].detach().cpu().numpy(), ref[i].numpy(), rtol=3e-6, atol=1e-7)


# ----------------------------------------------------------------------------------------------
class _FakeGaussians:
    """The attributes render() reads from GaussianModel (scene/gaussian_model.py:101-136)."""

    def __init__(self, sc, deg):
        p = {k: torch.nn.Parameter(v.to(DEV).clone()) for k, v in sc.params.items()}
        self._xyz, self._rotation, self._scaling, self._opacity = p["xyz"], p["rotation"], p["scaling"], p["opacity"]
        self._features_dc, self._features_rest = p["f_dc"], p["f_rest"]
        self.active_sh_degree, self.max_sh_degree = deg, 3
        self.P = torch.nn.Parameter(sc.poses.to(DEV).clone())

    get_xyz = property(lambda s: s._xyz)
    get_opacity = property(lambda s: torch.sigmoid(s._opacity))
    get_scaling = property(lambda s: torch.exp(s._scaling))
    get_features = property(lambda s: torch.cat((s._features_dc, s._features_rest), dim=1))

    def get_RT(self, idx):
        return self.P[idx]


class _Pipe:
    convert_SHs_python = False
    compute_cov3D_python = False
    debug = False


def test_render_dropin_matches_oracle_and_populates_grads():
    import instantsplat_b200 as I
    from instantsplat_b200.camera import SimpleCamera
    sc = random_scene(3000, 112, 80, seed=31)
    pc = _FakeGaussians(sc, 3)
    cam = SimpleCamera(sc.width, sc.height, sc.fovx, sc.fovy, device=DEV)
    bg = torch.tensor([0.0, 0.0, 0.0], device=DEV)
    gt = torch.rand(3, sc.height, sc.width, generator=torch.Generator().manual_seed(6))
    pkg = I.render(cam, pc, _Pipe(), bg, camera_pose=pc.get_RT(0))
    assert set(pkg) == {"render", "viewspace_points", "visibility_filter", "radii"}
    img = pkg["render"]
    # oracle arm first: its ambiguity mask zeroes the loss weights in both arms
    co = O.Camera.instantsplat(sc.width, sc.height, sc.fovx, sc.fovy, sh_degree=3)
    po = {k: v.clone().requires_grad_(True) for k, v in sc.params.items()}
    pose_o = sc.poses[0].clone().requires_grad_(True)
    m2o = torch.zeros(sc.P, 3, requires_grad=True)
    img_o, _, aux = O.render_instantsplat(po["xyz"], po["rotation"], po["scaling"], po["opacity"], po["f_dc"], po["f_rest"],
                                          pose_o, co, means2D=m2o, return_aux=True)
    assert_image(image_stats(img, img_o, aux["ambiguous"]), "render() drop-in")
    # the reference's loss expression (train.py:171-176) supplies dL/dimage; flagged pixels get zero weight
    im = img.detach().clone().requires_grad_(True)
    (0.8 * (im - gt.to(DEV)).abs().mean() + 0.2 * (1.0 - I.fused_ssim(im[None], gt.to(DEV)[None]))).backward()
    w = im.grad * (~aux["ambiguous"]).to(DEV)[None]
    w = w / w.abs().max()
    (img * w).sum().backward()
    (img_o * w.cpu()).sum().backward()
    ge = dict(pose=rel_err(pc.P.grad[0], pose_o.grad), xyz=rel_err(pc._xyz.grad, po["xyz"].grad),
              f_rest=rel_err(pc._features_rest.grad, po["f_rest"].grad),
              viewspace_points=rel_err(pkg["viewspace_points"].grad, m2o.grad))
    assert max(ge.values()) < GRAD_TOL, ge
    assert pkg["visibility_filter"].dtype == torch.bool


def test_pose_only_tracking_mode():
    """render.py:99-170 -- Gaussians frozen, only the camera pose requires grad: same pose gradient as the
    full backward, no per-Gaussian gradient tensors produced."""
    import instantsplat_b200 as I
    sc = random_scene(4000, 128, 96, seed=44)
    gt = torch.rand(3, sc.height, sc.width, generator=torch.Generator().manual_seed(1))
    _, _, _, g_full = cuda_run(sc, 3, torch.zeros(3), gt)
    prm = {k: v.to(DEV).clone() for k, v in sc.params.items()}                 # frozen
    pose = sc.poses[0].to(DEV).clone().requires_grad_(True)
    rs = settings_for(sc, 3, torch.zeros(3))
    img, _ = I.rasterize_fused(prm["xyz"], prm["rotation"], prm["scaling"], prm["opacity"], prm["f_dc"],
                               prm["f_rest"], pose, torch.zeros(sc.P, 3, device=DEV), rs)
    I.fused_training_loss(img, gt.to(DEV)).backward()
    assert rel_err(pose.grad, g_full["pose"]) < 1e-5
    assert all(v.grad is None for v in prm.values())


def test_trainer_step_matches_autograd_path_and_learns():
    import instantsplat_b200 as I
    sc = surface_scene(30_000, 3, 192, 128, seed=41, sh_degree=3)
    gts = torch.rand(3, 3, sc.height, sc.width, generator=torch.Generator().manual_seed(8))
    tr = I.JointTrainer(sc, DEV, gt_images=gts)
    # gradients written into the flat buffer == gradients of the autograd boundary
    tr.render(1)
    tr.loss_and_backward(1, tr.gt[1])
    sc1 = surface_scene(30_000, 3, 192, 128, seed=41, sh_degree=3)
    sc1.poses = sc.poses[1:2].clone()
    _, _, loss_c, g_c = cuda_run(sc1, 3, torch.zeros(3), gts[1])
    assert abs(float(tr.loss_value()) - float(loss_c)) < 1e-6
    for k in NAMES:
        assert rel_err(tr.view(tr.grads, k), g_c[k].reshape(sc.P, -1)) < 1e-4, k
    assert rel_err(tr.pose_grad[1], g_c["pose"]) < 1e-4
    assert float(tr.pose_grad[0].abs().max()) == 0.0
    # a few hundred iterations towards renders of a perturbed copy reduce the loss
    from instantsplat_b200.scenes import perturbed_copy
    tgt = I.JointTrainer(sc, DEV)
    pp = perturbed_copy(sc, sigma=0.05)
    for k, kk in (("xyz", 3), ("f_dc", 3), ("opacity", 1)):
        tgt.view(tgt.params, k).copy_(pp[k].reshape(sc.P, kk).to(DEV))
    gt_imgs = torch.stack([tgt.render(v).clone() for v in range(3)])
    tr2 = I.JointTrainer(sc, DEV, gt_images=gt_imgs)
    losses = []
    for it in range(60):
        tr2.step(it % 3)
        losses.append(float(tr2.loss_value()))
    assert np.mean(losses[-6:]) < 0.8 * np.mean(losses[:6]), losses[:6] + losses[-6:]
    assert torch.isfinite(tr2.params).all() and torch.isfinite(tr2.poses).all()


def test_full_size_properties_1080p():
    """Size-independent properties at the BASELINE resolution (1920x1080, 200k Gaussians, deg 3):
    determinism of the forward, lossless culling, T in [0,1], linearity of the backward in dL/dout."""
    import instantsplat_b200 as I
    import instantsplat_b200.rasterizer as R
    sc = surface_scene(200_000, 12, 1920, 1080, seed=1002, sh_degree=3)
    rs = settings_for(sc, 3, torch.zeros(3))
    prm = {k: v.to(DEV).clone().requires_grad_(True) for k, v in sc.params.items()}
    pose = sc.poses[5].to(DEV).clone().requires_grad_(True)

    def run(scale):
        for p in list(prm.values()) + [pose]:
            p.grad = None
        img, radii = I.rasterize_fused(prm["xyz"], prm["rotation"], prm["scaling"], prm["opacity"], prm["f_dc"],
                                       prm["f_rest"], pose, torch.zeros(sc.P, 3, device=DEV), rs)
        w = torch.linspace(0, 1, 1920, device=DEV)[None, None, :] * scale
        (img * w).sum().backward()
        return img.detach(), radii, {k: v.grad.clone() for k, v in prm.items()}, pose.grad.clone()

    img1, r1, g1, p1 = run(1.0)
    img2, r2, g2, p2 = run(2.0)
    assert torch.equal(img1, img2) and torch.equal(r1, r2)            # deterministic forward
    assert float(img1.min()) >= 0.0 and torch.isfinite(img1).all()
    for k in g1:
        assert rel_err(g2[k], 2.0 * g1[k]) < 1e-4, k                  # backward linear in dL/dout
    assert rel_err(p2, 2.0 * p1) < 1e-4
    try:
        R.EXACT_CULL = False
        img3, r3, g3, p3 = run(1.0)
    finally:
        R.EXACT_CULL = True
    assert float((img3 - img1).abs().max()) <= 1e-6 and torch.equal(r3, r1)


def test_knn_distcuda2_matches_bruteforce():
    """shims/simple_knn distCUDA2 (grid-hash exact 3-NN) vs brute force, on a surface cloud, a uniform cloud,
    a cloud with duplicates / far outliers, and tiny inputs."""
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "shims"))
    from simple_knn._C import distCUDA2
    g = torch.Generator().manual_seed(0)
    clouds = [surface_scene(6000, 3, 64, 64, seed=3).params["xyz"], torch.rand(5000, 3, generator=g) * 4 - 2]
    c = torch.randn(3000, 3, generator=g)
    c[:50] = c[50:100]                      # exact duplicates
    c[100] = torch.tensor([50.0, -40.0, 30.0])   # far outlier
    clouds.append(c)
    clouds += [torch.randn(7, 3, generator=g), torch.randn(4, 3, generator=g)]
    for pts in clouds:
        d = torch.cdist(pts.double(), pts.double())
        ref = (d * d).topk(4, dim=1, largest=False).values[:, 1:].mean(dim=1).float()
        got = distCUDA2(pts.to(DEV)).cpu()
        assert torch.allclose(got, ref, rtol=1e-4, atol=1e-7), float((got - ref).abs().max())


def test_per_point_adam_state_surgery_prune_and_cat():
    """Row f4: the reference's densify/prune code edits `optimizer.state[p]` and `param_groups[i]["params"]` in place
    (scene/gaussian_model.py:328-398: _prune_optimizer, cat_tensors_to_optimizer).  The drop-in keeps the
    same state layout, so the same surgery works and later steps match the oracle on the resized tensors."""
    import instantsplat_b200 as I
    g = torch.Generator().manual_seed(5)
    p0 = torch.randn(500, 3, generator=g)
    param = torch.nn.Parameter(p0.to(DEV).clone())
    opt = I.PerPointAdam([{"params": [param], "lr": 1e-2, "name": "xyz"}], lr=0.0, eps=1e-15)
    ref_p, ref_m, ref_v = p0.clone(), torch.zeros_like(p0), torch.zeros_like(p0)
    g1 = torch.randn(500, 3, generator=g) * 1e-2
    param.grad = g1.to(DEV)
    opt.step()
    O.per_point_adam_step(ref_p, g1, ref_m, ref_v, 1, 1e-2)
    # ---- prune (reference _prune_optimizer)
    mask = torch.rand(500, generator=g) > 0.3
    group = opt.param_groups[0]
    st = opt.state.get(group["params"][0])
    st["exp_avg"] = st["exp_avg"][mask.to(DEV)]
    st["exp_avg_sq"] = st["exp_avg_sq"][mask.to(DEV)]
    del opt.state[group["params"][0]]
    group["params"][0] = torch.nn.Parameter(group["params"][0][mask.to(DEV)].detach().clone().requires_grad_(True))
    opt.state[group["params"][0]] = st
    ref_p, ref_m, ref_v = ref_p[mask].clone(), ref_m[mask].clone(), ref_v[mask].clone()
    # ---- cat new points (reference cat_tensors_to_optimizer)
    ext = torch.randn(77, 3, generator=g)
    st = opt.state.get(group["params"][0])
    st["exp_avg"] = torch.cat((st["exp_avg"], torch.zeros(77, 3, device=DEV)), dim=0)
    st["exp_avg_sq"] = torch.cat((st["exp_avg_sq"], torch.zeros(77, 3, device=DEV)), dim=0)
    del opt.state[group["params"][0]]
    group["params"][0] = torch.nn.Parameter(torch.cat((group["params"][0].detach(), ext.to(DEV)), dim=0).requires_grad_(True))
    opt.state[group["params"][0]] = st
    ref_p = torch.cat((ref_p, ext)); ref_m = torch.cat((ref_m, torch.zeros(77, 3))); ref_v = torch.cat((ref_v, torch.zeros(77, 3)))
    newp = group["params"][0]
    for it in (2, 3):
        gi = torch.randn(newp.shape, generator=g) * 1e-2
        newp.grad = gi.to(DEV)
        opt.step()
        O.per_point_adam_step(ref_p, gi, ref_m, ref_v, it, 1e-2)
    np.testing.assert_allclose(newp.detach().cpu().numpy(), ref_p.numpy(), rtol=3e-6, atol=1e-7)
    assert opt.state[newp]["step"] == 3 and opt.state[newp]["exp_avg"].shape == newp.shape


def test_dgr_C_surface_matches_module_path():
    """shims/diff_gaussian_rasterization/_C: the upstream `_C.rasterize_gaussians(_backward)` / `mark_visible`
    signatures give the same image and gradients as the GaussianRasterizer module."""
    import sys
    import instantsplat_b200 as I
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "shims"))
    import diff_gaussian_rasterization as dgr
    sc = random_scene(2500, 120, 88, seed=19)
    rs = settings_for(sc, 3, torch.tensor([0.2, 0.1, 0.0]))
    dev_p = {k: v.to(DEV) for k, v in sc.params.items()}
    means = dev_p["xyz"].clone().requires_grad_(True)
    scales = torch.exp(dev_p["scaling"]).requires_grad_(True)
    rots = dev_p["rotation"].clone().requires_grad_(True)
    opac = torch.sigmoid(dev_p["opacity"]).requires_grad_(True)
    shs = torch.cat([dev_p["f_dc"], dev_p["f_rest"]], 1).requires_grad_(True)
    m2d = torch.zeros(sc.P, 3, device=DEV, requires_grad=True)
    img, radii = dgr.GaussianRasterizer(rs)(means3D=means, means2D=m2d, opacities=opac, shs=shs, scales=scales,
                                             rotations=rots)
    w = torch.rand(3, sc.height, sc.width, device=DEV)
    (img * w).sum().backward()
    e = torch.empty(0, device=DEV)
    nr, color, radii2, geom, binning, imgbuf = dgr._C.rasterize_gaussians(
        rs.bg, means.detach(), e, opac.detach(), scales.detach(), rots.detach(), 1.0, e, rs.viewmatrix, rs.projmatrix,
        rs.tanfovx, rs.tanfovy, sc.height, sc.width, shs.detach(), 3, rs.campos, False, False)
    assert nr > 0 and torch.equal(color, img.detach()) and torch.equal(radii2, radii)
    assert geom.dtype == torch.uint8 and binning.dtype == torch.uint8
    grads = dgr._C.rasterize_gaussians_backward(
        rs.bg, means.detach(), radii2, e, scales.detach(), rots.detach(), 1.0, e, rs.viewmatrix, rs.projmatrix, rs.tanfovx,
        rs.tanfovy, w, shs.detach(), 3, rs.campos, geom, nr, binning, imgbuf, False)
    d_m2d, d_col, d_op, d_m3d, d_cov, d_sh, d_sc, d_rot = grads
    assert d_col.numel() == 0 and d_cov.numel() == 0 and d_op.shape == (sc.P, 1)
    for a, b in ((d_m2d, m2d.grad), (d_op, opac.grad), (d_m3d, means.grad), (d_sh, shs.grad), (d_sc, scales.grad),
                 (d_rot, rots.grad)):
        assert rel_err(a, b) < 1e-4
    vis = dgr._C.mark_visible(means.detach(), rs.viewmatrix, rs.projmatrix)
    assert torch.equal(vis, means.detach()[:, 2] > 0.2)


def test_training_steps_are_bit_reproducible():
    """Two trainers running the same steps on the same inputs end bit-identical: the blend backward adds its
    per-Gaussian sums in fixed point, so their value does not depend on the order in which CTAs arrive (with float
    atomics it did, and Adam amplified the difference over a run)."""
    import instantsplat_b200 as I
    sc = surface_scene(30_000, 3, 320, 192, seed=19, sh_degree=3)
    gts = torch.rand(3, 3, sc.height, sc.width, generator=torch.Generator().manual_seed(6)).to(DEV)
    out = []
    for _ in range(2):
        tr = I.JointTrainer(sc, DEV, gt_images=gts)
        for s in range(12):
            tr.step(s % 3)
        torch.cuda.synchronize()
        out.append((tr.params.clone(), tr.poses.clone(), tr.color.clone(), tr.loss_value().clone()))
        del tr
    for a, b in zip(*out):
        assert torch.equal(a, b)
