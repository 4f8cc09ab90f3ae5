"""Adaptive density control in JointTrainer (-m gpu, DESIGN.md section 4.8): the statistics the per-Gaussian backward
accumulates, the densify / prune rows, and the whole train.py:195-211 schedule, each against the mirror GaussianModel
driven through the fused render() and PerPointAdam (tests/test_densify_cpu.py pins the mirror to the reference)."""
import copy
import os
import sys

import pytest
import torch

import instantsplat_b200 as I
from instantsplat_b200.camera import SimpleCamera
from instantsplat_b200.model import GaussianModel, optimization_defaults
from instantsplat_b200.scenes import perturbed_copy, surface_scene

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KEYS = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation")


def _quat_R(q):
    q = q / q.norm()
    r, x, y, z = q.tolist()
    return torch.tensor([[1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y)],
                         [2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x)],
                         [2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)]])


def inputs(P=20_000, n_views=3, W=160, H=96, seed=61, white=False, edge=True):
    """A surface scene with two edge populations: 400 Gaussians below the 1/255 opacity cutoff (radius > 0, no kept
    tile) and 400 placed behind view 0's camera (radius 0 there); ground truth from a perturbed copy."""
    sc = surface_scene(P, n_views, W, H, seed=seed, sh_degree=3)
    if edge:
        sc.params["opacity"][:400] = torch.logit(torch.tensor(0.002))
        R, t = _quat_R(sc.poses[0, :4]), sc.poses[0, 4:]
        behind = torch.stack([torch.tensor([0.1 * (k % 20 - 10), 0.1 * (k // 20 - 10), -1.0]) for k in range(400)])
        sc.params["xyz"][400:800] = ((behind - t) @ R)        # x = R^T (p - t): camera-frame z = -1
    if white:
        sc.bg = torch.ones(3)
    tgt = I.JointTrainer(sc, DEV)
    pp = perturbed_copy(sc, sigma=0.05)
    for k, kk in (("xyz", 3), ("f_dc", 3), ("opacity", 1), ("scaling", 3)):
        tgt.view(tgt.params, k)[800:].copy_(pp[k].reshape(sc.P, kk)[800:].to(DEV))
    gts = torch.stack([tgt.render(v).clone() for v in range(n_views)])
    cams = []
    for v in range(n_views):
        c = SimpleCamera(W, H, sc.fovx, sc.fovy, device=DEV)
        c.uid = v
        cams.append(c)
    return sc, gts, cams


def cfg_of(**over):
    c = I.OptimConfig()
    c.iterations = 1000
    c.densify = True
    c.densify_from_iter = c.densify_until_iter = 10 ** 9      # statistics only, unless overridden
    for k, v in over.items():
        setattr(c, k, v)
    return c


def mirror(sc, tr=None, kernel_size=None):
    gm = GaussianModel.from_scene(sc, DEV)
    gm.training_setup_pp(optimization_defaults(iterations=1000))
    gm.xyz_gradient_accum = torch.zeros(sc.P, 1, device=DEV)
    gm.denom = torch.zeros(sc.P, 1, device=DEV)
    gm.percent_dense = 0.01
    if kernel_size is not None:
        gm.filter_3D = tr.filter_3D[:, None].clone()
    return gm


PIPE = type("Pipe", (), dict(convert_SHs_python=False, compute_cov3D_python=False, debug=False))()


def mirror_stats(gm, pkg):
    vis, radii = pkg["visibility_filter"], pkg["radii"]
    gm.max_radii2D[vis] = torch.max(gm.max_radii2D[vis], radii[vis])
    gm.add_densification_stats(pkg["viewspace_points"], vis)


# ---- 1. statistics against the boundary ---------------------------------------------------------------------------
@pytest.mark.parametrize("kernel_size", [None, 0.1])
def test_statistics_match_the_boundary(kernel_size):
    from _geom import decode
    sc, gts, cams = inputs()
    tr = I.JointTrainer(sc, DEV, gt_images=gts, cfg=cfg_of(mip_kernel_size=kernel_size))
    gm = mirror(sc, tr, kernel_size)
    bg = sc.bg.to(DEV)
    seen_notile = 0
    for v in (0, 1, 2, 0, 2):
        tr.render(v)
        d = decode(tr.frame)
        seen_notile += int(((d["radii"] > 0) & (d["tiles"] == 0)).sum())
        if v == 0:
            assert int((d["radii"][400:800] == 0).sum()) == 400         # behind the camera
        tr.loss_and_backward(v, tr.gt[v], stats=True)
        pkg = I.render(cams[v], gm, PIPE, bg, camera_pose=gm.get_RT(v), kernel_size=kernel_size)
        pkg["render"].backward(tr.dL_dimg)           # the trainer's image gradient: the same dL/dmeans2D
        with torch.no_grad():
            mirror_stats(gm, pkg)
        gm.optimizer.zero_grad(set_to_none=True)
        gm.P.grad = None
    torch.cuda.synchronize()
    assert seen_notile > 0
    assert torch.equal(tr.denom, gm.denom)
    assert torch.equal(tr.max_radii2D, gm.max_radii2D.float())
    a, b = tr.xyz_gradient_accum, gm.xyz_gradient_accum
    assert float(b.max()) > 0 and int((b > 0).sum()) > sc.P // 4
    assert float(((a - b).abs() / b.abs().clamp_min(1e-30)).max()) <= 1e-6
    assert int(tr.denom[:400].count_nonzero()) > 0 and float(tr.xyz_gradient_accum[:400].abs().max()) == 0.0


def test_gradients_identical_with_statistics_on_and_off():
    sc, gts, _ = inputs(P=8000, seed=62)
    tr = I.JointTrainer(sc, DEV, gt_images=gts, cfg=cfg_of())
    out = []
    for stats in (False, True):
        tr.render(1)
        tr.loss_and_backward(1, tr.gt[1], stats=stats)
        out.append((tr.grads.clone(), tr.pose_grad.clone()))
    assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1])
    assert int(tr.denom.count_nonzero()) > 0


# ---- 2. overflow ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("use_graph", [False, True])
def test_overflowed_iteration_counts_once(use_graph):
    sc, gts, _ = inputs(P=30_000, W=256, H=160, seed=63)
    n = 10

    def run(sabotage_at=None):
        tr = I.JointTrainer(sc, DEV, gt_images=gts, cfg=cfg_of(), use_graph=use_graph)
        for k in range(n):
            if k == sabotage_at:
                tr._size_binning(0)
                assert tr.cap < tr.last_R
            tr.step(k % sc.n_views)
        torch.cuda.synchronize()
        return tr

    ref, ovf = run(), run(sabotage_at=6)
    assert ovf.overflows == 1 and ref.overflows == 0
    assert torch.equal(ref.denom, ovf.denom)
    assert torch.equal(ref.max_radii2D, ovf.max_radii2D)
    torch.testing.assert_close(ovf.xyz_gradient_accum, ref.xyz_gradient_accum, rtol=1e-4, atol=1e-9)


# ---- 3. surgery ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("clone_and_split", [False, True])
def test_densify_rows_match_the_mirror(clone_and_split):
    # no edge populations: a point no view sees would take a filter size that depends on the whole population
    sc, gts, cams = inputs(P=12_000, seed=64, edge=False)
    tr = I.JointTrainer(sc, DEV, gt_images=gts, cfg=cfg_of(mip_kernel_size=0.1))
    for k in range(4):
        tr.step(k % sc.n_views)
    tr.compute_filter_3D()                           # from the current poses, as the mirror's compute_3D_filter
    g = torch.Generator(device=DEV).manual_seed(3)
    P = tr.P
    denom = torch.randint(0, 4, (P,), device=DEV, generator=g).float()
    tr._stats[0] = denom * torch.rand(P, device=DEV, generator=g) * 4e-4
    tr._stats[1] = denom
    tr._stats[2] = torch.rand(P, device=DEV, generator=g) * 40
    # the mirror in the trainer's state
    gm = GaussianModel(3, DEV)
    shapes = dict(xyz=(P, 3), f_dc=(P, 1, 3), f_rest=(P, 15, 3), opacity=(P, 1), scaling=(P, 3), rotation=(P, 4))
    gm._set_params({k: tr.view(tr.params, k).reshape(shapes[k]).clone() for k in KEYS})
    gm.init_RT_seq(tr.poses.clone())
    gm.spatial_lr_scale = 1.0
    gm.training_setup_pp(optimization_defaults(iterations=1000), tr.per_point_lr[:P].reshape(P, 1).clone())
    for k in KEYS:
        p = getattr(gm, gm._ATTR[k])
        gm.optimizer.state[p] = dict(step=tr.step_count(k), exp_avg=tr.view(tr.exp_avg, k).reshape(shapes[k]).clone(),
                                     exp_avg_sq=tr.view(tr.exp_avg_sq, k).reshape(shapes[k]).clone())
    gm.xyz_gradient_accum, gm.denom = tr.xyz_gradient_accum.clone(), tr.denom.clone()
    gm.max_radii2D = tr.max_radii2D.clone()
    gm.percent_dense = tr.cfg.percent_dense
    gm.compute_3D_filter(cams)
    assert torch.equal(gm.filter_3D[:, 0], tr.filter_3D)
    # an extent that puts the median Gaussian at the clone / split boundary
    extent = float(torch.exp(tr.view(tr.params, "scaling")).max(1).values.median()) / tr.cfg.percent_dense
    args = (2e-4, 0.005, extent, 20)
    pa = tr.densify_and_prune(*args, clone_and_split=clone_and_split,
                              generator=torch.Generator(device=DEV).manual_seed(11))
    pb = gm.densify_and_prune(*args, clone_and_split=clone_and_split,
                              generator=torch.Generator(device=DEV).manual_seed(11))
    assert tr.P == gm._xyz.shape[0] == pa.P == pb.P
    assert int((~pa.keep).sum()) > 0
    if clone_and_split:
        assert int(pa.clone.sum()) > 0 and int(pa.split_sel.sum()) > 0
    for k in KEYS:
        p = getattr(gm, gm._ATTR[k])
        st = gm.optimizer.state[p]
        assert torch.equal(tr.view(tr.params, k), p.detach().reshape(tr.P, -1)), k
        assert torch.equal(tr.view(tr.exp_avg, k), st["exp_avg"].reshape(tr.P, -1)), k
        assert torch.equal(tr.view(tr.exp_avg_sq, k), st["exp_avg_sq"].reshape(tr.P, -1)), k
    assert torch.equal(tr.per_point_lr[:tr.P], gm.per_point_lr[:, 0])
    assert torch.equal(tr.filter_3D, gm.filter_3D[:, 0])
    assert torch.equal(tr.xyz_gradient_accum, gm.xyz_gradient_accum) and torch.equal(tr.denom, gm.denom)
    assert torch.equal(tr.max_radii2D, gm.max_radii2D)
    assert bool((tr.denom == 0).all()) == clone_and_split
    tr.step(0)                                       # the rebuilt trainer renders and trains
    assert torch.isfinite(tr.params).all()


# ---- 4. the whole loop ---------------------------------------------------------------------------------------------
LOOP = dict(densify_from_iter=5, densification_interval=5, opacity_reset_interval=20, densify_until_iter=36)
N_LOOP = 40


def grad_threshold(sc, gts):
    """A threshold that selects about 10 % of the seen Gaussians after a few iterations."""
    tr = I.JointTrainer(sc, DEV, gt_images=gts, cfg=cfg_of())
    for k in range(5):
        tr.step(k % sc.n_views)
    g = (tr.xyz_gradient_accum / tr.denom)[tr.denom > 0]
    return float(torch.quantile(g, 0.9))


def mirror_loop(sc, gts, cams, cfg, views):
    """train.py:140-211 with the densification block enabled, on the mirror."""
    if os.path.join(ROOT, "shims") not in sys.path:
        sys.path.insert(0, os.path.join(ROOT, "shims"))
    from fused_ssim import fused_ssim          # the shim, as train.py:39-43 imports it
    gm = GaussianModel.from_scene(sc, DEV)
    gm.training_setup_pp(optimization_defaults(iterations=cfg.iterations))
    gm.xyz_gradient_accum = torch.zeros(sc.P, 1, device=DEV)
    gm.denom = torch.zeros(sc.P, 1, device=DEV)
    gm.percent_dense = cfg.percent_dense
    gen = torch.Generator(device=DEV).manual_seed(cfg.densify_seed)
    extent = I.cameras_extent(sc.poses)
    bg = sc.bg.to(DEV)
    white = bool((sc.bg == 1).all())
    losses, sizes, steps = [], [], []
    for k, v in enumerate(views):
        iteration = 1 + k
        gm.update_learning_rate(iteration)
        if iteration % 1000 == 0:
            gm.oneupSHdegree()
        pkg = I.render(cams[v], gm, PIPE, bg, camera_pose=gm.get_RT(cams[v].uid))
        image = pkg["render"]
        Ll1 = torch.abs(image - gts[v]).mean()
        loss = (1.0 - cfg.lambda_dssim) * Ll1 + cfg.lambda_dssim * (1.0 - fused_ssim(image.unsqueeze(0),
                                                                                      gts[v].unsqueeze(0)))
        loss.backward()
        losses.append(loss.item())
        with torch.no_grad():
            if iteration < cfg.densify_until_iter:
                mirror_stats(gm, pkg)
                if iteration > cfg.densify_from_iter and iteration % cfg.densification_interval == 0:
                    size_threshold = 20 if iteration > cfg.opacity_reset_interval else None
                    gm.densify_and_prune(cfg.densify_grad_threshold, 0.005, extent, size_threshold,
                                         clone_and_split=cfg.densify_clone_split, generator=gen)
                if iteration % cfg.opacity_reset_interval == 0 or (white and iteration == cfg.densify_from_iter):
                    gm.reset_opacity()
            if iteration < cfg.iterations:
                gm.optimizer.step()
                gm.optimizer.zero_grad(set_to_none=True)
        sizes.append(gm._xyz.shape[0])
        steps.append({n: gm.optimizer.state[getattr(gm, gm._ATTR[n])]["step"] for n in KEYS})
    return gm, losses, sizes, steps


def trainer_loop(sc, gts, cfg, views, use_graph=False, watch=False):
    tr = I.JointTrainer(sc, DEV, gt_images=gts, cfg=cfg, use_graph=use_graph)
    losses, sizes, steps, frozen = [], [], [], []
    if watch:
        # what the densify / reset replaced must not move in the same iteration's optimizer step
        dp, ro = tr.densify_and_prune, tr.reset_opacity
        snap = {}

        def densify_and_prune(*a, **k):
            out = dp(*a, **k)
            snap["all"] = (tr.params.clone(), {n: tr.step_count(n) for n in KEYS})
            return out

        def reset_opacity():
            ro()
            snap["opacity"] = (tr.view(tr.params, "opacity").clone(), tr.step_count("opacity"))
            if "all" in snap:
                snap["all"] = (tr.params.clone(), snap["all"][1])

        tr.densify_and_prune, tr.reset_opacity = densify_and_prune, reset_opacity
    for v in views:
        tr.step(v)
        losses.append(float(tr.loss_value()))
        sizes.append(tr.P)
        steps.append({n: tr.step_count(n) for n in KEYS})
        if watch and snap:
            if "all" in snap:
                p, st = snap["all"]
                frozen.append(torch.equal(p, tr.params) and st == steps[-1])
            if "opacity" in snap:
                p, st = snap["opacity"]
                frozen.append(torch.equal(p, tr.view(tr.params, "opacity")) and st == steps[-1]["opacity"])
            snap.clear()
    torch.cuda.synchronize()
    return tr, losses, sizes, steps, frozen


@pytest.mark.parametrize("clone_split,white", [(False, False), (True, False), (True, True)])
def test_whole_loop_matches_the_mirror(clone_split, white):
    sc, gts, cams = inputs(P=15_000, seed=65, white=white)
    cfg = cfg_of(densify_clone_split=clone_split, densify_grad_threshold=grad_threshold(sc, gts), **LOOP)
    views = [k % sc.n_views for k in range(N_LOOP)]
    gm, l_m, s_m, st_m = mirror_loop(sc, gts, cams, cfg, views)
    tr, l_t, s_t, st_t, frozen = trainer_loop(sc, gts, cfg, views, watch=True)
    assert tr.densified_at == [10, 15, 20, 25, 30, 35] and tr.reset_at == ([5, 20] if white else [20])
    assert s_m == s_t, (s_m, s_t)
    assert len(set(s_t)) > 2, "the events are expected to change the Gaussian count"
    if clone_split and not white:              # (after the early reset of a white background, prunes outweigh)
        assert max(s_t) > sc.P
    assert st_m == st_t
    assert st_t[-1]["xyz"] == N_LOOP - 6 and st_t[-1]["opacity"] == N_LOOP - 6 - (1 if white else 0) \
        and tr.step_count("pose") == N_LOOP
    assert len(frozen) == 6 + (2 if white else 1) and all(frozen)
    d = max(abs(a - b) for a, b in zip(l_m, l_t))
    assert d < 1e-5, (d, l_m, l_t)
    for k in KEYS:
        diff = (tr.view(tr.params, k) - getattr(gm, gm._ATTR[k]).detach().reshape(tr.P, -1)).abs()
        assert float((diff > 1e-3).float().mean()) < 2e-3 and float(diff.max()) < 0.3, \
            (k, float(diff.max()), float((diff > 1e-3).float().mean()))


# ---- 5. replay and reproducibility ---------------------------------------------------------------------------------
def test_graph_replay_and_reruns_are_bit_identical():
    sc, gts, _ = inputs(P=15_000, seed=66)
    cfg = cfg_of(densify_clone_split=True, densify_grad_threshold=grad_threshold(sc, gts), **LOOP)
    views = [k % sc.n_views for k in range(N_LOOP)]
    a, la, sa, _, _ = trainer_loop(sc, gts, cfg, views)
    b, lb, sb, _, _ = trainer_loop(sc, gts, copy.copy(cfg), views)
    g, lg, sg, _, _ = trainer_loop(sc, gts, cfg, views, use_graph=True)
    assert len(g._graphs) > 0
    assert sa == sb == sg and la == lb == lg
    for t in (b, g):
        assert torch.equal(a.params, t.params) and torch.equal(a.exp_avg, t.exp_avg)
        assert torch.equal(a.exp_avg_sq, t.exp_avg_sq) and torch.equal(a.poses, t.poses)
        assert torch.equal(a._stats, t._stats)


def test_densify_needs_one_gpu():
    sc = surface_scene(1000, 2, 32, 32, seed=1, sh_degree=3)
    with pytest.raises(I.GsbError):
        I.JointTrainer(sc, DEV, cfg=cfg_of(), world_size=2, rank=0)
