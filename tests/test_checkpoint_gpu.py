"""Checkpoints of JointTrainer (-m gpu, DESIGN.md section 4.9): a run stopped at iteration k, saved, and continued by a
NEW trainer from the file ends bit-identical to the run that was not stopped; the tuple restores into the mirror; a
mirror-written checkpoint continues in the fused loop; the PLY / pose outputs round-trip; refusals raise."""
import os
import sys

import numpy as np
import pytest
import torch

import instantsplat_b200 as I
from instantsplat_b200 import scene_io
from instantsplat_b200.model import GaussianModel, optimization_defaults
from test_densify_gpu import LOOP, PIPE, cfg_of, grad_threshold, inputs

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KEYS = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation")
N_PLAIN, N_DENSIFY = 12, 40


def run(tr, views, record):
    for v in views:
        tr.step(v)
        record.append((tr.loss_value().clone(), tr.P))
    torch.cuda.synchronize()
    return tr


def snapshot(tr):
    s = {f"{b}_{k}": tr.view(getattr(tr, b), k).clone() for b in ("params", "exp_avg", "exp_avg_sq") for k in KEYS}
    s.update(poses=tr.poses.clone(), pose_m=tr.pose_m.clone(), pose_v=tr.pose_v.clone(),
             steps={k: tr.step_count(k) for k in KEYS + ("pose",)}, iteration=tr.iteration, opt_step=tr.opt_step,
             active_sh_degree=tr.active_sh_degree, stats=None if tr._stats is None else tr._stats.clone(),
             filter_3D=None if tr.filter_3D is None else tr.filter_3D.clone(),
             ppl=None if tr.per_point_lr is None else tr.per_point_lr[:tr.P].clone(),
             events=(list(tr.densified_at), list(tr.reset_at), list(tr.mip_recomputed_at)),
             gen=None if tr._stats is None else tr.densify_generator.get_state())
    return s


def assert_same(a, b):
    assert a.keys() == b.keys()
    for k in a:
        if torch.is_tensor(a[k]):
            assert torch.equal(a[k], b[k]), k
        else:
            assert a[k] == b[k], (k, a[k], b[k])


_FULL = {}


def full_run(key, sc, gts, cfg, views, use_graph):
    if key not in _FULL:
        rec = []
        tr = run(I.JointTrainer(sc, DEV, gt_images=gts, cfg=cfg, use_graph=use_graph), views, rec)
        _FULL[key] = (snapshot(tr), rec)
    return _FULL[key]


def resumed_run(sc, gts, cfg, views, k, use_graph, path):
    rec = []
    a = run(I.JointTrainer(sc, DEV, gt_images=gts, cfg=cfg, use_graph=use_graph), views[:k], rec)
    a.save_checkpoint(path)
    del a
    b = I.JointTrainer.from_checkpoint(path, sc, gt_images=gts, device=DEV, use_graph=use_graph)
    assert b.iteration == k and b.cap == 0 and not b._graphs
    run(b, views[k:], rec)
    return b, rec


def check_resume(full, rec, b):
    snap, rec_full = full
    assert len(rec) == len(rec_full)
    for i, ((la, pa), (lb, pb)) in enumerate(zip(rec_full, rec)):
        assert pa == pb and torch.equal(la, lb), (i + 1, pa, pb, float(la), float(lb))
    assert_same(snap, snapshot(b))


# ---- 1. bit-identical resume ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("use_graph", [False, True])
def test_resume_is_bit_identical_plain(use_graph, tmp_path):
    sc, gts, _ = inputs(P=12_000, seed=71)
    cfg = I.OptimConfig()
    cfg.iterations = 1000
    views = [i % sc.n_views for i in range(N_PLAIN)]
    full = full_run(("plain", use_graph), sc, gts, cfg, views, use_graph)
    assert sc.per_point_lr is not None and full[0]["ppl"] is not None
    b, rec = resumed_run(sc, gts, cfg, views, 5, use_graph, str(tmp_path / "chkpnt5.pth"))
    if use_graph:
        assert len(b._graphs) > 0
    check_resume(full, rec, b)


def densify_case():
    sc, gts, _ = inputs(P=15_000, seed=72, white=True)
    sc.sh_degree = 1                              # active degree 1 -> 2 -> 3 at iterations 12 and 24
    # an extent that puts the median Gaussian at the clone / split boundary, so that every event draws split samples
    extent = float(torch.exp(sc.params["scaling"]).max(1).values.median()) / 0.01
    cfg = cfg_of(densify_clone_split=True, densify_grad_threshold=grad_threshold(sc, gts), mip_kernel_size=0.1,
                 mip_filter3d_interval=7, sh_increase_interval=12, scene_extent=extent, **LOOP)
    return sc, gts, cfg


# k: white-background reset at 5; one before the densify at 10 and right after it; between the Mip recomputes at 14 and
# 21; on the SH-degree step at 24 (densify events at 10, 15, ..., 35, resets at 5 and 20)
@pytest.mark.parametrize("k", [5, 9, 10, 17, 24])
def test_resume_is_bit_identical_densify_mip_white(k, tmp_path):
    sc, gts, cfg = densify_case()
    views = [i % sc.n_views for i in range(N_DENSIFY)]
    full = full_run("densify", sc, gts, cfg, views, False)
    snap = full[0]
    assert snap["events"][0] == [10, 15, 20, 25, 30, 35] and snap["events"][1] == [5, 20]
    assert snap["events"][2] == [7, 14, 21, 28, 35] and snap["active_sh_degree"] == 3
    assert len(set(p for _, p in full[1])) > 2 and snap["steps"]["xyz"] < snap["steps"]["pose"]
    assert not torch.equal(snap["gen"], torch.Generator(device=DEV).manual_seed(cfg.densify_seed).get_state())
    b, rec = resumed_run(sc, gts, cfg, views, k, False, str(tmp_path / f"chkpnt{k}.pth"))
    check_resume(full, rec, b)


# ---- 2. the tuple is the reference's ---------------------------------------------------------------------------------
def test_capture_restores_into_the_mirror():
    sc, gts, cfg = densify_case()
    tr = run(I.JointTrainer(sc, DEV, gt_images=gts, cfg=cfg), [i % sc.n_views for i in range(22)], [])
    cap = tr.capture()
    assert isinstance(cap[1], torch.nn.Parameter) and cap[1].is_cuda and cap[12].requires_grad
    gm = GaussianModel(3, DEV)
    gm.restore(cap, optimization_defaults(iterations=cfg.iterations))
    shapes = tr._shapes()
    for k in KEYS:
        p = getattr(gm, gm._ATTR[k])
        assert tuple(p.shape) == shapes[k] and torch.equal(p.detach().reshape(tr.P, -1), tr.view(tr.params, k)), k
    assert torch.equal(gm.P.detach(), tr.poses) and gm.active_sh_degree == tr.active_sh_degree
    assert torch.equal(gm.xyz_gradient_accum, tr.xyz_gradient_accum) and torch.equal(gm.denom, tr.denom)
    assert torch.equal(gm.max_radii2D, tr.max_radii2D)
    sd = gm.optimizer.state_dict()
    names = [g["name"] for g in sd["param_groups"]]
    assert names == list(KEYS) + ["pose"] and type(gm.optimizer) is torch.optim.Adam
    assert [g["lr"] for g in sd["param_groups"]] == tr._group_lrs()
    assert torch.equal(sd["param_groups"][0]["per_point_lr"][:, 0], tr.per_point_lr[:tr.P])
    for i, g in enumerate(sd["param_groups"]):
        st = sd["state"][i]
        assert int(st["step"]) == tr.step_count(g["name"]), g["name"]
        if g["name"] == "pose":
            assert torch.equal(st["exp_avg"], tr.pose_m) and torch.equal(st["exp_avg_sq"], tr.pose_v)
        else:
            assert torch.equal(st["exp_avg"].reshape(tr.P, -1), tr.view(tr.exp_avg, g["name"]))
            assert torch.equal(st["exp_avg_sq"].reshape(tr.P, -1), tr.view(tr.exp_avg_sq, g["name"]))
    assert tr.step_count("opacity") < tr.step_count("xyz") < tr.step_count("pose")


def test_capture_without_densify_or_pose_optimisation():
    sc, gts, _ = inputs(P=4000, seed=73)
    cfg = I.OptimConfig()
    cfg.optim_pose = False
    tr = run(I.JointTrainer(sc, DEV, gt_images=gts, cfg=cfg), [0, 1, 2], [])
    cap = tr.capture()
    sd = cap[10]
    assert sorted(sd["state"]) == list(range(6))           # the pose group has no state, as in the reference
    assert all(float(t.abs().sum()) == 0 for t in cap[7:10])
    assert sd[I.CHECKPOINT_KEY]["densify_generator"] is None and sd[I.CHECKPOINT_KEY]["filter_3D"] is None


# ---- 3. a checkpoint without JointTrainer's state ------------------------------------------------------------------
def mirror_steps(gm, gts, cams, bg, cfg, views, first, losses):
    if os.path.join(ROOT, "shims") not in sys.path:
        sys.path.insert(0, os.path.join(ROOT, "shims"))
    from fused_ssim import fused_ssim
    for i, v in enumerate(views):
        iteration = first + 1 + i
        gm.update_learning_rate(iteration)
        pkg = I.render(cams[v], gm, PIPE, bg, camera_pose=gm.get_RT(v))
        image = pkg["render"]
        loss = (1.0 - cfg.lambda_dssim) * torch.abs(image - gts[v]).mean() + \
            cfg.lambda_dssim * (1.0 - fused_ssim(image.unsqueeze(0), gts[v].unsqueeze(0)))
        loss.backward()
        losses.append(loss.item())
        with torch.no_grad():
            gm.optimizer.step()
            gm.optimizer.zero_grad(set_to_none=True)
            gm.P.grad = None


def test_mirror_checkpoint_resumes_in_the_trainer(tmp_path):
    sc, gts, cams = inputs(P=15_000, seed=74)
    cfg = I.OptimConfig()
    cfg.iterations = 1000
    bg = sc.bg.to(DEV)
    gm = GaussianModel.from_scene(sc, DEV)
    gm.training_setup_pp(optimization_defaults(iterations=cfg.iterations), sc.per_point_lr.to(DEV).reshape(-1, 1))
    views = [i % sc.n_views for i in range(20)]
    mirror_steps(gm, gts, cams, bg, cfg, views[:10], 0, [])
    path = str(tmp_path / "chkpnt10.pth")
    torch.save((gm.capture(), 10), path)
    # a checkpoint without JointTrainer's state carries no OptimConfig: pass the run's (iterations sets the pose schedule)
    tr = I.JointTrainer.from_checkpoint(path, sc, gt_images=gts, cfg=cfg, device=DEV)
    assert tr.iteration == 10 and tr.opt_step == 10 and all(tr.step_count(k) == 10 for k in KEYS)
    assert torch.equal(tr.per_point_lr[:tr.P], gm.per_point_lr[:, 0])
    l_m, l_t = [], []
    mirror_steps(gm, gts, cams, bg, cfg, views[10:], 10, l_m)
    for v in views[10:]:
        tr.step(v)
        l_t.append(float(tr.loss_value()))
    assert type(gm.optimizer) is I.PerPointAdam
    d = max(abs(a - b) for a, b in zip(l_m, l_t))
    assert d < 1e-5, (d, l_m, l_t)
    for k in KEYS:
        diff = (tr.view(tr.params, k) - getattr(gm, gm._ATTR[k]).detach().reshape(tr.P, -1)).abs()
        assert float((diff > 1e-3).float().mean()) < 2e-3 and float(diff.max()) < 0.3, (k, float(diff.max()))


def test_checkpoint_without_extra_state_derives_it(tmp_path):
    sc, gts, cfg = densify_case()
    tr = run(I.JointTrainer(sc, DEV, gt_images=gts, cfg=cfg), [i % sc.n_views for i in range(22)], [])
    cap = tr.capture()
    del cap[10][I.CHECKPOINT_KEY]
    path = str(tmp_path / "bare.pth")
    torch.save((cap, tr.iteration), path)
    b = I.JointTrainer.from_checkpoint(path, sc, gt_images=gts, cfg=cfg, device=DEV)
    assert b.opt_step == tr.opt_step and all(b.step_count(k) == tr.step_count(k) for k in KEYS + ("pose",))
    ref = torch.empty_like(b.filter_3D)
    I.frame.mip_filter3d(b.view(b.params, "xyz"), b.poses, b.W, b.H, b.ident.tanfovx, b.ident.tanfovy, out=ref)
    assert torch.equal(b.filter_3D, ref)                   # recomputed from the restored xyz and poses
    g0 = torch.Generator(device=DEV).manual_seed(cfg.densify_seed)
    assert torch.equal(b.densify_generator.get_state(), g0.get_state())
    assert b.densified_at == [] and type(b) is I.JointTrainer


# ---- 4. render.py's inputs -----------------------------------------------------------------------------------------
def test_save_ply_and_poses_round_trip(tmp_path):
    sc, gts, cfg = densify_case()
    tr = run(I.JointTrainer(sc, DEV, gt_images=gts, cfg=cfg), [i % sc.n_views for i in range(12)], [])
    ply = str(tmp_path / "point_cloud" / "iteration_12" / "point_cloud.ply")
    tr.save_ply(ply)
    d = scene_io.load_gaussians_ply(ply)
    shapes = tr._shapes()
    for k in KEYS:
        assert d[k].shape == shapes[k], k
        assert torch.equal(torch.from_numpy(d[k]).reshape(tr.P, -1), tr.view(tr.params, k).cpu()), k
    assert "filter_3D" in d and torch.equal(torch.from_numpy(d["filter_3D"])[:, 0], tr.filter_3D.cpu())
    ids = [3, 1, 2]
    npy = str(tmp_path / "pose" / "ours_12" / "pose_optimized.npy")
    mats = tr.save_poses(npy, colmap_ids=ids)
    back = np.load(npy)
    assert np.array_equal(back, mats) and back.shape == (3, 4, 4)
    poses = tr.poses.cpu().numpy()
    for i in range(3):
        assert np.array_equal(back[i], scene_io.pose7_to_matrix(poses[ids.index(i + 1)]).astype(np.float32))
    plain = run(I.JointTrainer(sc, DEV, gt_images=gts), [0], [])
    plain.save_ply(str(tmp_path / "plain.ply"))
    assert "filter_3D" not in scene_io.load_gaussians_ply(str(tmp_path / "plain.ply"))


# ---- 5. refusals ---------------------------------------------------------------------------------------------------
def test_refusals(tmp_path):
    sc, gts, _ = inputs(P=4000, seed=75)
    tr = run(I.JointTrainer(sc, DEV, gt_images=gts), [0, 1], [])
    path = str(tmp_path / "c.pth")
    tr.save_checkpoint(path)
    multi = I.JointTrainer(sc, DEV, world_size=2, rank=0)
    with pytest.raises(I.GsbError, match="world_size"):
        multi.capture()
    with pytest.raises(I.GsbError, match="world_size"):
        multi.load_checkpoint(path)
    two = I.scenes.Scene({k: v.clone() for k, v in sc.params.items()}, sc.poses[:2].clone(), sc.width, sc.height,
                         sc.fovx, sc.fovy, sc.sh_degree, sc.bg.clone(), sc.per_point_lr)
    with pytest.raises(I.GsbError, match="pose table has 3 views"):
        I.JointTrainer.from_checkpoint(path, two, device=DEV)
    other = I.scenes.Scene(sc.params, sc.poses, sc.width + 16, sc.height, sc.fovx, sc.fovy, sc.sh_degree, sc.bg,
                           sc.per_point_lr)
    with pytest.raises(I.GsbError, match="another frame.*W"):
        I.JointTrainer.from_checkpoint(path, other, device=DEV)
    cap = tr.capture()
    cap = list(cap)
    cap[3] = cap[3][:, :8].contiguous()                       # SH degree 2
    for m in ("exp_avg", "exp_avg_sq"):
        cap[10]["state"][2][m] = cap[10]["state"][2][m][:, :8].contiguous()
    torch.save((tuple(cap), 2), path)
    with pytest.raises(I.GsbError, match="SH layout"):
        tr.load_checkpoint(path)
    cap = list(tr.capture())
    del cap[10][I.CHECKPOINT_KEY]["opt_step"]
    torch.save((tuple(cap), 2), path)
    with pytest.raises(I.GsbError, match="lacks"):
        tr.load_checkpoint(path)
    cap = list(tr.capture())
    cap[10][I.CHECKPOINT_KEY]["lag"]["opacity"] = 1
    torch.save((tuple(cap), 2), path)
    with pytest.raises(I.GsbError, match="step counts"):
        tr.load_checkpoint(path)
