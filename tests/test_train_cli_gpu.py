"""The training stage on the GPU (-m gpu, DESIGN.md section 4.14): the loaded scene against create_from_pcd and the
reference golden, the CLI against a JointTrainer(use_graph=True) driven directly with view_schedule (bit for bit:
ply, pose files, checkpoints, per-iteration losses), the first iterations against train.py's loop on the drop-ins,
--start_checkpoint, and stages 2 -> 5 of run_eval.sh end to end."""
import json
import os
import sys

import numpy as np
import pytest
import torch

import instantsplat_b200 as I
from instantsplat_b200 import metrics as M
from instantsplat_b200 import render_views as R
from instantsplat_b200 import scene_io as S
from instantsplat_b200 import train as T
from instantsplat_b200.model import GaussianModel
from instantsplat_b200.scenes import surface_scene
from instantsplat_b200.tracking import PoseTracker

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _source(root, P=3000, n=3, W=80, H=56, seed=41):
    """An init_geo-shaped source whose images are renders of the scene; its points3D.ply holds the scene's points."""
    sc = surface_scene(P, n, W, H, seed=seed, sh_degree=3)
    p = sc.params
    truth = PoseTracker(p["xyz"], p["rotation"], p["scaling"], p["opacity"], p["f_dc"], p["f_rest"], W, H, sc.fovx,
                        sc.fovy, sh_degree=3, device=DEV)
    from instantsplat_b200.freeview import quantise
    imgs = quantise(truth.render_batch(sc.poses).contiguous()).cpu().numpy()
    S.write_synthetic_source(root, sc, imgs)
    return root


def _args(src, model, *extra):
    return T.parse_args(["-s", src, "-m", model, "-r", "1", "--n_views", "3", "--quiet"] + list(extra))


def _same(a, b, path="") -> None:
    if torch.is_tensor(a):
        assert torch.is_tensor(b) and a.dtype == b.dtype and torch.equal(a.detach().cpu(), b.detach().cpu()), path
    elif isinstance(a, dict):
        assert a.keys() == b.keys(), path
        for k in a:
            _same(a[k], b[k], f"{path}.{k}")
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b), path
        for i, (x, y) in enumerate(zip(a, b)):
            _same(x, y, f"{path}[{i}]")
    else:
        assert a == b, (path, a, b)


def _drive(tr, rows, it0, args, model, ids):
    """JointTrainer driven with the schedule, saving where the CLI saves; returns the per-iteration losses."""
    losses = []
    for k, row in enumerate(rows):
        it = it0 + 1 + k
        tr.step(row)
        losses.append(tr.loss_value().clone())
        if it in args.save_iterations:
            tr.save_ply(os.path.join(model, "point_cloud", f"iteration_{it}", "point_cloud.ply"))
            tr.save_poses(os.path.join(model, "pose", f"ours_{it}", "pose_optimized.npy"), ids)
        if it in args.checkpoint_iterations:
            tr.save_checkpoint(os.path.join(model, f"chkpnt{it}.pth"))
    torch.cuda.synchronize()
    return torch.stack(losses).cpu()


def _compare_models(a, b, its, ckpts):
    rd = lambda *p: open(os.path.join(*p), "rb").read()
    for it in its:
        assert rd(a, "point_cloud", f"iteration_{it}", "point_cloud.ply") == rd(b, "point_cloud", f"iteration_{it}",
                                                                                 "point_cloud.ply"), it
        assert rd(a, "pose", f"ours_{it}", "pose_optimized.npy") == rd(b, "pose", f"ours_{it}", "pose_optimized.npy")
    for it in ckpts:
        _same(torch.load(os.path.join(a, f"chkpnt{it}.pth")), torch.load(os.path.join(b, f"chkpnt{it}.pth")))


# ---- 1. the scene -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("scaled", [False, True])
def test_scene_matches_create_from_pcd_and_golden(golden_dir, tmp_path, scaled):
    z = np.load(os.path.join(golden_dir, "train.npz"))
    src = tmp_path / "src"
    for i, rel in enumerate(z["src_files"]):
        p = src / str(rel)
        p.parent.mkdir(parents=True, exist_ok=True)
        p.write_bytes(z[f"src_blob_{i}"].tobytes())
    ts = T.load_training_scene(str(src), 4, 1, init_scale_from_view_depth=scaled)
    h = ts.host
    gm = GaussianModel(3, DEV)
    xyz, rgb, _ = S.read_points3d_ply(h.ply_path)
    gm.create_from_pcd(xyz, rgb / 255.0, h.extent, h.scale_gaussian)
    for name, attr in GaussianModel._ATTR.items():
        assert torch.equal(ts.scene.params[name], getattr(gm, attr).detach()), name
    tag = "init_scaled" if scaled else "init"
    got = lambda k: ts.scene.params[k].cpu().numpy()
    for k, ref in (("xyz", "_xyz"), ("f_rest", "_features_rest"), ("rotation", "_rotation")):
        assert np.array_equal(got(k), z[f"{tag}{ref}"]), k
    # RGB2SH's division and inverse_sigmoid's log round differently on the GPU than on the CPU the golden ran on
    np.testing.assert_allclose(got("f_dc"), z[f"{tag}_features_dc"], rtol=2.5e-7, atol=0)
    np.testing.assert_allclose(got("opacity"), z[f"{tag}_opacity"], rtol=1e-6, atol=0)
    # log sqrt of the knn mean: the GPU knn sums its fp32 squared distances in another order than the CPU stand-in
    np.testing.assert_allclose(got("scaling"), z[f"{tag}_scaling"], rtol=0, atol=1e-4)
    assert torch.equal(ts.scene.poses, torch.from_numpy(z["P"]))
    assert ts.scene.sh_degree == 0 and torch.equal(ts.scene.bg, torch.zeros(3))
    assert tuple(ts.targets.shape) == (4, 3, h.views.height, h.views.width)
    for r, i in enumerate(h.order):
        assert torch.equal(ts.targets[r], torch.from_numpy(h.views.images[i]).to(DEV).permute(2, 0, 1) / 255.0)


# ---- 2. the CLI adds nothing ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("white,iterations", [(False, 1004), (True, 25)])
def test_cli_equals_joint_trainer_driven_directly(tmp_path, white, iterations):
    src = _source(str(tmp_path / "src"), P=2000, W=64, H=48)
    extra = ["--iterations", str(iterations), "--pp_optimizer", "--optim_pose", "--save_iterations", "12",
             "--checkpoint_iterations", "12", "20"] + (["-w"] if white else [])
    args = _args(src, str(tmp_path / "cli"), *extra)
    res = T.run(args)
    assert res.first_iter == 0 and res.rows == T.view_schedule(3, iterations)[1]
    assert res.trainer.opt_step == iterations - 1                  # the last iteration takes no Adam step
    if iterations > 1000:
        assert res.trainer.active_sh_degree == 1                   # oneupSHdegree at 1000
    ts = T.load_training_scene(src, 3, 1, white_background=white)
    tr = I.JointTrainer(ts.scene, DEV, gt_images=ts.targets, cfg=T.optim_config(args, ts.host.extent), use_graph=True)
    direct = str(tmp_path / "direct")
    for it in args.save_iterations:
        tr.save_poses(os.path.join(direct, "pose", f"ours_{it}", "pose_org.npy"), ts.host.colmap_ids)
    losses = _drive(tr, T.view_schedule(3, iterations)[1], 0, args, direct, ts.host.colmap_ids)
    assert torch.equal(res.losses, losses)
    _compare_models(args.model_path, direct, [12, iterations], [12, 20])
    for it in (12, iterations):
        rd = lambda m: open(os.path.join(m, "pose", f"ours_{it}", "pose_org.npy"), "rb").read()
        assert rd(args.model_path) == rd(direct)
    files = sorted(os.listdir(args.model_path))
    assert files == ["cameras.json", "cfg_args", "chkpnt12.pth", "chkpnt20.pth", "input.ply", "point_cloud", "pose",
                     "train_time.txt"]
    lines = open(os.path.join(args.model_path, "train_time.txt")).read().splitlines()
    assert [l.split(":")[0] for l in lines] == ["[2] train_joint_TrainTime", "[2] train_joint"]
    assert "white_background=%s" % white in open(os.path.join(args.model_path, "cfg_args")).read()


# ---- 3. the drop-in loop -------------------------------------------------------------------------------------------
def test_first_iterations_agree_with_the_reference_loop(tmp_path):
    """20 iterations of the CLI against train.py:140-211 on the mirror GaussianModel (test_reference_loop.py), built
    from the same scene, rows and targets.  On this create_from_pcd initialisation the largest difference measured was
    2.4e-5, above test_three_ways_of_running_the_loop_agree's 1e-5 on its perturbed scene; the bar here is 5e-5."""
    sys.path.insert(0, os.path.join(ROOT, "shims"))
    from instantsplat_b200.camera import SimpleCamera
    from test_reference_loop import reference_loop
    src = _source(str(tmp_path / "src"), P=20_000, W=160, H=112, seed=43)
    n = 20
    res = T.run(_args(src, str(tmp_path / "cli"), "--iterations", str(n), "--pp_optimizer", "--optim_pose"))
    ts = T.load_training_scene(src, 3, 1)
    gm = GaussianModel(3, DEV)
    gm.create_from_pcd(ts.host.points, ts.host.colors, ts.host.extent)
    gm.init_RT_seq(ts.host.poses)
    gm.training_setup_pp(I.optimization_defaults(iterations=n), ts.host.per_point_lr.to(DEV))
    cams = []
    for v in range(3):
        c = SimpleCamera(ts.scene.width, ts.scene.height, ts.scene.fovx, ts.scene.fovy, device=DEV)
        c.uid = v
        cams.append(c)
    ref = reference_loop(gm, I.render, res.rows, ts.targets, cams, n, iterations=n)
    assert ref[-1] < ref[0]
    d = max(abs(a - b) for a, b in zip(ref, res.losses.tolist()))
    assert d < 5e-5, (d, ref, res.losses.tolist())


# ---- 4. resume -----------------------------------------------------------------------------------------------------
def test_start_checkpoint(tmp_path):
    src = _source(str(tmp_path / "src"), P=2500, W=64, H=48, seed=44)
    N, k = 30, 12
    a = _args(src, str(tmp_path / "first"), "--iterations", str(N), "--pp_optimizer", "--optim_pose",
              "--checkpoint_iterations", str(k))
    T.run(a)
    ck = os.path.join(a.model_path, f"chkpnt{k}.pth")
    b = _args(src, str(tmp_path / "resumed"), "--iterations", str(N), "--pp_optimizer", "--optim_pose",
              "--save_iterations", "5", "20", "--start_checkpoint", ck)
    res = T.run(b)
    assert res.first_iter == k and res.rows == T.view_schedule(3, N, k)[1] != T.view_schedule(3, N)[1][k:]
    ts = T.load_training_scene(src, 3, 1)
    tr = I.JointTrainer.from_checkpoint(ck, ts.scene, gt_images=ts.targets, cfg=T.optim_config(b, ts.host.extent),
                                        device=DEV, use_graph=True)
    restored = tr.poses.clone()
    direct = str(tmp_path / "direct")
    losses = _drive(tr, T.view_schedule(3, N, k)[1], k, b, direct, ts.host.colmap_ids)
    assert torch.equal(res.losses, losses)
    _compare_models(b.model_path, direct, [20, N], [])
    for it in (5, 20, N):                      # pose_org.npy: the restored table, past save points included
        org = np.load(os.path.join(b.model_path, "pose", f"ours_{it}", "pose_org.npy"))
        want = S.save_pose_npy(os.path.join(direct, "org.npy"), restored.detach().cpu().numpy(), ts.host.colmap_ids)
        assert np.array_equal(org, want)
    assert not os.path.isdir(os.path.join(b.model_path, "point_cloud", "iteration_5"))


# ---- 5. stages 2 -> 5 of run_eval.sh -------------------------------------------------------------------------------
def test_stages_2_to_5(tmp_path, capsys):
    from test_render_views_gpu import _source_and_model
    src, _, _ = _source_and_model(str(tmp_path))
    model = str(tmp_path / "trained")
    it = 300
    assert T.main(["-s", src, "-m", model, "-r", "1", "--n_views", "3", "--iterations", str(it), "--pp_optimizer",
                   "--optim_pose", "--test_iterations", str(it), "--checkpoint_iterations", "100"]) == 0
    out = capsys.readouterr().out
    assert f"[ITER {it}] Evaluating train: L1" in out and "[ITER 10] Loss" in out and "Training complete." in out
    for f in ("cfg_args", "input.ply", "cameras.json", "train_time.txt", "chkpnt100.pth",
              f"pose/ours_{it}/pose_org.npy", f"pose/ours_{it}/pose_optimized.npy",
              f"point_cloud/iteration_{it}/point_cloud.ply"):
        assert os.path.isfile(os.path.join(model, f)), f
    base = ["-s", src, "-m", model, "--n_views", "3", "--iterations", str(it), "-r", "1", "--workers", "2"]
    assert R.main(base) == 0
    assert R.main(base + ["--eval", "--optim_test_pose_iter", "20"]) == 0
    assert M.main(["-s", src, "-m", model, "--n_views", "3"]) == 0
    res = json.loads(open(os.path.join(model, "results.json")).read())[f"ours_{it}"]
    assert np.isfinite(res["PSNR"]) and np.isfinite(res["ATE"])
    assert len(os.listdir(os.path.join(model, "train", f"ours_{it}", "renders"))) == 3
    # the loss falls and the trained model beats the initial one on the training views
    args = _args(src, str(tmp_path / "again"), "--iterations", str(it), "--pp_optimizer", "--optim_pose")
    r = T.run(args)
    assert float(r.losses[-20:].mean()) < 0.8 * float(r.losses[:20].mean())
    ts = T.load_training_scene(src, 3, 1)
    init = I.JointTrainer(ts.scene, DEV, gt_images=ts.targets, cfg=T.optim_config(args, ts.host.extent))
    p0 = float(init.evaluate()["psnr"].mean())
    p1 = float(r.trainer.evaluate()["psnr"].mean())
    assert p1 > p0 + 1.0, (p0, p1)
