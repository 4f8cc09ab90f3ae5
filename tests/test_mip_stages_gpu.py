"""Mip-Splatting through the stage command lines on the GPU (-m gpu, DESIGN.md section 4.22): `train --kernel_size`
against a Mip JointTrainer(use_graph=True) driven directly (ply with filter_3D, pose files, checkpoints, per-iteration
losses, the 3D-filter recompute), --start_checkpoint with the flag against from_checkpoint, the render stages, the
fly-through and the frame-rate loop against a PoseTracker built with kernel_size and the ply's filter_3D, rendering
at another scale than the one trained at, and `pipeline eval|infer --kernel_size` against the stage CLIs."""
import contextlib
import os
import shutil

import numpy as np
import pytest
import torch

import instantsplat_b200 as I
from instantsplat_b200 import freeview as F
from instantsplat_b200 import metrics as M
from instantsplat_b200 import pipeline as P
from instantsplat_b200 import render_views as R
from instantsplat_b200 import scene_io as S
from instantsplat_b200 import train as T
from instantsplat_b200.frame import mip_filter3d
from instantsplat_b200.tracking import PoseTracker

pytestmark = pytest.mark.gpu
DEV = "cuda"
K = ["--kernel_size", "0.1"]


def _ply(model, it):
    return os.path.join(model, "point_cloud", f"iteration_{it}", "point_cloud.ply")


def _tracker(ply, W, H, fovx, fovy, kernel_size=None):
    """The tracker a user would build by hand: PoseTracker over the ply's tensors, with kernel_size and the
    ply's filter_3D when kernel_size is given, else with no filter."""
    g = {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in S.load_gaussians_ply(ply).items()}
    kw = {} if kernel_size is None else dict(kernel_size=kernel_size, filter_3D=g["filter_3D"])
    return PoseTracker(g["xyz"], g["rotation"], g["scaling"], g["opacity"], g["f_dc"], g["f_rest"], W, H, fovx, fovy,
                       sh_degree=3, device=DEV, **kw)


def _view_tracker(ply, views, kernel_size=None):
    return _tracker(ply, views.width, views.height, views.fovx, views.fovy, kernel_size)


def _all(chunks):
    return np.concatenate([c for _, c in chunks])


def _read(folder, names):
    from PIL import Image
    return np.stack([np.asarray(Image.open(os.path.join(folder, n))) for n in names])


def _files(root):
    out = []
    for d, _, fs in os.walk(root):
        out += [os.path.relpath(os.path.join(d, f), root) for f in fs]
    return sorted(out)


# ---- 1. train ------------------------------------------------------------------------------------------------------
def test_train_cli_equals_mip_joint_trainer_driven_directly(tmp_path):
    from test_train_cli_gpu import _compare_models, _drive, _source
    src = _source(str(tmp_path / "src"), P=2000, W=64, H=48)
    N = 230                                      # a 3D-filter recompute at 100; none at 200, within the last 100
    args = T.parse_args(["-s", src, "-m", str(tmp_path / "cli"), "-r", "1", "--n_views", "3", "--iterations", str(N),
                         "--pp_optimizer", "--optim_pose", "--save_iterations", "12", "--checkpoint_iterations", "12",
                         "150", "--test_iterations", str(N)] + K)
    lines = []
    res = T.run(args, log=lambda *a: lines.append(" ".join(map(str, a))))
    assert res.rows == T.view_schedule(3, N)[1] and res.trainer.mip_recomputed_at == [100]
    ts = T.load_training_scene(src, 3, 1)
    cfg = T.optim_config(args, ts.host.extent)
    assert cfg.mip_kernel_size == 0.1
    tr = I.JointTrainer(ts.scene, DEV, gt_images=ts.targets, cfg=cfg, use_graph=True)
    direct = str(tmp_path / "direct")
    for it in args.save_iterations:
        tr.save_poses(os.path.join(direct, "pose", f"ours_{it}", "pose_org.npy"), ts.host.colmap_ids)
    losses = _drive(tr, T.view_schedule(3, N)[1], 0, args, direct, ts.host.colmap_ids)
    assert tr.mip_recomputed_at == [100]
    assert torch.equal(res.losses, losses)
    _compare_models(args.model_path, direct, [12, N], [12, 150])
    for it in (12, N):
        rd = lambda m: open(os.path.join(m, "pose", f"ours_{it}", "pose_org.npy"), "rb").read()
        assert rd(args.model_path) == rd(direct)
        assert S.ply_properties(_ply(args.model_path, it))[-1] == "filter_3D"
    saved = S.load_gaussians_ply(_ply(args.model_path, N))["filter_3D"]
    assert np.array_equal(saved.reshape(-1), tr.filter_3D.cpu().numpy()) and (saved > 0).any()
    m = tr.evaluate()
    want = f"\n[ITER {N}] Evaluating train: L1 {sum(m['l1'].tolist()) / 3} PSNR {sum(m['psnr_channels'].mean(1).tolist()) / 3}"
    assert want in lines
    assert "kernel" not in open(os.path.join(args.model_path, "cfg_args")).read()


# ---- 2. resume -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("first_mip", [True, False])
def test_start_checkpoint_with_the_flag(tmp_path, first_mip):
    """A Mip checkpoint resumes with its filter; one from a run without Mip gets the filter recomputed from the
    restored xyz and poses.  Either way the CLI equals from_checkpoint driven with view_schedule(n, N, k)."""
    from test_train_cli_gpu import _compare_models, _drive, _source
    src = _source(str(tmp_path / "src"), P=2500, W=64, H=48, seed=44)
    N, k = 30, 12
    a = T.parse_args(["-s", src, "-m", str(tmp_path / "first"), "-r", "1", "--n_views", "3", "--iterations", str(N),
                      "--pp_optimizer", "--optim_pose", "--checkpoint_iterations", str(k), "--quiet"]
                     + (K if first_mip else []))
    T.run(a)
    ck = os.path.join(a.model_path, f"chkpnt{k}.pth")
    b = T.parse_args(["-s", src, "-m", str(tmp_path / "resumed"), "-r", "1", "--n_views", "3", "--iterations", str(N),
                      "--pp_optimizer", "--optim_pose", "--save_iterations", "20", "--start_checkpoint", ck, "--quiet"]
                     + K)
    res = T.run(b)
    assert res.first_iter == k and res.rows == T.view_schedule(3, N, k)[1]
    ts = T.load_training_scene(src, 3, 1)
    tr = I.JointTrainer.from_checkpoint(ck, ts.scene, gt_images=ts.targets, cfg=T.optim_config(b, ts.host.extent),
                                        device=DEV, use_graph=True)
    f0 = tr.filter_3D.clone()
    if not first_mip:
        want = mip_filter3d(tr.view(tr.params, "xyz"), tr.poses, tr.W, tr.H, tr.ident.tanfovx, tr.ident.tanfovy)
        assert torch.equal(f0, want)
    direct = str(tmp_path / "direct")
    losses = _drive(tr, T.view_schedule(3, N, k)[1], k, b, direct, ts.host.colmap_ids)
    assert torch.equal(res.losses, losses)
    _compare_models(b.model_path, direct, [20, N], [])
    # no recompute between k and N (N - 100 < 100): the ply holds the filter the restore left
    saved = S.load_gaussians_ply(_ply(b.model_path, N))["filter_3D"]
    assert np.array_equal(saved.reshape(-1), f0.cpu().numpy())


# ---- 3-5. the render stages, the scales, the fly-through and the frame rate ---------------------------------------
@pytest.fixture(scope="module")
def mip_model(tmp_path_factory):
    """test_render_views_gpu's render.py source (3 training views, 4 test views, 96 x 64) and a model trained on it by
    `train --kernel_size 0.1`."""
    from test_render_views_gpu import _source_and_model
    root = str(tmp_path_factory.mktemp("mip"))
    src, _, _ = _source_and_model(root)
    model, it = os.path.join(root, "mip_model"), 30
    with contextlib.redirect_stdout(open(os.devnull, "w")):
        assert T.main(["-s", src, "-m", model, "-r", "1", "--n_views", "3", "--iterations", str(it), "--pp_optimizer",
                       "--optim_pose", "--quiet"] + K) == 0
    return src, model, it


def test_render_stages(mip_model, tmp_path, capsys):
    src, model, it = mip_model
    copy = lambda name: shutil.copytree(model, str(tmp_path / name))
    mip, plain, timed = copy("mip"), copy("plain"), copy("timed")
    base = ["-s", src, "--n_views", "3", "--iterations", str(it), "-r", "1", "--workers", "2"]
    ev = ["--eval", "--optim_test_pose_iter", "20", "--max_batch", "3"]
    for m, extra in ((mip, K), (plain, [])):
        assert R.main(base + ["-m", m] + extra) == 0
        assert R.main(base + ["-m", m] + ev + extra) == 0
    assert R.main(base + ["-m", timed] + ev + ["--test_fps"] + K) == 0
    assert ">>> FPS = " in capsys.readouterr().out
    ply = _ply(model, it)
    # training views at the optimised poses
    views = S.load_views(src, 3, 0)
    poses = F.poses_from_w2c(np.load(os.path.join(model, "pose", f"ours_{it}", "pose_optimized.npy")))
    idx = [f"{i:05d}.png" for i in range(3)]
    folder = lambda m, split: os.path.join(m, split, f"ours_{it}")
    got = _read(os.path.join(folder(mip, "train"), "renders"), idx)
    assert np.array_equal(got, _all(F.frames_u8(_view_tracker(ply, views, 0.1), poses)))
    assert np.array_equal(_read(os.path.join(folder(mip, "train"), "gt"), idx), views.images)
    no = _read(os.path.join(folder(plain, "train"), "renders"), idx)
    assert np.array_equal(no, _all(F.frames_u8(_view_tracker(ply, views), poses)))       # filters ignored, as today
    assert not np.array_equal(got, no)
    # test views: tracked, then rendered at their best poses
    tv = S.load_views(src, 3, 1)
    names = [n + ".png" for n in tv.names]
    init, gts = F.poses_from_w2c(tv.w2c), R.gt_images(tv, DEV)
    for m, k in ((mip, 0.1), (plain, None)):
        tk = _view_tracker(ply, tv, k)
        best, _ = tk.optimize_batch(init, gts, num_iter=20, max_batch=3)
        assert np.array_equal(_read(os.path.join(folder(m, "test"), "renders"), names), _all(F.frames_u8(tk, best, 3)))
        assert np.array_equal(_read(os.path.join(folder(m, "test"), "gt"), names), tv.images)
    assert not np.array_equal(_read(os.path.join(folder(mip, "test"), "renders"), names),
                              _read(os.path.join(folder(plain, "test"), "renders"), names))
    # --test_fps: total_fps.json, and every PNG the run without it wrote
    fa, fb = _files(mip), _files(timed)
    assert sorted(set(fb) - set(fa)) == ["total_fps.json"]                 # train_time.txt is the train stage's
    assert open(os.path.join(timed, "train_time.txt")).read().splitlines()[-1].startswith("[4] render: ")
    assert not open(os.path.join(mip, "train_time.txt")).read().count("[4] render")
    pngs = [rel for rel in fa if rel.startswith("test") and rel.endswith(".png")]
    assert len(pngs) == 8
    for rel in pngs:
        assert open(os.path.join(mip, rel), "rb").read() == open(os.path.join(timed, rel), "rb").read(), rel


def test_render_at_another_scale(mip_model, tmp_path):
    """Trained at -r 2 (48 x 32, resampled), the test views rendered at -r 1 (96 x 64) with the filters."""
    src, _, _ = mip_model
    model, it = str(tmp_path / "half"), 30
    with contextlib.redirect_stdout(open(os.devnull, "w")):
        assert T.main(["-s", src, "-m", model, "-r", "2", "--resample_images", "--n_views", "3", "--iterations",
                       str(it), "--pp_optimizer", "--optim_pose", "--quiet"] + K) == 0
        assert R.main(["-s", src, "-m", model, "--n_views", "3", "--iterations", str(it), "-r", "1", "--workers", "2",
                       "--eval", "--optim_test_pose_iter", "20"] + K) == 0
    tv = S.load_views(src, 3, 1)
    assert (tv.width, tv.height) == (96, 64)
    tk = _view_tracker(_ply(model, it), tv, 0.1)
    best, _ = tk.optimize_batch(F.poses_from_w2c(tv.w2c), R.gt_images(tv, DEV), num_iter=20, max_batch=12)
    names = [n + ".png" for n in tv.names]
    got = _read(os.path.join(model, "test", f"ours_{it}", "renders"), names)
    assert got.shape == (4, 64, 96, 3) and np.array_equal(got, _all(F.frames_u8(tk, best, 12)))


def test_fly_through(mip_model, tmp_path):
    src, model, it = mip_model
    a, b = str(tmp_path / "freeview"), str(tmp_path / "infer_video")
    shutil.copytree(model, a)
    shutil.copytree(model, b)
    with contextlib.redirect_stdout(open(os.devnull, "w")):
        assert F.main(["-s", src, "-m", a, "--n_views", "3", "--iterations", str(it), "--workers", "2"] + K) == 0
        assert R.main(["-s", src, "-m", b, "--n_views", "3", "--iterations", str(it), "--workers", "2",
                       "--infer_video"] + K) == 0
    W, H, fovx, fovy = F.intrinsics(src, 3)
    path = F.interpolated_w2c(np.load(os.path.join(model, "pose", f"ours_{it}", "pose_optimized.npy")), 3)
    want = _all(F.frames_u8(_tracker(_ply(model, it), W, H, fovx, fovy, 0.1), F.poses_from_w2c(path), 4))
    idx = [f"{i:05d}.png" for i in range(len(path))]
    assert np.array_equal(_read(os.path.join(a, "interp", f"ours_{it}", "renders"), idx), want)
    plain = _all(F.frames_u8(_tracker(_ply(model, it), W, H, fovx, fovy), F.poses_from_w2c(path), 4))
    assert not np.array_equal(want, plain)
    fa = _files(a)
    assert fa == _files(b)
    for rel in fa:
        assert open(os.path.join(a, rel), "rb").read() == open(os.path.join(b, rel), "rb").read(), rel


# ---- 6. the pipeline -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["eval", "infer"])
def test_pipeline_equals_the_stage_clis(mip_model, tmp_path, mode):
    from test_pipeline_gpu import _compare_trees, _data_root
    src, _, _ = mip_model
    root = _data_root(str(tmp_path / "data"), src, mode)
    out = str(tmp_path / "out")
    ts = P.tasks(mode, root, out, ["D"], ["A"], [3], [20])
    clis = {"train": T.main, "render_train": R.main, "render_test": R.main, "metrics": M.main, "render": R.main}
    for t in ts:
        os.makedirs(t.model, exist_ok=True)
        for key, argv in P.stage_argv(t, kernel_size=0.1).items():
            assert (key == "metrics") != (argv[-2:] == K), key
            with open(os.path.join(t.model, P.STAGES[t.mode][key][0]), "w") as f, \
                    contextlib.redirect_stdout(f), contextlib.redirect_stderr(f):
                clis[key](argv)
    os.rename(out, str(tmp_path / "cli"))
    argv = [mode, "--data_root", root, "--output_dir", out, "--datasets", "D", "--scenes", "A", "--n_views", "3",
            "--iterations", "20", "--workers", "2"] + K
    with contextlib.redirect_stdout(open(os.devnull, "w")):
        assert P.main(argv) == 0
    files = _compare_trees(out, str(tmp_path / "cli"))
    pre = os.path.join("D", "A", "3_views")
    assert S.ply_properties(_ply(os.path.join(out, pre), 20))[-1] == "filter_3D"
    if mode == "eval":
        assert os.path.join(pre, "test", "ours_20", "renders", "t0.png") in files
    else:
        assert len([f for f in files if f.startswith(os.path.join(pre, "interp"))]) == 2 * int(300 / 3) + 1
