"""render.py's train / test stages and metrics.py on the GPU (-m gpu, DESIGN.md section 4.13): the test stage's best
poses against PoseTracker.optimize_batch at every --max_batch, its PNGs against the 8-bit renders and the source
images, the train stage against frames_u8, the metrics CLI against evaluate_batch, and the tracked poses against the
CPU restatement of render.py:113-161 (tests/test_tracking.py)."""
import json
import math
import os

import numpy as np
import pytest
import torch

import instantsplat_b200 as I
from instantsplat_b200 import freeview as F
from instantsplat_b200 import metrics as M
from instantsplat_b200 import render_views as R
from instantsplat_b200 import scene_io as S
from instantsplat_b200.frame import mip_filter3d
from instantsplat_b200.scenes import surface_scene
from instantsplat_b200.tracking import PoseTracker

pytestmark = pytest.mark.gpu
DEV = "cuda"
N_TRAIN, N_TEST, ITERS = 3, 4, 20


def _u8(img: torch.Tensor) -> np.ndarray:
    return F.quantise(img.to(DEV).contiguous()).cpu().numpy()


def _truth_tracker(sc, bg):
    p = sc.params
    return PoseTracker(p["xyz"], p["rotation"], p["scaling"], p["opacity"], p["f_dc"], p["f_rest"], sc.width, sc.height,
                       sc.fovx, sc.fovy, bg=bg, sh_degree=sc.sh_degree, device=DEV)


def _source_and_model(root, deg=3, white=False):
    """A source in render.py's layout (sparse_3/0 training views, sparse_3/1 test views at perturbed poses, images/,
    sparse/0/images.bin with 24 ground-truth poses) and a briefly trained model."""
    sc = surface_scene(6000, N_TRAIN, 96, 64, seed=31, sh_degree=deg)
    bg = torch.ones(3) if white else torch.zeros(3)
    sc.bg = bg
    src, model = os.path.join(root, "src"), os.path.join(root, "model")
    truth = _truth_tracker(sc, bg)
    train_u8 = _u8(truth.render_batch(sc.poses))
    S.write_synthetic_source(src, sc, train_u8)
    g = torch.Generator().manual_seed(4)
    true_test = sc.poses[torch.arange(N_TEST) % N_TRAIN] + 0.02 * torch.randn(N_TEST, 7, generator=g)
    test_u8 = _u8(truth.render_batch(true_test))
    init = true_test + torch.tensor([0.0, 0.004, -0.003, 0.002, 0.01, -0.008, 0.012])
    fx = sc.width / (2.0 * math.tan(sc.fovx / 2.0))
    fy = sc.height / (2.0 * math.tan(sc.fovy / 2.0))
    names = [f"t{i}.png" for i in (3, 1, 0, 2)]                     # not in image_name order
    S.write_colmap_text(os.path.join(src, f"sparse_{N_TRAIN}", "1"), sc.width, sc.height, fx, fy, init.numpy(), names)
    from PIL import Image
    for i, n in enumerate(names):
        Image.fromarray(test_u8[i]).save(os.path.join(src, "images", n))
    gt = np.concatenate([np.tile([1.0, 0, 0, 0], (24, 1)), np.random.default_rng(5).standard_normal((24, 3))], axis=1)
    gt[S.split_train_test(list(range(24)), N_TRAIN)[0]] = sc.poses.numpy()
    S.write_colmap_images_bin(os.path.join(src, "sparse", "0", "images.bin"), gt, [f"{i:03d}.png" for i in range(24)])
    tr = I.JointTrainer(sc, DEV, gt_images=torch.from_numpy(train_u8).permute(0, 3, 1, 2) / 255.0)
    for k in range(6):
        tr.step(k % N_TRAIN)
    tr.save_ply(os.path.join(model, "point_cloud", "iteration_6", "point_cloud.ply"))
    tr.save_poses(os.path.join(model, "pose", "ours_6", "pose_optimized.npy"))
    return src, model, 6


def _read(folder, names):
    from PIL import Image
    return np.stack([np.asarray(Image.open(os.path.join(folder, n))) for n in names])


@pytest.mark.parametrize("deg,mip,white", [(1, False, False), (3, False, False), (3, True, False), (3, False, True)])
def test_test_stage(tmp_path, deg, mip, white):
    src, model, it = _source_and_model(str(tmp_path), deg, white)
    views = S.load_views(src, N_TRAIN, 1, resolution=1)
    assert views.names == ["t0", "t1", "t2", "t3"]
    tk = R.tracker_for(model, it, views, white)
    assert tk.sh_degree == 3                       # the saved ply carries degree-3 coefficients, as render.py loads it
    kw = {}
    if mip:
        kw = dict(kernel_size=0.1, filter_3D=mip_filter3d(tk.xyz, F.poses_from_w2c(views.w2c).to(DEV), views.width,
                                                          views.height, math.tan(views.fovx / 2),
                                                          math.tan(views.fovy / 2)))
    if mip or deg != 3:
        tk = PoseTracker(tk.xyz, tk.rotation, tk.scaling, tk.opacity, tk.f_dc, tk.f_rest, views.width, views.height,
                         views.fovx, views.fovy, bg=torch.ones(3) if white else None, sh_degree=deg, device=DEV, **kw)
    init = F.poses_from_w2c(views.w2c)
    want, _ = tk.optimize_batch(init, R.gt_images(views, DEV), num_iter=ITERS)
    assert not torch.equal(want, init)
    names = [n + ".png" for n in views.names]
    for b in (1, 3, N_TEST):
        out = str(tmp_path / f"test_{b}")
        best = R.render_test(tk, views, out, ITERS, max_batch=b, workers=2)
        assert torch.equal(best, want), b
        assert sorted(os.listdir(os.path.join(out, "renders"))) == names == sorted(os.listdir(os.path.join(out, "gt")))
        assert np.array_equal(_read(os.path.join(out, "renders"), names), _u8(tk.render_batch(want))), b
        assert np.array_equal(_read(os.path.join(out, "gt"), names), views.images)
        assert np.array_equal(views.images, _read(os.path.join(src, "images"), names))


def test_cli_stages_and_metrics(tmp_path, capsys):
    src, model, it = _source_and_model(str(tmp_path))
    base = ["-s", src, "-m", model, "--n_views", str(N_TRAIN), "--iterations", "-1", "-r", "1", "--workers", "2"]
    # train stage: the training views at pose_optimized.npy
    assert R.main(base) == 0
    views = S.load_views(src, N_TRAIN, 0)
    tk = R.tracker_for(model, it, views)
    poses = F.poses_from_w2c(np.load(os.path.join(model, "pose", f"ours_{it}", "pose_optimized.npy")))
    folder = os.path.join(model, "train", f"ours_{it}")
    idx = [f"{i:05d}.png" for i in range(N_TRAIN)]
    assert sorted(os.listdir(os.path.join(folder, "renders"))) == idx
    want = np.concatenate([c for _, c in F.frames_u8(tk, poses)])
    assert np.array_equal(_read(os.path.join(folder, "renders"), idx), want)
    assert np.array_equal(_read(os.path.join(folder, "gt"), idx), views.images)
    # test stage, then metrics.py
    assert R.main(base + ["--eval", "--optim_test_pose_iter", str(ITERS), "--max_batch", "3"]) == 0
    tviews = S.load_views(src, N_TRAIN, 1)
    ttk = R.tracker_for(model, it, tviews)
    gts = R.gt_images(tviews, DEV)
    best, _ = ttk.optimize_batch(F.poses_from_w2c(tviews.w2c), gts, num_iter=ITERS)
    assert M.main(["-s", src, "-m", model, "--n_views", str(N_TRAIN)]) == 0
    per = json.loads(open(os.path.join(model, "per_view.json")).read())[f"ours_{it}"]
    res = json.loads(open(os.path.join(model, "results.json")).read())[f"ours_{it}"]
    names = [n + ".png" for n in tviews.names]
    assert list(per["PSNR"]) == names
    m = ttk.evaluate_batch(best, gts, mode="png8")
    assert torch.equal(torch.tensor([per["PSNR"][n] for n in names], dtype=torch.float64), m["psnr"].cpu())
    assert torch.equal(torch.tensor([per["SSIM"][n] for n in names], dtype=torch.float64), m["ssim"].cpu())
    p = M.pose_errors(np.load(os.path.join(model, "pose", f"ours_{it}", "pose_optimized.npy")),
                      M.train_gt_poses(src, N_TRAIN))
    assert {k: res[k] for k in ("RPE_t", "RPE_r", "ATE")} == p
    assert "LPIPS" not in res and "LPIPS: not computed" in capsys.readouterr().out


def test_tracking_agrees_with_reference_restatement():
    """2 test views, 20 iterations: the stage's best poses against render.py:113-161 restated on the CPU oracle with
    torch's Adam and CosineAnnealingLR, to tests/test_tracking.py's tolerance."""
    from oracle import gs_oracle as O
    from test_tracking import reference_tracking
    sc = surface_scene(6000, 3, 128, 96, seed=61, sh_degree=2)
    cam = O.Camera.instantsplat(sc.width, sc.height, sc.fovx, sc.fovy, sh_degree=2)
    gts, w2c = [], []
    for v in (0, 2):
        with torch.no_grad():
            img, _ = O.render_instantsplat(sc.params["xyz"], sc.params["rotation"], sc.params["scaling"],
                                           sc.params["opacity"], sc.params["f_dc"], sc.params["f_rest"], sc.poses[v], cam)
        gts.append(img.mul(255).add_(0.5).clamp_(0, 255).permute(1, 2, 0).to(torch.uint8).numpy())
        init = sc.poses[v] + torch.tensor([0.0, 0.004, -0.003, 0.002, 0.01, -0.008, 0.012])
        w2c.append(S.pose7_to_matrix(init.numpy()))
    views = S.Views(["a", "b"], np.stack(w2c), np.stack(gts), sc.width, sc.height, sc.fovx, sc.fovy)
    p = sc.params
    tk = PoseTracker(p["xyz"], p["rotation"], p["scaling"], p["opacity"], p["f_dc"], p["f_rest"], sc.width, sc.height,
                     sc.fovx, sc.fovy, sh_degree=2, device=DEV)
    best = R.track(tk, views, num_iter=20, max_batch=2)
    init = F.poses_from_w2c(views.w2c)
    gt_f = R.gt_images(views, "cpu")
    for i, v in enumerate((0, 2)):
        ref_pose, _, ref_losses, _ = reference_tracking(sc, v, gt_f[i], init[i], 20, 2)
        assert ref_losses[-1] < ref_losses[0]
        assert float((best[i] - ref_pose).abs().max()) < 2e-4, (i, best[i], ref_pose)
