"""The training stage's host side (instantsplat_b200/train.py, DESIGN.md section 4.14) against tests/golden/train.npz,
which oracle/make_golden_train.py writes from the reference's own parser, prepare_output_and_logger, Scene,
load_and_prepare_confidence, compute_scale_gaussian_by_project_pair_pcd and save_pose (and train.py's selection
lines): the view schedule, the camera order and pose table, the extent, the per-point learning rates, the init-scale
cap, the files written beside the model, the flag set and the refusals."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from instantsplat_b200 import scene_io as S
from instantsplat_b200 import train as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def z(golden_dir):
    return np.load(os.path.join(golden_dir, "train.npz"))


@pytest.fixture
def source(z, tmp_path):
    """The generator's source, file for file."""
    root = tmp_path / "src"
    for i, rel in enumerate(z["src_files"]):
        p = root / str(rel)
        p.parent.mkdir(parents=True, exist_ok=True)
        p.write_bytes(z[f"src_blob_{i}"].tobytes())
    return str(root)


def test_view_schedule_matches_train_py(z):
    for n, it, first in z["schedules"].tolist():
        order, rows = T.view_schedule(n, it, first)
        assert order == z[f"order_{n}"].tolist() == T.scene_order(n), (n, it, first)
        assert rows == z[f"sched_{n}_{it}_{first}"].tolist(), (n, it, first)
        assert len(rows) == max(0, it - first)


def test_view_schedule_resume_restarts_from_seed_0():
    """A resumed run's schedule is that of a fresh seed, not the rest of the uninterrupted one (train.py re-seeds)."""
    _, full = T.view_schedule(12, 200)
    _, resumed = T.view_schedule(12, 200, 100)
    assert resumed == full[:100] and resumed != full[100:]
    state = __import__("random").getstate()
    T.view_schedule(5, 50)
    assert __import__("random").getstate() == state        # the global RNG is not touched


def test_host_scene_matches_reference(z, source):
    n = 4
    h = T.load_host_scene(source, n, 1)
    names = [h.views.names[i] for i in h.order]
    assert names == z["uid_names"].tolist()
    assert h.colmap_ids == z["uid_colmap_ids"].tolist()
    assert h.views.names == sorted(h.views.names)
    assert torch.equal(h.poses, torch.from_numpy(z["P"]))
    assert h.extent == float(z["cameras_extent"])
    assert torch.equal(h.per_point_lr, torch.from_numpy(z["confidence"]))
    assert h.scale_gaussian is None
    assert np.array_equal(h.points, z["init_xyz"]) and h.points.dtype == np.float32
    # create_from_pcd's colour and constant tensors (the knn scales are checked on the GPU)
    sh = (torch.from_numpy(h.colors).float() - 0.5) / 0.28209479177387814
    assert torch.equal(sh, torch.from_numpy(z["init_features_dc"][:, 0]))
    hs = T.load_host_scene(source, n, 1, init_scale_from_view_depth=True)
    assert np.array_equal(hs.scale_gaussian, z["scale_gaussian"]) and hs.scale_gaussian.dtype == np.float64


def test_files_beside_the_model_are_byte_equal(z, source, tmp_path):
    argv = [str(a) for a in z["argv"]]
    args = T.parse_args(argv)
    ref = json.loads(str(z["ref_args_json"]))
    assert vars(args) == ref                                  # every flag and default as train.py parses them
    assert T.cfg_args_text(args).encode() == z["cfg_args"].tobytes()
    # the golden's paths are the generator's; write the source's files to a fresh model folder
    args.source_path, args.model_path = source, str(tmp_path / "model")
    h = T.load_host_scene(source, args.n_views, args.resolution)
    T.write_model_files(args, h)
    m = tmp_path / "model"
    assert (m / "cameras.json").read_bytes() == z["cameras_json"].tobytes()
    assert (m / "input.ply").read_bytes() == z["input_ply"].tobytes()
    assert (m / "cfg_args").read_text() == T.cfg_args_text(args)
    # save_pose's layout and COLMAP-id order; scene_io converts the quaternions in fp64, get_camera_from_tensor in fp32
    mats = S.save_pose_npy(str(m / "pose_org.npy"), h.poses.numpy(), h.colmap_ids)
    assert mats.dtype == z["pose_org"].dtype and mats.shape == z["pose_org"].shape
    np.testing.assert_allclose(mats, z["pose_org"], rtol=0, atol=6e-8)


def test_train_time_lines(tmp_path):
    T.save_time(str(tmp_path), "[2] train_joint_TrainTime", 125.9)
    T.save_time(str(tmp_path), "[2] train_joint", 7.2)
    assert (tmp_path / "train_time.txt").read_text() == "[2] train_joint_TrainTime: 2 min 5 sec\n[2] train_joint: 0 min 7 sec\n"


def test_every_train_py_flag_parses():
    argv = ["-s", "S", "-m", "M", "-i", "imgs", "-r", "1", "--sh_degree", "3", "-w", "--data_device", "cpu",
            "--n_views", "3", "--init_scale_from_view_depth", "--iterations", "20", "--position_lr_init", "1e-4",
            "--position_lr_final", "1e-6", "--position_lr_delay_mult", "0.02", "--position_lr_max_steps", "100",
            "--feature_lr", "0.003", "--opacity_lr", "0.04", "--scaling_lr", "0.004", "--rotation_lr", "0.002",
            "--percent_dense", "0.02", "--lambda_dssim", "0.3", "--densification_interval", "50",
            "--opacity_reset_interval", "100", "--densify_from_iter", "5", "--densify_until_iter", "10",
            "--densify_grad_threshold", "0.001", "--pp_optimizer", "--optim_pose", "--convert_SHs_python",
            "--compute_cov3D_python", "--debug", "--ip", "0.0.0.0", "--port", "1", "--debug_from", "3",
            "--detect_anomaly", "--test_iterations", "10", "20", "--save_iterations", "5", "--quiet",
            "--disable_viewer", "--checkpoint_iterations", "7", "--start_checkpoint", "c.pth"]
    a = T.parse_args(argv)
    assert a.images == "imgs" and a.white_background and a.data_device == "cpu" and a.save_iterations == [5, 20]
    assert a.test_iterations == [10, 20] and a.checkpoint_iterations == [7] and a.start_checkpoint == "c.pth"
    c = T.optim_config(a, 2.5)
    assert (c.iterations, c.position_lr_init, c.lambda_dssim, c.pp_optimizer, c.optim_pose) == (20, 1e-4, 0.3, True, True)
    assert c.spatial_lr_scale == 2.5 and c.max_sh_degree == 3 and c.densify is False
    d = T.optim_config(T.parse_args(["-s", "S", "-m", "M"]), 1.0)
    assert d.pp_optimizer is False and d.optim_pose is False and d.iterations == 30_000    # train.py's defaults


@pytest.mark.parametrize("extra,reason", [
    (["--eval"], "--eval: train.py would load sparse_<n>/1"),
    (["--random_background"], "--random_background: a fresh random background"),
    (["--sh_degree", "2"], "--sh_degree 2: the trainer's flat buffers hold degree-3 SH"),
    (["-r", "2"], "resampled images are not supported"),
    (["--start_checkpoint", "missing.pth"], "--start_checkpoint: missing.pth not found"),
])
def test_refusals_write_nothing(source, tmp_path, extra, reason):
    model = tmp_path / "model"
    with pytest.raises(SystemExit, match=reason.replace("<", ".").replace(">", ".").replace("(", ".")):
        T.main(["-s", source, "-m", str(model), "--n_views", "4", "--iterations", "3"] + extra)
    assert not model.exists()


def test_refuses_camera_ids_other_than_1_to_n(source, tmp_path):
    folder = os.path.join(source, "sparse_4", "0")
    txt = open(os.path.join(folder, "cameras.txt")).read().replace("\n4 PINHOLE", "\n5 PINHOLE")
    open(os.path.join(folder, "cameras.txt"), "w").write(txt)
    imgs = open(os.path.join(folder, "images.txt")).read().split("\n")
    imgs = [" ".join(l.split()[:8] + ["5"] + l.split()[9:]) if l.startswith("4 ") else l for l in imgs]
    open(os.path.join(folder, "images.txt"), "w").write("\n".join(imgs))
    model = tmp_path / "model"
    with pytest.raises(SystemExit, match=r"camera ids \[.*5.*\]; train.py's save_pose needs every camera id 1..4"):
        T.main(["-s", source, "-m", str(model), "--n_views", "4", "-r", "1"])
    assert not model.exists()


def test_refuses_missing_confidence(source, tmp_path):
    os.remove(os.path.join(source, "sparse_4", "0", "confidence_dsp.npy"))
    model = tmp_path / "model"
    with pytest.raises(SystemExit, match="confidence_dsp.npy not found"):
        T.main(["-s", source, "-m", str(model), "--n_views", "4", "-r", "1"])
    assert not model.exists()


def test_images_folder_flag(source, tmp_path):
    os.rename(os.path.join(source, "images"), os.path.join(source, "imgs"))
    with pytest.raises(FileNotFoundError):
        T.load_host_scene(source, 4, 1)
    v = T.load_host_scene(source, 4, 1, images="imgs").views
    assert v.names == ["a", "b", "c", "d"] and v.camera_ids == [2, 4, 1, 3]


def test_help_via_module():
    r = subprocess.run([sys.executable, "-m", "instantsplat_b200.train", "--help"], cwd=ROOT, capture_output=True,
                       text=True, timeout=120)
    assert r.returncode == 0, r.stderr
    for flag in ("--source_path", "--n_views", "--pp_optimizer", "--start_checkpoint", "--checkpoint_iterations"):
        assert flag in r.stdout
