"""render.py's train / test stages and metrics.py, host side (no GPU): the split, the images.bin reader and the pose
errors against the reference's own functions (tests/golden/pose_eval.npz, made by oracle/make_golden_pose_eval.py),
the camera loader and its refusals, the 8-bit gt round trip, and the layout of metrics.py's output files."""
import json
import os

import numpy as np
import pytest
import torch

from instantsplat_b200 import metrics as M
from instantsplat_b200 import render_views as R
from instantsplat_b200 import scene_io as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "pose_eval.npz")


@pytest.mark.parametrize("N", [24, 30])
@pytest.mark.parametrize("n", [3, 6, 12])
def test_split_matches_reference(N, n):
    z = np.load(GOLD)
    train, test = S.split_train_test(list(range(N)), n)
    assert train == z[f"split{N}_{n}_train"].tolist() and len(train) == n
    assert test == z[f"split{N}_{n}_test"].tolist() and len(test) == 12


def test_images_bin_matches_reference(tmp_path):
    z = np.load(GOLD)
    path = tmp_path / "sparse" / "0" / "images.bin"
    path.parent.mkdir(parents=True)
    path.write_bytes(z["bin_bytes"].tobytes())
    recs = S.read_colmap_images_bin(str(path))
    ids = list(recs)
    assert ids == z["bin_ids"].tolist()
    assert np.array_equal(np.stack([recs[i]["qvec"] for i in ids]), z["bin_qvec"])
    assert np.array_equal(np.stack([recs[i]["tvec"] for i in ids]), z["bin_tvec"])
    assert [recs[i]["camera_id"] for i in ids] == z["bin_camera_ids"].tolist()
    assert [recs[i]["name"] for i in ids] == z["bin_names"].tolist()
    assert [len(recs[i]["point3D_ids"]) for i in ids] == z["bin_n_points"].tolist()
    assert np.array_equal(np.concatenate([recs[i]["xys"] for i in ids]), z["bin_xys"])
    assert np.array_equal(np.concatenate([recs[i]["point3D_ids"] for i in ids]), z["bin_point_ids"])
    got = S.read_colmap_gt_pose(str(tmp_path))
    assert got.dtype == np.float64 and np.array_equal(got, z["bin_gt_pose"])
    # the writer gives the same bytes back
    pts = [np.column_stack([recs[i]["xys"], recs[i]["point3D_ids"]]) for i in ids]
    S.write_colmap_images_bin(str(tmp_path / "again.bin"), [np.concatenate([recs[i]["qvec"], recs[i]["tvec"]]) for i in ids],
                              [recs[i]["name"] for i in ids], ids, [recs[i]["camera_id"] for i in ids], pts)
    assert (tmp_path / "again.bin").read_bytes() == z["bin_bytes"].tobytes()
    (tmp_path / "cut.bin").write_bytes(z["bin_bytes"].tobytes()[:-5])
    with pytest.raises(ValueError, match="truncated"):
        S.read_colmap_images_bin(str(tmp_path / "cut.bin"))


CASES = ["traj3", "traj6", "traj12", "scale", "reflect"]


@pytest.mark.parametrize("case", CASES)
def test_alignment_matches_reference(case):
    z = np.load(GOLD)
    gt, est = z[f"{case}_gt"], z[f"{case}_est"]
    assert gt.dtype == np.float64 and est.dtype == np.float32
    t_gt, t_est, _ = M.align_pose(gt[:, :3, -1], est[:, :3, -1])
    assert np.array_equal(t_gt, z[f"{case}_t_gt"]) and np.array_equal(t_est, z[f"{case}_t_est"])
    g, e = gt.copy(), est.copy()
    g[:, :3, -1], e[:, :3, -1] = t_gt, t_est
    aligned = M.align_sim3(e, g)
    assert aligned.dtype == np.float32 and np.array_equal(aligned, z[f"{case}_aligned"])
    want = z[f"{case}_errors"]                                  # rpe_trans, rpe_rot, ate as the reference returns them
    got = np.array([*M.compute_rpe(g, aligned), M.compute_ate(g, aligned)])
    assert np.allclose(got, want, rtol=1e-12, atol=0), (got, want)
    p = M.pose_errors(est, gt)
    assert np.allclose([p["RPE_t"], p["RPE_r"], p["ATE"]], [want[0] * 100, want[1] * 180 / np.pi, want[2]],
                       rtol=1e-12, atol=0)


def test_reflected_case_takes_umeyama_flip():
    z = np.load(GOLD)
    assert bool(z["reflect_flipped"])
    # the fit is still a rotation
    R = z["reflect_aligned"][0, :3, :3].astype(np.float64) @ z["reflect_est"][0, :3, :3].astype(np.float64).T
    assert np.linalg.det(R) > 0


def test_gt_round_trip_is_identity():
    assert R.gt_round_trip_is_identity()
    k = torch.arange(256, dtype=torch.uint8)
    assert torch.equal((k / 255.0).mul(255).add_(0.5).clamp_(0, 255).to(torch.uint8), k)


def test_pil_resize_to_same_size_is_a_copy():
    """loadCam's PILtoTorch resizes to the loaded size; at -r 1 (and -r -1 up to 1600 wide) that is the image's own
    size, and PIL returns the pixels unchanged."""
    from PIL import Image
    a = np.random.default_rng(3).integers(0, 256, (37, 53, 3), dtype=np.uint8)
    im = Image.fromarray(a)
    assert np.array_equal(np.array(im.resize(im.size)), a)
    assert not np.array_equal(np.array(im.resize((26, 18))), a[::2, ::2])        # a real resize does resample
    assert S.loaded_size(53, 37, 1) == (53, 37) and S.loaded_size(53, 37, -1) == (53, 37)
    assert S.loaded_size(1600, 900, -1) == (1600, 900) and S.loaded_size(1700, 900, -1) != (1700, 900)
    assert S.loaded_size(54, 38, 2) == (27, 19)


def _source(root, names_train, names_test, W=24, H=16, n_views=None, mode="RGB", seed=0):
    """A source directory: images/<name>, sparse_<n>/0 (train) and sparse_<n>/1 (test), PINHOLE 20 x 21."""
    from PIL import Image
    g = np.random.default_rng(seed)
    n = len(names_train) if n_views is None else n_views
    os.makedirs(os.path.join(root, "images"), exist_ok=True)
    imgs = {}
    for name in names_train + names_test:
        a = g.integers(0, 256, (H, W, 4 if mode == "RGBA" else 3), dtype=np.uint8)
        Image.fromarray(a, mode).save(os.path.join(root, "images", name))
        imgs[name] = a
    for k, names in enumerate((names_train, names_test)):
        poses = np.concatenate([g.standard_normal((len(names), 4)), g.standard_normal((len(names), 3))], axis=1)
        S.write_colmap_text(os.path.join(root, f"sparse_{n}", str(k)), W, H, 20.0, 21.0, poses, names)
    return imgs


def test_load_views(tmp_path):
    imgs = _source(str(tmp_path), ["b.png", "a.png", "c.png"], ["z.png", "y.png"])
    v = S.load_views(str(tmp_path), 3, 0, resolution=1)
    assert v.names == ["a", "b", "c"] and len(v) == 3 and (v.width, v.height) == (24, 16)
    assert np.array_equal(v.images, np.stack([imgs[n] for n in ("a.png", "b.png", "c.png")]))
    assert abs(v.fovx - 2 * np.arctan(24 / 40.0)) < 1e-15 and abs(v.fovy - 2 * np.arctan(16 / 42.0)) < 1e-15
    _, ims = S.read_colmap_text(str(tmp_path / "sparse_3" / "0"))
    rec = [r for r in ims.values() if r["name"] == "a.png"][0]
    assert np.array_equal(v.w2c[0, :3, :3], S.qvec2rotmat(rec["qvec"])) and np.array_equal(v.w2c[0, :3, 3], rec["tvec"])
    t = S.load_views(str(tmp_path), 3, 1, resolution=-1)
    assert t.names == ["y", "z"]
    gts = R.gt_images(t, "cpu")
    assert gts.shape == (2, 3, 16, 24) and gts.dtype == torch.float32 and gts.is_contiguous()
    assert torch.equal(gts, torch.from_numpy(t.images).permute(0, 3, 1, 2) / 255.0)
    # SIMPLE_PINHOLE: one focal length for both axes
    cams = tmp_path / "sparse_3" / "0" / "cameras.txt"
    cams.write_text(cams.read_text().replace("PINHOLE 24 16 20 21", "SIMPLE_PINHOLE 24 16 20"))
    v = S.load_views(str(tmp_path), 3, 0)
    assert abs(v.fovy - 2 * np.arctan(16 / 40.0)) < 1e-15


def test_loader_refusals(tmp_path):
    _source(str(tmp_path), ["a.png", "b.png"], ["c.png"])
    with pytest.raises(ValueError, match="resampled"):
        S.load_views(str(tmp_path), 2, 0, resolution=2)
    with pytest.raises(ValueError, match="resampled"):
        S.load_views(str(tmp_path), 2, 0, resolution=12)
    cams = tmp_path / "sparse_2" / "0" / "cameras.txt"
    txt = cams.read_text()
    cams.write_text(txt.replace("2 PINHOLE 24 16 20 21", "2 PINHOLE 24 16 20 22"))
    with pytest.raises(ValueError, match="intrinsics differ"):
        S.load_views(str(tmp_path), 2, 0)
    cams.write_text(txt.replace("2 PINHOLE", "2 OPENCV"))
    with pytest.raises(ValueError, match="PINHOLE"):
        S.load_views(str(tmp_path), 2, 0)
    with pytest.raises(FileNotFoundError, match="sparse_5"):
        S.load_views(str(tmp_path), 5, 0)
    rgba = tmp_path / "rgba"
    _source(str(rgba), ["a.png", "b.png"], ["c.png"], mode="RGBA")
    with pytest.raises(ValueError, match="alpha"):
        S.load_views(str(rgba), 2, 0)
    wide = tmp_path / "wide"
    _source(str(wide), ["a.png"], ["c.png"], W=1601, H=4)
    with pytest.raises(ValueError, match="resampled"):
        S.load_views(str(wide), 1, 0, resolution=-1)
    assert S.load_views(str(wide), 1, 0, resolution=1).width == 1601


def test_render_views_refusals(tmp_path):
    src, model = tmp_path / "src", tmp_path / "model"
    _source(str(src), ["a.png", "b.png"], ["c.png"])
    (model / "point_cloud" / "iteration_7").mkdir(parents=True)
    with pytest.raises(FileNotFoundError, match="pose_optimized.npy"):
        R.main(["-s", str(src), "-m", str(model), "--n_views", "2", "--iterations", "-1"])
    with pytest.raises(FileNotFoundError, match="point_cloud.ply"):
        R.main(["-s", str(src), "-m", str(model), "--n_views", "2", "--eval"])
    with pytest.raises(SystemExit):
        R.main(["-s", str(src), "-m", str(model), "--n_views", "2", "--max_batch", "0"])
    v = S.load_views(str(src), 2, 0)
    with pytest.raises(ValueError, match="one to one"):
        R.render_train(None, v, np.stack([np.eye(4)] * 3), str(tmp_path / "out"))


def test_cli_entry_points():
    import importlib
    for mod in ("instantsplat_b200.render_views", "instantsplat_b200.metrics"):
        m = importlib.import_module(mod)
        assert callable(m.main)
        with pytest.raises(SystemExit) as e:
            m.main(["--help"])
        assert e.value.code == 0


def _fake_numbers(renders, gts, device="cuda"):
    """A stand-in for the GPU metrics: PSNR = 10 + the view's first render byte, SSIM = its first gt byte / 255."""
    return {"PSNR": torch.tensor([10.0 + float(r[0, 0, 0]) for r in renders], dtype=torch.float64),
            "SSIM": torch.tensor([float(g[0, 0, 0]) / 255 for g in gts], dtype=torch.float64)}


def _method_tree(scene, method, names, seed=0):
    from PIL import Image
    g = np.random.default_rng(seed)
    for sub in ("renders", "gt"):
        os.makedirs(os.path.join(scene, "test", method, sub), exist_ok=True)
        for n in names:
            Image.fromarray(g.integers(0, 256, (8, 12, 3), dtype=np.uint8)).save(os.path.join(scene, "test", method, sub, n))


def test_metrics_layout(tmp_path, monkeypatch, capsys):
    monkeypatch.setattr(M, "image_numbers", _fake_numbers)
    z = np.load(GOLD)
    src = tmp_path / "src"
    # 24 ground-truth poses; the 6 training views' are those of traj6
    gt_all = np.stack([np.eye(4)] * 24)
    train_idx = S.split_train_test(list(range(24)), 6)[0]
    gt_all[train_idx] = z["traj6_gt"]
    qt = []
    for p in gt_all:                                            # images.bin holds w2c: read_colmap_gt_pose transposes
        from scipy.spatial.transform import Rotation
        x, y, zz, w = Rotation.from_matrix(p[:3, :3].T).as_quat()
        qt.append([w, x, y, zz, *p[:3, 3]])
    S.write_colmap_images_bin(str(src / "sparse" / "0" / "images.bin"), np.array(qt), [f"{i:03d}.png" for i in range(24)])
    scene = tmp_path / "model"
    names = ["b.png", "a.png", "c.png"]
    _method_tree(str(scene), "ours_7", names)
    (scene / "pose" / "ours_7").mkdir(parents=True)
    np.save(scene / "pose" / "ours_7" / "pose_optimized.npy", z["traj6_est"])
    assert M.main(["-s", str(src), "-m", str(scene), "--n_views", "6"]) == 0
    out = capsys.readouterr().out
    assert "LPIPS: not computed" in out
    res = json.loads((scene / "results.json").read_text())
    per = json.loads((scene / "per_view.json").read_text())
    assert list(res) == ["ours_7"] and list(per) == ["ours_7"]
    assert set(res["ours_7"]) == {"SSIM", "PSNR", "RPE_t", "RPE_r", "ATE"}
    assert set(per["ours_7"]) == {"SSIM", "PSNR"} and list(per["ours_7"]["PSNR"]) == ["a.png", "b.png", "c.png"]
    from PIL import Image
    rd = lambda sub, n: np.asarray(Image.open(scene / "test" / "ours_7" / sub / n))
    for n in names:
        assert per["ours_7"]["PSNR"][n] == 10.0 + float(rd("renders", n)[0, 0, 0])
        assert per["ours_7"]["SSIM"][n] == float(rd("gt", n)[0, 0, 0]) / 255
    assert res["ours_7"]["PSNR"] == pytest.approx(np.mean(list(per["ours_7"]["PSNR"].values())), rel=1e-15)
    lines = (scene / "test" / "ours_7" / "metrics.txt").read_text().splitlines()
    p0, s0 = per["ours_7"]["PSNR"]["a.png"], per["ours_7"]["SSIM"]["a.png"]
    assert lines[0] == f"image namea.png, image idx: 0, PSNR: {p0:.2f}, SSIM: {s0:.4f}" and len(lines) == 3
    # the pose numbers are the reference's on traj6 (the rotations went through a quaternion on the way into
    # images.bin, so they agree to rounding, the positions exactly)
    want = z["traj6_errors"]
    got = res["ours_7"]
    assert np.allclose([got["RPE_t"], got["RPE_r"]], [want[0] * 100, want[1] * 180 / np.pi], rtol=1e-6, atol=0)
    assert got["ATE"] == float(want[2])
    txt = (scene / "pose" / "ours_7" / "pose_eval.txt").read_text()
    assert txt == "RPE_t: {:.04f}, RPE_r: {:.04f}, ATE: {:.04f}".format(got["RPE_t"], got["RPE_r"], got["ATE"])


def test_metrics_missing_pieces(tmp_path, monkeypatch, capsys):
    monkeypatch.setattr(M, "image_numbers", _fake_numbers)
    src = tmp_path / "src"
    src.mkdir()
    ok, no_test, bad = tmp_path / "ok", tmp_path / "no_test", tmp_path / "bad"
    _method_tree(str(ok), "ours_3", ["a.png", "b.png"])
    no_test.mkdir()
    _method_tree(str(bad), "ours_3", ["a.png"])
    os.remove(bad / "test" / "ours_3" / "gt" / "a.png")
    assert M.main(["-s", str(src), "-m", str(no_test), str(ok), str(bad), "--n_views", "3"]) == 1
    out = capsys.readouterr().out
    assert "poses: skipped" in out and "images.bin" in out                          # no sparse/0: images only
    res = json.loads((ok / "results.json").read_text())
    assert set(res["ours_3"]) == {"SSIM", "PSNR"}
    assert not (no_test / "results.json").exists() and not (bad / "results.json").exists()
    assert out.count("Unable to compute metrics") == 2
