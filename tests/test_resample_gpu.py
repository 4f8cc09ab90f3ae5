"""Pillow's bicubic resize on the GPU (-m gpu, DESIGN.md section 4.21): gsb_resample_u8_batch against Pillow byte for
byte, batched and alone, load_views with a CUDA resample_device, and --resample_images through train, render_views
(train stage and --eval) and freeview on a source wider than 1600 pixels."""
import json
import math
import os

import numpy as np
import pytest
import torch
from PIL import Image

import _resample as RS
import instantsplat_b200 as I
from instantsplat_b200 import freeview as F
from instantsplat_b200 import render_views as R
from instantsplat_b200 import resample
from instantsplat_b200 import scene_io as S
from instantsplat_b200 import train as T
from instantsplat_b200.scenes import surface_scene
from instantsplat_b200.tracking import PoseTracker

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _pillow(batch: np.ndarray, size) -> np.ndarray:
    return np.stack([np.asarray(Image.fromarray(a).resize(size)) for a in batch])


@pytest.mark.parametrize("src,dst", RS.GRID + [RS.BIG])
def test_kernel_equals_pillow(src, dst):
    V = 2 if (src, dst) == RS.BIG else 3
    batch = np.stack([RS.image(*src, seed=100 * v + src[0]) for v in range(V)])
    got = resample.resize_u8(torch.from_numpy(batch).to(DEV), dst)
    assert got.shape == (V, dst[1], dst[0], 3) and got.dtype == torch.uint8 and got.is_cuda
    assert np.array_equal(got.cpu().numpy(), _pillow(batch, dst))


def test_each_view_equals_resizing_it_alone():
    batch = torch.from_numpy(np.stack([RS.image(1920, 1080, seed=s) for s in range(5)])).to(DEV)
    together = resample.resize_u8(batch, (1600, 900))
    for v in range(5):
        assert torch.equal(together[v:v + 1], resample.resize_u8(batch[v:v + 1].contiguous(), (1600, 900)))
    assert torch.equal(resample.resize_u8(batch[:2].contiguous(), (1920, 1080)), batch[:2])         # same size: a copy


def test_bad_arguments_are_refused():
    x = torch.zeros(1, 8, 8, 3, dtype=torch.uint8, device=DEV)
    out = torch.empty(1, 4, 4, 3, dtype=torch.uint8, device=DEV)
    b, c = (torch.from_numpy(t.copy()).to(DEV) for t in resample.coefficients(8, 4))
    L = I.lib()
    s = I._lib.stream_ptr()
    args = lambda V, yb, scratch: (V, 8, 8, 4, 4, x.data_ptr(), out.data_ptr(), b.data_ptr(), c.data_ptr(),
                                   c.shape[1], yb, c.data_ptr(), c.shape[1], scratch, 10 ** 6, s)
    assert L.gsb_resample_u8_batch(*args(0, b.data_ptr(), out.data_ptr())) == -1          # no view
    assert L.gsb_resample_u8_batch(*args(1, None, out.data_ptr())) == -1                  # a missing table
    assert L.gsb_resample_u8_batch(*args(1, b.data_ptr(), None)) == -1                    # no scratch for two passes
    with pytest.raises(ValueError, match="at least 1 x 1"):
        resample.resize_u8(x, (0, 3))
    torch.cuda.synchronize()


# ---- the loader and the stage command lines --------------------------------------------------------------------
W, H, N_TRAIN, N_TEST = 1700, 64, 3, 2


def _source(root):
    """An init_geo-shaped source 1700 pixels wide (sparse_3/0 and sparse_3/1), its images renders of a scene."""
    sc = surface_scene(3000, N_TRAIN, W, H, seed=43, sh_degree=3)
    p = sc.params
    truth = PoseTracker(p["xyz"], p["rotation"], p["scaling"], p["opacity"], p["f_dc"], p["f_rest"], W, H, sc.fovx,
                        sc.fovy, sh_degree=3, device=DEV)
    S.write_synthetic_source(root, sc, F.quantise(truth.render_batch(sc.poses).contiguous()).cpu().numpy())
    g = torch.Generator().manual_seed(6)
    test = sc.poses[torch.arange(N_TEST)] + 0.01 * torch.randn(N_TEST, 7, generator=g)
    fx = W / (2.0 * math.tan(sc.fovx / 2.0))
    fy = H / (2.0 * math.tan(sc.fovy / 2.0))
    names = ["t1.png", "t0.png"]
    S.write_colmap_text(os.path.join(root, f"sparse_{N_TRAIN}", "1"), W, H, fx, fy, test.numpy(), names)
    test_u8 = F.quantise(truth.render_batch(test).contiguous()).cpu().numpy()
    for i, n in enumerate(names):
        Image.fromarray(test_u8[i]).save(os.path.join(root, "images", n))
    return root


@pytest.fixture(scope="module")
def source(tmp_path_factory):
    return _source(str(tmp_path_factory.mktemp("wide") / "src"))


def _decoded(src, split):
    v = S.load_views(src, N_TRAIN, split, 1)
    return v.images


def _host_pillow(images, size):
    """resample.resize_u8 with Pillow on the host in its place."""
    return torch.from_numpy(_pillow(images.cpu().numpy(), size)).to(images.device)


@pytest.mark.parametrize("r", [-1, 2, 4, 8, 1000])
def test_load_views_equals_pillow(source, r):
    for split in (0, 1):
        v = S.load_views(source, N_TRAIN, split, r, resample_device=DEV)
        size = S.loaded_size(W, H, r)
        assert (v.width, v.height) == size and (v.source_width, v.source_height) == (W, H)
        assert np.array_equal(v.images, _pillow(_decoded(source, split), size))
        full = S.load_views(source, N_TRAIN, split, 1)
        assert (v.fovx, v.fovy) == (full.fovx, full.fovy) and v.names == full.names


def _train(source, model, r, *extra):
    args = T.parse_args(["-s", source, "-m", model, "-r", str(r), "--n_views", str(N_TRAIN), "--iterations", "4",
                         "--quiet"] + list(extra))
    return T.run(args)


def _read(path):
    with open(path, "rb") as f:
        return f.read()


@pytest.fixture(scope="module")
def models(source, tmp_path_factory):
    """Runs of train: -r 1, and -r 2 / -r -1 with --resample_images, each also with Pillow on the host resizing."""
    root = tmp_path_factory.mktemp("models")
    out = {"r1": str(root / "r1")}
    _train(source, out["r1"], 1)
    for r in (2, -1):
        out[r] = str(root / f"gpu{r}")
        res = _train(source, out[r], r, "--resample_images")
        assert (res.trainer.W, res.trainer.H) == S.loaded_size(W, H, r)
        out[f"host{r}"] = str(root / f"host{r}")
        mp = pytest.MonkeyPatch()
        mp.setattr(resample, "resize_u8", _host_pillow)
        try:
            _train(source, out[f"host{r}"], r, "--resample_images")
        finally:
            mp.undo()
    return out


@pytest.mark.parametrize("r", [2, -1])
def test_train_at_the_loaded_size(models, r):
    a, b = models[r], models[f"host{r}"]
    for rel in (("point_cloud", "iteration_4", "point_cloud.ply"), ("pose", "ours_4", "pose_optimized.npy"),
                ("pose", "ours_4", "pose_org.npy")):
        assert _read(os.path.join(a, *rel)) == _read(os.path.join(b, *rel)), rel
    cams = _read(os.path.join(a, "cameras.json"))
    assert cams == _read(os.path.join(models["r1"], "cameras.json"))
    assert {(c["width"], c["height"]) for c in json.loads(cams)} == {(W, H)}
    assert b"resample" not in _read(os.path.join(a, "cfg_args"))


def _pngs(folder, names):
    return np.stack([np.asarray(Image.open(os.path.join(folder, n))) for n in names])


def test_render_views_at_the_loaded_size(source, models):
    model, r = models[2], 2
    size = S.loaded_size(W, H, r)
    base = ["-s", source, "-m", model, "--n_views", str(N_TRAIN), "-r", str(r), "--workers", "2"]
    with pytest.raises(ValueError, match="resampled images are not supported"):
        R.main(base)
    assert R.main(base + ["--resample_images"]) == 0
    folder = os.path.join(model, "train", "ours_4")
    idx = [f"{i:05d}.png" for i in range(N_TRAIN)]
    views = S.load_views(source, N_TRAIN, 0, r, resample_device=DEV)
    tk = R.tracker_for(model, 4, views)
    poses = F.poses_from_w2c(np.load(os.path.join(model, "pose", "ours_4", "pose_optimized.npy")))
    want = np.concatenate([c for _, c in F.frames_u8(tk, poses)])
    assert want.shape[1:3] == (size[1], size[0])
    assert np.array_equal(_pngs(os.path.join(folder, "renders"), idx), want)
    assert np.array_equal(_pngs(os.path.join(folder, "gt"), idx), _pillow(_decoded(source, 0), size))
    # --eval: the test views tracked and rendered at the loaded size
    assert R.main(base + ["--resample_images", "--eval", "--optim_test_pose_iter", "5"]) == 0
    tv = S.load_views(source, N_TRAIN, 1, r, resample_device=DEV)
    names = [n + ".png" for n in tv.names]
    folder = os.path.join(model, "test", "ours_4")
    ttk = R.tracker_for(model, 4, tv)
    best, _ = ttk.optimize_batch(F.poses_from_w2c(tv.w2c), R.gt_images(tv, DEV), num_iter=5)
    want = np.concatenate([c for _, c in F.frames_u8(ttk, best)])
    assert want.shape[1:3] == (size[1], size[0])
    assert np.array_equal(_pngs(os.path.join(folder, "renders"), names), want)
    assert np.array_equal(_pngs(os.path.join(folder, "gt"), names), _pillow(_decoded(source, 1), size))


def test_freeview_at_the_loaded_size(source, models):
    model = models[-1]
    argv = ["-s", source, "-m", model, "--n_views", str(N_TRAIN), "--iterations", "4", "--max_batch", "16"]
    folder = os.path.join(model, "interp", "ours_4", "renders")
    n = int(300 / N_TRAIN) * (N_TRAIN - 1) + 1
    names = [f"{i:05d}.png" for i in range(n)]
    path = lambda: F.poses_from_w2c(np.load(os.path.join(model, "pose", "ours_4", "pose_interpolated.npy")))
    # without the flag: the full-size frames, as before
    assert F.main(argv) == 0
    tk, _, _ = F.load(source, model, N_TRAIN, 4)
    assert (tk.W, tk.H) == (W, H)
    assert np.array_equal(_pngs(folder, names), np.concatenate([c for _, c in F.frames_u8(tk, path())]))
    with pytest.raises(ValueError, match="without --resample_images"):
        F.main(argv + ["-r", "-1"])
    # with it: render.py's size for -r -1
    assert F.main(argv + ["-r", "-1", "--resample_images"]) == 0
    tk, _, _ = F.load(source, model, N_TRAIN, 4, resolution=-1, resample_images=True)
    assert (tk.W, tk.H) == S.loaded_size(W, H, -1)
    got = _pngs(folder, names)
    assert got.shape[1:3] == (tk.H, tk.W)
    assert np.array_equal(got, np.concatenate([c for _, c in F.frames_u8(tk, path())]))
