"""Pillow's bicubic resize on the host side (instantsplat_b200/resample.py, DESIGN.md section 4.21): the integer
tables against Pillow through a numpy restatement of its two passes, the tables' sums in index order, the loader's
refusals and the --resample_images flags of the stage command lines."""
import os

import numpy as np
import pytest
import torch
from PIL import Image

import _resample as RS
from instantsplat_b200 import freeview as F
from instantsplat_b200 import render_views as R
from instantsplat_b200 import resample
from instantsplat_b200 import scene_io as S
from instantsplat_b200 import train as T


@pytest.mark.parametrize("src,dst", RS.GRID + [RS.BIG])
def test_restated_passes_equal_pillow(src, dst):
    a = RS.image(*src, seed=src[0] * 7 + src[1])
    assert np.array_equal(RS.resize(a, dst), np.asarray(Image.fromarray(a).resize(dst)))


def test_grid_covers_the_loaded_sizes():
    """The grid's sizes are loadCam's at -r 2 / 4 / 8 (odd sizes), -r -1 (1601 and 1920 wide, 4032 x 3024) and a
    numeric -r that upscales."""
    grid = RS.GRID + [RS.BIG]
    for src, r in (((37, 23), 2), ((37, 23), 4), ((101, 75), 8), ((1601, 5), -1), ((1920, 1080), -1), ((40, 24), 60),
                   ((4032, 3024), -1)):
        assert (src, S.loaded_size(*src, r)) in grid, (src, r)


def _sequential_tables(n_in, n_out):
    scale = n_in / n_out
    fs = max(scale, 1.0)
    support = 2.0 * fs
    rows = []
    for o in range(n_out):
        c = (o + 0.5) * scale
        first = max(int(c - support + 0.5), 0)
        n = min(int(c + support + 0.5), n_in) - first
        w = [resample._bicubic((x + first - c + 0.5) * (1.0 / fs)) for x in range(n)]
        total = 0.0
        for v in w:
            total += v
        rows.append((first, [int((-0.5 if v / total < 0 else 0.5) + v / total * (1 << 22)) for v in w]))
    return rows, total


@pytest.mark.parametrize("n_in,n_out", [(4032, 1600), (3024, 1200), (37, 18), (101, 13), (9, 1), (24, 36)])
def test_tables_sum_in_index_order(n_in, n_out):
    bounds, coefs = resample.coefficients(n_in, n_out)
    rows, _ = _sequential_tables(n_in, n_out)
    assert bounds.dtype == np.int32 and coefs.dtype == np.int32 and bounds.shape == (n_out, 2)
    for o, (first, w) in enumerate(rows):
        assert (bounds[o, 0], bounds[o, 1]) == (first, len(w))
        assert coefs[o, :len(w)].tolist() == w and not coefs[o, len(w):].any()
    assert resample.coefficients(n_in, n_out)[1] is coefs                   # cached per size pair
    assert not coefs.flags.writeable


def test_pairwise_sum_would_differ():
    """numpy's pairwise np.sum rounds differently from the sequential sum on rows of the 12 MP downscale: the order
    the tables use is a choice that matters in fp64."""
    scale = 4032 / 1600
    differ = 0
    for o in range(1600):
        c = (o + 0.5) * scale
        first = max(int(c - 2 * scale + 0.5), 0)
        n = min(int(c + 2 * scale + 0.5), 4032) - first
        w = [resample._bicubic((x + first - c + 0.5) * (1.0 / scale)) for x in range(n)]
        total = 0.0
        for v in w:
            total += v
        differ += float(np.sum(np.array(w))) != total
    assert differ > 0


def test_bad_sizes_and_host_tensors_are_refused():
    with pytest.raises(ValueError, match="sizes"):
        resample.coefficients(0, 3)
    with pytest.raises(ValueError, match="CUDA"):
        resample.resize_u8(torch.zeros(1, 4, 4, 3, dtype=torch.uint8), (2, 2))
    with pytest.raises(ValueError, match="CUDA"):
        resample.resize_u8(np.zeros((1, 4, 4, 3), np.uint8), (2, 2))


def _source(root, W=24, H=16, n=2):
    rng = np.random.default_rng(3)
    names = [f"{c}.png" for c in "ab"[:n]]
    poses = np.concatenate([np.tile([1.0, 0, 0, 0], (n, 1)), rng.standard_normal((n, 3))], axis=1)
    S.write_colmap_text(os.path.join(root, f"sparse_{n}", "0"), W, H, 20.0, 21.0, poses, names)
    os.makedirs(os.path.join(root, "images"), exist_ok=True)
    for name in names:
        Image.fromarray(rng.integers(0, 256, (H, W, 3), dtype=np.uint8)).save(os.path.join(root, "images", name))
    return root


def test_loader_refuses_a_host_resample_device(tmp_path):
    src = _source(str(tmp_path))
    for dev in ("cpu", torch.device("cpu"), "meta"):
        with pytest.raises(ValueError, match="CUDA device only"):
            S.load_views(src, 2, 0, resolution=2, resample_device=dev)
    with pytest.raises(ValueError, match="resampled images are not supported"):
        S.load_views(src, 2, 0, resolution=2)
    v = S.load_views(src, 2, 0, resolution=1)
    assert (v.source_width, v.source_height) == (v.width, v.height) == (24, 16)


def test_train_flag_parses_and_leaves_the_rest_unchanged():
    base = ["-s", "S", "-m", "M", "--n_views", "3", "-r", "2"]
    a, b = T.parse_args(base), T.parse_args(base + ["--resample_images"])
    assert not resample.requested(a) and resample.requested(b)
    assert "resample_images" not in vars(a)                                 # train.py's own namespace
    assert T.cfg_args_text(a) == T.cfg_args_text(b) and "resample" not in T.cfg_args_text(b)
    assert T.refusals(a) == T.refusals(b) == []
    bad = ["--eval", "--random_background", "--sh_degree", "2"]
    assert T.refusals(T.parse_args(base + bad)) == T.refusals(T.parse_args(base + bad + ["--resample_images"]))


def test_train_refusal_without_flag_writes_nothing(tmp_path):
    src = _source(str(tmp_path / "src"))
    model = tmp_path / "model"
    with pytest.raises(SystemExit, match=r"resampled images are not supported .* or --resample_images"):
        T.main(["-s", src, "-m", str(model), "--n_views", "2", "-r", "2"])
    assert not model.exists()


def test_render_views_flag_and_infer_video_forwarding(monkeypatch):
    a = R.parser().parse_args(["-s", "S", "-m", "M", "--n_views", "3"])
    assert not resample.requested(a)
    assert resample.requested(R.parser().parse_args(["-s", "S", "-m", "M", "--n_views", "3", "--resample_images"]))
    argvs = []
    monkeypatch.setattr(F, "main", lambda argv: argvs.append(argv) or 0)
    R.main(["-s", "S", "-m", "M", "--n_views", "3", "--infer_video"])
    assert "-r" not in argvs[-1] and "--resample_images" not in argvs[-1]             # the default -r -1 stays
    R.main(["-s", "S", "-m", "M", "--n_views", "3", "--infer_video", "-r", "4", "--resample_images"])
    assert argvs[-1][-3:] == ["-r", "4", "--resample_images"]
    R.main(["-s", "S", "-m", "M", "--n_views", "3", "--infer_video", "--resample_images"])
    assert argvs[-1][-3:] == ["-r", "-1", "--resample_images"]


def test_freeview_frame_size(tmp_path, monkeypatch):
    src = _source(str(tmp_path), W=1700, H=90)
    assert F.frame_size(src, 2) == (1700, 90)
    assert F.frame_size(src, 2, -1, True) == S.loaded_size(1700, 90, -1) == (1600, 84)
    assert F.frame_size(src, 2, 2, True) == (850, 45)
    with pytest.raises(ValueError, match="resampled images are not supported without --resample_images"):
        F.frame_size(src, 2, 2)
    # the command line: -r reaches load only with the flag's decision beside it
    seen = []
    monkeypatch.setattr(F, "load", lambda *a: seen.append(a) or (None, np.zeros((2, 4, 4)), 7))
    monkeypatch.setattr(F, "fly_through", lambda *a: (0, "x"))
    assert F.main(["-s", src, "-m", "M", "--n_views", "2"]) == 0
    assert seen[-1][-2:] == (1, False)
    assert F.main(["-s", src, "-m", "M", "--n_views", "2", "-r", "2", "--resample_images"]) == 0
    assert seen[-1][-2:] == (2, True)
