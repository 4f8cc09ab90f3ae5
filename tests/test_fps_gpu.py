"""render.py --test_fps on the GPU (-m gpu): PoseTracker.time_renders' replayed forward against render_batch, its
durations, its memory and its overflow check; render_views --eval --test_fps and pipeline eval --test_fps against
the same runs without the flag, file for file."""
import contextlib
import json
import math
import os
import re
import shutil

import pytest
import torch

from instantsplat_b200 import GsbError
from instantsplat_b200 import pipeline as P
from instantsplat_b200 import render_views as R
from instantsplat_b200.frame import mip_filter3d, read_R
from instantsplat_b200.scenes import surface_scene
from instantsplat_b200.tracking import PoseTracker

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _tracker(sc, white=False, mip=False, **kw):
    p = sc.params
    if mip:
        kw = dict(kernel_size=0.1, filter_3D=mip_filter3d(p["xyz"].to(DEV), sc.poses.to(DEV), sc.width, sc.height,
                                                          math.tan(sc.fovx / 2), math.tan(sc.fovy / 2)))
    return PoseTracker(p["xyz"], p["rotation"], p["scaling"], p["opacity"], p["f_dc"], p["f_rest"], sc.width, sc.height,
                       sc.fovx, sc.fovy, bg=torch.ones(3) if white else None, sh_degree=sc.sh_degree, device=DEV, **kw)


@pytest.mark.parametrize("deg,white,mip", [(0, False, False), (0, True, False), (3, False, False), (3, True, False),
                                           (3, False, True)])
def test_replayed_image_is_render_batch(deg, white, mip):
    sc = surface_scene(6000, 3, 96, 64, seed=41, sh_degree=deg)
    tk = _tracker(sc, white, mip)
    out = torch.empty(3, sc.height, sc.width, device=DEV)
    for v, n in ((0, 1), (2, 7)):
        pose = sc.poses[v] + 0.01 * v
        out.fill_(float("nan"))
        tk.time_renders(pose, n, out=out)
        assert torch.equal(out, tk.render_batch(pose.reshape(1, 7))[0]), (v, n)
    # a device pose row, and a frame of several tiles' worth of lists
    big = surface_scene(20000, 2, 256, 192, seed=42, sh_degree=deg)
    tk = _tracker(big, white)
    pose = big.poses[1].to(DEV)
    out = torch.empty(3, big.height, big.width, device=DEV)
    tk.time_renders(pose, 3, out=out)
    assert torch.equal(out, tk.render_batch(pose.reshape(1, 7))[0])
    assert float(out.std()) > 0


def test_durations_and_memory():
    sc = surface_scene(6000, 3, 96, 64, seed=43, sh_degree=3)
    tk = _tracker(sc)
    tk.render(sc.poses[0])
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    t1 = tk.time_renders(sc.poses[0], 200)
    after1 = torch.cuda.memory_allocated()
    t2 = tk.time_renders(sc.poses[1], 50)
    after2 = torch.cuda.memory_allocated()
    assert before == after1 == after2, (before, after1, after2)
    assert len(t1) == 200 and len(t2) == 50
    assert all(isinstance(t, float) and math.isfinite(t) and t > 0 for t in t1 + t2)
    fps, line = R.fps_from_times(t1 * 5)
    assert math.isfinite(fps) and fps > 0 and float(json.loads(line)) == fps
    with pytest.raises(ValueError):
        tk.time_renders(sc.poses[0], 0)
    with pytest.raises(ValueError):
        tk.time_renders(sc.poses[:2], 1)


def test_small_binning_capacity_raises():
    sc = surface_scene(100000, 3, 256, 192, seed=4, sh_degree=0)
    tk = _tracker(sc)
    tk.render_batch(sc.poses[:1])
    assert read_R(tk.host_status) > 65536 + 1000                 # more instances than the capacity floor
    assert len(tk.time_renders(sc.poses[0], 3)) == 3
    tk.headroom = 0.0                                             # binning buffer = the 65536-instance floor
    with pytest.raises(GsbError, match="binning buffer"):
        tk.time_renders(sc.poses[0], 3)
    torch.cuda.synchronize()


# ---- the command lines -------------------------------------------------------------------------------------------
def _files(root):
    out = []
    for d, _, fs in os.walk(root):
        out += [os.path.relpath(os.path.join(d, f), root) for f in fs]
    return sorted(out)


MASK = lambda s: re.sub(r"\d+(\.\d+)?(e[-+]?\d+)?", "#", s)
FPS_LINES = ">>> Calculate FPS: \n>>> FPS =  #\n"


def test_render_views_cli(tmp_path, capsys):
    from test_render_views_gpu import _source_and_model
    src, model, it = _source_and_model(str(tmp_path))
    plain, timed = str(tmp_path / "plain"), str(tmp_path / "timed")
    shutil.copytree(model, plain)
    shutil.copytree(model, timed)
    base = ["-s", src, "--n_views", "3", "--iterations", str(it), "--eval", "--optim_test_pose_iter", "20",
            "--max_batch", "3", "--workers", "2"]
    assert R.main(base + ["-m", plain]) == 0
    out_plain = capsys.readouterr().out
    assert R.main(base + ["-m", timed, "--test_fps"]) == 0
    out_timed = capsys.readouterr().out
    assert ">>> Calculate FPS: \n>>> FPS =  " in out_timed and ">>> FPS" not in out_plain
    assert FPS_LINES in MASK(out_timed)
    assert MASK(out_timed).replace(FPS_LINES, "", 1) == MASK(out_plain.replace(plain, timed))
    fa, fb = _files(plain), _files(timed)
    assert sorted(set(fb) - set(fa)) == ["total_fps.json", "train_time.txt"] and set(fa) <= set(fb)
    pngs = [f for f in fa if f.endswith(".png") and f.startswith("test")]
    assert len(pngs) == 8
    for rel in fa:
        assert open(os.path.join(plain, rel), "rb").read() == open(os.path.join(timed, rel), "rb").read(), rel
    lines = open(os.path.join(timed, "total_fps.json")).read().splitlines()
    assert len(lines) == 1 and float(json.loads(lines[0])) > 0
    assert re.fullmatch(r"\[4\] render: \d+ min \d+ sec\n", open(os.path.join(timed, "train_time.txt")).read())
    # a second run appends one line to each file
    assert R.main(base + ["-m", timed, "--test_fps"]) == 0
    assert len(open(os.path.join(timed, "total_fps.json")).read().splitlines()) == 2
    assert [l.split(":")[0] for l in open(os.path.join(timed, "train_time.txt"))] == ["[4] render"] * 2
    # without --eval the flag does nothing (render.py's train branch has no FPS loop)
    again = str(tmp_path / "train_only")
    shutil.copytree(model, again)
    assert R.main(["-s", src, "-m", again, "--n_views", "3", "--iterations", str(it), "--test_fps",
                   "--workers", "2"]) == 0
    assert not os.path.exists(os.path.join(again, "total_fps.json"))
    assert not os.path.exists(os.path.join(again, "train_time.txt"))


def test_pipeline_eval(tmp_path):
    from test_pipeline_gpu import _data_root
    from test_render_views_gpu import _source_and_model
    src, _, _ = _source_and_model(str(tmp_path / "gen"))
    root = _data_root(str(tmp_path / "data"), src, "eval")
    a, b = str(tmp_path / "plain"), str(tmp_path / "out")
    for extra in ([], ["--test_fps"]):             # both into OUT, the first moved aside: the paths in the files agree
        argv = ["eval", "--data_root", root, "--output_dir", b, "--datasets", "D", "--scenes", "A", "--n_views", "3",
                "--iterations", "20", "--workers", "2"] + extra
        with contextlib.redirect_stdout(open(os.devnull, "w")):
            assert P.main(argv) == 0
        if not extra:
            os.rename(b, a)
    fa, fb = _files(a), _files(b)
    model = os.path.join("D", "A", "3_views")
    assert fb == sorted(fa + [os.path.join(model, "total_fps.json")])
    lines = open(os.path.join(b, model, "total_fps.json")).read().splitlines()
    assert len(lines) == 1 and float(json.loads(lines[0])) > 0
    for rel in fa:
        x, y = (open(os.path.join(r, rel), "rb").read().decode(errors="replace") if rel.endswith((".log", ".txt"))
                else open(os.path.join(r, rel), "rb").read() for r in (a, b))
        if rel.endswith("train_time.txt"):
            names = lambda t: [l.split(":")[0] for l in t.splitlines()]
            assert names(y) == names(x) + ["[4] render"], rel
        elif rel.endswith("02_train.log"):
            assert sorted(MASK(x).splitlines()) == sorted(MASK(y).splitlines()), rel
        elif rel.endswith("04_render_test.log"):
            assert FPS_LINES in MASK(y) and MASK(y).replace(FPS_LINES, "", 1) == MASK(x), rel
        elif rel.endswith(".log"):
            assert MASK(x) == MASK(y), rel
        else:
            assert x == y, rel
