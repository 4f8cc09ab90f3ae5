"""The pipeline on the GPU (-m gpu, DESIGN.md section 4.18): `pipeline eval` and `pipeline infer` against the stage
CLIs run one after another into the same output directory (every file byte for byte, train_time.txt by line names,
the logs with their numbers masked), the tracker built from the trainer against load_tracker of the saved ply, the
in-memory metrics against metrics.main on the written PNGs, and the device memory left after a task."""
import contextlib
import os
import re
import shutil

import numpy as np
import pytest
import torch

from instantsplat_b200 import freeview as F
from instantsplat_b200 import metrics as M
from instantsplat_b200 import pipeline as P
from instantsplat_b200 import render_views as R
from instantsplat_b200 import scene_io as S
from instantsplat_b200 import train as T

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(scope="module")
def source(tmp_path_factory):
    """test_render_views_gpu's init_geo-shaped source: 3 training views and 4 test views at 96 x 64, images.bin."""
    from test_render_views_gpu import _source_and_model
    src, _, _ = _source_and_model(str(tmp_path_factory.mktemp("gen")))
    return src


def _data_root(root, source, mode):
    """Two scenes: A with sparse/0/images.bin, B without it (metrics then skips the pose errors)."""
    for scene in ("A", "B"):
        dst = os.path.join(root, "D", scene, "24_views" if mode == "eval" else "")
        shutil.copytree(source, dst)
        if scene == "B":
            shutil.rmtree(os.path.join(dst, "sparse"))
    return root


def _run_clis(ts):
    """The scripts' way: each stage's CLI on its line, what it prints sent to the script's log file."""
    clis = {"train": T.main, "render_train": R.main, "render_test": R.main, "metrics": M.main, "render": R.main}
    for t in ts:
        os.makedirs(t.model, exist_ok=True)
        for key, argv in P.stage_argv(t).items():
            with open(os.path.join(t.model, P.STAGES[t.mode][key][0]), "w") as f, \
                    contextlib.redirect_stdout(f), contextlib.redirect_stderr(f):
                clis[key](argv)


def _files(root):
    out = []
    for d, _, fs in os.walk(root):
        out += [os.path.relpath(os.path.join(d, f), root) for f in fs]
    return sorted(out)


def _compare_trees(a, b):
    fa = _files(a)
    assert fa == _files(b)
    mask = lambda s: re.sub(r"\d+(\.\d+)?(e[-+]?\d+)?", "#", s)
    for rel in fa:
        x, y = (open(os.path.join(r, rel), "rb").read() for r in (a, b))
        if rel.endswith("train_time.txt"):
            names = lambda t: [l.split(":")[0] for l in t.decode().splitlines()]
            assert names(x) == names(y), rel
        elif rel.endswith("02_train.log"):
            # the train stage prints its loss lines when their asynchronous copy lands, so where they fall among the
            # save lines depends on timing, in the CLI as much as here: the lines are compared, not their order
            assert sorted(mask(x.decode()).splitlines()) == sorted(mask(y.decode()).splitlines()), rel
        elif rel.endswith(".log"):
            assert mask(x.decode()) == mask(y.decode()), rel
        else:
            assert x == y, rel
    return fa


def _pipeline_and_clis(tmp_path, source, mode, scenes, iterations):
    """Runs the CLIs into OUT, moves OUT aside, runs the pipeline into OUT: the paths inside the files agree."""
    root = _data_root(str(tmp_path / "data"), source, mode)
    out = str(tmp_path / "out")
    ts = P.tasks(mode, root, out, ["D"], scenes, [3], iterations)
    _run_clis(ts)
    os.rename(out, str(tmp_path / "cli"))
    argv = [mode, "--data_root", root, "--output_dir", out, "--datasets", "D", "--scenes", *scenes, "--n_views", "3",
            "--iterations", *map(str, iterations), "--workers", "2"]
    assert P.main(argv) == 0
    return root, out, _compare_trees(out, str(tmp_path / "cli"))


def test_eval_equals_the_stage_clis(tmp_path, source, capsys):
    root, out, files = _pipeline_and_clis(tmp_path, source, "eval", ["A", "B"], [20, 30])
    con = capsys.readouterr().out
    assert con.count("Starting training...") == 4 and "Processing task 4 / 4" in con
    assert "All tasks completed! Processed 4 tasks in total." in con
    for scene in ("A", "B"):
        pre = os.path.join("D", scene, "3_views")
        for it in (20, 30):
            for f in ("renders/t0.png", "gt/t3.png", "metrics.txt"):
                assert os.path.join(pre, "test", f"ours_{it}", f) in files
            assert os.path.join(pre, "train", f"ours_{it}", "renders", "00002.png") in files
        assert (os.path.join(pre, "pose", "ours_30", "pose_eval.txt") in files) == (scene == "A")
        for log in ("02_train.log", "03_render_train.log", "04_render_test.log", "05_metrics.log"):
            assert os.path.join(pre, log) in files
        assert "poses: skipped" in open(os.path.join(out, pre, "05_metrics.log")).read() or scene == "A"
        # the in-memory numbers are metrics.main's on the written PNGs
        model = os.path.join(out, pre)
        again = str(tmp_path / f"again_{scene}")
        shutil.copytree(model, again)
        with contextlib.redirect_stdout(open(os.devnull, "w")):
            assert M.main(["-s", os.path.join(root, "D", scene, "24_views"), "-m", again, "--n_views", "3"]) == 0
        for rel in ["results.json", "per_view.json"] + [os.path.join("test", f"ours_{it}", "metrics.txt")
                                                        for it in (20, 30)]:
            assert open(os.path.join(model, rel), "rb").read() == open(os.path.join(again, rel), "rb").read(), rel


def test_infer_equals_the_stage_clis(tmp_path, source):
    _, _, files = _pipeline_and_clis(tmp_path, source, "infer", ["A"], [20])
    pre = os.path.join("D", "A", "3_views")
    frames = [f for f in files if f.startswith(os.path.join(pre, "interp", "ours_20", "renders"))]
    assert len(frames) == 2 * int(300 / 3) + 1
    assert os.path.join(pre, "pose", "ours_20", "pose_interpolated.npy") in files
    assert os.path.join(pre, "03_render.log") in files


def test_tracker_from_the_trainer_is_the_ply_tracker(tmp_path, source):
    args = T.parse_args(["-s", source, "-m", str(tmp_path / "m"), "-r", "1", "--n_views", "3", "--iterations", "20",
                         "--pp_optimizer", "--optim_pose", "--quiet"])
    res = T.run(args)
    assert res.trainer.active_sh_degree == 0 and res.trainer.stored_sh_degree == 3
    v = res.host.views
    got = F.tracker_from_gaussians(res.trainer.ply_tensors(), v.width, v.height, v.fovx, v.fovy)
    ply = os.path.join(args.model_path, "point_cloud", "iteration_20", "point_cloud.ply")
    want = F.load_tracker(ply, v.width, v.height, v.fovx, v.fovy)
    assert got.sh_degree == want.sh_degree == 3
    for k in ("xyz", "rotation", "scaling", "opacity", "f_dc", "f_rest"):
        a, b = getattr(got, k), getattr(want, k)
        assert a.dtype == b.dtype and a.shape == b.shape and torch.equal(a, b), k
    assert got.filter_3D is None and want.filter_3D is None
    assert (got.W, got.H, got.P) == (want.W, want.H, want.P)
    keys = S.pose_matrices(res.trainer.poses.detach().cpu().numpy(), res.colmap_ids)
    saved = np.load(os.path.join(args.model_path, "pose", "ours_20", "pose_optimized.npy"))
    assert keys.dtype == saved.dtype and np.array_equal(keys, saved)


def test_a_task_releases_its_device_memory(tmp_path, source):
    root = _data_root(str(tmp_path / "data"), source, "eval")
    after = []
    for k in range(2):
        ts = P.tasks("eval", root, str(tmp_path / f"out{k}"), ["D"], ["A"], [3], [20])
        with contextlib.redirect_stdout(open(os.devnull, "w")):
            assert P.run_tasks(ts, workers=2)[0] == 0
        torch.cuda.synchronize()
        after.append(torch.cuda.memory_allocated())
    assert after[0] == after[1], after
