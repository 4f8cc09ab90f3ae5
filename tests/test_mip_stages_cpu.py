"""Mip-Splatting on the stage command lines, host side (instantsplat_b200/mip.py, DESIGN.md section 4.22): train's
namespace and cfg_args with and without --kernel_size, the OptimConfig it makes, every refusal with nothing written,
the pipeline's stage lines, the fly-through forwarding, the loaders' argument and --help of every stage."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from instantsplat_b200 import freeview as F
from instantsplat_b200 import metrics as M
from instantsplat_b200 import mip
from instantsplat_b200 import pipeline as P
from instantsplat_b200 import render_views as R
from instantsplat_b200 import scene_io as S
from instantsplat_b200 import train as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BAD = ["-0.1", "nan", "inf", "-inf"]


@pytest.fixture
def source(golden_dir, tmp_path):
    """The train golden's 4-view source, file for file."""
    z = np.load(os.path.join(golden_dir, "train.npz"))
    root = tmp_path / "src"
    for i, rel in enumerate(z["src_files"]):
        p = root / str(rel)
        p.parent.mkdir(parents=True, exist_ok=True)
        p.write_bytes(z[f"src_blob_{i}"].tobytes())
    return str(root)


def _model(root, filter_3D: bool, it=7, P_=5, n=4):
    """A model folder as train writes it: point_cloud/iteration_<it>/point_cloud.ply (save_gaussians_ply, with or
    without filter_3D) and pose/ours_<it>/pose_optimized.npy."""
    rng = np.random.default_rng(1)
    g = lambda *s: rng.standard_normal(s).astype(np.float32)
    S.save_gaussians_ply(os.path.join(root, "point_cloud", f"iteration_{it}", "point_cloud.ply"), g(P_, 3), g(P_, 1, 3),
                         g(P_, 15, 3), g(P_, 1), g(P_, 3), g(P_, 4),
                         np.abs(g(P_)) if filter_3D else None)
    poses = np.concatenate([np.tile([1.0, 0, 0, 0], (n, 1)), rng.standard_normal((n, 3))], axis=1)
    S.save_pose_npy(os.path.join(root, "pose", f"ours_{it}", "pose_optimized.npy"), poses)
    return root


def _tree(root):
    out = []
    for d, _, fs in os.walk(root):
        out += [os.path.relpath(os.path.join(d, f), root) for f in fs]
    return sorted(out)


# ---- train ---------------------------------------------------------------------------------------------------
def test_train_namespace_and_cfg_args_are_unchanged():
    base = ["-s", "S", "-m", "M", "--n_views", "3", "--iterations", "500", "--pp_optimizer", "--optim_pose"]
    a, b = T.parse_args(base), T.parse_args(base + ["--kernel_size", "0.1"])
    assert "kernel_size" not in vars(a)                           # train.py's own namespace
    assert b.kernel_size == 0.1 and mip.kernel_size(a) is None and mip.kernel_size(b) == 0.1
    assert vars(a) == {k: v for k, v in vars(b).items() if k != "kernel_size"}
    assert T.cfg_args_text(a).encode() == T.cfg_args_text(b).encode() and "kernel" not in T.cfg_args_text(b)
    assert T.refusals(a) == T.refusals(b) == []
    ca, cb = T.optim_config(a, 1.5), T.optim_config(b, 1.5)
    assert "mip_kernel_size" not in vars(ca) and ca.mip_kernel_size is None          # the class default
    assert cb.mip_kernel_size == 0.1
    assert {k: v for k, v in vars(ca).items()} == {k: v for k, v in vars(cb).items() if k != "mip_kernel_size"}
    assert T.optim_config(T.parse_args(base + ["--kernel_size", "0"]), 1.0).mip_kernel_size == 0.0


def test_golden_namespace_with_the_flag(golden_dir):
    """train.py's own argv parses to train.py's namespace; with the flag added, only kernel_size is new."""
    import json
    z = np.load(os.path.join(golden_dir, "train.npz"))
    argv = [str(a) for a in z["argv"]]
    ref = json.loads(str(z["ref_args_json"]))
    b = T.parse_args(argv + ["--kernel_size", "0.1"])
    assert vars(T.parse_args(argv)) == ref == {k: v for k, v in vars(b).items() if k != "kernel_size"}
    assert T.cfg_args_text(b).encode() == z["cfg_args"].tobytes()


@pytest.mark.parametrize("k", BAD)
def test_train_refuses_a_bad_kernel_size(source, tmp_path, k):
    model = tmp_path / "model"
    with pytest.raises(SystemExit, match=r"--kernel_size .*: the 2D Mip filter's kernel size must be a finite number"):
        T.main(["-s", source, "-m", str(model), "--n_views", "4", "-r", "1", "--iterations", "3", f"--kernel_size={k}"])
    assert not model.exists()


def test_kernel_refusal():
    for k in (None, 0.0, -0.0, 0.1, 0.3, 1e6):
        assert mip.kernel_refusal(k) is None, k
    for k in (-1e-9, -0.1, float("nan"), float("inf"), float("-inf")):
        assert "finite number >= 0" in mip.kernel_refusal(k), k
    assert mip.argv(None) == [] and mip.argv(0.1) == ["--kernel_size", "0.1"]
    for k in (0.1, 1 / 3, 0.0, 2.5e-7):
        assert float(mip.argv(k)[1]) == k


# ---- the ply -------------------------------------------------------------------------------------------------
def test_ply_properties_and_refusal(tmp_path):
    with_f = _model(str(tmp_path / "a"), True)
    without = _model(str(tmp_path / "b"), False)
    ply = lambda m: os.path.join(m, "point_cloud", "iteration_7", "point_cloud.ply")
    pa, pb = S.ply_properties(ply(with_f)), S.ply_properties(ply(without))
    assert pb == S.gaussian_ply_fields(45) and pa == pb + ["filter_3D"]
    assert mip.ply_refusal(0.1, ply(with_f)) is None
    assert mip.ply_refusal(None, ply(without)) is None                     # no flag: filter_3D not needed
    assert "has no filter_3D property" in mip.ply_refusal(0.1, ply(without))
    assert mip.ply_refusal(0.1, str(tmp_path / "missing.ply")) is None     # left to the loader


def test_tracker_from_gaussians_needs_filter_3D_with_kernel_size():
    g = {k: torch.zeros(2, *s) for k, s in dict(xyz=(3,), f_dc=(1, 3), f_rest=(15, 3), opacity=(1,), scaling=(3,),
                                                  rotation=(4,)).items()}
    with pytest.raises(ValueError, match="the model: no filter_3D"):
        F.tracker_from_gaussians(g, 8, 8, 1.0, 1.0, kernel_size=0.1)
    with pytest.raises(ValueError, match="finite number >= 0"):
        F.tracker_from_gaussians(dict(g, filter_3D=torch.zeros(2, 1)), 8, 8, 1.0, 1.0, kernel_size=float("nan"))


# ---- render_views and freeview -------------------------------------------------------------------------------
def _render_argv(model, *extra):
    return ["-s", "nowhere", "-m", model, "--n_views", "4", "--iterations", "7", "-r", "1", *extra]


@pytest.mark.parametrize("extra", [[], ["--eval"], ["--eval", "--test_fps"], ["--infer_video"]])
def test_render_views_refusals_write_nothing(tmp_path, monkeypatch, extra):
    model = _model(str(tmp_path / "model"), False)
    before = _tree(model)
    monkeypatch.setattr(F, "fly_through", lambda *a, **k: pytest.fail("the fly-through ran"))
    with pytest.raises(SystemExit, match="has no filter_3D property, so there is no 3D filter to apply"):
        R.main(_render_argv(model, *extra, "--kernel_size", "0.1"))
    for k in BAD:
        with pytest.raises(SystemExit, match="the 2D Mip filter's kernel size must be a finite number >= 0"):
            R.main(_render_argv(_model(str(tmp_path / "f"), True), *extra, f"--kernel_size={k}"))
    assert _tree(model) == before


def test_freeview_refusals_write_nothing(tmp_path, monkeypatch):
    model = _model(str(tmp_path / "model"), False)
    before = _tree(model)
    monkeypatch.setattr(F, "fly_through", lambda *a, **k: pytest.fail("the fly-through ran"))
    for it in ("7", "-1"):
        argv = ["-s", "nowhere", "-m", model, "--n_views", "4", "--iterations", it]
        with pytest.raises(SystemExit, match="freeview: --kernel_size: .* has no filter_3D property"):
            F.main(argv + ["--kernel_size", "0.1"])
        for k in BAD:
            with pytest.raises(SystemExit, match="freeview: --kernel_size .*: the 2D Mip filter's kernel size"):
                F.main(argv + [f"--kernel_size={k}"])
    assert _tree(model) == before


def test_the_flag_reaches_the_loaders(tmp_path, monkeypatch):
    """render_views hands --kernel_size to tracker_for, forwards it to the fly-through, and freeview hands it to load;
    without the flag every call is what it was."""
    model = _model(str(tmp_path / "model"), True)
    seen = []

    def tracker_for(*a, **k):
        seen.append(k)
        raise RuntimeError("stop")
    monkeypatch.setattr(R, "tracker_for", tracker_for)
    monkeypatch.setattr(R, "load_views", lambda *a, **k: None)
    for extra, want in (([], {"kernel_size": None}), (["--kernel_size", "0.25"], {"kernel_size": 0.25})):
        for stage in ([], ["--eval"]):
            with pytest.raises(RuntimeError, match="stop"):
                R.main(_render_argv(model, *stage, *extra))
            assert seen[-1] == want
    argvs = []
    monkeypatch.setattr(F, "main", lambda argv: argvs.append(argv) or 0)
    R.main(["-s", "S", "-m", "M", "--n_views", "3", "--infer_video"])
    assert "--kernel_size" not in argvs[-1]
    R.main(["-s", "S", "-m", "M", "--n_views", "3", "--infer_video", "-r", "2", "--resample_images",
            "--kernel_size", "0.1"])
    assert argvs[-1][-5:] == ["-r", "2", "--resample_images", "--kernel_size", "0.1"]


def test_freeview_hands_the_flag_to_load(tmp_path, monkeypatch):
    model = _model(str(tmp_path / "model"), True)
    seen = []
    monkeypatch.setattr(F, "load", lambda *a, **k: seen.append((a, k)) or (None, np.zeros((2, 4, 4)), 7))
    monkeypatch.setattr(F, "fly_through", lambda *a: (0, "x"))
    argv = ["-s", "S", "-m", model, "--n_views", "2"]
    assert F.main(argv) == 0 and seen[-1][1] == {}
    assert F.main(argv + ["--kernel_size", "0.1"]) == 0 and seen[-1][1] == {"kernel_size": 0.1}


# ---- pipeline ------------------------------------------------------------------------------------------------
def test_stage_argv_with_and_without_the_flag():
    src, model = "/data/Tanks/Horse/24_views", "out/Tanks/Horse/3_views"
    base = ["-s", src, "-m", model, "-r", "1", "--n_views", "3", "--iterations", "1000"]
    k = ["--kernel_size", "0.1"]
    t = P.Task("eval", "Tanks", "Horse", 3, 1000, src, model)
    plain = {"train": base + ["--pp_optimizer", "--optim_pose"], "render_train": base,
             "render_test": base + ["--eval"], "metrics": ["-s", src, "-m", model, "--n_views", "3"]}
    assert P.stage_argv(t) == P.stage_argv(t, kernel_size=None) == plain
    assert P.stage_argv(t, kernel_size=0.1) == {"train": plain["train"] + k, "render_train": base + k,
                                                "render_test": base + ["--eval"] + k, "metrics": plain["metrics"]}
    assert P.stage_argv(t, "/w", True, 0.1)["render_test"] == base + ["--eval", "--test_fps"] + k
    ti = P.Task("infer", "sora", "Art", 3, 1000, "/assets/sora/Art", "out/sora/Art/3_views")
    bi = ["-s", ti.source, "-m", ti.model, "-r", "1", "--n_views", "3", "--iterations", "1000"]
    assert P.stage_argv(ti) == {"train": bi + ["--pp_optimizer", "--optim_pose"], "render": bi + ["--infer_video"]}
    assert P.stage_argv(ti, kernel_size=0.1) == {"train": bi + ["--pp_optimizer", "--optim_pose"] + k,
                                                 "render": bi + ["--infer_video"] + k}
    # each line parsed by its stage's parser: kappa where the flag is, and no attribute where it is not
    got = P.stage_args(t, kernel_size=0.1)
    assert [mip.kernel_size(got[s]) for s in ("train", "render_train", "render_test")] == [0.1] * 3
    assert vars(got["metrics"]) == vars(M.parser().parse_args(plain["metrics"]))
    assert all("kernel_size" not in vars(v) for v in P.stage_args(t).values())
    assert mip.kernel_size(P.stage_args(ti, kernel_size=0.1)["render"]) == 0.1


@pytest.fixture
def data_root(golden_dir, tmp_path):
    """test_pipeline_cpu's layout: ROOT/Tanks/Horse/24_views with test views, ROOT/sora/Art."""
    import shutil
    z = np.load(os.path.join(golden_dir, "train.npz"))
    root = tmp_path / "data"
    for src in (root / "Tanks" / "Horse" / "24_views", root / "sora" / "Art"):
        for i, rel in enumerate(z["src_files"]):
            p = src / str(rel)
            p.parent.mkdir(parents=True, exist_ok=True)
            p.write_bytes(z[f"src_blob_{i}"].tobytes())
    eval_src = root / "Tanks" / "Horse" / "24_views"
    (eval_src / "sparse_4" / "1").mkdir()
    for f in ("cameras.txt", "images.txt"):
        shutil.copy(eval_src / "sparse_4" / "0" / f, eval_src / "sparse_4" / "1" / f)
    return root


def test_pipeline_refusals_write_nothing(data_root, tmp_path):
    out = tmp_path / "out"
    for mode, d, s in (("eval", "Tanks", "Horse"), ("infer", "sora", "Art")):
        ts = P.tasks(mode, str(data_root), str(out), [d], [s], [4], [10])
        assert P.refusals(ts[0], kernel_size=0.1) == P.refusals(ts[0]) == [], mode
        for k in BAD:
            argv = [mode, "--data_root", str(data_root), "--output_dir", str(out), "--datasets", d, "--scenes", s,
                    "--n_views", "4", "--iterations", "10", f"--kernel_size={k}"]
            with pytest.raises(SystemExit) as e:
                P.main(argv)
            assert "the 2D Mip filter's kernel size must be a finite number >= 0" in str(e.value.code)
            assert f"{d}/{s} (4 views/10 iters)" in str(e.value.code)
            assert not out.exists()


# ---- --help --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("argv", [["train"], ["render_views"], ["freeview"], ["pipeline", "eval"],
                                  ["pipeline", "infer"]])
def test_help_lists_the_flag(argv):
    r = subprocess.run([sys.executable, "-m", f"instantsplat_b200.{argv[0]}", *argv[1:], "--help"], cwd=ROOT,
                       capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr
    assert "--kernel_size K" in r.stdout and "Mip" in r.stdout
