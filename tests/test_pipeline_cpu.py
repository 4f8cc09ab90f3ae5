"""The pipeline's host side (instantsplat_b200/pipeline.py, DESIGN.md section 4.18): its task list and paths against
run_eval.sh's and run_infer.sh's loops, each stage's arguments against the script's line parsed by the stage's own
parser, every refusal with nothing written, the PNG pool, the in-memory metrics path and --help."""
import filecmp
import json
import os
import shutil
import subprocess
import sys
import threading

import numpy as np
import pytest
import torch

from instantsplat_b200 import freeview as F
from instantsplat_b200 import metrics as M
from instantsplat_b200 import pipeline as P
from instantsplat_b200 import render_views as R
from instantsplat_b200 import train as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _scripts_loop(mode, root, out, datasets, scenes, n_views, iterations):
    """The scripts' main loop and run_on_gpu's SOURCE_PATH / MODEL_PATH, as the shell builds them."""
    rows = []
    for d in datasets:
        for s in scenes:
            for n in n_views:
                for it in iterations:
                    src = f"{root}/{d}/{s}/24_views/" if mode == "eval" else f"{root}/{d}/{s}/"
                    rows.append((d, s, n, it, src, f"./{out}/{d}/{s}/{n}_views"))
    return rows


@pytest.mark.parametrize("mode", ["eval", "infer"])
def test_task_order_and_paths(mode):
    args = ("ROOT", "out", ["Tanks", "MVimgNet"], ["Family", "Horse", "Barn"], [3, 6, 12], [200, 1000])
    ts = P.tasks(mode, *args)
    want = _scripts_loop(mode, *args)
    assert len(ts) == len(want) == 2 * 3 * 3 * 2
    for t, (d, s, n, it, src, model) in zip(ts, want):
        assert (t.mode, t.dataset, t.scene, t.n_views, t.iterations) == (mode, d, s, n, it)
        assert os.path.normpath(t.source) == os.path.normpath(src)
        assert os.path.normpath(t.model) == os.path.normpath(model)


def test_stage_arguments_are_the_scripts_lines():
    src, model = "/data/Tanks/Horse/24_views", "out/Tanks/Horse/3_views"
    t = P.Task("eval", "Tanks", "Horse", 3, 1000, src, model)
    got = P.stage_args(t)
    assert list(got) == ["train", "render_train", "render_test", "metrics"]
    sm = ["-s", src, "-m", model]
    want = {"train": T.parse_args(sm + ["-r", "1", "--n_views", "3", "--iterations", "1000", "--pp_optimizer",
                                        "--optim_pose"]),
            "render_train": R.parser().parse_args(sm + ["-r", "1", "--n_views", "3", "--iterations", "1000"]),
            "render_test": R.parser().parse_args(sm + ["-r", "1", "--n_views", "3", "--iterations", "1000", "--eval"]),
            "metrics": M.parser().parse_args(sm + ["--n_views", "3"])}
    for k in want:
        assert vars(got[k]) == vars(want[k]), k
    assert got["train"].save_iterations == [1000] and got["train"].pp_optimizer and got["train"].optim_pose
    assert got["render_test"].optim_test_pose_iter == 500 and got["render_test"].max_batch == 12
    lp = P.stage_args(t, lpips_weights="/w")["metrics"]
    assert vars(lp) == vars(M.parser().parse_args(sm + ["--n_views", "3", "--lpips_weights", "/w"]))
    ti = P.Task("infer", "sora", "Art", 3, 1000, "/assets/sora/Art", "out/sora/Art/3_views")
    got = P.stage_args(ti)
    assert list(got) == ["train", "render"]
    assert vars(got["render"]) == vars(R.parser().parse_args(
        ["-s", ti.source, "-m", ti.model, "-r", "1", "--n_views", "3", "--iterations", "1000", "--infer_video"]))
    assert got["render"].infer_video and not got["render"].eval


# ---- refusals ------------------------------------------------------------------------------------------------
@pytest.fixture
def data_root(golden_dir, tmp_path):
    """ROOT/Tanks/Horse/24_views (eval) and ROOT/sora/Art (infer): the train golden's 4-view source, with its
    training views copied as test views for eval; no sparse/0/images.bin."""
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


def _refused(argv, out):
    with pytest.raises(SystemExit) as e:
        P.main(argv)
    assert not os.path.exists(out), "a refused run wrote something"
    return str(e.value.code)


def _argv(mode, root, out, scenes=("Horse",), n=("4",), datasets=("Tanks",)):
    return [mode, "--data_root", str(root), "--output_dir", str(out), "--datasets", *datasets, "--scenes", *scenes,
            "--n_views", *n, "--iterations", "10", "20"]


def test_complete_sources_are_not_refused(data_root):
    for mode, d, s in (("eval", "Tanks", "Horse"), ("infer", "sora", "Art")):
        ts = P.tasks(mode, str(data_root), "out", [d], [s], [4], [10])
        assert P.refusals(ts[0]) == [], mode        # no sparse/0/images.bin: metrics skips the pose errors


@pytest.mark.parametrize("missing", ["sparse_4/0/points3D.ply", "sparse_4/0/confidence_dsp.npy", "sparse_4/1"])
def test_missing_init_geo_outputs_are_refused(data_root, tmp_path, missing):
    src = data_root / "Tanks" / "Horse" / "24_views"
    p = src / missing
    shutil.rmtree(p) if p.is_dir() else p.unlink()
    out = tmp_path / "out"
    msg = _refused(_argv("eval", data_root, out), out)
    assert str(p) in msg and "Tanks/Horse (4 views/10 iters)" in msg and "(4 views/20 iters)" in msg


def test_a_bad_task_stops_every_task(data_root, tmp_path):
    """Horse is complete, Barn is absent: nothing is written, Horse included."""
    out = tmp_path / "out"
    msg = _refused(_argv("eval", data_root, out, scenes=("Horse", "Barn")), out)
    assert "Barn" in msg and "Horse" not in msg
    assert os.path.join(str(data_root), "Tanks", "Barn", "24_views", "sparse_4", "0", "points3D.ply") in msg


def test_train_cli_refusals_are_reported(data_root, tmp_path):
    from PIL import Image
    img = data_root / "Tanks" / "Horse" / "24_views" / "images" / "b.png"
    Image.open(img).convert("RGBA").save(img)
    out = tmp_path / "out"
    msg = _refused(_argv("eval", data_root, out), out)
    assert "RGBA" in msg and str(img) in msg
    with pytest.raises(T.Refused, match="RGBA"):      # the train CLI's own refusal
        T.run(T.parse_args(["-s", str(img.parent.parent), "-m", str(out), "-r", "1", "--n_views", "4"]))
    assert not os.path.exists(out)


def test_other_refusals(data_root, tmp_path):
    out = tmp_path / "out"
    msg = _refused(_argv("infer", data_root, out, ("Art",), ("1",), ("sora",)), out)
    assert "--n_views must be at least 2" in msg
    ply = data_root / "sora" / "Art" / "sparse_4" / "0" / "points3D.ply"
    ply.unlink()
    assert str(ply) in _refused(_argv("infer", data_root, out, ("Art",), datasets=("sora",)), out)
    _refused(_argv("eval", data_root, out) + ["--lpips_weights", str(tmp_path / "none")], out)
    _refused(_argv("eval", data_root, out) + ["--workers", "0"], out)


# ---- the PNG pool --------------------------------------------------------------------------------------------
def _frames(n=7, H=6, W=10, seed=0):
    return np.random.default_rng(seed).integers(0, 256, (n, H, W, 3), dtype=np.uint8)


def test_png_writer_writes_what_write_pngs_writes(tmp_path):
    u8 = _frames()
    F.write_pngs([(0, u8[:3]), (3, u8[3:])], str(tmp_path / "a"), workers=2)
    names = [f"v{i}.png" for i in range(7)]
    F.write_pngs([(0, u8)], str(tmp_path / "na"), workers=1, names=names)
    w = P.PngWriter(workers=3)
    assert w.write([(0, u8[:3]), (3, u8[3:])], str(tmp_path / "b")) == 7
    assert w.write([(0, u8)], str(tmp_path / "nb"), None, names) == 7
    w.close()
    for a, b, files in (("a", "b", [f"{i:05d}.png" for i in range(7)]), ("na", "nb", names)):
        assert sorted(os.listdir(tmp_path / b)) == sorted(files)
        match, mismatch, errors = filecmp.cmpfiles(tmp_path / a, tmp_path / b, files, shallow=False)
        assert not mismatch and not errors


def test_png_writer_bounds_the_queue_and_does_not_wait(tmp_path, monkeypatch):
    gate, seen = threading.Event(), []
    real = F._save_png

    def slow(img, path):
        gate.wait()
        real(img, path)
    monkeypatch.setattr(F, "_save_png", slow)
    w = P.PngWriter(workers=1)
    assert w.cap == 4
    w.write([(0, _frames(3))], str(tmp_path / "q"))          # returns with all three encodes still blocked
    assert len(w._pending) == 3 and not os.listdir(tmp_path / "q")

    def frames():
        for i in range(6):
            seen.append(len(w._pending))
            yield i, _frames(1, seed=i)
    threading.Timer(0.3, gate.set).start()
    w.write(frames(), str(tmp_path / "r"))
    assert max(seen) <= w.cap
    w.close()
    assert len(os.listdir(tmp_path / "q")) == 3 and len(os.listdir(tmp_path / "r")) == 6


def test_a_failed_write_fails_the_run_and_names_the_file(tmp_path):
    folder = tmp_path / "f"
    (folder / "00001.png").mkdir(parents=True)               # a directory where a frame's file goes
    w = P.PngWriter(workers=2)
    with pytest.raises(P.WriteError, match="00001.png"):      # from whichever call finds it done first
        w.write([(0, _frames(3))], str(folder))
        w.close()
    w.close()
    assert (folder / "00000.png").is_file() and (folder / "00002.png").is_file()   # every other write finished


# ---- metrics from memory -------------------------------------------------------------------------------------
def _fake_numbers(renders, gts, device="cuda"):
    return {"PSNR": torch.tensor([10.0 + float(r.astype(np.float64).mean()) for r in renders], dtype=torch.float64),
            "SSIM": torch.tensor([float(g.astype(np.float64).mean()) / 255 for g in gts], dtype=torch.float64)}


def test_held_pairs_give_the_files_numbers(tmp_path, monkeypatch):
    """metrics.evaluate with the current method in memory writes what it writes from the PNGs, an earlier method
    read from its files alongside."""
    monkeypatch.setattr(M, "image_numbers", _fake_numbers)
    src = tmp_path / "src"
    src.mkdir()
    a = tmp_path / "a" / "model"
    names = ["t2.png", "t0.png", "t1.png", "t10.png"]
    u8 = {m: (_frames(4, seed=1 + k), _frames(4, seed=7 + k)) for k, m in enumerate(("ours_5", "ours_9"))}
    for m, (r, g) in u8.items():
        F.write_pngs([(0, r)], str(a / "test" / m / "renders"), 1, names)
        F.write_pngs([(0, g)], str(a / "test" / m / "gt"), 1, names)
    b = tmp_path / "b" / "model"
    shutil.copytree(a, b)
    assert M.evaluate([str(a)], str(src), 3) == 0
    order = sorted(range(4), key=names.__getitem__)
    r, g = u8["ours_9"]
    assert M.evaluate([str(b)], str(src), 3, held={"ours_9": (r[order], g[order], [names[i] for i in order])}) == 0
    for f in ("results.json", "per_view.json", "test/ours_5/metrics.txt", "test/ours_9/metrics.txt"):
        assert (a / f).read_bytes() == (b / f).read_bytes(), f
    assert list(json.loads((b / "per_view.json").read_text())["ours_9"]["PSNR"]) == sorted(names)


def test_help():
    for argv in ([], ["eval"], ["infer"]):
        r = subprocess.run([sys.executable, "-m", "instantsplat_b200.pipeline", *argv, "--help"], cwd=ROOT,
                           capture_output=True, text=True, timeout=120)
        assert r.returncode == 0, r.stderr
        for flag in (["eval", "infer"] if not argv else ["--data_root", "--output_dir", "--datasets", "--scenes",
                                                         "--n_views", "--iterations", "--workers"]):
            assert flag in r.stdout, (argv, flag)
    assert "--lpips_weights" in subprocess.run([sys.executable, "-m", "instantsplat_b200.pipeline", "eval", "--help"],
                                               cwd=ROOT, capture_output=True, text=True, timeout=120).stdout
