"""render.py --test_fps, host side (no GPU): the trim and rate against render.py:180-182 restated, the bytes appended
to total_fps.json and train_time.txt, the flag on render_views and pipeline eval (not pipeline infer), the refusal
when there is no test view to time, and the pipeline's stage lines with and without it."""
import json
import os
import random
import time

import pytest

from instantsplat_b200 import pipeline as P
from instantsplat_b200 import render_views as R
from test_pipeline_cpu import _argv, _refused, data_root  # noqa: F401  (data_root is a fixture)
from test_render_views_cpu import _source


def _render_py_fps(durations):
    """render.py:180-182 as written there."""
    fps_list = list(durations)
    fps_list.sort()
    fps_list = fps_list[100:900]
    fps = 1 / (sum(fps_list) / len(fps_list))
    return fps


def _lists():
    rng = random.Random(11)
    base = [rng.uniform(0.5e-3, 2e-3) for _ in range(1000)]
    ties = [rng.choice([1e-3, 1.25e-3, 2e-3]) for _ in range(1000)]
    outliers = [1e-3 + rng.uniform(0, 1e-5) for _ in range(800)] + [1e-6] * 100 + [0.5] * 100
    rng.shuffle(outliers)
    return {"unsorted": base, "ties": ties, "outliers": outliers, "sorted": sorted(base),
            "reversed": sorted(base, reverse=True), "all_equal": [7e-4] * 1000}


@pytest.mark.parametrize("case", list(_lists()))
def test_trim_and_rate_are_render_py_s(case):
    d = _lists()[case]
    fps, line = R.fps_from_times(d)
    assert fps == _render_py_fps(d)
    assert isinstance(fps, float) and line == json.dumps(str(fps)) + "\n"
    assert float(json.loads(line)) == fps
    if case == "outliers":
        # the fastest and slowest 100 move the plain mean; the trimmed rate is that of the middle 800 alone
        middle = sorted(d)[100:900]
        assert max(middle) < 0.5 and min(middle) > 1e-6
        assert abs(fps - len(d) / sum(d)) > 0.5 * fps
        assert fps == 1 / (sum(middle) / 800)


def test_input_is_not_reordered():
    d = _lists()["unsorted"]
    before = list(d)
    R.fps_from_times(d)
    assert d == before


class _Timer:
    """Stands in for PoseTracker.time_renders with fixed frame times."""

    def __init__(self, times):
        self.times, self.calls = times, []

    def time_renders(self, pose, n=1000):
        self.calls.append((pose, n))
        return list(self.times[len(self.calls) - 1])


def test_two_runs_append_render_py_s_bytes(tmp_path, capsys):
    lists = _lists()
    runs = [lists["unsorted"], lists["outliers"]]
    timer = _Timer(runs)
    got, want = tmp_path / "got", tmp_path / "want"
    got.mkdir()
    want.mkdir()
    for k, d in enumerate(runs):
        fps = R.report_fps(timer, "pose", str(got), time.time())
        assert timer.calls[k] == ("pose", 1000)
        out = capsys.readouterr().out
        assert out == f">>> Calculate FPS: \n>>> FPS =  {fps}\n"
        ref = _render_py_fps(d)
        assert fps == ref
        with open(f"{want}/total_fps.json", 'a') as fp:            # render.py:184-186
            json.dump(f'{ref}', fp, indent=True)
            fp.write('\n')
    assert (got / "total_fps.json").read_bytes() == (want / "total_fps.json").read_bytes()
    lines = (got / "total_fps.json").read_text().splitlines()
    assert len(lines) == 2 and [float(json.loads(s)) for s in lines] == [_render_py_fps(d) for d in runs]
    # each run ends the `[4] render` span of render.py's eval branch (render.py:219-231)
    assert (got / "train_time.txt").read_text() == "[4] render: 0 min 0 sec\n" * 2


def test_flag_is_parsed():
    base = ["-s", "S", "-m", "M", "--n_views", "3"]
    assert not R.parser().parse_args(base).test_fps
    assert R.parser().parse_args(base + ["--eval", "--test_fps"]).test_fps
    pipe = ["--data_root", "D", "--output_dir", "O", "--datasets", "d", "--scenes", "s", "--n_views", "3",
            "--iterations", "10"]
    assert not P.parser().parse_args(["eval"] + pipe).test_fps
    assert P.parser().parse_args(["eval"] + pipe + ["--test_fps"]).test_fps
    with pytest.raises(SystemExit):
        P.parser().parse_args(["infer"] + pipe + ["--test_fps"])
    assert not hasattr(P.parser().parse_args(["infer"] + pipe), "test_fps")


def test_stage_lines_with_and_without_the_flag():
    t = P.Task("eval", "Tanks", "Horse", 3, 1000, "/data/Tanks/Horse/24_views", "out/Tanks/Horse/3_views")
    plain, fps = P.stage_argv(t), P.stage_argv(t, test_fps=True)
    assert P.stage_argv(t, test_fps=False) == plain
    assert plain["render_test"] == ["-s", t.source, "-m", t.model, "-r", "1", "--n_views", "3", "--iterations", "1000",
                                    "--eval"]
    assert fps["render_test"] == plain["render_test"] + ["--test_fps"]
    assert {k: v for k, v in fps.items() if k != "render_test"} == {k: v for k, v in plain.items()
                                                                     if k != "render_test"}
    args = P.stage_args(t, test_fps=True)
    assert args["render_test"].test_fps and args["render_test"].eval
    assert not P.stage_args(t)["render_test"].test_fps and not args["render_train"].test_fps
    assert P.stage_argv(t, "/w", True)["metrics"] == P.stage_argv(t, "/w")["metrics"]
    ti = P.Task("infer", "sora", "Art", 3, 1000, "/assets/sora/Art", "out/sora/Art/3_views")
    assert P.stage_argv(ti, test_fps=True) == P.stage_argv(ti)


def test_no_test_view_is_refused_before_anything_is_written(tmp_path):
    src, model = tmp_path / "src", tmp_path / "model"
    _source(str(src), ["a.png", "b.png"], [])
    argv = ["-s", str(src), "-m", str(model), "--n_views", "2", "--iterations", "7", "--eval"]
    with pytest.raises(SystemExit) as e:
        R.main(argv + ["--test_fps"])
    assert "--test_fps" in str(e.value.code) and "lists none" in str(e.value.code)
    assert os.path.join(str(src), "sparse_2", "1") in str(e.value.code)
    assert not model.exists()
    assert R.fps_refusal(str(src), 2) is not None
    _source(str(tmp_path / "ok"), ["a.png"], ["c.png"])
    assert R.fps_refusal(str(tmp_path / "ok"), 1) is None
    assert R.fps_refusal(str(tmp_path / "none"), 1) is None                  # unreadable: load_views' to report


def test_pipeline_refuses_no_test_view_with_the_flag(data_root, tmp_path):  # noqa: F811
    txt = data_root / "Tanks" / "Horse" / "24_views" / "sparse_4" / "1" / "images.txt"
    txt.write_text("# Image list with two lines of data per image:\n")
    t = P.tasks("eval", str(data_root), "out", ["Tanks"], ["Horse"], [4], [10])[0]
    assert not any("--test_fps" in r for r in P.refusals(t))                # the flag's refusal needs the flag
    assert any("--test_fps" in r for r in P.refusals(t, test_fps=True))
    out = tmp_path / "out"
    msg = _refused(_argv("eval", data_root, out) + ["--test_fps"], out)
    assert "--test_fps times the last test view" in msg and str(txt.parent) in msg
    assert "(4 views/10 iters)" in msg and "(4 views/20 iters)" in msg
