"""point_cloud.ply on the GPU, host side (instantsplat_b200/ply.py, DESIGN.md section 4.23): the pack and unpack entry
points are declared, exported and typed and refuse bad arguments before any launch, the GPU writer's header is the
numpy writer's at every SH degree with and without filter_3D, only that exact layout takes the GPU reader (every
other file goes to the numpy reader), and --ply_io parses on every command line without changing a namespace or a
stage line when it is absent."""
import ctypes
import os
import re

import numpy as np
import pytest

from instantsplat_b200 import freeview as F
from instantsplat_b200 import pipeline as P
from instantsplat_b200 import ply
from instantsplat_b200 import render_views as R
from instantsplat_b200 import scene_io as S
from instantsplat_b200 import train as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEGREES = [0, 1, 2, 3]


def _tensors(P_, deg, filt, seed=0):
    rng = np.random.default_rng(seed)
    g = lambda *s: rng.standard_normal(s).astype(np.float32)
    rows = (deg + 1) ** 2 - 1
    return dict(xyz=g(P_, 3), f_dc=g(P_, 1, 3), f_rest=g(P_, rows, 3), opacity=g(P_, 1), scaling=g(P_, 3),
                rotation=g(P_, 4), filter_3D=np.abs(g(P_)) if filt else None)


def _numpy_file(path, P_, deg, filt, seed=0):
    S.save_gaussians_ply(path, **_tensors(P_, deg, filt, seed))
    return path


def _header(path):
    data = open(path, "rb").read()
    return data[:data.index(b"end_header\n") + len(b"end_header\n")]


# ---- the C ABI -----------------------------------------------------------------------------------------------
def test_entry_points_declared_exported_and_typed():
    import __graft_entry__ as G
    G.build()
    import instantsplat_b200 as I
    from instantsplat_b200._lib import GsbPlySegment
    L = I.lib()
    hdr = open(os.path.join(ROOT, "include", "gsb200.h")).read()
    declared = set(re.findall(r"GSB_API [^;(]*?\b(gsb_\w+)\(", hdr))
    for name in ("gsb_ply_pack", "gsb_ply_unpack"):
        assert name in declared and name in I._lib.EXPORTS and hasattr(L, name), name
        assert getattr(L, name).restype is ctypes.c_int
    vp, i32, i64 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64
    seg = ctypes.POINTER(GsbPlySegment)
    assert L.gsb_ply_pack.argtypes == [i64, i32, seg, vp, vp]
    assert L.gsb_ply_unpack.argtypes == [i64, vp, i32, seg, vp]
    assert [f[0] for f in GsbPlySegment._fields_] == ["data", "width", "inner"]
    assert re.search(r"#define GSB_PLY_MAX_SEGMENTS 8\b", hdr) and re.search(r"#define GSB_PLY_MAX_FLOATS 64\b", hdr)
    assert I._lib.PLY_MAX_SEGMENTS == 8
    for name, params in (("gsb_ply_pack", 5), ("gsb_ply_unpack", 5)):
        decl = re.search(name + r"\(([^)]*)\)", hdr).group(1)
        assert len(decl.split(",")) == params, name


def test_bad_arguments_are_refused_before_any_launch():
    import instantsplat_b200 as I
    from instantsplat_b200._lib import GsbPlySegment
    L = I.lib()
    launches = L.gsb_launch_count()
    table = lambda *segs: (GsbPlySegment * len(segs))(*[GsbPlySegment(d, w, k) for d, w, k in segs])
    ok = table((None, 3, 3), (None, 45, 3))
    for pack in (True, False):
        call = (lambda P_, n, segs, buf: L.gsb_ply_pack(P_, n, segs, buf, None)) if pack else \
            (lambda P_, n, segs, buf: L.gsb_ply_unpack(P_, buf, n, segs, None))
        assert call(0, 2, ok, 16) == 0                                # nothing to do: no launch
        assert call(-1, 2, ok, 16) == -1
        assert call(4, 0, ok, 16) == -1
        assert call(4, 9, table(*[(None, 1, 1)] * 9), 16) == -1       # more than GSB_PLY_MAX_SEGMENTS
        assert call(4, 2, None, 16) == -1
        assert call(4, 2, ok, None) == -1
        assert call(4, 2, ok, 18) == -1                               # buffer not 4-byte aligned
        assert call(4, 1, table((None, 45, 4)), 16) == -1             # inner does not divide width
        assert call(4, 1, table((None, 0, 1)), 16) == -1
        assert call(4, 1, table((None, 3, 0)), 16) == -1
        assert call(4, 1, table((18, 3, 3)), 16) == -1                # data not 4-byte aligned
        assert call(4, 2, table((None, 60, 3), (None, 5, 5)), 16) == -1     # 65 words > GSB_PLY_MAX_FLOATS
        assert call(1 << 62, 1, table((None, 3, 3)), 16) == -1        # more CTAs than grid.x holds
    assert "gsb_ply_unpack" in L.gsb_last_error().decode()
    assert L.gsb_launch_count() == launches


# ---- the header and the layout -------------------------------------------------------------------------------
@pytest.mark.parametrize("deg", DEGREES)
@pytest.mark.parametrize("filt", [False, True])
@pytest.mark.parametrize("P_", [0, 1, 129])
def test_header_is_the_numpy_writers(tmp_path, deg, filt, P_):
    path = _numpy_file(str(tmp_path / "a.ply"), P_, deg, filt)
    rows = (deg + 1) ** 2 - 1
    assert S.gaussian_ply_header(P_, 3 * rows, filt) == _header(path)
    assert ply.layout(path) == (P_, 3 * rows, filt, len(_header(path)))
    assert os.path.getsize(path) == len(_header(path)) + 4 * P_ * (17 + 3 * rows + filt)
    want = S.gaussian_ply_fields(3 * rows) + (["filter_3D"] if filt else [])
    assert S.ply_properties(path) == want


def _rewrite(path, out, edit):
    data = open(path, "rb").read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    open(out, "wb").write(edit(data[:end]) + data[end:])
    return out


EDITS = {
    "comment": lambda h: h.replace(b"format binary_little_endian 1.0\n", b"format binary_little_endian 1.0\ncomment x\n"),
    "version": lambda h: h.replace(b"binary_little_endian 1.0", b"binary_little_endian 1.1"),
    "float32": lambda h: h.replace(b"property float x\n", b"property float32 x\n"),
    "order": lambda h: h.replace(b"property float y\nproperty float z\n", b"property float z\nproperty float y\n"),
    "renamed": lambda h: h.replace(b"property float opacity\n", b"property float alpha\n"),
    "extra_element": lambda h: h.replace(b"end_header\n", b"element face 0\nproperty list uchar int vertex_indices\n"
                                                          b"end_header\n"),
    "signed_count": lambda h: h.replace(b"element vertex 5\n", b"element vertex +5\n"),
}


@pytest.mark.parametrize("edit", sorted(EDITS))
def test_other_headers_take_the_numpy_reader(tmp_path, edit):
    path = _numpy_file(str(tmp_path / "a.ply"), 5, 3, False)
    other = _rewrite(path, str(tmp_path / "b.ply"), EDITS[edit])
    assert open(other, "rb").read() != open(path, "rb").read()
    assert ply.layout(other) is None


def test_other_layouts_take_the_numpy_reader(tmp_path):
    # a property list the numpy writer writes, but not save_gaussians_ply's: 6 f_rest values (not a square degree)
    rng = np.random.default_rng(2)
    cols = [rng.standard_normal(4).astype(np.float32) for _ in range(23)]
    names = S.gaussian_ply_fields(6)
    S._write_ply(str(tmp_path / "six.ply"), [(n, "f4") for n in names], cols)
    assert ply.layout(str(tmp_path / "six.ply")) is None
    # doubles instead of floats
    S._write_ply(str(tmp_path / "f8.ply"), [(n, "f8") for n in S.gaussian_ply_fields(0)],
                 [c.astype(np.float64) for c in cols[:17]])
    assert ply.layout(str(tmp_path / "f8.ply")) is None
    # points3D.ply
    S.write_points3d_ply(str(tmp_path / "p.ply"), np.zeros((3, 3), np.float32), np.zeros((3, 3), np.uint8))
    assert ply.layout(str(tmp_path / "p.ply")) is None
    # truncated records, and extra bytes after them (the numpy reader ignores those)
    path = _numpy_file(str(tmp_path / "a.ply"), 5, 1, True)
    data = open(path, "rb").read()
    open(str(tmp_path / "short.ply"), "wb").write(data[:-4])
    assert ply.layout(str(tmp_path / "short.ply")) is None
    open(str(tmp_path / "long.ply"), "wb").write(data + b"\0" * 8)
    assert ply.layout(str(tmp_path / "long.ply")) == ply.layout(path)
    # no header end
    open(str(tmp_path / "none.ply"), "wb").write(b"ply\n" + b"x" * 10000)
    assert ply.layout(str(tmp_path / "none.ply")) is None


def test_load_refuses_a_host_device(tmp_path):
    path = _numpy_file(str(tmp_path / "a.ply"), 5, 3, False)
    with pytest.raises(ValueError, match="needs a CUDA device"):
        ply.load(path, "cpu")


# ---- the command lines ---------------------------------------------------------------------------------------
def test_train_namespace_and_cfg_args_are_unchanged():
    base = ["-s", "S", "-m", "M", "--n_views", "3", "--iterations", "500", "--pp_optimizer", "--optim_pose"]
    a = T.parse_args(base)
    assert "ply_io" not in vars(a) and ply.io(a) is None and ply.kwargs(a) == {}
    for v in ("numpy", "gpu"):
        b = T.parse_args(base + ["--ply_io", v])
        assert ply.io(b) == v and ply.kwargs(b) == {"ply_io": v}
        assert vars(a) == {k: x for k, x in vars(b).items() if k != "ply_io"}
        assert T.cfg_args_text(a).encode() == T.cfg_args_text(b).encode() and "ply" not in T.cfg_args_text(b)
    with pytest.raises(SystemExit):
        T.parse_args(base + ["--ply_io", "pil"])


@pytest.mark.parametrize("argv", [["-s", "S", "-m", "M", "--n_views", "3"],
                                  ["-s", "S", "-m", "M", "--n_views", "3", "--eval"]])
def test_render_views_and_freeview_namespaces(argv):
    a = R.parser().parse_args(argv)
    b = R.parser().parse_args(argv + ["--ply_io", "gpu"])
    assert "ply_io" not in vars(a) and b.ply_io == "gpu"
    assert vars(a) == {k: v for k, v in vars(b).items() if k != "ply_io"}


def test_the_flag_reaches_the_loaders(tmp_path, monkeypatch):
    """render_views hands --ply_io to tracker_for and forwards it to the fly-through; freeview hands it to load;
    without the flag every call is what it was."""
    model = tmp_path / "model"
    _numpy_file(str(model / "point_cloud" / "iteration_7" / "point_cloud.ply"), 5, 3, False)
    seen = []

    def tracker_for(*a, **k):
        seen.append(k)
        raise RuntimeError("stop")
    monkeypatch.setattr(R, "tracker_for", tracker_for)
    monkeypatch.setattr(R, "load_views", lambda *a, **k: None)
    (model / "pose" / "ours_7").mkdir(parents=True)
    np.save(str(model / "pose" / "ours_7" / "pose_optimized.npy"), np.zeros((3, 4, 4)))
    argv = ["-s", "nowhere", "-m", str(model), "--n_views", "3", "--iterations", "7"]
    for extra, want in (([], {"kernel_size": None}), (["--ply_io", "gpu"], {"kernel_size": None, "ply_io": "gpu"}),
                        (["--ply_io", "numpy"], {"kernel_size": None, "ply_io": "numpy"})):
        for stage in ([], ["--eval"]):
            with pytest.raises(RuntimeError, match="stop"):
                R.main(argv + stage + extra)
            assert seen[-1] == want
    argvs = []
    monkeypatch.setattr(F, "main", lambda argv: argvs.append(argv) or 0)
    R.main(["-s", "S", "-m", "M", "--n_views", "3", "--infer_video"])
    assert "--ply_io" not in argvs[-1]
    R.main(["-s", "S", "-m", "M", "--n_views", "3", "--infer_video", "--ply_io", "gpu"])
    assert argvs[-1][-2:] == ["--ply_io", "gpu"]


def test_freeview_hands_the_flag_to_load(tmp_path, monkeypatch):
    seen = []
    monkeypatch.setattr(F, "load", lambda *a, **k: seen.append((a, k)) or (None, np.zeros((2, 4, 4)), 7))
    monkeypatch.setattr(F, "fly_through", lambda *a: (0, "x"))
    argv = ["-s", "S", "-m", "M", "--n_views", "2"]
    assert F.main(argv) == 0 and seen[-1][1] == {}
    assert F.main(argv + ["--ply_io", "gpu"]) == 0 and seen[-1][1] == {"ply_io": "gpu"}


def test_stage_argv_with_and_without_the_flag():
    src, model = "/data/Tanks/Horse/24_views", "out/Tanks/Horse/3_views"
    for mode in ("eval", "infer"):
        t = P.Task(mode, "Tanks", "Horse", 3, 1000, src, model)
        plain = P.stage_argv(t)
        assert P.stage_argv(t, ply_io=None) == plain
        assert all("--ply_io" not in v for v in plain.values())
        got = P.stage_argv(t, ply_io="gpu")
        assert got["train"] == plain["train"] + ["--ply_io", "gpu"]
        assert {k: v for k, v in got.items() if k != "train"} == {k: v for k, v in plain.items() if k != "train"}
        assert P.stage_argv(t, kernel_size=0.1, ply_io="gpu")["train"] == plain["train"] + ["--kernel_size", "0.1",
                                                                                            "--ply_io", "gpu"]
        args = P.stage_args(t, ply_io="gpu")
        assert ply.io(args["train"]) == "gpu"
        assert all("ply_io" not in vars(v) for k, v in args.items() if k != "train")
        assert all("ply_io" not in vars(v) for v in P.stage_args(t).values())


@pytest.mark.parametrize("mode", ["eval", "infer"])
def test_pipeline_namespace(mode):
    argv = [mode, "--data_root", "R", "--output_dir", "O", "--datasets", "D", "--scenes", "S", "--n_views", "3",
            "--iterations", "10"]
    a, b = P.parser().parse_args(argv), P.parser().parse_args(argv + ["--ply_io", "gpu"])
    assert "ply_io" not in vars(a) and ply.io(b) == "gpu"
    assert vars(a) == {k: v for k, v in vars(b).items() if k != "ply_io"}


def test_pipeline_hands_the_flag_to_run_tasks(monkeypatch, tmp_path):
    seen = []
    monkeypatch.setattr(P, "refusals", lambda *a, **k: [])
    monkeypatch.setattr(P, "run_tasks", lambda *a, **k: seen.append(k) or (0, []))
    argv = ["infer", "--data_root", "R", "--output_dir", str(tmp_path), "--datasets", "D", "--scenes", "S",
            "--n_views", "3", "--iterations", "10"]
    assert P.main(argv) == 0 and seen[-1]["ply_io"] is None
    assert P.main(argv + ["--ply_io", "gpu"]) == 0 and seen[-1]["ply_io"] == "gpu"
