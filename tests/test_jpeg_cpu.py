"""CPU checks of the GPU JPEG decoder (instantsplat_b200/jpeg.py, csrc/gs_jpeg.cuh; DESIGN.md 4.24): the marker
parser against Pillow on a seeded corpus Pillow writes, the route of every kind of file, a sequential restatement
(tests/_jpeg.py) and the kernels' shared arithmetic built for the host (tests/host_jpeg.cpp) against Pillow byte for
byte, the subsequence synchronisation run serially against the sequential decode, the streams that must be flagged,
and --jpeg_decoder on every command line."""
import ctypes
import io
import os
import re

import numpy as np
import pytest

from instantsplat_b200 import _lib, jpeg as J, pipeline as P, render_views as R, train as TR
from instantsplat_b200 import freeview as F, metrics as M

import _jpeg as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SMALL = [(1, 1), (2, 2), (3, 5), (15, 16), (16, 17), (17, 33), (67, 45)]
QUALITIES = (1, 10, 50, 75, 95, 100)


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    return T.host_lib(str(tmp_path_factory.mktemp("hj")))


def _corpus():
    """(name, file) written by Pillow's encoder: every quality and subsampling, optimize, qtables, restart rows and
    blocks."""
    out = []
    for q in QUALITIES:
        for ss in (0, 1, 2):
            out.append((f"q{q}_ss{ss}", T.pil_jpeg(T.image(37, 61, q + ss), quality=q, subsampling=ss)))
    arr = T.image(40, 72, 5)
    out.append(("optimize", T.pil_jpeg(arr, quality=85, optimize=True)))
    out.append(("qtables", T.pil_jpeg(arr, qtables=[list(range(1, 65)), [7] * 64], subsampling=1)))
    out.append(("qtables16", T.pil_jpeg(arr, qtables=[[300] * 64, [2] * 64])))
    out.append(("rst_rows", T.pil_jpeg(arr, quality=90, restart_marker_rows=1)))
    out.append(("rst_blocks", T.pil_jpeg(arr, quality=60, subsampling=0, restart_marker_blocks=3)))
    return out


@pytest.mark.parametrize("name,data", _corpus())
def test_parser_agrees_with_pillow(name, data):
    from PIL import Image, JpegImagePlugin
    p = J.parse(data)
    with Image.open(io.BytesIO(data)) as im:
        assert (p.width, p.height) == im.size and im.mode == "RGB"
        assert {(1, 1): 0, (2, 1): 1, (2, 2): 2}[(p.h, p.v)] == JpegImagePlugin.get_sampling(im)
        for c in range(3):
            assert list(p.quant[c]) == list(im.quantization[p.qt_ids[c]])
    assert J.route(data) == "gpu"


def test_routes_of_files_outside_the_subset():
    from PIL import Image
    arr = T.image(24, 40, 2)
    buf = io.BytesIO()
    Image.fromarray(arr).convert("CMYK").save(buf, "JPEG")
    png = io.BytesIO()
    Image.fromarray(arr).save(png, "PNG")
    good = T.pil_jpeg(arr, quality=80)
    for data in (T.pil_jpeg(arr, progressive=True), T.pil_jpeg(arr[..., 0]), buf.getvalue(), png.getvalue(),
                 good[:len(good) // 2], good[:200], b"garbage" * 100, b"", good.replace(b"JFIF", b"XXXX")[:-2]):
        assert J.route(data) == "pil"
    # no JFIF: the component ids decide (R, G, B ids are RGB), and an Adobe transform 0 is RGB
    blocks = T.random_blocks(16, 16, 1, 1, 0)
    q = np.full((3, 64), 3, np.uint16)
    plain = T.encode(blocks, 16, 16, 1, 1, q, jfif=False)
    assert J.route(plain) == "gpu"
    frame_ids = bytes([3, 1, 0x11, 0, 2, 0x11, 1, 3, 0x11, 2])
    rgb_ids = plain.replace(frame_ids, bytes([3, 82, 0x11, 0, 71, 0x11, 1, 66, 0x11, 2]))
    assert rgb_ids != plain and J.route(rgb_ids) == "pil"
    app14 = b"\xff\xee\x00\x0eAdobe\x00\x64\x00\x00\x00\x00"
    adobe = lambda transform: plain[:2] + app14 + bytes([transform]) + plain[2:]
    assert J.route(adobe(0)) == "pil" and J.route(adobe(1)) == "gpu"


def test_derived_tables_refuse_what_libjpeg_refuses():
    with pytest.raises(J.Unsupported):
        J.Derived((3,) + (0,) * 15, bytes([0, 1, 2]), False)        # three 1-bit codes
    with pytest.raises(J.Unsupported):
        J.Derived((0, 1) + (0,) * 14, bytes([16]), True)             # a DC symbol above 15
    d = J.Derived(T.AC_BITS, T.AC_VALS, False)
    assert d.maxcode[8] == len(T.AC_VALS) - 1 and d.maxcode[9] == -1 and d.look[0] == (8 << 8) | 0


@pytest.mark.parametrize("ss", [0, 1, 2])
@pytest.mark.parametrize("restart", [{}, {"restart_marker_blocks": 1}, {"restart_marker_rows": 1}])
def test_restatement_and_host_build_equal_pillow(host, ss, restart):
    for h, w in SMALL:
        data = T.pil_jpeg(T.image(h, w, h * w + ss), quality=80, subsampling=ss, **restart)
        ref = T.pil_decode(data)
        assert np.array_equal(T.py_decode(data), ref), (h, w)
        got, st = T.host_decode(host, data)
        assert st == 0 and np.array_equal(got, ref), (h, w)


@pytest.mark.parametrize("q", QUALITIES)
def test_host_build_equals_pillow_at_every_quality(host, q):
    for ss in (0, 1, 2):
        data = T.pil_jpeg(T.image(83, 130, q), quality=q, subsampling=ss)
        got, st = T.host_decode(host, data)
        assert st == 0 and np.array_equal(got, T.pil_decode(data)), ss


def test_encoder_writes_440_that_pillow_and_the_decoders_agree_on(host):
    for name, data, flagged in T.flagged_corpus():
        if flagged:
            continue
        ref = T.pil_decode(data)
        assert np.array_equal(T.py_decode(data), ref), name
        got, st = T.host_decode(host, data)
        assert st == 0 and np.array_equal(got, ref), name


def test_flagged_streams_are_flagged(host):
    for name, data, flagged in T.flagged_corpus():
        if not flagged:
            continue
        assert J.route(data) == "gpu", name                  # the headers are fine: only the stream is not
        _, st = T.host_decode(host, data)
        assert st != 0, name
        for S in (J.MIN_SUBSEQ_BITS, 64, J.SUBSEQ_BITS):
            _, st_sync, _ = T.host_coefs(host, data, S)
            assert st_sync != 0 or name == "coef_range", (name, S)


@pytest.mark.parametrize("S", [32, 40, 64, 256, 1024, 8192])
def test_sync_decoder_equals_the_sequential_decode(host, S):
    rounds = []
    for ss, kw in [(2, {}), (0, {}), (1, {"restart_marker_rows": 1}), (2, {"restart_marker_blocks": 5})]:
        data = T.pil_jpeg(T.image(160, 232, S + ss), quality=90, subsampling=ss, **kw)
        seq, st, _ = T.host_coefs(host, data)
        got, st_sync, r = T.host_coefs(host, data, S)
        assert st == 0 and st_sync == 0
        assert np.array_equal(got, seq)
        rounds.append(r)
    if S <= 64:
        assert max(rounds) >= 1                 # the guessed states did not all hold: synchronisation was exercised


def test_exports_and_signatures_match_the_header():
    hdr = open(os.path.join(ROOT, "include", "gsb200.h")).read()
    for name in ("gsb_jpeg_scratch_bytes", "gsb_jpeg_decode_batch"):
        assert name in _lib.EXPORTS
        m = re.search(r"GSB_API [^;(]*?\b" + name + r"\(([^)]*)\)", hdr)
        assert m, name
    assert len(re.search(r"gsb_jpeg_decode_batch\(([^)]*)\)", hdr).group(1).split(",")) == 9
    assert len(re.search(r"gsb_jpeg_scratch_bytes\(([^)]*)\)", hdr).group(1).split(",")) == 3
    assert ctypes.sizeof(_lib.GsbJpegHuff) == 1424 and ctypes.sizeof(_lib.GsbJpegFile) == 8976
    assert int(re.search(r"#define GSB_JPEG_LOOKAHEAD (\d+)", hdr).group(1)) == _lib.JPEG_LOOKAHEAD


def test_decode_refuses_a_host_device(tmp_path):
    with pytest.raises(ValueError, match="CUDA device only"):
        J.decode_u8([], "cpu")
    from instantsplat_b200.scene_io import load_views
    with pytest.raises(ValueError, match="CUDA device only"):
        load_views(str(tmp_path), 3, decode_device="cpu")


# ---- the command lines ---------------------------------------------------------------------------------------
def test_train_namespace_and_cfg_args_are_unchanged():
    base = ["-s", "S", "-m", "M", "--n_views", "3", "--iterations", "500", "--pp_optimizer", "--optim_pose"]
    a = TR.parse_args(base)
    assert "jpeg_decoder" not in vars(a) and J.decoder(a) is None and not J.requested(a)
    for v in ("pil", "gpu"):
        b = TR.parse_args(base + ["--jpeg_decoder", v])
        assert J.decoder(b) == v and J.requested(b) == (v == "gpu")
        assert vars(a) == {k: x for k, x in vars(b).items() if k != "jpeg_decoder"}
        assert TR.cfg_args_text(a).encode() == TR.cfg_args_text(b).encode() and "jpeg" not in TR.cfg_args_text(b)
    with pytest.raises(SystemExit):
        TR.parse_args(base + ["--jpeg_decoder", "turbo"])


@pytest.mark.parametrize("argv", [["-s", "S", "-m", "M", "--n_views", "3"],
                                  ["-s", "S", "-m", "M", "--n_views", "3", "--eval"]])
def test_render_views_namespace(argv):
    a = R.parser().parse_args(argv)
    b = R.parser().parse_args(argv + ["--jpeg_decoder", "gpu"])
    assert "jpeg_decoder" not in vars(a) and b.jpeg_decoder == "gpu"
    assert vars(a) == {k: v for k, v in vars(b).items() if k != "jpeg_decoder"}


def test_freeview_and_metrics_do_not_take_the_flag():
    with pytest.raises(SystemExit):
        F.main(["-s", "S", "-m", "M", "--n_views", "2", "--jpeg_decoder", "gpu"])
    with pytest.raises(SystemExit):
        M.parser().parse_args(["-s", "S", "-m", "M", "--n_views", "2", "--jpeg_decoder", "gpu"])


def test_render_views_hands_the_flag_to_load_views(tmp_path, monkeypatch):
    seen = []

    def load_views(*a, **k):
        seen.append(k)
        raise RuntimeError("stop")
    monkeypatch.setattr(R, "load_views", load_views)
    model = tmp_path / "model"
    (model / "point_cloud" / "iteration_7").mkdir(parents=True)
    (model / "point_cloud" / "iteration_7" / "point_cloud.ply").write_bytes(b"")
    (model / "pose" / "ours_7").mkdir(parents=True)
    np.save(str(model / "pose" / "ours_7" / "pose_optimized.npy"), np.zeros((3, 4, 4)))
    argv = ["-s", "nowhere", "-m", str(model), "--n_views", "3", "--iterations", "7"]
    for extra, want in (([], None), (["--jpeg_decoder", "pil"], None), (["--jpeg_decoder", "gpu"], "cuda")):
        for stage in ([], ["--eval"]):
            with pytest.raises(RuntimeError, match="stop"):
                R.main(argv + stage + extra)
            assert seen[-1] == {"resample_device": None, "decode_device": want}


def test_stage_argv_with_and_without_the_flag():
    src, model = "/data/Tanks/Horse/24_views", "out/Tanks/Horse/3_views"
    for mode in ("eval", "infer"):
        t = P.Task(mode, "Tanks", "Horse", 3, 1000, src, model)
        plain = P.stage_argv(t)
        assert P.stage_argv(t, jpeg_decoder=None) == plain
        assert all("--jpeg_decoder" not in v for v in plain.values())
        got = P.stage_argv(t, jpeg_decoder="gpu")
        decoding = {"train", "render_test"}
        for k in plain:
            assert got[k] == plain[k] + (["--jpeg_decoder", "gpu"] if k in decoding else []), k
        args = P.stage_args(t, jpeg_decoder="gpu")
        assert J.requested(args["train"])
        assert all("jpeg_decoder" not in vars(v) for v in P.stage_args(t).values())


@pytest.mark.parametrize("mode", ["eval", "infer"])
def test_pipeline_namespace_and_hand_over(mode, monkeypatch, tmp_path):
    argv = [mode, "--data_root", "R", "--output_dir", str(tmp_path), "--datasets", "D", "--scenes", "S",
            "--n_views", "3", "--iterations", "10"]
    a, b = P.parser().parse_args(argv), P.parser().parse_args(argv + ["--jpeg_decoder", "gpu"])
    assert "jpeg_decoder" not in vars(a) and J.decoder(b) == "gpu"
    assert vars(a) == {k: v for k, v in vars(b).items() if k != "jpeg_decoder"}
    seen, refused = [], []
    monkeypatch.setattr(P, "refusals", lambda *a, **k: refused.append(a) or [])
    monkeypatch.setattr(P, "run_tasks", lambda *a, **k: seen.append(k) or (0, []))
    assert P.main(argv) == 0 and seen[-1]["jpeg_decoder"] is None and refused[-1][3] is None
    assert P.main(argv + ["--jpeg_decoder", "gpu"]) == 0 and seen[-1]["jpeg_decoder"] == "gpu"
    assert refused[-1][3] == "gpu"
