"""The GPU PNG encoder's host side without a GPU (DESIGN.md section 4.19): the numpy restatement of Pillow's scanline
filter against tests/golden/png.npz and against Pillow's own IDAT, the chunk framing, the Adler-32 combine of the pack
kernel, gsb_png_bound, the exports, and --png_encoder on the three command lines."""
import ctypes
import io
import os
import re
import zlib

import numpy as np
import pytest
from PIL import Image

import instantsplat_b200 as I
from instantsplat_b200 import freeview as F
from instantsplat_b200 import pipeline as P
from instantsplat_b200 import png
from instantsplat_b200 import render_views as R

import _png

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = np.load(os.path.join(HERE, "golden", "png.npz"))


def _pil_png(img: np.ndarray) -> bytes:
    buf = io.BytesIO()
    Image.fromarray(img).save(buf, "PNG")
    return buf.getvalue()


def _ties() -> np.ndarray:
    """Rows on which several filters cost the same: a constant row (None, Sub and Paeth tie under Up's zero row in
    row 0, Up and Paeth tie below), a ramp whose Sub and Up residuals are equal, and a row equal to the one above."""
    img = np.zeros((6, 9, 3), np.uint8)
    img[0] = 7
    img[1] = 7
    img[2] = np.arange(27).reshape(9, 3)
    img[3] = img[2] + 3
    img[4] = img[3]
    img[5] = 128
    return img


def _edge_images():
    rng = np.random.default_rng(11)
    return {
        "1x1": rng.integers(0, 256, (1, 1, 3), dtype=np.uint8),
        "1xN": rng.integers(0, 256, (1, 41, 3), dtype=np.uint8),
        "Nx1": rng.integers(0, 256, (33, 1, 3), dtype=np.uint8),
        "odd": rng.integers(0, 256, (7, 6, 3), dtype=np.uint8),         # 3W + 1 = 19
        "zero": np.zeros((9, 13, 3), np.uint8),
        "colour": np.full((12, 17, 3), (200, 30, 7), np.uint8),
        "noise": rng.integers(0, 256, (37, 53, 3), dtype=np.uint8),
        "ties": _ties(),
        "levels": (rng.integers(0, 4, (64, 96, 3)) * 60).astype(np.uint8),
    }


@pytest.mark.parametrize("name", ["santorini", "art"])
def test_filter_rule_reproduces_the_fixture(name):
    crop = GOLDEN[f"{name}_crop"]
    assert crop.shape == (384, 512, 3) and crop.dtype == np.uint8
    _, types = _png.filter_rows(crop)
    assert np.array_equal(types, GOLDEN[f"{name}_filters"])


@pytest.mark.parametrize("name", ["santorini", "art"] + list(_edge_images()))
def test_filter_rule_is_pillows_idat(name):
    img = GOLDEN[f"{name}_crop"] if name in ("santorini", "art") else _edge_images()[name]
    filtered, types = _png.filter_rows(img)
    assert zlib.decompress(_png.idat(_pil_png(img))) == filtered
    assert set(types.tolist()) <= {0, 1, 2, 4}


def test_ties_take_the_first_filter():
    _, types = _png.filter_rows(_ties())
    # row 0: None costs 7 x 27, Sub 7 x 3, Up 7 x 27, Paeth (= Sub against a zero row) 7 x 3 -> Sub, not Paeth
    # row 1: Up and Paeth are both all zero -> Up; row 4 equals row 3 -> Up
    assert types[0] == 1 and types[1] == 2 and types[4] == 2


@pytest.mark.parametrize("HW", [(1, 1), (5, 7), (384, 512)])
def test_framing_around_a_zlib_stream(HW):
    H, W = HW
    img = np.random.default_rng(H).integers(0, 256, (H, W, 3), dtype=np.uint8)
    filtered, _ = _png.filter_rows(img)
    data = png.png_file(H, W, zlib.compress(filtered))
    ch = _png.chunks(data)                                 # checks every CRC
    assert [k for k, _ in ch] == [b"IHDR", b"IDAT", b"IEND"]
    assert ch[0][1] == _png.chunks(_pil_png(img))[0][1]    # IHDR byte for byte
    assert zlib.decompress(_png.idat(data)) == filtered
    im = Image.open(io.BytesIO(data))
    im.verify()
    assert np.array_equal(np.asarray(Image.open(io.BytesIO(data))), img)


@pytest.mark.parametrize("N", [0, 1, 5, 32767, 32768, 32769, 3 * 32768 + 17, 6221880])
def test_adler_combine(N):
    data = np.random.default_rng(N).integers(0, 256, N, dtype=np.uint8).tobytes()
    assert _png.adler_combine(_png.adler_parts(data), N) == zlib.adler32(data)
    ones = b"\xff" * N                                     # the largest partial sums
    assert _png.adler_combine(_png.adler_parts(ones), N) == zlib.adler32(ones)


def test_bound_formula():
    L = I.lib()
    for H, W in [(1, 1), (5, 7), (8192, 1), (1, 10922), (99, 110), (512, 512), (1080, 1920), (2160, 3840)]:
        N = H * (3 * W + 1)
        nseg = -(-N // 32768)
        assert L.gsb_png_bound(H, W) == 2 + N + 10 * nseg + 2 + 4 == png.bound(H, W)
        # a stored segment is its bytes plus two 5-byte block heads; the stream adds 2 + 2 + 4
        assert L.gsb_png_scratch_bytes(3, H, W) == 3 * (-(-N // 16) * 16 + nseg * (32768 + 16 + 16))
    for H, W in [(0, 4), (4, 0), (-1, 4), (1 << 20, 1 << 20)]:
        assert L.gsb_png_bound(H, W) == 0
    assert L.gsb_png_scratch_bytes(0, 4, 4) == 0


def test_exports_and_signatures():
    L = I.lib()
    header = open(os.path.join(HERE, "..", "include", "gsb200.h")).read()
    declared = set(re.findall(r"GSB_API\s+[\w\s\*]+?\b(gsb_\w+)\s*\(", header))
    for name in ("gsb_png_bound", "gsb_png_scratch_bytes", "gsb_png_encode_batch"):
        assert name in declared and name in I._lib.EXPORTS and hasattr(L, name)
    assert L.gsb_png_bound.restype is ctypes.c_size_t and L.gsb_png_scratch_bytes.restype is ctypes.c_size_t
    assert L.gsb_png_encode_batch.restype is ctypes.c_int
    i32, vp = ctypes.c_int32, ctypes.c_void_p
    assert L.gsb_png_encode_batch.argtypes == [i32, i32, i32, vp, vp, ctypes.c_size_t, vp, vp, vp]
    # refused before anything is launched: bad sizes, NULL, misalignment, short scratch
    need = L.gsb_png_scratch_bytes(1, 4, 4)
    assert L.gsb_png_encode_batch(0, 4, 4, 16, 16, need, 16, 16, None) == -1
    assert L.gsb_png_encode_batch(1, 0, 4, 16, 16, need, 16, 16, None) == -1
    assert L.gsb_png_encode_batch(1, 4, 4, None, 16, need, 16, 16, None) == -1
    assert L.gsb_png_encode_batch(1, 4, 4, 16, 24, need, 16, 16, None) == -1        # scratch not 16-byte aligned
    assert L.gsb_png_encode_batch(1, 4, 4, 16, 16, need, 16, 20, None) == -1        # sizes not 8-byte aligned
    assert L.gsb_png_encode_batch(1, 4, 4, 16, 16, need - 1, 16, 16, None) == -1
    assert b"scratch" in L.gsb_last_error()


def test_encode_refuses_host_and_misshaped_frames():
    import torch
    with pytest.raises(ValueError):
        png.encode(torch.zeros(1, 4, 4, 3, dtype=torch.uint8))
    with pytest.raises(ValueError):
        png.encode(np.zeros((1, 4, 4, 3), np.uint8))


def test_flag_on_every_command_line():
    base = ["-s", "S", "-m", "M", "--n_views", "3"]
    assert R.parser().parse_args(base).png_encoder == "pil"
    assert R.parser().parse_args(base + ["--png_encoder", "gpu"]).png_encoder == "gpu"
    for mode in ("eval", "infer"):
        argv = [mode, "--data_root", "D", "--output_dir", "O", "--datasets", "d", "--scenes", "s", "--n_views", "3",
                "--iterations", "10"]
        assert P.parser().parse_args(argv).png_encoder == "pil"
        assert P.parser().parse_args(argv + ["--png_encoder", "gpu"]).png_encoder == "gpu"
    with pytest.raises(SystemExit):
        R.parser().parse_args(base + ["--png_encoder", "jpeg"])
    with pytest.raises(SystemExit):
        P.parser().parse_args(argv + ["--png_encoder", "jpeg"])
    assert F.png_writer("pil") is F.write_pngs and F.png_writer("gpu") is png.write_pngs
    with pytest.raises(ValueError):
        P.PngWriter(1, "jpeg")


def test_freeview_flag_reaches_fly_through(tmp_path, monkeypatch):
    seen = {}
    monkeypatch.setattr(F, "load", lambda *a: (None, np.zeros((3, 4, 4)), 7))
    monkeypatch.setattr(F, "fly_through", lambda *a: (seen.setdefault("write", a[7]), (0, "x"))[1])
    for enc, want in ((None, F.write_pngs), ("pil", F.write_pngs), ("gpu", png.write_pngs)):
        seen.clear()
        argv = ["-s", "S", "-m", "M", "--n_views", "3"] + ([] if enc is None else ["--png_encoder", enc])
        assert F.main(argv) == 0
        assert seen["write"] is want
    # render_views --infer_video hands the flag on to the fly-through
    argvs = []
    monkeypatch.setattr(F, "main", lambda argv: argvs.append(argv) or 0)
    R.main(["-s", "S", "-m", "M", "--n_views", "3", "--infer_video", "--png_encoder", "gpu"])
    assert argvs[-1][-2:] == ["--png_encoder", "gpu"]
