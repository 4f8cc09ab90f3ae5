"""The GPU PNG encoder (-m gpu, DESIGN.md section 4.19): every file's inflated IDAT equals the numpy restatement of
Pillow's filters and its pixels equal the input, on edge shapes, segment boundaries, the photo crops of
tests/golden/png.npz and PoseTracker renders; chunk CRCs and Image.verify(); the same bytes alone, at every position
of a batch and on a second call; sizes against gsb_png_bound and Pillow; and --png_encoder gpu through freeview,
render_views and the pipeline."""
import contextlib
import io
import json
import os
import shutil
import zlib

import numpy as np
import pytest
import torch
from PIL import Image

from instantsplat_b200 import freeview as F
from instantsplat_b200 import metrics as M
from instantsplat_b200 import pipeline as P
from instantsplat_b200 import png
from instantsplat_b200 import render_views as R
from instantsplat_b200 import train as T
from instantsplat_b200.scenes import surface_scene

import _png

pytestmark = pytest.mark.gpu
DEV = "cuda"
HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = np.load(os.path.join(HERE, "golden", "png.npz"))
SEG = 32768


def _pil_bytes(img):
    buf = io.BytesIO()
    Image.fromarray(img).save(buf, "PNG")
    return len(buf.getvalue())


def _check_file(data: bytes, img: np.ndarray) -> None:
    """CRCs, IHDR, the inflated scanlines (Pillow's filters), the decoded pixels and Image.verify()."""
    H, W, _ = img.shape
    ch = _png.chunks(data)
    assert ch[0] == (b"IHDR", png.ihdr(H, W)) and ch[-1] == (b"IEND", b"")
    assert all(k == b"IDAT" for k, _ in ch[1:-1]) and len(ch) >= 3
    stream = _png.idat(data)
    assert len(stream) <= png.bound(H, W)
    assert zlib.decompress(stream) == _png.filter_rows(img)[0]
    Image.open(io.BytesIO(data)).verify()
    im = Image.open(io.BytesIO(data))
    im.load()
    assert im.mode == "RGB" and np.array_equal(np.asarray(im), img)


def _encode_one(img: np.ndarray) -> bytes:
    return png.encode(torch.from_numpy(np.ascontiguousarray(img))[None].to(DEV))[0]


def _shape_with(N: int):
    """(H, W) with H (3W + 1) == N."""
    for d in range(4, N + 1, 3):
        if N % d == 0:
            return N // d, (d - 1) // 3
    raise ValueError(N)


def _edge_images():
    rng = np.random.default_rng(3)
    out = {"1x1": rng.integers(0, 256, (1, 1, 3), dtype=np.uint8),
           "1xN": rng.integers(0, 256, (1, 1000, 3), dtype=np.uint8),
           "Nx1": rng.integers(0, 256, (700, 1, 3), dtype=np.uint8),
           "odd": rng.integers(0, 256, (31, 6, 3), dtype=np.uint8),
           "zero": np.zeros((9, 13, 3), np.uint8),
           "colour": np.full((40, 33, 3), (200, 30, 7), np.uint8),
           "noise": rng.integers(0, 256, (37, 53, 3), dtype=np.uint8),
           "levels": (rng.integers(0, 4, (64, 96, 3)) * 60).astype(np.uint8)}
    from test_png_cpu import _ties
    out["ties"] = _ties()
    for tag, N in (("seg", SEG), ("seg+1", SEG + 1), ("seg-1", SEG - 1), ("2seg+4", 2 * SEG + 4)):
        H, W = _shape_with(N)
        y, x = np.mgrid[0:H, 0:W]
        out[tag] = ((np.stack([x * 7 + y, x ^ y, y * 3], -1) + rng.integers(0, 3, (H, W, 3))) % 256).astype(np.uint8)
    return out


@pytest.mark.parametrize("name", list(_edge_images()))
def test_edge_shapes_are_exact(name):
    img = _edge_images()[name]
    _check_file(_encode_one(img), img)


@pytest.mark.parametrize("name", ["santorini", "art"])
def test_crops_are_exact_and_small(name):
    img = GOLDEN[f"{name}_crop"]
    data = _encode_one(img)
    _check_file(data, img)
    types = np.frombuffer(zlib.decompress(_png.idat(data)), np.uint8)[::3 * img.shape[1] + 1]
    assert np.array_equal(types, GOLDEN[f"{name}_filters"])
    ratio = len(data) / int(GOLDEN[f"{name}_pil_bytes"])
    print(f"{name} crop: {len(data)} bytes, {ratio:.3f} x Pillow's")
    assert ratio <= 1.20


def _renders(H, W, white=False, n=3):
    sc = surface_scene(20000, n, W, H, seed=41 + H, sh_degree=3)
    tk = F.tracker_from_gaussians(sc.params, W, H, sc.fovx, sc.fovy, white, DEV)
    return np.concatenate([c for _, c in F.frames_u8(tk, sc.poses)])


@pytest.mark.parametrize("H,W,white", [(512, 512, False), (512, 512, True), (1080, 1920, False)])
def test_renders_are_exact_and_small(H, W, white):
    frames = _renders(H, W, white)
    files = png.encode(torch.from_numpy(frames).to(DEV))
    for f, img in zip(files, frames):
        _check_file(f, img)
    ours, pil = sum(map(len, files)), sum(_pil_bytes(img) for img in frames)
    print(f"renders {H}x{W} white={white}: {ours} bytes, {ours / pil:.3f} x Pillow's")
    assert ours <= 1.20 * pil


def test_bytes_do_not_depend_on_the_batch():
    rng = np.random.default_rng(8)
    frames = _renders(512, 512, n=16)
    frames[5] = rng.integers(0, 256, frames[5].shape, dtype=np.uint8)
    frames[9] = 0
    alone = [_encode_one(f) for f in frames]
    assert png.encode(torch.from_numpy(frames).to(DEV)) == alone
    assert png.encode(torch.from_numpy(frames).to(DEV)) == alone              # a second call
    for k in range(0, 16, 3):
        assert png.encode(torch.from_numpy(frames[k:k + 3]).to(DEV)) == alone[k:k + 3]
        trio = np.stack([frames[(k + 7) % 16], frames[k], frames[(k + 1) % 16]])
        assert png.encode(torch.from_numpy(trio).to(DEV))[1] == alone[k]
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        assert png.encode(torch.from_numpy(frames[:3]).to(DEV)) == alone[:3]


@pytest.mark.parametrize("H,W", [(512, 512), (1080, 1920)])
def test_noise_stays_near_its_filtered_size(H, W):
    img = np.random.default_rng(H).integers(0, 256, (H, W, 3), dtype=np.uint8)
    data = _encode_one(img)
    _check_file(data, img)
    stream = _png.idat(data)
    assert len(stream) <= png.bound(H, W) and len(stream) <= 1.002 * H * (3 * W + 1) + 64


@pytest.mark.parametrize("colour", [(0, 0, 0), (200, 30, 7), (255, 255, 255)])
def test_flat_1080p_frames_are_small(colour):
    img = np.empty((1080, 1920, 3), np.uint8)
    img[:] = colour
    data = _encode_one(img)
    _check_file(data, img)
    print(f"flat {colour}: {len(data)} bytes (Pillow {_pil_bytes(img)})")
    assert len(data) <= 64 * 1024


def test_repeated_encode_leaves_device_memory_unchanged():
    x = torch.from_numpy(_edge_images()["seg+1"]).to(DEV)[None].repeat(4, 1, 1, 1)
    png.encode(x)
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    for _ in range(3):
        png.encode(x)
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated() == before


def test_write_pngs_names_and_files(tmp_path):
    frames = _renders(64, 96, n=5)
    chunks = [(0, frames[:2]), (2, frames[2:])]
    assert png.write_pngs(chunks, str(tmp_path / "a"), workers=2) == 5
    assert sorted(os.listdir(tmp_path / "a")) == [f"{i:05d}.png" for i in range(5)]
    names = [f"v{i}.png" for i in range(5)]
    assert png.write_pngs(chunks, str(tmp_path / "b"), workers=1, names=names) == 5
    for i in range(5):
        data = open(tmp_path / "b" / names[i], "rb").read()
        assert data == open(tmp_path / "a" / f"{i:05d}.png", "rb").read()
        _check_file(data, frames[i])
    w = P.PngWriter(2, "gpu")
    assert w.write(chunks, str(tmp_path / "c")) == 5
    w.close()
    for i in range(5):
        assert open(tmp_path / "c" / f"{i:05d}.png", "rb").read() == open(tmp_path / "a" / f"{i:05d}.png", "rb").read()


# ---- the stages ------------------------------------------------------------------------------------------------
def _read_dir(folder):
    return {n: np.asarray(Image.open(os.path.join(folder, n))) for n in sorted(os.listdir(folder))}


def test_freeview_cli_gpu_decodes_to_the_pil_pixels(tmp_path):
    from test_freeview_gpu import _model_dir
    src, model, it = _model_dir(tmp_path, 3)
    argv = ["-s", str(src), "-m", str(model), "--n_views", "3", "--iterations", "-1", "--max_batch", "16"]
    folder = model / "interp" / f"ours_{it}" / "renders"
    assert F.main(argv + ["--png_encoder", "gpu"]) == 0
    gpu = _read_dir(folder)
    raw = {n: open(folder / n, "rb").read() for n in gpu}
    shutil.rmtree(folder)
    assert F.main(argv) == 0
    pil = _read_dir(folder)
    assert list(gpu) == list(pil) and len(gpu) == 2 * 100 + 1
    for n in gpu:
        assert np.array_equal(gpu[n], pil[n]), n
        _check_file(raw[n], pil[n])


def test_render_views_metrics_equal_for_both_encoders(tmp_path):
    from test_render_views_gpu import N_TRAIN, _source_and_model
    src, model, it = _source_and_model(str(tmp_path / "gen"))
    results = {}
    for enc in ("pil", "gpu"):
        m = str(tmp_path / enc)
        shutil.copytree(model, m)
        base = ["-s", src, "-m", m, "--n_views", str(N_TRAIN), "--iterations", str(it), "-r", "1", "--png_encoder", enc]
        with contextlib.redirect_stdout(io.StringIO()):
            assert R.main(base) == 0
            assert R.main(base + ["--eval", "--optim_test_pose_iter", "20"]) == 0
            assert M.main(["-s", src, "-m", m, "--n_views", str(N_TRAIN)]) == 0
        results[enc] = (json.load(open(os.path.join(m, "results.json"))),
                        json.load(open(os.path.join(m, "per_view.json"))))
        if enc == "gpu":
            for sub in ("train", "test"):
                for kind in ("renders", "gt"):
                    folder = os.path.join(m, sub, f"ours_{it}", kind)
                    want = _read_dir(os.path.join(str(tmp_path / "pil"), sub, f"ours_{it}", kind))
                    got = _read_dir(folder)
                    assert list(got) == list(want)
                    for n in got:
                        assert np.array_equal(got[n], want[n]), (sub, kind, n)
    assert results["pil"] == results["gpu"]


def _run_clis_gpu(ts):
    """The stage CLIs on the scripts' lines, the render stages with --png_encoder gpu."""
    clis = {"train": T.main, "render_train": R.main, "render_test": R.main, "metrics": M.main, "render": R.main}
    for t in ts:
        os.makedirs(t.model, exist_ok=True)
        for key, argv in P.stage_argv(t).items():
            extra = ["--png_encoder", "gpu"] if key.startswith("render") else []
            with open(os.path.join(t.model, P.STAGES[t.mode][key][0]), "w") as f, \
                    contextlib.redirect_stdout(f), contextlib.redirect_stderr(f):
                clis[key](argv + extra)


@pytest.mark.parametrize("mode", ["eval", "infer"])
def test_pipeline_gpu_equals_the_stage_clis_gpu(tmp_path, mode):
    from test_pipeline_gpu import _compare_trees, _data_root
    from test_render_views_gpu import _source_and_model
    src, _, _ = _source_and_model(str(tmp_path / "gen"))
    root = _data_root(str(tmp_path / "data"), src, mode)
    out = str(tmp_path / "out")
    ts = P.tasks(mode, root, out, ["D"], ["A"], [3], [20])
    _run_clis_gpu(ts)
    os.rename(out, str(tmp_path / "cli"))
    argv = [mode, "--data_root", root, "--output_dir", out, "--datasets", "D", "--scenes", "A", "--n_views", "3",
            "--iterations", "20", "--workers", "2", "--png_encoder", "gpu"]
    with contextlib.redirect_stdout(io.StringIO()):
        assert P.main(argv) == 0
    files = _compare_trees(out, str(tmp_path / "cli"))
    pngs = [f for f in files if f.endswith(".png")]
    assert pngs
    for f in pngs:
        data = open(os.path.join(out, f), "rb").read()
        _check_file(data, np.asarray(Image.open(io.BytesIO(data))))
