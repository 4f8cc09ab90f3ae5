"""The GPU JPEG decoder (gsb_jpeg_decode_batch, instantsplat_b200/jpeg.py, DESIGN.md 4.24) against Pillow, byte for
byte: the seeded corpus of tests/test_jpeg_cpu.py, the reference's asset shapes (1280x720 and 1920x1080 4:2:0), phone
sized 4032x3024 in 4:2:0 and 4:4:4 with and without restart markers, the smallest subsequence size, one mixed batch
and each file alone; the streams the kernels must flag; and no memory left behind."""
import os

import numpy as np
import pytest
import torch

from instantsplat_b200 import jpeg as J

import _jpeg as T

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


def _write(tmp_path, name: str, data: bytes) -> str:
    p = str(tmp_path / name)
    with open(p, "wb") as f:
        f.write(data)
    return p


def _corpus(tmp_path):
    out = []
    for (h, w) in [(1, 1), (2, 2), (3, 5), (15, 16), (16, 17), (17, 33), (67, 45), (240, 320)]:
        for ss in (0, 1, 2):
            for q, kw in [(1, {}), (10, {}), (50, {"optimize": True}), (75, {"restart_marker_blocks": 1}),
                          (95, {"restart_marker_rows": 1}), (100, {})]:
                arr = T.image(h, w, 7 * h + w + q + ss)
                data = T.pil_jpeg(arr, quality=q, subsampling=ss, **kw)
                out.append(_write(tmp_path, f"c_{h}x{w}_{ss}_{q}.jpg", data))
    return out


def _assert_pillow(paths, images, routes=None):
    for i, p in enumerate(paths):
        with open(p, "rb") as f:
            ref = T.pil_decode(f.read())
        got = images[i].cpu().numpy()
        assert got.shape == ref.shape and np.array_equal(got, ref), \
            f"{os.path.basename(p)}: {int((got != ref).sum()) if got.shape == ref.shape else got.shape} bytes differ"
        if routes is not None:
            assert routes[i] == "gpu", f"{os.path.basename(p)} went to Pillow"


@pytest.mark.parametrize("subseq_bits", [J.SUBSEQ_BITS, J.MIN_SUBSEQ_BITS])
def test_corpus_in_one_batch_equals_pillow(tmp_path, subseq_bits):
    paths = _corpus(tmp_path)
    images, routes = J.decode_u8(paths, DEV, subseq_bits=subseq_bits, return_routes=True)
    _assert_pillow(paths, images, routes)


def test_corpus_each_file_alone_equals_pillow(tmp_path):
    paths = _corpus(tmp_path)[::5]
    for p in paths:
        images, routes = J.decode_u8([p], DEV, return_routes=True)
        _assert_pillow([p], images, routes)


@pytest.mark.parametrize("w,h,ss,q,kw", [
    (1280, 720, 2, 75, {}), (1920, 1080, 2, 95, {}), (1920, 1080, 2, 75, {"restart_marker_rows": 2}),
    (4032, 3024, 2, 92, {}), (4032, 3024, 0, 92, {}), (4032, 3024, 2, 92, {"restart_marker_rows": 1}),
    (4032, 3024, 0, 75, {"restart_marker_blocks": 64})])
def test_large_images_equal_pillow(tmp_path, w, h, ss, q, kw):
    arr = T.image(h, w, w + h + q)
    p = _write(tmp_path, "big.jpg", T.pil_jpeg(arr, quality=q, subsampling=ss, **kw))
    images, routes = J.decode_u8([p], DEV, return_routes=True)
    _assert_pillow([p], images, routes)


def test_large_image_at_smallest_subsequence_size(tmp_path):
    arr = T.image(1080, 1920, 3)
    p = _write(tmp_path, "big.jpg", T.pil_jpeg(arr, quality=95, subsampling=2))
    images, routes = J.decode_u8([p], DEV, subseq_bits=J.MIN_SUBSEQ_BITS, return_routes=True)
    _assert_pillow([p], images, routes)


def test_mixed_sizes_in_one_batch_and_in_sub_batches(tmp_path):
    paths = []
    for i, (w, h, ss) in enumerate([(1280, 720, 2), (33, 17, 0), (1920, 1080, 2), (640, 480, 1), (7, 9, 2)]):
        paths.append(_write(tmp_path, f"m{i}.jpg", T.pil_jpeg(T.image(h, w, i), quality=85, subsampling=ss)))
    images, routes = J.decode_u8(paths, DEV, return_routes=True)
    _assert_pillow(paths, images, routes)
    images, routes = J.decode_u8(paths, DEV, budget=1, return_routes=True)     # one file per call
    _assert_pillow(paths, images, routes)


def test_same_size_batch_is_one_stack(tmp_path):
    paths = [_write(tmp_path, f"s{i}.jpg", T.pil_jpeg(T.image(72, 96, i), quality=90)) for i in range(4)]
    images = J.decode_u8(paths, DEV)
    st = J.stack(images)
    assert st.shape == (4, 72, 96, 3)
    _assert_pillow(paths, list(st))


def test_encoder_440_and_flagged_streams(tmp_path):
    cases = T.flagged_corpus()
    paths = [_write(tmp_path, f"f_{name}.jpg", data) for name, data, _ in cases]
    status = J.status_of(paths, DEV)
    for (name, data, flagged), st in zip(cases, status):
        assert st is not None, name
        assert (st != 0) == flagged, f"{name}: status {st}"
    for (name, data, flagged), p in zip(cases, paths):
        try:
            ref = T.pil_decode(data)
        except Exception as e:                          # Pillow's exception must come back as it is
            with pytest.raises(type(e)):
                J.decode_u8([p], DEV)
            continue
        images, routes = J.decode_u8([p], DEV, return_routes=True)
        assert routes[0] == ("pil" if flagged else "gpu"), name
        assert np.array_equal(images[0].cpu().numpy(), ref), name


def test_files_outside_the_subset_come_back_from_pillow(tmp_path):
    arr = T.image(40, 56, 1)
    datas = {"progressive": T.pil_jpeg(arr, progressive=True), "gray": T.pil_jpeg(arr[..., 0])}
    from PIL import Image
    import io
    buf = io.BytesIO()
    Image.fromarray(arr).convert("CMYK").save(buf, "JPEG")
    datas["cmyk"] = buf.getvalue()
    buf = io.BytesIO()
    Image.fromarray(arr).save(buf, "PNG")
    datas["png"] = buf.getvalue()
    paths = [_write(tmp_path, f"{k}.img", v) for k, v in datas.items()]
    images, routes = J.decode_u8(paths, DEV, return_routes=True)
    assert routes == ["pil"] * len(paths)
    for p, im in zip(paths, images):
        with Image.open(p) as ref:
            assert np.array_equal(im.cpu().numpy(), np.array(ref))


def test_no_memory_left_behind(tmp_path):
    paths = [_write(tmp_path, f"l{i}.jpg", T.pil_jpeg(T.image(300, 400, i), quality=90)) for i in range(3)]
    J.decode_u8(paths, DEV)
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    J.decode_u8(paths, DEV)
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated() == before


# ---- the loader and the stage command lines --------------------------------------------------------------------
N_TRAIN = 3


@pytest.fixture(scope="module")
def jpeg_source(tmp_path_factory):
    """test_render_views_gpu's source and model with the views' images re-encoded as JPEG (4:2:0, 4:4:4 and 4:2:2 in
    turn, one with restart markers) under .jpg names; one test view stays PNG, which Pillow decodes either way."""
    from PIL import Image
    from test_render_views_gpu import _source_and_model
    src, model, it = _source_and_model(str(tmp_path_factory.mktemp("jpeg")))
    folder = os.path.join(src, "images")
    keep_png = "t2.png"
    for k, name in enumerate(sorted(os.listdir(folder))):
        if name == keep_png:
            continue
        path = os.path.join(folder, name)
        with Image.open(path) as im:
            arr = np.array(im)
        os.remove(path)
        kw = {"restart_marker_rows": 1} if k == 1 else {}
        with open(path[:-4] + ".jpg", "wb") as f:
            f.write(T.pil_jpeg(arr, quality=90, subsampling=k % 3, **kw))
    for split in ("0", "1"):
        txt = os.path.join(src, f"sparse_{N_TRAIN}", split, "images.txt")
        lines = open(txt).read().replace(".png", ".jpg").replace(keep_png[:-4] + ".jpg", keep_png)
        open(txt, "w").write(lines)
    return src, model, it


def _same_views(a, b):
    assert a.names == b.names and a.camera_ids == b.camera_ids
    assert (a.width, a.height, a.source_width, a.source_height, a.fovx, a.fovy) == \
        (b.width, b.height, b.source_width, b.source_height, b.fovx, b.fovy)
    assert np.array_equal(a.w2c, b.w2c)
    assert a.images.dtype == b.images.dtype == np.uint8 and np.array_equal(a.images, b.images)


def test_load_views_with_and_without_the_decoder(jpeg_source):
    from instantsplat_b200 import scene_io as S
    src, _, _ = jpeg_source
    jpgs = sorted(os.path.join(src, "images", n) for n in os.listdir(os.path.join(src, "images")) if n.endswith(".jpg"))
    assert len(jpgs) == 6 and J.decode_u8(jpgs, DEV, return_routes=True)[1] == ["gpu"] * 6
    for split in (0, 1):
        plain = S.load_views(src, N_TRAIN, split, 1)
        _same_views(S.load_views(src, N_TRAIN, split, 1, decode_device=DEV), plain)
        plain = S.load_views(src, N_TRAIN, split, 2, resample_device=DEV)
        assert (plain.width, plain.height) == (48, 32)
        _same_views(S.load_views(src, N_TRAIN, split, 2, resample_device=DEV, decode_device=DEV), plain)


def _read(path):
    with open(path, "rb") as f:
        return f.read()


def test_train_writes_the_same_files(jpeg_source, tmp_path):
    from instantsplat_b200 import train as TR
    src, _, _ = jpeg_source
    models = {}
    m = str(tmp_path / "model")                 # one path for both runs: cfg_args records it
    for dec in ([], ["--jpeg_decoder", "gpu"]):
        TR.run(TR.parse_args(["-s", src, "-m", m, "-r", "1", "--n_views", str(N_TRAIN), "--iterations", "4",
                              "--quiet"] + dec))
        models[bool(dec)] = str(tmp_path / ("gpu" if dec else "pil"))
        os.rename(m, models[bool(dec)])
    for rel in (("point_cloud", "iteration_4", "point_cloud.ply"), ("pose", "ours_4", "pose_optimized.npy"),
                ("pose", "ours_4", "pose_org.npy"), ("cameras.json",), ("cfg_args",), ("input.ply",)):
        assert _read(os.path.join(models[True], *rel)) == _read(os.path.join(models[False], *rel)), rel


def test_render_views_writes_the_same_pngs(jpeg_source, tmp_path):
    import shutil
    from instantsplat_b200 import render_views as R
    src, model, it = jpeg_source
    trees = {}
    for dec in ([], ["--jpeg_decoder", "gpu"]):
        m = str(tmp_path / ("gpu" if dec else "pil"))
        shutil.copytree(model, m)
        base = ["-s", src, "-m", m, "--n_views", str(N_TRAIN), "--iterations", str(it), "--workers", "2"] + dec
        assert R.main(base) == 0
        assert R.main(base + ["--eval", "--optim_test_pose_iter", "5"]) == 0
        trees[bool(dec)] = m
    for stage in ("train", "test"):
        for kind in ("renders", "gt"):
            fa = os.path.join(trees[True], stage, f"ours_{it}", kind)
            fb = os.path.join(trees[False], stage, f"ours_{it}", kind)
            names = sorted(os.listdir(fb))
            assert names and sorted(os.listdir(fa)) == names
            for n in names:
                assert _read(os.path.join(fa, n)) == _read(os.path.join(fb, n)), (stage, kind, n)


def test_pipeline_eval_writes_the_same_files(jpeg_source, tmp_path):
    import shutil
    from instantsplat_b200 import pipeline as P
    from test_pipeline_gpu import _compare_trees
    src, _, _ = jpeg_source
    root = str(tmp_path / "data")
    shutil.copytree(src, os.path.join(root, "D", "A", "24_views"))
    outs = {}
    out = str(tmp_path / "out")                 # one path for both runs: the files record it
    for dec in ([], ["--jpeg_decoder", "gpu"]):
        argv = ["eval", "--data_root", root, "--output_dir", out, "--datasets", "D", "--scenes", "A", "--n_views",
                str(N_TRAIN), "--iterations", "10", "--workers", "2"] + dec
        assert P.main(argv) == 0
        outs[bool(dec)] = str(tmp_path / ("gpu" if dec else "pil"))
        os.rename(out, outs[bool(dec)])
    assert _compare_trees(outs[True], outs[False])
