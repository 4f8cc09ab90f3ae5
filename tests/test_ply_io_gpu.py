"""point_cloud.ply written and read on the GPU (-m gpu, instantsplat_b200/ply.py, DESIGN.md section 4.23): the GPU
writer's file is save_gaussians_ply's byte for byte at every SH degree, with and without filter_3D, at record counts
around the CTA size and across chunk boundaries, on NaN payloads, infinities, -0 and denormals; the GPU reader is
load_gaussians_ply bit for bit, including on files it hands to the numpy reader; the kernels at every 16-byte phase of
the record buffer, in device and pinned host memory; JointTrainer.save_ply(io="gpu"); the stage command lines with
--ply_io gpu against the same runs without it; and one round trip past 2^31 bytes."""
import contextlib
import filecmp
import os
import shutil

import numpy as np
import pytest
import torch

import instantsplat_b200 as I
from instantsplat_b200 import freeview as F
from instantsplat_b200 import pipeline as P
from instantsplat_b200 import ply
from instantsplat_b200 import render_views as R
from instantsplat_b200 import scene_io as S
from instantsplat_b200 import train as T
from instantsplat_b200.scenes import surface_scene
from instantsplat_b200.trainer import OptimConfig

pytestmark = pytest.mark.gpu
DEV = "cuda"
SPECIAL = np.array([0x7FC12345, 0xFFA00001, 0x7F800001, 0x7F800000, 0xFF800000, 0x80000000, 0x00000000, 0x00000001,
                    0x007FFFFF, 0x80400000, 0x7F7FFFFF], dtype=np.uint32).view(np.int32)


def _tensors(P_, deg, filt, seed=0, special=True):
    """save_gaussians_ply's inputs as CUDA tensors, with the special words scattered through every tensor."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    rows = (deg + 1) ** 2 - 1
    shapes = dict(xyz=(3,), f_dc=(1, 3), f_rest=(rows, 3), opacity=(1,), scaling=(3,), rotation=(4,))
    if filt:
        shapes["filter_3D"] = (1,)
    out = {}
    sp = torch.from_numpy(SPECIAL).to(DEV)
    for k, s in shapes.items():
        t = torch.randn(P_, *s, generator=g, device=DEV)
        if special and t.numel():
            w = t.view(-1).view(torch.int32)
            idx = torch.randint(0, t.numel(), (min(t.numel(), 64),), generator=g, device=DEV)
            w[idx] = sp[torch.arange(idx.numel(), device=DEV) % sp.numel()]
        out[k] = t
    return out


def _host(t):
    return {k: v.cpu().numpy() for k, v in t.items()}


def _numpy_write(path, t):
    h = _host(t)
    S.save_gaussians_ply(path, h["xyz"], h["f_dc"], h["f_rest"], h["opacity"], h["scaling"], h["rotation"],
                         h.get("filter_3D"))


def _bits_equal(got, want):
    """got (CUDA tensors) and want (load_gaussians_ply's arrays): the same keys, shapes and words."""
    assert sorted(got) == sorted(want)
    for k, v in want.items():
        g = got[k]
        assert g.is_cuda and g.dtype == torch.float32 and g.is_contiguous() and tuple(g.shape) == v.shape, k
        assert torch.equal(g.cpu().view(torch.int32), torch.from_numpy(np.ascontiguousarray(v)).view(torch.int32)), k


# ---- 1. byte-identical writes, bit-equal reads ----------------------------------------------------------------
@pytest.mark.parametrize("deg", [0, 1, 2, 3])
@pytest.mark.parametrize("filt", [False, True])
@pytest.mark.parametrize("P_", [0, 1, 127, 128, 129, 1000])
def test_write_and_read_equal_numpy(tmp_path, deg, filt, P_):
    t = _tensors(P_, deg, filt, seed=P_ + 10 * deg)
    a, b = str(tmp_path / "gpu.ply"), str(tmp_path / "numpy.ply")
    ply.save(a, t)
    _numpy_write(b, t)
    assert filecmp.cmp(a, b, shallow=False)
    want = S.load_gaussians_ply(b)
    _bits_equal(ply.load(a), want)
    # the written words are the tensors' own
    for k, v in t.items():
        assert torch.equal(v.cpu().view(torch.int32), torch.from_numpy(want[k]).view(torch.int32)), k


@pytest.mark.parametrize("per_chunk", [1, 7, 127, 128, 129, 999, 1000, 1001])
def test_chunk_boundaries_and_the_pinned_bound(tmp_path, monkeypatch, per_chunk):
    """chunk_bytes of per_chunk records (plus 4 bytes, not a whole record): the same file, the same values, and no
    pinned buffer above chunk_bytes."""
    t = _tensors(1000, 3, True, seed=per_chunk)
    rec = 4 * (17 + 45 + 1)
    sizes = []
    real = ply._pinned
    monkeypatch.setattr(ply, "_pinned", lambda n: sizes.append(n) or real(n))
    b = str(tmp_path / "numpy.ply")
    _numpy_write(b, t)
    want = S.load_gaussians_ply(b)
    for chunk in (per_chunk * rec, per_chunk * rec + 4):
        a = str(tmp_path / f"gpu{chunk}.ply")
        ply.save(a, t, chunk_bytes=chunk)
        assert filecmp.cmp(a, b, shallow=False)
        _bits_equal(ply.load(a, chunk_bytes=chunk), want)
        assert len(sizes) == 2 and all(n <= chunk for n in sizes) and sizes[0] == min(per_chunk, 1000) * rec
        sizes.clear()
    with pytest.raises(ValueError, match="smaller than one 252-byte record"):
        ply.save(str(tmp_path / "x.ply"), t, chunk_bytes=rec - 4)


def test_default_chunk_holds_at_most_64_mib(tmp_path, monkeypatch):
    t = _tensors(300_000, 3, False, seed=3, special=False)          # 74 MB of records: two chunks
    sizes = []
    real = ply._pinned
    monkeypatch.setattr(ply, "_pinned", lambda n: sizes.append(n) or real(n))
    a, b = str(tmp_path / "gpu.ply"), str(tmp_path / "numpy.ply")
    ply.save(a, t)
    _numpy_write(b, t)
    assert filecmp.cmp(a, b, shallow=False)
    _bits_equal(ply.load(a), S.load_gaussians_ply(b))
    assert ply.CHUNK_BYTES == 64 << 20 and sizes == [(64 << 20) // 248 * 248] * 2


@pytest.mark.parametrize("deg", [0, 3])
@pytest.mark.parametrize("P_", [1, 129, 1000])
@pytest.mark.parametrize("pinned", [False, True])
@pytest.mark.parametrize("offset", [0, 4, 8, 12])
def test_kernels_at_every_16_byte_phase(tmp_path, deg, P_, pinned, offset):
    """pack into, and unpack from, a device or pinned host buffer at byte offset 0, 4, 8 and 12: the file's records."""
    t = _tensors(P_, deg, True, seed=offset)
    path = str(tmp_path / "numpy.ply")
    _numpy_write(path, t)
    data = open(path, "rb").read()
    body = np.frombuffer(data[ply.layout(path)[3]:], np.uint8)
    n = body.size
    buf = torch.full((n + 32,), 0xA5, dtype=torch.uint8, device="cpu" if pinned else DEV)
    if pinned:
        buf = buf.pin_memory()
    ply.pack(t, buf, byte_offset=offset)
    torch.cuda.synchronize()
    got = buf.cpu().numpy()
    assert np.array_equal(got[offset:offset + n], body)
    assert (got[:offset] == 0xA5).all() and (got[offset + n:] == 0xA5).all()          # nothing outside the run
    out = {k: torch.full_like(v, float("nan")) for k, v in t.items()}
    ply.unpack(buf, out, byte_offset=offset)
    torch.cuda.synchronize()
    _bits_equal(out, S.load_gaussians_ply(path))
    # a slice of the records, as the chunked writer packs it
    k0, k = P_ // 3, P_ - P_ // 3
    rec = n // P_
    part = torch.zeros(k * rec + offset, dtype=torch.uint8, device=DEV)
    ply.pack(t, part, k0, k, offset)
    assert np.array_equal(part.cpu().numpy()[offset:], body[k0 * rec:])


def test_files_the_numpy_reader_takes(tmp_path):
    """Every file layout() sends to the numpy reader loads on the device with load_gaussians_ply's values, and one
    the numpy reader refuses is refused with the same error."""
    from test_ply_io_cpu import EDITS, _rewrite
    t = _tensors(5, 3, False, seed=7)
    path = str(tmp_path / "a.ply")
    _numpy_write(path, t)
    read = 0
    for name, edit in EDITS.items():
        other = _rewrite(path, str(tmp_path / f"{name}.ply"), edit)
        assert ply.layout(other) is None
        try:
            want = S.load_gaussians_ply(other)
        except Exception as e:
            with pytest.raises(type(e)):
                ply.load(other)
            continue
        _bits_equal(ply.load(other), want)
        read += 1
    assert read >= 5
    data = open(path, "rb").read()
    open(str(tmp_path / "long.ply"), "wb").write(data + b"\1" * 12)
    _bits_equal(ply.load(str(tmp_path / "long.ply")), S.load_gaussians_ply(path))
    six = str(tmp_path / "six.ply")
    rng = np.random.default_rng(2)
    S._write_ply(six, [(n, "f4") for n in S.gaussian_ply_fields(6)],
                 [rng.standard_normal(4).astype(np.float32) for _ in range(23)])
    _bits_equal(ply.load(six), S.load_gaussians_ply(six))


# ---- 2. the trainer ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("deg", [0, 1, 2, 3])
@pytest.mark.parametrize("mip", [None, 0.1])
def test_trainer_save_ply(tmp_path, deg, mip):
    sc = surface_scene(1003, 2, 48, 32, seed=9 + deg, sh_degree=deg)
    cfg = OptimConfig()
    cfg.max_sh_degree, cfg.mip_kernel_size = deg, mip
    tr = I.JointTrainer(sc, DEV, cfg=cfg)
    a, b = str(tmp_path / "d" / "gpu.ply"), str(tmp_path / "e" / "numpy.ply")
    tr.save_ply(a, io="gpu")
    tr.save_ply(b)
    assert filecmp.cmp(a, b, shallow=False)
    assert (S.ply_properties(a)[-1] == "filter_3D") == (mip is not None)
    _bits_equal(ply.load(a), {k: v.cpu().numpy() for k, v in tr.ply_tensors().items()})
    with pytest.raises(ValueError, match="io must be"):
        tr.save_ply(a, io="pil")


# ---- 3. the command lines ------------------------------------------------------------------------------------
def _files(root):
    out = []
    for d, _, fs in os.walk(root):
        out += [os.path.relpath(os.path.join(d, f), root) for f in fs]
    return sorted(out)


def test_train_cli(tmp_path):
    from test_train_cli_gpu import _source
    src = _source(str(tmp_path / "src"), P=2000, W=64, H=48)
    base = ["-s", src, "-r", "1", "--n_views", "3", "--iterations", "25", "--pp_optimizer", "--optim_pose",
            "--save_iterations", "7", "20", "--quiet"]
    a, b = str(tmp_path / "numpy"), str(tmp_path / "gpu")
    for m, extra in ((a, []), (b, ["--ply_io", "gpu"])):
        T.run(T.parse_args(base + ["-m", m] + extra))
    for it in (7, 20, 25):
        for rel in (("point_cloud", f"iteration_{it}", "point_cloud.ply"), ("pose", f"ours_{it}", "pose_optimized.npy"),
                    ("pose", f"ours_{it}", "pose_org.npy")):
            assert filecmp.cmp(os.path.join(a, *rel), os.path.join(b, *rel), shallow=False), rel
    for rel in ("cameras.json", "input.ply"):
        assert filecmp.cmp(os.path.join(a, rel), os.path.join(b, rel), shallow=False), rel
    cfg = lambda m: open(os.path.join(m, "cfg_args")).read().replace(m, "MODEL")      # each holds its model path
    assert cfg(a) == cfg(b) and "ply_io" not in cfg(b)
    assert _files(a) == _files(b)


def test_train_cli_with_mip(tmp_path):
    from test_train_cli_gpu import _source
    src = _source(str(tmp_path / "src"), P=1500, W=64, H=48, seed=43)
    base = ["-s", src, "-r", "1", "--n_views", "3", "--iterations", "12", "--save_iterations", "5", "--quiet",
            "--kernel_size", "0.1"]
    a, b = str(tmp_path / "numpy"), str(tmp_path / "gpu")
    T.run(T.parse_args(base + ["-m", a]))
    T.run(T.parse_args(base + ["-m", b, "--ply_io", "gpu"]))
    for it in (5, 12):
        rel = os.path.join("point_cloud", f"iteration_{it}", "point_cloud.ply")
        assert filecmp.cmp(os.path.join(a, rel), os.path.join(b, rel), shallow=False)
        assert S.ply_properties(os.path.join(b, rel))[-1] == "filter_3D"


@pytest.fixture(scope="module")
def model(tmp_path_factory):
    from test_render_views_gpu import _source_and_model
    return _source_and_model(str(tmp_path_factory.mktemp("ply")))


def _same_trees(a, b):
    fa = _files(a)
    assert fa == _files(b)
    for rel in fa:
        if rel.endswith("train_time.txt"):
            continue
        assert filecmp.cmp(os.path.join(a, rel), os.path.join(b, rel), shallow=False), rel
    return fa


@pytest.mark.parametrize("stage", [[], ["--eval", "--optim_test_pose_iter", "20"], ["--infer_video"]])
def test_render_stages(model, tmp_path, stage):
    src, m, it = model
    a, b = str(tmp_path / "numpy"), str(tmp_path / "gpu")
    shutil.copytree(m, a)
    shutil.copytree(m, b)
    base = ["-s", src, "--n_views", "3", "--iterations", str(it), "-r", "1", "--workers", "2"] + stage
    with contextlib.redirect_stdout(open(os.devnull, "w")):
        assert R.main(base + ["-m", a]) == 0
        assert R.main(base + ["-m", b, "--ply_io", "gpu"]) == 0
    files = _same_trees(a, b)
    assert len([f for f in files if f.endswith(".png")]) > 0


def test_freeview(model, tmp_path):
    src, m, it = model
    a, b = str(tmp_path / "numpy"), str(tmp_path / "gpu")
    shutil.copytree(m, a)
    shutil.copytree(m, b)
    base = ["-s", src, "--n_views", "3", "--iterations", str(it), "--workers", "2"]
    with contextlib.redirect_stdout(open(os.devnull, "w")):
        assert F.main(base + ["-m", a]) == 0
        assert F.main(base + ["-m", b, "--ply_io", "gpu"]) == 0
    files = _same_trees(a, b)
    assert len([f for f in files if f.startswith("interp")]) == 2 * int(300 / 3) + 1


def test_load_tracker(model):
    src, m, it = model
    path = os.path.join(m, "point_cloud", f"iteration_{it}", "point_cloud.ply")
    views = S.load_views(src, 3, 0)
    a = F.load_tracker(path, views.width, views.height, views.fovx, views.fovy)
    b = F.load_tracker(path, views.width, views.height, views.fovx, views.fovy, ply_io="gpu")
    poses = F.poses_from_w2c(views.w2c)
    assert torch.equal(a.render_batch(poses), b.render_batch(poses))


def test_pipeline_eval_on_two_tasks(model, tmp_path):
    from test_pipeline_gpu import _compare_trees, _data_root
    src, _, _ = model
    root = _data_root(str(tmp_path / "data"), src, "eval")
    out = str(tmp_path / "out")
    argv = ["eval", "--data_root", root, "--output_dir", out, "--datasets", "D", "--scenes", "A", "B", "--n_views",
            "3", "--iterations", "20", "--workers", "2"]
    with contextlib.redirect_stdout(open(os.devnull, "w")):
        assert P.main(argv) == 0
        os.rename(out, str(tmp_path / "numpy"))
        assert P.main(argv + ["--ply_io", "gpu"]) == 0
    files = _compare_trees(out, str(tmp_path / "numpy"))
    for scene in ("A", "B"):
        assert os.path.join("D", scene, "3_views", "point_cloud", "iteration_20", "point_cloud.ply") in files


# ---- 4. past 2^31 bytes --------------------------------------------------------------------------------------
def test_round_trip_past_2_31_bytes(tmp_path):
    P_ = 9_000_000                                      # 9e6 x 248 bytes = 2.23e9 > 2^31
    rec = 248
    need = 3 * P_ * rec + (1 << 30)
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip(f"needs {need / 2**30:.1f} GiB of free device memory, {free / 2**30:.1f} GiB free")
    t = _tensors(P_, 3, False, seed=1)
    buf = torch.empty(P_ * rec, dtype=torch.uint8, device=DEV)
    assert buf.numel() > 2 ** 31
    ply.pack(t, buf)                                     # one launch over all 2.23e9 bytes
    # records either side of byte 2^31 and the last one, against numpy's layout of the same rows
    lo = (2 ** 31) // rec - 2
    for first in (0, lo, P_ - 3):
        rows = {k: v[first:first + 3].contiguous() for k, v in t.items()}
        small = torch.empty(3 * rec, dtype=torch.uint8, device=DEV)
        ply.pack(rows, small)
        assert torch.equal(buf[first * rec:(first + 3) * rec], small), first
        path = str(tmp_path / f"rows{first}.ply")
        _numpy_write(path, rows)
        assert np.array_equal(small.cpu().numpy(), np.frombuffer(open(path, "rb").read()[ply.layout(path)[3]:], np.uint8))
    out = {k: torch.empty_like(v) for k, v in t.items()}
    ply.unpack(buf, out)
    for k in t:
        assert torch.equal(out[k].view(torch.int32), t[k].view(torch.int32)), k
    del out, buf
    if shutil.disk_usage(str(tmp_path)).free < 2 * P_ * rec:
        pytest.skip("the device round trip passed; not enough disk for the 2.2 GB file")
    path = str(tmp_path / "big.ply")
    ply.save(path, t)
    assert os.path.getsize(path) == len(S.gaussian_ply_header(P_, 45, False)) + P_ * rec
    back = ply.load(path)
    for k in t:
        assert torch.equal(back[k].view(torch.int32), t[k].view(torch.int32)), k
