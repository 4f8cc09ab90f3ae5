"""Generate tests/golden/train.npz from the REFERENCE's own training-stage code, run on CPU: train.py's argument
parser (arguments/__init__.py's ModelParams, OptimizationParams and PipelineParams plus train.py's flags),
`prepare_output_and_logger` (tensorboard off), `load_and_prepare_confidence(device="cpu", scale=(1, 100))`,
`random.seed(0)` then the real `Scene(args, gaussians)` (readColmapSceneInfo, the shuffle, getNerfppNorm,
cameraList_from_camInfos, input.ply, cameras.json, create_from_pcd with the stand-in distCUDA2, init_RT_seq) with and
without --init_scale_from_view_depth (compute_scale_gaussian_by_project_pair_pcd), and `save_pose`'s pose_org.npy.

Run like make_golden_checkpoint.py: `.cuda()` and device="cuda" stay on the CPU, the cameras' data_device is "cpu",
and the stand-ins of tests/cpu_standins serve distCUDA2 and the rasterizer imports.  cv2, roma, open3d, dust3r and
matplotlib are empty modules (their functions are not called here).  plyfile is not installed here, so fetchPly's
`PlyData.read(path)['vertex']` is served by instantsplat_b200.scene_io's binary PLY reader, which yields the same
named columns.

The view schedule (train.py:117-158) is recorded from train.py's selection lines restated below verbatim (RESTATEMENT:
`training()` renders and steps the optimizer on every iteration, which the CPU stand-ins cannot run at these counts),
after random.seed(0) and Scene's two shuffles of a list of n cameras.  The scene case checks that this restatement and
the real Scene draw the same shuffle.

    python oracle/make_golden_train.py <path to the InstantSplat checkout>
"""
import json
import os
import random
import sys
import tempfile
import types
from argparse import ArgumentParser

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if len(sys.argv) != 2:
    sys.exit(__doc__)
REF = sys.argv[1]
for p in (os.path.join(ROOT, "tests", "cpu_standins"), os.path.join(ROOT, "tests", "stubs"), ROOT):
    sys.path.insert(0, p)
sys.path.append(REF)

for name in ("matplotlib", "matplotlib.pyplot", "cv2", "roma", "open3d", "dust3r", "dust3r.utils",
             "dust3r.utils.image", "dust3r.utils.device", "plyfile"):
    sys.modules[name] = types.ModuleType(name)
sys.modules["matplotlib"].pyplot = sys.modules["matplotlib.pyplot"]
sys.modules["dust3r.utils.image"]._resize_pil_image = None
sys.modules["dust3r.utils.device"].to_numpy = None


class _PlyData:
    """plyfile.PlyData.read, as far as fetchPly uses it: data['vertex'][column]."""

    def __init__(self, vertex):
        self._vertex = vertex

    @classmethod
    def read(cls, path):
        from instantsplat_b200.scene_io import _read_ply
        return cls(_read_ply(path))

    def __getitem__(self, name):
        assert name == "vertex"
        return self._vertex


sys.modules["plyfile"].PlyData = _PlyData
sys.modules["plyfile"].PlyElement = None

import numpy as np  # noqa: E402
import torch  # noqa: E402

torch.Tensor.cuda = lambda self, *a, **k: self


class _TorchNoCuda:
    def __getattr__(self, name):
        obj = getattr(torch, name)
        if callable(obj) and not isinstance(obj, type):
            def call(*a, **k):
                if k.get("device") == "cuda":
                    k.pop("device")
                return obj(*a, **k)
            return call
        return obj


import scene as ref_scene  # noqa: E402
import scene.gaussian_model as ref_gm  # noqa: E402
from arguments import ModelParams, OptimizationParams, PipelineParams  # noqa: E402

ref_gm.torch = _TorchNoCuda()
import train as ref_train  # noqa: E402

ref_train.TENSORBOARD_FOUND = False

from instantsplat_b200 import scene_io  # noqa: E402
from instantsplat_b200.scenes import surface_scene  # noqa: E402

N_VIEWS = 4
NAMES = ["c.png", "a.png", "d.png", "b.png"]          # images.txt order; image_name order is a, b, c, d
SCHEDULES = [(n, it, first) for n in (1, 2, 3, 12, 24) for it, first in ((10, 0), (37, 0), (250, 0), (1000, 0),
                                                                           (250, 100), (1000, 537), (30, 30))]


def reference_parser() -> ArgumentParser:
    """train.py:299-312."""
    parser = ArgumentParser(description="Training script parameters")
    lp, op, pp = ModelParams(parser), OptimizationParams(parser), PipelineParams(parser)
    parser.add_argument('--ip', type=str, default="127.0.0.1")
    parser.add_argument('--port', type=int, default=6009)
    parser.add_argument('--debug_from', type=int, default=-1)
    parser.add_argument('--detect_anomaly', action='store_true', default=False)
    parser.add_argument("--test_iterations", nargs="+", type=int, default=[])
    parser.add_argument("--save_iterations", nargs="+", type=int, default=[])
    parser.add_argument("--quiet", action="store_true")
    parser.add_argument('--disable_viewer', action='store_true', default=True)
    parser.add_argument("--checkpoint_iterations", nargs="+", type=int, default=[])
    parser.add_argument("--start_checkpoint", type=str, default=None)
    return parser, lp, op, pp


def schedule(n: int, iterations: int, first_iter: int):
    """random.seed(0), Scene's shuffles, then train.py:117-118,122,124,152-157 (RESTATEMENT, verbatim but for the
    camera objects, which are their uids here)."""
    random.seed(0)
    train_cameras = list(range(n))
    random.shuffle(train_cameras)
    random.shuffle([])
    viewpoint_stack = list(range(n))                      # scene.getTrainCameras().copy(): uids 0..n-1
    viewpoint_indices = list(range(len(viewpoint_stack)))
    rows = []
    first_iter += 1
    for iteration in range(first_iter, iterations + 1):
        if not viewpoint_stack:
            viewpoint_stack = list(range(n))
            viewpoint_indices = list(range(len(viewpoint_stack)))
        rand_idx = random.randint(0, len(viewpoint_indices) - 1)
        viewpoint_cam = viewpoint_stack.pop(rand_idx)
        vind = viewpoint_indices.pop(rand_idx)
        assert viewpoint_cam == vind
        rows.append(viewpoint_cam)
    return train_cameras, rows


def write_source(root: str) -> None:
    """A tiny init_geo-shaped source: 300 points, 4 views listed out of image_name order, PNG images, camera ids 1..4,
    confidence values."""
    sc = surface_scene(300, N_VIEWS, 40, 28, seed=91, sh_degree=3)
    g = np.random.default_rng(91)
    imgs = g.integers(0, 256, (N_VIEWS, sc.height, sc.width, 3), dtype=np.uint8)
    folder = scene_io.write_synthetic_source(root, sc)
    fx = sc.width / (2.0 * np.tan(sc.fovx / 2.0))
    fy = sc.height / (2.0 * np.tan(sc.fovy / 2.0))
    scene_io.write_colmap_text(folder, sc.width, sc.height, fx, fy, sc.poses.numpy(), NAMES)
    np.save(os.path.join(folder, "confidence_dsp.npy"), (1.5 * g.standard_normal((sc.P, 1))).astype(np.float32))
    from PIL import Image
    os.makedirs(os.path.join(root, "images"), exist_ok=True)
    for i, n in enumerate(NAMES):
        Image.fromarray(imgs[i]).save(os.path.join(root, "images", n))


def read_tree(root: str):
    files = sorted(os.path.relpath(os.path.join(d, f), root) for d, _, fs in os.walk(root) for f in fs)
    return files, [np.frombuffer(open(os.path.join(root, f), "rb").read(), np.uint8).copy() for f in files]


def run_scene(src: str, model: str, argv, init_scale: bool, out: dict, tag: str) -> None:
    parser, lp, op, pp = reference_parser()
    args = parser.parse_args(argv)
    args.save_iterations.append(args.iterations)
    dataset = lp.extract(args)
    dataset.init_scale_from_view_depth = init_scale
    if not init_scale:
        out["argv"] = np.array(argv)
        out["ref_args_json"] = np.array(json.dumps(vars(args)))
        ref_train.prepare_output_and_logger(dataset)
        out["cfg_args"] = np.frombuffer(open(os.path.join(model, "cfg_args"), "rb").read(), np.uint8).copy()
    dataset.data_device = "cpu"
    confidence = ref_train.load_and_prepare_confidence(os.path.join(src, f"sparse_{N_VIEWS}/0", "confidence_dsp.npy"),
                                                       device="cpu", scale=(1, 100))
    recorded = {}
    real = ref_scene.compute_scale_gaussian_by_project_pair_pcd

    def record(*a, **k):
        recorded["scale"] = real(*a, **k)
        return recorded["scale"]

    ref_scene.compute_scale_gaussian_by_project_pair_pcd = record
    try:
        gaussians = ref_gm.GaussianModel(dataset.sh_degree)
        random.seed(0)
        sc = ref_scene.Scene(dataset, gaussians)
    finally:
        ref_scene.compute_scale_gaussian_by_project_pair_pcd = real
    cams = sc.getTrainCameras()
    for attr in ("_xyz", "_features_dc", "_features_rest", "_scaling", "_rotation", "_opacity"):
        out[f"{tag}{attr}"] = getattr(gaussians, attr).detach().numpy().copy()
    if init_scale:
        out["scale_gaussian"] = np.asarray(recorded["scale"])
        return
    out.update(uid_names=np.array([c.image_name for c in cams]), uid_colmap_ids=np.array([c.colmap_id for c in cams]),
               uids=np.array([c.uid for c in cams]), P=gaussians.P.detach().numpy().copy(),
               cameras_extent=np.asarray(sc.cameras_extent), confidence=confidence.numpy().copy())
    names_sorted = sorted(c.image_name for c in cams)
    order, _ = schedule(len(cams), 0, 0)
    assert [names_sorted[i] for i in order] == [c.image_name for c in cams], "the restated shuffle differs from Scene's"
    for f in ("cameras.json", "input.ply"):
        out[f.replace(".", "_")] = np.frombuffer(open(os.path.join(model, f), "rb").read(), np.uint8).copy()
    path = os.path.join(model, "pose", "ours_5", "pose_org.npy")
    os.makedirs(os.path.dirname(path), exist_ok=True)
    ref_train.save_pose(path, gaussians.P, sc.getTrainCameras().copy())
    out["pose_org"] = np.load(path)


def main():
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        src, model = os.path.join(tmp, "src"), os.path.join(tmp, "model")
        write_source(src)
        out["src_files"], blobs = read_tree(src)
        out["src_files"] = np.array(out["src_files"])
        for i, b in enumerate(blobs):
            out[f"src_blob_{i}"] = b
        os.makedirs(model)
        argv = ["-s", src, "-m", model, "-r", "1", "--n_views", str(N_VIEWS), "--iterations", "5", "--pp_optimizer",
                "--optim_pose"]
        out["source_path"], out["model_path"] = np.array(src), np.array(model)
        run_scene(src, model, argv, False, out, "init")
        run_scene(src, model, argv, True, out, "init_scaled")
    for n, it, first in SCHEDULES:
        order, rows = schedule(n, it, first)
        out[f"order_{n}"] = np.array(order, np.int64)
        out[f"sched_{n}_{it}_{first}"] = np.array(rows, np.int64)
    out["schedules"] = np.array(SCHEDULES, np.int64)
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "train.npz"), **out)
    print({k: getattr(v, "shape", None) for k, v in out.items() if not k.startswith("src_blob")})


if __name__ == "__main__":
    main()
