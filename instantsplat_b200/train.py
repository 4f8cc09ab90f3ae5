"""The training stage of InstantSplat's scripts (stage 2 of run_eval.sh and run_infer.sh): train.py's `training`
(train.py:88-231) from an init_geo-shaped source to the model render.py reads, with JointTrainer replayed from CUDA
graphs as the loop (DESIGN.md section 4.14).

    python -m instantsplat_b200.train -s SOURCE -m MODEL -r 1 --n_views N --iterations IT --pp_optimizer --optim_pose

What train.py does between the parts this package already has, and where it lives here:

  * load_host_scene / load_training_scene: Scene(dataset, gaussians) (scene/__init__.py:27-95).  The cameras of
    sparse_<n>/0 sorted by image_name, then random.seed(0)'s shuffle: pose row (uid) r is the r-th camera after it.
    The pose table is init_RT_seq's, the extent getNerfppNorm's radius, the Gaussians create_from_pcd's (knn on the
    GPU), the per-point learning rates load_and_prepare_confidence(scale=(1, 100))'s, and --init_scale_from_view_depth
    caps the scales with compute_scale_gaussian_by_project_pair_pcd.
  * view_schedule: train.py's random camera pick (train.py:117-158), seed 0 and the Scene's shuffle first.  A run
    resumed with --start_checkpoint re-seeds, so its schedule starts afresh; it is not the rest of the uninterrupted
    run's schedule.
  * run: the save, checkpoint and report points, pose_org.npy / pose_optimized.npy, train_time.txt, and the EMA loss
    read back asynchronously from a device ring (no host wait per iteration).
  * cfg_args_text, cameras_json and input.ply: the files train.py writes beside the model, byte for byte.

Refused with the reason before anything is written: --eval, --random_background, --sh_degree other than 3, a -r
that resamples the images without --resample_images (load_views' refusals), camera ids that are not 1..n, a missing
confidence_dsp.npy.

--resample_images (not one of train.py's flags, and not part of cfg_args) resizes the training images to loadCam's
size on the GPU, Pillow's bicubic resize byte for byte (resample.py), and trains at that size; cameras.json and the
view-depth scale cap keep the decoded size, as train.py's CameraInfo does.

--kernel_size K (Mip-Splatting, not one of train.py's flags, and not part of cfg_args; mip.py) trains with both
Mip-Splatting filters, OptimConfig.mip_kernel_size = K: the 3D filter is computed when the trainer is built (or
restored from --start_checkpoint) and recomputed every mip_filter3d_interval iterations except in the last 100,
point_cloud.ply gets the filter_3D property, checkpoints carry the filter, and the `Evaluating train` line renders with
the filters.  A K that is negative, NaN or infinite is refused.  Without the flag no filter is used.

--ply_io gpu (not one of train.py's flags, and not part of cfg_args; ply.py) writes point_cloud.ply at the save points
with JointTrainer.save_ply(io="gpu"): the records packed from the flat buffers on the GPU, the same bytes as without it.

--jpeg_decoder gpu (not one of train.py's flags, and not part of cfg_args; jpeg.py) decodes the training views' JPEG
files on the GPU in one call, Pillow's pixels byte for byte; other files, and JPEG files outside the decoder's subset,
go through Pillow as without it.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import random
import shutil
import sys
import time
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import freeview, jpeg, mip, ply, resample
from .scene_io import Views, load_views, read_points3d_ply

# ---- train.py's command line: arguments/__init__.py:47-94 and train.py:299-312 --------------------------------------
# A leading underscore gives the flag a one-letter shorthand, as ParamGroup does.
MODEL_PARAMS = (("sh_degree", 3), ("_source_path", ""), ("_model_path", ""), ("_images", "images"), ("_resolution", -1),
                ("_white_background", False), ("data_device", "cuda"), ("eval", False), ("n_views", 0),
                ("init_scale_from_view_depth", False))
OPTIMIZATION_PARAMS = (("iterations", 30_000), ("position_lr_init", 0.00016), ("position_lr_final", 0.0000016),
                       ("position_lr_delay_mult", 0.01), ("position_lr_max_steps", 30_000), ("feature_lr", 0.0025),
                       ("opacity_lr", 0.05), ("scaling_lr", 0.005), ("rotation_lr", 0.001), ("percent_dense", 0.01),
                       ("lambda_dssim", 0.2), ("densification_interval", 100), ("opacity_reset_interval", 3000),
                       ("densify_from_iter", 500), ("densify_until_iter", 15_000), ("densify_grad_threshold", 0.0002),
                       ("random_background", False), ("pp_optimizer", False), ("optim_pose", False))
PIPELINE_PARAMS = (("convert_SHs_python", False), ("compute_cov3D_python", False), ("debug", False))
# the OptimizationParams fields the training loop reads (the densify ones belong to its commented-out block)
LOOP_FIELDS = ("iterations", "position_lr_init", "position_lr_final", "position_lr_delay_mult", "position_lr_max_steps",
               "feature_lr", "opacity_lr", "scaling_lr", "rotation_lr", "lambda_dssim", "pp_optimizer", "optim_pose")


def _add_group(ap: argparse.ArgumentParser, title: str, fields) -> None:
    g = ap.add_argument_group(title)
    for key, value in fields:
        flags = ["--" + key.lstrip("_")] + (["-" + key[1]] if key.startswith("_") else [])
        if type(value) is bool:
            g.add_argument(*flags, default=value, action="store_true")
        else:
            g.add_argument(*flags, default=value, type=type(value))


def parser() -> argparse.ArgumentParser:
    """train.py's parser: ModelParams, OptimizationParams and PipelineParams in its order, then its own flags."""
    ap = argparse.ArgumentParser(prog="python -m instantsplat_b200.train",
                                 description="train.py: joint pose and Gaussian optimisation of an init_geo scene")
    _add_group(ap, "Loading Parameters", MODEL_PARAMS)
    _add_group(ap, "Optimization Parameters", OPTIMIZATION_PARAMS)
    _add_group(ap, "Pipeline Parameters", PIPELINE_PARAMS)
    ap.add_argument("--ip", type=str, default="127.0.0.1", help="ignored (train.py's viewer)")
    ap.add_argument("--port", type=int, default=6009, help="ignored (train.py's viewer)")
    ap.add_argument("--debug_from", type=int, default=-1, help="ignored")
    ap.add_argument("--detect_anomaly", action="store_true", default=False, help="ignored (no autograd)")
    ap.add_argument("--test_iterations", nargs="+", type=int, default=[])
    ap.add_argument("--save_iterations", nargs="+", type=int, default=[])
    ap.add_argument("--quiet", action="store_true")
    ap.add_argument("--disable_viewer", action="store_true", default=True, help="ignored (train.py's viewer)")
    ap.add_argument("--checkpoint_iterations", nargs="+", type=int, default=[])
    ap.add_argument("--start_checkpoint", type=str, default=None)
    resample.add_arg(ap)
    mip.add_arg(ap)
    ply.add_arg(ap)
    jpeg.add_arg(ap)
    return ap


def parse_args(argv: Optional[Sequence[str]] = None) -> argparse.Namespace:
    """The parsed flags, with --iterations appended to --save_iterations as train.py does."""
    args = parser().parse_args(argv)
    args.save_iterations.append(args.iterations)
    return args


def refusals(args: argparse.Namespace) -> List[str]:
    """The flag combinations this stage does not run, each with its reason."""
    out = []
    if not args.source_path or not args.model_path:
        out.append("-s/--source_path and -m/--model_path are required")
    if args.eval:
        out.append("--eval: train.py would load sparse_<n>/1, the test views, as its training cameras, and its "
                   "training_report would call get_RT_test on a test pose table that is never set")
    if args.random_background:
        out.append("--random_background: a fresh random background every iteration is not reproducible and does not "
                   "fit a captured CUDA graph")
    if args.sh_degree != 3:
        out.append(f"--sh_degree {args.sh_degree}: the trainer's flat buffers hold degree-3 SH, and a smaller layout "
                   "would change the ply and checkpoint shapes")
    if args.start_checkpoint is not None and not os.path.isfile(args.start_checkpoint):
        out.append(f"--start_checkpoint: {args.start_checkpoint} not found")
    why = mip.kernel_refusal(mip.kernel_size(args))
    if why:
        out.append(why)
    return out


def cfg_args_text(args: argparse.Namespace) -> str:
    """prepare_output_and_logger's cfg_args: str(Namespace) of the ModelParams group (ModelParams.extract: the fields
    in parse order, source_path made absolute), what get_combined_args evals."""
    keys = {k.lstrip("_") for k, _ in MODEL_PARAMS}
    d = {k: v for k, v in vars(args).items() if k in keys}
    d["source_path"] = os.path.abspath(d["source_path"])
    return str(argparse.Namespace(**d))


# ---- the scene: scene/__init__.py:27-95, scene/dataset_readers.py:50-71,315-369, train.py:63-97 ----------------------
def scene_order(n_views: int) -> List[int]:
    """Scene's shuffle after safe_state's random.seed(0): order[r] is the index (in image_name order) of the camera with
    uid r.  A local random.Random(0); the global state is not touched."""
    return _seeded(n_views)[1]


def _seeded(n_views: int) -> Tuple[random.Random, List[int]]:
    rng = random.Random(0)
    order = list(range(n_views))
    rng.shuffle(order)                   # random.shuffle(train_cameras)
    rng.shuffle([])                      # random.shuffle(test_cameras): empty without --eval
    return rng, order


def view_schedule(n_views: int, iterations: int, first_iter: int = 0) -> Tuple[List[int], List[int]]:
    """(scene_order(n_views), the pose row trained at each iteration first_iter + 1 .. iterations): train.py's stack of
    uids, refilled when empty, popped at randint(0, len - 1).  A resumed run (first_iter > 0) re-seeds and rebuilds
    the stack, as train.py does."""
    rng, order = _seeded(n_views)
    rows, stack = [], []
    for _ in range(first_iter + 1, iterations + 1):
        if not stack:
            stack = list(range(n_views))
        rows.append(stack.pop(rng.randint(0, len(stack) - 1)))
    return order, rows


def fov2focal(fov: float, pixels: int) -> float:
    return pixels / (2 * math.tan(fov / 2))


def nerfpp_radius(w2c: np.ndarray) -> float:
    """getNerfppNorm's radius (scene/dataset_readers.py:50-71): 1.1 x the largest distance of a camera centre from
    their mean, each centre from the inverse of getWorld2View2's fp32 matrix, in the reference's numpy dtypes."""
    centers = []
    for m in np.asarray(w2c):
        C2W = np.linalg.inv(freeview._world2view2(np.transpose(m[:3, :3]), m[:3, 3]))
        centers.append(C2W[:3, 3:4])
    cam_centers = np.hstack(centers)
    center = np.mean(cam_centers, axis=1, keepdims=True)
    diagonal = np.max(np.linalg.norm(cam_centers - center, axis=0, keepdims=True))
    return float(diagonal * 1.1)


def scale_from_view_depth(points: np.ndarray, w2c: np.ndarray, fx: float, fy: float) -> np.ndarray:
    """compute_scale_gaussian_by_project_pair_pcd (utils/graphics_utils.py:107-135) as Scene calls it: extrinsics
    np.linalg.inv of the [R^T | T] blocks (readColmapCameras' poses, R = qvec2rotmat^T, in image_name order), every
    view projecting every point; the per-point minimum depth, clipped below at 0.01, over the mean of the last view's
    focal lengths.  fp64 [P]."""
    poses = []
    for m in np.asarray(w2c):
        R, T = np.transpose(m[:3, :3]), np.array(m[:3, 3])
        poses.append(np.block([[R, T.reshape(3, 1)], [np.zeros((1, 3)), 1]]))
    depth_z = []
    for extrin in np.linalg.inv(np.array(poses)):
        R, t = extrin[:3, :3], extrin[:3, 3]
        depth_z.append((R @ points.T + t[:, np.newaxis])[2, :])
    depth_z = np.min(np.array(depth_z), 0)
    depth_z = np.clip(depth_z, 0.01, depth_z.max())
    return depth_z / ((fx + fy) / 2)


def load_confidence(path: str) -> torch.Tensor:
    """train.py's load_and_prepare_confidence(path, device="cpu", scale=(1, 100)): (1 - sigmoid(c)) * 99 + 1, fp32 on the
    CPU.  train.py reads the file unconditionally, so a missing one is an error."""
    if not os.path.isfile(path):
        raise FileNotFoundError(f"{path} not found (train.py reads the per-point confidence unconditionally)")
    c = torch.from_numpy(np.load(path)).float()
    min_scale, max_scale = 1, 100
    return (1.0 - torch.sigmoid(c)) * (max_scale - min_scale) + min_scale


@dataclass
class HostScene:
    """The host side of train.py's Scene.  views: the training cameras sorted by image_name; order[r]: the index into
    views of pose row (uid) r; colmap_ids[r]: that camera's COLMAP camera id; poses [n, 7] fp32: init_RT_seq's table in
    row order; extent: getNerfppNorm's radius; points [P, 3] fp32 and colors [P, 3] fp64 (u8 / 255): fetchPly's cloud;
    per_point_lr [P, 1] fp32; scale_gaussian [P] fp64 or None; ply_path: points3D.ply."""
    views: Views
    order: List[int]
    colmap_ids: List[int]
    poses: torch.Tensor
    extent: float
    points: np.ndarray
    colors: np.ndarray
    per_point_lr: torch.Tensor
    scale_gaussian: Optional[np.ndarray]
    ply_path: str


def load_host_scene(source_path: str, n_views: int, resolution: int, images: str = "images",
                    init_scale_from_view_depth: bool = False, resample_device=None, decode_device=None) -> HostScene:
    """Everything of load_training_scene that is computed on the CPU, except the image resize of a CUDA
    resample_device and the JPEG decode of a CUDA decode_device (load_views').  Raises, before anything is written,
    on what train.py cannot train: load_views' refusals, camera ids other than 1..n (save_pose looks up colmap ids
    1..n and would fail at the first save point), a missing points3D.ply or confidence_dsp.npy."""
    views = load_views(source_path, n_views, 0, resolution, images, resample_device, decode_device)
    ids = list(views.camera_ids)
    if sorted(ids) != list(range(1, len(views) + 1)):
        raise ValueError(f"sparse_{n_views}/0: camera ids {ids}; train.py's save_pose needs every camera id 1..{len(views)} "
                         "exactly once (one COLMAP camera per image, as init_geo writes them)")
    folder = os.path.join(source_path, f"sparse_{n_views}", "0")
    ply_path = os.path.join(folder, "points3D.ply")
    if not os.path.isfile(ply_path):
        raise FileNotFoundError(f"{ply_path} not found")
    ppl = load_confidence(os.path.join(folder, "confidence_dsp.npy"))
    xyz, rgb, _ = read_points3d_ply(ply_path)
    if ppl.shape[0] != xyz.shape[0]:
        raise ValueError(f"{folder}: confidence_dsp.npy has {ppl.shape[0]} values for {xyz.shape[0]} points")
    order = scene_order(len(views))
    sg = None
    if init_scale_from_view_depth:
        sg = scale_from_view_depth(xyz, views.w2c, fov2focal(views.fovx, views.source_width),
                                   fov2focal(views.fovy, views.source_height))
    return HostScene(views=views, order=order, colmap_ids=[ids[i] for i in order],
                     poses=freeview.poses_from_w2c(views.w2c[order]), extent=nerfpp_radius(views.w2c), points=xyz,
                     colors=rgb / 255.0, per_point_lr=ppl, scale_gaussian=sg, ply_path=ply_path)


@dataclass
class TrainingScene:
    """host: the HostScene; scene: the scenes.Scene JointTrainer trains (initial active SH degree 0, background by
    --white_background); targets [n, 3, H, W] fp32 u8 / 255 on the device, in pose-row order."""
    host: HostScene
    scene: "object"
    targets: torch.Tensor


def load_training_scene(source_path: str, n_views: int, resolution: int, images: str = "images", sh_degree: int = 3,
                        white_background: bool = False, init_scale_from_view_depth: bool = False,
                        device="cuda", resample_images: bool = False) -> TrainingScene:
    """train.py's Scene(dataset, gaussians) with its confidence: the cameras, their order, the pose table, the initial
    Gaussians (GaussianModel.create_from_pcd, spatial_lr_scale = the extent, its knn on the GPU), the per-point
    learning rates and the targets.  resample_images: resize the images on device when -r changes their size."""
    host = load_host_scene(source_path, n_views, resolution, images, init_scale_from_view_depth,
                           device if resample_images else None)
    return _device_scene(host, sh_degree, white_background, torch.device(device))


# ---- the files train.py writes beside the model ------------------------------------------------------------------
def cameras_json(views: Views) -> List[dict]:
    """camera_to_JSON (utils/camera_utils.py:66-86) of every camera in image_name order, before the shuffle, at the
    decoded size (CameraInfo's), whatever size the images are loaded at."""
    out = []
    for i, name in enumerate(views.names):
        Rt = np.zeros((4, 4))
        Rt[:3, :3] = views.w2c[i][:3, :3]
        Rt[:3, 3] = views.w2c[i][:3, 3]
        Rt[3, 3] = 1.0
        W2C = np.linalg.inv(Rt)
        W, H = views.source_width, views.source_height
        out.append({"id": i, "img_name": name, "width": W, "height": H,
                    "position": W2C[:3, 3].tolist(), "rotation": [x.tolist() for x in W2C[:3, :3]],
                    "fy": fov2focal(views.fovy, H), "fx": fov2focal(views.fovx, W)})
    return out


def write_model_files(args: argparse.Namespace, host: HostScene) -> None:
    """cfg_args (prepare_output_and_logger), input.ply (a byte copy of points3D.ply) and cameras.json (json.dump's
    default formatting), as train.py writes them."""
    os.makedirs(args.model_path, exist_ok=True)
    with open(os.path.join(args.model_path, "cfg_args"), "w") as f:
        f.write(cfg_args_text(args))
    shutil.copyfile(host.ply_path, os.path.join(args.model_path, "input.ply"))
    with open(os.path.join(args.model_path, "cameras.json"), "w") as f:
        json.dump(cameras_json(host.views), f)


def save_time(model_path: str, name: str, seconds: float) -> None:
    """utils/sfm_utils.py save_time: appends `<name>: <m> min <s> sec` to train_time.txt."""
    os.makedirs(model_path, exist_ok=True)
    minutes, secs = divmod(seconds, 60)
    with open(os.path.join(model_path, "train_time.txt"), "a") as f:
        f.write(f"{name}: {int(minutes)} min {int(secs)} sec\n")


def optim_config(args: argparse.Namespace, extent: float):
    """JointTrainer's OptimConfig from the command line: the OptimizationParams fields the loop reads (train.py's
    defaults, so pp_optimizer and optim_pose are off unless given), spatial_lr_scale = the extent, max_sh_degree, and
    mip_kernel_size = --kernel_size when it is given."""
    from .trainer import OptimConfig
    c = OptimConfig()
    for k in LOOP_FIELDS:
        setattr(c, k, getattr(args, k))
    c.spatial_lr_scale = float(extent)
    c.max_sh_degree = int(args.sh_degree)
    k = mip.kernel_size(args)
    if k is not None:
        c.mip_kernel_size = k
    return c


# ---- the run: train.py:88-231 ------------------------------------------------------------------------------------
class Refused(ValueError):
    """A source or a set of flags this stage does not train; raised before anything is written."""


@dataclass
class RunResult:
    """trainer: the JointTrainer at the end; rows: the pose row of each iteration run; first_iter: the iteration the
    run started after; losses [len(rows)] fp64 (CPU): each iteration's loss; phases: wall seconds per phase (load:
    PNG decode, PLY and confidence read; init: the Gaussians and targets on the GPU; trainer: trainer construction or
    restore; loop: the iterations without their saves; saves: ply, pose and checkpoint files); colmap_ids; host: the
    HostScene the run trained on (its views are the decoded training images)."""
    trainer: "object"
    rows: List[int]
    first_iter: int
    losses: torch.Tensor
    phases: Dict[str, float]
    colmap_ids: List[int]
    host: HostScene


def run(args: argparse.Namespace, device="cuda", log=print) -> RunResult:
    """train.py's training(): refuses first (nothing is written then), writes cfg_args, input.ply and cameras.json,
    builds the trainer (or restores --start_checkpoint), writes pose_org.npy for every save iteration, then runs the
    schedule with JointTrainer.step replayed from CUDA graphs.  Save and checkpoint points follow their iteration's
    step; train_time.txt gets train.py's two lines.  log prints the progress lines, unless --quiet."""
    from .trainer import JointTrainer
    bad = refusals(args)
    if bad:
        raise Refused("; ".join(bad))
    say = (lambda *a: None) if args.quiet else log
    dev = torch.device(device)
    phases = dict(load=0.0, init=0.0, trainer=0.0, loop=0.0, saves=0.0)
    t0 = time.perf_counter()
    try:
        host = load_host_scene(args.source_path, args.n_views, args.resolution, args.images,
                               args.init_scale_from_view_depth, dev if resample.requested(args) else None,
                               dev if jpeg.requested(args) else None)
    except (ValueError, FileNotFoundError) as e:
        raise Refused(str(e)) from e
    phases["load"] = time.perf_counter() - t0
    say(f"Optimizing {args.model_path}")
    write_model_files(args, host)
    say(f"Output folder: {args.model_path}")

    t0 = time.perf_counter()
    ts = _device_scene(host, args.sh_degree, args.white_background, dev)
    torch.cuda.synchronize(dev)
    phases["init"] = time.perf_counter() - t0
    cfg = optim_config(args, host.extent)
    t0 = time.perf_counter()
    if args.start_checkpoint:
        tr = JointTrainer.from_checkpoint(args.start_checkpoint, ts.scene, gt_images=ts.targets, cfg=cfg, device=dev,
                                          use_graph=True)
    else:
        tr = JointTrainer(ts.scene, dev, gt_images=ts.targets, cfg=cfg, use_graph=True)
    torch.cuda.synchronize(dev)
    phases["trainer"] = time.perf_counter() - t0
    first_iter = int(tr.iteration)
    ids = host.colmap_ids
    mp = args.model_path
    for it in args.save_iterations:
        tr.save_poses(os.path.join(mp, "pose", f"ours_{it}", "pose_org.npy"), ids)

    _, rows = view_schedule(len(ids), args.iterations, first_iter)
    n = len(rows)
    ring = torch.zeros(max(n, 1), 2, dtype=torch.float64, device=dev)
    pinned = torch.zeros(max(n, 1), 2, dtype=torch.float64).pin_memory()
    pending, state = [], dict(sent=0, ema=0.0)

    def drain(wait: bool) -> None:
        """EMA loss of the ring slices whose copy has landed (all of them when wait), printed every 10 iterations."""
        while pending and (wait or pending[0][0].query()):
            ev, lo, hi = pending.pop(0)
            ev.synchronize()
            for j, loss in enumerate(tr._loss(pinned[lo:hi]).tolist(), lo):
                state["ema"] = 0.4 * loss + 0.6 * state["ema"]
                it = first_iter + 1 + j
                if it % 10 == 0:
                    say(f"[ITER {it}] Loss {state['ema']:.7f}")

    start = time.time()
    t_loop = time.perf_counter()
    save_s = 0.0
    for k, row in enumerate(rows):
        it = first_iter + 1 + k
        tr.step(row)
        ring[k].copy_(tr.sums)
        if it % 10 == 0 or it == args.iterations:
            lo = state["sent"]
            pinned[lo:k + 1].copy_(ring[lo:k + 1], non_blocking=True)
            ev = torch.cuda.Event()
            ev.record()
            pending.append((ev, lo, k + 1))
            state["sent"] = k + 1
            drain(False)
        if it == args.iterations:
            torch.cuda.synchronize(dev)
            save_time(mp, "[2] train_joint_TrainTime", time.time() - start)
            if it in args.test_iterations or it % 5000 == 0:
                m = tr.evaluate()
                l1 = sum(m["l1"].tolist()) / len(ids)
                psnr = sum(m["psnr_channels"].mean(1).tolist()) / len(ids)
                say(f"\n[ITER {it}] Evaluating train: L1 {l1} PSNR {psnr}")
        ts0 = time.perf_counter()
        if it in args.save_iterations:
            say(f"\n[ITER {it}] Saving Gaussians")
            tr.save_ply(os.path.join(mp, "point_cloud", f"iteration_{it}", "point_cloud.ply"), ply.io(args) or "numpy")
            tr.save_poses(os.path.join(mp, "pose", f"ours_{it}", "pose_optimized.npy"), ids)
        if it in args.checkpoint_iterations:
            say(f"\n[ITER {it}] Saving Checkpoint")
            tr.save_checkpoint(os.path.join(mp, f"chkpnt{it}.pth"))
        save_s += time.perf_counter() - ts0
    torch.cuda.synchronize(dev)
    save_time(mp, "[2] train_joint", time.time() - start)
    drain(True)
    phases["loop"] = time.perf_counter() - t_loop - save_s
    phases["saves"] = save_s
    say("\nTraining complete.")
    return RunResult(tr, rows, first_iter, tr._loss(ring[:n]).cpu(), phases, ids, host)


def _device_scene(host: HostScene, sh_degree: int, white_background: bool, dev) -> TrainingScene:
    from .model import GaussianModel
    from .render_views import gt_images
    from .scenes import Scene
    gm = GaussianModel(sh_degree, dev)
    gm.create_from_pcd(host.points, host.colors, host.extent, host.scale_gaussian)
    params = {name: getattr(gm, attr).detach() for name, attr in GaussianModel._ATTR.items()}
    v = host.views
    scene = Scene(params, host.poses.clone(), v.width, v.height, v.fovx, v.fovy, sh_degree=0,
                  bg=torch.ones(3) if white_background else torch.zeros(3), per_point_lr=host.per_point_lr)
    targets = gt_images(v, dev)[torch.tensor(host.order, device=dev)].contiguous()
    return TrainingScene(host, scene, targets)


def main(argv: Optional[Sequence[str]] = None) -> int:
    args = parse_args(argv)
    try:
        run(args)
    except Refused as e:
        raise SystemExit(f"instantsplat_b200.train: {e}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
