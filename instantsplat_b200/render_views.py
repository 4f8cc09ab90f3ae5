"""The training- and test-view renders of a trained model: stages 3 and 4 of InstantSplat's scripts/run_eval.sh,
render.py's render_sets (render.py:189-248) with its branch logic, on the GPU.

  * no --eval (render_set "train", render.py:204-216): the training views of source/sparse_<n>/0 (sorted by
    image_name) at the poses of pose/ours_<it>/pose_optimized.npy, row i to view i as loadCameras pairs them, turned
    into render() 7-vectors by freeview.poses_from_w2c.  Writes train/ours_<it>/renders/{idx:05d}.png and
    gt/{idx:05d}.png.
  * --eval (render_set_optimize, render.py:99-170): the test views of source/sparse_<n>/1, each starting from
    get_tensor_from_camera of its own world_view_transform (the same conversion), are tracked for
    --optim_test_pose_iter iterations in PoseTracker.optimize_batch (render.py's Adam groups, weight decay, cosine
    schedule and best-candidate rule; each view bit-identical to tracking it alone), then rendered at their best
    poses.  Writes test/ours_<it>/renders/<image_name>.png and gt/<image_name>.png.
  * --infer_video without --eval: the fly-through, freeview.main.

Renders are save_image's 8-bit frames (freeview.frames_u8).  A ground-truth file is save_image of the loaded image,
uint8 -> /255 -> uint8; that round trip is the identity on all 256 levels (checked once, gt_round_trip_is_identity),
so the gt PNGs are encoded from the decoded bytes.  Every PNG is encoded on freeview.write_pngs' thread pool, or on the
GPU by png.write_pngs with --png_encoder gpu.

--resample_images lets -r change the images' size: each stage's views are resized on the GPU to loadCam's size
(Pillow's bicubic resize, byte for byte, resample.py), the renders are made at that size, and the gt files hold the
resized bytes, as save_image(PILtoTorch(...)) writes them.  With --infer_video it also forwards -r to the fly-through.
Without the flag such a -r is refused, and --infer_video renders at the full size as before.

--test_fps with --eval is render.py's frame-rate report (render.py:172-186, report_fps): after the test renders, the
last test view in sorted order is rendered 1000 times at its best pose, from a replayed CUDA graph
(PoseTracker.time_renders), the rate of the trimmed mean is printed and appended to MODEL/total_fps.json, and the
`[4] render` line of train_time.txt records the test stage's time with the loop in it.  Without the flag neither
file is written.

Like render.py, both stages render without Mip-Splatting's filters, and a ply's filter_3D property is then not used.
--kernel_size K (mip.py) builds the tracker with both filters, the 2D filter at K and the ply's filter_3D, so the
training-view renders, the test-view tracking, the best-pose renders and the --test_fps loop all run the filtered
forward; with --infer_video the flag is forwarded to the fly-through.  It is refused, before anything is written, for
a K that is negative, NaN or infinite and for a ply without filter_3D (a model trained without --kernel_size).

The background is black, or white with --white_background; the SH degree is the ply's.  The model's cfg_args is not
read: render.py's get_combined_args lets every command-line value that is not None win, and ModelParams is built
with sentinel=False, so its defaults (white_background False included) always override the saved config there too.

    python -m instantsplat_b200.render_views -s SOURCE -m MODEL --n_views N --iterations IT [--eval] [--infer_video]
        [--optim_test_pose_iter 500] [--white_background] [--max_batch B] [--workers K] [--png_encoder pil|gpu]
        [--test_fps] [-r R --resample_images] [--kernel_size K] [--ply_io numpy|gpu] [--jpeg_decoder pil|gpu]

--ply_io gpu reads point_cloud.ply on the GPU (ply.py), for the stage here or the fly-through it hands over to; the
renders are the same as without it.

--jpeg_decoder gpu decodes the stage's JPEG source images (the training split, or --eval's test split) on the GPU in
one call (jpeg.py), Pillow's pixels byte for byte, so the gt files and renders are the same as without it.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time
from typing import Optional, Sequence, Tuple

import numpy as np
import torch

from . import freeview, jpeg, mip, ply, resample
from .scene_io import Views, load_views, read_colmap_text
from .tracking import PoseTracker
from .train import save_time


def gt_round_trip_is_identity() -> bool:
    """save_image(PILtoTorch(k)) == k for every 8-bit level k: uint8(clamp(fp32(k / 255) * 255 + 0.5, 0, 255))."""
    k = torch.arange(256, dtype=torch.uint8)
    x = k / 255.0
    return torch.equal(x.mul(255).add_(0.5).clamp_(0, 255).to(torch.uint8), k)


def gt_images(views: Views, device) -> torch.Tensor:
    """The views' images as loadCam hands them to render.py: [V, 3, H, W] fp32 k / 255 on the device."""
    u8 = torch.from_numpy(np.ascontiguousarray(views.images)).to(device)
    return (u8 / 255.0).permute(0, 3, 1, 2).contiguous()


def tracker_for(model_path: str, it: int, views: Views, white_background: bool = False, device="cuda",
                kernel_size: Optional[float] = None, ply_io: str = "numpy") -> PoseTracker:
    """freeview.load_tracker of point_cloud/iteration_<it>/point_cloud.ply at the views' size and field of view;
    kernel_size: with Mip-Splatting's filters (the ply's filter_3D); ply_io: read it the numpy way or on the GPU."""
    ply = os.path.join(model_path, "point_cloud", f"iteration_{it}", "point_cloud.ply")
    if not os.path.isfile(ply):
        raise FileNotFoundError(f"{ply} not found")
    return freeview.load_tracker(ply, views.width, views.height, views.fovx, views.fovy, white_background, device,
                                 kernel_size, ply_io)


def _write_gt(views: Views, folder: str, names, workers: Optional[int], write=freeview.write_pngs) -> None:
    if not gt_round_trip_is_identity():
        raise RuntimeError("the 8-bit -> fp32 -> 8-bit round trip is not the identity; gt files cannot be copied")
    write([(0, views.images)], folder, workers, names)


def render_train(tracker: PoseTracker, views: Views, w2c_opt, out_dir: str, max_batch: Optional[int] = None,
                 workers: Optional[int] = None, write=freeview.write_pngs) -> torch.Tensor:
    """render_set("train"): views at the optimised world-to-camera matrices w2c_opt [V, 4, 4] (pose_optimized.npy,
    one row per view) -> out_dir/renders/{idx:05d}.png and out_dir/gt/{idx:05d}.png, each folder's frames handed to
    write (freeview.write_pngs' signature).  Returns the 7-vectors [V, 7]."""
    w2c_opt = np.asarray(w2c_opt)
    if w2c_opt.ndim != 3 or w2c_opt.shape[0] != len(views):
        raise ValueError(f"render_train: {w2c_opt.shape[0] if w2c_opt.ndim == 3 else w2c_opt.shape} optimised poses "
                         f"for {len(views)} training views; loadCameras pairs them one to one")
    poses = freeview.poses_from_w2c(w2c_opt)
    write(freeview.frames_u8(tracker, poses, max_batch), os.path.join(out_dir, "renders"), workers)
    _write_gt(views, os.path.join(out_dir, "gt"), None, workers, write)
    return poses


def track(tracker: PoseTracker, views: Views, num_iter: int = 500, max_batch: Optional[int] = None) -> torch.Tensor:
    """render.py:113-161 for every test view: best poses [V, 7] (CPU fp32), from the views' own 7-vectors, tracked in
    PoseTracker.optimize_batch chunks of max_batch views (None: all at once)."""
    init = freeview.poses_from_w2c(views.w2c)
    best, _ = tracker.optimize_batch(init, gt_images(views, tracker.dev), num_iter=num_iter, max_batch=max_batch)
    return best


def render_test(tracker: PoseTracker, views: Views, out_dir: str, num_iter: int = 500, max_batch: Optional[int] = None,
                workers: Optional[int] = None, write=freeview.write_pngs) -> torch.Tensor:
    """render_set_optimize: track, then out_dir/renders/<image_name>.png at the best poses and out_dir/gt/<image_name>.png,
    through write as in render_train.  Returns the best poses [V, 7]."""
    best = track(tracker, views, num_iter, max_batch)
    names = [n + ".png" for n in views.names]
    write(freeview.frames_u8(tracker, best, max_batch), os.path.join(out_dir, "renders"), workers, names)
    _write_gt(views, os.path.join(out_dir, "gt"), names, workers, write)
    return best


def fps_from_times(durations: Sequence[float]) -> Tuple[float, str]:
    """render.py:180-186 on frame times in seconds: (fps, the text appended to total_fps.json).  fps is the reciprocal
    of the mean of the sorted times [100:900] (the 100 fastest and all past the 900th dropped); the text is
    json.dump(f'{fps}', fp, indent=True) and a newline, a JSON string holding str(fps) on a line of its own."""
    kept = sorted(durations)[100:900]
    fps = 1 / (sum(kept) / len(kept))
    return fps, json.dumps(f"{fps}", indent=True) + "\n"


def report_fps(tracker: PoseTracker, pose: torch.Tensor, model_path: str, start: float, n: int = 1000) -> float:
    """render.py's --test_fps and the end of its `[4] render` span (render.py:172-186, :219-231): prints
    `>>> Calculate FPS: `, times n renders at pose [7] (PoseTracker.time_renders), prints `>>> FPS = ` and the rate,
    appends fps_from_times' line to model_path/total_fps.json, then appends `[4] render` with the seconds since start
    (a time.time() value) to model_path/train_time.txt.  Returns the rate."""
    print(">>> Calculate FPS: ")
    fps, line = fps_from_times(tracker.time_renders(pose, n))
    print(">>> FPS = ", fps)
    with open(os.path.join(model_path, "total_fps.json"), "a") as f:
        f.write(line)
    save_time(model_path, "[4] render", time.time() - start)
    return fps


def fps_refusal(source_path: str, n_views: int) -> Optional[str]:
    """Why --eval --test_fps cannot run, or None: it times the last test view, and render.py fails when
    sparse_<n_views>/1 lists none (its loop variable `view` is then undefined).  A folder that cannot be read is left
    to load_views, which names the problem."""
    folder = os.path.join(source_path, f"sparse_{n_views}", "1")
    try:
        _, images = read_colmap_text(folder, ("PINHOLE", "SIMPLE_PINHOLE"))
    except (OSError, ValueError):
        return None
    return None if images else f"--test_fps times the last test view, and {folder}/images.txt lists none"


def parser() -> argparse.ArgumentParser:
    """render.py's command line as this stage reads it."""
    ap = argparse.ArgumentParser(prog="python -m instantsplat_b200.render_views",
                                 description="render.py: the training views at their optimised poses, or (--eval) "
                                             "the test views after pose tracking")
    ap.add_argument("-s", "--source_path", required=True)
    ap.add_argument("-m", "--model_path", required=True)
    ap.add_argument("--n_views", type=int, required=True)
    ap.add_argument("--iterations", type=int, default=-1)
    ap.add_argument("-r", "--resolution", type=int, default=-1)
    ap.add_argument("--eval", action="store_true")
    ap.add_argument("--infer_video", action="store_true")
    ap.add_argument("--optim_test_pose_iter", type=int, default=500)
    ap.add_argument("--white_background", action="store_true")
    ap.add_argument("--max_batch", type=int, default=12,
                    help="views per batched loop; tracking scratch is about 150 P + 44 H W bytes a view")
    ap.add_argument("--workers", type=int, default=None, help="PNG encoder threads (default: up to 8)")
    freeview.add_png_encoder_arg(ap)
    ap.add_argument("--test_fps", action="store_true",
                    help="with --eval: time 1000 renders of the last test view and append the rate to total_fps.json")
    resample.add_arg(ap)
    mip.add_arg(ap)
    ply.add_arg(ap)
    jpeg.add_arg(ap)
    return ap


def main(argv=None) -> int:
    a = parser().parse_args(argv)
    if a.max_batch < 1:
        raise SystemExit("--max_batch must be at least 1")
    k = mip.kernel_size(a)
    why = mip.kernel_refusal(k)
    if why:
        raise SystemExit(f"render_views: {why}")
    if a.infer_video and not a.eval:
        fv = ["-s", a.source_path, "-m", a.model_path, "--n_views", str(a.n_views), "--iterations", str(a.iterations),
              "--max_batch", str(a.max_batch)] + (["--white_background"] if a.white_background else []) \
            + ([] if a.workers is None else ["--workers", str(a.workers)]) + ["--png_encoder", a.png_encoder] \
            + ply.argv(ply.io(a)) + (["-r", str(a.resolution), "--resample_images"] if resample.requested(a) else []) + mip.argv(k)
        return freeview.main(fv)
    write = freeview.png_writer(a.png_encoder)
    it = freeview.max_iteration(a.model_path) if a.iterations == -1 else a.iterations
    why = mip.ply_refusal(k, freeview.model_files(a.model_path, it)[0])
    if why:
        raise SystemExit(f"render_views: {why}")
    rdev = "cuda" if resample.requested(a) else None
    ddev = "cuda" if jpeg.requested(a) else None
    if a.eval:
        why = fps_refusal(a.source_path, a.n_views) if a.test_fps else None
        if why:
            raise SystemExit(f"render_views: {why}")
        views = load_views(a.source_path, a.n_views, 1, a.resolution, resample_device=rdev, decode_device=ddev)
        tracker = tracker_for(a.model_path, it, views, a.white_background, kernel_size=k, **ply.kwargs(a))
        out = os.path.join(a.model_path, "test", f"ours_{it}")
        start = time.time()
        best = render_test(tracker, views, out, a.optim_test_pose_iter, a.max_batch, a.workers, write)
        if a.test_fps:
            report_fps(tracker, best[-1], a.model_path, start)
    else:
        npy = os.path.join(a.model_path, "pose", f"ours_{it}", "pose_optimized.npy")
        if not os.path.isfile(npy):
            raise FileNotFoundError(f"{npy} not found")
        views = load_views(a.source_path, a.n_views, 0, a.resolution, resample_device=rdev, decode_device=ddev)
        tracker = tracker_for(a.model_path, it, views, a.white_background, kernel_size=k, **ply.kwargs(a))
        out = os.path.join(a.model_path, "train", f"ours_{it}")
        render_train(tracker, views, np.load(npy), out, a.max_batch, a.workers, write)
    print(f"{len(views)} views -> {out}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
