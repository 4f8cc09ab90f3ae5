"""The free-view fly-through of a trained model: stage 3 of InstantSplat's scripts/run_infer.sh,
`render.py --infer_video` without `--eval` (render.py:204-248), as batched forwards and one 8-bit pass on the GPU.

What render.py does, and what each function here restates:
  1. interpolated_w2c: save_interpolate_pose (render.py:36-56).  The n key poses of pose_optimized.npy
     (world-to-camera, COLMAP id order) are joined pair by pair with utils/camera_utils.py:127-195
     generate_interpolated_path: with two key poses that is a degree-1 smoothing spline (k = min(5, 1), s = 0.03)
     through (position, lookat, up) points at rot_weight 0.1, sampled at int(300 / n) steps per pair, and rebuilt
     with viewmatrix.  The last key pose is appended and every pose embedded in np.eye(4): [(n-1) int(300/n) + 1, 4, 4]
     fp64.  The spline treats world-to-camera matrices as if they were camera-to-world; that is the reference's
     behaviour and is kept.
  2. poses_from_w2c: loadCameras (scene/dataset_readers.py:87-103) sets each frame's world_view_transform to
     getWorld2View2(p[:3, :3]^T, p[:3, 3]) (utils/graphics_utils.py:38-49: two fp64 inversions, which change low bits,
     then fp32), and render_set (render.py:86) turns it into the 7-vector render() takes with get_tensor_from_camera:
     rotation2quad (utils/pose_utils.py:117-180, pytorch3d's best-conditioned candidate in fp32, neither normalised nor
     sign-canonicalised) followed by t.  This is not model.w2c_to_pose (the trace method).
  3. frames_u8: render() at each 7-vector with the training cameras' intrinsics (frame i takes camera i % n; they
     must all be equal here) and torchvision's save_image quantisation, uint8(clamp(x * 255 + 0.5, 0, 255)).
  4. write_pngs: save_image's PIL PNG encode with default parameters, to renders/{idx:05d}.png.

The training-view renders of render.py's `render_set("train")` (the views at their optimised poses) need nothing
else: frames_u8(tracker, poses_from_w2c(np.load(".../pose_optimized.npy"))) and write_pngs.

Not done: the mp4 (images_to_video needs imageio / ffmpeg), the pose plots (matplotlib) and save_time.

-r / --resolution (default 1) and --resample_images: render.py renders the fly-through at the training cameras' loaded
size, loaded_size of cameras.txt's width and height at -r (init_geo writes the images' own size there).  With
--resample_images the frames are rendered at that size; without it a -r that changes the size is refused, and the
frames are the full-size ones.

Like render.py, the fly-through renders without Mip-Splatting's filters, and a ply's filter_3D property is then not
used.  --kernel_size K (mip.py) renders every frame with both filters: the 2D filter at K and the ply's filter_3D.
It is refused, before anything is written, for a K that is negative, NaN or infinite and for a ply without filter_3D
(a model trained without --kernel_size).

--ply_io gpu (ply.py) reads point_cloud.ply on the GPU: the records unpacked by one kernel into the tracker's device
tensors, the same values as without it (a file not in save_gaussians_ply's exact layout is read the numpy way).

    python -m instantsplat_b200.freeview -s SOURCE -m MODEL --n_views N --iterations IT [--white_background]
        [--png_encoder pil|gpu] [-r R --resample_images] [--kernel_size K] [--ply_io numpy|gpu]
"""
from __future__ import annotations

import argparse
import os
import sys
from collections import deque
from concurrent.futures import ThreadPoolExecutor
from typing import Iterable, Iterator, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib, mip, ply, png, resample
from ._lib import check
from .frame import ST_OVERFLOW
from .tracking import PoseTracker

ROT_WEIGHT, SMOOTHNESS, SPLINE_DEGREE = 0.1, 0.03, 5     # generate_interpolated_path's defaults


# ---- 1. trajectory -------------------------------------------------------------------------------------------
def _unit(x: np.ndarray) -> np.ndarray:
    return x / np.linalg.norm(x)


def _spline_segment(keys: np.ndarray, n_interp: int) -> np.ndarray:
    """generate_interpolated_path(poses=keys, n_interp) for key poses [m, 4, 4] (or [m, 3, 4]): [n_interp (m-1), 3, 4].
    The same numpy / scipy calls in the same order as the reference, so the same bits."""
    from scipy.interpolate import splev, splprep
    pos = keys[:, :3, -1]
    points = np.stack([pos, pos - ROT_WEIGHT * keys[:, :3, 2], pos + ROT_WEIGHT * keys[:, :3, 1]], 1)
    m = points.shape[0]
    n = n_interp * (m - 1)
    tck, _ = splprep(np.reshape(points, (m, -1)).T, k=min(SPLINE_DEGREE, m - 1), s=SMOOTHNESS)
    u = np.linspace(0, 1, n, endpoint=False)
    samples = np.reshape(np.array(splev(u, tck)).T, (n, 3, 3))
    out = []
    for p, lookat, up in samples:                     # viewmatrix(p - lookat, up - p, p)
        z = _unit(p - lookat)
        x = _unit(np.cross(up - p, z))
        y = _unit(np.cross(z, x))
        out.append(np.stack([x, y, z, p], axis=1))
    return np.array(out)


def interpolated_w2c(w2c, n_views: int) -> np.ndarray:
    """save_interpolate_pose: key poses w2c [n, 4, 4] (pose_optimized.npy; rows 0 .. n_views - 2 start the segments,
    and the last row is appended, as the reference does) -> [(n_views-1) int(300/n_views) + 1, 4, 4] fp64."""
    w2c = np.asarray(w2c)
    if w2c.ndim != 3 or w2c.shape[1:] not in ((4, 4), (3, 4)):
        raise ValueError(f"interpolated_w2c: expected [n, 4, 4] key poses, got {w2c.shape}")
    n_views = int(n_views)
    if n_views < 2:
        raise ValueError(f"interpolated_w2c: a fly-through needs at least 2 key poses, got n_views = {n_views}")
    if n_views > w2c.shape[0]:
        raise ValueError(f"interpolated_w2c: n_views = {n_views} but only {w2c.shape[0]} key poses")
    n_interp = int(10 * 30 / n_views)
    if n_interp < 1:
        # the reference's loadCameras would then render the training cameras at their own poses instead
        raise ValueError(f"interpolated_w2c: n_views = {n_views} leaves no frame between key poses (at most 300)")
    segs = [_spline_segment(w2c[i:i + 2], n_interp) for i in range(n_views - 1)]
    path = np.concatenate([np.concatenate(segs, axis=0), w2c[-1][:3, :].reshape(1, 3, 4)], axis=0)
    out = np.stack([np.eye(4)] * path.shape[0], 0)
    out[:, :3, :3] = path[:, :3, :3]
    out[:, :3, 3] = path[:, :3, 3]
    return out


# ---- 2. camera pose ------------------------------------------------------------------------------------------
def _world2view2(R: np.ndarray, t: np.ndarray) -> np.ndarray:
    """getWorld2View2(R, t) with translate 0 and scale 1: [R^T | t] inverted, its centre re-set, inverted again; fp32."""
    Rt = np.zeros((4, 4))
    Rt[:3, :3] = R.transpose()
    Rt[:3, 3] = t
    Rt[3, 3] = 1.0
    C2W = np.linalg.inv(Rt)
    C2W[:3, 3] = (C2W[:3, 3] + np.array([0.0, 0.0, 0.0])) * 1.0
    return np.float32(np.linalg.inv(C2W))


def rotation2quad(m: torch.Tensor) -> torch.Tensor:
    """utils/pose_utils.py rotation2quad on [N, 3, 3]: the quaternion (real first) from the candidate with the largest
    |q| component, in m's dtype, neither normalised nor sign-canonicalised.  Every operation is elementwise and
    correctly rounded in IEEE fp32 (add, subtract, multiply, divide, sqrt), so the CPU gives the bits the reference
    gets on CUDA; argmax takes the first of equal maxima on both."""
    m00, m01, m02, m10, m11, m12, m20, m21, m22 = m.reshape(-1, 9).unbind(-1)
    s = torch.stack([1.0 + m00 + m11 + m22, 1.0 + m00 - m11 - m22, 1.0 - m00 + m11 - m22, 1.0 - m00 - m11 + m22], -1)
    q_abs = torch.where(s > 0, torch.sqrt(s), torch.zeros_like(s))
    rows = torch.stack([
        torch.stack([q_abs[:, 0] ** 2, m21 - m12, m02 - m20, m10 - m01], -1),
        torch.stack([m21 - m12, q_abs[:, 1] ** 2, m10 + m01, m02 + m20], -1),
        torch.stack([m02 - m20, m10 + m01, q_abs[:, 2] ** 2, m12 + m21], -1),
        torch.stack([m10 - m01, m20 + m02, m21 + m12, q_abs[:, 3] ** 2], -1)], -2)
    cand = rows / (2.0 * q_abs[..., None].max(torch.tensor(0.1, dtype=q_abs.dtype)))
    return cand[torch.arange(cand.shape[0]), q_abs.argmax(-1)]


def poses_from_w2c(w2c) -> torch.Tensor:
    """loadCameras + get_tensor_from_camera for world-to-camera matrices [N, 4, 4] (any float dtype): the 7-vectors
    [N, 7] (fp32, CPU) render() takes, quaternion first."""
    w2c = np.asarray(w2c)
    if w2c.ndim != 3 or w2c.shape[1:] not in ((4, 4), (3, 4)):
        raise ValueError(f"poses_from_w2c: expected [N, 4, 4] matrices, got {w2c.shape}")
    rt = torch.from_numpy(np.stack([_world2view2(np.transpose(p[:3, :3]), p[:3, 3]) for p in w2c])
                          if len(w2c) else np.zeros((0, 4, 4), np.float32))
    return torch.cat([rotation2quad(rt[:, :3, :3]), rt[:, :3, 3]], 1)


# ---- 3. 8-bit frames on the GPU ------------------------------------------------------------------------------
def quantise(img: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """gsb_frames_u8_batch: img [V, 3, H, W] contiguous fp32 CUDA -> [V, H, W, 3] uint8, save_image's levels."""
    if not isinstance(img, torch.Tensor) or img.dim() != 4 or img.shape[1] != 3 or img.dtype != torch.float32 \
            or not img.is_cuda or not img.is_contiguous():
        raise ValueError(f"quantise: expected a contiguous fp32 CUDA [V, 3, H, W] tensor, got "
                         f"{tuple(getattr(img, 'shape', ()))}")
    V, _, H, W = img.shape
    if out is None:
        out = torch.empty(V, H, W, 3, dtype=torch.uint8, device=img.device)
    with torch.cuda.device(img.device):
        check(_lib.lib().gsb_frames_u8_batch(V, H, W, img.data_ptr(), out.data_ptr(), _lib.stream_ptr()),
              "gsb_frames_u8_batch")
    return out


def frames_u8(tracker: PoseTracker, poses: torch.Tensor, max_batch: Optional[int] = None
              ) -> Iterator[Tuple[int, np.ndarray]]:
    """render() at every row of poses [N, 7] through save_image's quantisation: yields (first_index, uint8 [B, H, W, 3])
    host chunks in order; each array is the caller's.  Each chunk is one batched forward of the tracker (its SH degree,
    Mip filters and background, binning sized from the chunk's own preprocess count) followed by
    gsb_frames_u8_batch; the device-to-host copy of chunk k runs on a side stream into a double-buffered pinned ring
    while chunk k + 1 renders.  max_batch: frames per forward (None: all).  Raises GsbError if a tile list outgrew
    the binning buffer."""
    p = tracker._poses(poses, "frames_u8")
    if max_batch is not None and int(max_batch) < 1:
        raise ValueError("frames_u8: max_batch must be >= 1")
    N, H, W, dev = p.shape[0], tracker.H, tracker.W, tracker.dev
    if N == 0:
        return
    B = N if max_batch is None else min(N, int(max_batch))
    main, side = torch.cuda.current_stream(dev), torch.cuda.Stream(dev)
    frames = [torch.empty(B, H, W, 3, dtype=torch.uint8, device=dev) for _ in range(2)]
    ring = [torch.empty(B, H, W, 3, dtype=torch.uint8).pin_memory() for _ in range(2)]
    ovf = torch.zeros(2, dtype=torch.int32, device=dev)
    ovf_host = torch.zeros(2, dtype=torch.int32).pin_memory()
    ready = [torch.cuda.Event() for _ in range(2)]
    done = [torch.cuda.Event() for _ in range(2)]
    cam = tracker._cam()

    def launch(v0: int, n: int, s: int) -> None:
        with torch.cuda.device(dev):
            fr = tracker._frame_batch(n)
            tracker._forward_batch(fr, cam, tracker._gauss(p[v0:v0 + n]), p[v0:v0 + n], True)
            main.wait_event(done[s])                       # slot s's copy of chunk k - 2 has left the device buffer
            quantise(fr.color, frames[s][:n])
            ovf[s:s + 1].copy_(fr.word(ST_OVERFLOW))
            ready[s].record(main)
            side.wait_event(ready[s])
            with torch.cuda.stream(side):
                ring[s][:n].copy_(frames[s][:n], non_blocking=True)
                ovf_host[s:s + 1].copy_(ovf[s:s + 1], non_blocking=True)
                done[s].record(side)

    def collect(v0: int, n: int, s: int) -> Tuple[int, np.ndarray]:
        done[s].synchronize()
        if int(ovf_host[s]):
            raise _lib.GsbError("frames_u8: a tile list outgrew the binning buffer")
        return v0, ring[s][:n].numpy().copy()

    pending = None
    try:
        for k, v0 in enumerate(range(0, N, B)):
            chunk = (v0, min(N - v0, B), k % 2)
            launch(*chunk)
            if pending is not None:
                yield collect(*pending)                    # chunk k - 1, while chunk k renders
            pending = chunk
        yield collect(*pending)
    finally:
        side.synchronize()                                 # nothing in flight on buffers that are about to be freed


# ---- 4. PNG files --------------------------------------------------------------------------------------------
def _save_png(img: np.ndarray, path: str) -> None:
    from PIL import Image
    Image.fromarray(img).save(path)                       # what save_image does with the uint8 HWC array


def write_pngs(frames: Iterable[Tuple[int, np.ndarray]], folder: str, workers: Optional[int] = None,
               names: Optional[Sequence[str]] = None) -> int:
    """Writes every frame of (first_index, uint8 [B, H, W, 3]) chunks to folder/{idx:05d}.png (or folder/names[idx]),
    the file torchvision.utils.save_image writes for that image, encoding on a pool of `workers` threads (None: up to 8;
    Pillow's encoder releases the GIL).  At most 4 x workers frames wait for the encoder.  Returns the number of
    files."""
    os.makedirs(folder, exist_ok=True)
    workers = min(8, os.cpu_count() or 1) if workers is None else int(workers)
    if workers < 1:
        raise ValueError("write_pngs: workers must be >= 1")
    count, pending = 0, deque()
    with ThreadPoolExecutor(max_workers=workers) as pool:
        for first, chunk in frames:
            for i in range(chunk.shape[0]):
                name = f"{first + i:05d}.png" if names is None else names[first + i]
                pending.append(pool.submit(_save_png, chunk[i], os.path.join(folder, name)))
                count += 1
            while len(pending) > 4 * workers:
                pending.popleft().result()
        for f in pending:
            f.result()
    return count


def add_png_encoder_arg(ap: argparse.ArgumentParser) -> None:
    ap.add_argument("--png_encoder", choices=("pil", "gpu"), default="pil",
                    help="pil: save_image's files, byte for byte; gpu: encoded on the GPU (png.py), other bytes that "
                         "decode to the same pixels")


def png_writer(encoder: str):
    """write_pngs for --png_encoder pil, png.write_pngs for gpu."""
    return png.write_pngs if encoder == "gpu" else write_pngs


# ---- the command line: stage 3 of run_infer.sh ---------------------------------------------------------------
def max_iteration(model_path: str) -> int:
    """searchForMaxIteration (utils/system_utils.py:26-28) over model_path/point_cloud."""
    folder = os.path.join(model_path, "point_cloud")
    if not os.path.isdir(folder):
        raise FileNotFoundError(f"no saved iterations: {folder} does not exist")
    its = [int(f.split("_")[-1]) for f in os.listdir(folder)]
    if not its:
        raise FileNotFoundError(f"no saved iterations under {folder}")
    return max(its)


def intrinsics(source_path: str, n_views: int):
    """(width, height, fovx, fovy) of the PINHOLE cameras in source/sparse_<n_views>/0/cameras.txt at full resolution
    (`-r 1`), FoV by focal2fov.  Refuses cameras that differ: render.py would cycle them frame by frame, and
    run_infer.sh's --focal_avg makes them equal."""
    import math
    from .scene_io import read_colmap_text
    folder = os.path.join(source_path, f"sparse_{n_views}", "0")
    if not os.path.isfile(os.path.join(folder, "cameras.txt")):
        raise FileNotFoundError(f"{folder}/cameras.txt not found")
    cams, _ = read_colmap_text(folder)
    if not cams:
        raise ValueError(f"{folder}/cameras.txt lists no camera")
    keys = {(c["width"], c["height"], float(c["params"][0]), float(c["params"][1])) for c in cams.values()}
    if len(keys) != 1:
        raise ValueError(f"{folder}/cameras.txt: the cameras' intrinsics differ ({len(keys)} distinct); the "
                         "fly-through renders with one camera")
    W, H, fx, fy = keys.pop()
    focal2fov = lambda f, pixels: 2 * math.atan(pixels / (2 * f))
    return W, H, focal2fov(fx, W), focal2fov(fy, H)


def frame_size(source_path: str, n_views: int, resolution: int = 1, resample_images: bool = False) -> Tuple[int, int]:
    """The fly-through's (width, height): loaded_size of the cameras' size at -r resolution.  Raises ValueError for a
    resolution that changes the size unless resample_images, and for an empty frame."""
    from .scene_io import loaded_size
    W, H, _, _ = intrinsics(source_path, n_views)
    Wl, Hl = loaded_size(W, H, resolution)
    if (Wl, Hl) != (W, H) and not resample_images:
        raise ValueError(f"-r {resolution} resizes {W}x{H} to {Wl}x{Hl}; resampled images are not supported without "
                         "--resample_images")
    if Wl < 1 or Hl < 1:
        raise ValueError(f"-r {resolution} resizes {W}x{H} to {Wl}x{Hl}, an empty frame")
    return Wl, Hl


def model_files(model_path: str, iteration: int = -1) -> Tuple[str, str, int]:
    """(point_cloud/iteration_<it>/point_cloud.ply, pose/ours_<it>/pose_optimized.npy, it) of a trained model;
    iteration -1: the largest saved one, for the model and the poses alike (render.py looks the poses up under the
    literal `ours_-1`)."""
    it = max_iteration(model_path) if int(iteration) == -1 else int(iteration)
    return (os.path.join(model_path, "point_cloud", f"iteration_{it}", "point_cloud.ply"),
            os.path.join(model_path, "pose", f"ours_{it}", "pose_optimized.npy"), it)


def load(source_path: str, model_path: str, n_views: int, iteration: int = -1, white_background: bool = False,
         device="cuda", resolution: int = 1, resample_images: bool = False, kernel_size: Optional[float] = None,
         ply_io: str = "numpy"):
    """What render.py loads for the fly-through: (tracker over model_files' ply, key poses from its
    pose_optimized.npy, it).  Like render.py, no Mip-Splatting filters unless kernel_size is given; then the tracker
    applies the 2D filter with it and the ply's filter_3D (load_tracker).  The tracker renders at
    frame_size(resolution, resample_images); ply_io: load_tracker's."""
    ply, npy, it = model_files(model_path, iteration)
    for f in (ply, npy):
        if not os.path.isfile(f):
            raise FileNotFoundError(f"{f} not found")
    _, _, fovx, fovy = intrinsics(source_path, n_views)
    W, H = frame_size(source_path, n_views, resolution, resample_images)
    return load_tracker(ply, W, H, fovx, fovy, white_background, device, kernel_size, ply_io), np.load(npy), it


def load_tracker(path: str, width: int, height: int, fovx: float, fovy: float, white_background: bool = False,
                 device="cuda", kernel_size: Optional[float] = None, ply_io: str = "numpy") -> PoseTracker:
    """A PoseTracker over a saved point_cloud.ply as render.py renders it: the SH degree from the file's coefficient
    count, a black or white background.  No Mip-Splatting filters unless kernel_size is given (a filter_3D property
    in the file is then not used); with it, the 2D filter at kernel_size and the file's filter_3D, which it must
    carry (tracker_from_gaussians).  ply_io "numpy": scene_io.load_gaussians_ply; "gpu": ply.load, the tensors
    unpacked on the device (the same values)."""
    from .scene_io import load_gaussians_ply
    if ply_io == "gpu":
        g = ply.load(path, device)
    elif ply_io == "numpy":
        g = {k: torch.from_numpy(np.ascontiguousarray(a)) for k, a in load_gaussians_ply(path).items()}
    else:
        raise ValueError(f"load_tracker: ply_io must be 'numpy' or 'gpu', got {ply_io!r}")
    return tracker_from_gaussians(g, width, height, fovx, fovy, white_background, device, path, kernel_size)


def tracker_from_gaussians(g, width: int, height: int, fovx: float, fovy: float, white_background: bool = False,
                           device="cuda", where: str = "the model", kernel_size: Optional[float] = None) -> PoseTracker:
    """load_tracker without the file: g holds load_gaussians_ply's tensors (JointTrainer.ply_tensors gives them from a
    trainer).  Tensors already on the device, fp32 and contiguous are shared with the tracker, not copied.
    kernel_size: Mip-Splatting's filters, the 2D one at kernel_size and the 3D one from g["filter_3D"] (a ValueError
    when g has none); None: neither, whatever g holds."""
    M = 1 + g["f_rest"].shape[1]
    deg = int(round(M ** 0.5)) - 1
    if (deg + 1) ** 2 != M:
        raise ValueError(f"{where}: {M} SH coefficients per channel is not a square")
    kw = {}
    if kernel_size is not None:
        why = mip.kernel_refusal(kernel_size)
        if why:
            raise ValueError(why)
        if "filter_3D" not in g:
            raise ValueError(f"{where}: no filter_3D, so there is no 3D filter to apply with kernel_size {kernel_size}")
        kw = dict(kernel_size=float(kernel_size), filter_3D=g["filter_3D"])
    bg = torch.ones(3) if white_background else torch.zeros(3)
    return PoseTracker(g["xyz"], g["rotation"], g["scaling"], g["opacity"], g["f_dc"], g["f_rest"], width, height, fovx,
                       fovy, bg=bg, sh_degree=deg, device=device, **kw)


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(prog="python -m instantsplat_b200.freeview",
                                 description="render.py --infer_video: the interpolated fly-through of a trained model")
    ap.add_argument("-s", "--source_path", required=True)
    ap.add_argument("-m", "--model_path", required=True)
    ap.add_argument("--n_views", type=int, required=True)
    ap.add_argument("--iterations", type=int, default=-1)
    ap.add_argument("--white_background", action="store_true")
    ap.add_argument("--max_batch", type=int, default=4,
                    help="frames per batched forward; scratch grows by about 150 P + 60 H W bytes a frame")
    ap.add_argument("--workers", type=int, default=None, help="PNG encoder threads (default: up to 8)")
    add_png_encoder_arg(ap)
    ap.add_argument("-r", "--resolution", type=int, default=1,
                    help="render at the size the training cameras load at with this -r (needs --resample_images when "
                         "it changes the size)")
    resample.add_arg(ap)
    mip.add_arg(ap)
    ply.add_arg(ap)
    a = ap.parse_args(argv)
    if a.n_views < 2:
        raise SystemExit("--n_views must be at least 2: the fly-through joins consecutive key poses")
    k = mip.kernel_size(a)
    if k is not None:
        why = mip.kernel_refusal(k) or mip.ply_refusal(k, model_files(a.model_path, a.iterations)[0])
        if why:
            raise SystemExit(f"freeview: {why}")
    tracker, keys, it = load(a.source_path, a.model_path, a.n_views, a.iterations, a.white_background, "cuda",
                             a.resolution, resample.requested(a), **({} if k is None else {"kernel_size": k}),
                             **ply.kwargs(a))
    n, folder = fly_through(tracker, keys, it, a.model_path, a.n_views, a.max_batch, a.workers,
                            png_writer(a.png_encoder))
    print(f"{n} frames -> {folder}")
    return 0


def fly_through(tracker: PoseTracker, keys, it: int, model_path: str, n_views: int, max_batch: Optional[int] = None,
                workers: Optional[int] = None, write=write_pngs) -> Tuple[int, str]:
    """What main does after loading: pose/ours_<it>/pose_interpolated.npy from the key poses keys [n, 4, 4]
    (pose_optimized.npy's rows), then the frames through write (write_pngs' signature) to interp/ours_<it>/renders.
    Returns (frames, folder)."""
    path = interpolated_w2c(keys, n_views)
    np.save(os.path.join(model_path, "pose", f"ours_{it}", "pose_interpolated.npy"), path)
    folder = os.path.join(model_path, "interp", f"ours_{it}", "renders")
    return write(frames_u8(tracker, poses_from_w2c(path), max_batch), folder, workers), folder


if __name__ == "__main__":
    sys.exit(main())
