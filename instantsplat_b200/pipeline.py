"""InstantSplat's scripts/run_eval.sh and scripts/run_infer.sh from stage 2 on, for a list of scenes, in one process
on one GPU (DESIGN.md section 4.18).

    python -m instantsplat_b200.pipeline eval  --data_root ROOT --output_dir OUT --datasets D.. --scenes S..
        --n_views N.. --iterations IT.. [--lpips_weights DIR] [--workers W] [--png_encoder pil|gpu] [--test_fps]
        [--kernel_size K] [--ply_io numpy|gpu] [--jpeg_decoder pil|gpu]
    python -m instantsplat_b200.pipeline infer --data_root ROOT --output_dir OUT --datasets D.. --scenes S..
        --n_views N.. --iterations IT.. [--workers W] [--png_encoder pil|gpu] [--kernel_size K] [--ply_io numpy|gpu]
        [--jpeg_decoder pil|gpu]

Tasks run in the scripts' loop order (dataset, scene, n_views, iterations), one after another.  The source is
ROOT/D/S/24_views for eval and ROOT/D/S for infer; the model is OUT/D/S/<N>_views.  Each stage is the stage module's
own code on the arguments its own parser makes of the script's line (stage_argv), and writes what its CLI prints to
the log the script redirects it to.  What the stage CLIs read back from the previous stage's files is handed over in
memory instead:

  * train: train.run; its trainer's final Gaussians (JointTrainer.ply_tensors, what point_cloud.ply holds, at the
    stored SH degree) and pose_optimized.npy's rows (scene_io.pose_matrices) are kept, then the trainer is released.
  * training-view renders: render_views.render_train on the train stage's decoded views.
  * test-view renders: render_views.render_test on load_views(split=1), its 8-bit renders and gts kept; with
    --test_fps (render.py's flag on the stage's line, as run_eval.sh's commented-out line would add it), then
    render_views.report_fps at the last test view's best pose, which writes total_fps.json into the model directory.
  * metrics: metrics.evaluate with the current test/ours_<it> from memory, any earlier method from its files.
  * infer: freeview.fly_through.

Like the stage CLIs, the render stages use no Mip-Splatting filter unless --kernel_size K is given.  With it, the
train, render and fly-through lines carry --kernel_size K (metrics scores PNGs and needs nothing), the trainer trains
with both filters, and its filter_3D goes to the trackers with the rest of ply_tensors.  A K that is negative, NaN or
infinite is refused with the other refusals.

--ply_io gpu goes on the train stage's line only: its save points write point_cloud.ply on the GPU (ply.py).  The
render stages get the model in memory and read no ply.

--jpeg_decoder gpu goes on the train line and the test-view renders' line, the two stages that decode source images:
the refusal pass, the train stage and the test views loaded for stage 4 decode their JPEG files on the GPU (jpeg.py),
Pillow's pixels byte for byte.

Every PNG goes to one process-wide encoder pool (PngWriter) that the GPU stages do not wait for, up to a bound on the
frames queued; with --png_encoder gpu the frames are encoded on the GPU and the pool only writes the files.  Every
task is checked before anything is written (refusals).  The scripts' nvidia-smi GPU picker and init_geo (stage 1) are
not part of this.
"""
from __future__ import annotations

import argparse
import contextlib
import gc
import os
import sys
import time
from collections import deque
from concurrent.futures import ThreadPoolExecutor
from dataclasses import dataclass
from typing import Dict, Iterable, List, Optional, Sequence, Tuple

import numpy as np

from . import freeview, jpeg, metrics, mip, ply, png, render_views, train
from .scene_io import load_views, pose_matrices

# stage -> (log file, the script's start line, its completion line)
STAGES = {
    "eval": {"train": ("02_train.log", "Starting training...", "Training completed."),
             "render_train": ("03_render_train.log", "Starting rendering training views...", "Rendering completed."),
             "render_test": ("04_render_test.log", "Starting rendering testing views...", "Rendering completed."),
             "metrics": ("05_metrics.log", "Calculating metrics...", "Metrics calculation completed.")},
    "infer": {"train": ("02_train.log", "Starting training...", "Training completed."),
              "render": ("03_render.log", "Starting rendering training views...", "Rendering completed.")},
}


# ---- tasks ---------------------------------------------------------------------------------------------------
@dataclass
class Task:
    mode: str
    dataset: str
    scene: str
    n_views: int
    iterations: int
    source: str
    model: str

    @property
    def label(self) -> str:
        return f"{self.dataset}/{self.scene} ({self.n_views} views/{self.iterations} iters)"


def tasks(mode: str, data_root: str, output_dir: str, datasets: Sequence[str], scenes: Sequence[str],
          n_views: Sequence[int], iterations: Sequence[int]) -> List[Task]:
    """The scripts' main loop: dataset, then scene, then n_views, then iterations."""
    out = []
    for d in datasets:
        for s in scenes:
            for n in n_views:
                for it in iterations:
                    src = os.path.join(data_root, d, s, "24_views") if mode == "eval" else os.path.join(data_root, d, s)
                    out.append(Task(mode, d, s, int(n), int(it), src, os.path.join(output_dir, d, s, f"{n}_views")))
    return out


def stage_argv(t: Task, lpips_weights: Optional[str] = None, test_fps: bool = False,
               kernel_size: Optional[float] = None, ply_io: Optional[str] = None,
               jpeg_decoder: Optional[str] = None) -> Dict[str, List[str]]:
    """Each stage's command line as the script writes it; test_fps adds --test_fps to the test-view renders';
    kernel_size adds --kernel_size to the train, render and fly-through lines (not to metrics, which scores PNGs);
    ply_io adds --ply_io to the train line; jpeg_decoder adds --jpeg_decoder to the train and test-view render lines."""
    base = ["-s", t.source, "-m", t.model, "-r", "1", "--n_views", str(t.n_views), "--iterations", str(t.iterations)]
    k = mip.argv(kernel_size)
    out = {"train": base + ["--pp_optimizer", "--optim_pose"] + k + ply.argv(ply_io) + jpeg.argv(jpeg_decoder)}
    if t.mode == "eval":
        out["render_train"] = base + k
        out["render_test"] = base + ["--eval"] + (["--test_fps"] if test_fps else []) + k + jpeg.argv(jpeg_decoder)
        out["metrics"] = ["-s", t.source, "-m", t.model, "--n_views", str(t.n_views)] \
            + ([] if lpips_weights is None else ["--lpips_weights", lpips_weights])
    else:
        out["render"] = base + ["--infer_video"] + k
    return out


def stage_args(t: Task, lpips_weights: Optional[str] = None, test_fps: bool = False,
               kernel_size: Optional[float] = None, ply_io: Optional[str] = None,
               jpeg_decoder: Optional[str] = None) -> Dict[str, argparse.Namespace]:
    """stage_argv parsed by each stage's own parser."""
    parse = {"train": train.parse_args, "metrics": lambda a: metrics.parser().parse_args(a)}
    return {k: parse.get(k, lambda a: render_views.parser().parse_args(a))(v)
            for k, v in stage_argv(t, lpips_weights, test_fps, kernel_size, ply_io, jpeg_decoder).items()}


def refusals(t: Task, test_fps: bool = False, kernel_size: Optional[float] = None,
             jpeg_decoder: Optional[str] = None) -> List[str]:
    """Why the task cannot run, each reason with its path; empty when it can.  Reads the source, writes nothing.
    test_fps: the eval task's test-view renders carry --test_fps, which needs a test view; kernel_size: the stages
    carry --kernel_size, which must be a finite number >= 0.  The model the render stages read is the train stage's,
    in memory, and carries filter_3D whenever the train stage has the flag.  jpeg_decoder "gpu": the training views
    are decoded on the GPU, as the train stage will decode them."""
    out = []
    why = mip.kernel_refusal(kernel_size)
    if why:
        out.append(why)
    f0 = os.path.join(t.source, f"sparse_{t.n_views}", "0")
    for name in ("points3D.ply", "confidence_dsp.npy"):
        if not os.path.isfile(os.path.join(f0, name)):
            out.append(f"init_geo output missing: {os.path.join(f0, name)} not found")
    if t.mode == "eval" and not os.path.isdir(os.path.join(t.source, f"sparse_{t.n_views}", "1")):
        out.append(f"the test views are missing: {os.path.join(t.source, f'sparse_{t.n_views}', '1')} not found")
    if t.mode == "infer" and t.n_views < 2:
        out.append("--n_views must be at least 2: the fly-through joins consecutive key poses")
    why = render_views.fps_refusal(t.source, t.n_views) if test_fps and t.mode == "eval" else None
    if why:
        out.append(why)
    if out:
        return out
    a = stage_args(t, kernel_size=kernel_size, jpeg_decoder=jpeg_decoder)["train"]
    out += train.refusals(a)
    try:
        train.load_host_scene(a.source_path, a.n_views, a.resolution, a.images, a.init_scale_from_view_depth,
                              decode_device="cuda" if jpeg.requested(a) else None)
        if t.mode == "infer":
            freeview.intrinsics(t.source, t.n_views)
    except (ValueError, FileNotFoundError) as e:
        out.append(str(e))
    return out


# ---- PNG files -----------------------------------------------------------------------------------------------
class WriteError(RuntimeError):
    """A PNG could not be written; the message names the file."""


class PngWriter:
    """One pool of `workers` PNG encoder threads for a whole run (None: up to 8).  write queues frames and returns
    without waiting for their encodes; at most 4 x workers frames wait, so the host memory they hold stays bounded,
    and write blocks while the queue is full.  A failed write raises WriteError, naming the file, from the first call
    that finds it done (write, wait or close).  encoder "gpu": write encodes each chunk on the GPU (png.encode_host,
    on the current stream) and queues only the file writes."""

    def __init__(self, workers: Optional[int] = None, encoder: str = "pil"):
        self.workers = min(8, os.cpu_count() or 1) if workers is None else int(workers)
        if self.workers < 1:
            raise ValueError("PngWriter: workers must be >= 1")
        if encoder not in ("pil", "gpu"):
            raise ValueError(f"PngWriter: encoder must be 'pil' or 'gpu', got {encoder!r}")
        self.encoder = encoder
        self.cap = 4 * self.workers
        self._pool = ThreadPoolExecutor(max_workers=self.workers)
        self._pending = deque()                     # (future, path) in submission order

    def write(self, frames: Iterable[Tuple[int, np.ndarray]], folder: str, workers: Optional[int] = None,
              names: Optional[Sequence[str]] = None) -> int:
        """freeview.write_pngs' files for the same arguments (workers is the pool's own, the argument is ignored),
        queued.  Returns the number of files."""
        os.makedirs(folder, exist_ok=True)
        count = 0
        for first, chunk in frames:
            files = png.encode_host(chunk) if self.encoder == "gpu" else None
            for i in range(chunk.shape[0]):
                while len(self._pending) >= self.cap:
                    self._finish(*self._pending.popleft())
                path = os.path.join(folder, f"{first + i:05d}.png" if names is None else names[first + i])
                job = (freeview._save_png, chunk[i]) if files is None else (png.write_file, files[i])
                self._pending.append((self._pool.submit(*job, path), path))
                count += 1
            while self._pending and self._pending[0][0].done():
                self._finish(*self._pending.popleft())
        return count

    @staticmethod
    def _finish(fut, path: str) -> None:
        try:
            fut.result()
        except Exception as e:
            raise WriteError(f"writing {path} failed: {type(e).__name__}: {e}") from e

    def wait(self, select=lambda path: True) -> None:
        """Waits for the queued writes whose path select accepts."""
        for fut, path in list(self._pending):
            if select(path):
                self._finish(fut, path)

    def close(self) -> None:
        """Waits for every queued write, then raises the first failure."""
        first = None
        while self._pending:
            try:
                self._finish(*self._pending.popleft())
            except WriteError as e:
                first = first or e
        self._pool.shutdown(wait=True)
        if first is not None:
            raise first


# ---- one task ------------------------------------------------------------------------------------------------
def _say(msg: str) -> None:
    print(f"[{time.strftime('%Y-%m-%d %H:%M:%S')}] {msg}", flush=True)


@contextlib.contextmanager
def _stage(t: Task, key: str, times: Dict[str, float]):
    """The script's lines around a stage; what the stage prints goes to its log, as `> log 2>&1` sends it."""
    log, start, done = STAGES[t.mode][key]
    path = os.path.join(t.model, log)
    _say(start)
    t0 = time.perf_counter()
    with open(path, "w") as f, contextlib.redirect_stdout(f), contextlib.redirect_stderr(f):
        yield
    times[key] = time.perf_counter() - t0
    _say(f"{done} Log saved in {path}")


def run_task(t: Task, pool: PngWriter, lpips_net=None, lpips_weights: Optional[str] = None,
             device="cuda", test_fps: bool = False, kernel_size: Optional[float] = None,
             ply_io: Optional[str] = None, jpeg_decoder: Optional[str] = None) -> Tuple[int, Dict[str, float]]:
    """The script's run_on_gpu from stage 2 on, with test_fps: stage 4 with --test_fps; kernel_size: every stage but
    metrics with --kernel_size (the trainer's filter_3D handed to the trackers); ply_io: the train stage with
    --ply_io; jpeg_decoder: the train stage and the test views with --jpeg_decoder.  Returns (model directories
    metrics could not evaluate, wall seconds per stage).  The trainer and trackers are released before it returns."""
    a = stage_args(t, lpips_weights, test_fps, kernel_size, ply_io, jpeg_decoder)
    times, failed = {}, 0
    print("=" * 55)
    print(f"Starting process: {t.label}")
    print("=" * 55, flush=True)
    os.makedirs(t.model, exist_ok=True)
    with _stage(t, "train", times):
        res = train.run(a["train"], device, log=print)
        g = res.trainer.ply_tensors()
        keys = pose_matrices(res.trainer.poses.detach().cpu().numpy(), res.colmap_ids)
        views = res.host.views
        del res
        gc.collect()                                # the trainer, its graphs and scratch
    it = t.iterations
    tracker = lambda v, r: freeview.tracker_from_gaussians(g, v.width, v.height, v.fovx, v.fovy, r.white_background,
                                                           device, kernel_size=mip.kernel_size(r))
    if t.mode == "infer":
        r = a["render"]
        with _stage(t, "render", times):
            W, H, fovx, fovy = freeview.intrinsics(t.source, t.n_views)
            tk = freeview.tracker_from_gaussians(g, W, H, fovx, fovy, r.white_background, device,
                                                 kernel_size=mip.kernel_size(r))
            n, folder = freeview.fly_through(tk, keys, it, t.model, t.n_views, r.max_batch, write=pool.write)
            print(f"{n} frames -> {folder}")
    else:
        r = a["render_train"]
        with _stage(t, "render_train", times):
            out = os.path.join(t.model, "train", f"ours_{it}")
            render_views.render_train(tracker(views, r), views, keys, out, r.max_batch,
                                      write=pool.write)
            print(f"{len(views)} views -> {out}")
        r = a["render_test"]
        held = {}

        def keep(frames, folder, workers=None, names=None):
            held[folder] = np.concatenate([c for _, c in frames])
            return pool.write([(0, held[folder])], folder, workers, names)

        with _stage(t, "render_test", times):
            views = load_views(t.source, t.n_views, 1, r.resolution,
                               decode_device=device if jpeg.requested(r) else None)
            out = os.path.join(t.model, "test", f"ours_{it}")
            tk = tracker(views, r)
            start = time.time()
            best = render_views.render_test(tk, views, out, r.optim_test_pose_iter, r.max_batch, write=keep)
            if r.test_fps:
                render_views.report_fps(tk, best[-1], t.model, start)
            del tk
            print(f"{len(views)} views -> {out}")
        names = [n + ".png" for n in views.names]
        order = sorted(range(len(names)), key=names.__getitem__)         # metrics pairs the files in sorted order
        pairs = (held[os.path.join(out, "renders")][order], held[os.path.join(out, "gt")][order],
                 [names[i] for i in order])
        del held, views
        m = a["metrics"]
        with _stage(t, "metrics", times):
            test_dir = os.path.join(t.model, "test") + os.sep
            pool.wait(lambda p: p.startswith(test_dir) and not p.startswith(out + os.sep))    # earlier methods' files
            failed = metrics.evaluate(m.model_paths, m.source_path, m.n_views, device, lpips_net,
                                      held={f"ours_{it}": pairs})
    del g
    gc.collect()
    print("=" * 55)
    print(f"Task completed: {t.label}")
    print("=" * 55, flush=True)
    return failed, times


def run_tasks(ts: Sequence[Task], workers: Optional[int] = None, lpips_net=None, lpips_weights: Optional[str] = None,
              device="cuda", png_encoder: str = "pil", test_fps: bool = False,
              kernel_size: Optional[float] = None, ply_io: Optional[str] = None,
              jpeg_decoder: Optional[str] = None) -> Tuple[int, List[Dict[str, float]]]:
    """Every task in order on one encoder pool (PngWriter with png_encoder), then every write waited for; test_fps,
    kernel_size, ply_io and jpeg_decoder: run_task's.  Returns (model directories metrics could not evaluate,
    per-task stage times).  Raises WriteError when a PNG could not be written."""
    pool = PngWriter(workers, png_encoder)
    failed, times = 0, []
    try:
        for k, t in enumerate(ts, 1):
            print(f"Processing task {k} / {len(ts)}", flush=True)
            f, s = run_task(t, pool, lpips_net, lpips_weights, device, test_fps, kernel_size, ply_io, jpeg_decoder)
            failed += f
            times.append(s)
    finally:
        pool.close()
    return failed, times


# ---- the command line ----------------------------------------------------------------------------------------
def parser() -> argparse.ArgumentParser:
    ap = argparse.ArgumentParser(prog="python -m instantsplat_b200.pipeline",
                                 description="run_eval.sh / run_infer.sh from stage 2 on, for a list of scenes, in one "
                                             "process on one GPU")
    sub = ap.add_subparsers(dest="mode", required=True)
    for mode, what in (("eval", "train, render the training and test views, metrics (run_eval.sh)"),
                       ("infer", "train, render the fly-through (run_infer.sh)")):
        p = sub.add_parser(mode, help=what, description=what)
        p.add_argument("--data_root", required=True, help="eval: ROOT/D/S/24_views is the source; infer: ROOT/D/S")
        p.add_argument("--output_dir", required=True, help="the model of a task is OUTPUT_DIR/D/S/<N>_views")
        p.add_argument("--datasets", nargs="+", required=True)
        p.add_argument("--scenes", nargs="+", required=True)
        p.add_argument("--n_views", nargs="+", type=int, required=True)
        p.add_argument("--iterations", nargs="+", type=int, required=True)
        if mode == "eval":
            p.add_argument("--lpips_weights", metavar="DIR", default=None, help="as metrics --lpips_weights")
            p.add_argument("--test_fps", action="store_true", help="render.py --test_fps on the test-view renders: "
                                                                    "each task's rate appended to total_fps.json")
        p.add_argument("--workers", type=int, default=None, help="PNG encoder threads for the whole run (default: up "
                                                                  "to 8)")
        freeview.add_png_encoder_arg(p)
        mip.add_arg(p)
        ply.add_arg(p)
        jpeg.add_arg(p)
    return ap


def main(argv=None) -> int:
    ap = parser()
    a = ap.parse_args(argv)
    if a.workers is not None and a.workers < 1:
        ap.error("--workers must be at least 1")
    weights, test_fps = getattr(a, "lpips_weights", None), getattr(a, "test_fps", False)
    k = mip.kernel_size(a)
    ts = tasks(a.mode, a.data_root, a.output_dir, a.datasets, a.scenes, a.n_views, a.iterations)
    dec = jpeg.decoder(a)
    bad = [f"{t.label}: {r}" for t in ts for r in refusals(t, test_fps, k, dec)]
    if bad:
        raise SystemExit("\n".join(f"instantsplat_b200.pipeline: {b}" for b in bad))
    net = None
    if weights is not None:
        from . import lpips as LP
        try:
            net = LP.LpipsVGG.from_dir(weights, "cuda")
        except (OSError, ValueError) as e:
            ap.error(str(e))
    try:
        failed, _ = run_tasks(ts, a.workers, net, weights, png_encoder=a.png_encoder, test_fps=test_fps,
                              kernel_size=k, ply_io=ply.io(a), jpeg_decoder=dec)
    except WriteError as e:
        raise SystemExit(f"instantsplat_b200.pipeline: {e}")
    print("=" * 55)
    print(f"All tasks completed! Processed {len(ts)} tasks in total.")
    print("=" * 55)
    return 1 if failed else 0


if __name__ == "__main__":
    sys.exit(main())
