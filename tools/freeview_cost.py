"""Cost of the free-view fly-through (render.py --infer_video) at BASELINE configs[2] (1M Gaussians, 1920x1080, SH 3),
with the first 3 and all 12 of its views as key poses (201 and 276 frames):

  * gpu_ms_per_frame: batched forward + gsb_frames_u8_batch per frame at max_batch 1, 4 and 16 (CUDA events around
    the chunk loop, no device-to-host copy);
  * stream_ms_per_frame: frames_u8 end to end (the same, plus the pinned-ring copies and the host arrays);
  * quantise: gsb_frames_u8_batch alone on 16 frames, against its HBM floor of 15 bytes per pixel at 3.35 TB/s;
  * d2h_ms: one chunk's device-to-host copy into pinned memory at 1, 4 and 16 frames;
  * png_fps: write_pngs at 1, 4 and 8 workers on 48 rendered frames;
  * cli_s against the render.py-shaped loop: `python -m instantsplat_b200.freeview` (main(), from the ply on disk,
    all frames) against drop-in render() and torchvision.utils.save_image per frame on the same model and poses, timed
    over the first --loop-frames frames and scaled to all of them;
  * test_fps: render.py's --test_fps protocol (1000 timed calls, sorted, mean of [100:900]) for the drop-in render()
    and PoseTracker.render.

Prints one JSON line with the GPU and its power limit.  Usage: python tools/freeview_cost.py [--views 3 12]
"""
import argparse
import dataclasses
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import instantsplat_b200 as I  # noqa: E402
from instantsplat_b200 import freeview as F  # noqa: E402
from instantsplat_b200.camera import SimpleCamera  # noqa: E402
from instantsplat_b200.scene_io import save_gaussians_ply, save_pose_npy, write_synthetic_source  # noqa: E402
from instantsplat_b200.scenes import make_config  # noqa: E402
from instantsplat_b200.tracking import PoseTracker  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30)
        return out.stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        return None


def log(key, value):
    """One partial result per line as it is measured; the last line holds them all."""
    print(json.dumps({key: value}), flush=True)


def events(fn, iters=1):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, r


def gpu_loop(tk, poses, B):
    """Forward + quantise over all poses in chunks of B, on the current stream (frames_u8 without the copies)."""
    out = torch.empty(B, tk.H, tk.W, 3, dtype=torch.uint8, device=tk.dev)
    cam = tk._cam()
    for v0 in range(0, poses.shape[0], B):
        p = poses[v0:v0 + B]
        fr = tk._frame_batch(p.shape[0])
        tk._forward_batch(fr, cam, tk._gauss(p), p, True)
        F.quantise(fr.color, out[:p.shape[0]])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, nargs="+", default=[3, 12])
    ap.add_argument("--png-frames", type=int, default=48)
    ap.add_argument("--loop-frames", type=int, default=40, help="frames timed in the render.py-shaped loop")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("freeview_cost.py needs a CUDA device")
    dev = "cuda"
    sc = make_config(2)
    H, W = sc.height, sc.width
    prm = {k: v.to(dev) for k, v in sc.params.items()}
    tk = PoseTracker(prm["xyz"], prm["rotation"], prm["scaling"], prm["opacity"], prm["f_dc"], prm["f_rest"], W, H,
                       sc.fovx, sc.fovy, sh_degree=3, device=dev)
    model = I.GaussianModel.from_scene(sc, dev)
    cam = SimpleCamera(W, H, sc.fovx, sc.fovy, device=dev)
    pipe, bg = I.PipelineDefaults(), torch.zeros(3, device=dev)
    res = dict(gpu=torch.cuda.get_device_name(0), power_limit=power_limit(), P=sc.P, W=W, H=H, sh_degree=3)
    log("device", res)

    with tempfile.TemporaryDirectory() as tmp:
        keys_all = save_pose_npy(os.path.join(tmp, "keys.npy"), sc.poses.numpy())
        per_views = {}
        for n in a.views:
            keys = keys_all[:n]
            poses = F.poses_from_w2c(F.interpolated_w2c(keys, n)).to(dev)
            N = poses.shape[0]
            r = dict(frames=N, gpu_ms_per_frame={}, stream_ms_per_frame={})
            for B in (1, 4, 16):
                gpu_loop(tk, poses[:B], B)                                   # warm-up at this chunk size
                r["gpu_ms_per_frame"][B] = round(events(lambda: gpu_loop(tk, poses, B)) / N, 3)
                t, _ = wall(lambda: sum(c.shape[0] for _, c in F.frames_u8(tk, poses, max_batch=B)))
                r["stream_ms_per_frame"][B] = round(t * 1e3 / N, 3)
            # the CLI from files on disk against a render.py-shaped loop, same model and key poses
            src, mdir = os.path.join(tmp, f"src{n}"), os.path.join(tmp, f"model{n}")
            write_synthetic_source(src, dataclasses.replace(sc, poses=sc.poses[:n].clone()))
            p = {k: v.numpy() for k, v in sc.params.items()}
            save_gaussians_ply(os.path.join(mdir, "point_cloud", "iteration_1000", "point_cloud.ply"), p["xyz"],
                               p["f_dc"], p["f_rest"], p["opacity"], p["scaling"], p["rotation"])
            os.makedirs(os.path.join(mdir, "pose", "ours_1000"))
            np.save(os.path.join(mdir, "pose", "ours_1000", "pose_optimized.npy"), keys)
            log(f"views{n}_gpu", r)
            t_cli, _ = wall(lambda: F.main(["-s", src, "-m", mdir, "--n_views", str(n), "--iterations", "1000",
                                            "--max_batch", "16"]))
            r["cli_s"] = round(t_cli, 3)
            import torchvision
            out = os.path.join(tmp, f"ref{n}")
            os.makedirs(out)

            def render_py_loop():
                for i in range(a.loop_frames):
                    with torch.no_grad():
                        img = I.render(cam, model, pipe, bg, camera_pose=poses[i])["render"]
                    torchvision.utils.save_image(img, os.path.join(out, f"{i:05d}.png"))
            t_ref, _ = wall(render_py_loop)
            r["render_py_loop_s_per_frame"] = round(t_ref / a.loop_frames, 4)
            r["render_py_loop_s_extrapolated"] = round(t_ref / a.loop_frames * N, 2)
            r["cli_speedup"] = round(t_ref / a.loop_frames * N / t_cli, 2)
            per_views[n] = r
            log(f"views{n}", r)
        res["views"] = per_views

        # the quantise kernel alone, 16 frames
        imgs = tk.render_batch(poses[:16])
        u8 = torch.empty(16, H, W, 3, dtype=torch.uint8, device=dev)
        F.quantise(imgs, u8)
        ms = events(lambda: F.quantise(imgs, u8), 200)
        nbytes = 16 * H * W * 15
        res["quantise"] = dict(frames=16, ms=round(ms, 4), hbm_floor_ms=round(nbytes / HBM_BYTES_PER_S * 1e3, 4),
                               TB_per_s=round(nbytes / (ms * 1e-3) / 1e12, 3),
                               share_of_floor=round(nbytes / HBM_BYTES_PER_S * 1e3 / ms, 3))
        log("quantise", res["quantise"])
        # one chunk's device-to-host copy
        res["d2h_ms"] = {}
        for B in (1, 4, 16):
            host = torch.empty(B, H, W, 3, dtype=torch.uint8).pin_memory()
            host.copy_(u8[:B])
            res["d2h_ms"][B] = round(events(lambda: host.copy_(u8[:B], non_blocking=True), 20), 3)
        # PNG encode
        frames = u8[:16].cpu().numpy()
        frames = np.concatenate([frames] * ((a.png_frames + 15) // 16))[:a.png_frames]
        res["png_fps"] = {}
        for w in (1, 4, 8):
            d = os.path.join(tmp, f"png{w}")
            t0 = time.perf_counter()
            F.write_pngs([(0, frames)], d, workers=w)
            res["png_fps"][w] = round(len(frames) / (time.perf_counter() - t0), 2)
        res["host_cpus"] = os.cpu_count()
        log("png_fps", res["png_fps"])

    # render.py --test_fps: 1000 calls timed on the host as render.py times them (no synchronise of its own)
    pose = poses[0]

    def test_fps(fn):
        for _ in range(20):
            fn()
        ts = []
        for _ in range(1000):
            t0 = time.perf_counter()
            fn()
            ts.append(time.perf_counter() - t0)
        ts = sorted(ts)[100:900]
        return round(1.0 / (sum(ts) / len(ts)), 1)

    with torch.no_grad():
        res["test_fps"] = dict(dropin_render=test_fps(lambda: I.render(cam, model, pipe, bg, camera_pose=pose)),
                               tracker_render=test_fps(lambda: tk.render(pose)))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
