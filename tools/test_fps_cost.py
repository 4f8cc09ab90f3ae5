"""Cost of render.py --test_fps's rate, three ways, at BASELINE configs[1] (200k Gaussians, 512x512, SH 0) and
configs[2] (1M Gaussians, 1920x1080, SH 3), on a tracked view: view 0's pose perturbed by 0.01 N(0, 1) and tracked
for --iters iterations (PoseTracker.optimize against the render at its true pose), then timed at the best pose.

  * time_renders: PoseTracker.time_renders (what `render_views --eval --test_fps` reports): a CUDA-graph replay of
    the single-view forward per frame, host clock around each replay and its stream synchronise;
  * render_batch: an eager PoseTracker.render_batch loop, each call sizing its binning buffer from a host copy of the
    instance count (one host wait inside every call), host clock around each call and a synchronise;
  * render_py: render.py:172-179 itself through the drop-in renderer.render(): host clock around each call, no
    synchronise of its own (render() waits for the instance count inside).

Each is render.py's protocol (n = 1000 timed frames, sorted, the mean of [100:900], fps = 1 / mean), repeated
--rounds times with the three ways alternating, after 20 untimed frames of each.  Also: the graph replay's GPU time
per frame from CUDA events over 1000 back-to-back replays, and whether the replayed image equals render_batch's.

Prints one JSON line per measurement and a last one with them all, with the GPU's name and power limit.
Usage: python tools/test_fps_cost.py [--configs 1 2] [--rounds 3] [--iters 500]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import instantsplat_b200 as I  # noqa: E402
from instantsplat_b200.camera import SimpleCamera  # noqa: E402
from instantsplat_b200.render_views import fps_from_times  # noqa: E402
from instantsplat_b200.scenes import make_config  # noqa: E402
from instantsplat_b200.tracking import PoseTracker  # noqa: E402

N = 1000


def device_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                              "-i", "0"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        return None


def log(key, value):
    print(json.dumps({key: value}), flush=True)


def host_times(fn, sync):
    """render.py's loop around fn, n times; sync: a device synchronise inside the timed window after each call."""
    for _ in range(20):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(N):
        t0 = time.perf_counter()
        fn()
        if sync:
            torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    torch.cuda.synchronize()
    return ts


def replay_gpu_ms(tk, pose):
    """GPU time per frame of the captured forward: CUDA events around N back-to-back replays."""
    from instantsplat_b200.frame import Frame
    p = pose.reshape(1, 7).to(tk.dev).contiguous()
    fr = Frame(tk.dev, tk.P, tk.W, tk.H, views=1)
    cam = tk._cam()
    tk._forward_batch(fr, cam, tk._gauss(p), p, True)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fr.preprocess_batch(cam, tk._gauss(p), p, None, tk.filt)
        fr.render_batch(cam)
    for _ in range(20):
        g.replay()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(N):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / N


def run_config(idx, rounds, iters, dev="cuda"):
    sc = make_config(idx)
    prm = {k: v.to(dev) for k, v in sc.params.items()}
    tk = PoseTracker(prm["xyz"], prm["rotation"], prm["scaling"], prm["opacity"], prm["f_dc"], prm["f_rest"], sc.width,
                     sc.height, sc.fovx, sc.fovy, sh_degree=sc.sh_degree, device=dev)
    gt = tk.render(sc.poses[0])
    init = sc.poses[0] + 0.01 * torch.randn(7, generator=torch.Generator().manual_seed(5))
    pose, loss = tk.optimize(init, gt, num_iter=iters)
    r = dict(P=sc.P, W=sc.width, H=sc.height, sh_degree=sc.sh_degree, tracked_loss=round(loss, 6),
             pose_err=round(float((pose - sc.poses[0]).abs().max()), 6))
    img = torch.empty(3, sc.height, sc.width, device=dev)
    tk.time_renders(pose, 1, out=img)
    r["replay_equals_render_batch"] = bool(torch.equal(img, tk.render_batch(pose.reshape(1, 7))[0]))

    model = I.GaussianModel.from_scene(sc, dev)
    cam = SimpleCamera(sc.width, sc.height, sc.fovx, sc.fovy, device=dev)
    pipe, bg = I.PipelineDefaults(), torch.zeros(3, device=dev)
    pose_dev = pose.to(dev)
    p1 = pose.reshape(1, 7)
    ways = {"time_renders": lambda: tk.time_renders(pose, N),
            "render_batch": lambda: host_times(lambda: tk.render_batch(p1), sync=True),
            "render_py": lambda: host_times(lambda: I.render(cam, model, pipe, bg, camera_pose=pose_dev), sync=False)}
    tk.time_renders(pose, 20)
    fps = {k: [] for k in ways}
    ms = {k: [] for k in ways}
    with torch.no_grad():
        for _ in range(rounds):
            for k, fn in ways.items():
                f, _ = fps_from_times(fn())
                fps[k].append(round(f, 1))
                ms[k].append(round(1e3 / f, 4))
    r["fps"], r["trimmed_mean_ms"] = fps, ms
    r["replay_gpu_ms"] = round(replay_gpu_ms(tk, pose), 4)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", type=int, nargs="+", default=[1, 2])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=500)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("test_fps_cost.py needs a CUDA device")
    res = dict(gpu=torch.cuda.get_device_name(0), nvidia_smi=device_info(), host_cpus=os.cpu_count(),
               frames=N, rounds=a.rounds)
    log("device", res)
    for idx in a.configs:
        res[f"configs[{idx}]"] = run_config(idx, a.rounds, a.iters)
        log(f"configs[{idx}]", res[f"configs[{idx}]"])
    print(json.dumps(res))


if __name__ == "__main__":
    main()
