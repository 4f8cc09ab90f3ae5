"""Cost of render.py --eval (run_eval.sh stage 4: track every test view, render it at its best pose, write the render
and gt PNGs) through `python -m instantsplat_b200.render_views --eval`, against a render.py-shaped loop, at
  * BASELINE configs[2]: 1M Gaussians, 12 views, 1920x1080, SH 3;
  * InstantSplat's evaluation size: surface_scene 450k Gaussians, 12 views, 512x288, SH 3.

The test views' images are renders at the scene's poses; sparse_<n>/1 lists the poses perturbed by 0.01 N(0, 1).
Per workload:
  * cli_s: main(["--eval", ...]) end to end from files on disk, and its parts, each timed on its own (host clock
    around work that ends in a device synchronise): load (views decoded, ply read, tracker built), track
    (optimize_batch), render (the batched forward at the best poses, CUDA events), quantise (gsb_frames_u8_batch,
    CUDA events), copy (one device-to-host copy of the 8-bit frames into pinned memory, CUDA events) and png (the
    24 render and gt files on --workers threads);
  * render_py_loop: render.py:113-170 for --loop-views views (drop-in render() with a grad-carrying camera_pose,
    torch.optim.Adam, CosineAnnealingLR, l1_loss_mask, the candidate rule, then render() and save_image of render and
    gt), scaled to all views.

Prints one JSON line per measurement and a last one with them all, with the GPU and its power limit and SM clock.
Usage: python tools/render_views_cost.py [--iters 500] [--loop-views 2] [--workers 8]
"""
import argparse
import json
import math
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
from instantsplat_b200 import render_views as R  # noqa: E402
from instantsplat_b200 import scene_io as S  # noqa: E402
from instantsplat_b200.camera import SimpleCamera  # noqa: E402
from instantsplat_b200.scenes import make_config, surface_scene  # noqa: E402
from instantsplat_b200.tracking import PoseTracker  # noqa: E402


def device_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                              "0"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        return None


def log(key, value):
    print(json.dumps({key: value}), flush=True)


def wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, r


def events(fn, iters=1):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def write_inputs(sc, root):
    """source/sparse_<n>/1 + images/ (the test views) and model/point_cloud/iteration_1000/point_cloud.ply."""
    src, model = os.path.join(root, "src"), os.path.join(root, "model")
    p = sc.params
    tk = PoseTracker(p["xyz"], p["rotation"], p["scaling"], p["opacity"], p["f_dc"], p["f_rest"], sc.width, sc.height,
                     sc.fovx, sc.fovy, sh_degree=3, device="cuda")
    u8 = np.concatenate([c for _, c in F.frames_u8(tk, sc.poses, max_batch=4)])
    del tk
    g = torch.Generator().manual_seed(7)
    init = sc.poses + 0.01 * torch.randn(sc.poses.shape, generator=g)
    names = [f"{i:06d}.png" for i in range(sc.n_views)]
    fx = sc.width / (2.0 * math.tan(sc.fovx / 2.0))
    fy = sc.height / (2.0 * math.tan(sc.fovy / 2.0))
    S.write_colmap_text(os.path.join(src, f"sparse_{sc.n_views}", "1"), sc.width, sc.height, fx, fy, init.numpy(), names)
    F.write_pngs([(0, u8)], os.path.join(src, "images"), names=names)
    q = {k: v.numpy() for k, v in p.items()}
    S.save_gaussians_ply(os.path.join(model, "point_cloud", "iteration_1000", "point_cloud.ply"), q["xyz"], q["f_dc"],
                         q["f_rest"], q["opacity"], q["scaling"], q["rotation"])
    return src, model


def render_py_loop(sc, views, n_views, iters, out):
    """render.py:113-170 on the drop-in render() for the first n_views views."""
    import torchvision
    dev = "cuda"
    model = I.GaussianModel.from_scene(sc, dev)
    for t in (model._xyz, model._features_dc, model._features_rest, model._opacity, model._scaling, model._rotation):
        t.requires_grad_(False)
    cam = SimpleCamera(views.width, views.height, views.fovx, views.fovy, device=dev)
    pipe, bg = I.PipelineDefaults(), torch.zeros(3, device=dev)
    init = F.poses_from_w2c(views.w2c).to(dev)
    gts = R.gt_images(views, dev)
    os.makedirs(out, exist_ok=True)
    for v in range(n_views):
        T = init[v, 4:].clone().requires_grad_()
        q = init[v, :4].clone().requires_grad_()
        opt = torch.optim.Adam([{"params": [T], "lr": 0.003}, {"params": [q], "lr": 0.001}], betas=(0.9, 0.999),
                               weight_decay=1e-4)
        sched = torch.optim.lr_scheduler.CosineAnnealingLR(opt, T_max=iters, eta_min=0.0001)
        cq, cT, best = q.clone().detach(), T.clone().detach(), float(1e20)
        for _ in range(iters):
            img = I.render(cam, model, pipe, bg, camera_pose=torch.cat([q, T]))["render"]
            mask = (img > 0.0).float()
            loss = (torch.abs(img - gts[v]) * mask).sum() / mask.sum()
            loss.backward()
            with torch.no_grad():
                opt.step()
                opt.zero_grad(set_to_none=True)
                if loss < best:
                    best = loss
                    cq, cT = q.clone().detach(), T.clone().detach()
            sched.step()
        with torch.no_grad():
            img = I.render(cam, model, pipe, bg, camera_pose=torch.cat([cq, cT]))["render"]
        torchvision.utils.save_image(img, os.path.join(out, f"r{v}.png"))
        torchvision.utils.save_image(gts[v], os.path.join(out, f"g{v}.png"))


def workload(sc, a):
    res = dict(P=sc.P, views=sc.n_views, W=sc.width, H=sc.height, sh_degree=3, iters=a.iters, workers=a.workers)
    with tempfile.TemporaryDirectory() as tmp:
        src, model = write_inputs(sc, tmp)
        n = sc.n_views
        cli = lambda iters: R.main(["-s", src, "-m", model, "--n_views", str(n), "--iterations", "1000", "--eval",
                                    "-r", "1", "--optim_test_pose_iter", str(iters), "--max_batch", str(n),
                                    "--workers", str(a.workers)])
        cli(3)                                                                       # warm-up
        t_cli, _ = wall(lambda: cli(a.iters))
        res["cli_s"] = round(t_cli, 3)

        def load():
            v = S.load_views(src, n, 1, 1)
            return v, R.tracker_for(model, 1000, v)
        t_load, (views, tk) = wall(load)
        res["load_s"] = round(t_load, 3)
        t_track, best = wall(lambda: R.track(tk, views, a.iters, n))
        res["track_s"] = round(t_track, 3)
        res["track_ms_per_view_iter"] = round(t_track * 1e3 / (n * a.iters), 4)
        best = best.to("cuda")
        tk.render_batch(best)
        res["render_ms"] = round(events(lambda: tk.render_batch(best), 5), 3)
        imgs = tk.render_batch(best)
        u8 = torch.empty(n, sc.height, sc.width, 3, dtype=torch.uint8, device="cuda")
        F.quantise(imgs, u8)
        res["quantise_ms"] = round(events(lambda: F.quantise(imgs, u8), 20), 4)
        host = torch.empty(n, sc.height, sc.width, 3, dtype=torch.uint8).pin_memory()
        host.copy_(u8)
        res["copy_ms"] = round(events(lambda: host.copy_(u8, non_blocking=True), 10), 3)
        frames = host.numpy()
        t0 = time.perf_counter()
        F.write_pngs([(0, frames)], os.path.join(tmp, "png_r"), a.workers)
        F.write_pngs([(0, views.images)], os.path.join(tmp, "png_g"), a.workers)
        res["png_s"] = round(time.perf_counter() - t0, 3)
        del tk
        torch.cuda.empty_cache()
        render_py_loop(sc, views, 1, 3, os.path.join(tmp, "warm"))                 # warm-up
        t_ref, _ = wall(lambda: render_py_loop(sc, views, a.loop_views, a.iters, os.path.join(tmp, "ref")))
        res["render_py_loop_s_per_view"] = round(t_ref / a.loop_views, 3)
        res["render_py_loop_s_extrapolated"] = round(t_ref / a.loop_views * n, 2)
        res["cli_speedup"] = round(t_ref / a.loop_views * n / t_cli, 2)
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=500)
    ap.add_argument("--loop-views", type=int, default=2, help="views timed in the render.py-shaped loop")
    ap.add_argument("--workers", type=int, default=8)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("render_views_cost.py needs a CUDA device")
    out = dict(gpu=torch.cuda.get_device_name(0), power_limit_and_max_sm_clock=device_info(), host_cpus=os.cpu_count())
    log("device", out)
    out["a_configs2_1M_12x1920x1080"] = workload(make_config(2), a)
    log("a", out["a_configs2_1M_12x1920x1080"])
    out["b_eval_450k_12x512x288"] = workload(surface_scene(450_000, 12, 512, 288, seed=1005, sh_degree=3), a)
    log("b", out["b_eval_450k_12x512x288"])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
