"""Cost of adaptive density control (DESIGN.md section 4.8) at the bench workload (configs[2]: 1M Gaussians, 12 views,
1920x1080):

  * k_preprocess_bwd with the densification statistics off and on (gsb_backward_ex vs gsb_backward_stats), from the
    library's CUDA-event instrumentation (gsb_profile_*), off and on alternating round by round;
  * one densify event of JointTrainer on that scene: the selection and row arithmetic alone (densify_plan), the
    whole JointTrainer.densify_and_prune (selection and the one flat-buffer rebuild), and the two steps after it (an
    eager one that sizes the binning buffer, then the capture of a new graph and its first replay), each timed with
    CUDA events, for the prune-only and the clone + split body.

Prints one JSON object.

    python tools/densify_cost.py [--rounds 5] [--iters 20]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    import torch
    import instantsplat_b200 as I
    from instantsplat_b200._lib import KERNEL_IDS, GsbGrads
    from instantsplat_b200.frame import Frame, IdentityView, capacity, densify_stats, gaussians, read_R
    from instantsplat_b200.scenes import make_config
    if not torch.cuda.is_available():
        raise SystemExit("densify_cost.py measures on the GPU; none is available")
    dev = torch.device("cuda")
    L = I.lib()
    sc = make_config(2)
    # ---- 1. the per-Gaussian backward with the statistics off and on
    prm = {k: v.to(dev).float().contiguous() for k, v in sc.params.items()}
    poses = sc.poses.to(dev).float().contiguous()
    iv = IdentityView(sc.width, sc.height, sc.fovx, sc.fovy, sc.bg, dev)
    cam = iv.camera(3, 16)
    g = gaussians(sc.P, prm["xyz"], prm["rotation"], prm["scaling"], prm["opacity"], prm["f_dc"], prm["f_rest"], poses[0])
    fr = Frame(dev, sc.P, sc.width, sc.height)
    status = torch.zeros(8, dtype=torch.int32).pin_memory()
    dL = torch.rand(3, sc.height, sc.width, device=dev) * 1e-6
    grads = {k: torch.empty_like(v) for k, v in prm.items()}
    dpose = torch.empty(7, device=dev)
    gr = GsbGrads()
    for f, k in (("dL_dmeans3D", "xyz"), ("dL_dscales", "scaling"), ("dL_drotations", "rotation"),
                 ("dL_dopacities", "opacity"), ("dL_dsh_dc", "f_dc"), ("dL_dsh_rest", "f_rest")):
        setattr(gr, f, grads[k].data_ptr())
    gr.dL_dpose = dpose.data_ptr()
    acc = torch.zeros(3, sc.P, device=dev)
    modes = {"off": None, "on": densify_stats(fr.radii, acc[0], acc[1], acc[2])}
    fr.preprocess(cam, g, status)
    torch.cuda.synchronize()
    R = read_R(status)
    fr.alloc_binning(capacity(R, 1.2))
    fr.preprocess(cam, g)
    fr.render(cam)
    for st in modes.values():
        fr.backward(cam, g, dL, gr, None, st)
    torch.cuda.synchronize()
    n_ids = len(KERNEL_IDS)
    kid = KERNEL_IDS.index("preprocess_bwd")
    times = {m: [] for m in modes}
    for _ in range(args.rounds):
        for m, st in modes.items():
            ms = (ctypes.c_double * n_ids)()
            cnt = (ctypes.c_int64 * n_ids)()
            L.gsb_profile_enable(1)
            for _ in range(args.iters):
                fr.backward(cam, g, dL, gr, None, st)
            torch.cuda.synchronize()
            L.gsb_profile_collect(ms, cnt, n_ids)
            L.gsb_profile_enable(0)
            times[m].append(ms[kid] / max(1, cnt[kid]))
    del fr, grads
    med = lambda v: sorted(v)[len(v) // 2]
    # ---- 2. one densify event of the trainer
    event = {}
    for body in ("prune_only", "clone_split"):
        cfg = I.OptimConfig()
        cfg.densify = True
        cfg.densify_from_iter = cfg.densify_until_iter = 10 ** 9
        tr = I.JointTrainer(sc, dev, gt_images=torch.rand(sc.n_views, 3, sc.height, sc.width), cfg=cfg,
                            use_graph=True)
        for k in range(4):                               # statistics, Adam moments and a captured graph of view 0
            tr.step(0)
        torch.cuda.synchronize()
        gm = tr.xyz_gradient_accum / tr.denom
        thr = float(torch.quantile(gm[tr.denom > 0][:1 << 24], 0.9))
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        P0 = tr.P
        t0 = time.perf_counter()
        ev[0].record()
        v = lambda name: tr.view(tr.params, name)
        plan = I.densify_plan(v("xyz"), v("scaling"), v("rotation"), v("opacity"), tr.xyz_gradient_accum, tr.denom,
                              tr.max_radii2D, thr, cfg.min_opacity, tr.scene_extent, cfg.size_threshold,
                              cfg.percent_dense, body == "clone_split", tr.densify_generator)
        ev[1].record()
        tr.densify_and_prune(thr, cfg.min_opacity, tr.scene_extent, cfg.size_threshold, body == "clone_split",
                             torch.Generator(device=dev).manual_seed(0))
        ev[2].record()
        tr.step(0)                                       # eager sizing forward (first after the rebuild)
        tr.step(0)                                       # capture + first replay
        ev[3].record()
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
        event[body] = dict(P_before=P0, P_after=tr.P, plan_ms=ev[0].elapsed_time(ev[1]),
                           densify_and_prune_ms=ev[1].elapsed_time(ev[2]),
                           two_steps_after_ms=ev[2].elapsed_time(ev[3]), wall_s=wall, selected=plan.P)
        del tr
        torch.cuda.empty_cache()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(
        gpu=smi, workload=f"configs[2]: P={sc.P}, {sc.n_views} views, {sc.width}x{sc.height}, view 0", instances=R,
        rounds=args.rounds, iters=args.iters,
        preprocess_bwd_ms={m: dict(median=med(t), min=min(t), max=max(t)) for m, t in times.items()},
        stats_extra_ms=med(times["on"]) - med(times["off"]), densify_event=event)))


if __name__ == "__main__":
    main()
