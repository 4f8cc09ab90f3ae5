"""Cost of densify in batched training (DESIGN.md section 4.10) on two workloads: InstantSplat's size (450k Gaussians,
12 views, 512x288, SH 3) and BASELINE configs[2] (1M Gaussians, 12 views, 1920x1080, SH 3).

  * k_preprocess_bwd of a 12-view batch without and with the densification statistics (k_preprocess_bwd<., false,
    true> against <., true, true>, all 12 views counted), from the library's CUDA-event instrumentation (gsb_profile_*),
    the two alternating round by round;
  * ms per view-iteration of a densify-on run (OptimConfig.densify, InstantSplat's prune-only body), sequential step()
    against step_batch at V = 3 and V = 12, with graph replay.  After 24 view-iterations of warm-up, the timed window
    covers iterations 25..72, which hold four densify events (36, 48, 60, 72) and two opacity resets (36, 72) in every
    arm; their selection, rebuilds and the graph captures after them are part of the time.  The prune criteria are
    switched off (min_opacity 0, no screen- or world-size limit), so every event rebuilds the buffers at an unchanged
    Gaussian count and the arms, which take different numbers of Adam steps, keep the same workload.  Each round builds
    fresh trainers and runs the arms one after another; a first round (first-use costs of the torch operations of the
    densify selection, graph pools) is run and discarded.

Prints one JSON line: the GPU, its power limit and the numbers.

    python tools/densify_batch_cost.py [--rounds 2] [--iters 20]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import instantsplat_b200 as I  # noqa: E402
from instantsplat_b200._lib import KERNEL_IDS  # noqa: E402
from instantsplat_b200.scenes import make_config, surface_scene  # noqa: E402
from instantsplat_b200.trainer import JointTrainer, OptimConfig  # noqa: E402

WARMUP, WINDOW = 24, 48


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                              "-i", "0"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        return None


def densify_cfg(**over):
    c = OptimConfig()
    c.densify, c.densify_batches = True, True
    for k, v in over.items():
        setattr(c, k, v)
    return c


def kernel_times(sc, gts, rounds, iters):
    """Median / min / max ms of k_preprocess_bwd per 12-view batch, statistics off and on."""
    tr = JointTrainer(sc, "cuda", gt_images=gts, cfg=densify_cfg(densify_from_iter=10 ** 9, densify_until_iter=10 ** 9))
    tr.headroom = 2.0
    views = list(range(12))
    tr.step_batch(views)                               # sizes the batch frame's binning buffer
    b = tr._batch
    L = I.lib()
    n_ids = len(KERNEL_IDS)
    kid = KERNEL_IDS.index("preprocess_bwd")
    modes = {"off": 0, "on": 12}
    for n in modes.values():
        tr._enqueue_batch(b, tr.gt, False, n)
    torch.cuda.synchronize()
    times = {m: [] for m in modes}
    for _ in range(rounds):
        for m, n in modes.items():
            ms = (ctypes.c_double * n_ids)()
            cnt = (ctypes.c_int64 * n_ids)()
            L.gsb_profile_enable(1)
            for _ in range(iters):
                tr._enqueue_batch(b, tr.gt, False, n)
            torch.cuda.synchronize()
            L.gsb_profile_collect(ms, cnt, n_ids)
            L.gsb_profile_enable(0)
            times[m].append(ms[kid] / max(1, cnt[kid]))
    assert int(b.host_status[1, 1]) == 0, "binning overflow in the timed batches"
    del tr, b
    torch.cuda.empty_cache()
    med = lambda v: sorted(v)[len(v) // 2]
    out = {m: dict(median=round(med(t), 4), min=round(min(t), 4), max=round(max(t), 4)) for m, t in times.items()}
    out["stats_extra_ms"] = round(med(times["on"]) - med(times["off"]), 4)
    return out


def training_times(sc, gts, rounds):
    """ms per view-iteration over the timed window, per arm and round, and the events each arm saw."""
    cfg = lambda: densify_cfg(densify_from_iter=WARMUP, densification_interval=12, opacity_reset_interval=36,
                              min_opacity=0.0, size_threshold=None, scene_extent=1e9)
    arms = {"step": 1, "batch_V3": 3, "batch_V12": 12}
    res = {a: dict(ms_per_view_iter=[]) for a in arms}
    for r in range(rounds + 1):
        for arm, V in arms.items():
            tr = JointTrainer(sc, "cuda", gt_images=gts, cfg=cfg(), use_graph=True)
            batches = [[(k * V + j) % sc.n_views for j in range(V)] for k in range((WARMUP + WINDOW) // V)]

            def run(bs):
                for views in bs:
                    if arm == "step":
                        tr.step(views[0])
                    else:
                        tr.step_batch(views)

            n_warm = WARMUP // V
            run(batches[:n_warm])
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            run(batches[n_warm:])
            torch.cuda.synchronize()
            if r > 0:
                res[arm]["ms_per_view_iter"].append(round((time.perf_counter() - t0) * 1e3 / WINDOW, 4))
            res[arm].update(densified_at=list(tr.densified_at), reset_at=list(tr.reset_at), P_end=tr.P)
            del tr
            torch.cuda.empty_cache()
    for arm in arms:
        if arm != "step":
            res[arm]["speedup_vs_step"] = round(min(res["step"]["ms_per_view_iter"]) /
                                                min(res[arm]["ms_per_view_iter"]), 3)
    return res


def workload(sc, rounds, iters):
    gts = torch.rand(sc.n_views, 3, sc.height, sc.width, generator=torch.Generator().manual_seed(3)).cuda()
    return dict(P=sc.P, views=sc.n_views, W=sc.width, H=sc.height,
                preprocess_bwd_12_views_ms=kernel_times(sc, gts, rounds * 2, iters),
                densify_run=training_times(sc, gts, rounds))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("densify_batch_cost.py measures on the GPU; none is available")
    out = dict(gpu=gpu_info(), rounds=a.rounds, iters=a.iters)
    out["a_eval_450k_12x512x288"] = workload(surface_scene(450_000, 12, 512, 288, seed=1005, sh_degree=3), a.rounds,
                                             a.iters)
    out["b_configs2_1M_12x1920x1080"] = workload(make_config(2), a.rounds, a.iters)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
