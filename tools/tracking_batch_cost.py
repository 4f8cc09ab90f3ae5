"""Cost of tracking V test views one after another (PoseTracker.optimize per view) against one batched loop
(PoseTracker.optimize_batch), on two workloads: BASELINE configs[2] (1M Gaussians, 12 views, 1920x1080, SH 3) and
InstantSplat's evaluation size (450k Gaussians, 12 views, 512x288, SH 3).  Targets are renders at the true poses,
tracking starts from seeded perturbations.  The two arms alternate over several rounds; the script checks that their
outputs are identical.  (optimize is the batched loop at V = 1, so the sequential arm is V single-view loops.)

Prints one JSON line: the GPU, its power limit, and per workload ms per view-iteration of each arm and their ratio.
Usage: python tools/tracking_batch_cost.py [--iters 50] [--rounds 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from instantsplat_b200.scenes import make_config, surface_scene  # noqa: E402
from instantsplat_b200.tracking import PoseTracker  # noqa: E402


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30)
        return out.stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        return None


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, (time.perf_counter() - t0) * 1e3


def workload(sc, iters, rounds):
    p = sc.params
    tr = PoseTracker(p["xyz"], p["rotation"], p["scaling"], p["opacity"], p["f_dc"], p["f_rest"], sc.width, sc.height,
                     sc.fovx, sc.fovy, sh_degree=3, device="cuda")
    V = sc.poses.shape[0]
    gts = tr.render_batch(sc.poses)
    g = torch.Generator().manual_seed(7)
    init = sc.poses + 0.01 * torch.randn(sc.poses.shape, generator=g)

    def seq(n=iters):
        outs = [tr.optimize(init[v], gts[v], num_iter=n, return_trace=True) for v in range(V)]
        return (torch.stack([o[0] for o in outs]), torch.tensor([o[1] for o in outs]), torch.stack([o[2] for o in outs]))

    def bat(n=iters):
        return tr.optimize_batch(init, gts, num_iter=n, return_trace=True)

    seq(3), bat(3)                                                  # warm-up: every shape of the timed calls
    t_seq, t_bat, same = [], [], True
    for _ in range(rounds):
        a, ta = timed(seq)
        b, tb = timed(bat)
        same &= all(torch.equal(x, y) for x, y in zip(a, b))
        t_seq.append(ta); t_bat.append(tb)
    n = V * iters
    res = dict(P=tr.P, views=V, W=sc.width, H=sc.height, iters=iters, rounds=rounds, identical=bool(same),
               seq_ms_per_view_iter=[round(t / n, 4) for t in t_seq],
               batch_ms_per_view_iter=[round(t / n, 4) for t in t_bat])
    res["speedup"] = round(min(t_seq) / min(t_bat), 3)
    del tr
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tracking_batch_cost.py needs a CUDA device")
    out = dict(gpu=torch.cuda.get_device_name(0), power_limit=power_limit())
    out["a_configs2_1M_12x1920x1080"] = workload(make_config(2), a.iters, a.rounds)
    out["b_eval_450k_12x512x288"] = workload(surface_scene(450_000, 12, 512, 288, seed=1005, sh_degree=3), a.iters,
                                             a.rounds)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
