"""Cost of training on V views one optimizer step each (V sequential JointTrainer.step calls) against one optimizer
step over all V (JointTrainer.step_batch), for V in {1, 3, 12}, on two workloads: BASELINE configs[2] (1M Gaussians,
12 views, 1920x1080, SH 3) and InstantSplat's size (450k Gaussians, 12 views, 512x288, SH 3).  Both arms replay CUDA
graphs and alternate over several rounds; each round consumes the same number of views in both.  The two arms take
different optimizer steps for V > 1 (that is the point of the batch), so only the V = 1 arm is checked against step():
after every round its parameters, moments and pose table must equal the sequential arm's.

Prints one JSON line: the GPU, its power limit, and per workload and V the ms per view-iteration of each arm and their
ratio.  Usage: python tools/train_batch_cost.py [--views-per-round 24] [--rounds 3]
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
from instantsplat_b200.trainer import JointTrainer, OptimConfig  # noqa: E402


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
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def state(tr):
    return [tr.params, tr.exp_avg, tr.exp_avg_sq, tr.poses, tr.pose_m, tr.pose_v]


def workload(sc, per_round, rounds):
    n = sc.n_views
    gts = torch.rand(n, 3, sc.height, sc.width, generator=torch.Generator().manual_seed(3)).cuda()
    res = dict(P=sc.P, views=n, W=sc.width, H=sc.height, views_per_round=per_round, rounds=rounds)
    for V in (1, 3, 12):
        cfg = OptimConfig()
        seq = JointTrainer(sc, "cuda", gt_images=gts, cfg=cfg, use_graph=True)
        bat = JointTrainer(sc, "cuda", gt_images=gts, cfg=cfg, use_graph=True)
        batches = [[(k * V + j) % n for j in range(V)] for k in range(per_round // V)]

        def run_seq():
            for views in batches:
                for v in views:
                    seq.step(v)

        def run_bat():
            for views in batches:
                bat.step_batch(views)

        run_seq(), run_bat()                                       # warm-up: graph capture of every key
        t_seq, t_bat, same = [], [], True
        for _ in range(rounds):
            t_seq.append(timed(run_seq))
            t_bat.append(timed(run_bat))
            if V == 1:
                same &= all(torch.equal(a, b) for a, b in zip(state(seq), state(bat)))
        m = len(batches) * V
        r = dict(seq_ms_per_view_iter=[round(t / m, 4) for t in t_seq],
                 batch_ms_per_view_iter=[round(t / m, 4) for t in t_bat],
                 speedup=round(min(t_seq) / min(t_bat), 3))
        if V == 1:
            r["identical_to_step"] = bool(same)
        res[f"V{V}"] = r
        del seq, bat
        torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views-per-round", type=int, default=24, help="a multiple of 12")
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("train_batch_cost.py needs a CUDA device")
    out = dict(gpu=torch.cuda.get_device_name(0), power_limit=power_limit())
    out["a_configs2_1M_12x1920x1080"] = workload(make_config(2), a.views_per_round, a.rounds)
    out["b_eval_450k_12x512x288"] = workload(surface_scene(450_000, 12, 512, 288, seed=1005, sh_degree=3),
                                             a.views_per_round, a.rounds)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
