"""Stage-level cost of Mip-Splatting's filters (--kernel_size, DESIGN.md section 4.22): `train` (1000 iterations,
InstantSplat's flags) and `render_views --eval` (500 tracking iterations per test view, then the renders and PNGs), each
with and without --kernel_size 0.1, at
  * BASELINE configs[1]: 200k Gaussians, 3 views, 512x512;
  * BASELINE configs[2]: 1M Gaussians, 12 views, 1920x1080.

The source is scene_io.write_synthetic_source's (the config's points and confidence, PNG images rendered from the
config's Gaussians); its test views (sparse_<n>/1) are the training images at the training poses perturbed by
0.01 N(0, 1).  Each arm trains its own model, and render_views --eval runs on that model with the same flag.  Per
round the two arms alternate (the order swaps every round); each time is end to end on the host clock around work
that ends in a device synchronise, after one warm-up of each arm (20 training iterations, 3 tracking iterations).
train's loop phase (its iterations without the saves) is reported apart.

Prints one JSON line per measurement and a last one with them all, with the GPU, its power limit and max SM clock.
Usage: python tools/mip_stages_cost.py [--iterations 1000] [--rounds 2]
"""
import argparse
import contextlib
import json
import math
import os
import shutil
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from instantsplat_b200 import freeview as F  # noqa: E402
from instantsplat_b200 import render_views as R  # noqa: E402
from instantsplat_b200 import scene_io as S  # noqa: E402
from instantsplat_b200 import train as T  # noqa: E402
from instantsplat_b200.scenes import make_config  # noqa: E402
from instantsplat_b200.tracking import PoseTracker  # noqa: E402

ARMS = {"plain": [], "mip": ["--kernel_size", "0.1"]}


def device_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                              "0"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        return None


def log(key, value):
    print(json.dumps({key: value}), flush=True)


def write_source(sc, root):
    """Training views (sparse_<n>/0, images/<6 digits>.png) and test views (sparse_<n>/1, images/t<3 digits>.png)."""
    p = sc.params
    tk = PoseTracker(p["xyz"], p["rotation"], p["scaling"], p["opacity"], p["f_dc"], p["f_rest"], sc.width, sc.height,
                     sc.fovx, sc.fovy, sh_degree=sc.sh_degree, device="cuda")
    u8 = np.concatenate([c for _, c in F.frames_u8(tk, sc.poses, max_batch=4)])
    del tk
    S.write_synthetic_source(root, sc, u8)
    g = torch.Generator().manual_seed(7)
    init = sc.poses + 0.01 * torch.randn(sc.poses.shape, generator=g)
    names = [f"t{i:03d}.png" for i in range(sc.n_views)]
    fx = sc.width / (2.0 * math.tan(sc.fovx / 2.0))
    fy = sc.height / (2.0 * math.tan(sc.fovy / 2.0))
    S.write_colmap_text(os.path.join(root, f"sparse_{sc.n_views}", "1"), sc.width, sc.height, fx, fy, init.numpy(),
                        names)
    F.write_pngs([(0, u8)], os.path.join(root, "images"), names=names)
    return root


def wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, r


def arm(src, model, n, iterations, track_iters, extra):
    """train, then render_views --eval, into model; returns the times."""
    targs = T.parse_args(["-s", src, "-m", model, "-r", "1", "--n_views", str(n), "--iterations", str(iterations),
                          "--pp_optimizer", "--optim_pose", "--quiet"] + extra)
    t_train, res = wall(lambda: T.run(targs))
    out = dict(train_s=round(t_train, 3), train_loop_s=round(res.phases["loop"], 3),
               train_it_per_s=round(iterations / res.phases["loop"], 1), last_loss=float(res.losses[-1]),
               filter3d_recomputes=len(res.trainer.mip_recomputed_at))
    del res
    torch.cuda.empty_cache()
    argv = ["-s", src, "-m", model, "--n_views", str(n), "--iterations", str(iterations), "--eval", "-r", "1",
            "--optim_test_pose_iter", str(track_iters)] + extra
    with contextlib.redirect_stdout(open(os.devnull, "w")):
        t_render, _ = wall(lambda: R.main(argv))
    out["render_eval_s"] = round(t_render, 3)
    torch.cuda.empty_cache()
    return out


def workload(idx, a):
    sc = make_config(idx)
    res = dict(P=sc.P, views=sc.n_views, W=sc.width, H=sc.height, iterations=a.iterations,
               track_iters=a.track_iters, rounds=[])
    n = sc.n_views
    with tempfile.TemporaryDirectory() as tmp:
        src = write_source(sc, os.path.join(tmp, "src"))
        del sc
        for name, extra in ARMS.items():                                        # warm-up: imports, modules, graphs
            arm(src, os.path.join(tmp, f"warm_{name}"), n, 20, 3, extra)
            shutil.rmtree(os.path.join(tmp, f"warm_{name}"))
        for r in range(a.rounds):
            rnd = {}
            for name in (list(ARMS) if r % 2 == 0 else list(ARMS)[::-1]):
                model = os.path.join(tmp, f"{name}{r}")
                rnd[name] = arm(src, model, n, a.iterations, a.track_iters, ARMS[name])
                shutil.rmtree(model)
            res["rounds"].append(rnd)
            log(f"configs[{idx}] round {r}", rnd)
    for key in ("train_s", "train_loop_s", "render_eval_s"):
        for name in ARMS:
            res[f"{name}_{key}_median"] = statistics.median(x[name][key] for x in res["rounds"])
        res[f"mip_over_plain_{key}"] = round(res[f"mip_{key}_median"] / res[f"plain_{key}_median"], 3)
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iterations", type=int, default=1000)
    ap.add_argument("--track_iters", type=int, default=500)
    ap.add_argument("--rounds", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mip_stages_cost.py needs a CUDA device")
    out = dict(gpu=torch.cuda.get_device_name(0), name_power_limit_max_sm_clock=device_info(),
               host_cpus=os.cpu_count(), rounds=a.rounds)
    log("device", out)
    for idx in (1, 2):
        out[f"configs{idx}"] = workload(idx, a)
        log(f"configs{idx}", out[f"configs{idx}"])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
