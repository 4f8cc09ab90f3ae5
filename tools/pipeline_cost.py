"""Wall time of run_eval.sh's and run_infer.sh's stages 2 onward on one GPU, two ways, on the same tasks:
  * scripts: each stage's CLI as its own sequential subprocess (`python -m instantsplat_b200.train`, `render_views`,
    `render_views --eval`, `metrics`; infer: `train`, `render_views --infer_video`), as run_eval.sh runs them on one
    GPU, each paying its own interpreter, torch import, CUDA context, library load, image decode and ply read;
  * pipeline: one `instantsplat_b200.pipeline` process over the same tasks (the trained model handed over on the
    GPU, PNG encoding on one pool overlapped with the GPU stages).
Both are timed from the first task's start to the last file written (the newest mtime under the output directory,
which is also each process's end, since both wait for their writes), with wall seconds per stage: per subprocess for
the scripts, per in-process stage for the pipeline.

Tasks: dataset D, scenes C1a and C1b at BASELINE configs[1] (200k Gaussians, 3 views, 512x512) and C2 at configs[2]
(1M Gaussians, 12 views, 1920x1080), 1000 iterations; sources are written by scene_io.write_synthetic_source with
images rendered from the config's Gaussians, 12 test views at perturbed poses and a sparse/0/images.bin.  Prints JSON
lines, the last one holding everything, with the GPU's name and power limit read in the same run.
Usage: python tools/pipeline_cost.py [--iterations 1000] [--workers 8] [--modes eval infer]
"""
import argparse
import dataclasses
import json
import math
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from instantsplat_b200 import freeview as F  # noqa: E402
from instantsplat_b200 import pipeline as P  # noqa: E402
from instantsplat_b200 import scene_io as S  # noqa: E402
from instantsplat_b200.scenes import make_config  # noqa: E402
from instantsplat_b200.tracking import PoseTracker  # noqa: E402

SCENES = (("C1a", 1), ("C1b", 1), ("C2", 2))
N_TEST = 12


def device_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                              "0"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        return None


def log(key, value):
    print(json.dumps({key: value}), flush=True)


def write_source(idx, root):
    """An init_geo-shaped source of configs[idx]: training views, N_TEST test views in sparse_<n>/1, images.bin."""
    sc = make_config(idx)
    p = sc.params
    tk = PoseTracker(p["xyz"], p["rotation"], p["scaling"], p["opacity"], p["f_dc"], p["f_rest"], sc.width, sc.height,
                     sc.fovx, sc.fovy, sh_degree=3, device="cuda")
    n = sc.n_views
    S.write_synthetic_source(root, sc)
    u8 = np.concatenate([c for _, c in F.frames_u8(tk, sc.poses, max_batch=4)])
    F.write_pngs([(0, u8)], os.path.join(root, "images"), names=[f"{i:06d}.png" for i in range(n)])
    g = torch.Generator().manual_seed(4)
    test = sc.poses[torch.arange(N_TEST) % n] + 0.02 * torch.randn(N_TEST, 7, generator=g)
    names = [f"t{i:02d}.png" for i in range(N_TEST)]
    F.write_pngs(F.frames_u8(tk, test, max_batch=4), os.path.join(root, "images"), names=names)
    fx = sc.width / (2.0 * math.tan(sc.fovx / 2.0))
    fy = sc.height / (2.0 * math.tan(sc.fovy / 2.0))
    init = test + torch.tensor([0.0, 0.004, -0.003, 0.002, 0.01, -0.008, 0.012])
    S.write_colmap_text(os.path.join(root, f"sparse_{n}", "1"), sc.width, sc.height, fx, fy, init.numpy(), names)
    gt = np.concatenate([np.tile([1.0, 0, 0, 0], (24, 1)), np.random.default_rng(5).standard_normal((24, 3))], axis=1)
    gt[S.split_train_test(list(range(24)), n)[0]] = sc.poses.numpy()
    S.write_colmap_images_bin(os.path.join(root, "sparse", "0", "images.bin"), gt, [f"{i:03d}.png" for i in range(24)])
    del tk
    torch.cuda.empty_cache()
    return dict(P=sc.P, views=n, W=sc.width, H=sc.height, test_views=N_TEST)


def last_file(folder):
    return max(os.path.getmtime(os.path.join(d, f)) for d, _, fs in os.walk(folder) for f in fs)


def scripts_way(ts):
    """Each stage's CLI as a subprocess, one after another, its output in the script's log file."""
    mods = {"train": "train", "render_train": "render_views", "render_test": "render_views", "metrics": "metrics",
            "render": "render_views"}
    times = []
    for t in ts:
        os.makedirs(t.model, exist_ok=True)
        st = {}
        for key, argv in P.stage_argv(t).items():
            with open(os.path.join(t.model, P.STAGES[t.mode][key][0]), "w") as f:
                t0 = time.perf_counter()
                subprocess.run([sys.executable, "-m", f"instantsplat_b200.{mods[key]}", *argv], cwd=ROOT, stdout=f,
                               stderr=subprocess.STDOUT, check=True)
                st[key] = round(time.perf_counter() - t0, 3)
        times.append(st)
    return times


def child(spec):
    """The pipeline process: run_tasks over the spec's tasks, its stage times to spec['times']."""
    a = json.loads(spec)
    failed, times = P.run_tasks([P.Task(**t) for t in a["tasks"]], a["workers"])
    with open(a["times"], "w") as f:
        json.dump([{k: round(v, 3) for k, v in s.items()} for s in times], f)
    return 1 if failed else 0


def measure(mode, root, tmp, views, a):
    """Both ways over the same tasks (each scene at its config's view count), the scripts' way first."""
    res = {}
    for way in ("scripts", "pipeline"):
        out = os.path.join(tmp, f"{mode}_{way}")
        ts = [t for name, idx in SCENES for t in P.tasks(mode, root, out, ["D"], [name], [views[idx]], [a.iterations])]
        start = time.time()
        if way == "scripts":
            times = scripts_way(ts)
        else:
            spec = dict(tasks=[dataclasses.asdict(t) for t in ts], workers=a.workers,
                        times=os.path.join(tmp, f"{mode}_times.json"))
            subprocess.run([sys.executable, os.path.abspath(__file__), "--child", json.dumps(spec)], cwd=ROOT,
                           stdout=subprocess.DEVNULL, check=True)
            times = json.load(open(spec["times"]))
        res[way] = dict(wall_s=round(last_file(out) - start, 3),
                        stages_s={f"{t.scene} ({t.n_views} views)": s for t, s in zip(ts, times)})
    res["speedup"] = round(res["scripts"]["wall_s"] / res["pipeline"]["wall_s"], 2)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iterations", type=int, default=1000)
    ap.add_argument("--workers", type=int, default=8)
    ap.add_argument("--modes", nargs="+", default=["eval", "infer"], choices=["eval", "infer"])
    ap.add_argument("--child", default=None, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.child is not None:
        return child(a.child)
    if not torch.cuda.is_available():
        raise SystemExit("pipeline_cost.py needs a CUDA device")
    info = dict(gpu=torch.cuda.get_device_name(0), name_power_limit_max_sm_clock=device_info(), host_cpus=os.cpu_count(),
                iterations=a.iterations, workers=a.workers)
    log("device", info)
    # a throwaway interpreter first, so that neither way pays the first load of torch and the library from disk
    subprocess.run([sys.executable, "-c", "import instantsplat_b200 as I; I.lib(); import torch; torch.zeros(1).cuda()"],
                   cwd=ROOT, check=True)
    with tempfile.TemporaryDirectory() as tmp:
        views = {}
        for idx in (1, 2):
            info[f"configs{idx}"] = write_source(idx, os.path.join(tmp, f"src{idx}"))
            views[idx] = info[f"configs{idx}"]["views"]
        log("sources", {k: v for k, v in info.items() if k.startswith("configs")})
        for mode in a.modes:
            root = os.path.join(tmp, f"{mode}_root")
            for name, idx in SCENES:
                link = os.path.join(root, "D", name, "24_views") if mode == "eval" else os.path.join(root, "D", name)
                os.makedirs(os.path.dirname(link), exist_ok=True)
                os.symlink(os.path.join(tmp, f"src{idx}"), link)
            info[mode] = measure(mode, root, tmp, views, a)
            log(mode, info[mode])
    print(json.dumps(info))
    return 0


if __name__ == "__main__":
    sys.exit(main())
