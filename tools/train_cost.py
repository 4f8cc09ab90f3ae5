"""Cost of the training stage (run_eval.sh / run_infer.sh stage 2) through `python -m instantsplat_b200.train`, against
a train.py-shaped loop through the drop-in API on the same scene and schedule, at
  * BASELINE configs[1]: 200k Gaussians, 3 views, 512x512;
  * BASELINE configs[2]: 1M Gaussians, 12 views, 1920x1080.

The source is written by scene_io.write_synthetic_source: the config's points and confidence, and PNG images rendered
from the config's own Gaussians.  Per workload and round (the two arms alternate):
  * cli: train.run() with InstantSplat's flags (--iterations 1000 --pp_optimizer --optim_pose), wall time end to end
    and its phases (host clock around work that ends in a device synchronise): load (PNG decode, PLY and confidence
    read), init (create_from_pcd with the GPU knn, targets uploaded), trainer (JointTrainer construction), loop (the
    1000 iterations, CUDA-graph captures included, saves excluded), saves (ply, poses at the final iteration);
  * dropin_loop: train.py:140-211 on the same Gaussians, targets and schedule: update_learning_rate, the fused
    render(), L1 + fused_ssim, backward, PerPointAdam (training_setup_pp with the confidence), loss.item() every
    iteration.

Prints one JSON line per measurement and a last one with them all, with the GPU and its power limit and SM clock.
Usage: python tools/train_cost.py [--iterations 1000] [--rounds 2]
"""
import argparse
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
from instantsplat_b200 import scene_io as S  # noqa: E402
from instantsplat_b200 import train as T  # noqa: E402
from instantsplat_b200.camera import SimpleCamera  # noqa: E402
from instantsplat_b200.scenes import make_config  # noqa: E402
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


def write_source(sc, root):
    p = sc.params
    tk = PoseTracker(p["xyz"], p["rotation"], p["scaling"], p["opacity"], p["f_dc"], p["f_rest"], sc.width, sc.height,
                     sc.fovx, sc.fovy, sh_degree=3, device="cuda")
    u8 = np.concatenate([c for _, c in F.frames_u8(tk, sc.poses, max_batch=4)])
    del tk
    S.write_synthetic_source(root, sc, u8)
    return root


def dropin_loop(src, n_views, iterations):
    """train.py:140-211 with the drop-ins; returns (seconds for the loop, last loss)."""
    from instantsplat_b200 import fused_ssim
    dev = "cuda"
    ts = T.load_training_scene(src, n_views, 1)
    gm = I.GaussianModel(3, dev)
    gm.create_from_pcd(ts.host.points, ts.host.colors, ts.host.extent)
    gm.init_RT_seq(ts.host.poses)
    gm.training_setup_pp(I.optimization_defaults(iterations=iterations), ts.host.per_point_lr.to(dev))
    cams = []
    for v in range(n_views):
        c = SimpleCamera(ts.scene.width, ts.scene.height, ts.scene.fovx, ts.scene.fovy, device=dev)
        c.uid = v
        cams.append(c)
    pipe, bg = I.PipelineDefaults(), torch.zeros(3, device=dev)
    rows = T.view_schedule(n_views, iterations)[1]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    loss_v = None
    for k, row in enumerate(rows):
        it = k + 1
        gm.update_learning_rate(it)
        if it % 1000 == 0:
            gm.oneupSHdegree()
        img = I.render(cams[row], gm, pipe, bg, camera_pose=gm.get_RT(row))["render"]
        gt = ts.targets[row]
        loss = 0.8 * torch.abs(img - gt).mean() + 0.2 * (1.0 - fused_ssim(img.unsqueeze(0), gt.unsqueeze(0)))
        loss.backward()
        loss_v = loss.item()
        if it < iterations:
            gm.optimizer.step()
            gm.optimizer.zero_grad(set_to_none=True)
    torch.cuda.synchronize()
    return time.perf_counter() - t0, loss_v


def workload(idx, a):
    sc = make_config(idx)
    res = dict(P=sc.P, views=sc.n_views, W=sc.width, H=sc.height, iterations=a.iterations, rounds=[])
    with tempfile.TemporaryDirectory() as tmp:
        src = write_source(sc, os.path.join(tmp, "src"))
        del sc
        argv = lambda m: ["-s", src, "-m", os.path.join(tmp, m), "-r", "1", "--n_views", str(res["views"]),
                          "--pp_optimizer", "--optim_pose", "--quiet"]
        T.run(T.parse_args(argv("warm") + ["--iterations", "20"]))                    # warm-up: imports, modules
        dropin_loop(src, res["views"], 20)
        for r in range(a.rounds):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = T.run(T.parse_args(argv(f"cli{r}") + ["--iterations", str(a.iterations)]))
            torch.cuda.synchronize()
            t_cli = time.perf_counter() - t0
            last, phases = float(out.losses[-1]), {k: round(v, 3) for k, v in out.phases.items()}
            loop_rate = round(a.iterations / out.phases["loop"], 1)
            del out
            torch.cuda.empty_cache()
            t_loop, last_ref = dropin_loop(src, res["views"], a.iterations)
            torch.cuda.empty_cache()
            rnd = dict(cli_s=round(t_cli, 3), cli_phases_s=phases, cli_loop_it_per_s=loop_rate, dropin_loop_s=round(t_loop, 3),
                       dropin_it_per_s=round(a.iterations / t_loop, 1), cli_last_loss=last, dropin_last_loss=last_ref)
            res["rounds"].append(rnd)
            log(f"configs[{idx}] round {r}", rnd)
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iterations", type=int, default=1000)
    ap.add_argument("--rounds", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("train_cost.py needs a CUDA device")
    out = dict(gpu=torch.cuda.get_device_name(0), power_limit_and_max_sm_clock=device_info(), host_cpus=os.cpu_count())
    log("device", out)
    for idx in (1, 2):
        out[f"configs{idx}"] = workload(idx, a)
        log(f"configs{idx}", out[f"configs{idx}"])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
