"""Cost of train.py's random background in JointTrainer (DESIGN.md section 4.17) on BASELINE configs[2] (1M Gaussians,
12 views, 1920x1080, SH degree 3), the option off against on, alternating in one process.

  * it/s: step() replayed from CUDA graphs, and step_batch with V = --views replayed from graphs.  Each round builds
    both arms afresh from the same scene, captures every graph, then times --steps optimizer steps per arm (it/s
    counts views, one per reference iteration).  Fresh arms keep the two runs on the same stretch of training: over
    longer runs the arms learn different things (the option changes what is optimised), and with them their tile
    lists and blend work.
  * kernels: the view-batched blend forward and backward (`blend_fwd`, `blend_bwd`, CUDA events of the library's
    profiler) of one step_batch frame, launched --launches times with the shared background (gsb_render_batch /
    gsb_backward_batch_stats) and with a [V, 3] table of drawn colours (the *_bg entry points), alternating; the
    same binning lists and dL/dimage, so both do the same work.  Then the V draws of one step into the batch slot,
    timed with CUDA events.

Prints one JSON line per round and a last one with the medians, the GPU, its power limit and SM clock.
Usage: python tools/random_background_cost.py [--steps 200] [--launches 100] [--rounds 3] [--views 4] [--out F]
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
from instantsplat_b200 import _lib  # noqa: E402
from instantsplat_b200.scenes import make_config  # noqa: E402

KERNELS = ("blend_fwd", "blend_bwd")


def device_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                              "0"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        return None


def log(key, value):
    print(json.dumps({key: value}), flush=True)


class Arm:
    """One trainer and its view schedule: step() (V = 1) or step_batch over V consecutive views."""

    def __init__(self, sc, gts, random_background, V):
        cfg = I.OptimConfig()
        cfg.random_background = random_background
        self.tr = I.JointTrainer(sc, "cuda", gt_images=gts, cfg=cfg, use_graph=True)
        self.V, self.n, self.k = V, sc.n_views, 0

    def run(self, steps):
        for _ in range(steps):
            views = [(self.k + j) % self.n for j in range(self.V)]
            self.tr.step(views[0]) if self.V == 1 else self.tr.step_batch(views)
            self.k += self.V


def timed(arm, steps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    arm.run(steps)
    torch.cuda.synchronize()
    return round(steps * arm.V / (time.perf_counter() - t0), 1)


def blend_ms(tr, bg, n):
    """ms per launch of the blend forward and backward of tr's batch frame over n launches each, with bg (None: the
    camera's shared background, else a [V, 3] table)."""
    L = _lib.lib()
    nk = len(_lib.KERNEL_IDS)
    ms, cnt = (ctypes.c_double * nk)(), (ctypes.c_int64 * nk)()
    b = tr._batch
    cam, g = tr._camera(), tr._gauss(b.poses)
    torch.cuda.synchronize()
    L.gsb_profile_enable(1)
    for _ in range(n):
        b.frame.render_batch(cam, None, bg)
        b.frame.backward_batch(cam, g, b.poses, b.dL, tr._grads(), b.dpose, tr.filt, None, 0, bg)
    torch.cuda.synchronize()
    L.gsb_profile_collect(ms, cnt, nk)
    L.gsb_profile_enable(0)
    return {name: round(ms[_lib.KERNEL_IDS.index(name)] / n, 4) for name in KERNELS}


def kernels_part(sc, gts, a):
    arm = Arm(sc, gts, False, a.views)
    arm.run(2)
    tr = arm.tr
    gen = torch.Generator(device="cuda").manual_seed(0)
    table = torch.rand(a.views, 3, generator=gen, device="cuda")
    blend_ms(tr, None, 5)                    # warm both entry points
    blend_ms(tr, table, 5)
    rounds = []
    for r in range(a.rounds):
        order = ("shared", "table") if r % 2 == 0 else ("table", "shared")
        rnd = {name: blend_ms(tr, None if name == "shared" else table, a.launches) for name in order}
        rounds.append(rnd)
        log(f"kernels round {r}", rnd)
    med = {name: {k: sorted(x[name][k] for x in rounds)[len(rounds) // 2] for k in KERNELS}
           for name in ("shared", "table")}
    # what the option adds to a step besides the kernels: the V draws into the slot, timed with CUDA events
    tr.background_generator = torch.Generator(device="cuda").manual_seed(0)
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(a.launches):
        tr._draw_backgrounds(tr._batch)
    end.record()
    torch.cuda.synchronize()
    return dict(V=a.views, launches=a.launches, instances=tr.last_R, rounds=rounds, median=med,
                draws_ms_per_step=round(start.elapsed_time(end) / a.launches, 4))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--launches", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--views", type=int, default=4)
    ap.add_argument("--out", default=None, help="also write the final JSON here")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("random_background_cost.py needs a CUDA device")
    res = dict(gpu=torch.cuda.get_device_name(0), power_limit_and_max_sm_clock=device_info(), config="configs[2]",
               views_per_batch=a.views, steps=a.steps)
    sc = make_config(2)
    gts = torch.rand(sc.n_views, 3, sc.height, sc.width, generator=torch.Generator().manual_seed(2)).to("cuda")
    for path, V in (("step", 1), ("step_batch", a.views)):
        rounds = []
        for r in range(a.rounds):
            order = ("off", "on") if r % 2 == 0 else ("on", "off")
            rnd = {}
            for name in order:
                arm = Arm(sc, gts, name == "on", V)
                arm.run(2 * sc.n_views + 2)          # every view (or batch) graph captured, binning capacity settled
                rnd[name] = dict(it_per_s=timed(arm, a.steps), instances=arm.tr.last_R)
                del arm
                torch.cuda.empty_cache()
            rounds.append(rnd)
            log(f"{path} round {r}", rnd)
        res[path] = dict(V=V, it_per_s=rounds,
                         median={name: sorted(x[name]["it_per_s"] for x in rounds)[len(rounds) // 2] for name in ("off", "on")})
        log(path, res[path]["median"])
    res["blend_kernels_ms"] = kernels_part(sc, gts, a)
    log("blend_kernels_ms", res["blend_kernels_ms"]["median"])
    print(json.dumps(res), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
