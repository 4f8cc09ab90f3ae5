"""Cost of JointTrainer at SH degrees 0..3 (DESIGN.md section 4.16) on BASELINE configs[2] (1M Gaussians, 12 views,
1920x1080), its f_rest cut to (D+1)^2 - 1 rows and max_sh_degree = D (active degree D from the first step).

  * train: per degree, step() replayed from CUDA graphs (it/s over --steps steps after every view's graph is
    captured), then --prof-steps eager steps with CUDA events around every kernel (ms per step of the per-Gaussian
    forward `preprocess`, the per-Gaussian backward `preprocess_bwd` and `adam`), and the bytes of the four flat
    buffers (params, grads, exp_avg, exp_avg_sq).
  * kernels (with --parent-lib, a libgsb200.so built from the parent commit, whose per-Gaussian kernels stage a
    CTA's inputs and write the SH gradients with per-thread copies at M = 4 and 9): per degree 1 and 2, two trainers
    on the same scene, one on each library, stepped eagerly in alternating rounds of --prof-steps steps with the
    same kernel events; their parameters must stay bit-identical.

Prints one JSON line per measurement and a last one with them all, with the GPU and its power limit and SM clock.
Usage: python tools/sh_degree_cost.py [--steps 200] [--prof-steps 40] [--rounds 3] [--parent-lib PATH]
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
from instantsplat_b200.scenes import Scene, make_config  # noqa: E402

ROWS = {0: 0, 1: 3, 2: 8, 3: 15}
KERNELS = ("preprocess", "preprocess_bwd", "adam")


def device_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                              "0"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        return None


def log(key, value):
    print(json.dumps({key: value}), flush=True)


def at_degree(sc: Scene, D: int) -> Scene:
    p = dict(sc.params, f_rest=sc.params["f_rest"][:, :ROWS[D]].contiguous())
    return Scene(p, sc.poses, sc.width, sc.height, sc.fovx, sc.fovy, 3, sc.bg, sc.per_point_lr, sc.name)


def trainer(sc, D, gts, use_graph):
    cfg = I.OptimConfig()
    cfg.max_sh_degree = D
    return I.JointTrainer(at_degree(sc, D), "cuda", gt_images=gts, cfg=cfg, use_graph=use_graph)


def profiled(tr, n, first):
    """ms per step of KERNELS over n eager steps, from the current library's kernel events."""
    L = _lib.lib()
    nk = len(_lib.KERNEL_IDS)
    ms, cnt = (ctypes.c_double * nk)(), (ctypes.c_int64 * nk)()
    L.gsb_profile_enable(1)                          # also drops the records of earlier calls
    for k in range(n):
        tr.step((first + k) % tr.n_views)
    torch.cuda.synchronize()
    L.gsb_profile_collect(ms, cnt, nk)
    L.gsb_profile_enable(0)
    return {name: round(ms[_lib.KERNEL_IDS.index(name)] / n, 4) for name in KERNELS}


def train_part(sc, gts, a):
    out = {}
    for D in (0, 1, 2, 3):
        tr = trainer(sc, D, gts, use_graph=True)
        for k in range(2 * sc.n_views + 2):          # every view's graph captured, binning capacity settled
            tr.step(k % sc.n_views)
        torch.cuda.synchronize()
        k0 = 2 * sc.n_views + 2
        t0 = time.perf_counter()
        for k in range(a.steps):
            tr.step((k0 + k) % sc.n_views)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        tr.use_graph = False
        prof = profiled(tr, a.prof_steps, k0 + a.steps)
        res = dict(M=tr.sh_coeffs, floats_per_gaussian=sum(k for _, k in tr.widths), P=tr.P,
                   flat_buffer_bytes=4 * 4 * tr.total, it_per_s=round(a.steps / dt, 1),
                   kernel_ms_per_step=prof, adam_algorithmic_bytes=tr.algorithmic_bytes()["adam"])
        log(f"train D={D}", res)
        out[f"D{D}"] = res
        del tr
        torch.cuda.empty_cache()
    return out


def use_lib(path):
    """Point the package at the library at `path` (loaded once, then swapped in and out by reference)."""
    _lib._lib = None
    _lib.LIB_PATH = path
    return _lib.lib()


def kernels_part(sc, gts, a):
    new_path = _lib.LIB_PATH
    libs = dict(new=use_lib(new_path), parent=use_lib(os.path.abspath(a.parent_lib)))
    out = {}
    for D in (1, 2):
        trs = {}
        for name, L in libs.items():
            _lib._lib = L
            trs[name] = trainer(sc, D, gts, use_graph=False)
            for k in range(3):
                trs[name].step(k % sc.n_views)
        rounds = []
        for r in range(a.rounds):
            rnd = {}
            for name in (("new", "parent") if r % 2 == 0 else ("parent", "new")):
                _lib._lib = libs[name]
                rnd[name] = profiled(trs[name], a.prof_steps, 3 + r * a.prof_steps)
            rounds.append(rnd)
            log(f"kernels D={D} round {r}", rnd)
        same = all(torch.equal(trs["new"].__dict__[b], trs["parent"].__dict__[b])
                   for b in ("params", "exp_avg", "exp_avg_sq", "poses"))
        med = lambda lib, k: sorted(x[lib][k] for x in rounds)[len(rounds) // 2]
        out[f"D{D}"] = dict(M=(D + 1) ** 2, rounds=rounds, bit_identical=same,
                            median_ms={lib: {k: med(lib, k) for k in KERNELS} for lib in libs})
        log(f"kernels D={D}", out[f"D{D}"])
        del trs
        torch.cuda.empty_cache()
    _lib._lib = libs["new"]
    _lib.LIB_PATH = new_path
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--prof-steps", type=int, default=40)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--parent-lib", default=None)
    ap.add_argument("--out", default=None, help="also write the final JSON here")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sh_degree_cost.py needs a CUDA device")
    res = dict(gpu=torch.cuda.get_device_name(0), power_limit_and_max_sm_clock=device_info(), config="configs[2]")
    sc = make_config(2)
    g = torch.Generator().manual_seed(2)
    gts = torch.rand(sc.n_views, 3, sc.height, sc.width, generator=g).to("cuda")
    res["train"] = train_part(sc, gts, a)
    if a.parent_lib:
        res["kernels_vs_parent"] = kernels_part(sc, gts, a)
    else:
        res["kernels_vs_parent"] = "not measured (no --parent-lib)"
    print(json.dumps(res), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
