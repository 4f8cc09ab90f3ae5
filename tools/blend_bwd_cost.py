"""Cost of the blend backward's moment reduction (DESIGN.md section 4.3) at the bench workload (configs[2]: 1M
Gaussians, 1920x1080, view 0): the time of the blend backward (k_abs_max + k_blend_bwd2) with the batched reduction
(default) and with the per-entry warp butterfly it replaced (gsb_set_option("blend_bwd_batch", 0)), in a full and a
pose-only (tracking) backward.  Kernel times come from the library's CUDA-event instrumentation (gsb_profile_*); the
two reductions alternate round by round in one process.  Prints one JSON object.

    python tools/blend_bwd_cost.py [--rounds 7] [--iters 30]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=30)
    args = ap.parse_args()
    import torch
    import instantsplat_b200 as I
    from instantsplat_b200._lib import KERNEL_IDS, GsbGrads
    from instantsplat_b200.frame import Frame, IdentityView, capacity, gaussians, read_R
    from instantsplat_b200.scenes import make_config
    if not torch.cuda.is_available():
        raise SystemExit("blend_bwd_cost.py measures on the GPU; none is available")
    dev = torch.device("cuda")
    L = I.lib()
    sc = make_config(2)
    prm = {k: v.to(dev).float().contiguous() for k, v in sc.params.items()}
    poses = sc.poses.to(dev).float().contiguous()
    iv = IdentityView(sc.width, sc.height, sc.fovx, sc.fovy, sc.bg, dev)
    cam = iv.camera(3, 16)
    view = 0
    g = gaussians(sc.P, prm["xyz"], prm["rotation"], prm["scaling"], prm["opacity"], prm["f_dc"], prm["f_rest"],
                  poses[view])
    fr = Frame(dev, sc.P, sc.width, sc.height)
    status = torch.zeros(8, dtype=torch.int32).pin_memory()
    dL = (torch.rand(3, sc.height, sc.width, generator=torch.Generator().manual_seed(3)) * 1e-6).to(dev)
    grads = {k: torch.empty_like(v) for k, v in prm.items()}
    dpose = torch.empty(7, device=dev)
    full, pose_only = GsbGrads(), GsbGrads()
    for f, k in (("dL_dmeans3D", "xyz"), ("dL_dscales", "scaling"), ("dL_drotations", "rotation"),
                 ("dL_dopacities", "opacity"), ("dL_dsh_dc", "f_dc"), ("dL_dsh_rest", "f_rest")):
        setattr(full, f, grads[k].data_ptr())
    full.dL_dpose = pose_only.dL_dpose = dpose.data_ptr()
    fr.preprocess(cam, g, status)
    torch.cuda.synchronize()
    R = read_R(status)
    fr.alloc_binning(capacity(R, 1.2))
    fr.preprocess(cam, g, None)
    fr.render(cam)
    torch.cuda.synchronize()
    modes = {"butterfly": 0, "batch": 1}
    kid = KERNEL_IDS.index("blend_bwd")
    n_ids = len(KERNEL_IDS)
    out = {}
    try:
        for m, on in modes.items():        # warm up both, and check they give the same accumulator words
            assert L.gsb_set_option(b"blend_bwd_batch", on) == 0
            for gr in (full, pose_only):
                fr.backward(cam, g, dL, gr)
            fr.backward(cam, g, dL, full)
            torch.cuda.synchronize()
            out[m] = {k: v.clone() for k, v in grads.items()}
        identical = all(torch.equal(out["butterfly"][k], out["batch"][k]) for k in grads)
        res = {m: {"full": [], "pose_only": []} for m in modes}
        for _ in range(args.rounds):
            for m, on in modes.items():
                L.gsb_set_option(b"blend_bwd_batch", on)
                for mode, gr in (("full", full), ("pose_only", pose_only)):
                    ms = (ctypes.c_double * n_ids)()
                    cnt = (ctypes.c_int64 * n_ids)()
                    L.gsb_profile_enable(1)
                    for _ in range(args.iters):
                        fr.backward(cam, g, dL, gr)
                    torch.cuda.synchronize()
                    L.gsb_profile_collect(ms, cnt, n_ids)
                    L.gsb_profile_enable(0)
                    res[m][mode].append(ms[kid] / max(1, cnt[kid]))
    finally:
        L.gsb_set_option(b"blend_bwd_batch", 1)
    med = lambda v: sorted(v)[len(v) // 2]
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(
        gpu=smi, workload=f"configs[2]: P={sc.P}, {sc.width}x{sc.height}, view {view}, R={R}",
        rounds=args.rounds, iters=args.iters, gradients_identical=identical,
        blend_bwd_median_ms={m: {k: med(v) for k, v in r.items()} for m, r in res.items()},
        blend_bwd_spread_ms={m: {k: [min(v), max(v)] for k, v in r.items()} for m, r in res.items()},
        blend_bwd_ms={m: r for m, r in res.items()})))


if __name__ == "__main__":
    main()
