"""Cost of the Mip-Splatting filters (DESIGN.md section 4.7) at the bench workload (configs[2]: 1M Gaussians, 12 views,
1920x1080): per-kernel times of the projection (k_preprocess), the per-Gaussian backward (k_preprocess_bwd), the blend
backward of a full backward and of a pose-only (tracking) backward, with the filters off and on, and the time of
gsb_mip_filter3d.  Kernel times come from the library's CUDA-event instrumentation (gsb_profile_*); off and on
alternate round by round.  Prints one JSON object.

    python tools/mip_cost.py [--rounds 5] [--iters 20]
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
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--kernel-size", type=float, default=0.1)
    args = ap.parse_args()
    import torch
    import instantsplat_b200 as I
    from instantsplat_b200._lib import KERNEL_IDS, GsbGrads
    from instantsplat_b200.frame import Frame, IdentityView, capacity, gaussians, mip_filter, mip_filter3d, read_R
    from instantsplat_b200.scenes import make_config
    if not torch.cuda.is_available():
        raise SystemExit("mip_cost.py measures on the GPU; none is available")
    dev = torch.device("cuda")
    L = I.lib()
    sc = make_config(2)
    prm = {k: v.to(dev).float().contiguous() for k, v in sc.params.items()}
    poses = sc.poses.to(dev).float().contiguous()
    iv = IdentityView(sc.width, sc.height, sc.fovx, sc.fovy, sc.bg, dev)
    cam = iv.camera(3, 16)
    f3d = mip_filter3d(prm["xyz"], poses, sc.width, sc.height, iv.tanfovx, iv.tanfovy)
    filters = {"off": None, "on": mip_filter(args.kernel_size, f3d)}
    view = 0
    g = gaussians(sc.P, prm["xyz"], prm["rotation"], prm["scaling"], prm["opacity"], prm["f_dc"], prm["f_rest"],
                  poses[view])
    fr = Frame(dev, sc.P, sc.width, sc.height)
    status = torch.zeros(8, dtype=torch.int32).pin_memory()
    dL = torch.rand(3, sc.height, sc.width, device=dev) * 1e-6
    grads = {k: torch.empty_like(v) for k, v in prm.items()}
    dpose = torch.empty(7, device=dev)
    full, pose_only = GsbGrads(), GsbGrads()
    for f, k in (("dL_dmeans3D", "xyz"), ("dL_dscales", "scaling"), ("dL_drotations", "rotation"),
                 ("dL_dopacities", "opacity"), ("dL_dsh_dc", "f_dc"), ("dL_dsh_rest", "f_rest")):
        setattr(full, f, grads[k].data_ptr())
    full.dL_dpose = pose_only.dL_dpose = dpose.data_ptr()
    names = ("preprocess", "blend_bwd", "preprocess_bwd")
    ids = {n: KERNEL_IDS.index(n) for n in names}
    res = {m: {"full": {n: [] for n in names}, "pose_only": {n: [] for n in names}} for m in filters}
    R = {}
    for m, filt in filters.items():            # size the binning buffer for both, warm up
        fr.preprocess(cam, g, status, filt)
        torch.cuda.synchronize()
        R[m] = read_R(status)
    fr.alloc_binning(capacity(max(R.values()), 1.2))
    for m, filt in filters.items():
        for gr in (full, pose_only):
            fr.preprocess(cam, g, None, filt)
            fr.render(cam)
            fr.backward(cam, g, dL, gr, filt)
    torch.cuda.synchronize()
    n_ids = len(KERNEL_IDS)
    for _ in range(args.rounds):
        for m, filt in filters.items():
            for mode, gr in (("full", full), ("pose_only", pose_only)):
                ms = (ctypes.c_double * n_ids)()
                cnt = (ctypes.c_int64 * n_ids)()
                L.gsb_profile_enable(1)
                for _ in range(args.iters):
                    fr.preprocess(cam, g, None, filt)
                    fr.render(cam)
                    fr.backward(cam, g, dL, gr, filt)
                torch.cuda.synchronize()
                L.gsb_profile_collect(ms, cnt, n_ids)
                L.gsb_profile_enable(0)
                for n in names:
                    res[m][mode][n].append(ms[ids[n]] / max(1, cnt[ids[n]]))
    # gsb_mip_filter3d: CUDA events around repeated launches
    out = torch.empty(sc.P, device=dev)
    for _ in range(3):
        mip_filter3d(prm["xyz"], poses, sc.width, sc.height, iv.tanfovx, iv.tanfovy, out=out)
    t_f3d = []
    for _ in range(args.rounds):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(args.iters):
            mip_filter3d(prm["xyz"], poses, sc.width, sc.height, iv.tanfovx, iv.tanfovy, out=out)
        b.record()
        b.synchronize()
        t_f3d.append(a.elapsed_time(b) / args.iters)
    med = lambda v: sorted(v)[len(v) // 2]
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(
        gpu=smi, workload=f"configs[2]: P={sc.P}, {sc.n_views} views, {sc.width}x{sc.height}, view {view}",
        kernel_size=args.kernel_size, instances=R, rounds=args.rounds, iters=args.iters,
        median_ms={m: {mode: {n: med(v) for n, v in d.items()} for mode, d in r.items()} for m, r in res.items()},
        spread_ms={m: {mode: {n: [min(v), max(v)] for n, v in d.items()} for mode, d in r.items()}
                   for m, r in res.items()},
        mip_filter3d_ms=dict(median=med(t_f3d), min=min(t_f3d), max=max(t_f3d)))))


if __name__ == "__main__":
    main()
