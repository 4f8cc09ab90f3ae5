#!/usr/bin/env python
"""bench.py -- the BASELINE.json metric on H100: train iters/sec (+ render Mpix/s fwd+bwd) of the
joint pose+Gaussian optimisation loop at 1M Gaussians / 12 views / 1920x1080 / SH degree 3
(BASELINE.json configs[2]; configs[0] is the CPU-only correctness case, configs[1] a parity size).

    python bench.py --gpus 1 --steps 20 --warmup 5
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 \
        --master-port P bench.py --gpus N --steps K --warmup W
    python bench.py --impl reference ...      # the oracle port of the path on the host cores

One "iteration" = one reference training iteration (train.py:140-211) on ONE view: render (fused pose
transform + rasterizer) -> L1+DSSIM -> backward -> optimizer step.  With N GPUs the views are sharded
(view v -> rank v mod N): every optimizer step consumes N views, gradients are summed with one NCCL
all-reduce; value = views processed by all ranks / time ("weak" scaling: one view per GPU per step).
Prints ONE JSON line (rank 0).
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

METRIC = "train_iters_per_sec"
UNIT = "iters/s"


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--config", type=int, default=2, help="BASELINE.json configs index (2 = headline)")
    ap.add_argument("--scale", type=float, default=1.0, help="shrink P (debug only; invalidates the number)")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--blend-version", type=int, default=0, help="debug: force blend kernel version 1|2|3")
    ap.add_argument("--graph", action="store_true",
                    help="multi-GPU with --exchange fused_p2p: replay each rank's iteration (exchange included) from CUDA graphs")
    ap.add_argument("--no-graph", action="store_true",
                    help="do not replay the iteration from CUDA graphs (single GPU, and multi-GPU with --exchange fused_p2p)")
    ap.add_argument("--exchange", default="fused_p2p", choices=["allreduce", "fused_p2p", "fused_p2p_nccl"],
                    help="multi-GPU gradient exchange: NCCL all-reduce + Adam, or the fused P2P "
                         "reduce-scatter->Adam->all-gather kernel (default)")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write what the last timed step computed (rendered image, loss, "
                         "poses, a fixed seeded row sample of every parameter tensor) as DIR/<name>.npy")
    return ap.parse_args()


def workload_name(idx, sc):
    return (f"BASELINE.configs[{idx}]: {sc.P} Gaussians, {sc.n_views} views {sc.width}x{sc.height}, "
            f"SH deg {sc.sh_degree}, joint pose+Gaussian optimisation (InstantSplat path), synthetic surface scene")


class ClockSampler:
    """nvidia-smi clocks / throttle reasons during the timed region."""
    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,"
         "clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index=0):
        self.rows, self.proc, self.idx = [], None, gpu_index

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits",
                                          "-lms", "20", "-i", str(self.idx)], stdout=subprocess.PIPE,
                                         stderr=subprocess.DEVNULL, text=True)
            self.t = threading.Thread(target=self._read, daemon=True)
            self.t.start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append(line.strip())

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        time.sleep(0.05)
        self.proc.terminate()
        sm, mx, reasons = [], [], set()
        for r in self.rows:
            f = [x.strip() for x in r.split(",")]
            if len(f) < 9:
                continue
            try:
                sm.append(float(f[1])); mx.append(float(f[2]))
            except ValueError:
                continue
            for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), f[5:9]):
                if v.lower().startswith("active"):
                    reasons.add(name)
        sm.sort()
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "reasons": sorted(reasons), "samples": len(sm)}


def measured_peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        return float(d["hbm_gbs"]), "measured (MEASURED_PEAKS.json hbm_gbs)"
    return 3350.0, "not measured: H100 SXM data sheet HBM3 bandwidth (3.35 TB/s)"


def gpu_identity(dev):
    """The card a number was measured on: name, SM count, L2 size and (from nvidia-smi) power limit and max SM clock."""
    props = torch.cuda.get_device_properties(dev)
    out = {"name": props.name, "sm_count": props.multi_processor_count,
           "l2_mb": getattr(props, "L2_cache_size", 0) / 2**20, "power_limit_w": None, "sm_max_mhz": None}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                            "-i", str(dev.index or 0)], capture_output=True, text=True, timeout=30).stdout.split(",")
        out["power_limit_w"], out["sm_max_mhz"] = float(q[0]), float(q[1])
    except Exception:
        pass
    return out


# ----------------------------------------------------------------------------------------------
# --dump-outputs: what the timed path computed in its last step, so that two builds can be compared output for output
# ----------------------------------------------------------------------------------------------
DUMP_IMAGE_PIXELS = 1 << 21     # 25 MB of image: every pixel up to 1920x1080, a fixed sample above
DUMP_PARAM_ROWS = 1 << 16       # 15 MB of parameters (59 floats per Gaussian)


def grab_outputs(tr):
    """Host copies of the last step's results: the rendered image of its view, its loss, and -- after its optimizer
    update -- the pose table and every parameter tensor.  Larger outputs are reduced to a sample fixed by a seed and
    the shapes alone, so every run with the same arguments samples the same elements."""
    g = torch.Generator().manual_seed(0)

    def sample(n, cap):
        return None if n <= cap else torch.randperm(n, generator=g)[:cap].sort().values.to(tr.dev)

    img = tr.color.reshape(3, -1)
    pix = sample(img.shape[1], DUMP_IMAGE_PIXELS)
    out = {"image": img.reshape(tr.color.shape) if pix is None else img[:, pix],
           "loss": tr.loss_value().double().reshape(1), "poses": tr.poses}
    rows = sample(tr.P, DUMP_PARAM_ROWS)
    from instantsplat_b200.trainer import SEGMENTS
    for name, _ in SEGMENTS:
        p = tr.view(tr.params, name)
        out[name] = p if rows is None else p[rows]
    return {k: v.detach().cpu().numpy().copy() for k, v in out.items()}


def write_outputs(out_dir, arrays):
    import numpy as np
    os.makedirs(out_dir, exist_ok=True)
    for name, a in arrays.items():
        np.save(os.path.join(out_dir, name + ".npy"), a)


# ----------------------------------------------------------------------------------------------
# CPU arm: the oracle port of the path on the host cores, on a bounded, DETERMINISTIC sample of the workload
# ----------------------------------------------------------------------------------------------
def cpu_sample_plan(sc, n_steps):
    """What one CPU step computes -- a pure function of the workload and of the number of steps (no wall-clock
    probing, so two runs sample the same work).  About 12 s of CPU work per step (all Gaussians, 128 stratified tiles,
    the full frame's loss) for up to 32 steps -- the default bench's cpu_baseline (1 warm-up + 3 timed) and
    `--impl reference --steps 20 --warmup 5` (about 5 minutes) -- and a sample shrinking to no less than 1/8 of that for
    longer runs.  Smaller samples are NOT used: PyTorch's per-operator overhead dominates small tensors and the
    extrapolation then under-reports the CPU."""
    gx, gy = (sc.width + 15) // 16, (sc.height + 15) // 16
    T = gx * gy
    shrink = 1 if n_steps <= 32 else min(8, (n_steps + 31) // 32)
    n_g = max(2_000, min(sc.P, sc.P // shrink))                      # Gaussians projected (fwd+bwd) and Adam-updated
    n_t = max(4, min(T, 128 // shrink))                              # tiles blended (fwd+bwd), stratified over the frame
    rows = max(32, min(sc.height, sc.height // shrink))              # image rows of the L1+SSIM loss (fwd+bwd)
    stride = max(1, T // n_t)
    tiles = list(range(stride // 2, T, stride))[:n_t]
    return dict(n_gauss=n_g, tiles=tiles, rows=rows, T=T)


def cpu_reference_step(sc, view, gt, plan, proj_full, threads):
    """One sampled iteration of the oracle.  Returns seconds for (projection fwd+bwd + pose pre-transform over
    n_gauss Gaussians, blend fwd+bwd of the FULL cloud's lists on the plan's tiles, loss fwd+bwd on `rows` image rows,
    per-point Adam on n_gauss) and the number of tile instances blended."""
    from oracle import gs_oracle as O
    torch.set_num_threads(threads)
    n_g, tiles, rows = plan["n_gauss"], plan["tiles"], plan["rows"]
    cam = O.Camera.instantsplat(sc.width, sc.height, sc.fovx, sc.fovy, sh_degree=sc.sh_degree)
    prm = {k: v[:n_g].clone().requires_grad_(True) for k, v in sc.params.items()}
    pose = sc.poses[view].clone().requires_grad_(True)
    t0 = time.perf_counter()
    means, rots = O.pose_pretransform(prm["xyz"], prm["rotation"], pose)
    shs = torch.cat([prm["f_dc"], prm["f_rest"]], dim=1)
    proj = O.project(means, torch.exp(prm["scaling"]), rots, torch.sigmoid(prm["opacity"]), shs, cam)
    (proj["xy"].sum() + proj["conic"].sum() + proj["rgb"].sum() + proj["opacity"].sum()).backward()
    t1 = time.perf_counter()
    # blend: the tile lists of the WHOLE cloud (projected once, outside the timed region), leaves re-attached so that
    # the backward of the blend itself is timed
    leaves = {k: proj_full[k].detach().clone().requires_grad_(True) for k in ("xy", "conic", "opacity", "rgb")}
    pf = dict(proj_full)
    pf.update(leaves)
    t1b = time.perf_counter()
    img, aux = O.blend(pf, cam, tiles=tiles, return_aux=True)
    (img * torch.ones_like(img)).sum().backward()
    t2 = time.perf_counter()
    inst = int(sum(int(aux["ranges"][t, 1] - aux["ranges"][t, 0]) for t in tiles))
    im = img.detach()[:, :rows].clone().requires_grad_(True)
    O.training_loss(im, gt[:, :rows]).backward()
    t3 = time.perf_counter()
    for k, p in prm.items():
        g = p.grad if p.grad is not None else torch.zeros_like(p)
        O.per_point_adam_step(p.data, g, torch.zeros_like(p), torch.zeros_like(p), 1, 1e-3)
    t4 = time.perf_counter()
    return (t1 - t0), (t2 - t1b), (t3 - t2), (t4 - t3), inst


def cpu_arm(sc, steps, warmup):
    """Returns dict(value iters/s extrapolated to the full workload, spread over the timed steps, sample description).
    Extrapolation: projection and Adam by Gaussian count, blend by TILE-INSTANCE count (sum of list lengths: the
    quantity its cost is proportional to), loss by image rows."""
    from oracle import gs_oracle as O
    threads = min(os.cpu_count() or 1, 32)   # more threads only add sync overhead on these op sizes
    total_steps = max(1, steps + warmup)
    plan = cpu_sample_plan(sc, total_steps)
    gt = torch.rand(3, sc.height, sc.width, generator=torch.Generator().manual_seed(0))
    torch.set_num_threads(threads)
    cam = O.Camera.instantsplat(sc.width, sc.height, sc.fovx, sc.fovy, sh_degree=sc.sh_degree)
    view = 0
    with torch.no_grad():                    # untimed set-up: the full cloud's projection (tile lists, R)
        means, rots = O.pose_pretransform(sc.params["xyz"], sc.params["rotation"], sc.poses[view])
        shs = torch.cat([sc.params["f_dc"], sc.params["f_rest"]], dim=1)
        proj_full = O.project(means, torch.exp(sc.params["scaling"]), rots, torch.sigmoid(sc.params["opacity"]), shs, cam)
    R_full = int(proj_full["ntiles"].sum())
    times, parts = [], None
    for s in range(total_steps):
        tp, tb, tl, ta, inst = cpu_reference_step(sc, view, gt, plan, proj_full, threads)
        if s >= warmup:
            est = (tp + ta) * (sc.P / plan["n_gauss"]) + tb * (R_full / max(1, inst)) + tl * (sc.height / plan["rows"])
            times.append(est)
            parts = dict(projection_s=tp, blend_s=tb, loss_s=tl, adam_s=ta, instances_blended=inst)
    times.sort()
    med = times[len(times) // 2]
    return dict(value=1.0 / med, unit=UNIT, cores=threads, kind="port",
                spread={"n": len(times), "min_s_per_iter": times[0], "median_s_per_iter": med, "max_s_per_iter": times[-1]},
                sample=(f"oracle/gs_oracle.py (PyTorch CPU, {threads} threads), fixed sample (function of the workload and the "
                        f"step count only): per step pose pre-transform + projection fwd+bwd and Adam on {plan['n_gauss']} of "
                        f"{sc.P} Gaussians, blend fwd+bwd of the full cloud's tile lists on {len(plan['tiles'])} of {plan['T']} "
                        f"tiles ({parts['instances_blended']} of {R_full} tile instances, reference rect binning), L1+SSIM "
                        f"fwd+bwd on {plan['rows']} of {sc.height} rows; extrapolated by Gaussian count / instance count / "
                        f"rows; median of {len(times)} timed steps (view {view})"),
                sec_per_iter_extrapolated=med, last_step_parts=parts)


def gpu_torch_pieces(sc, dev, img, gt, reps=10):
    """BASELINE.md row B-ref-py: the reference's Python-side pieces of the path (pose pre-transform + activations +
    feature cat, l1 + PyTorch ssim, PerPointAdam), restated in oracle/gs_oracle.py, run with plain torch ops on
    the SAME GPU -- what the fused preprocess / loss / Adam kernels replace.  Baseline leg only."""
    from oracle import gs_oracle as O

    def clock(fn):
        for _ in range(2):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / reps

    prm = {k: v.to(dev).clone().requires_grad_(True) for k, v in sc.params.items()}
    pose = sc.poses[0].to(dev).clone().requires_grad_(True)

    def pre():
        means, rots = O.pose_pretransform(prm["xyz"], prm["rotation"], pose)
        shs = torch.cat([prm["f_dc"], prm["f_rest"]], dim=1)
        out = means.sum() + rots.sum() + torch.exp(prm["scaling"]).sum() + torch.sigmoid(prm["opacity"]).sum() + shs.sum()
        out.backward()
        for p in list(prm.values()) + [pose]:
            p.grad = None

    im = img.detach().clone().requires_grad_(True)

    def loss():
        O.training_loss(im, gt).backward()
        im.grad = None

    ps = [v.detach().clone() for v in prm.values()]
    gs_ = [torch.randn_like(p) * 1e-3 for p in ps]
    ms = [torch.zeros_like(p) for p in ps]
    vs = [torch.zeros_like(p) for p in ps]
    ppl = sc.per_point_lr.to(dev) if sc.per_point_lr is not None else None
    state = {"t": 0}

    def adam():
        state["t"] += 1
        for i, p in enumerate(ps):
            O.per_point_adam_step(p, gs_[i], ms[i], vs[i], state["t"], 1e-3, per_point_lr=ppl if i == 0 else None)

    return {"pose_pretransform_activations_cat_fwd_bwd_ms": clock(pre), "l1_ssim_fwd_bwd_ms": clock(loss),
            "per_point_adam_ms": clock(adam),
            "what": "torch restatement (oracle/gs_oracle.py) of the reference's gaussian_renderer/__init__.py:81-92,102,121, "
                    "utils/loss_utils.py:39-85 and scene/per_point_adam.py:34-98 run on the same GPU"}


def run_reference(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return None
    from instantsplat_b200.scenes import make_config
    sc = make_config(args.config, args.scale)
    r = cpu_arm(sc, args.steps, args.warmup)
    line = {"impl": "reference", "metric": METRIC, "value": r["value"], "unit": UNIT, "n_gpus": args.gpus,
            "steps": args.steps, "warmup": args.warmup, "ms_per_step": 1000.0 * r["sec_per_iter_extrapolated"],
            "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32",
            "data": "synthetic", "config": {"workload": workload_name(args.config, sc)},
            "cpu_baseline": {"value": r["value"], "unit": UNIT, "cores": r["cores"], "kind": "port",
                             "sample": r["sample"], "spread": r["spread"]},
            "e2e": {"value": r["value"], "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
            "note": "reference CUDA path (diff-gaussian-rasterization / fused-ssim) is an empty submodule in "
                    "the reference checkout: this arm is the CPU oracle port of the same path"}
    return line


# ----------------------------------------------------------------------------------------------
def run_b200(args):
    import instantsplat_b200 as I
    from instantsplat_b200 import _lib
    from instantsplat_b200.parallel import init_from_env, view_for_step
    from instantsplat_b200.scenes import make_config, perturbed_copy
    import torch.distributed as dist

    rank, local, world = init_from_env("nccl")
    assert world == args.gpus or world == 1, f"WORLD_SIZE {world} != --gpus {args.gpus}"
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    L = I.lib()
    if args.blend_version:
        L.gsb_set_option(b"blend_version", args.blend_version)
    sc = make_config(args.config, args.scale)
    # ground-truth images: our own render of a perturbed copy of the scene (non-trivial loss)
    tgt = I.JointTrainer(sc, dev)
    pp = perturbed_copy(sc, sigma=0.05)
    for k, kk in (("xyz", 3), ("f_dc", 3), ("opacity", 1), ("scaling", 3)):
        tgt.view(tgt.params, k).copy_(pp[k].reshape(sc.P, kk).to(dev))
    gt_dev = torch.stack([tgt.render(v).clone() for v in range(sc.n_views)])
    del tgt
    torch.cuda.empty_cache()
    gt_host = gt_dev.cpu().pin_memory()
    # N=1: graph replay is the default.  N>1: capturable with the flag-barrier exchange and bit-exact
    # (tests/test_multigpu.py "fused_p2p+graph"), but no faster than eager launches at N=2 when it was measured: the
    # host already runs ahead of a step that waits on its peers, so eager stays the default there and --graph opts in
    use_graph = (world == 1 and not args.no_graph) or (world > 1 and args.graph and args.exchange == "fused_p2p")
    tr = I.JointTrainer(sc, dev, gt_images=gt_dev, world_size=world, rank=rank, exchange=args.exchange,
                        use_graph=use_graph)
    # ---- e2e pipeline through the public API: this step's GT image is copied H2D from pinned memory on a copy
    # stream (double buffered, so the copy of step s+1 overlaps the compute of step s) and every step's loss is
    # read back to the host (asynchronously, consumed one step later).
    stages = [torch.empty_like(gt_dev[0]) for _ in range(2)]
    stage = stages[0]
    loss_host = torch.zeros(2, dtype=torch.float64).pin_memory()
    copy_stream = torch.cuda.Stream(device=dev)
    ev_copied = [torch.cuda.Event() for _ in range(2)]
    ev_free = [torch.cuda.Event() for _ in range(2)]
    ev_loss = [torch.cuda.Event() for _ in range(2)]
    losses = []
    e2e_state = {"primed": -1}

    def barrier():
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def device_step(s):
        tr.step(view_for_step(sc.n_views, world, rank, s))

    def prefetch(s):
        i = s & 1
        with torch.cuda.stream(copy_stream):
            copy_stream.wait_event(ev_free[i])
            stages[i].copy_(gt_host[view_for_step(sc.n_views, world, rank, s)], non_blocking=True)
            ev_copied[i].record(copy_stream)

    def e2e_step(s):
        i = s & 1
        if e2e_state["primed"] != s:
            prefetch(s)
        prefetch(s + 1)
        e2e_state["primed"] = s + 1
        cur = torch.cuda.current_stream()
        cur.wait_event(ev_copied[i])
        tr.step(view_for_step(sc.n_views, world, rank, s), gt=stages[i])
        ev_free[i].record(cur)
        loss_host[i:i + 1].copy_(tr.loss_value().reshape(1), non_blocking=True)   # D2H of this step's result
        ev_loss[i].record(cur)
        if e2e_state.get("have_prev"):
            ev_loss[1 - i].synchronize()
            losses.append(float(loss_host[1 - i]))
        e2e_state["have_prev"] = True

    def timed(fn, n, first):
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for s in range(n):
            fn(first + s)
        e1.record()
        barrier()
        ms = torch.tensor([e0.elapsed_time(e1)], device=dev, dtype=torch.float64)
        if world > 1:
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        return float(ms[0])

    W_, K = max(3, args.warmup), args.steps
    if use_graph:
        # first visit of a view is eager, the second captures its graph (a rank visits ceil(n_views / world) views)
        W_ = max(W_, 2 * ((sc.n_views + world - 1) // world) + 2)
    for s in range(W_):
        device_step(s)
    sampler = ClockSampler(local)
    if rank == 0:
        sampler.start()
    Rs = []
    import ctypes
    nk = len(_lib.KERNEL_IDS)
    ms_sum = (ctypes.c_double * nk)()
    cnt = (ctypes.c_int64 * nk)()
    if use_graph:
        # timed region 1 (the reported value): the iteration replayed from CUDA graphs, no instrumentation inside
        ms_dev = timed(lambda s: (device_step(s), Rs.append(tr.last_R)), K, W_)
        clocks = sampler.stop() if rank == 0 else None
        dumped = grab_outputs(tr) if args.dump_outputs and rank == 0 else None
        # timed region 2 (per-kernel table / roofline): the same steps launched eagerly with CUDA events around
        # every kernel on the launching stream
        tr.use_graph = False
        Kp = min(K, 40)
        L.gsb_profile_enable(1)
        launches0 = L.gsb_launch_count()
        ms_prof = timed(device_step, Kp, W_ + K)
        launches = int(round((L.gsb_launch_count() - launches0) * K / Kp))
        L.gsb_profile_collect(ms_sum, cnt, nk)
        L.gsb_profile_enable(0)
    else:
        L.gsb_profile_enable(1)
        launches0 = L.gsb_launch_count()
        ms_dev = timed(lambda s: (device_step(s), Rs.append(tr.last_R)), K, W_)
        dumped = grab_outputs(tr) if args.dump_outputs and rank == 0 else None
        launches = int(L.gsb_launch_count() - launches0)
        L.gsb_profile_collect(ms_sum, cnt, nk)
        L.gsb_profile_enable(0)
        clocks = sampler.stop() if rank == 0 else None
        ms_prof, Kp = ms_dev, K
    # e2e through JointTrainer.step(view, gt=<staging buffer>): graphs are keyed on (view, staging buffer), so warm
    # up until every pair this rank will visit has been captured
    tr.use_graph = use_graph
    n_e2e_warm = 2 * ((sc.n_views + world - 1) // world) + 2 if use_graph else 2
    for s in range(n_e2e_warm):
        e2e_step(W_ + K + s)
    ms_e2e = timed(e2e_step, K, W_ + K + n_e2e_warm)
    # ---- the same iteration through the reference's own operator API (boundaries B1-B4): the loop body of
    # the reference's train.py:140-211 transcribed onto the repo's mirror of GaussianModel (the reference tree is not
    # a dependency of this repository; tests/test_reference_shims_cpu.py checks the mirror against it on the CPU).
    dropin, e2e_plugin = None, None
    if world == 1:
        sys.path.insert(0, os.path.join(ROOT, "shims"))
        from fused_ssim import fused_ssim as shim_fused_ssim            # as train.py:39-43 imports it
        import instantsplat_b200.renderer as RD
        from instantsplat_b200.camera import SimpleCamera
        camv = SimpleCamera(sc.width, sc.height, sc.fovx, sc.fovy, device=dev)
        pipe = I.PipelineDefaults()
        bgz = torch.zeros(3, device=dev)
        oargs = I.optimization_defaults(iterations=30_000)
        nd = min(K, 60)

        def make_model():
            m = I.GaussianModel.from_scene(sc, dev)
            m.training_setup_pp(oargs)
            return m

        def verbatim_loop(model, n, first):
            """train.py:140-211 incl. update_learning_rate, the SH schedule and the per-iteration loss.item()."""
            for s in range(first, first + n):
                iteration = s + 1
                model.update_learning_rate(iteration)
                if iteration % 1000 == 0:
                    model.oneupSHdegree()
                v = s % sc.n_views
                pkg = I.render(camv, model, pipe, bgz, camera_pose=model.get_RT(v))
                image = pkg["render"]
                gt_image = gt_dev[v]                     # cameras keep original_image on the GPU (scene/cameras.py)
                Ll1 = torch.abs(image - gt_image).mean()
                ssim_value = shim_fused_ssim(image.unsqueeze(0), gt_image.unsqueeze(0))
                loss = 0.8 * Ll1 + 0.2 * (1.0 - ssim_value)
                loss.backward()
                loss.item()
                model.optimizer.step()
                model.optimizer.zero_grad(set_to_none=True)

        dropin = {}
        try:
            for name, fused in (("dropin_unchanged", False), ("dropin_fused", True)):
                RD.FUSED = fused
                model = make_model()
                verbatim_loop(model, 3, 0)
                ms = timed(lambda s0, m=model: verbatim_loop(m, 1, s0), nd, 3)
                dropin[name] = {"value": nd / (ms / 1e3), "unit": UNIT, "ms_per_step": ms / nd, "steps": nd}
                del model
            dropin["dropin_unchanged"]["api"] = (
                "train.py:140-211 verbatim (update_learning_rate, render, l1 + fused_ssim, backward, loss.item(), "
                "PerPointAdam.step) with the reference-shaped render body: PyTorch pose pre-transform / activations / "
                "feature cat -> GaussianRasterizer shim -- what an UNCHANGED checkout gets from PYTHONPATH=shims")
            dropin["dropin_fused"]["api"] = ("same loop with the fused render() (instantsplat_b200/hooks.py swaps it in "
                                             "without editing the reference)")
            # ---- headline e2e through the plugin API: fused render + fused_ssim + backward + PerPointAdam.step, this
            # step's GT copied H2D from pinned memory (double buffered on a copy stream), loss read back D2H every
            # step (asynchronously, consumed one step later) -- no blocking .item() in the loop
            RD.FUSED = True
            model = make_model()
            p_loss = torch.zeros(2, dtype=torch.float32).pin_memory()
            pst = {"primed": -1, "have_prev": False}

            def plugin_step(s):
                i = s & 1
                if pst["primed"] != s:
                    prefetch(s)
                prefetch(s + 1)
                pst["primed"] = s + 1
                cur = torch.cuda.current_stream()
                cur.wait_event(ev_copied[i])
                v = view_for_step(sc.n_views, world, rank, s)
                model.update_learning_rate(s + 1)
                pkg = I.render(camv, model, pipe, bgz, camera_pose=model.get_RT(v))
                image = pkg["render"]
                loss = 0.8 * torch.abs(image - stages[i]).mean() + 0.2 * (1.0 - shim_fused_ssim(image.unsqueeze(0), stages[i].unsqueeze(0)))
                loss.backward()
                ev_free[i].record(cur)
                p_loss[i:i + 1].copy_(loss.detach().reshape(1), non_blocking=True)
                ev_loss[i].record(cur)
                if pst["have_prev"]:
                    ev_loss[1 - i].synchronize()
                    losses.append(float(p_loss[1 - i]))
                pst["have_prev"] = True
                model.optimizer.step()
                model.optimizer.zero_grad(set_to_none=True)

            base = W_ + 2 * K + 8
            for s in range(3):
                plugin_step(base + s)
            ms_pl = timed(plugin_step, K, base + 3)
            e2e_plugin = {"value": K / (ms_pl / 1e3), "unit": UNIT, "ms_per_step": ms_pl / K,
                          "h2d_bytes_per_step": int(stage.numel() * 4), "d2h_bytes_per_step": 4,
                          "api": "reference operator API: render() [fused] + l1 + fused_ssim + loss.backward() + "
                                 "PerPointAdam.step() + update_learning_rate; GT H2D from pinned memory every step "
                                 "(copy stream, double buffered), loss D2H every step (async, read one step later)"}
            del model
        finally:
            RD.FUSED = True
    tr.check_peer_errors()
    if rank != 0:
        if world > 1:
            dist.destroy_process_group()
        return None
    views = K * world
    value = views / (ms_dev / 1e3)
    e2e_value = views / (ms_e2e / 1e3)
    # ---- per-kernel table and the roofline of the dominant kernel
    peak, peak_src = measured_peaks()
    tr.last_R = int(sum(Rs) / max(1, len(Rs)))
    alg = tr.algorithmic_bytes()
    alg_map = {"preprocess": alg["preprocess_fwd"], "blend_fwd": alg["blend_fwd"], "blend_bwd": alg["blend_bwd"],
               "preprocess_bwd": alg["preprocess_bwd"], "adam": alg["adam"],
               "loss_fwd": alg["loss"] * 0.5, "loss_bwd": alg["loss"] * 0.5}
    kernels = {}
    for i, name in enumerate(_lib.KERNEL_IDS):
        if cnt[i] == 0:
            continue
        avg = ms_sum[i] / cnt[i]
        row = {"ms": round(avg, 4), "launches_timed": int(cnt[i]), "share_of_step": round(ms_sum[i] / ms_prof, 4)}
        if name in alg_map:
            gbs = alg_map[name] / (avg * 1e-3) / 1e9
            row.update(alg_bytes=int(alg_map[name]), gbs=round(gbs, 1), frac_hbm=round(gbs / peak, 4))
        kernels[name] = row
    dom = max((k for k in kernels if k in alg_map), key=lambda k: kernels[k]["ms"])
    gpu = gpu_identity(dev)
    # pair statistics (instrumented re-run of the blend kernels, outside the timed region): the blend kernels are
    # bound by instruction issue over (pixel, Gaussian) pairs, so the pair rate is the roof that binds them
    pair = None
    try:
        ps = tr.blend_stats(view_for_step(sc.n_views, world, rank, 0))
        sm_clk = (clocks or {}).get("sm_mhz") or gpu["sm_max_mhz"] or 1980.0
        issue_peak = gpu["sm_count"] * 4 * sm_clk * 1e6    # warp instructions / s (4 schedulers per SM)
        pair = dict(ps)
        for d, kname in (("fwd", "blend_fwd"), ("bwd", "blend_bwd")):
            if kname in kernels:
                t = kernels[kname]["ms"] * 1e-3
                pair[f"{d}_pairs_per_s"] = ps[f"{d}_pairs_evaluated"] / t
                pair[f"{d}_warp_inst_per_64_pairs_at_full_issue"] = issue_peak * t / max(1, ps[f"{d}_warp_iters"])
        pair["issue_peak_warp_inst_per_s"] = issue_peak
        pair["note"] = ("pairs_evaluated = 64 x warp iterations (two 8x4 pixel blocks x one Gaussian); "
                        "warp_inst_per_64_pairs_at_full_issue = the instruction budget per iteration if every issue "
                        "slot were used: compare with the kernel's SASS count per iteration")
    except Exception as e:
        pair = {"error": f"{type(e).__name__}: {e}"}
    roof = {"bound": "hbm", "kernel": dom, "pairs": pair, "achieved": kernels[dom]["gbs"], "peak": peak, "unit": "GB/s",
            "frac": kernels[dom]["frac_hbm"], "peak_source": peak_src,
            "alg_bytes_per_launch": kernels[dom]["alg_bytes"], "ms_per_launch": kernels[dom]["ms"],
            "note": "algorithmic bytes = SURVEY.md 8(d) formulas with the measured R; the blend kernels are "
                    "bound by FP32/MUFU issue on (pixel,Gaussian) pairs, not by HBM (see DESIGN.md)"}
    t_render = sum(kernels[k]["ms"] for k in kernels if k not in ("loss_fwd", "loss_bwd", "adam"))
    torch_pieces = None
    if world == 1 and not args.no_cpu_baseline:
        try:
            torch_pieces = gpu_torch_pieces(sc, dev, tr.color, gt_dev[0])
            torch_pieces["ours_ms"] = {"preprocess_fwd+bwd (whole kernels, incl. EWA/SH)": kernels["preprocess"]["ms"] + kernels["preprocess_bwd"]["ms"],
                                       "loss_fwd+bwd": kernels["loss_fwd"]["ms"] + kernels["loss_bwd"]["ms"],
                                       "adam": kernels["adam"]["ms"]}
        except Exception as e:
            torch_pieces = {"error": f"{type(e).__name__}: {e}"}
    cpu_base = None
    if world == 1 and not args.no_cpu_baseline:
        try:
            c = cpu_arm(sc, 3, 1)
            cpu_base = {k: c[k] for k in ("value", "unit", "cores", "kind", "sample", "spread")}
        except Exception as e:          # never lose the GPU measurement to the CPU leg
            cpu_base = {"value": None, "unit": UNIT, "cores": os.cpu_count(), "kind": "port",
                        "sample": f"failed: {type(e).__name__}: {e}"}
    e2e_trainer = {"value": e2e_value, "unit": UNIT, "ms_per_step": ms_e2e / K,
                   "h2d_bytes_per_step": int(stage.numel() * 4), "d2h_bytes_per_step": 8,
                   "api": "JointTrainer.step(view, gt=<pinned host image, H2D on a copy stream, double buffered>) + "
                          "loss_value() D2H every step"}
    line = {
        "metric": METRIC, "value": value, "unit": UNIT, "n_gpus": world, "steps": K, "warmup": W_,
        "ms_per_step": ms_dev / K, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": "f32", "data": "synthetic",
        "config": {"workload": workload_name(args.config, sc), "views_per_step": world,
                   "parallelism": f"view-sharded dp{world}", "exchange": tr.exchange if world > 1 else "none", "P": sc.P, "R_mean": tr.last_R,
                   "launch_mode": ("CUDA-graph replay of the whole iteration (one graph per view); per-kernel table from "
                                   f"a second, eagerly launched timed region of {Kp} steps at {ms_prof / Kp:.3f} ms/step")
                   if use_graph else "eager launches",
                   "l2": f"working set (params+grads+moments 944 MB at 1M) exceeds the {gpu['l2_mb']:.0f} MB L2; "
                         "no explicit flush",
                   "iteration": "one view: render fwd + L1/DSSIM + bwd + per-point Adam (+ all-reduce if N>1)",
                   "scaling_note": "iters/s counts VIEWS; with N GPUs one optimizer step consumes N views (mean gradient) "
                                   "at the reference's per-view learning-rate schedule, so N-GPU numbers are throughput, "
                                   "not time-to-quality"},
        "render_mpix_per_s_fwd_bwd": sc.width * sc.height / (t_render * 1e-3) / 1e6,
        "e2e": e2e_plugin if e2e_plugin is not None else e2e_trainer,
        "e2e_trainer": e2e_trainer,
        "gpu_launches": launches, "gpu_launches_note": "every kernel on the path is libgsb200.so's own (no library sort/scan)",
        "dropin_boundary": dropin, "ref_python_pieces_gpu": torch_pieces, "kernels": kernels, "roofline": roof, "clocks": clocks, "cpu_baseline": cpu_base, "impl": "b200",
        "gpu": gpu,
    }
    if dumped is not None:
        write_outputs(args.dump_outputs, dumped)
        line["dumped_outputs"] = {k: [list(v.shape), str(v.dtype)] for k, v in dumped.items()}
    if world > 1:
        dist.destroy_process_group()
    return line


class _QuietStdout:
    """Libraries (NCCL's version banner, torchrun notices) must not pollute stdout: the contract is ONE JSON
    line.  Route fd 1 to stderr for the duration of the run and restore it for the final print."""

    def __enter__(self):
        sys.stdout.flush()
        self.saved = os.dup(1)
        os.dup2(2, 1)
        return self

    def __exit__(self, *exc):
        sys.stdout.flush()
        os.dup2(self.saved, 1)
        os.close(self.saved)


if __name__ == "__main__":
    a = parse()
    with _QuietStdout():
        line = run_reference(a) if a.impl == "reference" else run_b200(a)
    if line is not None:
        print(json.dumps(line), flush=True)
