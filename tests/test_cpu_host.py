"""CPU tests (-m "not gpu"): the C-ABI library loads and exports every symbol include/gsb200.h declares
(no compute without a GPU), host-side logic (LR schedule, view sharding, buffer sizing), the drop-in
shims import, and the N>1 exchange path under gloo with world_size 2."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_build_and_exports_match_header():
    import __graft_entry__ as G
    G.build()
    import instantsplat_b200 as I
    L = I.lib()
    hdr = open(os.path.join(ROOT, "include", "gsb200.h")).read()
    declared = set(re.findall(r"GSB_API [^;(]*?\b(gsb_\w+)\(", hdr))
    assert len(declared) >= 17
    for name in declared:
        assert hasattr(L, name), f"{name} declared in gsb200.h but not exported"
    assert set(I._lib.EXPORTS) == declared
    assert L.gsb_abi_version() == 2
    # sizing helpers are pure host code
    assert L.gsb_geom_bytes(1000) > 1000 * (16 * 3 + 48)
    assert L.gsb_binning_bytes(5000, 1920, 1080) > 5000 * 12
    assert L.gsb_image_bytes(1920, 1080) >= 2 * 4 * 1920 * 1080
    assert L.gsb_launch_count() == 0


def test_product_path_never_imports_oracle():
    for dirpath, _, files in os.walk(os.path.join(ROOT, "instantsplat_b200")):
        for f in files:
            if f.endswith(".py"):
                src = open(os.path.join(dirpath, f)).read()
                assert "oracle" not in re.sub(r'""".*?"""', "", src, flags=re.S), f"{f} references the oracle"


def test_no_cpu_fallback():
    import instantsplat_b200 as I
    a = torch.rand(1, 3, 8, 8)
    with pytest.raises(I.GsbError):
        I.fused_ssim(a, a)
    p = torch.nn.Parameter(torch.zeros(4, 3))
    p.grad = torch.ones(4, 3)
    with pytest.raises(I.GsbError):
        I.PerPointAdam([p], lr=1e-3).step()


def test_shims_import():
    sys.path.insert(0, os.path.join(ROOT, "shims"))
    try:
        import diff_gaussian_rasterization as d
        import fused_ssim as f
        from simple_knn._C import distCUDA2
        assert d.GaussianRasterizationSettings._fields == (
            "image_height", "image_width", "tanfovx", "tanfovy", "bg", "scale_modifier", "viewmatrix",
            "projmatrix", "sh_degree", "campos", "prefiltered", "debug")
        assert callable(f.fused_ssim) and callable(distCUDA2)
        pts = torch.rand(50, 3)
        d2 = distCUDA2(pts)
        ref = torch.cdist(pts, pts).pow(2).topk(4, largest=False).values[:, 1:].mean(1)
        assert torch.allclose(d2, ref, atol=1e-6)
    finally:
        sys.path.pop(0)


def test_lr_schedule_matches_reference_formula():
    from instantsplat_b200.trainer import get_expon_lr_func
    f = get_expon_lr_func(1.6e-4, 1.6e-6, lr_delay_mult=0.01, max_steps=30000)
    assert abs(f(0) - 1.6e-4) < 1e-12 and abs(f(30000) - 1.6e-6) < 1e-12
    assert abs(f(15000) - np.sqrt(1.6e-4 * 1.6e-6)) < 1e-12
    assert get_expon_lr_func(0.0, 0.0)(5) == 0.0 and f(-1) == 0.0


def test_view_sharding():
    from instantsplat_b200.parallel import shard_views, view_for_step
    assert shard_views(12, 4, 1) == [1, 5, 9]
    allv = sorted(v for r in range(8) for v in shard_views(24, 8, r))
    assert allv == list(range(24))
    assert [view_for_step(12, 4, 2, s) for s in range(4)] == [2, 6, 10, 2]
    assert view_for_step(3, 8, 5, 0) in range(3)          # more ranks than views
    with pytest.raises(ValueError):
        shard_views(4, 2, 2)


_WORKER = r'''
import os, sys, torch, torch.distributed as dist
sys.path.insert(0, sys.argv[1])
from instantsplat_b200.parallel import init_from_env, allreduce_sum_, view_for_step
rank, local, world = init_from_env("gloo")
assert world == 2
g = torch.Generator().manual_seed(100 + rank)
flat = torch.randn(1000, generator=g)
pose = torch.zeros(4, 7); pose[view_for_step(4, world, rank, 0)] = rank + 1.0
ref = sum(torch.randn(1000, generator=torch.Generator().manual_seed(100 + r)) for r in range(2))
allreduce_sum_((flat, pose))
assert torch.allclose(flat, ref), "flat gradient sum mismatch"
assert pose[0, 0] == 1.0 and pose[1, 0] == 2.0 and float(pose[2:].abs().sum()) == 0.0
dist.barrier(); dist.destroy_process_group()
print("rank", rank, "ok")
'''


def test_gloo_world2_gradient_exchange(tmp_path):
    script = tmp_path / "w.py"
    script.write_text(_WORKER)
    port = 29650 + os.getpid() % 200
    procs = []
    for r in range(2):
        env = dict(os.environ, RANK=str(r), LOCAL_RANK=str(r), WORLD_SIZE="2", MASTER_ADDR="127.0.0.1",
                   MASTER_PORT=str(port))
        procs.append(subprocess.Popen([sys.executable, str(script), ROOT], env=env, stdout=subprocess.PIPE,
                                      stderr=subprocess.STDOUT, text=True))
    outs = [p.communicate(timeout=120)[0] for p in procs]
    for r, (p, o) in enumerate(zip(procs, outs)):
        assert p.returncode == 0, o
        assert f"rank {r} ok" in o


def test_shard_bounds_cover_and_align():
    from instantsplat_b200.parallel import shard_bounds
    total = 59_000_123
    edges = [shard_bounds(total, 8, r) for r in range(8)]
    assert edges[0][0] == 0 and edges[-1][1] == total
    for (a, b), (c, d) in zip(edges[:-1], edges[1:]):
        assert b == c and a % 768 == 0 and c % 768 == 0
    assert shard_bounds(100, 4, 3) == (100, 100)          # tiny buffer: trailing shards are empty


def test_bench_reference_arm_prints_one_json_line():
    """`bench.py --impl reference` (the oracle port on the host cores) works without a GPU and prints exactly
    one JSON line on stdout with the contract keys."""
    import json
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--scale", "0.01",
                          "--steps", "1", "--warmup", "0"], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    lines = [l for l in out.stdout.splitlines() if l.strip()]
    assert len(lines) == 1
    d = json.loads(lines[0])
    for k in ("impl", "metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better",
              "cpu_baseline", "e2e", "config"):
        assert k in d, k
    assert d["impl"] == "reference" and d["cpu_baseline"]["kind"] == "port" and d["value"] > 0


def test_cpu_sample_plan_is_a_pure_function_and_never_tiny():
    """The CPU arm's per-step sample depends on the workload and the step count only (two runs time the same work), is
    the FULL sample for the runs the driver makes (<= 32 steps) and never shrinks below 1/8 of it."""
    import importlib.util
    spec = importlib.util.spec_from_file_location("bench_mod", os.path.join(ROOT, "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    import types
    sc = types.SimpleNamespace(P=1_000_000, width=1920, height=1080)
    full = bench.cpu_sample_plan(sc, 4)
    assert full == bench.cpu_sample_plan(sc, 4)
    assert full["n_gauss"] == sc.P and len(full["tiles"]) == 128 and full["rows"] == sc.height
    assert bench.cpu_sample_plan(sc, 25) == full                      # --steps 20 --warmup 5
    big = bench.cpu_sample_plan(sc, 1000)
    assert big["n_gauss"] * 8 >= sc.P and len(big["tiles"]) * 8 >= 128 and big["rows"] * 8 >= sc.height
    assert len(set(full["tiles"])) == 128 and max(full["tiles"]) < full["T"]


def test_debug_mode_writes_snapshot_of_failing_call(tmp_path, monkeypatch):
    """Upstream's Python wrapper dumps the arguments of a failing forward to snapshot_fw.dump in debug mode and
    re-raises (SURVEY.md section 8b, boundary B2 error behaviour)."""
    import instantsplat_b200 as I
    monkeypatch.chdir(tmp_path)
    eye = torch.eye(4)
    rs = I.GaussianRasterizationSettings(32, 32, 1.0, 1.0, torch.zeros(3), 1.0, eye, eye, 0, torch.zeros(3), False, True)
    bad = torch.zeros(5, 4)                       # means3D must be [P,3]
    with pytest.raises(RuntimeError):
        I.GaussianRasterizer(rs)(means3D=bad, means2D=torch.zeros(5, 3), opacities=torch.ones(5, 1),
                                 colors_precomp=torch.ones(5, 3), scales=torch.ones(5, 3), rotations=torch.ones(5, 4))
    dump = torch.load(tmp_path / "snapshot_fw.dump", weights_only=False)
    assert tuple(dump[0].shape) == (5, 4) and dump[-1][0] == 32


def test_scene_generation_does_not_depend_on_the_thread_count():
    """The synthetic scenes are the benchmark's and the tests' inputs: they must be bit-identical whatever the core
    count (large elementwise CPU ops are split into per-thread chunks that round transcendental functions differently)."""
    from instantsplat_b200.scenes import perturbed_copy, surface_scene
    n = torch.get_num_threads()
    out = []
    try:
        for threads in (1, 4, 7):
            torch.set_num_threads(threads)
            sc = surface_scene(300_000, 3, 320, 180, seed=11, sh_degree=3)
            out.append([sc.poses, sc.per_point_lr] + [sc.params[k] for k in sorted(sc.params)] +
                       [v for _, v in sorted(perturbed_copy(sc, sigma=0.05).items())])
    finally:
        torch.set_num_threads(n)
    assert torch.get_num_threads() == n
    for a, b, c in zip(*out):
        assert torch.equal(a, b) and torch.equal(a, c)
