"""Cost of writing and reading point_cloud.ply the numpy way (scene_io) and on the GPU (ply.py, --ply_io gpu), on one
GPU, at the model sizes the train CLI writes for BASELINE configs[1] (200k Gaussians) and configs[2] (1M), degree-3
records (248 bytes each):

  * write_numpy: save_gaussians_ply split into d2h (each tensor's .cpu()), concat (the [P, 62] np.concatenate),
    columns (62 strided assignments into the structured array), tobytes and write (the header and the body);
  * write_gpu: ply.save split into pack (gsb_ply_pack), copy (device to pinned host) and write, summed over chunks;
  * read_numpy: load_gaussians_ply split into read (the file into a structured array), columns (the np.stack per field
    group and the transposes) and h2d (each tensor to the device, as the tracker uploads them);
  * read_gpu: ply.load split into read (readinto the pinned buffer), copy (pinned to device) and unpack;
  * each end to end, and `fsync` of the written file (what making it durable would add, not part of either writer);
  * cli: the train CLI's `saves` phase (train.run, --iterations, save at the last one) and `render_views --eval` as a
    process (end to end), each with and without --ply_io gpu.

Rounds alternate the two ways; medians over --rounds.  Prints JSON lines, the last one holding everything, with the
GPU's name, power limit and SM clock read in the same run.
Usage: python tools/ply_cost.py [--rounds 5] [--cli_rounds 2] [--iterations 1000] [--no-cli]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from instantsplat_b200 import ply  # noqa: E402
from instantsplat_b200 import scene_io as S  # noqa: E402
from instantsplat_b200 import train as T  # noqa: E402
from pipeline_cost import device_info, write_source  # noqa: E402

SIZES = ((1, 200_000), (2, 1_000_000))


def log(key, value):
    print(json.dumps({key: value}), flush=True)


def now(sync=False):
    if sync:
        torch.cuda.synchronize()
    return time.perf_counter()


def tensors(P):
    g = torch.Generator(device="cuda").manual_seed(P)
    shapes = dict(xyz=(3,), f_dc=(1, 3), f_rest=(15, 3), opacity=(1,), scaling=(3,), rotation=(4,))
    return {k: torch.randn(P, *s, generator=g, device="cuda") for k, s in shapes.items()}


def write_numpy(path, t):
    s = {}
    t0 = now(True)
    h = {k: v.cpu().numpy() for k, v in t.items()}
    t1 = now()
    P = h["xyz"].shape[0]
    cm = lambda a: a.reshape(P, -1, 3).transpose(0, 2, 1).reshape(P, -1)
    attrs = np.concatenate([h["xyz"], np.zeros_like(h["xyz"]), cm(h["f_dc"]), cm(h["f_rest"]), h["opacity"],
                            h["scaling"], h["rotation"]], axis=1)
    t2 = now()
    fields = [(n, "f4") for n in S.gaussian_ply_fields(45)]
    arr = np.empty(P, dtype=np.dtype([(n, "<f4") for n, _ in fields]))
    for (n, _), i in zip(fields, range(attrs.shape[1])):
        arr[n] = attrs[:, i]
    t3 = now()
    body = arr.tobytes()
    t4 = now()
    with open(path, "wb") as f:
        f.write(S._ply_header(P, fields))
        f.write(body)
    t5 = now()
    s.update(d2h=t1 - t0, concat=t2 - t1, columns=t3 - t2, tobytes=t4 - t3, write=t5 - t4, total=t5 - t0)
    return s


def write_gpu(path, t):
    P = t["xyz"].shape[0]
    rec = 248
    per = min(ply.CHUNK_BYTES // rec, P)
    s = dict(pack=0.0, copy=0.0, write=0.0)
    t0 = now(True)
    stage = torch.empty(per * rec, dtype=torch.uint8, device="cuda")
    host = ply._pinned(per * rec)
    view = memoryview(host.numpy())
    ta = now(True)
    with open(path, "wb") as f:
        f.write(S.gaussian_ply_header(P, 45, False))
        for first in range(0, P, per):
            k = min(per, P - first)
            a = now()
            ply.pack(t, stage, first, k)
            b = now(True)
            host[:k * rec].copy_(stage[:k * rec], non_blocking=True)
            c = now(True)
            f.write(view[:k * rec])
            d = now()
            s["pack"] += b - a
            s["copy"] += c - b
            s["write"] += d - c
    s["buffers"] = ta - t0
    s["total"] = now() - t0
    return s


def read_numpy(path):
    t0 = now(True)
    d = S._read_ply(path)
    t1 = now()
    P = d.shape[0]
    col = lambda prefix: np.stack([d[n] for n in sorted((n for n in d.dtype.names if n.startswith(prefix)),
                                                        key=lambda s: int(s.split("_")[-1]))], axis=1)
    rest = col("f_rest_")
    out = dict(xyz=np.stack([d["x"], d["y"], d["z"]], axis=1), f_dc=col("f_dc_").reshape(P, 3, 1).transpose(0, 2, 1).copy(),
               f_rest=rest.reshape(P, 3, rest.shape[1] // 3).transpose(0, 2, 1).copy(),
               opacity=d["opacity"].reshape(P, 1).copy(), scaling=col("scale_"), rotation=col("rot_"))
    t2 = now()
    g = {k: torch.from_numpy(np.ascontiguousarray(v)).to("cuda") for k, v in out.items()}
    t3 = now(True)
    return dict(read=t1 - t0, columns=t2 - t1, h2d=t3 - t2, total=t3 - t0), g


def read_gpu(path):
    P, n_rest, filt, offset = ply.layout(path)
    rec = 248
    per = min(ply.CHUNK_BYTES // rec, P)
    s = dict(read=0.0, copy=0.0, unpack=0.0)
    t0 = now(True)
    out = {k: torch.empty(P, *sh, device="cuda") for k, sh in
           dict(xyz=(3,), f_dc=(1, 3), f_rest=(15, 3), opacity=(1,), scaling=(3,), rotation=(4,)).items()}
    stage = torch.empty(per * rec, dtype=torch.uint8, device="cuda")
    host = ply._pinned(per * rec)
    view = memoryview(host.numpy())
    with open(path, "rb") as f:
        f.seek(offset)
        for first in range(0, P, per):
            k = min(per, P - first)
            a = now()
            f.readinto(view[:k * rec])
            b = now()
            stage[:k * rec].copy_(host[:k * rec], non_blocking=True)
            c = now(True)
            ply.unpack(stage, out, first, k)
            d = now(True)
            s["read"] += b - a
            s["copy"] += c - b
            s["unpack"] += d - c
    s["total"] = now() - t0
    return s, out


def med(rows):
    return {k: statistics.median(r[k] for r in rows) for k in rows[0]}


def io_costs(P, rounds, tmp):
    t = tensors(P)
    a, b = os.path.join(tmp, "numpy.ply"), os.path.join(tmp, "gpu.ply")
    rows = {k: [] for k in ("write_numpy", "write_gpu", "read_numpy", "read_gpu", "save_numpy", "save_gpu",
                            "load_numpy", "load_gpu", "fsync")}
    for _ in range(rounds + 1):                       # round 0 warms up (pinned allocator, page cache, kernels)
        r = dict(write_numpy=write_numpy(a, t), write_gpu=write_gpu(b, t))
        assert open(a, "rb").read() == open(b, "rb").read()
        r["read_numpy"], g0 = read_numpy(a)
        r["read_gpu"], g1 = read_gpu(b)
        assert all(torch.equal(g0[k], g1[k]) for k in g0)
        t0 = now(True)
        S.save_gaussians_ply(a, *(t[k].cpu().numpy() for k in ("xyz", "f_dc", "f_rest", "opacity", "scaling",
                                                               "rotation")))
        t1 = now()
        ply.save(b, t)
        t2 = now()
        S.load_gaussians_ply(a)
        t3 = now()
        ply.load(b)
        t4 = now(True)
        fd = os.open(b, os.O_RDONLY)
        os.fsync(fd)
        os.close(fd)
        t5 = now()
        r.update(save_numpy=dict(total=t1 - t0), save_gpu=dict(total=t2 - t1), load_numpy=dict(total=t3 - t2),
                 load_gpu=dict(total=t4 - t3), fsync=dict(total=t5 - t4))
        if _:
            for k, v in r.items():
                rows[k].append(v)
    return {k: med(v) for k, v in rows.items()}


def cli_costs(idx, iterations, rounds, tmp):
    src = os.path.join(tmp, f"src{idx}")
    info = write_source(idx, src)
    n = info["views"]
    out = dict(saves={"numpy": [], "gpu": []}, render_eval={"numpy": [], "gpu": []})
    models = {}
    for r in range(rounds):
        for io in (("numpy", "gpu") if r % 2 == 0 else ("gpu", "numpy")):
            m = os.path.join(tmp, f"m{idx}_{io}_{r}")
            argv = ["-s", src, "-m", m, "-r", "1", "--n_views", str(n), "--iterations", str(iterations),
                    "--pp_optimizer", "--optim_pose", "--quiet"] + (["--ply_io", "gpu"] if io == "gpu" else [])
            res = T.run(T.parse_args(argv))
            out["saves"][io].append(res.phases["saves"])
            del res
            torch.cuda.empty_cache()
            models[io] = m
    ply_a = os.path.join(models["numpy"], "point_cloud", f"iteration_{iterations}", "point_cloud.ply")
    ply_b = os.path.join(models["gpu"], "point_cloud", f"iteration_{iterations}", "point_cloud.ply")
    same = open(ply_a, "rb").read() == open(ply_b, "rb").read()
    for r in range(rounds):
        for io in (("numpy", "gpu") if r % 2 == 0 else ("gpu", "numpy")):
            argv = [sys.executable, "-m", "instantsplat_b200.render_views", "-s", src, "-m", models["numpy"],
                    "--n_views", str(n), "--iterations", str(iterations), "-r", "1", "--eval"] \
                + (["--ply_io", "gpu"] if io == "gpu" else [])
            t0 = time.perf_counter()
            subprocess.run(argv, cwd=ROOT, check=True, capture_output=True)
            out["render_eval"][io].append(time.perf_counter() - t0)
    return dict(source=info, same_ply=same, **{k: {io: dict(median=statistics.median(v), all=v) for io, v in d.items()}
                                               for k, d in out.items()})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--cli_rounds", type=int, default=2)
    ap.add_argument("--iterations", type=int, default=1000)
    ap.add_argument("--no-cli", dest="cli", action="store_false")
    a = ap.parse_args()
    res = dict(device=device_info(), rounds=a.rounds, chunk_bytes=ply.CHUNK_BYTES, io={}, cli={})
    log("device", res["device"])
    with tempfile.TemporaryDirectory() as tmp:
        for idx, P in SIZES:
            res["io"][f"configs[{idx}]"] = io_costs(P, a.rounds, tmp)
            log(f"io configs[{idx}]", res["io"][f"configs[{idx}]"])
        if a.cli:
            for idx, _ in SIZES:
                res["cli"][f"configs[{idx}]"] = cli_costs(idx, a.iterations, a.cli_rounds, tmp)
                log(f"cli configs[{idx}]", res["cli"][f"configs[{idx}]"])
    log("ply_cost", res)


if __name__ == "__main__":
    main()
