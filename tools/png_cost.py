"""Cost of the GPU PNG encoder (png.py, gsb_png_encode_batch) against save_image's Pillow encoder, on one GPU:

  * encode: per-frame time at 512x512 and 1920x1080 on BASELINE configs[1] / configs[2] renders.  Pillow on 1 and 8
    threads (wall time over 16 frames); the GPU at V = 1, 4 and 16 frames per call, split into the kernels (CUDA
    events around gsb_png_encode_batch), the device-to-host copy of the used bytes (with its byte count) and the host
    framing (chunks and CRC-32), and png.encode end to end;
  * ratio: compressed bytes against Pillow's on those renders and on the two crops of tests/golden/png.npz;
  * freeview: `python -m instantsplat_b200.freeview` at configs[2] with 3 and 12 key views (201 and 276 frames), each
    encoder in its own process, the two alternated for --rounds rounds;
  * infer: `python -m instantsplat_b200.pipeline infer` over DESIGN.md section 4.18's tasks (C1a, C1b at configs[1],
    C2 at configs[2], --iterations) with each encoder, one process per view count, timed to the last file written
    (skipped with --no-infer).

Prints JSON lines, the last one holding everything, with the GPU's name and power limit read in the same run.
Usage: python tools/png_cost.py [--rounds 2] [--iterations 1000] [--no-infer]
"""
import argparse
import dataclasses
import io
import json
import os
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from instantsplat_b200 import _lib  # noqa: E402
from instantsplat_b200 import freeview as F  # noqa: E402
from instantsplat_b200 import png  # noqa: E402
from instantsplat_b200.scene_io import save_gaussians_ply, save_pose_npy, write_synthetic_source  # noqa: E402
from instantsplat_b200.scenes import make_config  # noqa: E402
from pipeline_cost import SCENES, device_info, last_file, write_source  # noqa: E402


def log(key, value):
    print(json.dumps({key: value}), flush=True)


def pil_bytes(img) -> bytes:
    from PIL import Image
    buf = io.BytesIO()
    Image.fromarray(img).save(buf, "PNG")
    return buf.getvalue()


def renders(idx, n):
    sc = make_config(idx)
    tk = F.tracker_from_gaussians(sc.params, sc.width, sc.height, sc.fovx, sc.fovy, False, "cuda")
    poses = sc.poses[torch.arange(n) % sc.n_views] + 0.01 * torch.randn(n, 7, generator=torch.Generator().manual_seed(1))
    out = np.concatenate([c for _, c in F.frames_u8(tk, poses, max_batch=4)])
    del tk
    torch.cuda.empty_cache()
    return out


def gpu_split(frames, V, reps=5):
    """ms per frame: kernels (events), device-to-host copy of the used bytes, host framing; and bytes copied."""
    L = _lib.lib()
    x = torch.from_numpy(frames[:V]).cuda()
    _, H, W, _ = x.shape
    nb = L.gsb_png_bound(H, W)
    scratch = torch.empty(L.gsb_png_scratch_bytes(V, H, W), dtype=torch.uint8, device="cuda")
    out = torch.empty(V, nb, dtype=torch.uint8, device="cuda")
    sizes = torch.empty(V, dtype=torch.int64, device="cuda")
    run = lambda: _lib.check(L.gsb_png_encode_batch(V, H, W, x.data_ptr(), scratch.data_ptr(), scratch.numel(),
                                                    out.data_ptr(), sizes.data_ptr(), _lib.stream_ptr()), "encode")
    run()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        run()
    e1.record()
    torch.cuda.synchronize()
    kern = e0.elapsed_time(e1) / reps
    t0 = time.perf_counter()
    for _ in range(reps):
        n = sizes.cpu().tolist()
        streams = [out[v, :n[v]].cpu().numpy().tobytes() for v in range(V)]
    d2h = (time.perf_counter() - t0) * 1e3 / reps
    t0 = time.perf_counter()
    for _ in range(reps):
        [png.png_file(H, W, s) for s in streams]
    host = (time.perf_counter() - t0) * 1e3 / reps
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        png.encode(x)
    e2e = (time.perf_counter() - t0) * 1e3 / reps
    return dict(kernels_ms=round(kern / V, 3), d2h_ms=round(d2h / V, 3), d2h_bytes=int(sum(n)) // V,
                framing_ms=round(host / V, 3), encode_ms=round(e2e / V, 3))


def encode_costs(frames):
    r = {}
    for threads in (1, 8):
        with ThreadPoolExecutor(threads) as pool:
            t0 = time.perf_counter()
            list(pool.map(pil_bytes, frames))
            r[f"pil_{threads}_threads_ms"] = round((time.perf_counter() - t0) * 1e3 / len(frames), 2)
    for V in (1, 4, 16):
        r[f"gpu_V{V}"] = gpu_split(frames, V)
    ours = sum(map(len, png.encode_host(frames)))
    pil = sum(len(pil_bytes(f)) for f in frames)
    r["ratio_vs_pil"] = round(ours / pil, 4)
    return r


def freeview_cli(tmp, rounds):
    sc = make_config(2)
    keys_all = save_pose_npy(os.path.join(tmp, "keys.npy"), sc.poses.numpy())
    p = {k: v.numpy() for k, v in sc.params.items()}
    res = {}
    for n in (3, 12):
        src, mdir = os.path.join(tmp, f"fv_src{n}"), os.path.join(tmp, f"fv_model{n}")
        write_synthetic_source(src, dataclasses.replace(sc, poses=sc.poses[:n].clone()))
        save_gaussians_ply(os.path.join(mdir, "point_cloud", "iteration_1000", "point_cloud.ply"), p["xyz"], p["f_dc"],
                           p["f_rest"], p["opacity"], p["scaling"], p["rotation"])
        os.makedirs(os.path.join(mdir, "pose", "ours_1000"))
        np.save(os.path.join(mdir, "pose", "ours_1000", "pose_optimized.npy"), keys_all[:n])
        res[n] = {"pil": [], "gpu": []}
        folder = os.path.join(mdir, "interp", "ours_1000", "renders")
        for _ in range(rounds):
            for enc in ("pil", "gpu"):
                t0 = time.perf_counter()
                subprocess.run([sys.executable, "-m", "instantsplat_b200.freeview", "-s", src, "-m", mdir, "--n_views",
                                str(n), "--iterations", "1000", "--max_batch", "16", "--png_encoder", enc], cwd=ROOT,
                               stdout=subprocess.DEVNULL, check=True)
                res[n][enc].append(round(time.perf_counter() - t0, 2))
                res[n][f"{enc}_bytes"] = sum(os.path.getsize(os.path.join(folder, f)) for f in os.listdir(folder))
        log(f"freeview_views{n}", res[n])
    return res


def infer(tmp, iterations):
    root = os.path.join(tmp, "infer_root")
    views = {}
    for idx in (1, 2):
        views[idx] = write_source(idx, os.path.join(tmp, f"src{idx}"))["views"]
    for name, idx in SCENES:
        os.makedirs(os.path.join(root, "D"), exist_ok=True)
        os.symlink(os.path.join(tmp, f"src{idx}"), os.path.join(root, "D", name))
    res = {}
    for enc in ("pil", "gpu"):
        out = os.path.join(tmp, f"infer_{enc}")
        start = time.time()
        argv = ["infer", "--data_root", root, "--output_dir", out, "--datasets", "D", "--workers", "8",
                "--png_encoder", enc, "--iterations", str(iterations)]
        # one process per view count, as the scripts' loop would need (configs[1] and configs[2] differ in views)
        for scenes, n in ((["C1a", "C1b"], views[1]), (["C2"], views[2])):
            subprocess.run([sys.executable, "-m", "instantsplat_b200.pipeline", *argv, "--scenes", *scenes,
                            "--n_views", str(n)], cwd=ROOT, stdout=subprocess.DEVNULL, check=True)
        res[enc] = dict(wall_s=round(last_file(out) - start, 2))
        log(f"infer_{enc}", res[enc])
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--iterations", type=int, default=1000)
    ap.add_argument("--no-infer", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("png_cost.py needs a CUDA device")
    info = dict(gpu=torch.cuda.get_device_name(0), name_power_limit_max_sm_clock=device_info(), host_cpus=os.cpu_count())
    log("device", info)
    for idx in (1, 2):
        frames = renders(idx, 16)
        key = f"configs{idx}_{frames.shape[1]}x{frames.shape[2]}"
        info[key] = encode_costs(frames)
        log(key, info[key])
    g = np.load(os.path.join(ROOT, "tests", "golden", "png.npz"))
    info["crops_ratio_vs_pil"] = {k: round(len(png.encode_host(g[f"{k}_crop"][None])[0]) / int(g[f"{k}_pil_bytes"]), 4)
                                  for k in ("santorini", "art")}
    log("crops", info["crops_ratio_vs_pil"])
    subprocess.run([sys.executable, "-c", "import instantsplat_b200 as I; I.lib(); import torch; torch.zeros(1).cuda()"],
                   cwd=ROOT, check=True)
    with tempfile.TemporaryDirectory() as tmp:
        info["freeview_cli_s"] = freeview_cli(tmp, a.rounds)
        if not a.no_infer:
            info["infer"] = infer(tmp, a.iterations)
    print(json.dumps(info))
    return 0


if __name__ == "__main__":
    sys.exit(main())
