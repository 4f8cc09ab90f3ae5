"""Cost of the GPU resize (resample.py, gsb_resample_u8_batch) against Pillow's, on one GPU, with V = 12 views:

  * pillow: Image.resize of each view on one thread (PILtoTorch's call), milliseconds per view;
  * kernel: resample.resize_u8 of the 12 uploaded views in one call (its table upload included), CUDA events around
    each call after 3 warm-up calls, and the bytes it reads and writes over that time;
  * load_views: scene_io.load_views of 12 PNG files (written by Pillow at compress_level 1) with
    resample_device="cuda", against the same call at -r 1 (decode only) and the decode followed by Pillow's resize
    of every view on one thread, each end to end on the host clock.

Cases: 1920x1080 at -r -1; 4032x3024 at -r -1, -r 2 and -r 8.  Each number is the median of --rounds rounds; the
rounds are printed too.  Prints JSON lines, the last one holding everything, with the GPU's name and power limit read
in the same run.
Usage: python tools/resample_cost.py [--rounds 3]
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

from instantsplat_b200 import resample  # noqa: E402
from instantsplat_b200 import scene_io as S  # noqa: E402

V = 12
CASES = [((1920, 1080), -1), ((4032, 3024), -1), ((4032, 3024), 2), ((4032, 3024), 8)]


def device_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                              "0"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        return None


def log(key, value):
    print(json.dumps({key: value}), flush=True)


def views(W, H, seed):
    """V smooth, noisy uint8 [H, W, 3] images: photo-like enough that PNG decoding is not trivial."""
    rng = np.random.default_rng(seed)
    y = np.linspace(0, 1, H, dtype=np.float32)[:, None, None]
    x = np.linspace(0, 1, W, dtype=np.float32)[None, :, None]
    out = []
    for v in range(V):
        f = rng.uniform(2, 12, 3).astype(np.float32)
        base = 127.5 + 100 * np.sin(f * x * 6.3 + v) * np.cos(f * y * 4.1)
        out.append(np.clip(base + rng.normal(0, 12, (H, W, 3)).astype(np.float32), 0, 255).astype(np.uint8))
    return np.stack(out)


def write_source(root, imgs):
    from PIL import Image
    H, W = imgs.shape[1:3]
    names = [f"{i:03d}.png" for i in range(V)]
    poses = np.concatenate([np.tile([1.0, 0, 0, 0], (V, 1)), np.zeros((V, 3))], axis=1)
    S.write_colmap_text(os.path.join(root, f"sparse_{V}", "0"), W, H, 0.8 * W, 0.8 * W, poses, names)
    os.makedirs(os.path.join(root, "images"), exist_ok=True)
    for n, a in zip(names, imgs):
        Image.fromarray(a).save(os.path.join(root, "images", n), compress_level=1)


def pillow_ms(imgs, size):
    from PIL import Image
    pil = [Image.fromarray(a) for a in imgs]
    t = time.perf_counter()
    for im in pil:
        im.resize(size)
    return (time.perf_counter() - t) * 1e3 / len(pil)


def kernel_ms(dev_imgs, size, reps=10):
    for _ in range(3):
        resample.resize_u8(dev_imgs, size)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        resample.resize_u8(dev_imgs, size)
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def load_s(src, r, dev):
    t = time.perf_counter()
    v = S.load_views(src, V, 0, r, resample_device=dev)
    if dev is not None:
        torch.cuda.synchronize()
    return time.perf_counter() - t, v


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    info = dict(gpu=torch.cuda.get_device_name(0), name_power_limit_max_sm_clock=device_info(), host_cpus=os.cpu_count(),
                rounds=a.rounds, views=V)
    log("device", info)
    results = []
    with tempfile.TemporaryDirectory() as tmp:
        made = {}
        for (W, H), r in CASES:
            if (W, H) not in made:
                imgs = views(W, H, seed=W)
                src = os.path.join(tmp, f"{W}x{H}")
                write_source(src, imgs)
                made[(W, H)] = (imgs, src, torch.from_numpy(imgs).cuda())
            imgs, src, dev_imgs = made[(W, H)]
            size = S.loaded_size(W, H, r)
            got = resample.resize_u8(dev_imgs, size).cpu().numpy()
            from PIL import Image
            exact = all(np.array_equal(got[v], np.asarray(Image.fromarray(imgs[v]).resize(size))) for v in range(V))
            rounds = []
            for _ in range(a.rounds):
                k = kernel_ms(dev_imgs, size)
                p = pillow_ms(imgs, size)
                t_gpu, _ = load_s(src, r, "cuda")
                t_dec, dec = load_s(src, 1, None)
                t0 = time.perf_counter()
                pillow_ms(dec.images, size)
                t_host = t_dec + (time.perf_counter() - t0)
                rounds.append(dict(kernel_ms=k, pillow_ms_per_view=p, load_views_gpu_s=t_gpu, load_views_decode_s=t_dec,
                                   decode_then_pillow_s=t_host))
            med = {key: statistics.median(x[key] for x in rounds) for key in rounds[0]}
            moved = V * (W * H * 3 + size[0] * size[1] * 3 + (H * size[0] * 3 * 2 if size[0] != W and size[1] != H else 0))
            res = dict(source=[W, H], r=r, loaded=list(size), bytes_equal_pillow=exact, median=med, rounds=rounds,
                       kernel_bytes=moved, kernel_GBps=moved / (med["kernel_ms"] * 1e-3) / 1e9,
                       pillow_ms_all_views=med["pillow_ms_per_view"] * V)
            log("case", res)
            results.append(res)
            torch.cuda.empty_cache()
    log("all", dict(device=info, cases=results))


if __name__ == "__main__":
    main()
