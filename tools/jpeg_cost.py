"""Cost of decoding JPEG source images with Pillow (one thread, one file at a time, as scene_io.load_views does) and
on the GPU (jpeg.decode_u8, --jpeg_decoder gpu), batches of 12 files:

  * pillow: np.array(Image.open(path)) of each file, summed over the batch;
  * gpu_e2e: decode_u8 of the 12 paths (file reads, marker parsing, upload, decode, status read), a host clock around
    work that ends in a device synchronise;
  * gpu_kernels: the gsb_jpeg_decode_batch call alone with the entropy bytes already on the device, CUDA events;
  * the cases: 1280x720, 1920x1080 and 4032x3024, 4:2:0 and 4:4:4, q75 and q95, with and without a restart marker
    per MCU row; every GPU decode is checked against Pillow's bytes first;
  * subseq: gpu_kernels at 4032x3024 q95 4:2:0 without restart markers for several subsequence sizes;
  * loader: scene_io.load_views of 12 JPEG views (4032x3024 q95 4:2:0) end to end with and without decode_device,
    and train's `load` phase (train.load_host_scene, what train.run times as `load`) with and without it.

Rounds alternate the ways; medians over --rounds with min and max.  Prints JSON lines, the last one holding
everything, with the GPU's name, power limit and SM clock read in the same run; with --out the last one is also
written to that file.
Usage: python tools/jpeg_cost.py [--rounds 5] [--sizes 1280x720,1920x1080,4032x3024] [--quick] [--out FILE]
"""
import argparse
import json
import os
import statistics
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from instantsplat_b200 import _lib, jpeg as J  # noqa: E402
from instantsplat_b200 import scene_io as S  # noqa: E402
from instantsplat_b200 import train as T  # noqa: E402
from pipeline_cost import device_info  # noqa: E402

N = 12
SIZES = ((1280, 720), (1920, 1080), (4032, 3024))


def log(key, value):
    print(json.dumps({key: value}), flush=True)


def stat(xs):
    return dict(median=statistics.median(xs), min=min(xs), max=max(xs), n=len(xs))


def images(w, h):
    """12 distinct photo-like views: a smooth field, texture and edges, shifted per view."""
    rng = np.random.default_rng(w * h)
    y, x = np.mgrid[0:h, 0:w].astype(np.float32)
    base = np.stack([128 + 90 * np.sin(x / (50 + 30 * c)) * np.cos(y / (70 - 20 * c)) for c in range(3)], -1)
    base += rng.normal(0, 12, base.shape).astype(np.float32)
    base = np.clip(base, 0, 255).astype(np.uint8)
    return [np.roll(base, (37 * v, 53 * v), (0, 1)) for v in range(N)]


def encode(arrs, folder, tag, ss, q, rst):
    from PIL import Image
    paths = []
    for v, a in enumerate(arrs):
        p = os.path.join(folder, f"{tag}_{v:02d}.jpg")
        kw = {"restart_marker_rows": 1} if rst else {}
        Image.fromarray(a).save(p, "JPEG", quality=q, subsampling=ss, **kw)
        paths.append(p)
    return paths


def pillow(paths):
    from PIL import Image
    t0 = time.perf_counter()
    out = []
    for p in paths:
        with Image.open(p) as im:
            out.append(np.array(im))
    return time.perf_counter() - t0, out


def gpu_e2e(paths):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out, routes = J.decode_u8(paths, "cuda", return_routes=True)
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out, routes


class Kernels:
    """gsb_jpeg_decode_batch on one batch with its inputs on the device, timed with CUDA events."""

    def __init__(self, paths, subseq_bits=J.SUBSEQ_BITS):
        datas = [open(p, "rb").read() for p in paths]
        parsed = [J.parse(d) for d in datas]
        self.S = subseq_bits
        self.files, total = J._table(list(range(len(paths))), parsed)
        sizes = [p.height * p.width * 3 for p in parsed]
        offs = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int64)
        for k in range(len(paths)):
            self.files[k].out_offset = int(offs[k])
        stream = np.concatenate([np.frombuffer(d, np.uint8)[p.scan_begin:p.scan_end] for d, p in zip(datas, parsed)])
        self.host = torch.from_numpy(stream).pin_memory()
        self.data = self.host.cuda()
        self.out = torch.empty(sum(sizes), dtype=torch.uint8, device="cuda")
        L = _lib.lib()
        self.nb = L.gsb_jpeg_scratch_bytes(len(paths), self.files, subseq_bits)
        self.scratch = torch.empty(self.nb + 256, dtype=torch.uint8, device="cuda")
        self.status = torch.empty(len(paths), dtype=torch.int32, device="cuda")
        self.n = len(paths)

    def run(self, upload=False):
        L = _lib.lib()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        if upload:
            self.data.copy_(self.host, non_blocking=True)
        _lib.check(L.gsb_jpeg_decode_batch(self.n, self.files, self.data.data_ptr(), self.S,
                                           (self.scratch.data_ptr() + 255) & ~255, self.nb, self.out.data_ptr(),
                                           self.status.data_ptr(), _lib.stream_ptr()), "gsb_jpeg_decode_batch")
        e1.record()
        torch.cuda.synchronize()
        assert not any(self.status.cpu().tolist())
        return e0.elapsed_time(e1) / 1e3


def case(arrs, tmp, tag, ss, q, rst, rounds):
    paths = encode(arrs, tmp, tag, ss, q, rst)
    _, ref = pillow(paths)
    _, got, routes = gpu_e2e(paths)                               # warm-up, and the bytes checked
    assert routes == ["gpu"] * N and all(np.array_equal(g.cpu().numpy(), r) for g, r in zip(got, ref))
    del got
    k = Kernels(paths)
    k.run()
    rows = dict(pillow=[], gpu_e2e=[], gpu_kernels=[], gpu_kernels_upload=[])
    for _ in range(rounds):
        rows["pillow"].append(pillow(paths)[0])
        rows["gpu_e2e"].append(gpu_e2e(paths)[0])
        rows["gpu_kernels"].append(k.run())
        rows["gpu_kernels_upload"].append(k.run(upload=True))
    mb = sum(os.path.getsize(p) for p in paths) / 1e6
    res = {key: stat(v) for key, v in rows.items()}
    res.update(file_mb=mb, scratch_mb=k.nb / 1e6)
    for p in paths:
        os.remove(p)
    return res


def subseq_sweep(arrs, tmp, rounds):
    paths = encode(arrs, tmp, "sweep", 2, 95, False)
    out = {}
    for S_ in (256, 512, 1024, 2048, 4096, 8192):
        k = Kernels(paths, S_)
        k.run()
        out[S_] = stat([k.run() for _ in range(rounds)])
        del k
    return out


def loader(arrs, tmp, rounds):
    """load_views and train's load phase on a 12-view JPEG source (4:2:0 q95)."""
    from instantsplat_b200.scenes import surface_scene
    h, w = arrs[0].shape[:2]
    src = os.path.join(tmp, "src")
    sc = surface_scene(2000, N, w, h, seed=3, sh_degree=3)
    S.write_synthetic_source(src, sc)
    import math
    fx = w / (2.0 * math.tan(sc.fovx / 2.0))
    fy = h / (2.0 * math.tan(sc.fovy / 2.0))
    names = [f"{i:06d}.jpg" for i in range(N)]
    S.write_colmap_text(os.path.join(src, f"sparse_{N}", "0"), w, h, fx, fy, sc.poses.numpy(), names)
    os.makedirs(os.path.join(src, "images"), exist_ok=True)
    from PIL import Image
    for i, a in enumerate(arrs):
        Image.fromarray(a).save(os.path.join(src, "images", names[i]), "JPEG", quality=95)
    ways = {"load_views_pil": lambda: S.load_views(src, N, 0, 1),
            "load_views_gpu": lambda: S.load_views(src, N, 0, 1, decode_device="cuda"),
            "train_load_pil": lambda: T.load_host_scene(src, N, 1),
            "train_load_gpu": lambda: T.load_host_scene(src, N, 1, decode_device="cuda")}
    a, b = ways["load_views_pil"](), ways["load_views_gpu"]()
    assert np.array_equal(a.images, b.images)
    rows = {k: [] for k in ways}
    for _ in range(rounds):
        for key, f in ways.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            f()
            torch.cuda.synchronize()
            rows[key].append(time.perf_counter() - t0)
    return {k: stat(v) for k, v in rows.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--sizes", default=",".join(f"{w}x{h}" for w, h in SIZES),
                    help="comma-separated WxH; the subsequence sweep and the loader run at 4032x3024")
    ap.add_argument("--quick", action="store_true", help="the first size only, one case each way")
    ap.add_argument("--out", default=None, help="also write the results as JSON to this file")
    a = ap.parse_args()
    sizes = [tuple(int(v) for v in s.split("x")) for s in a.sizes.split(",")]
    res = {"device": device_info(), "torch_device": torch.cuda.get_device_name(0), "batch": N,
           "subseq_bits": J.SUBSEQ_BITS}
    log("device", res["device"])
    with tempfile.TemporaryDirectory() as tmp:
        for w, h in sizes[:1] if a.quick else sizes:
            arrs = images(w, h)
            for ss in (2, 0):
                for q in (75, 95):
                    for rst in (False, True):
                        if a.quick and (q, rst) != (95, False):
                            continue
                        key = f"{w}x{h}_{'420' if ss == 2 else '444'}_q{q}{'_rst' if rst else ''}"
                        res[key] = case(arrs, tmp, key, ss, q, rst, a.rounds)
                        log(key, res[key])
            if w == 4032 or a.quick:
                res["subseq"] = subseq_sweep(arrs, tmp, a.rounds)
                log("subseq", res["subseq"])
            if w == 4032 or a.quick:
                res[f"loader_{w}x{h}"] = loader(arrs, tmp, a.rounds)
                log(f"loader_{w}x{h}", res[f"loader_{w}x{h}"])
            del arrs
    log("all", res)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
