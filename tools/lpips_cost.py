"""Cost of LPIPS (VGG) for 12 pairs at 288x512 (the evaluation size) and at 1080x1920, on seeded random weights
(oracle.lpips_oracle.seeded_weights) and random image pairs:

  * ours: LpipsVGG end to end (12 pairs, max_batch 4), ending in a device synchronise;
  * layers: each conv layer's kernel alone (gsb_lpips_conv3x3_relu on the activation shape of 8 images, CUDA events
    over repeated launches), its FLOPs from the shapes (2 * pixels * Cout * 9 * Cin) and the achieved rate as a share
    of the H100 SXM data sheet's 67 TFLOP/s dense FP32 (a data-sheet figure, for a card allowed 700 W);
  * cudnn_fp32 / cudnn_tf32: the same network through torch's conv2d (cuDNN, NCHW) with TF32 off and on.  TF32 on is
    the reference's default (torch.backends.cudnn.allow_tf32 is True), so the largest |LPIPS(tf32) - LPIPS(ours)| says
    how comparable our numbers are to a reference run;
  * reference_loop: the shape of lpips() in metrics.py's loop: per pair, both weight files loaded and the network
    rebuilt and moved to the GPU, then one forward in fp32 with TF32 on;
  * cli: `python -m instantsplat_b200.metrics` on 12 PNG pairs, with and without --lpips_weights.

Prints one JSON line with the GPU's name and power limit.  Usage: python tools/lpips_cost.py [--rounds 3]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import instantsplat_b200 as I  # noqa: E402
from instantsplat_b200 import lpips as LP  # noqa: E402
from instantsplat_b200 import metrics as M  # noqa: E402
from oracle.lpips_oracle import seeded_weights, weights_of  # noqa: E402

PAIRS = 12


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30)
        return out.stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        return None


def timed(fn, rounds):
    fn()
    torch.cuda.synchronize()
    best = float("inf")
    for _ in range(rounds):
        t0 = time.perf_counter()
        r = fn()
        torch.cuda.synchronize()
        best = min(best, (time.perf_counter() - t0) * 1e3)
    return best, r


def torch_lpips(x, y, w, chunk=4):
    """The reference's forward on NCHW fp32 with torch.conv2d, chunk pairs at a time: [V] fp64."""
    out = []
    for i in range(0, x.shape[0], chunk):
        mean = torch.tensor(LP_MEAN, device=x.device)[None, :, None, None]
        std = torch.tensor(LP_STD, device=x.device)[None, :, None, None]
        h = (torch.cat([x[i:i + chunk], y[i:i + chunk]]) - mean) / std
        n, total = h.shape[0] // 2, 0
        for k, (cw, cb) in enumerate(w["conv"]):
            h = F.relu(F.conv2d(h, cw, cb, padding=1))
            if k in LP.TAP_AFTER:
                f = h / (torch.sqrt(torch.sum(h ** 2, 1, keepdim=True)) + 1e-10)
                lw = w["lin"][LP.TAP_AFTER.index(k)].reshape(1, -1, 1, 1)
                total = total + F.conv2d((f[:n] - f[n:]) ** 2, lw).mean((2, 3)).flatten()
            if k in LP.POOL_AFTER:
                h = F.max_pool2d(h, 2, 2)
        out.append(total.double())
    return torch.cat(out)


LP_MEAN, LP_STD = [-.030, -.088, -.188], [.458, .448, .450]


def layer_times(net, H, W, iters):
    L = I.lib()
    B = 8
    rows, h, w, cin = [], H, W, 3
    st = I._lib.stream_ptr()
    for i, cout in enumerate(LP.VGG_CHANNELS):
        x = torch.rand(B, h, w, cin, device="cuda")
        out = torch.empty(B, h, w, cout, device="cuda")
        call = lambda: L.gsb_lpips_conv3x3_relu(B, h, w, cin, cout, x.data_ptr(), net.w[i].data_ptr(),
                                                net.b[i].data_ptr(), out.data_ptr(), st)
        I._lib.check(call(), "conv")
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            call()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / iters
        flop = 2.0 * B * h * w * cout * 9 * cin
        rows.append({"layer": i, "HxW": f"{h}x{w}", "cin": cin, "cout": cout, "ms": round(ms, 4),
                     "tflops": round(flop / ms / 1e9, 2), "share_of_67_tflops": round(flop / ms / 1e9 / 67, 3)})
        cin = cout
        if i in LP.POOL_AFTER:
            h, w = h // 2, w // 2
        del x, out
    return rows


def reference_loop(x, y, vgg_path, lin_path):
    """Per pair: load both files, build the network, move it to the GPU, run it (lpips() per image)."""
    vals = []
    for i in range(x.shape[0]):
        vgg = torch.load(vgg_path, map_location="cpu", weights_only=True)
        lin = LP.rename_lin_keys(torch.load(lin_path, map_location="cpu", weights_only=True))
        convs = [torch.nn.Conv2d(wt.shape[1], wt.shape[0], 3, padding=1) for wt in
                 (vgg[f"features.{m}.weight"] for m in LP.VGG_CONV)]
        for c, m in zip(convs, LP.VGG_CONV):
            c.weight.data.copy_(vgg[f"features.{m}.weight"])
            c.bias.data.copy_(vgg[f"features.{m}.bias"])
        w = {"conv": [(c.weight.cuda(), c.bias.cuda()) for c in convs],
             "lin": [lin[f"{k}.1.weight"].cuda() for k in range(5)]}
        vals.append(torch_lpips(x[i:i + 1], y[i:i + 1], w))
    return torch.cat(vals)


def cli_times(x, y, wdir, rounds):
    from PIL import Image
    u8 = lambda t: (t.clamp(0, 1) * 255 + 0.5).to(torch.uint8).permute(0, 2, 3, 1).cpu().numpy()
    with tempfile.TemporaryDirectory() as root:
        scene = os.path.join(root, "model")
        for sub, imgs in (("renders", u8(x)), ("gt", u8(y))):
            d = os.path.join(scene, "test", "ours_1", sub)
            os.makedirs(d)
            for i, a in enumerate(imgs):
                Image.fromarray(a).save(os.path.join(d, f"{i:05d}.png"))
        src = os.path.join(root, "src")
        os.makedirs(src)
        base = ["-s", src, "-m", scene, "--n_views", "3"]
        out = {}
        with open(os.devnull, "w") as null:
            for name, extra in (("without", []), ("with", ["--lpips_weights", wdir])):
                old, sys.stdout = sys.stdout, null
                try:
                    out[name] = round(timed(lambda: M.main(base + extra), rounds)[0], 1)
                finally:
                    sys.stdout = old
        return out


@torch.no_grad()
def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--kernel-iters", type=int, default=20)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    vgg, lin, _ = seeded_weights(1)
    net = LP.LpipsVGG(*LP.check_weights(vgg, lin), device="cuda")
    w = weights_of(vgg, lin)
    wc = {"conv": [(cw.cuda(), cb.cuda()) for cw, cb in w["conv"]], "lin": [l.cuda() for l in w["lin"]]}
    res = {"gpu": torch.cuda.get_device_name(0), "power_limit": power_limit(), "pairs": PAIRS}
    with tempfile.TemporaryDirectory() as wdir:
        torch.save(vgg, os.path.join(wdir, LP.VGG_FILE))
        torch.save(lin, os.path.join(wdir, LP.LIN_FILE))
        for H, W in ((288, 512), (1080, 1920)):
            g = torch.Generator(device="cuda").manual_seed(H)
            x = torch.rand(PAIRS, 3, H, W, device="cuda", generator=g)
            y = (x + 0.05 * torch.randn(PAIRS, 3, H, W, device="cuda", generator=g)).clamp(0, 1)
            r = {}
            ms, ours = timed(lambda: net(x, y)[0], a.rounds)
            flop = 2 * PAIRS * sum(2.0 * h * ww * co * 9 * ci for (h, ww), co, ci in
                                   zip([LP.layer_sizes(H, W)[k] for k in (0, 0, 1, 1, 2, 2, 2, 3, 3, 3, 4, 4, 4)],
                                       LP.VGG_CHANNELS, (3,) + LP.VGG_CHANNELS[:-1]))
            r["ours_ms"] = round(ms, 2)
            r["ours_tflops_end_to_end"] = round(flop / ms / 1e9, 2)
            r["conv_tflop"] = round(flop / 1e12, 3)
            for arm, tf32 in (("cudnn_fp32", False), ("cudnn_tf32", True)):
                torch.backends.cudnn.allow_tf32 = tf32
                ms, v = timed(lambda: torch_lpips(x, y, wc), a.rounds)
                r[f"{arm}_ms"] = round(ms, 2)
                r[f"{arm}_max_abs_diff_vs_ours"] = float((v - ours).abs().max())
            r["lpips_mean_ours"] = float(ours.mean())
            torch.backends.cudnn.allow_tf32 = True
            ms, _ = timed(lambda: reference_loop(x, y, os.path.join(wdir, LP.VGG_FILE), os.path.join(wdir, LP.LIN_FILE)),
                          1)
            r["reference_loop_ms"] = round(ms, 2)
            r["layers"] = layer_times(net, H, W, a.kernel_iters)
            if H == 288:
                r["cli_ms"] = cli_times(x, y, wdir, a.rounds)
            res[f"{H}x{W}"] = r
            del x, y
            torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
