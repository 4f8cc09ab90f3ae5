"""Cost of evaluating the training views at BASELINE configs[2] (1M Gaussians, 12 views, 1920x1080, SH 3), three ways:

  * report_loop: the shape of train.py's training_report (train.py:256-290) on the fused path: per view the fused
    render() under no_grad at get_RT(v), clamp of render and target, L1 and PSNR as utils/loss_utils.py l1_loss and
    utils/image_utils.py psnr compute them, `.mean().double()` accumulated; one host read of the totals at the end;
  * evaluate: JointTrainer.evaluate() over the 12 views (one batched forward, one metrics call), ending in a host read;
  * kernel: image_metrics alone on 12 views [12, 3, 1080, 1920], CUDA events over many launches, against its HBM floor
    of 2 * V * 3 * H * W * 4 bytes read at the data sheet's 3.35 TB/s.

The first two report the same mean L1 and mean per-channel PSNR (printed, with their difference).  Prints one JSON
line with the GPU and its power limit.  Usage: python tools/eval_cost.py [--rounds 5] [--kernel-iters 50]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import instantsplat_b200 as I  # noqa: E402
from instantsplat_b200.camera import SimpleCamera  # noqa: E402
from instantsplat_b200.evaluation import image_metrics  # noqa: E402
from instantsplat_b200.scenes import make_config  # noqa: E402
from instantsplat_b200.trainer import JointTrainer  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30)
        return out.stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        return None


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--kernel-iters", type=int, default=50)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("eval_cost.py needs a CUDA device")
    dev = "cuda"
    sc = make_config(2)
    V, H, W = sc.n_views, sc.height, sc.width
    gts = torch.rand(V, 3, H, W, generator=torch.Generator().manual_seed(3)).to(dev)
    tr = JointTrainer(sc, dev, gt_images=gts)
    model = I.GaussianModel.from_scene(sc, dev)
    cam = SimpleCamera(W, H, sc.fovx, sc.fovy, device=dev)
    pipe, bg = I.PipelineDefaults(), torch.zeros(3, device=dev)

    def report_loop():
        l1_test, psnr_test = 0.0, 0.0
        with torch.no_grad():
            for v in range(V):
                image = torch.clamp(I.render(cam, model, pipe, bg, camera_pose=model.get_RT(v))["render"], 0.0, 1.0)
                gt_image = torch.clamp(gts[v], 0.0, 1.0)
                l1_test += torch.abs(image - gt_image).mean().mean().double()
                mse = ((image - gt_image) ** 2).view(image.shape[0], -1).mean(1, keepdim=True)
                psnr_test += (20 * torch.log10(1.0 / torch.sqrt(mse))).mean().double()
        return float(l1_test / V), float(psnr_test / V)

    def evaluate():
        m = tr.evaluate()
        return float(m["l1"].mean()), float(m["psnr_channels"].mean(1).mean())

    report_loop(), evaluate()                                     # warm-up
    t_ref, t_ev = [], []
    for _ in range(a.rounds):
        t, ref = timed(report_loop)
        t_ref.append(t)
        t, ev = timed(evaluate)
        t_ev.append(t)
    # the metrics kernel alone
    imgs = torch.stack([tr.render(v).clone() for v in range(V)])
    image_metrics(imgs, gts)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    kern = {}
    for mode in ("clamp", "png8"):
        torch.cuda.synchronize()
        e0.record()
        for _ in range(a.kernel_iters):
            image_metrics(imgs, gts, mode=mode)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / a.kernel_iters
        floor_ms = 2 * V * 3 * H * W * 4 / HBM_BYTES_PER_S * 1e3
        kern[mode] = dict(ms=round(ms, 4), hbm_floor_ms=round(floor_ms, 4), read_TB_per_s=round(
            2 * V * 3 * H * W * 4 / (ms * 1e-3) / 1e12, 3), share_of_floor=round(floor_ms / ms, 3))
    out = dict(gpu=torch.cuda.get_device_name(0), power_limit=power_limit(), P=sc.P, views=V, W=W, H=H,
               report_loop_ms=[round(t, 3) for t in t_ref], evaluate_ms=[round(t, 3) for t in t_ev],
               speedup=round(min(t_ref) / min(t_ev), 3),
               report_loop_l1_psnr=ref, evaluate_l1_psnr=ev,
               diff_l1=abs(ref[0] - ev[0]), diff_psnr_db=abs(ref[1] - ev[1]), kernel=kern)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
