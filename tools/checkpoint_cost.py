"""Cost of JointTrainer's checkpoints (DESIGN.md section 4.9) at the bench workload (configs[2]: 1M Gaussians, 12
views, 1920x1080): after a few training steps, the time of `save_checkpoint` and of `JointTrainer.from_checkpoint`,
each ending in a device synchronise, and the file size.  The file goes to a temporary directory, which is removed.

Prints one JSON object.

    python tools/checkpoint_cost.py [--rounds 3] [--steps 5]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    args = ap.parse_args()
    import torch
    import instantsplat_b200 as I
    from instantsplat_b200.scenes import make_config
    if not torch.cuda.is_available():
        raise SystemExit("checkpoint_cost.py measures on the GPU; none is available")
    dev = torch.device("cuda")
    sc = make_config(2)
    gts = torch.rand(sc.n_views, 3, sc.height, sc.width, generator=torch.Generator().manual_seed(0))
    cfg = I.OptimConfig()
    cfg.iterations = 1000
    tr = I.JointTrainer(sc, dev, gt_images=gts, cfg=cfg)
    for k in range(args.steps):
        tr.step(k % sc.n_views)
    torch.cuda.synchronize()
    tmp = tempfile.mkdtemp(prefix="gsb_ckpt_")
    save_ms, load_ms = [], []
    try:
        path = os.path.join(tmp, "chkpnt.pth")
        for _ in range(args.rounds):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            tr.save_checkpoint(path)
            torch.cuda.synchronize()
            save_ms.append((time.perf_counter() - t0) * 1e3)
            size = os.path.getsize(path)
            t0 = time.perf_counter()
            b = I.JointTrainer.from_checkpoint(path, sc, gt_images=gts, cfg=cfg, device=dev)
            torch.cuda.synchronize()
            load_ms.append((time.perf_counter() - t0) * 1e3)
            assert torch.equal(b.params, tr.params) and b.opt_step == tr.opt_step
            del b
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    print(json.dumps(dict(config="configs[2]", P=sc.P, n_views=sc.n_views, width=sc.width, height=sc.height,
                          file_bytes=size, save_ms=[round(x, 1) for x in save_ms],
                          from_checkpoint_ms=[round(x, 1) for x in load_ms],
                          device=torch.cuda.get_device_name(0), nvidia_smi=smi[:1])))


if __name__ == "__main__":
    main()
