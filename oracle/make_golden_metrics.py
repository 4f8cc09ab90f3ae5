"""Generate tests/golden/metrics.npz from the REFERENCE's own evaluation code, run on CPU:
`utils.loss_utils.ssim` / `l1_loss` and `utils.image_utils.psnr` (the functions train.py's training_report and
metrics.py call), in both of the reference's evaluation pipelines:

  * clamp: training_report (train.py:256-290): render and target clamped to [0, 1], images [3, H, W], so `psnr`
    returns one value per channel and the report averages them;
  * png8: render.py:163-170 writes render and target with torchvision.utils.save_image, metrics.py reads them back
    (readImages, utils/sfm_utils.py:452-462: PIL.Image.open -> to_tensor -> unsqueeze(0)[:, :3]) and takes `psnr` of
    the [1, 3, H, W] image (one value from the whole image's MSE) and `ssim`.  Real PNG files are written and read.

Seeded inputs: four views at 37x53 (not a multiple of the 32x16 tile; values below 0 and above 1; view 2 identical
to its target; view 3's render made of 8-bit ties, fp32 values whose x*255 is exactly k + 0.5, and their nextafter
neighbours) and one 100x170 view that spans many tiles.  `ties` holds every tie value and its neighbours, and
`ties_png8` what save_image -> to_tensor makes of them.

    python oracle/make_golden_metrics.py <path to the InstantSplat checkout>
"""
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if len(sys.argv) != 2:
    sys.exit(__doc__)
sys.path.append(sys.argv[1])

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torchvision  # noqa: E402
import torchvision.transforms.functional as tf  # noqa: E402
from PIL import Image  # noqa: E402
from utils.image_utils import psnr  # noqa: E402
from utils.loss_utils import l1_loss, ssim  # noqa: E402


def tie_values() -> np.ndarray:
    """Every fp32 x in (0, 1) with fl(x * 255) == k + 0.5 for some k, with both nextafter neighbours."""
    out = []
    for k in range(255):
        c = np.float32((k + 0.5) / 255.0)
        for d in range(-4, 5):
            x = c
            for _ in range(abs(d)):
                x = np.nextafter(x, np.float32(np.sign(d)), dtype=np.float32)
            if np.float32(x) * np.float32(255) == np.float32(k + 0.5):
                out += [np.nextafter(x, np.float32(0), dtype=np.float32), x,
                        np.nextafter(x, np.float32(1), dtype=np.float32)]
    return np.unique(np.array(out, dtype=np.float32))


def png8(img: torch.Tensor, path: str) -> torch.Tensor:
    """[3, H, W] through save_image and readImages' to_tensor: [1, 3, H, W]."""
    torchvision.utils.save_image(img, path)
    return tf.to_tensor(Image.open(path)).unsqueeze(0)[:, :3, :, :]


def metrics(renders: torch.Tensor, gts: torch.Tensor, tmp: str) -> dict:
    out = {}
    for mode in ("clamp", "png8"):
        rows = {k: [] for k in ("l1", "ssim", "psnr_channels", "psnr")}
        for v in range(renders.shape[0]):
            if mode == "clamp":
                a, b = torch.clamp(renders[v], 0.0, 1.0), torch.clamp(gts[v], 0.0, 1.0)
            else:
                a = png8(renders[v], os.path.join(tmp, f"render_{v}.png"))[0]
                b = png8(gts[v], os.path.join(tmp, f"gt_{v}.png"))[0]
            rows["l1"].append(float(l1_loss(a, b).mean().double()))
            rows["psnr_channels"].append(psnr(a, b).reshape(3).double().numpy())
            rows["psnr"].append(float(psnr(a[None], b[None]).double()))
            rows["ssim"].append(float(ssim(a[None], b[None]).double()))
        for k, r in rows.items():
            out[f"{mode}_{k}"] = np.array(r, dtype=np.float64)
    return out


def main():
    g = torch.Generator().manual_seed(20261016)
    ties = tie_values()
    small_r = torch.rand(4, 3, 37, 53, generator=g) * 1.3 - 0.15
    small_g = torch.rand(4, 3, 37, 53, generator=g) * 1.2 - 0.1
    small_g[2] = small_r[2]
    small_r[3] = torch.from_numpy(ties)[torch.randint(len(ties), (3, 37, 53), generator=g)]
    big_r = torch.rand(1, 3, 100, 170, generator=g) * 1.3 - 0.15
    big_g = (big_r + 0.1 * torch.randn(1, 3, 100, 170, generator=g)).float()
    data = dict(ties=ties)
    with tempfile.TemporaryDirectory() as tmp:
        side = int(np.ceil(np.sqrt(len(ties))))
        plane = np.zeros(side * side, dtype=np.float32)
        plane[:len(ties)] = ties
        q = png8(torch.from_numpy(plane.reshape(1, side, side)).expand(3, side, side), os.path.join(tmp, "ties.png"))
        data["ties_png8"] = q[0, 0].reshape(-1)[:len(ties)].numpy()
        for name, r, t in (("small", small_r, small_g), ("big", big_r, big_g)):
            data[f"{name}_render"], data[f"{name}_gt"] = r.numpy(), t.numpy()
            data.update({f"{name}_{k}": v for k, v in metrics(r, t, tmp).items()})
    np.savez(os.path.join(ROOT, "tests", "golden", "metrics.npz"), **data)
    print({k: v.shape for k, v in data.items()})
    print("small clamp psnr", data["small_clamp_psnr"], "png8 psnr", data["small_png8_psnr"])


if __name__ == "__main__":
    main()
