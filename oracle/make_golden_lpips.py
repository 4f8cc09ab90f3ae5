"""Generate tests/golden/lpips.npz from the REFERENCE's own LPIPS (lpipsPyTorch.LPIPS('vgg'), the network metrics.py:69
builds), run on CPU with seeded weights in fp32 and, converted with .double(), in fp64.

The reference builds its network from torchvision's pretrained VGG16 and downloads the lin layers.  Before anything is
constructed, torchvision.models.vgg16 (as lpipsPyTorch's networks module calls it) is replaced by a VGG16 that
holds oracle.lpips_oracle.seeded_weights(SEED), lpipsPyTorch's get_state_dict by one that returns the seeded lin
layers renamed by the reference's own get_state_dict, and torch.hub.load_state_dict_from_url raises, so nothing can
reach the network.  The weights are not stored: the fixture holds the seed and the SHA-256 of the generated arrays.

Cases (u8 images, read as to_tensor reads them): 16x16 (every pool down to 1x1), 37x53 (odd sizes, floor pooling),
64x96, 100x170 (many tiles), and at 32x48 an identical pair, a black image against a random one, a noisy pair and a
very different pair.  Per case: the fp32 and fp64 LPIPS and the five per-layer means.  `lin_keys` / `lin_renamed`
record get_state_dict's renaming of vgg.pth's keys.

    python oracle/make_golden_lpips.py <path to the InstantSplat checkout>
"""
import copy
import os
import sys
from collections import OrderedDict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if len(sys.argv) != 2:
    sys.exit(__doc__)
sys.path.insert(0, ROOT)
sys.path.append(sys.argv[1])

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torchvision  # noqa: E402
import torchvision.transforms.functional as tf  # noqa: E402
from lpipsPyTorch.modules import lpips as ref_lpips  # noqa: E402
from lpipsPyTorch.modules import networks as ref_networks  # noqa: E402
from lpipsPyTorch.modules import utils as ref_utils  # noqa: E402

from oracle.lpips_oracle import seeded_weights  # noqa: E402

SEED = 20240915


def no_network(*a, **k):
    raise RuntimeError("make_golden_lpips: the generator never downloads anything")


def cases():
    g = np.random.default_rng(7)
    rnd = lambda h, w: g.integers(0, 256, (h, w, 3), dtype=np.uint8)
    out = OrderedDict()
    for name, (h, w) in (("s16", (16, 16)), ("odd", (37, 53)), ("m64", (64, 96)), ("big", (100, 170))):
        out[name] = (rnd(h, w), rnd(h, w))
    base = rnd(32, 48)
    out["same"] = (base, base.copy())
    out["black"] = (np.zeros_like(base), rnd(32, 48))
    noisy = np.clip(base.astype(np.int16) + g.integers(-12, 13, base.shape), 0, 255).astype(np.uint8)
    out["noisy"] = (base, noisy)
    yy, xx = np.mgrid[0:32, 0:48]
    smooth = np.stack([xx * 5, yy * 7, (xx + yy) * 3], -1).astype(np.uint8)
    out["diff"] = (smooth, 255 - base)
    return out


def per_layer(net, x, y):
    """LPIPS.forward's terms: the lin layer of each tap's squared difference, averaged over the map."""
    fx, fy = net.net(x), net.net(y)
    return torch.cat([l((a - b) ** 2).mean((2, 3), True).flatten() for a, b, l in zip(fx, fy, net.lin)])


def main():
    vgg_sd, lin_raw, sha = seeded_weights(SEED)
    torch.hub.load_state_dict_from_url = lambda *a, **k: OrderedDict(lin_raw)
    renamed = ref_utils.get_state_dict("vgg", "0.1")
    torch.hub.load_state_dict_from_url = no_network
    build_vgg16 = torchvision.models.vgg16

    def seeded_vgg16(*a, **k):
        m = build_vgg16(weights=None)
        m.features.load_state_dict({key[len("features."):]: v for key, v in vgg_sd.items()})
        return m

    ref_networks.models.vgg16 = seeded_vgg16
    ref_lpips.get_state_dict = lambda *a, **k: renamed
    net32 = ref_lpips.LPIPS("vgg", "0.1").eval()
    net64 = copy.deepcopy(net32).double()
    z = {"seed": np.int64(SEED), "sha256": np.array(sha), "lin_keys": np.array(list(lin_raw)),
         "lin_renamed": np.array(list(renamed))}
    names = []
    with torch.no_grad():
        for name, (a, b) in cases().items():
            x, y = tf.to_tensor(a).unsqueeze(0), tf.to_tensor(b).unsqueeze(0)
            z[f"x_{name}"], z[f"y_{name}"] = a, b
            z[f"ref32_{name}"] = np.float64(net32(x, y).item())
            z[f"ref64_{name}"] = np.float64(net64(x.double(), y.double()).item())
            z[f"layers32_{name}"] = per_layer(net32, x, y).double().numpy()
            z[f"layers64_{name}"] = per_layer(net64, x.double(), y.double()).numpy()
            print(f"{name:6s} {a.shape[0]}x{a.shape[1]}: fp32 {z[f'ref32_{name}']:.9f}  fp64 {z[f'ref64_{name}']:.12f}")
            names.append(name)
    z["cases"] = np.array(names)
    path = os.path.join(ROOT, "tests", "golden", "lpips.npz")
    np.savez_compressed(path, **z)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
