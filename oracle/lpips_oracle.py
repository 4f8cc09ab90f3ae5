"""fp64 restatement of LPIPS('vgg') v0.1  --  TEST INFRASTRUCTURE, NOT PRODUCT CODE.

lpipsPyTorch/modules/lpips.py (LPIPS.forward), networks.py (BaseNet.z_score / forward, VGG16: target_layers
[4, 9, 16, 23, 30] of vgg16().features) and utils.py (normalize_activation), in torch's conv2d / max_pool2d on any
device.  Only tests/ and tools/ import it; instantsplat_b200.lpips never does.
"""
import torch
import torch.nn.functional as F

LPIPS_MEAN = (-.030, -.088, -.188)
LPIPS_STD = (.458, .448, .450)
TAPS = (1, 3, 6, 9, 12)      # index among the 13 convs whose ReLU is tapped (relu1_2 .. relu5_3)
POOLS = (1, 3, 6, 9)         # MaxPool2d(2, 2) after these; the fifth pool (module 30) is never run


def lpips_vgg_fp64(x, y, weights):
    """LPIPS('vgg') of x[v] against y[v] ([V, 3, H, W] in [0, 1], any device) in fp64.  weights: {"conv":
    [(weight [Cout, Cin, 3, 3], bias [Cout]) x 13] in vgg16().features order, "lin": [weight [C] or [1, C, 1, 1] x 5]}.
    The z-score constants are rounded to fp32 first, as BaseNet's buffers hold them.  Returns (lpips [V], layers
    [V, 5]): each tap's mean over its map, and their sum."""
    dev = x.device
    d = lambda t: torch.as_tensor(t).to(device=dev, dtype=torch.float64)
    mean = torch.tensor(LPIPS_MEAN, dtype=torch.float32).to(dev, torch.float64)[None, :, None, None]
    std = torch.tensor(LPIPS_STD, dtype=torch.float32).to(dev, torch.float64)[None, :, None, None]

    def feats(img):
        h = (d(img) - mean) / std
        out = []
        for i, (w, b) in enumerate(weights["conv"]):
            h = F.relu(F.conv2d(h, d(w), d(b), padding=1))
            if i in TAPS:
                out.append(h / (torch.sqrt((h * h).sum(1, keepdim=True)) + 1e-10))
            if i in POOLS:
                h = F.max_pool2d(h, 2, 2)
        return out

    layers = []
    for fx, fy, lw in zip(feats(x), feats(y), weights["lin"]):
        layers.append(((fx - fy) ** 2 * d(lw).reshape(1, -1, 1, 1)).sum(1).mean((1, 2)))
    layers = torch.stack(layers, 1)
    return layers.sum(1), layers


VGG_CONV = (0, 2, 5, 7, 10, 12, 14, 17, 19, 21, 24, 26, 28)
VGG_CHANNELS = (64, 64, 128, 128, 256, 256, 256, 512, 512, 512, 512, 512, 512)
LIN_CHANNELS = (64, 128, 256, 512, 512)


def seeded_weights(seed):
    """Stand-ins for the hub files, from np.random.default_rng(seed): (vgg, lin, sha256).  vgg holds
    features.{m}.weight / bias as torchvision's VGG16 state dict names them (He-scaled normal weights, small normal
    biases), lin holds lin{k}.model.1.weight [1, C, 1, 1] as vgg.pth names them (positive).  sha256 is the hex digest
    of every array's fp32 bytes in that order, so a fixture can store the seed and the digest instead of the 14.7M
    weights."""
    import hashlib
    from collections import OrderedDict

    import numpy as np
    g = np.random.default_rng(seed)
    h = hashlib.sha256()
    vgg, lin, cin = OrderedDict(), OrderedDict(), 3
    for m, cout in zip(VGG_CONV, VGG_CHANNELS):
        w = (g.standard_normal((cout, cin, 3, 3), dtype=np.float32) * np.float32(np.sqrt(2.0 / (9 * cin))))
        b = g.standard_normal(cout, dtype=np.float32) * np.float32(0.02)
        for k, a in ((f"features.{m}.weight", w), (f"features.{m}.bias", b)):
            h.update(a.tobytes())
            vgg[k] = torch.from_numpy(a)
        cin = cout
    for k, c in enumerate(LIN_CHANNELS):
        a = g.uniform(0.01, 0.1, (1, c, 1, 1)).astype(np.float32)
        h.update(a.tobytes())
        lin[f"lin{k}.model.1.weight"] = torch.from_numpy(a)
    return vgg, lin, h.hexdigest()


def weights_of(vgg, lin):
    """The `weights` argument of lpips_vgg_fp64 from hub-format state dicts."""
    return {"conv": [(vgg[f"features.{m}.weight"], vgg[f"features.{m}.bias"]) for m in VGG_CONV],
            "lin": [lin[f"lin{k}.model.1.weight"] for k in range(len(LIN_CHANNELS))]}
