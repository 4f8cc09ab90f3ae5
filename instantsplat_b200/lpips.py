"""LPIPS (VGG16, v0.1), the third number of metrics.py (metrics.py:69: lpips(render, gt, net_type='vgg')), on the GPU
from the user's own weight files (DESIGN.md section 4.15).

The weights are the two files torch hub keeps after the reference's metrics.py has run once, under
$TORCH_HOME/hub/checkpoints/: torchvision's VGG16 state dict (vgg16-397923af.pth) and the LPIPS v0.1 linear layers
(vgg.pth).  Nothing is downloaded and no weights ship with the project.  What is computed is lpipsPyTorch's LPIPS on
inputs in [0, 1] (the 3DGS convention metrics.py keeps, not LPIPS's [-1, 1]): z-score, the 13 conv3x3 + ReLU layers
of vgg16().features with 2x2 max pooling after blocks 1-4, at relu1_2, relu2_2, relu3_3, relu4_3 and relu5_3 the
per-pixel normalisation f / (|f| + 1e-10), the lin layers' weighted squared difference, its mean over the map, and the
sum over the five layers.

    net = LpipsVGG.from_dir(os.path.expanduser("~/.cache/torch/hub/checkpoints"), "cuda")
    lpips, layers = net(renders, gts)       # [V] and [V, 5], fp64, on the device
"""
from __future__ import annotations

import os
from collections import OrderedDict
from typing import Dict, List, Tuple

import torch

from . import _lib
from ._lib import check
from .evaluation import _images

VGG_FILE = "vgg16-397923af.pth"
LIN_FILE = "vgg.pth"
VGG_CONV = (0, 2, 5, 7, 10, 12, 14, 17, 19, 21, 24, 26, 28)     # Conv2d modules of vgg16().features
VGG_CHANNELS = (64, 64, 128, 128, 256, 256, 256, 512, 512, 512, 512, 512, 512)
TAP_AFTER = (1, 3, 6, 9, 12)         # index in VGG_CONV whose ReLU is tapped (relu1_2, relu2_2, relu3_3, relu4_3, relu5_3)
POOL_AFTER = (1, 3, 6, 9)            # MaxPool2d(2, 2) follows these convs; the fifth pool is never run
LIN_CHANNELS = (64, 128, 256, 512, 512)
MIN_SIZE = 16                        # below this, the fourth pool leaves an empty map (the reference raises there)


def rename_lin_keys(state: Dict[str, torch.Tensor]) -> "OrderedDict[str, torch.Tensor]":
    """lpipsPyTorch/modules/utils.py get_state_dict's renaming of vgg.pth's keys: 'lin' and 'model.' dropped
    (lin{k}.model.1.weight -> {k}.1.weight, the keys of LinLayers)."""
    return OrderedDict((k.replace("lin", "").replace("model.", ""), v) for k, v in state.items())


def _load(path: str, what: str) -> dict:
    if not os.path.isfile(path):
        raise FileNotFoundError(f"LPIPS weights: {what} file {path} not found")
    try:
        state = torch.load(path, map_location="cpu", weights_only=True)
    except Exception as e:                                              # noqa: BLE001 -- report any unreadable file
        raise ValueError(f"LPIPS weights: {path} is not a readable state dict ({type(e).__name__}: {e})") from e
    if not isinstance(state, dict):
        raise ValueError(f"LPIPS weights: {path} holds a {type(state).__name__}, expected a state dict")
    return state


def _tensor(state: dict, key: str, shape: Tuple[int, ...], path: str) -> torch.Tensor:
    if key not in state:
        raise ValueError(f"LPIPS weights: {path} lacks {key}")
    t = state[key]
    if not isinstance(t, torch.Tensor) or not t.is_floating_point():
        raise ValueError(f"LPIPS weights: {path}: {key} is not a floating-point tensor")
    if tuple(t.shape) != shape:
        raise ValueError(f"LPIPS weights: {path}: {key} has shape {tuple(t.shape)}, expected {shape}")
    return t.float()


def check_weights(vgg: dict, lin: dict, vgg_path: str = VGG_FILE, lin_path: str = LIN_FILE):
    """Every conv weight / bias of vgg16().features and every lin weight, checked by name and shape and converted to
    fp32: ([(weight [Cout, Cin, 3, 3], bias [Cout]) x 13], [lin weight [C] x 5]).  vgg may hold other keys (the
    classifier of torchvision's file); the renamed lin keys must be exactly LinLayers', as its strict load wants."""
    convs, cin = [], 3
    for m, cout in zip(VGG_CONV, VGG_CHANNELS):
        w = _tensor(vgg, f"features.{m}.weight", (cout, cin, 3, 3), vgg_path)
        b = _tensor(vgg, f"features.{m}.bias", (cout,), vgg_path)
        convs.append((w, b))
        cin = cout
    renamed = rename_lin_keys(lin)
    want = [f"{k}.1.weight" for k in range(len(LIN_CHANNELS))]
    extra = sorted(set(renamed) - set(want))
    if extra:
        raise ValueError(f"LPIPS weights: {lin_path}: unexpected keys {extra} (after get_state_dict's renaming)")
    lins = []
    for k, c in enumerate(LIN_CHANNELS):
        if want[k] not in renamed:
            raise ValueError(f"LPIPS weights: {lin_path} lacks lin{k}.model.1.weight")
        lins.append(_tensor(renamed, want[k], (1, c, 1, 1), lin_path).reshape(c))
    return convs, lins


def read_weights(vgg_path: str, lin_path: str):
    """check_weights of the two files (loaded with torch.load(weights_only=True) onto the CPU)."""
    return check_weights(_load(vgg_path, "VGG16"), _load(lin_path, "LPIPS lin"), vgg_path, lin_path)


def check_pair(x, y) -> Tuple[int, int, int]:
    """(V, H, W) of two [V, 3, H, W] image batches of one shape, at least MIN_SIZE pixels in each dimension."""
    shape = lambda t: tuple(getattr(t, "shape", ()))
    if len(shape(x)) != 4 or shape(x)[1] != 3:
        raise ValueError(f"LpipsVGG: x: expected a [V, 3, H, W] tensor, got {shape(x)}")
    if shape(x) != shape(y):
        raise ValueError(f"LpipsVGG: x {shape(x)} and y {shape(y)} differ in shape")
    V, _, H, W = shape(x)
    if V == 0:
        raise ValueError("LpipsVGG: no images")
    if H < MIN_SIZE or W < MIN_SIZE:
        raise ValueError(f"LpipsVGG: images of {H}x{W} are below {MIN_SIZE} pixels in a dimension: VGG16's fourth "
                         "max pool would leave an empty feature map")
    return V, H, W


def layer_sizes(H: int, W: int) -> List[Tuple[int, int]]:
    """(H, W) of the five tapped maps: floor halving after each of the first four blocks."""
    out = [(H, W)]
    for _ in range(4):
        H, W = H // 2, W // 2
        out.append((H, W))
    return out


class LpipsVGG:
    """LPIPS with VGG16 features, weights packed once for the kernels (gsb_lpips_*, include/gsb200.h)."""

    def __init__(self, convs, lins, device="cuda"):
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise ValueError(f"LpipsVGG: expected a CUDA device (there is no CPU path), got {self.device}")
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        # [Cin, 3, 3, Cout]: row (ci, tap) holds the Cout weights the implicit GEMM reads together
        self.w = [w.permute(1, 2, 3, 0).contiguous().to(self.device) for w, _ in convs]
        self.b = [b.contiguous().to(self.device) for _, b in convs]
        self.lin = [l.contiguous().to(self.device) for l in lins]

    @classmethod
    def from_files(cls, vgg_path: str, lin_path: str, device="cuda") -> "LpipsVGG":
        """From torchvision's VGG16 state dict and the LPIPS v0.1 vgg lin layers, by path."""
        return cls(*read_weights(vgg_path, lin_path), device=device)

    @classmethod
    def from_dir(cls, path: str, device="cuda") -> "LpipsVGG":
        """From a directory holding the files under torch hub's names (vgg16-397923af.pth, vgg.pth), such as
        $TORCH_HOME/hub/checkpoints."""
        if not os.path.isdir(path):
            raise FileNotFoundError(f"LPIPS weights: directory {path} not found")
        return cls.from_files(os.path.join(path, VGG_FILE), os.path.join(path, LIN_FILE), device)

    def _chunk(self, x: torch.Tensor, y: torch.Tensor, out: torch.Tensor, scratch: torch.Tensor) -> None:
        """x, y [B, 3, H, W] (contiguous fp32 on self.device) -> out [B, 5], the per-layer sums over pixels."""
        L = _lib.lib()
        B, _, H, W = x.shape
        act = 2 * B * H * W * 64
        f = scratch[: 2 * act * 4].view(torch.float32)
        bufs = (f[:act], f[act:])
        parts = scratch[2 * act * 4:].view(torch.float64)
        st = _lib.stream_ptr()
        check(L.gsb_lpips_prepare(B, H, W, x.data_ptr(), y.data_ptr(), bufs[0].data_ptr(), st), "gsb_lpips_prepare")
        cur, h, w, cin, tap = 0, H, W, 3, 0
        for i, cout in enumerate(VGG_CHANNELS):
            check(L.gsb_lpips_conv3x3_relu(2 * B, h, w, cin, cout, bufs[cur].data_ptr(), self.w[i].data_ptr(),
                                           self.b[i].data_ptr(), bufs[1 - cur].data_ptr(), st),
                  "gsb_lpips_conv3x3_relu")
            cur, cin = 1 - cur, cout
            if i in TAP_AFTER:
                check(L.gsb_lpips_head(B, h, w, cout, bufs[cur].data_ptr(), self.lin[tap].data_ptr(), tap,
                                       out.data_ptr(), parts.data_ptr(), st), "gsb_lpips_head")
                tap += 1
            if i in POOL_AFTER:
                check(L.gsb_lpips_maxpool2(2 * B, h, w, cout, bufs[cur].data_ptr(), bufs[1 - cur].data_ptr(), st),
                      "gsb_lpips_maxpool2")
                cur, h, w = 1 - cur, h // 2, w // 2

    def __call__(self, x: torch.Tensor, y: torch.Tensor, max_batch: int = 4):
        """LPIPS of x[v] against y[v], x and y [V, 3, H, W] fp32 CUDA tensors with values in [0, 1] (k / 255 as
        metrics.py reads them), H and W at least 16.  Returns (lpips [V], layers [V, 5]) in fp64 on the device, without
        waiting for the GPU: layers holds each tap's mean over its map, lpips their sum.  x and y of up to max_batch
        views run as one batch of 2 max_batch images; scratch grows with it (gsb_lpips_scratch_bytes: 1 KiB per pixel
        of each of the max_batch pairs).  Each view's values are bit-identical from run to run and do not depend on max_batch or on
        the other views."""
        V, H, W = check_pair(x, y)
        x = _images(x, "LpipsVGG: x", self.device)
        y = _images(y, "LpipsVGG: y", self.device)
        if int(max_batch) < 1:
            raise ValueError(f"LpipsVGG: max_batch must be at least 1, got {max_batch}")
        B = min(V, int(max_batch))
        L = _lib.lib()
        sums = torch.empty(V, 5, dtype=torch.float64, device=self.device)
        with torch.cuda.device(self.device):
            scratch = torch.empty(L.gsb_lpips_scratch_bytes(B, H, W), dtype=torch.uint8, device=self.device)
            for v0 in range(0, V, B):
                v1 = min(V, v0 + B)
                self._chunk(x[v0:v1], y[v0:v1], sums[v0:v1], scratch)
        # divided by Python scalars: a device tensor of the areas would be a blocking copy from pageable memory
        layers = torch.stack([sums[:, k] / float(h * w) for k, (h, w) in enumerate(layer_sizes(H, W))], 1)
        return layers.sum(1), layers
