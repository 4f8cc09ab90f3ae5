"""Evaluation metrics, host side (no GPU): the entry points are exported and declared, tests/golden/metrics.npz (made by
the reference's own ssim / l1_loss / psnr, oracle/make_golden_metrics.py) agrees with an fp64 restatement of those
formulas, the 8-bit round trip is save_image's, the sums -> metrics conversion is right, and image_metrics refuses
what it cannot measure before it touches the library."""
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from instantsplat_b200.evaluation import image_metrics, metrics_from_sums

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "metrics.npz")


def test_metrics_symbols_exported_and_declared():
    import __graft_entry__ as G
    G.build()
    import instantsplat_b200 as I
    L = I.lib()
    hdr = open(os.path.join(ROOT, "include", "gsb200.h")).read()
    declared = set(re.findall(r"GSB_API [^;(]*?\b(gsb_\w+)\(", hdr))
    for name in ("gsb_image_metrics_scratch_bytes", "gsb_image_metrics_batch"):
        assert name in declared and name in I._lib.EXPORTS and hasattr(L, name), name
    assert re.search(r"#define GSB_METRIC_CLAMP 1\b", hdr) and re.search(r"#define GSB_METRIC_PNG8 2\b", hdr)
    # one fp64 partial triple per 32x16 tile and plane
    assert L.gsb_image_metrics_scratch_bytes(2, 3, 37, 53) == 2 * 3 * (2 * 3) * 3 * 8
    assert L.gsb_image_metrics_scratch_bytes(12, 3, 1080, 1920) == 12 * 3 * (60 * 68) * 3 * 8
    assert L.gsb_image_metrics_scratch_bytes(0, 3, 8, 8) == 0
    assert L.gsb_abi_version() == 2


def png8(x: np.ndarray) -> np.ndarray:
    """save_image's x.mul(255).add_(0.5).clamp_(0, 255).to(uint8) and to_tensor's /255, in fp32 numpy."""
    x = np.asarray(x, dtype=np.float32)
    q = np.clip(x * np.float32(255) + np.float32(0.5), np.float32(0), np.float32(255)).astype(np.uint8)
    return q.astype(np.float32) / np.float32(255)


def _window64():
    g = np.exp(-((np.arange(11) - 5.0) ** 2) / 4.5)
    g /= g.sum()
    return torch.from_numpy(np.outer(g, g))[None, None].expand(3, 1, 11, 11).contiguous()


def reference64(a: np.ndarray, b: np.ndarray) -> dict:
    """utils/loss_utils.py ssim / l1_loss and utils/image_utils.py psnr on [3, H, W] images, in fp64."""
    a, b = torch.from_numpy(np.asarray(a, np.float64))[None], torch.from_numpy(np.asarray(b, np.float64))[None]
    w = _window64()
    conv = lambda x: F.conv2d(x, w, padding=5, groups=3)
    mu1, mu2 = conv(a), conv(b)
    s1, s2, s12 = conv(a * a) - mu1 ** 2, conv(b * b) - mu2 ** 2, conv(a * b) - mu1 * mu2
    C1, C2 = 0.01 ** 2, 0.03 ** 2
    smap = ((2 * mu1 * mu2 + C1) * (2 * s12 + C2)) / ((mu1 ** 2 + mu2 ** 2 + C1) * (s1 + s2 + C2))
    d2 = (a - b) ** 2
    ps = lambda m: 20 * torch.log10(1.0 / torch.sqrt(m))
    return dict(l1=float((a - b).abs().mean()), ssim=float(smap.mean()),
                psnr_channels=ps(d2[0].reshape(3, -1).mean(1)).numpy(), psnr=float(ps(d2.mean())))


@pytest.mark.parametrize("name", ["small", "big"])
@pytest.mark.parametrize("mode", ["clamp", "png8"])
def test_golden_matches_fp64_restatement(name, mode):
    z = np.load(GOLD)
    r, g = z[f"{name}_render"], z[f"{name}_gt"]
    assert r.dtype == np.float32 and r.shape == g.shape and r.shape[1] == 3
    for v in range(r.shape[0]):
        if mode == "clamp":
            a, b = np.clip(r[v], 0, 1), np.clip(g[v], 0, 1)
        else:
            a, b = png8(r[v]), png8(g[v])
        want = reference64(a, b)
        assert abs(z[f"{name}_{mode}_l1"][v] - want["l1"]) <= 1e-6 * max(want["l1"], 1e-30), (v, want["l1"])
        assert abs(z[f"{name}_{mode}_ssim"][v] - want["ssim"]) <= 2e-6, (v, want["ssim"])
        for key in ("psnr", "psnr_channels"):
            got, exp = np.asarray(z[f"{name}_{mode}_{key}"][v]), np.asarray(want[key])
            assert np.array_equal(np.isinf(got), np.isinf(exp)), (v, key, got, exp)
            fin = np.isfinite(exp)
            assert np.all(np.abs(got[fin] - exp[fin]) <= 1e-4), (v, key, got, exp)
    # the inputs cover what the issue of each convention turns on
    assert (r < 0).any() and (r > 1).any() and (g < 0).any() and (g > 1).any()
    if name == "small":
        assert np.array_equal(r[2], g[2]) and np.isinf(z[f"small_{mode}_psnr"][2])
        assert np.isin(r[3], z["ties"]).all()


def test_png8_is_save_image_with_ties_rounding_up():
    z = np.load(GOLD)
    ties, want = z["ties"], z["ties_png8"]
    assert len(ties) > 3 * 200
    assert np.array_equal(png8(ties), want)
    exact = ties[ties * np.float32(255) == np.round(ties * np.float32(255) - np.float32(0.5)) + np.float32(0.5)]
    assert len(exact) > 200                      # the ties themselves, not only their neighbours
    # the two variants a kernel must not use disagree with torchvision on these values
    half_even = (np.rint(np.clip(ties * np.float32(255), 0, 255)).astype(np.float32) / np.float32(255))
    recip = (np.clip(ties * np.float32(255) + np.float32(0.5), 0, 255).astype(np.uint8).astype(np.float32) *
             np.float32(1 / 255))
    assert not np.array_equal(half_even, want) and not np.array_equal(recip, want)


def test_metrics_from_sums():
    H, W = 4, 5
    n = 3 * H * W
    sums = torch.tensor([[6.0, 54.0, 0.6, 1.2, 2.4],
                         [0.0, 60.0, 0.0, 0.0, 0.0],
                         [1.0, 30.0, 0.0, 0.2, 0.0]], dtype=torch.float64)
    m = metrics_from_sums(sums, H, W)
    assert torch.allclose(m["l1"], sums[:, 0] / n) and torch.allclose(m["ssim"], sums[:, 1] / n)
    assert torch.allclose(m["mse"], sums[:, 2:] / (H * W))
    mse0 = torch.tensor([0.6, 1.2, 2.4], dtype=torch.float64) / (H * W)
    assert torch.allclose(m["psnr_channels"][0], -10 * torch.log10(mse0))
    assert abs(float(m["psnr"][0]) - (-10 * np.log10(4.2 / n))) < 1e-12
    # identical images: inf in both conventions, as the reference's 20 * log10(1 / sqrt(0))
    assert torch.isinf(m["psnr"][1]) and torch.isinf(m["psnr_channels"][1]).all() and float(m["l1"][1]) == 0.0
    # one channel identical: that channel's PSNR is inf, the whole image's is not
    assert torch.isinf(m["psnr_channels"][2, 0]) and torch.isinf(m["psnr_channels"][2, 2])
    assert torch.isfinite(m["psnr"][2]) and m["psnr"].dtype == torch.float64
    assert {k: tuple(v.shape) for k, v in m.items()} == dict(l1=(3,), mse=(3, 3), psnr_channels=(3, 3), psnr=(3,),
                                                               ssim=(3,))


def test_image_metrics_refuses_bad_inputs():
    x = torch.zeros(2, 3, 8, 8)
    with pytest.raises(ValueError, match="CUDA"):
        image_metrics(x, x)
    with pytest.raises(ValueError, match="mode"):
        image_metrics(x, x, mode="png16")
    with pytest.raises(ValueError, match=r"\[V, 3, H, W\]"):
        image_metrics(torch.zeros(3, 8, 8), x)
    with pytest.raises(ValueError, match=r"\[V, 3, H, W\]"):
        image_metrics(torch.zeros(2, 4, 8, 8), x)
    with pytest.raises(ValueError, match="float32"):
        image_metrics(x.double(), x)
