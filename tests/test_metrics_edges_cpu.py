"""The restatement of the evaluation metrics kernel (tests/_metrics.py) and its bounds, checked without a device.

* Its per-tile sums add up to the whole frame's fp64 SSIM map (`O.ssim_map`), L1 and per-channel squared error, and
  each tile's sum is that of its own 32 x 16 box in the kernel's slot order.
* Its png8 transform is torchvision's save_image -> PIL -> to_tensor round trip on the special-value table.
* `metrics_from_sums` is utils/image_utils.py's psnr and utils/loss_utils.py's l1_loss restated in fp64, for zero,
  tiny, NaN and ordinary sums.
* The bounds discriminate: the correct formula in fp32 passes them, and each planted bug of a kernel (computed the way
  that kernel would) exceeds them tenfold or gives a finite number where fp64 gives NaN.
"""
import io
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import _loss as L
import _metrics as M
from instantsplat_b200.evaluation import metrics_from_sums
from oracle import gs_oracle as O

MODES = ("clamp", "png8")


def _batch(H, W, seed=0):
    """Two raw renders (in [-0.2, 3]) against three raw target planes, gt_row = [1, 0]."""
    img = L.content("raw", 6, H, W, seed=seed)[0].view(2, 3, H, W)
    gt = L.content("raw", 9, H, W, seed=seed + 1)[0].view(3, 3, H, W)
    return img, gt, [1, 0]


@pytest.mark.parametrize("shape", [(1, 1), (5, 11), (16, 32), (17, 33), (37, 70), (53, 77)])
@pytest.mark.parametrize("mode", MODES)
def test_tile_sums_add_up_to_the_frame(mode, shape):
    H, W = shape
    img, gt, rows = _batch(H, W, seed=H * W)
    R = M.restate(img, gt, rows, mode)
    gy, gx = M.grid(H, W)
    assert R["part"].shape == (6, gy, gx, 3)
    for v in range(2):
        a, b = M.transform(img[v], mode).double(), M.transform(gt[rows[v]], mode).double()
        smap, d = O.ssim_map(a, b), a - b
        want = [d.abs().sum(), smap.sum()] + [(d[c] ** 2).sum() for c in range(3)]
        tot = [d.abs().sum(), smap.abs().sum()] + [(d[c] ** 2).sum() for c in range(3)]
        for j in range(5):
            assert abs(float(R["out"][v, j] - want[j])) <= 1e-12 * float(tot[j]), (v, j)
        # each slot is its own tile's sum
        for c in range(3):
            for by in range(gy):
                for bx in range(gx):
                    ys, xs = slice(by * L.TH, (by + 1) * L.TH), slice(bx * L.TW, (bx + 1) * L.TW)
                    box = torch.stack([d[c, ys, xs].abs().sum(), smap[c, ys, xs].sum(), (d[c, ys, xs] ** 2).sum()])
                    got = R["part"][v * 3 + c, by, bx]
                    assert float((got - box).abs().max()) <= 1e-12 * (float(box.abs().max()) + 1e-300), (v, c, by, bx)


def test_tile_regions_partition_the_tiles():
    for H, W in ((1, 1), (37, 70), (240, 416), (2160, 3840)):
        R = M.tile_regions(H, W)
        tot = sum(m.int() for m in R.values())
        assert torch.equal(tot, torch.ones(*M.grid(H, W), dtype=tot.dtype)), (H, W)
    R = M.tile_regions(240, 416)          # 15 x 13 tiles, the outer ring touches the frame's 10 px
    assert int(R["seam"].sum()) == 13 * 11 and bool(R["border"][0, 5]) and bool(R["border"][14, 5])
    assert bool(R["border"][7, 12]) and bool(R["seam"][7, 11])


def test_special_values_cover_the_edges():
    S = M.SPECIALS
    assert any(math.isnan(s) for s in S) and math.inf in S and -math.inf in S and M.SUB in S
    assert any(s == 0 and math.copysign(1, s) < 0 for s in S)
    ties = [s for s in S if math.isfinite(s) and float(np.float32(s) * np.float32(255)) % 1 == 0.5]
    assert len(ties) >= 4, ties
    assert all(math.isnan(s) or float(np.float32(s)) == s for s in S)        # fp32 values


def test_png8_is_save_image_then_to_tensor():
    """The png8 restatement against torchvision's own round trip through a PNG file, bit for bit, NaN -> 0 included
    (what torch's float -> uint8 conversion gives on the CPU)."""
    from PIL import Image
    from torchvision.transforms.functional import to_tensor
    from torchvision.utils import save_image
    vals = torch.tensor(M.SPECIALS + [0.5, 0.2, 2.0, -0.7, 0.999, 1e-3], dtype=torch.float32)
    n = vals.numel()
    x = torch.stack([vals, vals.flip(0), vals.roll(3)])[:, None, :]       # [3, 1, n]
    buf = io.BytesIO()
    save_image(x, buf, format="png")
    buf.seek(0)
    want = to_tensor(Image.open(buf))
    assert want.shape == (3, 1, n) and want.dtype == torch.float32
    assert torch.equal(M.png8(x), want)
    assert float(M.png8(torch.tensor([math.nan]))) == 0.0
    assert M.png8(torch.tensor([math.inf, -math.inf])).tolist() == [1.0, 0.0]
    # the clamp convention keeps NaN, as torch.clamp does
    assert math.isnan(float(M.transform(torch.tensor([math.nan]), "clamp")))


# ---- metrics_from_sums ---------------------------------------------------------------------------------------------
def _psnr64(sq, n):
    """utils/image_utils.py psnr restated on a sum of squares over n values in fp64: 20 log10(1 / sqrt(mse))."""
    with np.errstate(divide="ignore", invalid="ignore"):
        return float(20.0 * np.log10(np.float64(1.0) / np.sqrt(np.float64(sq) / np.float64(n))))


def _close(got, want):
    if math.isnan(want) or math.isinf(want):
        return (math.isnan(got) and math.isnan(want)) or got == want
    return abs(got - want) <= 1e-12 * max(abs(want), 1e-300)


@pytest.mark.parametrize("sums", [[6.0, 54.0, 0.6, 1.2, 2.4],                     # ordinary
                                  [0.0, 60.0, 0.0, 0.0, 0.0],                     # identical images
                                  [1e-300, 59.9, 1e-310, 5e-324, 0.0],            # tiny and subnormal
                                  [math.nan, math.nan, math.nan, 0.2, 0.3],       # a NaN in channel 0
                                  [3.0, -1.5, 1e30, 0.4, 7.0]])                   # large, negative SSIM
def test_metrics_from_sums_restates_psnr_and_l1(sums):
    H, W = 4, 5
    n = 3 * H * W
    m = metrics_from_sums(torch.tensor([sums], dtype=torch.float64), H, W)
    assert _close(float(m["l1"][0]), sums[0] / n) and _close(float(m["ssim"][0]), sums[1] / n)
    for c in range(3):
        assert _close(float(m["mse"][0, c]), sums[2 + c] / (H * W)), c
        assert _close(float(m["psnr_channels"][0, c]), _psnr64(sums[2 + c], H * W)), c
    assert _close(float(m["psnr"][0]), _psnr64(sum(sums[2:]), n))


def test_metrics_from_sums_equals_the_reference_formulas_on_images():
    """Sums taken from fp64 images give utils/image_utils.py psnr of the [3, H, W] image per channel (training_report)
    and of the [1, 3, H, W] image (metrics.py), and l1_loss."""
    g = torch.Generator().manual_seed(3)
    a, b = torch.rand(2, 3, 9, 14, generator=g, dtype=torch.float64)
    b[1] = a[1]
    psnr = lambda x, y: 20 * torch.log10(1.0 / torch.sqrt(((x - y) ** 2).view(x.shape[0], -1).mean(1, keepdim=True)))
    d = a - b
    sums = torch.tensor([[float(d.abs().sum()), 0.0] + [float((d[c] ** 2).sum()) for c in range(3)]],
                        dtype=torch.float64)
    m = metrics_from_sums(sums, 9, 14)
    want_c = psnr(a, b)[:, 0]
    assert torch.isposinf(m["psnr_channels"][0, 1]) and torch.isposinf(want_c[1])
    fin = torch.isfinite(want_c)
    assert torch.allclose(m["psnr_channels"][0][fin], want_c[fin], rtol=1e-12, atol=0)
    assert abs(float(m["psnr"][0]) - float(psnr(a[None], b[None]))) <= 1e-12 * abs(float(m["psnr"][0]))
    assert abs(float(m["l1"][0]) - float(O.l1_loss(a, b))) <= 1e-15


# ---- the bounds discriminate ---------------------------------------------------------------------------------------
def kernel_like(img, gt, rows, mode, bug=None):
    """The partials [V C, gy, gx, 3] a kernel computing in fp32 would write, with one planted bug:
      pad_half      metric_input clamps to [0.5, 1] and is applied to the zero padding too
      png8_no_half  save_image's level without the + 0.5
      sq_raw        the squared error of the untransformed pixels
      nan_to_zero   the clamp maps NaN to 0 (fminf / fmaxf alone)"""
    V, C, H, W = img.shape
    tf = lambda x: M.transform(x, mode)
    if bug == "pad_half":
        tf = lambda x: torch.clamp(x, 0.5, 1)
    elif bug == "png8_no_half":
        tf = lambda x: x.mul(255).clamp(0, 255).to(torch.uint8).float().div(255)
    elif bug == "nan_to_zero":
        tf = lambda x: torch.where(torch.isnan(x), torch.zeros_like(x), torch.clamp(x, 0, 1))
    a, b = tf(img).reshape(V * C, H, W), tf(gt[rows]).reshape(V * C, H, W)
    if bug == "pad_half":
        pad = lambda x: F.pad(x, (L.HALO,) * 4, value=0.5)
        t = M.terms(pad(a), pad(b), torch.float32)[..., L.HALO:-L.HALO, L.HALO:-L.HALO]
    else:
        t = M.terms(a, b, torch.float32)
    if bug == "sq_raw":
        d = (img - gt[rows]).reshape(V * C, H, W)
        t[2] = d * d
    return M.tile_sums(t).double().permute(1, 2, 3, 0).contiguous()


def reduce_like(part, V, C, bug=None):
    """k_metrics_reduce's out [V, 2 + C] from partials, with one planted bug:
      skip_last   every sum leaves out its last partial (i < n - 1)
      sq_is_ssim  the per-channel offset (j - 2) T 3 + 1: the SSIM partials taken for the squared error"""
    p = part.reshape(V, C, -1, 3)
    if bug == "skip_last":
        l1 = p[..., 0].reshape(V, -1)[:, :-1].sum(1)
        ss = p[..., 1].reshape(V, -1)[:, :-1].sum(1)
        return torch.cat([l1[:, None], ss[:, None], p[..., :-1, 2].sum(2)], 1)
    out = M.view_sums(part, V, C)
    if bug == "sq_is_ssim":
        out[:, 2:] = p[..., 1].sum(2)
    return out


def _records(part, out, R, H, W):
    return M.check_partials("cpu", part, R) + M.check_views("cpu", out, metrics_from_sums(out, H, W), R)


def _worst_ratio(recs):
    return max(v["ratio"] for r in recs for v in r.values() if isinstance(v, dict) and "ratio" in v)


@pytest.mark.parametrize("mode", MODES)
def test_the_fp32_restatement_is_within_the_bounds(mode):
    img, gt, rows = _batch(53, 77, seed=2)
    R = M.restate(img, gt, rows, mode)
    part = kernel_like(img, gt, rows, mode)
    recs = _records(part, reduce_like(part, 2, 3), R, 53, 77)
    assert all(r["ok"] for r in recs), recs


@pytest.mark.parametrize("mode,bug", [("clamp", "pad_half"), ("png8", "png8_no_half"), ("clamp", "sq_raw"),
                                      ("png8", "sq_raw")])
def test_partial_mutants_exceed_the_bound_tenfold(mode, bug):
    img, gt, rows = _batch(53, 77, seed=3)
    R = M.restate(img, gt, rows, mode)
    part = kernel_like(img, gt, rows, mode, bug)
    recs = M.check_partials("cpu", part, R)
    assert _worst_ratio(recs) >= 10, recs
    if bug == "pad_half":               # the padding shows in the SSIM of the border tiles
        assert next(r for r in recs if r["region"] == "border")["ssim"]["ratio"] >= 10


@pytest.mark.parametrize("bug", ["skip_last", "sq_is_ssim"])
def test_reduce_mutants_exceed_the_bound_tenfold(bug):
    img, gt, rows = _batch(53, 77, seed=4)
    R = M.restate(img, gt, rows, "clamp")
    part = kernel_like(img, gt, rows, "clamp")
    recs = M.check_views("cpu", reduce_like(part, 2, 3, bug), metrics_from_sums(reduce_like(part, 2, 3, bug), 53, 77),
                         R)
    assert _worst_ratio(recs) >= 10 and not recs[0]["ok"], recs


def test_nan_to_zero_is_caught():
    """The clamp that maps NaN to 0 gives finite partials where fp64 has NaN."""
    img = torch.rand(1, 3, 37, 70, generator=torch.Generator().manual_seed(5))
    gt = torch.rand(1, 3, 37, 70, generator=torch.Generator().manual_seed(6))
    img[0, 1, 16, 32] = math.nan
    R = M.restate(img, gt, [0], "clamp")
    good = M.check_partials("cpu", kernel_like(img, gt, [0], "clamp"), R)
    bad = M.check_partials("cpu", kernel_like(img, gt, [0], "clamp", "nan_to_zero"), R)
    assert all(r["ok"] for r in good), good
    assert not all(r["ok"] for r in bad) and sum(r["ssim"]["nan_mismatch"] for r in bad) > 0, bad
