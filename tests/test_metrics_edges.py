"""The evaluation metrics kernel (gsb_image_metrics_batch, gs_loss.cu) tile by tile against fp64 at frame borders,
tile seams, small and large frames, special values and the batch's addressing (-m gpu).

The C ABI is called with a scratch buffer the test owns, so every CTA's three partials {sum |a - b|, sum ssim,
sum (a - b)^2} are compared with the fp64 sums over its tile of the transformed planes (tests/_metrics.py), with the
loss's calibrated bound K sum|t32 - t64| + 10 2^-24 sum|t64| (tests/_loss.py); border and seam tiles are recorded
apart.  Each view's out[v] is bounded the same way, its PSNRs by what the squared-error bound allows, and `inf` must
appear exactly where the fp64 squared error is 0.  Each case's numbers go to the parity report (kind "metrics").
Exact checks: zero L1 and squared-error partials wherever the transformed planes agree on a whole tile, NaN metrics
for a NaN pixel under the clamp convention (torch.clamp keeps NaN), bit-identical views alone and in any batch, and
the cross-mode identities that tie render.py's 8-bit frames to the metrics they feed.
"""
import math

import pytest
import torch

import _loss as L
import _metrics as M
from _parity import DEV, REPORT
from instantsplat_b200 import GsbError
from instantsplat_b200.evaluation import image_metrics, metrics_from_sums
from instantsplat_b200.freeview import quantise
from test_loss_edges import HS, WS

pytestmark = pytest.mark.gpu

MODES = ("clamp", "png8")


def run(case, img, gt, rows, mode, ref_device="cpu"):
    """Kernel vs restatement for imgs [V, C, H, W] against gts[rows] (restatement computed on ref_device) ->
    (records, (partials, out, metrics) of the kernel, restatement)."""
    V, C, H, W = img.shape
    part, out = M.metrics_kernel(img.to(DEV).contiguous(), gt.to(DEV).contiguous(), rows, mode)
    metrics = metrics_from_sums(out, H, W)
    R = M.restate(img.to(ref_device), gt.to(ref_device), rows, mode)
    recs = M.check_partials(case, part, R) + M.check_views(case, out, metrics, R)
    return recs, (part, out, metrics), R


def zero_where_equal(part, R):
    """Exact: the L1 and squared-error partials are 0 on every tile where the transformed planes agree pixel for
    pixel (and on no other)."""
    V, C, H, W = R["a"].shape
    same = M.tile_sums((R["a"] != R["b"]).double().reshape(V * C, H, W)).to(part.device) == 0
    return bool((part[..., 0][same] == 0).all()) and bool((part[..., 2][same] == 0).all()) and \
        bool((part[..., 0][~same] > 0).all())


def assert_ok(recs, exact=()):
    REPORT.extend(recs)
    bad = [r for r in recs if not r["ok"]]
    assert not bad, f"{len(bad)} of {len(recs)} checks over the bound (K = {L.K}, worst k_needed " \
                    f"{M.worst(recs):.3g}): {bad[:4]}"
    wrong = [name for name, ok in exact if not ok]
    assert not wrong, f"exact checks that failed: {wrong}"


def _raw(n, H, W, seed):
    """n planes of a render in [-0.2, 3]: both conventions saturate it on both sides."""
    return L.content("raw", n, H, W, seed=seed)[0]


# ---- 1. sizes ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", MODES)
def test_size_sweep(mode):
    """Frames smaller than the window, than one tile, and one pixel either side of a tile seam: two views against
    three target planes with gt_row = [1, 0]."""
    recs, exact = [], []
    for H in HS:
        for W in WS:
            img = _raw(6, H, W, seed=100 * H + W).view(2, 3, H, W)
            gt = _raw(9, H, W, seed=100 * H + W + 1).view(3, 3, H, W)
            rs, (part, _, _), R = run(f"sizes {mode} 2x3x{H}x{W}", img, gt, [1, 0], mode)
            recs += rs
            exact.append((f"{H}x{W}: zero where equal", zero_where_equal(part.cpu(), R)))
    assert_ok(recs, exact)


# ---- 2. content ----------------------------------------------------------------------------------------------------
def far_tiles(a, H, W):
    """[gy, gx]: tiles with no non-zero pixel of a [C, H, W] within 10 px of them."""
    hot = (a != 0).any(0).float()[None, None]
    near = torch.nn.functional.max_pool2d(hot, 2 * L.CTX + 1, stride=1, padding=L.CTX)[0, 0] > 0
    return M.tile_sums(near.double()) == 0


@pytest.mark.parametrize("shape", [(3, 53, 77), (3, 240, 416)])
@pytest.mark.parametrize("kind", L.CONTENTS + ("one_equal",))
@pytest.mark.parametrize("mode", MODES)
def test_content_regimes(mode, kind, shape):
    C, H, W = shape
    if kind == "one_equal":                        # channel 1 identical, the others not
        a, b = L.content("uniform", *shape, seed=7)
        b[1] = a[1]
    else:
        a, b = L.content(kind, *shape, seed=7)
    case = f"{kind} {mode} {'x'.join(map(str, shape))}"
    recs, (part, out, m), R = run(case, a[None], b[None], [0], mode)
    part, m = part.cpu(), {k: v.cpu() for k, v in m.items()}
    exact = [("zero where equal", zero_where_equal(part, R))]
    if kind in ("equal", "flat"):                  # flat saturates both planes to the same value in both modes
        exact.append(("equal: l1 / sq partials 0", bool((part[..., 0] == 0).all() and (part[..., 2] == 0).all())))
        exact.append(("equal: psnr inf", bool(torch.isposinf(m["psnr"]).all())))
        exact.append(("equal: psnr_channels inf", bool(torch.isposinf(m["psnr_channels"]).all())))
    if kind == "one_equal":
        pc = m["psnr_channels"][0]
        exact.append(("one equal: its PSNR only is inf",
                      bool(torch.isposinf(pc[1])) and bool(torch.isfinite(pc[[0, 2]]).all())))
        exact.append(("one equal: whole-image PSNR finite", bool(torch.isfinite(m["psnr"]).all())))
        exact.append(("one equal: its partials 0", bool((part[1, ..., 0] == 0).all() and (part[1, ..., 2] == 0).all())))
    if kind == "impulses":
        far = far_tiles(a, H, W)
        assert bool(far.any())
        exact.append(("impulses: l1 / sq partials 0 far from them",
                      bool((part[:, far][..., 0] == 0).all() and (part[:, far][..., 2] == 0).all())))
    assert_ok(recs, exact)


# ---- 3. special values ---------------------------------------------------------------------------------------------
SPECIAL_PIXELS = lambda H, W: [(0, 0), (H - 1, W - 1), (L.TH - 1, L.TW - 1), (L.TH, L.TW), (20, 40)]


def special_batch(H=37, W=70):
    """View k: a uniform render with SPECIALS[k] at five pixels of channel k % 3 (the first, the last of the plane,
    either side of a tile seam crossing, one inside), against a uniform target with SPECIALS[k + 1] at the same
    pixels.  -> (img [V, 3, H, W], gt [V, 3, H, W], channel of each view)."""
    S = M.SPECIALS
    V = len(S)
    g = torch.Generator().manual_seed(5)
    img, gt = torch.rand(V, 3, H, W, generator=g), torch.rand(V, 3, H, W, generator=g)
    chan = [k % 3 for k in range(V)]
    for k in range(V):
        for (y, x) in SPECIAL_PIXELS(H, W):
            img[k, chan[k], y, x] = S[k]
            gt[k, chan[k], y, x] = S[(k + 1) % V]
    return img, gt, chan


@pytest.mark.parametrize("mode", MODES)
def test_special_values(mode):
    """clamp: torch.clamp's semantics, so a NaN in either image makes the view's l1, ssim and psnr NaN, and the
    psnr of its channel, while its other channels stay finite.  png8: save_image + to_tensor on the CPU (NaN -> 0,
    +inf -> 1, -inf -> 0).  Every view is bit-identical to its result evaluated alone."""
    img, gt, chan = special_batch()
    V, C, H, W = img.shape
    rows = list(range(V))
    recs, (part, out, m), R = run(f"special values {mode}", img, gt, rows, mode)
    m = {k: v.cpu() for k, v in m.items()}
    exact = []
    for k, s in enumerate(M.SPECIALS):
        nan = mode == "clamp" and (math.isnan(s) or math.isnan(M.SPECIALS[(k + 1) % V]))
        views = (m["l1"][k], m["ssim"][k], m["psnr"][k])
        pc = m["psnr_channels"][k]
        others = [c for c in range(C) if c != chan[k]]
        if nan:
            exact.append((f"view {k} ({s}): l1, ssim, psnr NaN", all(bool(torch.isnan(x)) for x in views)))
            exact.append((f"view {k} ({s}): its channel's psnr NaN", bool(torch.isnan(pc[chan[k]]))))
        else:
            exact.append((f"view {k} ({s}): finite", all(bool(torch.isfinite(x)) for x in views) and
                          bool(torch.isfinite(pc[chan[k]]))))
        exact.append((f"view {k} ({s}): other channels finite", bool(torch.isfinite(pc[others]).all())))
        p1, o1 = M.metrics_kernel(img[k:k + 1].to(DEV), gt.to(DEV), [k], mode)
        exact.append((f"view {k} ({s}): alone", M.same_bits(p1, part[k * C:(k + 1) * C]) and
                      M.same_bits(o1[0], out[k])))
    assert_ok(recs, exact)


# ---- 4. cross-mode identities --------------------------------------------------------------------------------------
def test_png8_equals_clamp_on_8bit_inputs():
    """u8 / 255 in fp32 (what to_tensor yields) is a fixed point of both transforms: png8 partials and sums equal the
    clamp ones bit for bit."""
    g = torch.Generator().manual_seed(8)
    H, W = 53, 77
    img = torch.randint(0, 256, (3, 3, H, W), generator=g, dtype=torch.uint8).float().div(255).to(DEV)
    gt = torch.randint(0, 256, (3, 3, H, W), generator=g, dtype=torch.uint8).float().div(255).to(DEV)
    img[0, :, :8, :8] = gt[2, :, :8, :8]
    pc, oc = M.metrics_kernel(img, gt, [2, 0, 1], "clamp")
    pp, op = M.metrics_kernel(img, gt, [2, 0, 1], "png8")
    assert M.same_bits(pc, pp) and M.same_bits(oc, op)


@pytest.mark.parametrize("H,W", [(48, 64), (37, 53)])
def test_png8_is_clamp_of_the_saved_frames(H, W):
    """image_metrics(render, gt, "png8") equals image_metrics in clamp mode of gsb_frames_u8_batch(render) / 255
    against gsb_frames_u8_batch(gt) / 255, bit for bit: render.py's PNG frames feed metrics.py exactly the images
    the png8 convention assumes.  H W % 4 == 0 takes k_frames_u8's vector path, 37 x 53 the scalar one."""
    g = torch.Generator().manual_seed(H)
    img = (torch.rand(4, 3, H, W, generator=g) * 3.2 - 0.2).to(DEV)
    gt = (torch.rand(4, 3, H, W, generator=g) * 1.4 - 0.2).to(DEV)
    img[1, :, 3, 5] = torch.tensor([math.nan, math.inf, -math.inf])
    # to_tensor divides on the CPU; torch's CUDA division by a scalar multiplies by its reciprocal, which is one ulp
    # off at 126 of the 256 levels
    u8 = lambda x: quantise(x).cpu().permute(0, 3, 1, 2).float().div(255).contiguous().to(DEV)
    rows = [3, 1, 1, 0]
    want = image_metrics(u8(img), u8(gt), rows=rows, mode="clamp")
    got = image_metrics(img, gt, rows=rows, mode="png8")
    for k in got:
        assert M.same_bits(got[k], want[k]), (k, got[k], want[k])


# ---- 5. batch and addressing ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", MODES)
def test_rows_permuted_and_repeated(mode):
    """gt_row permuted and repeated, with rows at the first and the last target plane: every view bit-identical to its
    solo call, partials included, and within its bounds."""
    H, W, G = 37, 70, 4
    img, gt = _raw(15, H, W, seed=11).view(5, 3, H, W), _raw(12, H, W, seed=12).view(G, 3, H, W)
    rows = [3, 0, 3, 1, 2]
    recs, (part, out, _), _ = run(f"rows {mode}", img, gt, rows, mode)
    exact = []
    for v, r in enumerate(rows):
        p1, o1 = M.metrics_kernel(img[v:v + 1].to(DEV), gt.to(DEV), [r], mode)
        exact.append((f"view {v} alone", M.same_bits(p1, part[3 * v:3 * v + 3]) and M.same_bits(o1[0], out[v])))
        p2, o2 = M.metrics_kernel(img[v:v + 1].to(DEV), gt[r:r + 1].to(DEV), [0], mode)
        exact.append((f"view {v} against its plane alone", M.same_bits(p2, p1) and M.same_bits(o2, o1)))
    assert_ok(recs, exact)


@pytest.mark.parametrize("mode", MODES)
def test_misaligned_inputs(mode):
    """img and gt 4 bytes past a 16-byte boundary give the partials of an aligned copy, bit for bit."""
    V, C, H, W = 2, 3, 37, 70
    img, gt = _raw(V * C, H, W, seed=13).view(V, C, H, W), _raw(V * C, H, W, seed=14).view(V, C, H, W)
    bi = torch.empty(img.numel() + 4, device=DEV)
    bg = torch.empty(gt.numel() + 4, device=DEV)
    mi, mg = bi[1:1 + img.numel()].view(V, C, H, W), bg[1:1 + gt.numel()].view(V, C, H, W)
    mi.copy_(img)
    mg.copy_(gt)
    assert mi.data_ptr() % 16 == 4 and mg.data_ptr() % 16 == 4
    pa, oa = M.metrics_kernel(img.to(DEV), gt.to(DEV), [1, 0], mode)
    pm, om = M.metrics_kernel(mi, mg, [1, 0], mode)
    assert M.same_bits(pa, pm) and M.same_bits(oa, om)


@pytest.mark.parametrize("mode", MODES)
def test_batch_at_the_grid_z_limit(mode):
    """V C = 65535 planes (the grid's z limit) on 4 x 4 frames: accepted, and every view within its bounds; one more
    view is refused."""
    V, C, H, W, G = 21845, 3, 4, 4, 7
    g = torch.Generator().manual_seed(V)
    img = torch.rand(V, C, H, W, generator=g) * 1.4 - 0.2
    gt = torch.rand(G, C, H, W, generator=g) * 1.4 - 0.2
    rows = torch.randint(0, G, (V,), generator=g).tolist()
    recs, _, _ = run(f"grid z limit {mode}", img, gt, rows, mode)
    assert_ok(recs)
    with pytest.raises(GsbError):
        M.metrics_kernel(torch.zeros(V + 1, C, H, W, device=DEV), gt.to(DEV), rows + [0], mode)


# ---- 6. large frames -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", MODES)
def test_4k_frames(mode):
    """Two 3840 x 2160 views: all 16 200 x 3 partials of each against the fp64 restatement computed on the device,
    and both views' sums.  T = 16 200 partials per plane takes k_metrics_reduce far past its 256 threads, with
    T mod 256 = 72 and 3 T mod 256 = 216."""
    V, C, H, W = 2, 3, 2160, 3840
    g = torch.Generator(device=DEV).manual_seed(4)
    img = torch.rand(V, C, H, W, generator=g, device=DEV) * 3.2 - 0.2
    gt = torch.rand(V, C, H, W, generator=g, device=DEV)
    assert M.grid(H, W) == (135, 120)
    recs, (part, out, _), R = run(f"4K {mode}", img, gt, [1, 0], mode, ref_device=DEV)
    exact = [("every slot written", bool((part != M.SENTINEL).all()) and bool((out != M.SENTINEL).all()))]
    assert_ok(recs, exact)
