"""The blend backward's batched moment reduction (k_blend_bwd2 with BATCH, DESIGN.md section 4.3) against the per-entry
warp butterfly it replaces (gsb_set_option("blend_bwd_batch", 0)), word for word: for the same forward state, every
64-bit fixed-point accumulator word, and every gradient the backward returns, must be identical.

The batches hold 3 list entries and may span a staging chunk (kChunkB = 192 entries in the batched backward, 224 in
the butterfly one).  The populations end a warp's walk on every batch phase, inside a chunk and on both sides of a
chunk boundary, give one tile entries that each reach a single lane, and cover tracking mode (8 values per entry),
the Mip 2D filter on and off, cooperative staging and frames that are not a multiple of 16.
"""
import pytest
import torch

from _parity import DEV, settings_for
from test_blend_edges import clamp_scene, edge_scene, saturation_scene, signed_dL
from test_projection_edges import build_scene, camera_of

CHUNK_B = 192                  # kChunkB (GSB_BWD_CHUNK) of the batched backward


def _run(sc, dL, batch, pose_only=False, kernel_size=None, bulk=1):
    import _blend as BD
    import _geom as GM
    import instantsplat_b200 as I
    L = I.lib()
    assert L.gsb_set_option(b"blend_bwd_batch", int(batch)) == 0 and L.gsb_set_option(b"stage_bulk", bulk) == 0
    try:
        prm = {k: v.to(DEV).clone().requires_grad_(not pose_only) for k, v in sc.params.items()}
        pose = sc.poses[0].to(DEV).clone().requires_grad_(True)
        m2 = torch.zeros(sc.P, 3, device=DEV, requires_grad=not pose_only)
        rs = settings_for(sc, 0, torch.tensor((0.3, 0.6, 0.9)))
        if kernel_size is not None:
            rs = rs._replace(kernel_size=kernel_size)
        img, _ = I.rasterize_fused(prm["xyz"], prm["rotation"], prm["scaling"], prm["opacity"], prm["f_dc"],
                                   prm["f_rest"], pose, m2, rs)
        st = img.grad_fn.st
        img.backward(dL.to(DEV))
        torch.cuda.synchronize()
        raw = BD.decode_moments(st, GM.decode(st))["raw"]
        grads = {k: v.grad.detach().cpu() for k, v in prm.items() if v.grad is not None}
        grads["pose"] = pose.grad.detach().cpu()
        if m2.grad is not None:
            grads["means2D"] = m2.grad.detach().cpu()
        return raw, grads, img.detach().cpu()
    finally:
        L.gsb_set_option(b"blend_bwd_batch", 1)
        L.gsb_set_option(b"stage_bulk", 1)


def check_same(sc, make_dL, **kw):
    """Both reductions on the same frame: identical image, accumulator words and gradients.  -> number of
    non-zero accumulator words."""
    dL = make_dL(sc.height, sc.width).float()
    raw0, g0, img0 = _run(sc, dL, False, **kw)
    raw1, g1, img1 = _run(sc, dL, True, **kw)
    assert torch.equal(img0, img1)
    assert torch.equal(raw0, raw1), f"{int((raw0 != raw1).sum())} of {raw0.numel()} accumulator words differ"
    assert g0.keys() == g1.keys()
    for k in g0:
        assert torch.equal(g0[k], g1[k]), k
    return int(raw1.count_nonzero())


def stack_scene(n, W=16, H=16, seed=501):
    """n wide, faint Gaussians (sigma 24-30 px, opacity 0.012-0.015) over the middle of a W x H frame at distinct
    depths: every entry of every tile list reaches every pixel of the tile and no pixel terminates (T stays above
    0.985^n), so each warp's walk reduces exactly n entries."""
    g = torch.Generator().manual_seed(seed)
    _, _, tx, ty, fx = camera_of(W, H)
    r = lambda *s: torch.rand(*s, generator=g, dtype=torch.float64)
    z = 2.0 + 2.0 * (torch.arange(n, dtype=torch.float64) + r(n)) / max(n, 1)
    u, v = W / 2 - 0.5 + r(n) - 0.5, H / 2 - 0.5 + r(n) - 0.5
    pc = torch.stack([((2 * u + 1) / W - 1) * z * tx, ((2 * v + 1) / H - 1) * z * ty, z], 1)
    sig = ((24.0 + 6.0 * r(n)) * z / fx)[:, None].expand(n, 3).contiguous()
    return build_scene([(pc, sig, 0.012 + 0.003 * r(n))], W, H, seed=seed + 1)


def single_lane_scene(W=16, H=16, seed=511):
    """300 tiny, faint Gaussians (sigma 0.25 px, 0.6 px after the 0.3 px^2 dilation; opacity 0.006-0.012) on pixel
    centres of one tile: alpha >= 1/255 at the centre pixel only (o G < 1/255 one pixel away), so each entry
    contributes to one lane of one warp and every batch row holds one non-zero column."""
    g = torch.Generator().manual_seed(seed)
    _, _, tx, ty, fx = camera_of(W, H)
    n = 300
    z = 2.0 + 3.0 * torch.rand(n, generator=g, dtype=torch.float64)
    u = torch.randint(0, W, (n,), generator=g).double()
    v = torch.randint(0, H, (n,), generator=g).double()
    pc = torch.stack([((2 * u + 1) / W - 1) * z * tx, ((2 * v + 1) / H - 1) * z * ty, z], 1)
    sig = (0.25 * z / fx)[:, None].expand(n, 3).contiguous()
    return build_scene([(pc, sig, 0.006 + 0.006 * torch.rand(n, generator=g, dtype=torch.float64))], W, H, seed=seed + 1)


# list lengths (= entries reduced per warp) at every batch phase and around the batched backward's chunk boundaries
STACKS = (1, 2, 3, 4, 5, 6, 7, 100, CHUNK_B - 1, CHUNK_B, CHUNK_B + 1, CHUNK_B + 2, 2 * CHUNK_B, 2 * CHUNK_B + 1, 224)


@pytest.mark.gpu
@pytest.mark.parametrize("pose_only", [False, True])
def test_batch_ends(pose_only):
    """Lists whose walk ends mid-batch (n mod 3 = 1, 2), on a full batch, mid-chunk and on, one before and one after
    a chunk boundary."""
    for n in STACKS:
        sc = stack_scene(n)
        nz = check_same(sc, signed_dL(600 + n), pose_only=pose_only)
        assert nz >= 6 * n, (n, nz)


@pytest.mark.gpu
@pytest.mark.parametrize("pose_only", [False, True])
def test_single_lane_entries(pose_only):
    sc = single_lane_scene()
    assert check_same(sc, signed_dL(610), pose_only=pose_only) > 0


@pytest.mark.gpu
@pytest.mark.parametrize("pose_only", [False, True])
@pytest.mark.parametrize("kernel_size", [None, 0.1])
def test_saturation_and_clamp(pose_only, kernel_size):
    """Long lists ending anywhere in the first three chunks (early termination), and clamped alphas; Mip off / on."""
    for sc, seed in ((saturation_scene(), 620), (clamp_scene(), 621)):
        assert check_same(sc, signed_dL(seed), pose_only=pose_only, kernel_size=kernel_size) > 0


@pytest.mark.gpu
def test_cooperative_staging():
    assert check_same(saturation_scene(), signed_dL(630), bulk=0) > 0


@pytest.mark.gpu
@pytest.mark.parametrize("pose_only", [False, True])
def test_frames_not_multiple_of_16(pose_only):
    for k, (W, H) in enumerate(((17, 9), (33, 20), (47, 31), (100, 75))):
        assert check_same(edge_scene(W, H, 640 + k), signed_dL(641 + k), pose_only=pose_only) > 0


@pytest.mark.gpu
def test_bad_option_value():
    import instantsplat_b200 as I
    L = I.lib()
    assert L.gsb_set_option(b"blend_bwd_batch", 2) != 0 and L.gsb_set_option(b"blend_bwd_batch", -1) != 0
