"""Batched pose tracking (-m gpu): PoseTracker.optimize_batch / render_batch against V single-view calls, bit for bit
(torch.equal), and one small case against the CPU restatement of render.py:113-161."""
import math

import pytest
import torch

from instantsplat_b200 import GsbError
from instantsplat_b200.frame import mip_filter3d, read_R
from instantsplat_b200.scenes import surface_scene
from instantsplat_b200.tracking import PoseTracker

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _tracker(sc, deg, mip=False, **kw):
    p = sc.params
    f3d = None
    if mip:
        f3d = mip_filter3d(p["xyz"].to(DEV), sc.poses.to(DEV), sc.width, sc.height, math.tan(sc.fovx / 2),
                           math.tan(sc.fovy / 2))
    return PoseTracker(p["xyz"], p["rotation"], p["scaling"], p["opacity"], p["f_dc"], p["f_rest"], sc.width, sc.height,
                       sc.fovx, sc.fovy, sh_degree=deg, device=DEV, kernel_size=0.1 if mip else None, filter_3D=f3d, **kw)


def _with_big_gaussian(sc):
    """Append one faint Gaussian that covers the whole frame of every view, so k_big_rects has work."""
    p = dict(sc.params)
    c = sc.params["xyz"].mean(0, keepdim=True)
    p["xyz"] = torch.cat([p["xyz"], c])
    p["rotation"] = torch.cat([p["rotation"], torch.tensor([[1.0, 0, 0, 0]])])
    p["scaling"] = torch.cat([p["scaling"], torch.full((1, 3), math.log(4.0))])
    p["opacity"] = torch.cat([p["opacity"], torch.full((1, 1), -3.0)])
    p["f_dc"] = torch.cat([p["f_dc"], torch.full((1, 1, 3), 0.3)])
    p["f_rest"] = torch.cat([p["f_rest"], torch.zeros(1, *p["f_rest"].shape[1:])])
    sc.params = p
    return sc


def _inputs(tr, poses, seed, blind=None):
    """Targets rendered at the true poses, seeded perturbations as starts; row `blind` starts behind the scene."""
    gts = torch.stack([tr.render(p).cpu() for p in poses])
    g = torch.Generator().manual_seed(seed)
    init = poses + 0.01 * torch.randn(poses.shape, generator=g)
    if blind is not None:
        init[blind, 4:] = torch.tensor([0.0, 0.0, -100.0])       # every Gaussian behind the camera: mask sum 0
    return init, gts


def _assert_batch_equals_single(tr, init, gts, n_it, **kw):
    bp, bl, btr = tr.optimize_batch(init, gts, num_iter=n_it, return_trace=True, **kw)
    assert bp.shape == (init.shape[0], 7) and bl.shape == (init.shape[0],) and btr.shape == (init.shape[0], n_it)
    for v in range(init.shape[0]):
        p, l, t = tr.optimize(init[v], gts[v], num_iter=n_it, return_trace=True)
        assert torch.equal(bp[v], p), (v, bp[v], p)
        assert float(bl[v]) == l, (v, float(bl[v]), l)
        assert torch.equal(btr[v], t), (v, btr[v], t)
    rb = tr.render_batch(bp)
    for v in range(init.shape[0]):
        assert torch.equal(rb[v], tr.render(bp[v])), v
    return bp, bl, btr


CASES = [  # (V, deg, mip, blind view, big Gaussian)
    (1, 3, False, None, False),
    (3, 3, False, 1, True),
    (5, 3, False, 4, True),
    (3, 0, False, None, True),
    (3, 3, True, 0, True),
]


@pytest.mark.parametrize("V,deg,mip,blind,big", CASES)
def test_optimize_batch_equals_single_view(V, deg, mip, blind, big):
    sc = surface_scene(6000, 5, 215, 167, seed=61, sh_degree=deg)      # W, H not multiples of 16; 154 tiles
    if big:
        sc = _with_big_gaussian(sc)
    tr = _tracker(sc, deg, mip)
    init, gts = _inputs(tr, sc.poses[:V], seed=V, blind=blind)
    _, bl, btr = _assert_batch_equals_single(tr, init, gts, 6)
    if blind is not None:
        assert float(btr[blind, 0]) == 0.0                        # no pixel passes the mask: loss 0
    if big:                                                       # its tile rect exceeds kBigRect = 128 tiles
        tr.render(sc.poses[0])
        assert int(tr.frame.radii[0, -1]) > 215, int(tr.frame.radii[0, -1])


def test_optimize_batch_long_tile_lists():
    """Tile lists in every size class of the per-tile sort (<= 2048, <= 8192, longer), in every view of the batch."""
    from test_binning_lists import lengths_scene
    sc, _ = lengths_scene()
    tr = _tracker(sc, 0)
    poses = sc.poses[0].expand(3, 7).clone()
    init, gts = _inputs(tr, poses, seed=5)
    init = poses + 0.1 * (init - poses)                           # keep the lists in their classes
    tr.render_batch(init)
    st = tr.frame.status.cpu().tolist()
    assert st[4] >= 3 and st[5] >= 3, st                         # both long-list queues are non-empty
    _assert_batch_equals_single(tr, init, gts, 4)


def test_render_batch_beyond_65536_tiles():
    sc = surface_scene(3000, 12, 1920, 1080, seed=9, sh_degree=3)
    tr = _tracker(sc, 3)
    assert 12 * 120 * 68 > 65536
    rb = tr.render_batch(sc.poses)
    assert rb.shape == (12, 3, 1080, 1920)
    for v in range(12):
        assert torch.equal(rb[v], tr.render(sc.poses[v])), v


def test_max_batch_chunks_equal_unchunked():
    sc = surface_scene(5000, 5, 96, 72, seed=3, sh_degree=3)
    tr = _tracker(sc, 3)
    init, gts = _inputs(tr, sc.poses, seed=11)
    a = tr.optimize_batch(init, gts, num_iter=5, return_trace=True)
    b = tr.optimize_batch(init, gts, num_iter=5, return_trace=True, max_batch=2)
    for x, y in zip(a, b):
        assert torch.equal(x, y)


def test_odd_frame_chunks_and_device_targets():
    """3 H W odd: every other view of a [V, 3, H, W] tensor starts unaligned.  Chunks of two (chunk bases unaligned)
    and targets passed as a CUDA tensor (optimize then reads unaligned slices) give the single-view bits."""
    sc = surface_scene(6000, 5, 215, 167, seed=61, sh_degree=3)
    assert (3 * 215 * 167) % 4 != 0
    tr = _tracker(sc, 3)
    init, gts = _inputs(tr, sc.poses, seed=13)
    gts_dev = gts.to(DEV)
    whole = tr.optimize_batch(init, gts, num_iter=5, return_trace=True)
    chunked = _assert_batch_equals_single(tr, init, gts_dev, 5, max_batch=2)
    for x, y in zip(whole, chunked):
        assert torch.equal(x, y)


def test_masked_l1_partition_ignores_alignment():
    """The masked L1 sums of a slice that starts 4 bytes past a 16-byte boundary equal those of an aligned copy."""
    from instantsplat_b200 import _lib
    L = _lib.lib()
    g = torch.Generator().manual_seed(3)
    shape = (3, 37, 53)
    n = 3 * 37 * 53
    buf_i = (torch.rand(2 * n + 1, generator=g) - 0.3).to(DEV)
    buf_g = torch.rand(2 * n + 1, generator=g).to(DEV)
    img, gt = buf_i[1:].view(2, *shape), buf_g[1:].view(2, *shape)          # views 0 and 1 both unaligned
    res = []
    for a, b in ((img, gt), (img.clone(), gt.clone())):
        sums = torch.zeros(2, 2, dtype=torch.float64, device=DEV)
        dL = torch.empty(2 * n + 1, device=DEV)[1:].view(2, *shape) if a.data_ptr() % 16 else torch.empty_like(a)
        _lib.check(L.gsb_l1_mask_fwd_bwd_batch(2, *shape, a.data_ptr(), b.data_ptr(), 0.0, sums.data_ptr(),
                                               dL.data_ptr(), _lib.stream_ptr()), "gsb_l1_mask_fwd_bwd_batch")
        res.append((sums.cpu(), dL.cpu()))
    assert img.data_ptr() % 16 != 0
    assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1])


def test_optimize_batch_matches_reference_restatement():
    from test_tracking import reference_tracking
    sc = surface_scene(6000, 3, 128, 96, seed=61, sh_degree=2)
    n_it = 12
    tr = _tracker(sc, 2)
    from oracle import gs_oracle as O
    cam = O.Camera.instantsplat(sc.width, sc.height, sc.fovx, sc.fovy, sh_degree=2)
    views = (1, 2)
    gts, inits = [], []
    with torch.no_grad():
        for i, view in enumerate(views):
            gt, _ = O.render_instantsplat(sc.params["xyz"], sc.params["rotation"], sc.params["scaling"],
                                          sc.params["opacity"], sc.params["f_dc"], sc.params["f_rest"], sc.poses[view], cam)
            gts.append(gt)
            inits.append(sc.poses[view] + (i + 1) * torch.tensor([0.0, 0.004, -0.003, 0.002, 0.01, -0.008, 0.012]))
    pose, best, trace = tr.optimize_batch(torch.stack(inits), torch.stack(gts), num_iter=n_it, return_trace=True)
    for i, view in enumerate(views):
        ref_pose, ref_best, ref_losses, _ = reference_tracking(sc, view, gts[i], inits[i], n_it, 2)
        dl = max(abs(a - float(b)) for a, b in zip(ref_losses, trace[i]))
        assert dl < 2e-5, (view, dl)
        assert abs(float(best[i]) - ref_best) < 2e-5
        assert float((pose[i] - ref_pose).abs().max()) < 2e-4, (view, pose[i], ref_pose)


def test_overflow_and_bad_input():
    sc = surface_scene(20000, 12, 256, 192, seed=4, sh_degree=0)
    tr = _tracker(sc, 0)
    tr.render_batch(sc.poses)
    assert read_R(tr.host_status) > 65536 + 1000                 # more instances than the capacity floor
    small = _tracker(sc, 0)
    small.headroom = 0.0                                           # binning buffer = the 65536-instance floor
    gts = torch.zeros(12, 3, 192, 256)
    with pytest.raises(GsbError):
        small.optimize_batch(sc.poses, gts, num_iter=2)
    with pytest.raises(ValueError):
        tr.optimize_batch(sc.poses[:, :6], gts, num_iter=2)
    with pytest.raises(ValueError):
        tr.optimize_batch(sc.poses, gts[:11], num_iter=2)
    with pytest.raises(ValueError):
        tr.optimize_batch(sc.poses, gts[:, :, :100], num_iter=2)
    with pytest.raises(ValueError):
        tr.render_batch(sc.poses[0])
    p, l = tr.optimize_batch(sc.poses[:0], gts[:0], num_iter=2)
    assert p.shape == (0, 7) and l.shape == (0,)
