"""Per-tile lists of the binning stage (gs_bin.cu), checked directly, at every list-length class of the per-tile sort:

    <= 2048 entries          k_tile_sort: bucket pass + insertion sort, or flip-bitonic in shared memory when one
                             bucket holds more than 24 keys (skew)
    2049 .. 8192             k_tile_sort_long, the same in 96 KB of shared memory
    > 8192                   k_tile_sort_long, HUGE: flip-bitonic in place in global memory

The scenes are built from one-tile Gaussians (sigma < 1 px, radius <= 4, centre near the tile centre), so each tile's
list length is exactly the number placed in it, with the cull on or off.  Every scene's lists are checked exactly
(tests/_binning.py) and compared with the oracle's rect lists, with the cull on and off; then image and gradients are
compared with the fp64 oracle over the full frame for three blend kernels, gradients also per Gaussian.
"""
import math

import numpy as np
import pytest
import torch

import _binning as BL
from _parity import DEV, ROW_TOL_SCENES, compare_fused, settings_for
from instantsplat_b200.scenes import Scene, _single_threaded, make_config, random_scene

BLEND_VARIANTS = ((2, 1), (2, 0), (1, 0))    # (blend_version, stage_bulk): v2 bulk TMA staging, v2 cooperative, v1


def test_decoder_layout_matches_library():
    """tests/_binning.py restates the BinView layout of gs_internal.cuh; its total must be gsb_binning_bytes."""
    import __graft_entry__ as G
    G.build()
    import instantsplat_b200 as I
    L = I.lib()
    for cap in (0, 1, 7, 8, 31, 1000, 65536, 12345678):
        for W, H in ((1, 1), (16, 16), (17, 33), (80, 56), (64, 48), (1920, 1080), (3840, 2160), (4095, 17)):
            lay = BL.bin_layout(cap, W, H)
            assert lay["total"] == L.gsb_binning_bytes(cap, W, H), (cap, W, H)
            ntiles = ((W + 15) // 16) * ((H + 15) // 16)
            assert lay["ranges"][1] == 8 * ntiles and lay["ids"][1] == 4 * (max(cap, 1) + 8)
            assert all(v[0] % 256 == 0 for k, v in lay.items() if k != "total")


def test_max_bucket_restates_the_kernel():
    """The skew probe: keys that share their depth land in one bucket; spread depths do not."""
    ids = np.arange(100, dtype=np.int64)
    same = (np.int64(0x40200000) << 32) | ids
    assert BL.max_bucket(same[:25], 2048) == 25
    spread = ((np.int64(0x40000000) + 4096 * ids) << 32) | ids
    assert BL.max_bucket(spread, 2048) == 1


# ---- scenes -------------------------------------------------------------------------------------------------------
@_single_threaded
def one_tile_scene(W, H, per_tile, seed, fovx_deg=60.0):
    """per_tile: list of (tile, depths [n], opacities [n]) -> Scene of one-tile Gaussians (identity pose, SH degree 0).
    Centres are pixel centres 5..11 px into the tile and sigma is 0.5-0.75 px on screen.  With the 0.3 px^2 low-pass,
    the view-angle stretch (<= 1.52 in variance) and the eigenvalue floor sqrt(0.1), the 3-sigma radius is 3 or 4 px
    (at most 3.64 before ceil), so the rect is exactly one tile.  Gaussian ids are shuffled, so id order is not the
    order of emission."""
    g = torch.Generator().manual_seed(seed)
    fovx = math.radians(fovx_deg)
    fovy = 2.0 * math.atan(math.tan(fovx / 2) * H / W)
    tx_, ty_ = math.tan(fovx / 2), math.tan(fovy / 2)
    fx = W / (2 * tx_)
    gx = (W + 15) // 16
    cols = []
    for t, z, op in per_tile:
        n = len(z)
        z = torch.as_tensor(z, dtype=torch.float64)
        ty, tx = divmod(t, gx)
        u = 16 * tx + torch.randint(5, 12, (n,), generator=g).double()
        v = 16 * ty + torch.randint(5, 12, (n,), generator=g).double()
        x = ((2 * u + 1) / W - 1) * z * tx_
        y = ((2 * v + 1) / H - 1) * z * ty_
        s_px = 0.5 + 0.25 * torch.rand(n, generator=g).double()
        cols.append((torch.stack([x, y, z], 1), s_px * z / fx, torch.as_tensor(op, dtype=torch.float64)))
    xyz = torch.cat([c[0] for c in cols]).float()
    sig = torch.cat([c[1] for c in cols])
    op = torch.cat([c[2] for c in cols])
    P = xyz.shape[0]
    perm = torch.randperm(P, generator=g)
    xyz = xyz[perm].contiguous()
    scaling = torch.log(sig[perm]).float()[:, None].expand(P, 3).contiguous()
    opacity = torch.log(op[perm] / (1 - op[perm])).float()[:, None].contiguous()
    rotation = torch.zeros(P, 4)
    rotation[:, 0] = 1.0
    f_dc = torch.randn(P, 1, 3, generator=g)
    f_rest = torch.zeros(P, 15, 3)
    return Scene(dict(xyz=xyz, f_dc=f_dc, f_rest=f_rest, opacity=opacity, scaling=scaling, rotation=rotation),
                 torch.tensor([[1.0, 0, 0, 0, 0, 0, 0]]), W, H, fovx, fovy, 0, name="one-tile")


def lengths_scene():
    """64x48 frame, one tile per list-length class boundary: 1, 24, 25, 2047, 2048, 2049, 8191, 8192, 8193, 12 345 and
    40 000 entries (one tile empty).  Depths are continuous (no skew).  Lists >= 2047 are faint (opacity 0.005-0.007:
    alpha >= 1/255 at the centre pixel and at most its four neighbours), so they are walked to the end without early
    termination: at 40 000 entries T stays above 1e-3 and n_contrib passes 8192."""
    g = torch.Generator().manual_seed(61)
    counts = (1, 24, 25, 2047, 2048, 2049, 8191, 8192, 8193, 12_345, 40_000, 0)
    per = []
    for t, n in enumerate(counts):
        z = 2.0 + 6.0 * torch.rand(n, generator=g, dtype=torch.float64)
        op = (0.005 + 0.002 * torch.rand(n, generator=g, dtype=torch.float64)) if n >= 2047 else \
            (0.05 + 0.5 * torch.rand(n, generator=g, dtype=torch.float64))
        per.append((t, z, op))
    return one_tile_scene(64, 48, per, seed=62), dict(max_list=40_000, n_large=3, n_huge=3)


def ties_and_skew_scene():
    """64x32 frame.  Exact depth ties (z in {2, 2.5, 3}, exactly representable, identity pose) in lists of 24 (one
    bucket of exactly kSkew: insertion sort on the id), 25 (skew fallback), 2048, 2049, 8192 and 8193 entries; and skew
    without ties -- a band of depths 1e-4 wide plus three outliers at z = 40 -- in lists of 2003 and 6003 entries."""
    g = torch.Generator().manual_seed(71)
    tie = lambda n, vals=(2.0, 2.5, 3.0): torch.tensor(vals, dtype=torch.float64)[
        torch.randint(0, len(vals), (n,), generator=g)]
    band = lambda n: torch.cat([3.0 + 1e-4 * torch.rand(n, generator=g, dtype=torch.float64),
                                torch.full((3,), 40.0, dtype=torch.float64)])
    zs = [tie(24, (2.5,)), tie(25, (2.5,)), tie(2048), tie(2049), tie(8192), tie(8193), band(2000), band(6000)]
    per = [(t, z, 0.02 + 0.4 * torch.rand(len(z), generator=g, dtype=torch.float64)) for t, z in enumerate(zs)]
    return one_tile_scene(64, 32, per, seed=72), dict(max_list=8193, n_large=3, n_huge=1)


SKEWED_TILES = {"ties_and_skew": (1, 2, 3, 4, 6, 7), "lengths": ()}


# ---- GPU ----------------------------------------------------------------------------------------------------------
def forward_state(sc, view=0, deg=0, cull=True):
    import instantsplat_b200 as I
    import instantsplat_b200.rasterizer as R
    prm = {k: v.to(DEV).clone().requires_grad_(True) for k, v in sc.params.items()}
    pose = sc.poses[view].to(DEV).clone().requires_grad_(True)
    saved = R.EXACT_CULL
    try:
        R.EXACT_CULL = cull
        img, _ = I.rasterize_fused(prm["xyz"], prm["rotation"], prm["scaling"], prm["opacity"], prm["f_dc"],
                                   prm["f_rest"], pose, torch.zeros(sc.P, 3, device=DEV), settings_for(sc, deg, sc.bg))
    finally:
        R.EXACT_CULL = saved
    return img.grad_fn.st


def check_scene_lists(sc, expect, exact, deg=0, view=0, skewed=()):
    """List checks with the cull off and on; returns the records."""
    proj = BL.oracle_proj(sc, view, deg)
    out = {}
    for cull in (False, True):
        d = BL.decode(forward_state(sc, view, deg, cull))
        s = BL.check_lists(d)
        for k, v in (expect or {}).items():
            assert s[k] == v, (cull, k, s)
        s.update(BL.compare_with_oracle(d, proj, cull, exact=exact))
        if not cull:
            for t in skewed:       # the scene drives these tiles into the bitonic fallback
                lo, hi = (int(v) for v in d["ranges"][t])
                cap = BL.SMALL_LIST if hi - lo <= BL.SMALL_LIST else BL.LARGE_LIST
                if hi - lo <= BL.LARGE_LIST:
                    assert BL.max_bucket(d["pairs"][lo:hi].cpu().numpy(), cap) > BL.SKEW, t
        out["cull" if cull else "no_cull"] = s
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["lengths", "ties_and_skew"])
def test_constructed_scene_lists_and_parity(which):
    import instantsplat_b200 as I
    from _parity import REPORT
    sc, expect = lengths_scene() if which == "lengths" else ties_and_skew_scene()
    lists = check_scene_lists(sc, expect, exact=True, skewed=SKEWED_TILES[which])
    for k in ("no_cull", "cull"):
        assert lists[k]["mismatched_tiles"] == 0, lists
    if which == "lengths":
        st = forward_state(sc)
        hw = sc.width * sc.height
        nc = st.image[BL.align_up(hw * 4):BL.align_up(hw * 4) + hw * 4].view(torch.int32).cpu()
        assert int(nc.max()) > 8192, int(nc.max())      # the blend walked past list position 8192
        lists["n_contrib_max"] = int(nc.max())
        lists["pixels_n_contrib_over_8192"] = int((nc > 8192).sum())
    L = I.lib()
    cache = {}
    try:
        for ver, bulk in BLEND_VARIANTS:
            assert L.gsb_set_option(b"blend_version", ver) == 0 and L.gsb_set_option(b"stage_bulk", bulk) == 0
            rec = compare_fused(f"{which} (one-tile Gaussians, {sc.P}) blend v{ver} bulk {bulk}", sc, 0, 0,
                                torch.tensor([0.1, 0.2, 0.3]), row_tol=ROW_TOL_SCENES, oracle_cache=cache)
            rec["list_checks"] = lists
    finally:
        L.gsb_set_option(b"blend_version", 2)
        L.gsb_set_option(b"stage_bulk", 1)
    ft = cache["aux"]["final_T"]
    if which == "lengths":
        assert float(ft[:16, 48:64].min()) > 1e-3      # tile 11 is empty; tile 10 (40 000 entries): no early stop
        assert float(ft[32:48, 32:48].min()) > 1e-3
    REPORT.append(dict(case=f"{which}: oracle final_T min per tile",
                       final_T_min=[float(ft[ty * 16:(ty + 1) * 16, tx * 16:(tx + 1) * 16].min())
                                    for ty in range(sc.height // 16) for tx in range(sc.width // 16)]))


@pytest.mark.gpu
def test_general_scene_lists_match_oracle():
    """Lists of random scenes against the oracle's rect lists, cull off and on.  Mismatches are allowed only where
    the oracle's rect bound or depth lies within rounding (counted in the report); config 0 has ~50 tiles in the
    2049-8192 class."""
    from _parity import REPORT
    for name, sc, deg in (("random 600 80x56", random_scene(600, 80, 56, seed=21, sh_degree=0), 0),
                          ("configs[0] 10k 256x256", make_config(0), 3)):
        lists = check_scene_lists(sc, None, exact=False, deg=deg)
        if name.startswith("configs[0]"):
            assert lists["no_cull"]["n_large"] > 0, lists
        REPORT.append(dict(case=f"list checks: {name}", list_checks=lists))
        for k in ("no_cull", "cull"):
            assert lists[k]["mismatched_tiles"] <= max(2, lists[k]["tiles"] // 100), lists
