"""JointTrainer's SH layout at degrees 0..3 without a GPU (DESIGN.md section 4.16): the flat-buffer segments of each
degree, the refusals raised before anything is allocated, and point_cloud.ply files with 0, 9, 24 and 45 f_rest
columns (degree 0 has none)."""
import numpy as np
import pytest
import torch

from instantsplat_b200 import _lib
from instantsplat_b200 import scene_io as S
from instantsplat_b200.scenes import Scene
from instantsplat_b200.trainer import (SEGMENTS, JointTrainer, OptimConfig, _parse_capture, flat_layout,
                                       segment_widths, sh_rest_rows)

ROWS = {0: 0, 1: 3, 2: 8, 3: 15}


@pytest.mark.parametrize("D", [0, 1, 2, 3])
@pytest.mark.parametrize("P", [0, 1, 63, 64, 1000, 12_345])
def test_layout_of_each_degree(D, P):
    widths = segment_widths(ROWS[D])
    assert [n for n, _ in widths] == [n for n, _ in SEGMENTS]
    assert dict(widths)["f_rest"] == 3 * ROWS[D]
    assert sum(k for _, k in widths) == (14, 23, 38, 59)[D]
    seg, total = flat_layout(P, widths)
    end = 0
    for name, k in widths:
        b, e = seg[name]
        assert b == end and b % 64 == 0 and e % 64 == 0           # contiguous, every segment 256-byte aligned
        assert e - b == (P * k + 63) // 64 * 64 and e - b >= P * k
        end = e
    assert total == end
    if D == 0:
        assert seg["f_rest"][0] == seg["f_rest"][1]               # empty: no space, no tensor to launch
    if D == 3:
        assert (seg, total) == flat_layout(P)                     # the degree-3 layout is SEGMENTS'


@pytest.mark.parametrize("shape,rows", [((5, 0, 3), 0), ((5, 3, 3), 3), ((5, 8, 3), 8), ((5, 15, 3), 15),
                                        ((5, 45), 15), ((5, 9), 3)])
def test_rest_rows(shape, rows):
    assert sh_rest_rows(torch.zeros(shape), 5) == rows


@pytest.mark.parametrize("shape,match", [((5, 4, 3), "0, 3, 8 or 15"), ((5, 24, 3), "degree 4"),
                                         ((5, 1, 3), "0, 3, 8 or 15"), ((5, 3, 2), r"\[P, M-1, 3\]"),
                                         ((4, 3, 3), r"\[P, M-1, 3\]"), ((5, 10), r"\[P, M-1, 3\]")])
def test_rest_rows_refused(shape, match):
    with pytest.raises(_lib.GsbError, match=match):
        sh_rest_rows(torch.zeros(shape), 5)


def _scene(rows, P=7):
    g = torch.Generator().manual_seed(0)
    params = dict(xyz=torch.randn(P, 3, generator=g), f_dc=torch.randn(P, 1, 3, generator=g),
                  f_rest=torch.randn(P, rows, 3, generator=g), opacity=torch.randn(P, 1, generator=g),
                  scaling=torch.randn(P, 3, generator=g), rotation=torch.randn(P, 4, generator=g))
    poses = torch.tensor([[1.0, 0, 0, 0, 0, 0, 0]] * 2)
    return Scene(params, poses, 32, 24, 0.9, 0.7, sh_degree=0)


@pytest.mark.parametrize("D,max_deg", [(0, 1), (0, 3), (1, 2), (1, 3), (2, 3)])
def test_max_sh_degree_above_the_stored_degree_is_refused(D, max_deg):
    """Refused in the constructor before the first device allocation (this machine may have no GPU at all)."""
    cfg = OptimConfig()
    cfg.max_sh_degree = max_deg
    with pytest.raises(_lib.GsbError, match=f"max_sh_degree {max_deg} exceeds the scene's stored SH degree {D}"):
        JointTrainer(_scene(ROWS[D]), "cuda", cfg=cfg)


@pytest.mark.parametrize("rows", [1, 2, 5, 24])
def test_rest_rows_not_a_square_minus_one_are_refused(rows):
    cfg = OptimConfig()
    cfg.max_sh_degree = 0
    with pytest.raises(_lib.GsbError, match="rows per Gaussian"):
        JointTrainer(_scene(rows), "cuda", cfg=cfg)


@pytest.mark.parametrize("D", [0, 1, 2, 3])
def test_capture_parser_takes_each_degree(D):
    """A capture() tuple of GaussianModel(D) passes the checkpoint parser, f_rest [P, M-1, 3] and its moments."""
    P, r = 6, ROWS[D]
    t = lambda *s: torch.zeros(*s)
    shapes = dict(xyz=(P, 3), f_dc=(P, 1, 3), f_rest=(P, r, 3), opacity=(P, 1), scaling=(P, 3), rotation=(P, 4))
    groups = [dict(name=n, params=[i], lr=0.0) for i, n in enumerate(list(shapes) + ["pose"])]
    state = {i: dict(step=3, exp_avg=t(*shapes[n]), exp_avg_sq=t(*shapes[n])) for i, n in enumerate(shapes)}
    cap = (0, t(P, 3), t(P, 1, 3), t(P, r, 3), t(P, 3), t(P, 4), t(P, 1), t(P), t(P, 1), t(P, 1),
           dict(state=state, param_groups=groups), 1.0, t(2, 7))
    parsed = _parse_capture(cap, 5)
    assert tuple(parsed["f_rest"].shape) == (P, r, 3) and parsed["steps"]["f_rest"] == 3


@pytest.mark.parametrize("D", [0, 1, 2, 3])
@pytest.mark.parametrize("filt", [False, True])
def test_ply_round_trip_at_each_degree(tmp_path, D, filt):
    P, r = 11, ROWS[D]
    rng = np.random.default_rng(D)
    a = dict(xyz=rng.standard_normal((P, 3)), f_dc=rng.standard_normal((P, 1, 3)), f_rest=rng.standard_normal((P, r, 3)),
             opacity=rng.standard_normal((P, 1)), scaling=rng.standard_normal((P, 3)),
             rotation=rng.standard_normal((P, 4)))
    a = {k: v.astype(np.float32) for k, v in a.items()}
    f3 = rng.random((P, 1)).astype(np.float32) if filt else None
    path = str(tmp_path / "point_cloud.ply")
    S.save_gaussians_ply(path, a["xyz"], a["f_dc"], a["f_rest"], a["opacity"], a["scaling"], a["rotation"], f3)
    names = list(S._read_ply(path).dtype.names)
    assert names == S.gaussian_ply_fields(3 * r) + (["filter_3D"] if filt else [])
    if D == 0:
        assert not any(n.startswith("f_rest_") for n in names)
    b = S.load_gaussians_ply(path)
    assert tuple(b["f_rest"].shape) == (P, r, 3) and b["f_rest"].dtype == np.float32
    for k in a:
        assert np.array_equal(a[k], b[k]), k
    assert ("filter_3D" in b) == filt
