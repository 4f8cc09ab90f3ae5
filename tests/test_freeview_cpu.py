"""The free-view fly-through, host side (no GPU): the 8-bit frame entry point is declared and exported, the trajectory
and the 7-vectors equal the reference's own functions bit for bit (tests/golden/freeview.npz, made by
oracle/make_golden_freeview.py), the PNG writer writes save_image's files, and the refusals fire before any device work."""
import os
import re

import numpy as np
import pytest
import torch

from instantsplat_b200 import freeview as F
from instantsplat_b200.scene_io import write_colmap_text

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "freeview.npz")


def test_frames_symbol_exported_and_declared():
    import __graft_entry__ as G
    G.build()
    import instantsplat_b200 as I
    L = I.lib()
    hdr = open(os.path.join(ROOT, "include", "gsb200.h")).read()
    declared = set(re.findall(r"GSB_API [^;(]*?\b(gsb_\w+)\(", hdr))
    assert "gsb_frames_u8_batch" in declared and "gsb_frames_u8_batch" in I._lib.EXPORTS
    assert hasattr(L, "gsb_frames_u8_batch")
    # refused before any launch: no view, no pixel, no pointer
    assert L.gsb_frames_u8_batch(0, 4, 4, 16, 16, None) != 0
    assert L.gsb_frames_u8_batch(1, 0, 4, 16, 16, None) != 0
    assert L.gsb_frames_u8_batch(1, 4, 4, None, 16, None) != 0


@pytest.mark.parametrize("n", [2, 3, 5, 12])
def test_trajectory_matches_reference(n):
    z = np.load(GOLD)
    keys, want = z[f"traj{n}_keys"], z[f"traj{n}_w2c"]
    assert keys.dtype == np.float32 and keys.shape == (n, 4, 4)
    got = F.interpolated_w2c(keys, n)
    assert got.dtype == np.float64 and got.shape == ((n - 1) * int(300 / n) + 1, 4, 4) == want.shape
    assert got.shape[0] == {2: 151, 3: 201, 5: 241, 12: 276}[n]
    assert np.array_equal(got, want)
    assert np.array_equal(got[-1, :3], keys[-1, :3].astype(np.float64))     # the last key pose, appended as is


def test_trajectory_near_180_degrees():
    z = np.load(GOLD)
    assert np.array_equal(F.interpolated_w2c(z["flip_keys"], 2), z["flip_w2c"])


@pytest.mark.parametrize("case", ["traj2", "traj3", "traj5", "traj12", "flip", "quad"])
def test_poses_match_reference(case):
    z = np.load(GOLD)
    got = F.poses_from_w2c(z[f"{case}_w2c"])
    assert got.dtype == torch.float32 and got.shape == (z[f"{case}_w2c"].shape[0], 7)
    assert torch.equal(got, torch.from_numpy(z[f"{case}_pose"]))


def test_golden_reaches_every_candidate():
    """The quad set takes each of rotation2quad's four candidates, and the near-180-degree path two of them."""
    z = np.load(GOLD)
    assert set(z["quad_pick"].tolist()) == {0, 1, 2, 3}
    assert len(set(z["flip_pick"].tolist())) >= 2
    # the 7-vectors are not normalised, and a rotation and its negated quaternion are not canonicalised
    q = torch.from_numpy(z["quad_pose"][:, :4])
    assert (q[:, 0] < 0).any() and not torch.allclose(q.norm(dim=1), torch.ones(len(q)), atol=0, rtol=0)


def test_rotation2quad_is_not_the_trace_method():
    """At 180 degrees about x the trace method divides by ~0; rotation2quad takes the x candidate."""
    m = torch.tensor([[[1.0, 0, 0], [0, -1.0, 0], [0, 0, -1.0]]])
    q = F.rotation2quad(m)
    assert torch.equal(q, torch.tensor([[0.0, 1.0, 0.0, 0.0]]))


def _save_image_bytes(x: torch.Tensor, path: str) -> bytes:
    import torchvision
    torchvision.utils.save_image(x, path)
    with open(path, "rb") as f:
        return f.read()


def test_write_pngs_is_save_image(tmp_path):
    g = torch.Generator().manual_seed(5)
    imgs = torch.rand(3, 3, 37, 53, generator=g) * 1.4 - 0.2
    u8 = imgs.mul(255).add_(0.5).clamp_(0, 255).permute(0, 2, 3, 1).to(torch.uint8).numpy()
    n = F.write_pngs([(0, u8[:2]), (2, u8[2:])], str(tmp_path / "renders"), workers=2)
    assert n == 3 and sorted(os.listdir(tmp_path / "renders")) == ["00000.png", "00001.png", "00002.png"]
    for i in range(3):
        want = _save_image_bytes(imgs[i], str(tmp_path / f"ref{i}.png"))
        with open(tmp_path / "renders" / f"{i:05d}.png", "rb") as f:
            assert f.read() == want, i


def test_refusals(tmp_path):
    keys = np.stack([np.eye(4, dtype=np.float32)] * 3)
    with pytest.raises(ValueError, match="at least 2"):
        F.interpolated_w2c(keys, 1)
    with pytest.raises(ValueError, match="key poses"):
        F.interpolated_w2c(keys, 4)
    with pytest.raises(ValueError, match="at most 300"):
        F.interpolated_w2c(np.stack([np.eye(4)] * 301), 301)
    with pytest.raises(SystemExit):
        F.main(["-s", str(tmp_path), "-m", str(tmp_path), "--n_views", "1"])
    # differing intrinsics
    src = tmp_path / "src"
    folder = src / "sparse_2" / "0"
    poses = np.array([[1.0, 0, 0, 0, 0, 0, 0]] * 2)
    write_colmap_text(str(folder), 64, 48, 50.0, 50.0, poses, ["a.png", "b.png"])
    assert F.intrinsics(str(src), 2)[:2] == (64, 48)
    txt = (folder / "cameras.txt").read_text().replace("2 PINHOLE 64 48 50 50", "2 PINHOLE 64 48 51 50")
    (folder / "cameras.txt").write_text(txt)
    with pytest.raises(ValueError, match="intrinsics differ"):
        F.intrinsics(str(src), 2)
    # a missing ply, then a missing npy
    model = tmp_path / "model"
    (model / "point_cloud" / "iteration_7").mkdir(parents=True)
    with pytest.raises(FileNotFoundError, match="point_cloud.ply"):
        F.load(str(src), str(model), 2, -1)
    (model / "point_cloud" / "iteration_7" / "point_cloud.ply").write_bytes(b"ply\n")
    with pytest.raises(FileNotFoundError, match="pose_optimized.npy"):
        F.load(str(src), str(model), 2, 7)
    with pytest.raises(FileNotFoundError, match="point_cloud"):
        F.load(str(src), str(tmp_path / "nothing"), 2, -1)
