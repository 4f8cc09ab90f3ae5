"""The free-view fly-through on the GPU (-m gpu, DESIGN.md section 4.12): gsb_frames_u8_batch against save_image's
quantisation exactly, frames_u8 against PoseTracker.render and itself at every batch size, the 8-bit frames against
the drop-in render(), and the command line end to end on a trained synthetic model."""
import math
import os

import numpy as np
import pytest
import torch

import instantsplat_b200 as I
from instantsplat_b200 import freeview as F
from instantsplat_b200.camera import SimpleCamera
from instantsplat_b200.frame import mip_filter3d
from instantsplat_b200.scene_io import write_synthetic_source
from instantsplat_b200.scenes import surface_scene
from instantsplat_b200.tracking import PoseTracker

pytestmark = pytest.mark.gpu
DEV = "cuda"
GOLD = os.path.dirname(os.path.abspath(__file__))


def save_image_u8(x: torch.Tensor) -> torch.Tensor:
    """torchvision.utils.save_image's array for each image of x [V, 3, H, W], on the CPU: [V, H, W, 3] uint8."""
    return x.cpu().mul(255).add_(0.5).clamp_(0, 255).permute(0, 2, 3, 1).to(torch.uint8)


def _ties() -> torch.Tensor:
    """Every fp32 value whose x * 255 is exactly k + 0.5, with its neighbours (tests/golden/metrics.npz)."""
    return torch.from_numpy(np.load(os.path.join(GOLD, "golden", "metrics.npz"))["ties"])


@pytest.mark.parametrize("V", [1, 5])
@pytest.mark.parametrize("HW", [(37, 53), (1080, 1920)])
def test_kernel_is_save_image(V, HW):
    H, W = HW
    g = torch.Generator().manual_seed(V * 7 + H)
    x = torch.rand(V, 3, H, W, generator=g) * 1.6 - 0.3           # values below 0 and above 1
    ties = _ties()
    flat = x.view(-1)
    sel = torch.randint(flat.numel(), (flat.numel() // 3,), generator=g)
    flat[sel] = ties[torch.randint(len(ties), (len(sel),), generator=g)]
    flat[:len(ties)] = ties                                        # every tie value at least once
    flat[-6:] = torch.tensor([-1e30, 1e30, -0.0, 0.0, 1.0, float("inf")])
    got = F.quantise(x.to(DEV))
    assert got.shape == (V, H, W, 3) and got.dtype == torch.uint8
    assert torch.equal(got.cpu(), save_image_u8(x))
    # a view on its own gives the same bytes
    assert torch.equal(F.quantise(x[V - 1:].to(DEV)).cpu(), save_image_u8(x[V - 1:]))


def _scene(deg=3):
    return surface_scene(6000, 3, 96, 64, seed=23, sh_degree=deg)


def _tracker(sc, deg, mip=False, white=False):
    p = sc.params
    kw = {}
    if mip:
        kw = dict(kernel_size=0.1, filter_3D=mip_filter3d(p["xyz"].to(DEV), sc.poses.to(DEV), sc.width, sc.height,
                                                          math.tan(sc.fovx / 2), math.tan(sc.fovy / 2)))
    return PoseTracker(p["xyz"], p["rotation"], p["scaling"], p["opacity"], p["f_dc"], p["f_rest"], sc.width, sc.height,
                       sc.fovx, sc.fovy, bg=torch.ones(3) if white else None, sh_degree=deg, device=DEV, **kw)


def _path(sc):
    from instantsplat_b200.scene_io import pose7_to_matrix
    keys = np.stack([pose7_to_matrix(p) for p in sc.poses.numpy()]).astype(np.float32)
    return F.poses_from_w2c(F.interpolated_w2c(keys, sc.n_views))


def _all(chunks):
    firsts, arrs = zip(*list(chunks))
    out = np.concatenate(arrs)
    assert list(firsts) == list(np.cumsum([0] + [a.shape[0] for a in arrs[:-1]]))
    return out


@pytest.mark.parametrize("deg,mip,white", [(1, False, False), (3, False, False), (3, True, False), (3, False, True)])
def test_frames_u8_matches_render_at_every_batch(deg, mip, white):
    sc = _scene()
    tk = _tracker(sc, deg, mip, white)
    poses = _path(sc)[::9]                                         # 23 poses along the path: the chunks of 3 are ragged
    assert poses.shape[0] == 23
    ref = _all(F.frames_u8(tk, poses))
    assert ref.shape == (23, sc.height, sc.width, 3) and ref.dtype == np.uint8
    for b in (1, 3, 23, 64):
        assert np.array_equal(_all(F.frames_u8(tk, poses, max_batch=b)), ref), b
    for i in range(23):
        want = save_image_u8(tk.render(poses[i].to(DEV))[None])[0].numpy()
        assert np.array_equal(ref[i], want), i
    if white:                                                      # the background shows through somewhere
        assert not np.array_equal(ref, _all(F.frames_u8(_tracker(sc, deg, mip, False), poses)))
    assert len(list(F.frames_u8(tk, poses[:0]))) == 0


def test_frames_u8_against_dropin_render():
    """The 8-bit frames against save_image of the drop-in render() at the same 7-vectors.  The two forwards agree to
    the parity tolerance, so a pixel may sit on the other side of a level boundary: at most one level apart."""
    sc = _scene()
    tk = _tracker(sc, 3)
    poses = _path(sc)[::20]
    ours = _all(F.frames_u8(tk, poses, max_batch=4)).astype(np.int16)
    model = I.GaussianModel.from_scene(sc, DEV)
    cam = SimpleCamera(sc.width, sc.height, sc.fovx, sc.fovy, device=DEV)
    pipe, bg = I.PipelineDefaults(), torch.zeros(3, device=DEV)
    with torch.no_grad():
        ref = torch.stack([I.render(cam, model, pipe, bg, camera_pose=p.to(DEV))["render"] for p in poses])
    d = np.abs(ours - save_image_u8(ref).numpy().astype(np.int16))
    n_diff = int((d > 0).sum())
    print(f"frames_u8 vs drop-in render(): {n_diff} of {d.size} values differ, max {int(d.max())} level(s)")
    assert int(d.max()) <= 1 and n_diff <= 1e-3 * d.size


def _model_dir(tmp_path, n_views, white=False):
    """A synthetic source and a briefly trained model saved in render.py's layout."""
    sc = surface_scene(6000, n_views, 96, 64, seed=31, sh_degree=3)
    if white:
        sc.bg = torch.ones(3)
    src, model = tmp_path / "src", tmp_path / "model"
    write_synthetic_source(str(src), sc)
    gts = torch.rand(n_views, 3, sc.height, sc.width, generator=torch.Generator().manual_seed(2))
    tr = I.JointTrainer(sc, DEV, gt_images=gts)
    for k in range(6):
        tr.step(k % n_views)
    it = 6
    tr.save_ply(str(model / "point_cloud" / f"iteration_{it}" / "point_cloud.ply"))
    tr.save_poses(str(model / "pose" / f"ours_{it}" / "pose_optimized.npy"))
    (model / "point_cloud" / "iteration_2").mkdir(parents=True)    # an older save point: -1 takes the largest
    return src, model, it


def _read_pngs(folder, n):
    from PIL import Image
    return np.stack([np.asarray(Image.open(os.path.join(folder, f"{i:05d}.png"))) for i in range(n)])


@pytest.mark.parametrize("white", [False, True])
def test_cli_end_to_end(tmp_path, white):
    n = 3
    src, model, it = _model_dir(tmp_path, n, white)
    argv = ["-s", str(src), "-m", str(model), "--n_views", str(n), "--iterations", "-1", "--max_batch", "16"]
    assert F.main(argv + (["--white_background"] if white else [])) == 0
    folder = model / "interp" / f"ours_{it}" / "renders"
    N = int(300 / n) * (n - 1) + 1
    assert sorted(os.listdir(folder)) == [f"{i:05d}.png" for i in range(N)]
    keys = np.load(model / "pose" / f"ours_{it}" / "pose_optimized.npy")
    path = np.load(model / "pose" / f"ours_{it}" / "pose_interpolated.npy")
    assert np.array_equal(path, F.interpolated_w2c(keys, n))
    tk, keys2, it2 = F.load(str(src), str(model), n, it, white)
    assert it2 == it and np.array_equal(keys2, keys)
    want = _all(F.frames_u8(tk, F.poses_from_w2c(path)))
    assert np.array_equal(_read_pngs(folder, N), want)


def test_training_view_renders(tmp_path):
    """render.py's render_set("train"): the training views at their optimised poses, from pose_optimized.npy."""
    n = 3
    src, model, it = _model_dir(tmp_path, n)
    tk, keys, _ = F.load(str(src), str(model), n, it)
    poses = F.poses_from_w2c(keys)
    out = tmp_path / "train" / "renders"
    assert F.write_pngs(F.frames_u8(tk, poses), str(out), workers=2) == n
    assert np.array_equal(_read_pngs(out, n), save_image_u8(tk.render_batch(poses)).numpy())
