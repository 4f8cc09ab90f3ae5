"""Generate tests/golden/freeview.npz from the REFERENCE's own free-view functions, run on CPU:
`utils.camera_utils.generate_interpolated_path` (the trajectory of render.py --infer_video),
`utils.graphics_utils.getWorld2View2` (loadCameras, scene/dataset_readers.py:87-103) and
`utils.pose_utils.get_tensor_from_camera` / `rotation2quad` (render.py:86).

render.py itself imports the renderer, imageio and the scene loader, so its ten-line save_interpolate_pose
(render.py:36-56) is restated below around the reference's generate_interpolated_path, call for call.  matplotlib
(camera_utils imports pyplot for its pose plots) is not installed; it is replaced by an empty module in sys.modules.

Cases:
  * traj<n> for n_views = 2, 3, 5, 12: key poses written by scene_io.save_pose_npy (what JointTrainer.save_poses
    calls) from a synthetic scene's pose table, the interpolated path (151, 201, 241, 276 poses) and the 7-vector of
    every pose;
  * flip: a pair whose rotations differ by 179.5 degrees;
  * quad: rotations that make rotation2quad pick each of its four candidates (near identity, and about 180 degrees
    about x, y and z), plus random ones; `quad_pick` records the candidate each one took.

    python oracle/make_golden_freeview.py <path to the InstantSplat checkout>
"""
import os
import sys
import tempfile
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if len(sys.argv) != 2:
    sys.exit(__doc__)
REF = sys.argv[1]
for p in (os.path.join(ROOT, "tests", "cpu_standins"), os.path.join(ROOT, "tests", "stubs"), ROOT):
    sys.path.insert(0, p)
sys.path.append(REF)

_mpl = types.ModuleType("matplotlib")
_mpl.pyplot = types.ModuleType("matplotlib.pyplot")
sys.modules["matplotlib"], sys.modules["matplotlib.pyplot"] = _mpl, _mpl.pyplot

import numpy as np  # noqa: E402
import torch  # noqa: E402
import scene  # noqa: E402,F401  (first: utils.camera_utils and the scene package import each other)
from utils.camera_utils import generate_interpolated_path  # noqa: E402
from utils.graphics_utils import getWorld2View2  # noqa: E402
from utils.pose_utils import get_tensor_from_camera  # noqa: E402

from instantsplat_b200.scene_io import save_pose_npy  # noqa: E402
from instantsplat_b200.scenes import surface_scene  # noqa: E402


def save_interpolate_pose(org_pose: np.ndarray, n_views: int) -> np.ndarray:
    """render.py:36-56 without the file I/O and the plots."""
    n_interp = int(10 * 30 / n_views)
    all_inter_pose = []
    for i in range(n_views - 1):
        all_inter_pose.append(generate_interpolated_path(poses=org_pose[i:i + 2], n_interp=n_interp))
    all_inter_pose = np.concatenate(all_inter_pose, axis=0)
    all_inter_pose = np.concatenate([all_inter_pose, org_pose[-1][:3, :].reshape(1, 3, 4)], axis=0)
    inter_pose_list = []
    for p in all_inter_pose:
        tmp_view = np.eye(4)
        tmp_view[:3, :3] = p[:3, :3]
        tmp_view[:3, 3] = p[:3, 3]
        inter_pose_list.append(tmp_view)
    return np.stack(inter_pose_list, 0)


def pose7(w2c: np.ndarray) -> np.ndarray:
    """loadCameras' world_view_transform (getWorld2View2(R, T) with R = p[:3, :3]^T, T = p[:3, 3], transposed) and
    render_set's get_tensor_from_camera(world_view_transform.transpose(0, 1)), on CPU."""
    out = []
    for p in w2c:
        R, T = np.transpose(p[:3, :3]), p[:3, 3]
        wvt = torch.tensor(getWorld2View2(R, T)).transpose(0, 1)
        out.append(get_tensor_from_camera(wvt.transpose(0, 1)).numpy())
    return np.stack(out).astype(np.float32)


def rot(axis, deg: float) -> np.ndarray:
    a = np.asarray(axis, np.float64)
    a = a / np.linalg.norm(a)
    t = np.radians(deg)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + np.sin(t) * K + (1 - np.cos(t)) * K @ K


def pick(w2c: np.ndarray) -> np.ndarray:
    """Which of rotation2quad's candidates each matrix takes (argmax of the four 1 +- m00 +- m11 +- m22)."""
    out = []
    for p in w2c:
        m = torch.tensor(getWorld2View2(np.transpose(p[:3, :3]), p[:3, 3]))[:3, :3]
        s = torch.stack([1 + m[0, 0] + m[1, 1] + m[2, 2], 1 + m[0, 0] - m[1, 1] - m[2, 2],
                         1 - m[0, 0] + m[1, 1] - m[2, 2], 1 - m[0, 0] - m[1, 1] + m[2, 2]])
        out.append(int(torch.sqrt(torch.clamp(s, min=0)).argmax()))
    return np.array(out, np.int32)


def main():
    data = {}
    for n in (2, 3, 5, 12):
        sc = surface_scene(64 * n, n, 64, 48, seed=100 + n, sh_degree=1)
        with tempfile.TemporaryDirectory() as tmp:
            keys = save_pose_npy(os.path.join(tmp, "pose_optimized.npy"), sc.poses.numpy())
        traj = save_interpolate_pose(keys, n)
        assert traj.shape == ((n - 1) * int(300 / n) + 1, 4, 4), traj.shape
        data[f"traj{n}_keys"], data[f"traj{n}_w2c"], data[f"traj{n}_pose"] = keys, traj, pose7(traj)

    g = np.random.default_rng(20261016)
    flip = np.stack([np.eye(4), np.eye(4)]).astype(np.float32)
    flip[0, :3, :3] = rot([0.1, 1.0, 0.05], 3.0)
    flip[1, :3, :3] = rot([0.1, 1.0, 0.05], 182.5)
    flip[:, :3, 3] = [[0.1, -0.2, 0.3], [-0.4, 0.1, 2.0]]
    traj = save_interpolate_pose(flip, 2)
    data.update(flip_keys=flip, flip_w2c=traj, flip_pose=pose7(traj))

    mats = [rot([1, 0, 0], 0.0), rot([0.3, -0.2, 1.0], 20.0)]
    for axis in ([1, 0, 0], [0, 1, 0], [0, 0, 1]):
        for deg in (170.0, 180.0, 190.0):
            mats.append(rot(np.asarray(axis) + 0.02 * g.standard_normal(3), deg))
    for _ in range(24):
        mats.append(rot(g.standard_normal(3), g.uniform(0.0, 360.0)))
    quad = np.stack([np.eye(4)] * len(mats)).astype(np.float32)
    quad[:, :3, :3] = np.stack(mats)
    quad[:, :3, 3] = g.standard_normal((len(mats), 3))
    data.update(quad_w2c=quad, quad_pose=pose7(quad), quad_pick=pick(quad))
    assert set(data["quad_pick"].tolist()) == {0, 1, 2, 3}, data["quad_pick"]
    data["flip_pick"] = pick(data["flip_w2c"])
    np.savez(os.path.join(ROOT, "tests", "golden", "freeview.npz"), **data)
    print({k: v.shape for k, v in data.items()})
    print("quad picks", np.bincount(data["quad_pick"], minlength=4), "flip picks",
          np.bincount(data["flip_pick"], minlength=4))


if __name__ == "__main__":
    main()
