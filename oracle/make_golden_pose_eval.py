"""Generate tests/golden/pose_eval.npz from the REFERENCE's own pose-evaluation functions, run on CPU:
`scene.colmap_loader.read_extrinsics_binary`, `utils.sfm_utils.split_train_test`, `read_colmap_gt_pose` and
`align_pose`, `utils.utils_poses.align_traj.align_ate_c2b_use_a2b` and `utils.utils_poses.comp_ate.compute_ATE` /
`compute_rpe`, chained as metrics.py:88-111 chains them (torch tensors in, the same casts).

utils/sfm_utils.py imports cv2, roma, open3d and dust3r at module level for functions not used here; they are
replaced by empty modules in sys.modules (as is matplotlib, for the scene package's plots).

Cases:
  * split<N>_<n>: split_train_test on lists of N = 24 and 30 items at n_views = 3, 6, 12 (indices of the train and
    test items);
  * traj<n> for n = 3, 6, 12: a ground-truth trajectory (fp64, the layout read_colmap_gt_pose returns) and an
    estimate (fp32, as pose_optimized.npy) that is the truth under a similarity transform plus noise;
  * scale: an estimate 1e-3 times the truth's size; reflect: an estimate whose positions are mirrored, so the
    Umeyama fit flips its last singular direction (`reflect_flipped` records that it did);
  * bin: an images.bin written by instantsplat_b200.scene_io.write_colmap_images_bin (names out of order, 2D points
    on some images), its bytes, what read_extrinsics_binary reads from it and read_colmap_gt_pose's poses.

    python oracle/make_golden_pose_eval.py <path to the InstantSplat checkout>
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

for name in ("matplotlib", "matplotlib.pyplot", "cv2", "roma", "open3d", "dust3r", "dust3r.utils",
             "dust3r.utils.image", "dust3r.utils.device"):
    sys.modules[name] = types.ModuleType(name)
sys.modules["matplotlib"].pyplot = sys.modules["matplotlib.pyplot"]
sys.modules["dust3r.utils.image"]._resize_pil_image = None
sys.modules["dust3r.utils.device"].to_numpy = None

import numpy as np  # noqa: E402
import torch  # noqa: E402
import scene  # noqa: E402,F401  (first: utils.camera_utils and the scene package import each other)
from scene.colmap_loader import read_extrinsics_binary  # noqa: E402
from utils.sfm_utils import align_pose, read_colmap_gt_pose, split_train_test  # noqa: E402
from utils.utils_poses.align_traj import align_ate_c2b_use_a2b  # noqa: E402
from utils.utils_poses.comp_ate import compute_ATE, compute_rpe  # noqa: E402

from instantsplat_b200.scene_io import write_colmap_images_bin  # noqa: E402


def rot(g) -> np.ndarray:
    q = g.standard_normal(4)
    q /= np.linalg.norm(q)
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def trajectory(g, n: int, scale: float, mirror: bool):
    """(gt [n, 4, 4] fp64, est [n, 4, 4] fp32): est = a similarity transform of gt plus noise, mirrored in x."""
    gt = np.stack([np.eye(4)] * n)
    for i in range(n):
        gt[i, :3, :3] = rot(g)
        gt[i, :3, 3] = [np.cos(0.5 * i), np.sin(0.5 * i), 0.1 * i] + 0.05 * g.standard_normal(3)
    Rs, ts = rot(g), g.standard_normal(3)
    est = np.stack([np.eye(4)] * n)
    for i in range(n):
        est[i, :3, :3] = Rs @ gt[i, :3, :3]
        est[i, :3, 3] = scale * (Rs @ gt[i, :3, 3]) + ts + 0.02 * scale * g.standard_normal(3)
        if mirror:
            est[i, 0, 3] = -est[i, 0, 3]
    return gt, est.astype(np.float32)


def metrics_pose_part(pose_optimized: np.ndarray, gt_train_pose):
    """metrics.py's pose evaluation on the reference's functions: the aligned translations, the aligned estimate and
    the raw (rpe_trans, rpe_rot, ate)."""
    est = torch.from_numpy(pose_optimized.copy())
    gt = torch.from_numpy(np.array(gt_train_pose))
    t_gt, t_est, _ = align_pose(gt[:, :3, -1].numpy(), est[:, :3, -1].numpy())
    gt[:, :3, -1] = torch.from_numpy(t_gt)
    est[:, :3, -1] = torch.from_numpy(t_est)
    aligned = align_ate_c2b_use_a2b(est, gt)
    ate = compute_ATE(gt.cpu().numpy(), aligned.cpu().numpy())
    rpe_t, rpe_r = compute_rpe(gt.cpu().numpy(), aligned.cpu().numpy())
    return t_gt, t_est, aligned.numpy(), np.array([rpe_t, rpe_r, ate], np.float64)


def flipped(est: np.ndarray, gt: np.ndarray) -> bool:
    """Whether the Umeyama fit of the aligned positions needs its reflection fix (det U det V < 0)."""
    t_gt, t_est, _ = align_pose(gt[:, :3, 3], est[:, :3, 3])
    a, b = t_est.astype(np.float32), t_gt.astype(np.float32)
    C = (b - b.mean(0)).T @ (a - a.mean(0))
    U, _, Vt = np.linalg.svd(C)
    return bool(np.linalg.det(U) * np.linalg.det(Vt.T) < 0)


def main():
    data = {}
    for N in (24, 30):
        for n in (3, 6, 12):
            train, test = split_train_test(list(range(N)), llffhold=8, n_views=n, verbose=False)
            data[f"split{N}_{n}_train"] = np.array(train, np.int64)
            data[f"split{N}_{n}_test"] = np.array(test, np.int64)

    g = np.random.default_rng(20261016)
    cases = {f"traj{n}": (n, 0.37, False) for n in (3, 6, 12)}
    cases.update(scale=(6, 1e-3, False), reflect=(6, 0.8, True))
    for name, (n, scale, mirror) in cases.items():
        gt, est = trajectory(g, n, scale, mirror)
        t_gt, t_est, aligned, errs = metrics_pose_part(est, list(gt))
        data.update({f"{name}_gt": gt, f"{name}_est": est, f"{name}_t_gt": t_gt, f"{name}_t_est": t_est,
                     f"{name}_aligned": aligned, f"{name}_errors": errs})
        assert aligned.dtype == np.float32 and aligned.shape == (n, 4, 4)
    data["reflect_flipped"] = np.array(flipped(data["reflect_est"], data["reflect_gt"]))
    assert data["reflect_flipped"], "the mirrored case should need Umeyama's reflection fix"

    names = ["c.png", "a.png", "e.png", "b.png", "d.png"]
    qt = np.concatenate([g.standard_normal((5, 4)), g.standard_normal((5, 3))], axis=1)
    qt[:, :4] /= np.linalg.norm(qt[:, :4], axis=1, keepdims=True)
    pts = [np.zeros((0, 3)), np.array([[1.5, 2.25, 7], [3.0, -1.0, -1]]), np.zeros((0, 3)),
           np.array([[0.125, 9.5, 123456789012]]), np.zeros((0, 3))]
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "sparse", "0", "images.bin")
        write_colmap_images_bin(path, qt, names, image_ids=[7, 3, 9, 1, 4], camera_ids=[1, 1, 2, 2, 1], points2d=pts)
        with open(path, "rb") as f:
            data["bin_bytes"] = np.frombuffer(f.read(), np.uint8).copy()
        recs = read_extrinsics_binary(path)
        gt_pose = read_colmap_gt_pose(tmp)
    ids = list(recs)
    data.update(bin_ids=np.array(ids), bin_qvec=np.stack([recs[i].qvec for i in ids]),
                bin_tvec=np.stack([recs[i].tvec for i in ids]), bin_camera_ids=np.array([recs[i].camera_id for i in ids]),
                bin_names=np.array([recs[i].name for i in ids]),
                bin_n_points=np.array([len(recs[i].point3D_ids) for i in ids]),
                bin_xys=np.concatenate([recs[i].xys.reshape(-1, 2) for i in ids]),
                bin_point_ids=np.concatenate([np.asarray(recs[i].point3D_ids, np.int64).reshape(-1) for i in ids]),
                bin_gt_pose=gt_pose)
    np.savez(os.path.join(ROOT, "tests", "golden", "pose_eval.npz"), **data)
    print({k: v.shape for k, v in data.items()})


if __name__ == "__main__":
    main()
