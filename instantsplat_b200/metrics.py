"""The numbers InstantSplat reports: stage 5 of scripts/run_eval.sh, metrics.py's evaluate (metrics.py:35-125), per
model directory and per test/<method>.

  * Images: every file of test/<method>/renders paired with the gt file of the same name (the reference's os.listdir
    pairing, in sorted order here), decoded by PIL to k / 255 (to_tensor) and measured in one batched
    evaluation.image_metrics call (mode "png8", the identity on k / 255): PSNR of the whole image's MSE and the
    loss's SSIM, per view in fp64.  Written as metrics.txt lines in the reference's format, results.json (the means)
    and per_view.json (per file name), with the reference's keys and nesting.  LPIPS (VGG) needs pretrained weights:
    with --lpips_weights DIR (a directory holding torch hub's vgg16-397923af.pth and vgg.pth, such as
    $TORCH_HOME/hub/checkpoints) it is computed on the GPU by lpips.LpipsVGG, built once per run, and written where
    the reference writes it; without it its key is left out and the run says so.
  * Poses: source/sparse/0/images.bin (read_colmap_gt_pose), thinned to the training views by split_train_test,
    against pose/<method>/pose_optimized.npy: align_pose (scale and centre the translations, orthogonal Procrustes),
    then align_ate_c2b_use_a2b (a sim3 Umeyama fit in fp32), then compute_ATE and compute_rpe.  RPE_t is reported x
    100 and RPE_r in degrees, in pose/<method>/pose_eval.txt and results.json.  Each function below restates the
    reference's numpy / scipy calls in their order and dtypes.  The pose plots are not drawn.

A model directory without test/ is reported and skipped; a method without sparse/0/images.bin or pose_optimized.npy
keeps its image numbers and skips the pose part, with a message.

    python -m instantsplat_b200.metrics -s SOURCE -m MODEL [MODEL ...] --n_views N [--lpips_weights DIR]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
from typing import Dict, List, Tuple

import numpy as np
import torch

from . import lpips as LP
from .scene_io import read_colmap_gt_pose, split_train_test


# ---- pose errors (utils/sfm_utils.py, utils/utils_poses) -----------------------------------------------------
def align_pose(pose1, pose2):
    """sfm_utils.align_pose on two [N, 3] point sets: both centred and scaled to unit Frobenius norm, the second
    multiplied by the orthogonal-Procrustes scale.  Returns (points1, points2, R) in fp64; R is not applied."""
    from scipy.linalg import orthogonal_procrustes
    m1 = np.array(pose1, dtype=np.double, copy=True)
    m2 = np.array(pose2, dtype=np.double, copy=True)
    if m1.ndim != 2 or m2.ndim != 2:
        raise ValueError("align_pose: expected two-dimensional point sets")
    if m1.shape != m2.shape:
        raise ValueError(f"align_pose: point sets of shapes {m1.shape} and {m2.shape} differ")
    if m1.size == 0:
        raise ValueError("align_pose: empty point sets")
    m1 -= np.mean(m1, 0)
    m2 -= np.mean(m2, 0)
    n1, n2 = np.linalg.norm(m1), np.linalg.norm(m2)
    if n1 == 0 or n2 == 0:
        raise ValueError("align_pose: a point set has fewer than 2 distinct points")
    m1 /= n1
    m2 /= n2
    R, s = orthogonal_procrustes(m1, m2)
    return m1, m2 * s, R


def umeyama(model: np.ndarray, data: np.ndarray):
    """ATE/align_trajectory.align_umeyama with a free scale: (s, R, t) with model ~ s R data + t, the last singular
    direction flipped when the fit would be a reflection."""
    mu_m, mu_d = model.mean(0), data.mean(0)
    mz, dz = model - mu_m, data - mu_d
    n = np.shape(model)[0]
    C = 1.0 / n * np.dot(mz.transpose(), dz)
    sigma2 = 1.0 / n * np.multiply(dz, dz).sum()
    U, D, Vt = np.linalg.svd(C)
    D = np.diag(D)
    V = np.transpose(Vt)
    S = np.eye(3)
    if np.linalg.det(U) * np.linalg.det(V) < 0:
        S[2, 2] = -1
    R = np.dot(U, np.dot(S, np.transpose(V)))
    s = 1.0 / sigma2 * np.trace(np.dot(D, S))
    t = mu_m - s * np.dot(R, mu_d)
    return s, R, t


def align_sim3(traj_a, traj_b) -> np.ndarray:
    """align_traj.align_ate_c2b_use_a2b(a, b, method='sim3') with c = a: both trajectories [N, 3|4, 4] in fp32, the
    sim3 that maps a's positions onto b's (alignTrajectory -> Umeyama over all frames), applied to a.  Returns
    [N, 4, 4] fp32.  (alignTrajectory also converts the rotations to quaternions, which the sim3 fit never reads.)"""
    a = np.asarray(traj_a).astype(np.float32)
    b = np.asarray(traj_b).astype(np.float32)
    if a.shape[0] < 2:
        raise ValueError("align_sim3: a sim3 alignment needs at least 2 poses")
    # contiguous copies of the positions, as alignSIM3's index selection makes them (the sums then run in one order)
    s, R, t = umeyama(np.ascontiguousarray(b[:, :3, 3]), np.ascontiguousarray(a[:, :3, 3]))
    R = R[None, :, :].astype(np.float32)
    t = t[None, :, None].astype(np.float32)
    s = float(s)
    out = np.concatenate([R @ a[:, :3, :3], s * (R @ a[:, :3, 3:4]) + t], axis=2)
    out = np.concatenate([out, np.zeros_like(out[:, 0:1])], axis=1)
    out[:, 3, 3] = 1.0
    return out


def compute_ate(gt, pred) -> float:
    """comp_ate.compute_ATE: the RMS of the position errors |t_gt - t_pred|."""
    errors = [np.sqrt(np.sum((gt[i][:3, 3] - pred[i][:3, 3]) ** 2)) for i in range(len(pred))]
    return np.sqrt(np.mean(np.asarray(errors) ** 2))


def compute_rpe(gt, pred) -> Tuple[float, float]:
    """comp_ate.compute_rpe: mean translation and rotation (radians) error of consecutive relative poses."""
    trans, rot = [], []
    for i in range(len(gt) - 1):
        gt_rel = np.linalg.inv(gt[i]) @ gt[i + 1]
        pred_rel = np.linalg.inv(pred[i]) @ pred[i + 1]
        e = np.linalg.inv(gt_rel) @ pred_rel
        trans.append(np.sqrt(e[0, 3] ** 2 + e[1, 3] ** 2 + e[2, 3] ** 2))
        d = 0.5 * (e[0, 0] + e[1, 1] + e[2, 2] - 1.0)
        rot.append(np.arccos(max(min(d, 1.0), -1.0)))
    return np.mean(np.asarray(trans)), np.mean(np.asarray(rot))


def pose_errors(pose_optimized, gt_poses) -> Dict[str, float]:
    """metrics.py:88-111 on pose_optimized [n, 4, 4] (any float dtype, kept) and the training views' ground truth
    [n, 4, 4]: {"RPE_t": x 100, "RPE_r": degrees, "ATE"}."""
    est = np.array(pose_optimized, copy=True)
    gt = np.array(gt_poses, dtype=np.float64, copy=True)
    t_gt, t_est, _ = align_pose(gt[:, :3, -1], est[:, :3, -1])
    gt[:, :3, -1] = t_gt
    est[:, :3, -1] = t_est
    aligned = align_sim3(est, gt)
    ate = compute_ate(gt, aligned)
    rpe_t, rpe_r = compute_rpe(gt, aligned)
    return {"RPE_t": float(rpe_t * 100), "RPE_r": float(rpe_r * 180 / np.pi), "ATE": float(ate)}


def train_gt_poses(source_path: str, n_views: int) -> np.ndarray:
    """read_colmap_gt_pose + split_train_test: the ground-truth poses of the n_views training views."""
    train, _ = split_train_test(list(read_colmap_gt_pose(source_path)), n_views)
    return np.array(train)


# ---- images ----------------------------------------------------------------------------------------------------
def read_pairs(method_dir: str) -> Tuple[np.ndarray, np.ndarray, List[str]]:
    """readImages: (renders, gts) uint8 [V, H, W, 3] and the file names, every file of renders/ with the gt file of
    the same name (sorted by name).  Only the first three channels are kept, as readImages keeps them."""
    from PIL import Image
    rdir, gdir = os.path.join(method_dir, "renders"), os.path.join(method_dir, "gt")
    names = sorted(os.listdir(rdir))
    if not names:
        raise ValueError(f"{rdir} holds no image")
    renders, gts = [], []
    for n in names:
        for folder, out in ((rdir, renders), (gdir, gts)):
            with Image.open(os.path.join(folder, n)) as im:
                a = np.asarray(im)
            if a.ndim != 3 or a.shape[2] < 3 or a.dtype != np.uint8:
                raise ValueError(f"{os.path.join(folder, n)}: expected an 8-bit image with 3 or 4 channels, got "
                                 f"{a.dtype} {a.shape}")
            out.append(a[..., :3])
    shapes = {a.shape for a in renders + gts}
    if len(shapes) != 1:
        raise ValueError(f"{method_dir}: the images differ in size ({sorted(shapes)}); one batched call measures one size")
    return np.stack(renders), np.stack(gts), names


def image_numbers(renders: np.ndarray, gts: np.ndarray, device="cuda") -> Dict[str, torch.Tensor]:
    """PSNR and SSIM per view of uint8 [V, H, W, 3] images, as to_tensor + psnr / ssim see them: fp64 CPU tensors.
    The values k / 255 go in through mode "png8", whose 8-bit round trip leaves them unchanged
    (render_views.gt_round_trip_is_identity), so a file's numbers are those PoseTracker.evaluate_batch(mode="png8")
    gives for the render it holds, bit for bit; mode "clamp", the identity on them too, was measured to differ from
    it in the last bits."""
    from .evaluation import image_metrics
    f = lambda u8: (torch.from_numpy(np.ascontiguousarray(u8)).to(device) / 255.0).permute(0, 3, 1, 2).contiguous()
    m = image_metrics(f(renders), f(gts), mode="png8")
    return {"PSNR": m["psnr"].cpu(), "SSIM": m["ssim"].cpu()}


def lpips_numbers(renders: np.ndarray, gts: np.ndarray, net, device="cuda") -> torch.Tensor:
    """LPIPS per view of uint8 [V, H, W, 3] images read as to_tensor reads them (k / 255), by lpips.LpipsVGG `net`:
    an fp64 CPU tensor [V]."""
    f = lambda u8: (torch.from_numpy(np.ascontiguousarray(u8)).to(device) / 255.0).permute(0, 3, 1, 2).contiguous()
    return net(f(renders), f(gts))[0].cpu()


def evaluate_method(scene_dir: str, method: str, source_path: str, n_views: int, device="cuda", lpips_net=None,
                    pairs=None):
    """One test/<method> of one model directory: writes test/<method>/metrics.txt and (when the pose inputs exist)
    pose/<method>/pose_eval.txt.  Returns (full, per_view) entries for results.json and per_view.json.  LPIPS is
    measured with lpips_net (an lpips.LpipsVGG) when it is given.  pairs: what read_pairs would return for the method,
    held in memory (renders and gts uint8 [V, H, W, 3] in sorted file-name order, the names); None reads the files."""
    method_dir = os.path.join(scene_dir, "test", method)
    renders, gts, names = read_pairs(method_dir) if pairs is None else pairs
    m = image_numbers(renders, gts, device)
    psnr, ssim = m["PSNR"].tolist(), m["SSIM"].tolist()
    lp = lpips_numbers(renders, gts, lpips_net, device) if lpips_net is not None else None
    with open(os.path.join(method_dir, "metrics.txt"), "w") as f:
        for idx, name in enumerate(names):
            tail = "" if lp is None else f", LPIPS: {lp[idx].item():.4f}"
            f.write(f"image name{name}, image idx: {idx}, PSNR: {psnr[idx]:.2f}, SSIM: {ssim[idx]:.4f}{tail}\n")
    full = {"SSIM": float(m["SSIM"].mean()), "PSNR": float(m["PSNR"].mean())}
    per_view = {"SSIM": dict(zip(names, ssim)), "PSNR": dict(zip(names, psnr))}
    if lp is not None:
        full["LPIPS"] = float(lp.mean())
        per_view["LPIPS"] = dict(zip(names, lp.tolist()))
    print(f"  SSIM : {full['SSIM']:>12.7f}")
    print(f"  PSNR : {full['PSNR']:>12.7f}")
    if lp is None:
        print("  LPIPS: not computed (it needs pretrained VGG weights)")
    else:
        print(f"  LPIPS: {full['LPIPS']:>12.7f}")
    pose_dir = os.path.join(scene_dir, "pose", method)
    npy = os.path.join(pose_dir, "pose_optimized.npy")
    try:
        gt_poses = train_gt_poses(source_path, n_views)
    except FileNotFoundError as e:
        print(f"  poses: skipped ({e})")
        return full, per_view
    if not os.path.isfile(npy):
        print(f"  poses: skipped ({npy} not found)")
        return full, per_view
    p = pose_errors(np.load(npy), gt_poses)
    print(f"  RPE_t: {p['RPE_t']:>12.7f}")
    print(f"  RPE_r: {p['RPE_r']:>12.7f}")
    print(f"  ATE  : {p['ATE']:>12.7f}")
    full.update(p)
    with open(os.path.join(pose_dir, "pose_eval.txt"), "w") as f:
        f.write("RPE_t: {:.04f}, RPE_r: {:.04f}, ATE: {:.04f}".format(p["RPE_t"], p["RPE_r"], p["ATE"]))
    return full, per_view


def evaluate(scene_dirs, source_path: str, n_views: int, device="cuda", lpips_net=None, held=None) -> int:
    """metrics.py's evaluate over model directories: <scene>/results.json and <scene>/per_view.json for each.
    Returns the number of model directories that could not be evaluated (each is reported with its reason).
    held: {method: pairs} (evaluate_method's pairs) for methods whose images are in memory; the rest are read."""
    held = held or {}
    failed = 0
    for scene_dir in scene_dirs:
        print("Scene:", scene_dir)
        full, per_view = {}, {}
        try:
            test_dir = os.path.join(scene_dir, "test")
            if not os.path.isdir(test_dir):
                raise FileNotFoundError(f"{test_dir} not found")
            for method in sorted(os.listdir(test_dir)):
                if not os.path.isdir(os.path.join(test_dir, method)):
                    continue
                print("Method:", method)
                full[method], per_view[method] = evaluate_method(scene_dir, method, source_path, n_views, device,
                                                                  lpips_net, held.get(method))
        except (OSError, ValueError) as e:
            print(f"Unable to compute metrics for model {scene_dir}: {e}")
            failed += 1
            continue
        with open(os.path.join(scene_dir, "results.json"), "w") as fp:
            json.dump(full, fp, indent=True)
        with open(os.path.join(scene_dir, "per_view.json"), "w") as fp:
            json.dump(per_view, fp, indent=True)
    return failed


def parser() -> argparse.ArgumentParser:
    """metrics.py's command line as this stage reads it."""
    ap = argparse.ArgumentParser(prog="python -m instantsplat_b200.metrics",
                                 description="metrics.py: PSNR / SSIM (and LPIPS) of the test renders and the pose errors")
    ap.add_argument("-s", "--source_path", required=True)
    ap.add_argument("-m", "--model_paths", required=True, nargs="+")
    ap.add_argument("--n_views", type=int, required=True)
    ap.add_argument("--lpips_weights", metavar="DIR", default=None,
                    help=f"directory holding {LP.VGG_FILE} and {LP.LIN_FILE} (torch hub's checkpoints directory): "
                         "also report LPIPS (VGG)")
    return ap


def main(argv=None) -> int:
    ap = parser()
    a = ap.parse_args(argv)
    net = None
    if a.lpips_weights is not None:
        try:
            net = LP.LpipsVGG.from_dir(a.lpips_weights, "cuda")
        except (OSError, ValueError) as e:
            ap.error(str(e))
    return 1 if evaluate(a.model_paths, a.source_path, a.n_views, lpips_net=net) else 0


if __name__ == "__main__":
    sys.exit(main())
