"""Adaptive density control of the reference (scene/gaussian_model.py:420-474, train.py:195-206) as one row plan that
both the mirror `GaussianModel` and `JointTrainer` apply.

`densify_plan` runs the selection and new-row arithmetic of densify_and_clone, densify_and_split and the prune of
densify_and_prune with the reference's torch ops, in the reference's order, and returns where every row of the result
comes from.  Applying it is one gather per tensor, so the trainer rebuilds its flat buffers once per densify event
and lands on the same rows as the mirror, bit for bit.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import torch


@dataclass
class DensifyPlan:
    """Rows after a densify event.  `src[j]` is the old row that final row j copies; rows with `new[j]` were added by
    clone or split and start with zero Adam moments; the split copies at `split` take `split_xyz` / `split_scaling`
    (raw, log-space) instead of the copied values.  `keep` is the final prune over the rows before it (`src2`), which
    `new2` / `split2` describe like `new` / `split`.  `clone` / `split_sel` are the reference's selected_pts_mask of
    clone (over the P old rows) and of split (over the rows after clone).  `reset_stats`: the densification statistics restart at zero (densification_postfix ran)."""
    src: torch.Tensor
    new: torch.Tensor
    split: torch.Tensor
    split_xyz: torch.Tensor
    split_scaling: torch.Tensor
    keep: torch.Tensor
    src2: torch.Tensor
    new2: torch.Tensor
    split2: torch.Tensor
    clone: Optional[torch.Tensor]
    split_sel: Optional[torch.Tensor]
    reset_stats: bool

    @property
    def P(self) -> int:
        return int(self.src.shape[0])

    def gather(self, t: torch.Tensor, computed: Optional[torch.Tensor] = None, prune: bool = True) -> torch.Tensor:
        """Rows of `t` (first dimension: the old rows) in the new order; `computed` replaces the split copies.
        prune=False: the rows before the final prune."""
        out = t[self.src if prune else self.src2]
        if computed is not None:
            out[self.split if prune else self.split2] = computed[self.keep[self.split2]] if prune else computed
        return out

    def moments(self, m: torch.Tensor) -> torch.Tensor:
        """An Adam moment in the new order; new rows start at zero (cat_tensors_to_optimizer)."""
        out = m[self.src]
        out[self.new] = 0
        return out


def _rotation_matrices(rot: torch.Tensor) -> torch.Tensor:
    q = torch.nn.functional.normalize(rot)
    r, x, y, z = q.unbind(-1)
    return torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y), 2 * (x * y + r * z),
                        1 - 2 * (x * x + z * z), 2 * (y * z - r * x), 2 * (x * z - r * y), 2 * (y * z + r * x),
                        1 - 2 * (x * x + y * y)], -1).reshape(-1, 3, 3)


@torch.no_grad()
def densify_plan(xyz, scaling, rotation, opacity, grad_accum, denom, max_radii2D, max_grad, min_opacity, extent,
                 max_screen_size, percent_dense, clone_and_split=False, generator=None, N=2) -> DensifyPlan:
    """densify_and_prune (gaussian_model.py:455-474) on raw parameters: xyz [P,3], scaling [P,3] (log), rotation [P,4]
    (unnormalised), opacity [P,1] (logit), grad_accum / denom [P,1], max_radii2D [P].

    clone_and_split=False is InstantSplat's body (the prune alone); True runs densify_and_clone and densify_and_split
    (N copies, samples from torch.normal(..., generator=generator)) first, whose densification_postfix zeroes the
    statistics, so the size test of the prune then sees zeros."""
    dev = xyz.device
    P = xyz.shape[0]
    src = torch.arange(P, device=dev)
    scales = torch.exp(scaling)
    clone = split_sel = None
    split_xyz = torch.empty(0, 3, device=dev)
    split_scaling = torch.empty(0, 3, device=dev)
    new = torch.zeros(P, dtype=torch.bool, device=dev)
    split2 = torch.empty(0, dtype=torch.long, device=dev)
    radii = max_radii2D
    if clone_and_split:
        grads = grad_accum / denom
        grads[grads.isnan()] = 0.0
        # densify_and_clone: copies of the selected rows are appended
        clone = (torch.norm(grads, dim=-1) >= max_grad) & (torch.max(scales, dim=1).values <= percent_dense * extent)
        src = torch.cat((src, src[clone]))
        new = torch.cat((new, torch.ones(int(clone.sum()), dtype=torch.bool, device=dev)))
        # densify_and_split over the rows after clone (the clones' padded gradient is 0)
        n1 = src.shape[0]
        padded = torch.zeros(n1, device=dev)
        padded[:grads.shape[0]] = grads.squeeze()
        split_sel = (padded >= max_grad) & (torch.max(scales[src], dim=1).values > percent_dense * extent)
        stds = scales[src][split_sel].repeat(N, 1)
        samples = torch.normal(mean=torch.zeros_like(stds), std=stds, generator=generator)
        R = _rotation_matrices(rotation[src][split_sel]).repeat(N, 1, 1)
        split_xyz = torch.bmm(R, samples.unsqueeze(-1)).squeeze(-1) + xyz[src][split_sel].repeat(N, 1)
        split_scaling = torch.log(scales[src][split_sel].repeat(N, 1) / (0.8 * N))
        # postfix appends the split copies, then prune_points removes their sources
        n_split = split_xyz.shape[0]
        src = torch.cat((src[~split_sel], src[split_sel].repeat(N)))
        new = torch.cat((new[~split_sel], torch.ones(n_split, dtype=torch.bool, device=dev)))
        split2 = torch.arange(src.shape[0] - n_split, src.shape[0], device=dev)
        radii = torch.zeros(src.shape[0], device=dev)
    # the prune of densify_and_prune over the rows as they are now
    scaling2 = scaling[src]
    scaling2[split2] = split_scaling
    prune = (torch.sigmoid(opacity[src]) < min_opacity).squeeze(-1)
    if max_screen_size:
        prune = prune | (radii > max_screen_size) | (torch.exp(scaling2).max(dim=1).values > 0.1 * extent)
    keep = ~prune
    pos = torch.cumsum(keep, 0) - 1
    return DensifyPlan(src=src[keep], new=new[keep], split=pos[split2][keep[split2]], split_xyz=split_xyz,
                       split_scaling=split_scaling, keep=keep, src2=src, new2=new, split2=split2, clone=clone,
                       split_sel=split_sel, reset_stats=bool(clone_and_split))


def cameras_extent(poses7: torch.Tensor) -> float:
    """Scene extent of getNerfppNorm (scene/dataset_readers.py:50-71) from the pose table (qw,qx,qy,qz,tx,ty,tz) of
    world-to-camera transforms: camera centres C = -R^T t, radius 1.1 * max |C - mean C| (fp64)."""
    p = poses7.detach().double().cpu().reshape(-1, 7)
    q = torch.nn.functional.normalize(p[:, :4], dim=1)
    r, x, y, z = q.unbind(-1)
    R = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y), 2 * (x * y + r * z),
                     1 - 2 * (x * x + z * z), 2 * (y * z - r * x), 2 * (x * z - r * y), 2 * (y * z + r * x),
                     1 - 2 * (x * x + y * y)], -1).reshape(-1, 3, 3)
    C = -(R.transpose(1, 2) @ p[:, 4:, None]).squeeze(-1)
    return float(1.1 * (C - C.mean(0, keepdim=True)).norm(dim=1).max())
