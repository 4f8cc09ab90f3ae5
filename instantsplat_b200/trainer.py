"""The joint pose + Gaussian optimisation inner loop of train.py:124-211, H100-first.

One `JointTrainer.step(view)` = update_learning_rate -> render (fused pose transform + rasterizer)
-> L1 + DSSIM loss -> backward -> (multi-GPU: NCCL sum of the flat per-Gaussian gradient buffer)
-> per-point Adam, i.e. exactly one iteration of the reference loop, but:

  * all Gaussian parameters, gradients and Adam moments live in FLAT fp32 buffers (one tensor per
    kind, 256-byte aligned segments) so the backward kernels write gradients straight into the
    buffer NCCL reduces, and Adam is one launch over all seven tensors;
  * ~12 kernel launches per iteration instead of the reference's several hundred ATen launches,
    and exactly one host sync (the instance count R that sizes the binning buffers).

Multi-GPU (SURVEY.md section 8e): one process per GPU, a full replica of the cloud per GPU,
training views sharded round-robin (view v -> rank v mod G); per step every rank renders one of
its views, gradients are summed with one all-reduce over NVLink and scaled by 1/G inside the Adam
kernel, so all replicas stay bit-identical.  An "iteration" in the reported iters/s is one VIEW
(one reference iteration); one optimizer step consumes G views.

One GPU, V views per optimizer step (`JointTrainer.step_batch(views)`, DESIGN.md section 4.10): the same semantics as
G = V ranks, computed by one view-batched forward, loss and backward whose per-Gaussian gradients are summed over the
views in view order, and one Adam launch with grad_scale = 1/V.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import numpy as np
import torch
from torch import nn

from . import _lib
from ._lib import GsbGaussians, GsbGrads, check
from .frame import (ST_OVERFLOW, ST_SEQ, ST_WORDS, Frame, IdentityView, capacity, gaussians, mip_filter, mip_filter3d,
                    read_R)
from .densify import cameras_extent, densify_plan
from .frame import densify_stats
from .per_point_adam import launch_adam
from .scenes import Scene

# The six per-Gaussian tensors and their floats per Gaussian at SH degree 3 (15 f_rest rows).  A trainer's own widths
# follow its scene's f_rest (segment_widths, JointTrainer.widths); the names and their order are the same at every degree.
SEGMENTS = (("xyz", 3), ("f_dc", 3), ("f_rest", 45), ("opacity", 1), ("scaling", 3), ("rotation", 4))
ADAM_BETAS, ADAM_EPS = (0.9, 0.999), 1e-15       # training_setup_pp's PerPointAdam (scene/gaussian_model.py:221)


def get_expon_lr_func(lr_init, lr_final, lr_delay_steps=0, lr_delay_mult=1.0, max_steps=1000000):
    """utils/general_utils.py:29-62 (host-side, fp64 numpy, unchanged semantics)."""

    def helper(step):
        if step < 0 or (lr_init == 0.0 and lr_final == 0.0):
            return 0.0
        if lr_delay_steps > 0:
            delay_rate = lr_delay_mult + (1 - lr_delay_mult) * np.sin(
                0.5 * np.pi * np.clip(step / lr_delay_steps, 0, 1))
        else:
            delay_rate = 1.0
        t = np.clip(step / max_steps, 0, 1)
        return delay_rate * np.exp(np.log(lr_init) * (1 - t) + np.log(lr_final) * t)

    return helper


class OptimConfig:
    """arguments/__init__.py:73-94 defaults."""
    iterations = 30_000
    position_lr_init = 0.00016
    position_lr_final = 0.0000016
    position_lr_delay_mult = 0.01
    position_lr_max_steps = 30_000
    feature_lr = 0.0025
    opacity_lr = 0.05
    scaling_lr = 0.005
    rotation_lr = 0.001
    lambda_dssim = 0.2
    pp_optimizer = True
    optim_pose = True
    spatial_lr_scale = 1.0
    sh_increase_interval = 1000      # train.py:146-147: oneupSHdegree() when iteration % 1000 == 0
    max_sh_degree = 3
    # Mip-Splatting (DESIGN.md section 4.7): None = off; else the 2D Mip filter's kernel size (0.1 in Mip-Splatting)
    # together with the 3D smoothing filter, computed at construction and after every change of the Gaussian count, and
    # recomputed from the current poses and xyz each time the iteration count crosses a multiple of `mip_filter3d_interval`, except in the last 100.
    mip_kernel_size = None
    mip_filter3d_interval = 100
    # Adaptive density control (DESIGN.md section 4.8), train.py:195-206 with the block enabled; one GPU only.
    # densify_clone_split=False is InstantSplat's prune-only densify_and_prune, True the vanilla-3DGS clone + split.
    # scene_extent=None: getNerfppNorm's radius of the initial pose table (densify.cameras_extent).
    densify = False
    densify_from_iter = 500
    densify_until_iter = 15_000
    densification_interval = 100
    opacity_reset_interval = 3000
    densify_grad_threshold = 0.0002
    min_opacity = 0.005
    percent_dense = 0.01
    size_threshold = 20
    densify_clone_split = False
    scene_extent = None
    densify_seed = 0                 # seed of the generator the split samples are drawn from
    # step_batch with densify (DESIGN.md section 4.10): the statistics of every view of a batch, and the densify / reset
    # events of the iterations a batch covers fired once at its end.  Off: step_batch refuses densify=True, so that a
    # run configured for train.py's per-iteration schedule does not move its events by switching to step_batch.
    densify_batches = False
    # train.py's random background (DESIGN.md section 4.17), one GPU only: every iteration's forward and backward blend
    # over a fresh colour, torch.rand((3), device="cuda") from a CUDA generator seeded with background_seed (safe_state's
    # torch.manual_seed(0)).  render(), evaluate() and PoseTracker keep the scene's background.
    random_background = False
    background_seed = 0


def lr_schedules(args, spatial_lr_scale):
    """training_setup_pp's xyz and pose learning-rate schedules (scene/gaussian_model.py:223-232).  args: anything with
    the OptimizationParams field names (OptimConfig, optimization_defaults())."""
    xyz = get_expon_lr_func(args.position_lr_init * spatial_lr_scale, args.position_lr_final * spatial_lr_scale,
                            lr_delay_mult=args.position_lr_delay_mult, max_steps=args.position_lr_max_steps)
    pose = get_expon_lr_func(args.rotation_lr * 0.1, args.rotation_lr * 0.001, lr_delay_mult=args.position_lr_delay_mult,
                             max_steps=args.iterations)
    return xyz, pose


def group_lrs(args, spatial_lr_scale, iteration: Optional[int] = None) -> Dict[str, float]:
    """The `lr` of the seven param groups (SEGMENTS order, then "pose"): training_setup_pp's initial values, or, given
    an iteration, those after update_learning_rate(iteration)."""
    lrs = dict(xyz=args.position_lr_init * spatial_lr_scale, f_dc=args.feature_lr * 10,
               f_rest=args.feature_lr / 20.0 * 10, opacity=args.opacity_lr, scaling=args.scaling_lr * 10,
               rotation=args.rotation_lr * 10, pose=args.rotation_lr * 0.1)
    if iteration is not None:
        xyz, pose = lr_schedules(args, spatial_lr_scale)
        lrs.update(xyz=xyz(iteration), pose=pose(iteration))
    return lrs


def adam_step_sizes(cfg, iteration: int, opt_step: int, lag: Dict[str, int]) -> Dict[str, float]:
    """PerPointAdam's step size lr * sqrt(1-b2^t)/(1-b1^t) of the seven groups after update_learning_rate(iteration),
    where t = opt_step - lag[name] is the group's step count (the pose table has no lag).  A group that has taken no
    step yet gets the size of t = 1; it is not stepped with it."""
    b1, b2 = ADAM_BETAS
    out = {}
    for name, lr in group_lrs(cfg, cfg.spatial_lr_scale, iteration).items():
        t = max(1, opt_step - lag.get(name, 0))
        out[name] = lr * ((1 - b2 ** t) ** 0.5 / (1 - b1 ** t))
    return out


def batch_events(cfg, before: int, V: int) -> Dict[str, object]:
    """What one optimizer step over V views does to the schedules, starting from `before` views consumed (step() with
    G ranks, JointTrainer.step_batch with V views): the new iteration count; whether it crosses an SH-degree step
    (oneupSHdegree) or a 3D-filter recompute (not within the last 100 iterations); whether Adam steps (not at or
    after cfg.iterations).  The learning rates are those of the new iteration (adam_step_sizes)."""
    it = before + V
    return dict(iteration=it, sh_up=it // cfg.sh_increase_interval > before // cfg.sh_increase_interval,
                mip=it // cfg.mip_filter3d_interval > before // cfg.mip_filter3d_interval and it < cfg.iterations - 100,
                do_opt=it < cfg.iterations)


def batch_densify_events(cfg, before: int, V: int, white_background: bool) -> Dict[str, object]:
    """The densification schedule of one optimizer step over V views starting from `before` views consumed
    (JointTrainer.step_batch with densify, and step(), which densifies on one GPU only, with V = 1): view k of the
    batch stands for iteration before + 1 + k.
      n_stats: how many leading views count their statistics (those whose iteration is < densify_until_iter);
      densify: some covered iteration j is a densify point of step() (densify_from_iter < j < densify_until_iter,
               j % densification_interval == 0);
      reset: some covered j < densify_until_iter is an opacity reset (j % opacity_reset_interval == 0, or a white
             background and j == densify_from_iter);
      size_threshold: the screen-size limit of the densify, that of the last densify point covered (cfg.size_threshold
             when it is past opacity_reset_interval, else None); None without a densify.
    Each event fires at most once per step.  With V = 1 these are train.py's per-iteration rules."""
    its = range(before + 1, before + V + 1)
    dens = [j for j in its if cfg.densify_from_iter < j < cfg.densify_until_iter and j % cfg.densification_interval == 0]
    reset = any(j < cfg.densify_until_iter and (j % cfg.opacity_reset_interval == 0 or
                                                (white_background and j == cfg.densify_from_iter)) for j in its)
    size = None
    if dens and dens[-1] > cfg.opacity_reset_interval:
        size = cfg.size_threshold
    return dict(n_stats=min(max(cfg.densify_until_iter - 1 - before, 0), V), densify=bool(dens), reset=reset,
                size_threshold=size)


def L_sig_words():
    return (_lib.lib().gsb_peer_signal_bytes() + 3) // 4


def sh_rest_rows(f_rest: torch.Tensor, P: int) -> int:
    """The f_rest rows per Gaussian, M - 1 = (D+1)^2 - 1 for SH degree D (0, 3, 8 or 15), of an f_rest tensor
    [P, M-1, 3] (or [P, 3(M-1)]); GsbError with the reason for any other shape."""
    shape = tuple(f_rest.shape)
    if len(shape) == 3 and shape[0] == P and shape[2] == 3:
        rows = shape[1]
    elif len(shape) == 2 and shape[0] == P and shape[1] % 3 == 0:
        rows = shape[1] // 3
    else:
        raise _lib.GsbError(f"f_rest has shape {shape}; expected [P, M-1, 3] with P = {P}")
    d = int(round((rows + 1) ** 0.5)) - 1
    if rows not in (0, 3, 8, 15):
        raise _lib.GsbError(f"f_rest has {rows} rows per Gaussian; SH degree D stores (D+1)^2 - 1 of them, so one of "
                            "0, 3, 8 or 15 (degrees 0 to 3)" + (" (degree 4 and above are not supported)"
                                                                 if (d + 1) ** 2 == rows + 1 else ""))
    return rows


def segment_widths(rest_rows: int):
    """(name, floats per Gaussian) of the six per-Gaussian tensors of a model with `rest_rows` f_rest rows: SEGMENTS
    with f_rest at 3 * rest_rows (empty at degree 0)."""
    return tuple((name, 3 * rest_rows if name == "f_rest" else k) for name, k in SEGMENTS)


def flat_layout(P: int, widths=SEGMENTS):
    """Where the per-Gaussian tensors (name, width) of P Gaussians lie in the flat buffers: {name: (begin, end)}, each
    segment padded to a multiple of 64 floats (256 bytes; an empty f_rest takes no space), and the buffers' length."""
    segments, total = {}, 0
    for name, k in widths:
        segments[name] = (total, total + (P * k + 63) // 64 * 64)
        total = segments[name][1]
    return segments, total


class JointTrainer:
    def __init__(self, scene: Scene, device, gt_images: Optional[torch.Tensor] = None,
                 cfg: Optional[OptimConfig] = None, world_size: int = 1, rank: int = 0,
                 process_group=None, exchange: str = "allreduce", use_graph: bool = False):
        self.cfg = cfg or OptimConfig()
        if self.cfg.densify and world_size > 1:
            raise _lib.GsbError("densify=True needs world_size == 1: every rank would accumulate different "
                                "densification statistics")
        if self.cfg.random_background and world_size > 1:
            raise _lib.GsbError("random_background=True needs world_size == 1: the ranks' views of one step would need "
                                "consecutive colours of one shared sequence, which several GPUs do not draw")
        self.dev = torch.device(device)
        self.world_size, self.rank, self.pg = world_size, rank, process_group
        if exchange not in ("allreduce", "fused_p2p", "fused_p2p_nccl"):
            raise ValueError(f"unknown exchange mode {exchange!r}")
        self.exchange = exchange if world_size > 1 else "allreduce"
        # fused_p2p: peer-memory kernel bracketed by flag barriers over the same peer memory (default);
        # fused_p2p_nccl: same kernel bracketed by two tiny NCCL collectives (round-1 behaviour, kept for A/B runs)
        self._fused = self.exchange in ("fused_p2p", "fused_p2p_nccl")
        self.P = P = scene.P
        self.W, self.H = scene.width, scene.height
        self.fovx, self.fovy = float(scene.fovx), float(scene.fovy)
        self.sh_degree = scene.sh_degree
        self.n_views = scene.n_views
        # ---- the SH layout: the stored degree follows the scene's f_rest; cfg.max_sh_degree may not exceed it
        rows = sh_rest_rows(scene.params["f_rest"], P)
        self.stored_sh_degree = int(round((rows + 1) ** 0.5)) - 1
        self.sh_coeffs = rows + 1
        if self.cfg.max_sh_degree > self.stored_sh_degree:
            raise _lib.GsbError(f"OptimConfig.max_sh_degree {self.cfg.max_sh_degree} exceeds the scene's stored SH "
                                f"degree {self.stored_sh_degree} (f_rest has {rows} rows per Gaussian): the trainer "
                                "would raise the active degree past the coefficients it holds")
        self.widths = segment_widths(rows)
        # ---- flat buffers
        self.segments, self.total = flat_layout(P, self.widths)
        total = self.total
        if self._fused:
            # peer-visible parameter / gradient buffers (CUDA IPC) and shard-sized Adam moments
            from .parallel import PeerBuffer, shard_bounds
            self._peer_params = PeerBuffer(total, self.dev, process_group)
            self._peer_grads = PeerBuffer(total, self.dev, process_group)
            self.params, self.grads = self._peer_params.tensor, self._peer_grads.tensor
            self.shard = shard_bounds(total, world_size, rank)
            n_sh = max(4, self.shard[1] - self.shard[0])
            self.exp_avg = torch.zeros(n_sh, dtype=torch.float32, device=self.dev)
            self.exp_avg_sq = torch.zeros(n_sh, dtype=torch.float32, device=self.dev)
            self._sync = torch.zeros(1, dtype=torch.float32, device=self.dev)
            self._xch = torch.zeros(8 + scene.n_views * 7, dtype=torch.float32, device=self.dev)
            if self.exchange == "fused_p2p":
                self._peer_sig = PeerBuffer(L_sig_words(), self.dev, process_group)
        else:
            self.params = torch.zeros(total, dtype=torch.float32, device=self.dev)
            self.grads = torch.zeros(total, dtype=torch.float32, device=self.dev)
            self.exp_avg = torch.zeros(total, dtype=torch.float32, device=self.dev)
            self.exp_avg_sq = torch.zeros(total, dtype=torch.float32, device=self.dev)
        for name, k in self.widths:
            self.view(self.params, name).copy_(scene.params[name].reshape(P, k).to(self.dev))
        self.poses = scene.poses.to(self.dev).float().contiguous()              # [n_views,7]
        if self.exchange == "fused_p2p_nccl":
            self.pose_grad = self._xch[8:].view(scene.n_views, 7)
            self._pg_buf = None
        elif self.exchange == "fused_p2p":
            self.pose_grad = torch.zeros_like(self.poses)
            self._pg_buf = None
        else:
            # [n_views*7] pose gradients + 1 word carrying this rank's binning-overflow flag through the all-reduce
            self._pg_buf = torch.zeros(scene.n_views * 7 + 1, dtype=torch.float32, device=self.dev)
            self.pose_grad = self._pg_buf[:-1].view(scene.n_views, 7)
        self.pose_m = torch.zeros_like(self.poses)
        self.pose_v = torch.zeros_like(self.poses)
        self._set_per_point_lr(scene.per_point_lr if self.cfg.pp_optimizer else None)
        self.gt = None if gt_images is None else gt_images.to(self.dev).float().contiguous()
        self.ident = IdentityView(self.W, self.H, scene.fovx, scene.fovy, scene.bg, self.dev)
        self._single = self._Slot(self.dev, P, self.W, self.H)   # step()'s forward; sized by the first forward
        self.headroom = 1.5
        self.filter_3D, self.filt, self.mip_recomputed_at = None, None, []
        self._mip_setup()
        self.dL_dimg = torch.empty_like(self.color)
        self.maps = torch.empty(3, 3, self.H, self.W, dtype=torch.float32, device=self.dev)
        self.sums = torch.zeros(2, dtype=torch.float64, device=self.dev)
        self._ev_pre = torch.cuda.Event()
        self._ovf = None
        self.flags = torch.zeros(8, dtype=torch.int32, device=self.dev)
        self._pose_flags = torch.zeros(8, dtype=torch.int32, device=self.dev)
        if world_size > 1:    # the word the optimizer kernels test: overflow flags summed over the ranks
            self._ovf = self.flags[7:8] if self._fused else self._pg_buf[-1:]
        # CUDA-graph replay of the whole iteration: one graph per (view, ground-truth buffer); everything that changes
        # from step to step reaches the kernels through device memory (Adam step sizes, the flag barriers' epoch) or is
        # part of the graph's identity (view pose row, active SH degree, binning capacity).  Multi-GPU: only the
        # "fused_p2p" exchange is capturable (its collectives are this library's own kernels over peer memory; every
        # rank replays its own graph and the flag barriers inside keep the ranks in step).
        self.use_graph = bool(use_graph) and (world_size == 1 or self.exchange == "fused_p2p")
        self._graphs = {}
        self._after_backward = None   # test hook: called (and captured) between the backward and the optimizer step
        self._step_dev = torch.zeros(8, dtype=torch.float32, device=self.dev)   # every update's step sizes (_advance)
        self._polling = False
        self.iteration = 0            # reference iterations = views consumed (by all ranks)
        self.opt_step = 0
        self.last_R = 0
        self.overflows = 0
        self.exact_cull = True
        self.active_sh_degree = min(scene.sh_degree, self.cfg.max_sh_degree)
        c = self.cfg
        self._keep = None
        # per-tensor Adam step counts are opt_step minus the optimizer steps that skipped the tensor (the densify and
        # opacity-reset iterations replace tensors, which then have no gradient in the reference)
        self._lag = {name: 0 for name, _ in self.widths}
        self._stats = None
        if c.densify:
            self._stats = torch.zeros(3, P, dtype=torch.float32, device=self.dev)
            self.scene_extent = cameras_extent(scene.poses) if c.scene_extent is None else float(c.scene_extent)
            self.densify_generator = torch.Generator(device=self.dev).manual_seed(int(c.densify_seed))
            self.white_background = bool((scene.bg == 1).all())
        self.densified_at, self.reset_at = [], []
        # one generator for the run's background colours, drawn from outside any graph into the slots' fixed rows
        self.background_generator = None
        if c.random_background:
            self.background_generator = torch.Generator(device=self.dev).manual_seed(int(c.background_seed))
        self._batch = None            # step_batch's slot for the view count of its last call (_batch_scratch)
        self._batch_sums = None       # per-view loss sums of the last step_batch (batch_loss_values)

    # ------------------------------------------------------------------------------------------
    def view(self, flat: torch.Tensor, name: str) -> torch.Tensor:
        k = dict(self.widths)[name]
        o = self.segments[name][0]
        return flat[o:o + self.P * k].view(self.P, k)

    def my_views(self) -> List[int]:
        from .parallel import shard_views
        return shard_views(self.n_views, self.world_size, self.rank)

    @property
    def frame(self) -> Frame:
        """The Frame of step() and render() (one view)."""
        return self._single.frame

    @property
    def host_status(self) -> torch.Tensor:
        """The pinned [2, ST_WORDS] status words of that frame's last forward: [0] after preprocess, [1] after render."""
        return self._single.host_status

    @property
    def color(self) -> torch.Tensor:
        """The last rendered image [3, H, W]."""
        return self.frame.color

    @property
    def cap(self) -> int:
        """Instance capacity of the binning buffer (0: not sized yet)."""
        return self.frame.cap

    # densification statistics with the reference's names and shapes (None unless cfg.densify)
    @property
    def xyz_gradient_accum(self) -> Optional[torch.Tensor]:
        return None if self._stats is None else self._stats[0].view(self.P, 1)

    @property
    def denom(self) -> Optional[torch.Tensor]:
        return None if self._stats is None else self._stats[1].view(self.P, 1)

    @property
    def max_radii2D(self) -> Optional[torch.Tensor]:
        return None if self._stats is None else self._stats[2]

    def step_count(self, name: str) -> int:
        """Adam step count of one tensor ("pose" or a per-Gaussian tensor's name)."""
        return self.opt_step - self._lag.get(name, 0)

    def _mip_setup(self) -> None:
        """A filter_3D buffer for the current P, filled; the GsbFilter points at it for the buffer's lifetime, so the
        recompute (outside any captured graph) changes what graph replays read without changing the graphs."""
        if self.cfg.mip_kernel_size is None:
            return
        self.filter_3D = torch.empty(self.P, dtype=torch.float32, device=self.dev)
        self.filt = mip_filter(self.cfg.mip_kernel_size, self.filter_3D)
        self.compute_filter_3D()

    def compute_filter_3D(self) -> None:
        """Recompute the 3D smoothing filter from the current xyz and pose table (gsb_mip_filter3d, deterministic)."""
        mip_filter3d(self.view(self.params, "xyz"), self.poses, self.W, self.H, self.ident.tanfovx, self.ident.tanfovy,
                     out=self.filter_3D)

    def _gauss(self, poses: torch.Tensor) -> GsbGaussians:
        """The Gaussians at a pose row [7] (or, for the batched entry points, rows [V, 7])."""
        p = self.params
        return gaussians(self.P, *(self.view(p, n) for n in ("xyz", "rotation", "scaling", "opacity", "f_dc")),
                         self.view(p, "f_rest") if self.sh_coeffs > 1 else None, poses)

    def _camera(self, bg: Optional[torch.Tensor] = None):
        """The frame's camera at the active SH degree; bg: a [3] device tensor to blend over instead of the scene's."""
        cam = self.ident.camera(self.active_sh_degree, self.sh_coeffs, self.exact_cull)
        if bg is not None:
            cam.bg = bg.data_ptr()
        return cam

    def _train_bg(self, slot: "_Slot") -> Optional[torch.Tensor]:
        """The background a training forward on `slot` blends over: its drawn colours with random_background (step():
        [3], step_batch: [V, 3]), else None (the scene's)."""
        return slot.bg if self.background_generator is not None else None

    def _draw_backgrounds(self, slot: "_Slot") -> None:
        """train.py:164's bg = torch.rand((3), device="cuda") once for each iteration a step covers, into `slot`'s rows
        (row k: iteration before + k + 1), on the current stream and outside any graph, so a graph reads the new colours
        at the same address.  One torch draw of 3 per row: a single draw of [V, 3] would not give train.py's sequence."""
        for row in slot.bg.view(-1, 3):
            row.uniform_(0.0, 1.0, generator=self.background_generator)

    def _nonempty(self):
        """The (name, width) of the per-Gaussian tensors the kernels update: all six, but f_rest only above degree 0."""
        return [(name, k) for name, k in self.widths if k > 0]

    # ------------------------------------------------------------------------------------------
    def _size_binning(self, R: int, slot: Optional["_Slot"] = None) -> None:
        """A binning buffer for R instances plus headroom, in `slot`'s frame (None: step()'s)."""
        (slot or self._single).frame.alloc_binning(capacity(R, self.headroom))

    def _forward(self, slot: "_Slot", cam, g: GsbGaussians, poses: Optional[torch.Tensor] = None,
                 bg: Optional[torch.Tensor] = None) -> None:
        """Enqueue a forward of `slot`'s frame (poses: the [V, 7] rows of a batch slot; bg: its [V, 3] background
        table, None: cam's background) without ever waiting for the GPU: the instance count R stays on the device; the
        host only provides a capacity (sized from the counts seen so far, +50 %) and reads R back lazily."""
        fr, hs = slot.frame, slot.host_status
        if slot.V is None:
            fr.preprocess(cam, g, hs[0], self.filt)
        else:
            fr.preprocess_batch(cam, g, poses, hs[0], self.filt)
        if not torch.cuda.is_current_stream_capturing():
            slot.fwd_count += 1
            self._polling = False
            self._ev_pre.record()
            if fr.cap == 0:                           # very first forward: size the buffer from the real count
                self._ev_pre.synchronize()
                self._size_binning(read_R(hs[0]), slot)
        if slot.V is None:
            fr.render(cam, hs[1])
        else:
            fr.render_batch(cam, hs[1], bg)

    def _launch_forward(self, view: int, bg: Optional[torch.Tensor] = None) -> None:
        cam, g = self._camera(bg), self._gauss(self.poses[view])
        self._forward(self._single, cam, g)
        self._keep = (cam, g)

    def _settle(self, slot: Optional["_Slot"] = None) -> bool:
        """Wait for the status words of the preprocess phase of `slot`'s last forward (None: step()'s slot; early in
        the stream: the GPU still has the rest of the iteration queued, so this never starves it).  Returns True if the
        binning buffer was big enough; otherwise grows it (the device skipped the optimizer update by itself) and
        returns False."""
        slot = slot or self._single
        fr, hs = slot.frame, slot.host_status
        if self._polling:
            # graph replay: no host-visible event inside the graph, so watch the pinned status words for this forward's
            # serial number (written by the tile scan, copied by the memcpy node right behind it)
            want = slot.fwd_count & 0x7FFFFFFF
            n = 0
            while (int(hs[0, ST_SEQ]) & 0x7FFFFFFF) != want:
                n += 1
                if n > 20_000_000:
                    raise _lib.GsbError("graph replay: the forward's status words never arrived")
        else:
            self._ev_pre.synchronize()
        R = read_R(hs[0])
        self.last_R = R
        if R > fr.cap:
            self.overflows += 1
            self._size_binning(R, slot)
            return False
        if R > 0.85 * fr.cap:                          # grow ahead of need
            self._size_binning(R, slot)
        return True

    def _settled(self, enqueue, local: bool = False, batch: Optional["_Slot"] = None) -> None:
        """enqueue() launches a forward, possibly with the rest of an iteration; then wait for its instance count.  When
        the binning buffer was too small, the device has skipped the optimizer update by itself (gated on the overflow
        word, summed over the ranks in multi-GPU mode), so parameters and moments are untouched, and _settle has grown
        the buffer: enqueue once more.  Several ranks cannot do that within a training iteration, because the other
        ranks cannot know yet; they stop loudly.  local: only this rank's forward, which any rank may repeat.
        batch: the slot whose frame makes that forward (None: step()'s single-view slot)."""
        for _ in range(2):
            enqueue()
            if self._settle(batch):
                return
            if self.world_size > 1 and not local:
                raise _lib.GsbError(f"rank {self.rank}: {self.last_R} instances exceeded the binning capacity; the "
                                    "optimizer update of this step was skipped on every rank (parameters are "
                                    "consistent).  Raise JointTrainer.headroom.")
        raise _lib.GsbError(f"{self.last_R} instances exceeded the binning capacity twice in a row")

    def render(self, view: int) -> torch.Tensor:
        """Forward only (exact: repeated with a larger buffer in the unlikely case the capacity was exceeded)."""
        self._settled(lambda: self._launch_forward(view), local=True)
        return self.color

    def loss_and_backward(self, view: int, gt: torch.Tensor, stats: bool = False) -> None:
        """stats: the backward also accumulates the densification statistics (train.py:197-199)."""
        L = _lib.lib()
        st = _lib.stream_ptr()
        cam, g = self._keep
        self.sums.zero_()
        check(L.gsb_loss_forward(3, self.H, self.W, self.color.data_ptr(), gt.data_ptr(), self.sums.data_ptr(),
                                 self.maps.data_ptr(), st), "gsb_loss_forward")
        check(L.gsb_loss_backward(3, self.H, self.W, self.color.data_ptr(), gt.data_ptr(), self.maps.data_ptr(),
                                  float(self.cfg.lambda_dssim), self.dL_dimg.data_ptr(), st), "gsb_loss_backward")
        gr = self._grads()
        self.pose_grad.zero_()
        gr.dL_dpose = self.pose_grad[view].data_ptr()
        st = None
        if stats:
            st = densify_stats(self.frame.radii, self._stats[0], self._stats[1], self._stats[2])
        self.frame.backward(cam, g, self.dL_dimg, gr, self.filt, st)

    def _grads(self) -> GsbGrads:
        """GsbGrads over the per-Gaussian segments of the flat gradient buffer (no pose gradient)."""
        gr = GsbGrads()
        gd = self.grads
        gr.dL_dmeans3D = self.view(gd, "xyz").data_ptr()
        gr.dL_dscales = self.view(gd, "scaling").data_ptr()
        gr.dL_drotations = self.view(gd, "rotation").data_ptr()
        gr.dL_dopacities = self.view(gd, "opacity").data_ptr()
        gr.dL_dsh_dc = self.view(gd, "f_dc").data_ptr()
        gr.dL_dsh_rest = self.view(gd, "f_rest").data_ptr() if self.sh_coeffs > 1 else None
        return gr

    def _loss(self, sums: torch.Tensor) -> torch.Tensor:
        """train.py's loss (1 - lambda_dssim) L1 + lambda_dssim (1 - SSIM) from loss sums [..., 2] (L1, SSIM)."""
        n = 3 * self.H * self.W
        lam = self.cfg.lambda_dssim
        return (1.0 - lam) * sums[..., 0] / n + lam * (1.0 - sums[..., 1] / n)

    def loss_value(self) -> torch.Tensor:
        return self._loss(self.sums)

    def reduce_grads(self) -> None:
        if self.world_size > 1:
            from .parallel import allreduce_sum_
            self._pg_buf[-1:].copy_(self.frame.word(ST_OVERFLOW))
            allreduce_sum_((self.grads, self._pg_buf), self.pg)

    def _stepped(self, skip=()) -> List[str]:
        """The tensors an optimizer update steps, in launch order: entry i of the update reads _step_dev[i].  An empty
        f_rest (degree 0) is not launched; its step count still advances with the others (_lag)."""
        names = [name for name, _ in self._nonempty() if name not in skip]
        return names + ["pose"] if self.cfg.optim_pose else names

    def _advance(self, skip=()) -> None:
        """Count one optimizer step, which the tensors in `skip` do not take (they were replaced in this iteration, so
        the reference's parameter has no gradient; their step counts stay), and upload the update's step sizes to
        _step_dev, stream-ordered before whatever is enqueued next.  The pinned staging buffer comes from PyTorch's
        caching host allocator, which hands it out again only after the copy has run."""
        self.opt_step += 1
        for name in skip:
            self._lag[name] += 1
        sizes = adam_step_sizes(self.cfg, self.iteration, self.opt_step, self._lag)
        names = self._stepped(skip)
        host = torch.tensor([float(sizes[name]) for name in names], dtype=torch.float32, pin_memory=True)
        self._step_dev[:len(names)].copy_(host, non_blocking=True)

    def _adam_entry(self, name: str, grad_scale: float) -> dict:
        """launch_adam's entry of one tensor ("pose" or a per-Gaussian tensor's name); its step size is in _step_dev."""
        if name == "pose":
            t = dict(param=self.poses, grad=self.pose_grad, exp_avg=self.pose_m, exp_avg_sq=self.pose_v, row_len=7,
                     per_point_lr=None)
        else:
            t = dict(param=self.view(self.params, name), grad=self.view(self.grads, name),
                     exp_avg=self.view(self.exp_avg, name), exp_avg_sq=self.view(self.exp_avg_sq, name),
                     row_len=dict(self.widths)[name], per_point_lr=self.per_point_lr if name == "xyz" else None)
        return dict(t, beta1=ADAM_BETAS[0], beta2=ADAM_BETAS[1], eps=ADAM_EPS, weight_decay=0.0, grad_scale=grad_scale)

    def optimizer_step(self, grad_scale: Optional[float] = None, skip=()) -> None:
        """PerPointAdam.step over the 6 Gaussian tensors + the pose table in one launch
        (param groups and LRs of scene/gaussian_model.py:203-243).  skip: Gaussian tensors that take no step."""
        self._advance(skip)
        self._launch_adam(grad_scale, skip)

    def _launch_adam(self, grad_scale: Optional[float] = None, skip=(), skip_ptr=None) -> None:
        gs = 1.0 / self.world_size if grad_scale is None else grad_scale
        launch_adam([self._adam_entry(name, gs) for name in self._stepped(skip)], self.flags,
                    skip_ptr=self._skip_ptr() if skip_ptr is None else skip_ptr, step_sizes_dev=self._step_dev)

    def _skip_ptr(self):
        """Device word that makes the optimizer kernels skip the update: the forward's overflow status
        (multi-GPU: its sum over ranks, so that every replica takes the same decision)."""
        if self.world_size > 1:
            return self._ovf.data_ptr()
        return self.frame.word(ST_OVERFLOW).data_ptr()

    def fused_exchange_step(self) -> None:
        """Multi-GPU: gate flags + pose gradients summed over the ranks (one tiny kernel over peer memory, or a tiny
        NCCL all-reduce; either doubles as the pre-barrier), then ONE kernel per rank doing reduce-scatter ->
        per-point Adam -> all-gather over NVLink peer memory (csrc/gs_comm.cu), then a barrier before anyone reads
        the new parameters."""
        self._advance()
        self._launch_fused()

    def _launch_fused(self) -> None:
        import torch.distributed as dist
        from ._lib import GsbAdamTensor, GsbShardPiece
        L = _lib.lib()
        st = _lib.stream_ptr()
        # 1. whole-tensor gates on the local gradients, OR-ed across ranks
        segs = self._nonempty()
        arr = (GsbAdamTensor * len(segs))()
        for a, (name, k) in zip(arr, segs):
            g = self.view(self.grads, name)
            a.param = a.exp_avg = a.exp_avg_sq = a.grad = g.data_ptr()
            a.numel, a.row_len, a.grad_scale = g.numel(), k, 1.0
        check(L.gsb_adam_gate(len(segs), arr, self.flags.data_ptr(), st), "gsb_adam_gate")
        if self.exchange == "fused_p2p":
            # gate flags, the binning-overflow word and the pose-gradient table are summed over the ranks by ONE tiny
            # kernel through peer memory; its flag barrier is also "every rank's gradients are written".  Epoch 0 = the
            # device-resident epoch counter (advanced by this kernel), so the launch is identical every step
            check(L.gsb_peer_exchange(self.world_size, self.rank, self._peer_sig.ptr_array(), 0,
                                      self.flags.data_ptr(), self.frame.word(ST_OVERFLOW).data_ptr(),
                                      self.pose_grad.data_ptr(),
                                      self.pose_grad.numel(), st), "gsb_peer_exchange")
        else:
            # one small SUM all-reduce carries both the gate flags (as counts) and the pose-gradient table
            # (self.pose_grad is a view of self._xch[8:]); it is also the pre-barrier of the fused kernel
            self._xch[:8].copy_(self.flags)
            self._xch[7:8].copy_(self.frame.word(ST_OVERFLOW))  # slot 7: binning overflow (summed over ranks)
            dist.all_reduce(self._xch, op=dist.ReduceOp.SUM, group=self.pg)
            self.flags.copy_(self._xch[:8])
        # 2. the fused kernel over this rank's shard; a piece of segment i reads step size i of _step_dev (nothing is
        # skipped: the number of Gaussians is fixed with peer-memory buffers)
        lo, hi = self.shard
        pieces = []
        for fi, (name, k) in enumerate(segs):
            s0, s1 = self.segments[name]
            b, e = max(lo, s0), min(hi, s1)
            if e > b:
                pc = GsbShardPiece()
                pc.begin, pc.end, pc.seg_begin = b, e, s0
                pc.per_point_lr = self.per_point_lr.data_ptr() if (name == "xyz" and self.per_point_lr is not None) else None
                pc.row_len, pc.flag_index = k, fi
                pc.beta1, pc.beta2, pc.eps = ADAM_BETAS[0], ADAM_BETAS[1], ADAM_EPS
                pieces.append(pc)
        parr = (GsbShardPiece * max(1, len(pieces)))(*pieces)
        check(L.gsb_fused_rs_adam_ag(self.world_size, self.rank, self._peer_grads.ptr_array(),
                                     self._peer_params.ptr_array(), self.exp_avg.data_ptr(),
                                     self.exp_avg_sq.data_ptr(), lo, len(pieces), parr, self.flags.data_ptr(),
                                     self._ovf.data_ptr(), 1.0 / self.world_size, self._step_dev.data_ptr(), st),
              "gsb_fused_rs_adam_ag")
        # 3. pose table: replicated Adam on the all-reduced pose gradients
        if self.cfg.optim_pose:
            launch_adam([self._adam_entry("pose", 1.0 / self.world_size)], self._pose_flags, skip_ptr=self._ovf.data_ptr(),
                        step_sizes_dev=self._step_dev[len(segs):])
        # 4. nobody may start the next forward before every rank's parameter stores have landed
        if self.exchange == "fused_p2p":
            check(L.gsb_peer_barrier(self.world_size, self.rank, self._peer_sig.ptr_array(), 0, 1, st),
                  "gsb_peer_barrier")
        else:
            dist.all_reduce(self._sync, group=self.pg)

    def _enqueue_iteration(self, view: int, gt: torch.Tensor, do_opt: bool, stats: bool = False) -> None:
        """One iteration on `view` with no wait, launched eagerly or captured into a graph: forward, loss + backward,
        the test hook, and (do_opt) the exchange and update with the step sizes _advance uploaded."""
        self._launch_forward(view, self._train_bg(self._single))
        self.loss_and_backward(view, gt, stats)
        if self._after_backward is not None:
            self._after_backward()
        if not do_opt:
            return
        if self._fused:
            self._launch_fused()
        else:
            self.reduce_grads()
            self._launch_adam()

    def _replay(self, key: tuple, slot: "_Slot", enqueue) -> None:
        """Replay the CUDA graph cached under `key`, capturing enqueue() (an iteration whose forward runs on `slot`'s
        frame) into it on first use."""
        g = self._graphs.get(key)
        if g is None:
            if len(self._graphs) > 64:
                self._graphs.clear()
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                enqueue()
            self._graphs[key] = g
        slot.fwd_count += 1
        self._polling = True
        g.replay()

    def close(self) -> None:
        """Release the peer-visible buffers of the fused exchange (collective over the process group)."""
        for name in ("_peer_params", "_peer_grads", "_peer_sig"):
            pb = getattr(self, name, None)
            if pb is not None:
                if name == "_peer_params":
                    self.params = None
                if name == "_peer_grads":
                    self.grads = None
                pb.close(self.pg)
                setattr(self, name, None)

    def check_peer_errors(self) -> None:
        """Raise if a flag-barrier wait timed out on this rank (a peer died or fell out of step)."""
        if getattr(self, "_peer_sig", None) is not None:
            if int(self._peer_sig.tensor[60:61].view(torch.int32).item()) != 0:
                raise _lib.GsbError(f"rank {self.rank}: a peer flag barrier timed out")

    def step(self, view: int, gt: Optional[torch.Tensor] = None) -> None:
        """One reference iteration on `view` (train.py:140-211): update_learning_rate(iteration), oneupSHdegree every
        1000 iterations, render, loss, backward, optimizer step (skipped on the very last iteration, :209-211).
        With G GPUs one call consumes G views (one per rank): `iteration` counts VIEWS, so the learning-rate and
        SH-degree schedules advance per view as in the reference, while Adam's bias correction counts optimizer
        steps.  Nothing in here waits for the GPU except `_settle()`, which waits for an event early in the stream.
        With cfg.random_background the iteration renders over its own colour (train.py:164), drawn once per call."""
        if gt is None:
            gt = self.gt[view]
        self._run_step(self.world_size, self._single, ("step", view, gt.data_ptr()),
                       lambda do_opt, n_stats: self._enqueue_iteration(view, gt, do_opt, n_stats > 0))

    def _run_step(self, n: int, slot: "_Slot", head: tuple, enqueue, grad_scale: Optional[float] = None,
                  skip_ptr=None) -> None:
        """One optimizer step that consumes n views, whose forward runs on `slot`'s frame.  The schedules come from
        batch_events and batch_densify_events.  enqueue(do_opt, n_stats) enqueues the iteration with no wait, its
        backward adding the densification statistics of its first n_stats views; it is launched eagerly or replayed
        from the graph cached under `head` plus the state a graph bakes in.  An iteration that densifies or resets the
        opacity runs eagerly without its update, and Adam follows the event with grad_scale and skip_ptr (None:
        _launch_adam's defaults, read after the event has rebuilt the buffers)."""
        c = self.cfg
        ev = batch_events(c, self.iteration, n)
        de = dict(n_stats=0, densify=False, reset=False, size_threshold=None)
        if self._stats is not None:
            de = batch_densify_events(c, self.iteration, n, self.white_background)
        n_stats = de["n_stats"]
        self.iteration = ev["iteration"]
        if self.background_generator is not None:
            self._draw_backgrounds(slot)   # once per step: a repeat after an overflow and an eager event reuse them
        if ev["sh_up"]:
            self.active_sh_degree = min(self.active_sh_degree + 1, c.max_sh_degree)     # oneupSHdegree
        do_opt = ev["do_opt"]
        if de["densify"] or de["reset"]:
            # train.py:201-211: densify / reset between the backward and the optimizer step, eagerly (the optimizer's
            # tensor set differs); the replaced tensors take no step.  densify_and_prune rebuilds the buffers and the
            # slots (`slot` stays alive here).
            self._settled(lambda: enqueue(False, n_stats), batch=slot)
            skip = set()
            if de["densify"]:
                self.densify_and_prune(c.densify_grad_threshold, c.min_opacity, self.scene_extent, de["size_threshold"],
                                       c.densify_clone_split, self.densify_generator)
                self.densified_at.append(self.iteration)
                skip.update(name for name, _ in self.widths)
            if de["reset"]:
                self.reset_opacity()
                self.reset_at.append(self.iteration)
                skip.add("opacity")
            if do_opt:
                skip = [name for name, _ in self.widths if name in skip]
                self._advance(skip)
                self._launch_adam(grad_scale, skip, skip_ptr)
        else:
            if do_opt:
                self._advance()        # once per step: a repeat after an overflow takes the same step
            if self.use_graph and slot.frame.cap > 0:
                run = lambda: self._replay(head + (do_opt, self.active_sh_degree, slot.frame.cap, self.exact_cull,
                                                   n_stats), slot, lambda: enqueue(do_opt, n_stats))
            else:
                run = lambda: enqueue(do_opt, n_stats)
            self._settled(run, batch=slot)
        if self.filt is not None and ev["mip"]:
            self.compute_filter_3D()
            self.mip_recomputed_at.append(self.iteration)

    # ---- several views per optimizer step on one GPU (DESIGN.md section 4.10) ----------------------------------
    def step_batch(self, views: Sequence[int], gts: Optional[torch.Tensor] = None) -> None:
        """One optimizer step over the V views `views` (distinct indices into the pose table), with the semantics of
        step() on V ranks: `iteration` advances by V, and the SH-degree, learning-rate and Mip-filter schedules fire
        when it crosses their points; every view is rendered at its own pose row, its loss is train.py's on its target
        (gts[k] for views[k], or the trainer's own targets when gts is None); the per-Gaussian gradients are summed in
        the order of `views`, each view's dL/dpose lands in its row of pose_grad (the other rows are zero); one Adam
        step with grad_scale = 1/V over the six tensors and the whole pose table (skipped at the last iteration).
        step_batch([v]) equals step(v) bit for bit.  The per-view losses stay on the device (batch_loss_values()).
        With cfg.random_background, views[k] renders over the colour of iteration `iteration + k + 1` (the V colours
        step() would draw over the same V iterations).

        With OptimConfig.densify, cfg.densify_batches must be set: each view whose iteration is below densify_until_iter
        adds its own statistics (batch_densify_events), and the densify / opacity-reset events of the iterations the
        step covers run once, after the step's backward and before its Adam step, eagerly.  step_batch([v]) then still
        equals step(v) bit for bit.

        With use_graph, the captured graph is keyed on the address of the targets: pass gts=None (the trainer's own
        targets) or the same held buffer on every call.  A fresh tensor per call (or a non-contiguous one, which is
        copied) makes every call capture a new graph, and beyond 64 graphs the cache, step()'s graphs included, is
        cleared."""
        if self.world_size > 1:
            raise _lib.GsbError("step_batch needs world_size == 1 (batches on several GPUs are not implemented)")
        if self._stats is not None and not self.cfg.densify_batches:
            raise _lib.GsbError("step_batch with OptimConfig.densify=True needs OptimConfig.densify_batches=True: it "
                                "moves the densify and opacity-reset events to batch boundaries (or use step())")
        views = [int(v) for v in views]
        V = len(views)
        if V == 0:
            raise ValueError("step_batch: no views")
        if len(set(views)) != V:
            raise ValueError(f"step_batch: duplicate views in {views} (each view owns one pose row)")
        if any(not 0 <= v < self.n_views for v in views):
            raise ValueError(f"step_batch: views {views} out of range 0..{self.n_views - 1}")
        if gts is None:
            if self.gt is None:
                raise ValueError("step_batch: no targets (the trainer has no gt_images and gts is None)")
            target, rows = self.gt, views
        else:
            dev = self.dev if self.dev.index is not None else torch.device(self.dev.type, torch.cuda.current_device())
            if not isinstance(gts, torch.Tensor) or tuple(gts.shape) != (V, 3, self.H, self.W) or \
                    gts.dtype != torch.float32 or gts.device != dev:
                raise ValueError(f"step_batch: gts must be a float32 tensor of shape {(V, 3, self.H, self.W)} on {dev}, "
                                 f"got {getattr(gts, 'dtype', type(gts))} {tuple(getattr(gts, 'shape', ()))} on "
                                 f"{getattr(gts, 'device', None)}")
            target, rows = gts.contiguous(), list(range(V))
        b = self._batch_scratch(V)
        # the view ids and target rows reach the (possibly captured) iteration through device memory
        b.sel.copy_(torch.tensor([views, rows], dtype=torch.int64, pin_memory=True), non_blocking=True)
        self._run_step(V, b, ("batch", V, target.data_ptr()),
                       lambda do_opt, n_stats: self._enqueue_batch(b, target, do_opt, n_stats),
                       1.0 / V, b.frame.word(ST_OVERFLOW).data_ptr())
        self._batch_sums = b.sums

    def batch_loss_values(self) -> torch.Tensor:
        """loss_value() of each view of the last step_batch call, [V] on the device (views in the call's order)."""
        if self._batch_sums is None:
            raise _lib.GsbError("batch_loss_values: no step_batch call since the trainer was built, resized or restored")
        return self._loss(self._batch_sums)

    # ---- evaluation (train.py:256-290 training_report; DESIGN.md section 4.11) ----------------------------------
    def evaluate(self, views: Optional[Sequence[int]] = None, poses: Optional[torch.Tensor] = None,
                 gts: Optional[torch.Tensor] = None, mode: str = "clamp",
                 max_batch: Optional[int] = None) -> Dict[str, torch.Tensor]:
        """training_report's loop: render views and measure them against their targets (evaluation.image_metrics).
        views: indices into the pose table (None: every training view), each rendered at its pose row and compared
        with gts[k] for views[k], or with the trainer's own target when gts is None.  poses [V, 7] with gts
        [V, 3, H, W] instead: explicit poses (the test views at get_RT_test), not together with views.
        Each chunk of up to max_batch views (None: all at once) is one batched forward as in a step (active SH
        degree, Mip filters, exact_cull) with its own scratch, its binning buffer sized exactly from the preprocess
        count, then one metrics call.  Returns image_metrics' dict over all views (fp64 device tensors); view k's
        values do not depend on max_batch or on the other views.  Reads only the parameters, poses and targets and
        writes no training state; the scratch is released on return."""
        from .evaluation import _images, _mode, metric_sums, metrics_from_sums
        if self.world_size > 1:
            raise _lib.GsbError("evaluate needs world_size == 1 (evaluation on several GPUs is not implemented)")
        m = _mode(mode)
        if max_batch is not None and int(max_batch) < 1:
            raise ValueError("evaluate: max_batch must be >= 1")
        dev = self.dev if self.dev.index is not None else torch.device(self.dev.type, torch.cuda.current_device())
        if poses is not None:
            if views is not None:
                raise ValueError("evaluate: pass views or poses, not both")
            if not isinstance(poses, torch.Tensor) or poses.dim() != 2 or poses.shape[1] != 7 or \
                    poses.dtype != torch.float32 or poses.device != dev:
                raise ValueError(f"evaluate: poses must be a float32 [V, 7] tensor on {dev}, got "
                                 f"{getattr(poses, 'dtype', type(poses))} {tuple(getattr(poses, 'shape', ()))} on "
                                 f"{getattr(poses, 'device', None)}")
            if gts is None:
                raise ValueError("evaluate: explicit poses need their targets gts")
            pose_rows = poses.detach().contiguous()
            V = pose_rows.shape[0]
        else:
            views = list(range(self.n_views)) if views is None else [int(v) for v in views]
            if any(not 0 <= v < self.n_views for v in views):
                raise ValueError(f"evaluate: views {views} out of range 0..{self.n_views - 1}")
            V = len(views)
            if gts is None and self.gt is None:
                raise ValueError("evaluate: no targets (the trainer has no gt_images and gts is None)")
        if V == 0:
            raise ValueError("evaluate: no views")
        if gts is not None:
            gts = _images(gts, "evaluate: gts", dev)
            if tuple(gts.shape) != (V, 3, self.H, self.W):
                raise ValueError(f"evaluate: gts must have shape {(V, 3, self.H, self.W)}, got {tuple(gts.shape)}")
            target, rows = gts, list(range(V))
        else:
            target, rows = self.gt, views
        if poses is None:
            with torch.no_grad():      # a restored pose table may carry requires_grad from the checkpoint's Parameter
                pose_rows = self.poses.detach()[torch.tensor(views, dtype=torch.int64, device=dev)].contiguous()
        step = V if max_batch is None else int(max_batch)
        cam = self._camera()
        host_status = torch.zeros(ST_WORDS, dtype=torch.int32).pin_memory()
        sums, ovf = [], torch.zeros(1, dtype=torch.int32, device=dev)
        fr = None
        for v0 in range(0, V, step):
            v1 = min(V, v0 + step)
            pr = pose_rows[v0:v1]
            if fr is None or fr.views != v1 - v0:
                fr = None
                fr = Frame(dev, self.P, self.W, self.H, views=v1 - v0)
            g = self._gauss(pr)
            fr.preprocess_batch(cam, g, pr, host_status, self.filt)
            torch.cuda.current_stream(dev).synchronize()
            fr.alloc_binning(max(1, read_R(host_status)))
            fr.render_batch(cam)
            ovf |= fr.word(ST_OVERFLOW)
            sums.append(metric_sums(fr.color, target, rows[v0:v1], m))
        if int(ovf.item()):
            raise _lib.GsbError("evaluate: a tile list outgrew the binning buffer sized from the preprocess count")
        return metrics_from_sums(torch.cat(sums), self.H, self.W)

    class _Slot:
        """Where a forward runs: a Frame, the pinned [2, ST_WORDS] buffer its status words are copied to ([0] after
        preprocess, [1] after render) and the count of its forwards.  Each frame numbers its forwards in its own status
        words and copies them to its own pinned buffer, so a serial number is only ever compared with the count of the
        frame that wrote it (_settle); bg: the colours random_background draws for the slot's forward ([3], or [V, 3]
        for a batch).  V None: step()'s single view.  Otherwise step_batch's buffers for V views:
        sel [2, V] (view ids, target rows; uploaded per call), the gathered poses and their gradients [V, 7],
        dL/dimage, loss maps and per-view loss sums."""

        def __init__(self, dev, P, W, H, V=None):
            self.V = V
            self.frame = Frame(dev, P, W, H, views=V)
            self.frame.status.zero_()          # the forward serial number lives in these words
            self.fwd_count = 0
            self.host_status = torch.zeros(2, ST_WORDS, dtype=torch.int32).pin_memory()
            self.bg = torch.empty(3 if V is None else (V, 3), dtype=torch.float32, device=dev)
            if V is None:
                return
            self.sel = torch.zeros(2, V, dtype=torch.int64, device=dev)
            self.rows = torch.zeros(V, dtype=torch.int32, device=dev)
            self.poses = torch.zeros(V, 7, dtype=torch.float32, device=dev)
            self.dpose = torch.zeros(V, 7, dtype=torch.float32, device=dev)
            self.dL = torch.empty_like(self.frame.color)
            self.maps = torch.empty(3, V, 3, H, W, dtype=torch.float32, device=dev)
            self.sums = torch.zeros(V, 2, dtype=torch.float64, device=dev)

    def _batch_scratch(self, V: int) -> "_Slot":
        """The slot for V views; one is held at a time (a call with another V replaces it, and with it the graphs
        captured over it).  One graph per (V, target buffer, do_opt, active SH degree, capacity, exact_cull, n_stats)
        serves every choice of views: they are read from sel."""
        if self._batch is None or self._batch.V != V:
            self._batch = None
            self._graphs = {k: g for k, g in self._graphs.items() if k[0] != "batch"}
            self._batch = self._Slot(self.dev, self.P, self.W, self.H, V)
        return self._batch

    def _enqueue_batch(self, b: "_Slot", target: torch.Tensor, do_opt: bool, n_stats: int = 0) -> None:
        """One step_batch iteration with no wait, launched eagerly or captured into a graph: gather the pose rows,
        forward, loss, backward summed over the views (and the densification statistics of views 0..n_stats-1),
        scatter dL/dpose into pose_grad, the test hook, and (do_opt) the update, gated on the batch's binning-overflow
        word."""
        L = _lib.lib()
        st = _lib.stream_ptr()
        fr, V = b.frame, b.V
        idx = b.sel[0]
        b.rows.copy_(b.sel[1])
        with torch.no_grad():          # a restored pose table may carry requires_grad from the checkpoint's Parameter
            torch.index_select(self.poses, 0, idx, out=b.poses)
        cam, g, bg = self._camera(), self._gauss(b.poses), self._train_bg(b)
        self._forward(b, cam, g, b.poses, bg)
        b.sums.zero_()
        check(L.gsb_loss_forward_batch(V, 3, self.H, self.W, fr.color.data_ptr(), target.data_ptr(),
                                       b.rows.data_ptr(), b.sums.data_ptr(), b.maps.data_ptr(), st),
              "gsb_loss_forward_batch")
        check(L.gsb_loss_backward_batch(V, 3, self.H, self.W, fr.color.data_ptr(), target.data_ptr(),
                                        b.rows.data_ptr(), b.maps.data_ptr(), float(self.cfg.lambda_dssim),
                                        b.dL.data_ptr(), st), "gsb_loss_backward_batch")
        st = None
        if n_stats > 0:
            st = densify_stats(fr.radii, self._stats[0], self._stats[1], self._stats[2])
        fr.backward_batch(cam, g, b.poses, b.dL, self._grads(), b.dpose, self.filt, st, n_stats, bg)
        self.pose_grad.zero_()
        with torch.no_grad():
            self.pose_grad.index_copy_(0, idx, b.dpose)
        if self._after_backward is not None:
            self._after_backward()
        if do_opt:
            self._launch_adam(1.0 / V, skip_ptr=fr.word(ST_OVERFLOW).data_ptr())

    # ---- densify / prune / opacity reset on the flat buffers (SURVEY.md section 8 row f4) -----------------------
    # Semantics of scene/gaussian_model.py: prune_points (:359-374) keeps the surviving rows of every
    # parameter AND of both Adam moments; densification_postfix (:399-418) appends rows with zero moments;
    # reset_opacity (:280-283) clamps the opacity to 0.01 (in logit space) and zeroes that tensor's moments.  The
    # optimizer's step counter is untouched by all three, as in the reference (state["step"] survives the surgery).
    def _resize(self, new_P: int, rows, stats: Optional[torch.Tensor] = None) -> None:
        """rows(name, old_param_view, old_m_view, old_v_view) -> (param, m, v) tensors of shape [new_P, k].
        stats: the densification statistics [3, new_P] of the new rows (None: zeros, as densification_postfix)."""
        if self._fused:
            raise _lib.GsbError("changing the number of Gaussians is not supported with peer-memory buffers "
                                "(exchange='fused_p2p'); use exchange='allreduce'")
        new = {name: rows(name, self.view(self.params, name), self.view(self.exp_avg, name),
                          self.view(self.exp_avg_sq, name)) for name, _ in self.widths}
        self.P = new_P
        self.segments, total = flat_layout(new_P, self.widths)
        self.total = total
        self.params = torch.zeros(total, dtype=torch.float32, device=self.dev)
        self.grads = torch.zeros(total, dtype=torch.float32, device=self.dev)
        self.exp_avg = torch.zeros(total, dtype=torch.float32, device=self.dev)
        self.exp_avg_sq = torch.zeros(total, dtype=torch.float32, device=self.dev)
        for name, k in self.widths:
            p_, m_, v_ = new[name]
            self.view(self.params, name).copy_(p_.reshape(new_P, k))
            self.view(self.exp_avg, name).copy_(m_.reshape(new_P, k))
            self.view(self.exp_avg_sq, name).copy_(v_.reshape(new_P, k))
        if self._stats is not None:
            self._stats = torch.zeros(3, new_P, dtype=torch.float32, device=self.dev) if stats is None else \
                stats.contiguous()
        self._single = self._Slot(self.dev, new_P, self.W, self.H)   # the next forward sizes its binning buffer
        self._batch = None
        self._batch_sums = None
        self._mip_setup()
        self._keep = None
        self._graphs.clear()

    def _set_per_point_lr(self, values: Optional[torch.Tensor]) -> None:
        """The xyz tensor's per-point learning-rate multiplier [P] (None: off), padded with ones over the xyz
        segment's padded tail."""
        if values is None:
            self.per_point_lr = None
            return
        begin, end = self.segments["xyz"]
        ppl = torch.ones((end - begin) // 3 + 1, dtype=torch.float32, device=self.dev)
        ppl[:self.P] = values.to(self.dev).float().reshape(self.P)
        self.per_point_lr = ppl

    def prune_points(self, mask: torch.Tensor) -> None:
        """Remove the Gaussians where `mask` [P] is True."""
        keep = ~mask.to(self.dev).bool()
        ppl = None if self.per_point_lr is None else self.per_point_lr[:self.P][keep]
        stats = None if self._stats is None else self._stats[:, keep]
        self._resize(int(keep.sum()), lambda name, p, m, v: (p[keep], m[keep], v[keep]), stats)
        self._set_per_point_lr(ppl)

    def densification_postfix(self, new_xyz, new_features_dc, new_features_rest, new_opacities, new_scaling,
                              new_rotation, new_per_point_lr=None) -> None:
        """Append Gaussians; their Adam moments start at zero."""
        ext = dict(xyz=new_xyz, f_dc=new_features_dc, f_rest=new_features_rest, opacity=new_opacities,
                   scaling=new_scaling, rotation=new_rotation)
        n_new = int(new_xyz.shape[0])
        k_of = dict(self.widths)
        ppl = None
        if self.per_point_lr is not None:
            add = torch.ones(n_new, device=self.dev) if new_per_point_lr is None else \
                new_per_point_lr.to(self.dev).float().reshape(n_new)
            ppl = torch.cat((self.per_point_lr[:self.P], add))

        def rows(name, p, m, v):
            e = ext[name].to(self.dev).float().reshape(n_new, k_of[name])
            z = torch.zeros_like(e)
            return torch.cat((p, e)), torch.cat((m, z)), torch.cat((v, z))

        self._resize(self.P + n_new, rows)
        self._set_per_point_lr(ppl)

    def densify_and_prune(self, max_grad, min_opacity, extent, max_screen_size, clone_and_split=False, generator=None):
        """GaussianModel.densify_and_prune on the flat buffers from the accumulated statistics: the rows of
        densify.densify_plan (the mirror's), one rebuild; returns the plan."""
        if self._stats is None:
            raise _lib.GsbError("densify_and_prune needs the densification statistics (OptimConfig.densify=True)")
        v = lambda name: self.view(self.params, name)
        plan = densify_plan(v("xyz"), v("scaling"), v("rotation"), v("opacity"), self.xyz_gradient_accum, self.denom,
                            self.max_radii2D, max_grad, min_opacity, extent, max_screen_size, self.cfg.percent_dense,
                            clone_and_split, generator)
        computed = dict(xyz=plan.split_xyz, scaling=plan.split_scaling)
        ppl = None if self.per_point_lr is None else plan.gather(self.per_point_lr[:self.P])
        stats = None if plan.reset_stats else self._stats[:, plan.src]
        self._resize(plan.P, lambda name, p, m, v_: (plan.gather(p, computed.get(name)), plan.moments(m),
                                                      plan.moments(v_)), stats)
        self._set_per_point_lr(ppl)
        return plan

    def reset_opacity(self) -> None:
        op = self.view(self.params, "opacity")
        cur = torch.sigmoid(op)
        new = torch.min(cur, torch.full_like(cur, 0.01))
        op.copy_(torch.log(new / (1 - new)))
        self.view(self.exp_avg, "opacity").zero_()
        self.view(self.exp_avg_sq, "opacity").zero_()

    # ---- save points (train.py:103-105, :220-227; DESIGN.md section 4.9) ---------------------------------------
    def _shapes(self):
        m1 = self.sh_coeffs - 1
        return dict(xyz=(self.P, 3), f_dc=(self.P, 1, 3), f_rest=(self.P, m1, 3), opacity=(self.P, 1),
                    scaling=(self.P, 3), rotation=(self.P, 4))

    def _group_lrs(self):
        """The `lr` of every param group as the reference's optimizer holds it after update_learning_rate(iteration)
        (before the first iteration: training_setup_pp's initial values)."""
        c = self.cfg
        return [float(lr) for lr in group_lrs(c, c.spatial_lr_scale, self.iteration or None).values()]

    def capture(self):
        """The reference's 13-tuple (GaussianModel.capture) built from the flat buffers: copies, as nn.Parameters on
        this device; a PerPointAdam state dict (seven groups, current LRs, `step` = step_count(name)) that also carries
        what the tuple has no slot for under CHECKPOINT_KEY."""
        if self.world_size > 1:
            raise _lib.GsbError("checkpoints need world_size == 1: the fused exchange shards the Adam moments")
        shapes = self._shapes()
        prm = {name: nn.Parameter(self.view(self.params, name).reshape(shapes[name]).clone()) for name, _ in self.widths}
        pose = nn.Parameter(self.poses.clone())
        groups, state = [], {}
        for i, ((name, _), lr) in enumerate(zip(self.widths + (("pose", 7),), self._group_lrs())):
            ppl = None
            if name == "xyz" and self.per_point_lr is not None:
                ppl = self.per_point_lr[:self.P].reshape(self.P, 1).clone()
            groups.append(dict(lr=lr, betas=ADAM_BETAS, eps=ADAM_EPS, weight_decay=0.0, per_point_lr=ppl, name=name,
                               params=[i]))
            if name == "pose":
                if self.cfg.optim_pose and self.opt_step > 0:
                    state[i] = dict(step=self.opt_step, exp_avg=self.pose_m.clone(), exp_avg_sq=self.pose_v.clone())
            elif self.step_count(name) > 0:
                state[i] = dict(step=self.step_count(name),
                                exp_avg=self.view(self.exp_avg, name).reshape(shapes[name]).clone(),
                                exp_avg_sq=self.view(self.exp_avg_sq, name).reshape(shapes[name]).clone())
        c = self.cfg
        gen = getattr(self, "densify_generator", None)
        extra = dict(
            version=1, iteration=self.iteration, opt_step=self.opt_step, lag=dict(self._lag),
            densify_generator=None if gen is None else gen.get_state(),
            scene_extent=getattr(self, "scene_extent", None),
            filter_3D=None if self.filter_3D is None else self.filter_3D.clone(),
            mip_recomputed_at=list(self.mip_recomputed_at), densified_at=list(self.densified_at),
            reset_at=list(self.reset_at),
            cfg={k: getattr(c, k) for k in dir(OptimConfig) if not k.startswith("_")},
            frame=dict(W=self.W, H=self.H, fovx=self.fovx, fovy=self.fovy,
                       bg=[float(b) for b in self.ident.bg.tolist()], n_views=self.n_views, sh_degree=self.sh_degree))
        if self.background_generator is not None:
            extra["background_generator"] = self.background_generator.get_state()
        sd = {"state": state, "param_groups": groups, CHECKPOINT_KEY: extra}
        if self._stats is not None:
            accum, denom, radii = self.xyz_gradient_accum.clone(), self.denom.clone(), self.max_radii2D.clone()
        else:
            accum = torch.zeros(self.P, 1, device=self.dev)
            denom, radii = torch.zeros_like(accum), torch.zeros(self.P, device=self.dev)
        return (self.active_sh_degree, prm["xyz"], prm["f_dc"], prm["f_rest"], prm["scaling"], prm["rotation"],
                prm["opacity"], radii, accum, denom, sd, float(c.spatial_lr_scale), pose)

    def save_checkpoint(self, path: str) -> None:
        """train.py:225-227: torch.save((capture(), iteration), path).  train.py:104 reads it back unchanged, and so does
        torch.load's default weights_only=True (tensors, nn.Parameter, dicts, lists, tuples and primitives only)."""
        torch.save((self.capture(), self.iteration), path)

    def load_checkpoint(self, path: str) -> None:
        """Continue from a checkpoint: this trainer's frame, views and SH layout, the checkpoint's Gaussians."""
        self.restore(*read_checkpoint(path, self.dev))

    @classmethod
    def from_checkpoint(cls, path: str, scene: Scene, gt_images: Optional[torch.Tensor] = None,
                        cfg: Optional[OptimConfig] = None, device="cuda", use_graph: bool = False) -> "JointTrainer":
        """A trainer that continues the run saved in `path` on `scene`'s views (frame size, intrinsics, background,
        number of views, SH layout; its Gaussians are replaced by the checkpoint's).  cfg=None: the OptimConfig the
        checkpoint was written with (the defaults for a checkpoint without JointTrainer's state)."""
        model_args, first_iter = read_checkpoint(path, torch.device(device))
        if cfg is None:
            cfg = OptimConfig()
            extra = model_args[10].get(CHECKPOINT_KEY) if isinstance(model_args[10], dict) else None
            for k, v in (extra or {}).get("cfg", {}).items():
                if hasattr(OptimConfig, k):
                    setattr(cfg, k, v)
        tr = cls(scene, device, gt_images=gt_images, cfg=cfg, use_graph=use_graph)
        tr.restore(model_args, first_iter)
        return tr

    def restore(self, model_args, first_iter: int) -> None:
        """Load a capture()d tuple (this trainer's or the reference's / mirror's) and continue after iteration
        `first_iter`.  With CHECKPOINT_KEY present the continuation is bit-identical to the run that was not stopped.
        Without it (DESIGN.md section 4.9): opt_step and the lags come from the per-group step counts, the densify
        generator restarts from densify_seed, filter_3D is recomputed from the restored xyz and poses, and the update
        stays PerPointAdam's (the reference's restore switches to torch.optim.Adam)."""
        if self.world_size > 1:
            raise _lib.GsbError("checkpoints need world_size == 1: the fused exchange shards the Adam moments, and "
                                "multi-GPU resume is not implemented")
        t = _parse_capture(model_args, first_iter)
        extra = t["extra"]
        P, n_views = t["P"], t["pose"].shape[0]
        if n_views != self.n_views:
            raise _lib.GsbError(f"checkpoint: the pose table has {n_views} views, the scene {self.n_views}")
        shapes = self._shapes()
        m1 = shapes["f_rest"][1]
        if tuple(t["f_rest"].shape[1:]) != (m1, 3):
            rows = t["f_rest"].shape[1]
            d = int(round((rows + 1) ** 0.5)) - 1
            held = f"SH degree {d}" if (d + 1) ** 2 == rows + 1 else f"{rows} SH rows"
            raise _lib.GsbError(f"checkpoint: f_rest is {tuple(t['f_rest'].shape)}, the trainer's SH layout needs "
                                f"[P,{m1},3]" + ("" if self.stored_sh_degree == 3 else
                                                 f" (the checkpoint holds {held}, the trainer's scene SH degree "
                                                 f"{self.stored_sh_degree}; build the trainer on a scene of the "
                                                 "checkpoint's degree)"))
        if not 0 <= t["active_sh_degree"] <= self.cfg.max_sh_degree:
            raise _lib.GsbError(f"checkpoint: active_sh_degree {t['active_sh_degree']} is out of range")
        if extra is not None:
            fr = extra["frame"]
            mine = dict(W=self.W, H=self.H, fovx=self.fovx, fovy=self.fovy,
                        bg=[float(b) for b in self.ident.bg.tolist()], n_views=self.n_views, sh_degree=self.sh_degree)
            bad = [k for k in mine if fr.get(k) != mine[k]]
            if bad:
                raise _lib.GsbError("checkpoint: written for another frame: " +
                                    ", ".join(f"{k} {fr.get(k)} != {mine[k]}" for k in bad))
        steps = t["steps"]
        if extra is not None:
            opt_step, lag = int(extra["opt_step"]), {name: int(extra["lag"][name]) for name, _ in self.widths}
            want = {name: opt_step - lag[name] for name, _ in self.widths if opt_step - lag[name] > 0}
            if "pose" in steps:
                want["pose"] = opt_step
            if steps != want:
                raise _lib.GsbError(f"checkpoint: step counts {steps} disagree with opt_step {opt_step} and the lags")
        else:
            opt_step = steps.get("pose", 0) or max(steps.get(name, 0) for name, _ in self.widths)
            lag = {name: opt_step - steps.get(name, 0) for name, _ in self.widths}
        dev = self.dev
        self.poses.copy_(t["pose"].to(dev))
        for buf, key in ((self.pose_m, "m"), (self.pose_v, "v")):
            mv = t["moments"].get("pose")
            buf.copy_(mv[key].to(dev)) if mv is not None else buf.zero_()
        stats = None
        if self._stats is not None:
            stats = torch.stack((t["xyz_gradient_accum"].reshape(P), t["denom"].reshape(P),
                                 t["max_radii2D"].reshape(P))).to(dev).float()

        def rows(name, p, m, v):
            k = dict(self.widths)[name]
            new = t[name].detach().to(dev).float().reshape(P, k)
            mv = t["moments"].get(name)
            if mv is None:
                return new, torch.zeros_like(new), torch.zeros_like(new)
            return new, mv["m"].to(dev).float().reshape(P, k), mv["v"].to(dev).float().reshape(P, k)

        self._resize(P, rows, stats)         # also rebuilds the Frame, clears the graphs, recomputes filter_3D
        ppl = t["per_point_lr"]
        self._set_per_point_lr(ppl if self.cfg.pp_optimizer else None)
        self.iteration, self.opt_step, self._lag = int(first_iter), opt_step, lag
        self.active_sh_degree = t["active_sh_degree"]
        self.densified_at, self.reset_at = [], []
        if self.filt is not None:
            self.mip_recomputed_at = []
        if extra is not None:
            self.densified_at, self.reset_at = list(extra["densified_at"]), list(extra["reset_at"])
            if self.filt is not None:
                self.mip_recomputed_at = list(extra["mip_recomputed_at"])
                if extra["filter_3D"] is not None:
                    self.filter_3D.copy_(extra["filter_3D"].to(dev).reshape(P))
        if self._stats is not None:
            if extra is not None and extra["scene_extent"] is not None:
                self.scene_extent = float(extra["scene_extent"])
            gen = None if extra is None else extra["densify_generator"]
            if gen is not None:
                self.densify_generator.set_state(gen.cpu())
            else:
                self.densify_generator.manual_seed(int(self.cfg.densify_seed))
        if self.background_generator is not None:
            gen = None if extra is None else extra.get("background_generator")
            if gen is not None:
                self.background_generator.set_state(gen.cpu())
            else:
                self.background_generator.manual_seed(int(self.cfg.background_seed))

    def save_ply(self, path: str, io: str = "numpy") -> None:
        """scene.save: point_cloud.ply of the current Gaussians (with the filter_3D property when Mip is on).  io
        "numpy": scene_io.save_gaussians_ply of host copies; "gpu": ply.save, records packed straight from the flat
        buffers on the device (the same bytes)."""
        if io == "gpu":
            from . import ply
            t = {name: self.view(self.params, name) for name, _ in self.widths}
            ply.save(path, dict(t, filter_3D=self.filter_3D))
            return
        if io != "numpy":
            raise ValueError(f"save_ply: io must be 'numpy' or 'gpu', got {io!r}")
        from .scene_io import save_gaussians_ply
        v = lambda name: self.view(self.params, name).cpu().numpy()
        save_gaussians_ply(path, v("xyz"), v("f_dc"), v("f_rest"), v("opacity"), v("scaling"), v("rotation"),
                           None if self.filter_3D is None else self.filter_3D.cpu().numpy())

    def ply_tensors(self) -> Dict[str, torch.Tensor]:
        """The Gaussians save_ply writes, as scene_io.load_gaussians_ply reads them back, without the file: device
        copies (not views of the flat buffers) xyz [P,3], f_dc [P,1,3], f_rest [P,M-1,3] at the stored SH degree,
        opacity [P,1], scaling [P,3], rotation [P,4]; and filter_3D [P,1] when Mip is on."""
        P, w = self.P, dict(self.widths)
        v = lambda name, *shape: self.view(self.params, name).reshape(P, *shape).clone()
        out = dict(xyz=v("xyz", 3), f_dc=v("f_dc", 1, 3), f_rest=v("f_rest", w["f_rest"] // 3, 3),
                   opacity=v("opacity", 1), scaling=v("scaling", 3), rotation=v("rotation", 4))
        if self.filter_3D is not None:
            out["filter_3D"] = self.filter_3D.reshape(P, 1).clone()
        return out

    def save_poses(self, path: str, colmap_ids: Optional[List[int]] = None):
        """train.py save_pose: the pose table as [n_views,4,4] world-to-camera matrices in COLMAP id order."""
        from .scene_io import save_pose_npy
        return save_pose_npy(path, self.poses.detach().cpu().numpy(), colmap_ids)

    def blend_stats(self, view: int, gt: Optional[torch.Tensor] = None) -> Dict[str, int]:
        """Pair statistics of the blend kernels for one forward+backward of `view` (instrumented re-run of the same
        kernels, outside any timed region): evaluated / contributing (pixel, Gaussian) pairs."""
        self.render(view)
        self.loss_and_backward(view, self.gt[view] if gt is None else gt)
        cam, _ = self._keep
        stats = torch.zeros(8, dtype=torch.int64, device=self.dev)
        self.frame.blend_stats(cam, self.dL_dimg, stats)
        s = stats.cpu().tolist()
        return dict(instances=self.last_R, fwd_warp_iters=s[0], fwd_pairs_evaluated=64 * s[0], fwd_pairs_contributing=s[1],
                    bwd_warp_iters=s[2], bwd_pairs_evaluated=64 * s[2], bwd_pairs_contributing=s[3],
                    bwd_warp_iters_reduced=s[4])

    # ------------------------------------------------------------------------------------------
    def algorithmic_bytes(self) -> Dict[str, float]:
        """SURVEY.md section 8(d) per-kernel algorithmic HBM bytes for the last step (fp32)."""
        P, R, HW = self.P, self.last_R, self.W * self.H
        T = ((self.W + 15) // 16) * ((self.H + 15) // 16)
        K = (min(self.sh_degree, self.stored_sh_degree) + 1) ** 2
        F = sum(k for _, k in self.widths)          # floats per Gaussian in each flat buffer: 14 / 23 / 38 / 59 at D = 0..3
        V = P
        return dict(
            preprocess_fwd=P * (12 + 12 + 16 + 4) + V * 12 * K + V * (8 + 4 + 16 + 12 + 4) + P * 4,
            blend_fwd=R * 40 + HW * 20 + T * 8,
            blend_bwd=R * 40 + HW * 20 + T * 8 + V * 36,
            preprocess_bwd=P * 44 + V * (12 * K + 36) + P * 44 + V * 12 * K,
            loss=HW * 36,
            adam=F * P * 28 + P * 4,
        )


# ---- checkpoint files (DESIGN.md section 4.9) ----------------------------------------------------------------------
# The top-level key of the optimizer state dict under which JointTrainer stores what the reference tuple has no slot for;
# torch.optim.Optimizer.load_state_dict reads only "state" and "param_groups", so the reference's restore() ignores it.
CHECKPOINT_KEY = "joint_trainer"
_GROUP_NAMES = tuple(name for name, _ in SEGMENTS) + ("pose",)
_EXTRA_KEYS = ("iteration", "opt_step", "lag", "densify_generator", "scene_extent", "filter_3D", "mip_recomputed_at",
               "densified_at", "reset_at", "cfg", "frame")
# ... and, from a run with random_background, "background_generator": the state of the colours' generator.  Optional: a
# file without it (any other run's) continues the colours from background_seed.


def read_checkpoint(path: str, device=None):
    """(model_args, first_iter) of a train.py checkpoint, with torch.load's default weights_only=True.  The reference's
    (and the mirror's) state dicts hold the scheduled learning rates as numpy float64 scalars, so those two numpy globals
    are allowed as well; JointTrainer writes Python floats."""
    mod = getattr(np, "_core", None) or np.core
    with torch.serialization.safe_globals([mod.multiarray.scalar, np.dtype, type(np.dtype(np.float64))]):
        obj = torch.load(path, map_location=device)
    if not (isinstance(obj, (tuple, list)) and len(obj) == 2):
        raise _lib.GsbError(f"checkpoint {path}: expected (model_params, first_iter), got {type(obj).__name__}")
    return obj[0], obj[1]


def _parse_capture(model_args, first_iter) -> dict:
    """Check a GaussianModel.capture() tuple entry by entry; returns its parts by name, the moments and step count of
    every param group by group name, and the extra state (None when absent)."""
    def bad(msg):
        raise _lib.GsbError("checkpoint: " + msg)

    if not (isinstance(model_args, (tuple, list)) and len(model_args) == 13):
        bad("model_params must be GaussianModel.capture()'s 13-tuple")
    if isinstance(first_iter, bool) or not isinstance(first_iter, int) or first_iter < 0:
        bad(f"first_iter must be a non-negative int, got {first_iter!r}")
    names = ("active_sh_degree", "xyz", "f_dc", "f_rest", "scaling", "rotation", "opacity", "max_radii2D",
             "xyz_gradient_accum", "denom", "optimizer", "spatial_lr_scale", "pose")
    t = dict(zip(names, model_args))
    if isinstance(t["active_sh_degree"], bool) or not isinstance(t["active_sh_degree"], int):
        bad("active_sh_degree must be an int")
    for k in names[1:10] + ("pose",):
        if not torch.is_tensor(t[k]):
            bad(f"{k} must be a tensor, got {type(t[k]).__name__}")
    P = int(t["xyz"].shape[0]) if t["xyz"].dim() == 2 else -1
    want = dict(xyz=(P, 3), f_dc=(P, 1, 3), scaling=(P, 3), rotation=(P, 4), opacity=(P, 1), max_radii2D=(P,),
                xyz_gradient_accum=(P, 1), denom=(P, 1))
    for k, s in want.items():
        if tuple(t[k].shape) != s:
            bad(f"{k} has shape {tuple(t[k].shape)}, expected {s}")
    if t["f_rest"].dim() != 3 or t["f_rest"].shape[0] != P or t["f_rest"].shape[2] != 3:
        bad(f"f_rest has shape {tuple(t['f_rest'].shape)}, expected [P,M-1,3]")
    if t["pose"].dim() != 2 or t["pose"].shape[1] != 7:
        bad(f"the pose table has shape {tuple(t['pose'].shape)}, expected [n_views,7]")
    sd = t["optimizer"]
    if not (isinstance(sd, dict) and isinstance(sd.get("state"), dict) and isinstance(sd.get("param_groups"), list)):
        bad("the optimizer state dict needs 'state' and 'param_groups'")
    groups = {}
    for g in sd["param_groups"]:
        if not (isinstance(g, dict) and g.get("name") in _GROUP_NAMES and len(g.get("params", ())) == 1):
            bad(f"unexpected param group {g.get('name') if isinstance(g, dict) else g!r}")
        groups[g["name"]] = g
    if sorted(groups) != sorted(_GROUP_NAMES) or len(sd["param_groups"]) != len(_GROUP_NAMES):
        bad(f"param groups {[g.get('name') for g in sd['param_groups']]}, expected {list(_GROUP_NAMES)}")
    steps, moments = {}, {}
    for name, g in groups.items():
        st = sd["state"].get(g["params"][0])
        if not st:
            continue
        shape = tuple(t[name].shape)
        if not all(k in st for k in ("step", "exp_avg", "exp_avg_sq")) or \
                any(not torch.is_tensor(st[k]) or tuple(st[k].shape) != shape for k in ("exp_avg", "exp_avg_sq")):
            bad(f"the optimizer state of '{name}' needs step, exp_avg and exp_avg_sq of shape {shape}")
        steps[name] = int(float(st["step"]))
        moments[name] = dict(m=st["exp_avg"], v=st["exp_avg_sq"])
    ppl = groups["xyz"].get("per_point_lr")
    if ppl is not None and not (torch.is_tensor(ppl) and ppl.numel() == P):
        bad("the xyz group's per_point_lr must be a tensor with one value per Gaussian")
    extra = sd.get(CHECKPOINT_KEY)
    if extra is not None:
        missing = [k for k in _EXTRA_KEYS if k not in extra] if isinstance(extra, dict) else list(_EXTRA_KEYS)
        if missing:
            bad(f"'{CHECKPOINT_KEY}' lacks {missing}")
        if int(extra["iteration"]) != first_iter:
            bad(f"first_iter {first_iter} differs from the saved iteration {extra['iteration']}")
        if extra["filter_3D"] is not None and extra["filter_3D"].numel() != P:
            bad("filter_3D must have one value per Gaussian")
        bg_gen = extra.get("background_generator")
        if bg_gen is not None and not (torch.is_tensor(bg_gen) and bg_gen.dtype == torch.uint8):
            bad("background_generator must be a generator state (a uint8 tensor)")
    t.update(P=P, steps=steps, moments=moments, extra=extra, per_point_lr=None if ppl is None else ppl.reshape(P))
    return t
