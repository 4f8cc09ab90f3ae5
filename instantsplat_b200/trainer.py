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
"""
from __future__ import annotations

from typing import Dict, List, Optional

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

SEGMENTS = (("xyz", 3), ("f_dc", 3), ("f_rest", 45), ("opacity", 1), ("scaling", 3), ("rotation", 4))


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


def L_sig_words():
    return (_lib.lib().gsb_peer_signal_bytes() + 3) // 4


def _align(n, a=64):
    return (n + a - 1) // a * a


class JointTrainer:
    def __init__(self, scene: Scene, device, gt_images: Optional[torch.Tensor] = None,
                 cfg: Optional[OptimConfig] = None, world_size: int = 1, rank: int = 0,
                 process_group=None, exchange: str = "allreduce", use_graph: bool = False):
        self.cfg = cfg or OptimConfig()
        if self.cfg.densify and world_size > 1:
            raise _lib.GsbError("densify=True needs world_size == 1: every rank would accumulate different "
                                "densification statistics")
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
        # ---- flat buffers
        offs, total = {}, 0
        for name, k in SEGMENTS:
            offs[name] = total
            total += _align(P * k)
        self.offs, self.total = offs, total
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
        for name, k in SEGMENTS:
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
        self.per_point_lr = None
        if self.cfg.pp_optimizer and scene.per_point_lr is not None:
            ppl = torch.ones(_align(P * 3) // 3 + 1, dtype=torch.float32, device=self.dev)   # covers the padded tail
            ppl[:P] = scene.per_point_lr.to(self.dev).float().reshape(P)
            self.per_point_lr = ppl
        self.gt = None if gt_images is None else gt_images.to(self.dev).float().contiguous()
        self.ident = IdentityView(self.W, self.H, scene.fovx, scene.fovy, scene.bg, self.dev)
        self.frame = Frame(self.dev, P, self.W, self.H)     # scratch; its binning buffer is sized by the first forward
        self.headroom = 1.5
        self.filter_3D, self.filt, self.mip_recomputed_at = None, None, []
        self._mip_setup()
        self.dL_dimg = torch.empty_like(self.color)
        self.maps = torch.empty(3, 3, self.H, self.W, dtype=torch.float32, device=self.dev)
        self.sums = torch.zeros(2, dtype=torch.float64, device=self.dev)
        self.host_status = torch.zeros(2, ST_WORDS, dtype=torch.int32).pin_memory()   # [0] after preprocess, [1] after render
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
        self._step_host = torch.zeros(8, dtype=torch.float32).pin_memory()
        self._step_dev = torch.zeros(8, dtype=torch.float32, device=self.dev)
        self.frame.status.zero_()     # the forward serial number lives in these words
        self._fwd_count = 0
        self._polling = False
        self.iteration = 0            # reference iterations = views consumed (by all ranks)
        self.opt_step = 0
        self.last_R = 0
        self.overflows = 0
        self.exact_cull = True
        self.active_sh_degree = min(scene.sh_degree, self.cfg.max_sh_degree)
        c = self.cfg
        self.xyz_sched = get_expon_lr_func(c.position_lr_init * c.spatial_lr_scale,
                                           c.position_lr_final * c.spatial_lr_scale,
                                           lr_delay_mult=c.position_lr_delay_mult,
                                           max_steps=c.position_lr_max_steps)
        self.cam_sched = get_expon_lr_func(c.rotation_lr * 0.1, c.rotation_lr * 0.001,
                                           lr_delay_mult=c.position_lr_delay_mult, max_steps=c.iterations)
        self._keep = None
        # per-tensor Adam step counts are opt_step minus the optimizer steps that skipped the tensor (the densify and
        # opacity-reset iterations replace tensors, which then have no gradient in the reference)
        self._lag = {name: 0 for name, _ in SEGMENTS}
        self._stats = None
        if c.densify:
            self._stats = torch.zeros(3, P, dtype=torch.float32, device=self.dev)
            self.scene_extent = cameras_extent(scene.poses) if c.scene_extent is None else float(c.scene_extent)
            self.densify_generator = torch.Generator(device=self.dev).manual_seed(int(c.densify_seed))
            self.white_background = bool((scene.bg == 1).all())
        self.densified_at, self.reset_at = [], []

    # ------------------------------------------------------------------------------------------
    def view(self, flat: torch.Tensor, name: str) -> torch.Tensor:
        k = dict(SEGMENTS)[name]
        o = self.offs[name]
        return flat[o:o + self.P * k].view(self.P, k)

    def my_views(self) -> List[int]:
        from .parallel import shard_views
        return shard_views(self.n_views, self.world_size, self.rank)

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
        """Adam step count of one tensor ("pose" or a SEGMENTS name)."""
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

    def _gauss(self, view: int) -> GsbGaussians:
        p = self.params
        return gaussians(self.P, *(self.view(p, n) for n in ("xyz", "rotation", "scaling", "opacity", "f_dc", "f_rest")),
                         self.poses[view])

    # ------------------------------------------------------------------------------------------
    def _size_binning(self, R: int) -> None:
        self.frame.alloc_binning(capacity(R, self.headroom))

    def _launch_forward(self, view: int) -> None:
        """Enqueue the forward without ever waiting for the GPU: the instance count R stays on the device; the
        host only provides a capacity (sized from the counts seen so far, +50 %) and reads R back lazily."""
        cam, g = self.ident.camera(self.active_sh_degree, 16, self.exact_cull), self._gauss(view)
        capturing = torch.cuda.is_current_stream_capturing()
        self.frame.preprocess(cam, g, self.host_status[0], self.filt)
        if not capturing:
            self._fwd_count += 1
            self._polling = False
            self._ev_pre.record()
            if self.cap == 0:                         # very first forward: size the buffer from the real count
                self._ev_pre.synchronize()
                self._size_binning(read_R(self.host_status[0]))
        self.frame.render(cam, self.host_status[1])
        self._keep = (cam, g)

    def _settle(self) -> bool:
        """Wait for the status words of the last forward's preprocess phase (early in the stream: the GPU still has
        the rest of the iteration queued, so this never starves it).  Returns True if the binning buffer was big
        enough; otherwise grows it (the device skipped the optimizer update by itself) and returns False."""
        if self._polling:
            # graph replay: no host-visible event inside the graph, so watch the pinned status words for this forward's
            # serial number (written by the tile scan, copied by the memcpy node right behind it)
            want = self._fwd_count & 0x7FFFFFFF
            hs = self.host_status
            n = 0
            while (int(hs[0, ST_SEQ]) & 0x7FFFFFFF) != want:
                n += 1
                if n > 20_000_000:
                    raise _lib.GsbError("graph replay: the forward's status words never arrived")
        else:
            self._ev_pre.synchronize()
        R = read_R(self.host_status[0])
        self.last_R = R
        if R > self.cap:
            self.overflows += 1
            self._size_binning(R)
            return False
        if R > 0.85 * self.cap:                        # grow ahead of need
            self._size_binning(R)
        return True

    def render(self, view: int) -> torch.Tensor:
        """Forward only (exact: repeated with a larger buffer in the unlikely case the capacity was exceeded)."""
        self._launch_forward(view)
        if not self._settle():
            self._launch_forward(view)
            assert self._settle()
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
        gr = GsbGrads()
        gd = self.grads
        gr.dL_dmeans3D = self.view(gd, "xyz").data_ptr()
        gr.dL_dscales = self.view(gd, "scaling").data_ptr()
        gr.dL_drotations = self.view(gd, "rotation").data_ptr()
        gr.dL_dopacities = self.view(gd, "opacity").data_ptr()
        gr.dL_dsh_dc = self.view(gd, "f_dc").data_ptr()
        gr.dL_dsh_rest = self.view(gd, "f_rest").data_ptr()
        self.pose_grad.zero_()
        gr.dL_dpose = self.pose_grad[view].data_ptr()
        st = None
        if stats:
            st = densify_stats(self.frame.radii, self._stats[0], self._stats[1], self._stats[2])
        self.frame.backward(cam, g, self.dL_dimg, gr, self.filt, st)

    def loss_value(self) -> torch.Tensor:
        n = 3 * self.H * self.W
        lam = self.cfg.lambda_dssim
        return (1.0 - lam) * self.sums[0] / n + lam * (1.0 - self.sums[1] / n)

    def reduce_grads(self) -> None:
        if self.world_size > 1:
            from .parallel import allreduce_sum_
            self._pg_buf[-1:].copy_(self.frame.word(ST_OVERFLOW))
            allreduce_sum_((self.grads, self._pg_buf), self.pg)

    def _step_sizes(self):
        """lr * sqrt(1-b2^t)/(1-b1^t) per tensor for the current counters (host, double)."""
        c = self.cfg
        t = max(1, self.opt_step)
        corr = (1 - 0.999 ** t) ** 0.5 / (1 - 0.9 ** t)
        lrs = self._lrs()
        out = [lrs[name] * self._corr(max(1, self.step_count(name))) for name, _ in SEGMENTS]
        if c.optim_pose:
            out.append(self.cam_sched(self.iteration) * corr)
        return out

    def _upload_step_sizes(self) -> None:
        ss = self._step_sizes()
        for i, v in enumerate(ss):
            self._step_host[i] = v
        self._step_dev.copy_(self._step_host, non_blocking=True)

    @staticmethod
    def _corr(t: int) -> float:
        return (1 - 0.999 ** t) ** 0.5 / (1 - 0.9 ** t)

    def optimizer_step(self, grad_scale: Optional[float] = None, _advance: bool = True, _dev_steps: bool = False,
                       skip=()) -> None:
        """PerPointAdam.step over the 6 Gaussian tensors + the pose table in one launch
        (param groups and LRs of scene/gaussian_model.py:203-243).  skip: Gaussian tensors that take no step (they
        were replaced in this iteration, so the reference's parameter has no gradient); their step counts stay."""
        c = self.cfg
        if _advance:
            self.opt_step += 1
        for name in skip:
            self._lag[name] += 1
        t = self.opt_step
        b1, b2, eps = 0.9, 0.999, 1e-15
        corr = (1 - b2 ** t) ** 0.5 / (1 - b1 ** t)
        lrs = dict(xyz=self.xyz_sched(self.iteration), f_dc=c.feature_lr * 10, f_rest=c.feature_lr / 20.0 * 10,
                   opacity=c.opacity_lr, scaling=c.scaling_lr * 10, rotation=c.rotation_lr * 10)
        gs = 1.0 / self.world_size if grad_scale is None else grad_scale
        entries = []
        for name, k in SEGMENTS:
            if name in skip:
                continue
            entries.append(dict(param=self.view(self.params, name), grad=self.view(self.grads, name),
                                exp_avg=self.view(self.exp_avg, name), exp_avg_sq=self.view(self.exp_avg_sq, name),
                                per_point_lr=self.per_point_lr if name == "xyz" else None, row_len=k,
                                step_size=lrs[name] * self._corr(self.step_count(name)), beta1=b1, beta2=b2, eps=eps,
                                weight_decay=0.0, grad_scale=gs))
        if c.optim_pose:
            entries.append(dict(param=self.poses, grad=self.pose_grad, exp_avg=self.pose_m, exp_avg_sq=self.pose_v,
                                per_point_lr=None, row_len=7, step_size=self.cam_sched(self.iteration) * corr,
                                beta1=b1, beta2=b2, eps=eps, weight_decay=0.0, grad_scale=gs))
        launch_adam(entries, self.flags, skip_ptr=self._skip_ptr(), step_sizes_dev=self._step_dev if _dev_steps else None)

    def _skip_ptr(self):
        """Device word that makes the optimizer kernels skip the update: the forward's overflow status
        (multi-GPU: its sum over ranks, so that every replica takes the same decision)."""
        if self.world_size > 1:
            return self._ovf.data_ptr()
        return self.frame.word(ST_OVERFLOW).data_ptr()

    def _lrs(self):
        c = self.cfg
        return dict(xyz=self.xyz_sched(self.iteration), f_dc=c.feature_lr * 10, f_rest=c.feature_lr / 20.0 * 10,
                    opacity=c.opacity_lr, scaling=c.scaling_lr * 10, rotation=c.rotation_lr * 10)

    def fused_exchange_step(self, _advance: bool = True, _dev_steps: bool = False) -> None:
        """Multi-GPU: gate flags + pose gradients summed over the ranks (one tiny kernel over peer memory, or a tiny
        NCCL all-reduce; either doubles as the pre-barrier), then ONE kernel per rank doing reduce-scatter ->
        per-point Adam -> all-gather over NVLink peer memory (csrc/gs_comm.cu), then a barrier before anyone reads
        the new parameters.  _dev_steps: the kernels read their Adam step sizes from self._step_dev (graph replay)."""
        import torch.distributed as dist
        from ._lib import GsbAdamTensor, GsbShardPiece
        L = _lib.lib()
        st = _lib.stream_ptr()
        c = self.cfg
        if _advance:
            self.opt_step += 1
        t = self.opt_step
        step_dev = self._step_dev if _dev_steps else None
        b1, b2, eps = 0.9, 0.999, 1e-15
        corr = (1 - b2 ** t) ** 0.5 / (1 - b1 ** t)
        lrs = self._lrs()
        # 1. whole-tensor gates on the local gradients, OR-ed across ranks
        arr = (GsbAdamTensor * len(SEGMENTS))()
        for a, (name, k) in zip(arr, SEGMENTS):
            g = self.view(self.grads, name)
            a.param = a.exp_avg = a.exp_avg_sq = a.grad = g.data_ptr()
            a.numel, a.row_len, a.grad_scale = g.numel(), k, 1.0
            a.step_size, a.beta1, a.beta2, a.eps, a.weight_decay = 0.0, b1, b2, eps, 0.0
        check(L.gsb_adam_gate(len(SEGMENTS), arr, self.flags.data_ptr(), st), "gsb_adam_gate")
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
        # 2. the fused kernel over this rank's shard
        lo, hi = self.shard
        pieces = []
        for fi, (name, k) in enumerate(SEGMENTS):
            s0 = self.offs[name]
            s1 = s0 + _align(self.P * k)
            b, e = max(lo, s0), min(hi, s1)
            if e > b:
                pc = GsbShardPiece()
                pc.begin, pc.end, pc.seg_begin = b, e, s0
                pc.per_point_lr = self.per_point_lr.data_ptr() if (name == "xyz" and self.per_point_lr is not None) else None
                pc.row_len, pc.flag_index = k, fi
                pc.step_size, pc.beta1, pc.beta2, pc.eps = lrs[name] * corr, b1, b2, eps
                pieces.append(pc)
        parr = (GsbShardPiece * max(1, len(pieces)))(*pieces)
        check(L.gsb_fused_rs_adam_ag(self.world_size, self.rank, self._peer_grads.ptr_array(),
                                     self._peer_params.ptr_array(), self.exp_avg.data_ptr(),
                                     self.exp_avg_sq.data_ptr(), lo, len(pieces), parr, self.flags.data_ptr(),
                                     self._ovf.data_ptr(), 1.0 / self.world_size,
                                     None if step_dev is None else step_dev.data_ptr(), st), "gsb_fused_rs_adam_ag")
        # 3. pose table: replicated Adam on the all-reduced pose gradients
        if c.optim_pose:
            launch_adam([dict(param=self.poses, grad=self.pose_grad, exp_avg=self.pose_m, exp_avg_sq=self.pose_v,
                              per_point_lr=None, row_len=7, step_size=self.cam_sched(self.iteration) * corr,
                              beta1=b1, beta2=b2, eps=eps, weight_decay=0.0, grad_scale=1.0 / self.world_size)],
                        self._pose_flags, skip_ptr=self._ovf.data_ptr(),
                        step_sizes_dev=None if step_dev is None else step_dev[len(SEGMENTS):])
        # 4. nobody may start the next forward before every rank's parameter stores have landed
        if self.exchange == "fused_p2p":
            check(L.gsb_peer_barrier(self.world_size, self.rank, self._peer_sig.ptr_array(), 0, 1, st),
                  "gsb_peer_barrier")
        else:
            dist.all_reduce(self._sync, group=self.pg)

    def _graph_iteration(self, view: int, gt: torch.Tensor, do_opt: bool, stats: bool = False) -> None:
        """Replay (capturing on first use) the CUDA graph of one iteration on `view`."""
        if do_opt:
            self.opt_step += 1
            self._upload_step_sizes()                    # stream-ordered before the replay
        for _attempt in range(2):
            key = (view, gt.data_ptr(), do_opt, self.active_sh_degree, self.cap, self.exact_cull, stats)
            g = self._graphs.get(key)
            if g is None:
                if len(self._graphs) > 64:
                    self._graphs.clear()
                torch.cuda.synchronize()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    self._launch_forward(view)
                    self.loss_and_backward(view, gt, stats)
                    if self._after_backward is not None:
                        self._after_backward()
                    if do_opt and self._fused:
                        self.fused_exchange_step(_advance=False, _dev_steps=True)
                    elif do_opt:
                        self.optimizer_step(_advance=False, _dev_steps=True)
                self._graphs[key] = g
            self._fwd_count += 1
            self._polling = True
            g.replay()
            if self._settle():
                return
            if self.world_size > 1:
                raise _lib.GsbError(f"rank {self.rank}: {self.last_R} instances exceeded the binning capacity; the "
                                    "optimizer update of this step was skipped on every rank (parameters are "
                                    "consistent).  Raise JointTrainer.headroom.")
            # capacity exceeded: the device skipped the update, the buffer has been enlarged -> new graph, once more
        raise _lib.GsbError("graph replay: binning capacity exceeded twice in a row")

    def _run_iteration(self, view: int, gt: torch.Tensor, do_opt: bool, stats: bool = False) -> None:
        self._launch_forward(view)
        self.loss_and_backward(view, gt, stats)
        if self._after_backward is not None:
            self._after_backward()
        if not do_opt:
            return
        if self._fused:
            self.fused_exchange_step()
        else:
            self.reduce_grads()
            self.optimizer_step()

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
        steps.  Nothing in here waits for the GPU except `_settle()`, which waits for an event early in the stream."""
        c = self.cfg
        before = self.iteration
        self.iteration += self.world_size
        if self.iteration // c.sh_increase_interval > before // c.sh_increase_interval:
            self.active_sh_degree = min(self.active_sh_degree + 1, c.max_sh_degree)     # oneupSHdegree
        if gt is None:
            gt = self.gt[view]
        do_opt = self.iteration < c.iterations
        it = self.iteration
        stats = self._stats is not None and it < c.densify_until_iter
        densify_now = stats and it > c.densify_from_iter and it % c.densification_interval == 0
        reset_now = stats and (it % c.opacity_reset_interval == 0 or
                               (self.white_background and it == c.densify_from_iter))
        if densify_now or reset_now:
            # train.py:201-211: densify / reset between the backward and the optimizer step, eagerly (the optimizer's
            # tensor set differs); the replaced tensors take no step in this iteration
            self._run_iteration_settled(view, gt, False, stats)
            skip = set()
            if densify_now:
                size = c.size_threshold if it > c.opacity_reset_interval else None
                self.densify_and_prune(c.densify_grad_threshold, c.min_opacity, self.scene_extent, size,
                                       c.densify_clone_split, self.densify_generator)
                self.densified_at.append(it)
                skip.update(name for name, _ in SEGMENTS)
            if reset_now:
                self.reset_opacity()
                self.reset_at.append(it)
                skip.add("opacity")
            if do_opt:
                self.optimizer_step(skip=[name for name, _ in SEGMENTS if name in skip])
        elif self.use_graph and self.cap > 0:
            self._graph_iteration(view, gt, do_opt, stats)
        else:
            self._run_iteration_settled(view, gt, do_opt, stats)
        # crossing a multiple of the interval (with G ranks `iteration` advances by G per step)
        if self.filt is not None and self.iteration // c.mip_filter3d_interval > before // c.mip_filter3d_interval and \
                self.iteration < c.iterations - 100:
            self.compute_filter_3D()
            self.mip_recomputed_at.append(self.iteration)

    def _run_iteration_settled(self, view: int, gt: torch.Tensor, do_opt: bool, stats: bool = False) -> None:
        self._run_iteration(view, gt, do_opt, stats)
        if not self._settle():
            # The binning capacity was exceeded: the device skipped the update by itself (gated on the overflow word,
            # summed over ranks in multi-GPU mode), so parameters and moments are untouched.  Single GPU: repeat the
            # iteration with the larger buffer.  Multi GPU: the other ranks cannot know yet -- stop loudly.
            if self.world_size > 1:
                raise _lib.GsbError(f"rank {self.rank}: {self.last_R} instances exceeded the binning capacity; the "
                                    "optimizer update of this step was skipped on every rank (parameters are "
                                    "consistent).  Raise JointTrainer.headroom.")
            if do_opt:
                self.opt_step -= 1
            self._run_iteration(view, gt, do_opt, stats)
            assert self._settle()

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
                          self.view(self.exp_avg_sq, name)) for name, _ in SEGMENTS}
        offs, total = {}, 0
        for name, k in SEGMENTS:
            offs[name] = total
            total += _align(new_P * k)
        self.P, self.offs, self.total = new_P, offs, total
        self.params = torch.zeros(total, dtype=torch.float32, device=self.dev)
        self.grads = torch.zeros(total, dtype=torch.float32, device=self.dev)
        self.exp_avg = torch.zeros(total, dtype=torch.float32, device=self.dev)
        self.exp_avg_sq = torch.zeros(total, dtype=torch.float32, device=self.dev)
        for name, k in SEGMENTS:
            p_, m_, v_ = new[name]
            self.view(self.params, name).copy_(p_.reshape(new_P, k))
            self.view(self.exp_avg, name).copy_(m_.reshape(new_P, k))
            self.view(self.exp_avg_sq, name).copy_(v_.reshape(new_P, k))
        if self._stats is not None:
            self._stats = torch.zeros(3, new_P, dtype=torch.float32, device=self.dev) if stats is None else \
                stats.contiguous()
        self.frame = Frame(self.dev, new_P, self.W, self.H)   # the next forward sizes its binning buffer
        self._mip_setup()
        self._keep = None
        self._graphs.clear()
        self.frame.status.zero_()
        self._fwd_count = 0

    def _set_per_point_lr(self, values: Optional[torch.Tensor]) -> None:
        if values is None:
            self.per_point_lr = None
            return
        ppl = torch.ones(_align(self.P * 3) // 3 + 1, dtype=torch.float32, device=self.dev)
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
        k_of = dict(SEGMENTS)
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
        m1 = dict(SEGMENTS)["f_rest"] // 3
        return dict(xyz=(self.P, 3), f_dc=(self.P, 1, 3), f_rest=(self.P, m1, 3), opacity=(self.P, 1),
                    scaling=(self.P, 3), rotation=(self.P, 4))

    def _group_lrs(self):
        """The `lr` of every param group as the reference's optimizer holds it after update_learning_rate(iteration)
        (before the first iteration: training_setup_pp's initial values)."""
        c = self.cfg
        lrs = self._lrs()
        if self.iteration == 0:
            lrs["xyz"], pose = c.position_lr_init * c.spatial_lr_scale, c.rotation_lr * 0.1
        else:
            pose = self.cam_sched(self.iteration)
        return [float(lrs[name]) for name, _ in SEGMENTS] + [float(pose)]

    def capture(self):
        """The reference's 13-tuple (GaussianModel.capture) built from the flat buffers: copies, as nn.Parameters on
        this device; a PerPointAdam state dict (seven groups, current LRs, `step` = step_count(name)) that also carries
        what the tuple has no slot for under CHECKPOINT_KEY."""
        if self.world_size > 1:
            raise _lib.GsbError("checkpoints need world_size == 1: the fused exchange shards the Adam moments")
        shapes = self._shapes()
        prm = {name: nn.Parameter(self.view(self.params, name).reshape(shapes[name]).clone()) for name, _ in SEGMENTS}
        pose = nn.Parameter(self.poses.clone())
        groups, state = [], {}
        for i, ((name, _), lr) in enumerate(zip(SEGMENTS + (("pose", 7),), self._group_lrs())):
            ppl = None
            if name == "xyz" and self.per_point_lr is not None:
                ppl = self.per_point_lr[:self.P].reshape(self.P, 1).clone()
            groups.append(dict(lr=lr, betas=(0.9, 0.999), eps=1e-15, weight_decay=0.0, per_point_lr=ppl, name=name,
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
            raise _lib.GsbError(f"checkpoint: f_rest is {tuple(t['f_rest'].shape)}, the trainer's SH layout needs "
                                f"[P,{m1},3]")
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
            opt_step, lag = int(extra["opt_step"]), {name: int(extra["lag"][name]) for name, _ in SEGMENTS}
            want = {name: opt_step - lag[name] for name, _ in SEGMENTS if opt_step - lag[name] > 0}
            if "pose" in steps:
                want["pose"] = opt_step
            if steps != want:
                raise _lib.GsbError(f"checkpoint: step counts {steps} disagree with opt_step {opt_step} and the lags")
        else:
            opt_step = steps.get("pose", 0) or max(steps.get(name, 0) for name, _ in SEGMENTS)
            lag = {name: opt_step - steps.get(name, 0) for name, _ in SEGMENTS}
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
            k = dict(SEGMENTS)[name]
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

    def save_ply(self, path: str) -> None:
        """scene.save: point_cloud.ply of the current Gaussians (with the filter_3D property when Mip is on)."""
        from .scene_io import save_gaussians_ply
        v = lambda name: self.view(self.params, name).cpu().numpy()
        save_gaussians_ply(path, v("xyz"), v("f_dc"), v("f_rest"), v("opacity"), v("scaling"), v("rotation"),
                           None if self.filter_3D is None else self.filter_3D.cpu().numpy())

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
        K = (self.sh_degree + 1) ** 2
        V = P
        return dict(
            preprocess_fwd=P * (12 + 12 + 16 + 4) + V * 12 * K + V * (8 + 4 + 16 + 12 + 4) + P * 4,
            blend_fwd=R * 40 + HW * 20 + T * 8,
            blend_bwd=R * 40 + HW * 20 + T * 8 + V * 36,
            preprocess_bwd=P * 44 + V * (12 * K + 36) + P * 44 + V * 12 * K,
            loss=HW * 36,
            adam=59 * P * 28 + P * 4,
        )


# ---- checkpoint files (DESIGN.md section 4.9) ----------------------------------------------------------------------
# The top-level key of the optimizer state dict under which JointTrainer stores what the reference tuple has no slot for;
# torch.optim.Optimizer.load_state_dict reads only "state" and "param_groups", so the reference's restore() ignores it.
CHECKPOINT_KEY = "joint_trainer"
_GROUP_NAMES = tuple(name for name, _ in SEGMENTS) + ("pose",)
_EXTRA_KEYS = ("iteration", "opt_step", "lag", "densify_generator", "scene_extent", "filter_3D", "mip_recomputed_at",
               "densified_at", "reset_at", "cfg", "frame")


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
    t.update(P=P, steps=steps, moments=moments, extra=extra, per_point_lr=None if ppl is None else ppl.reshape(P))
    return t
