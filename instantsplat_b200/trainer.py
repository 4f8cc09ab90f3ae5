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

import ctypes
import math
from typing import Dict, List, Optional

import numpy as np
import torch

from . import _lib
from ._lib import GsbCamera, GsbGaussians, GsbGrads, check
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


def L_sig_words():
    return (_lib.lib().gsb_peer_signal_bytes() + 3) // 4


def _align(n, a=64):
    return (n + a - 1) // a * a


class JointTrainer:
    def __init__(self, scene: Scene, device, gt_images: Optional[torch.Tensor] = None,
                 cfg: Optional[OptimConfig] = None, world_size: int = 1, rank: int = 0,
                 process_group=None, exchange: str = "allreduce", use_graph: bool = False):
        self.cfg = cfg or OptimConfig()
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
        # ---- camera constants (identity view, reference gaussian_renderer/__init__.py:55-59)
        from .camera import projection_matrix
        self.tanfovx, self.tanfovy = math.tan(scene.fovx * 0.5), math.tan(scene.fovy * 0.5)
        self.viewmatrix = torch.eye(4, device=self.dev)
        self.projmatrix = projection_matrix(0.01, 100.0, scene.fovx, scene.fovy).t().contiguous().to(self.dev)
        self.campos = torch.zeros(3, device=self.dev)
        self.bg = scene.bg.to(self.dev).float().contiguous()
        # ---- scratch
        L = _lib.lib()
        self.geom_bytes = L.gsb_geom_bytes(P)
        self.geom = torch.empty(self.geom_bytes, dtype=torch.uint8, device=self.dev)
        self.image_buf = torch.empty(L.gsb_image_bytes(self.W, self.H), dtype=torch.uint8, device=self.dev)
        self.binning = None
        self.bin_bytes = 0
        self.cap = 0                  # instance capacity of the binning buffer (0: not sized yet)
        self.headroom = 1.5
        self.radii = torch.empty(P, dtype=torch.int32, device=self.dev)
        self.color = torch.empty(3, self.H, self.W, dtype=torch.float32, device=self.dev)
        self.dL_dimg = torch.empty_like(self.color)
        self.maps = torch.empty(3, 3, self.H, self.W, dtype=torch.float32, device=self.dev)
        self.sums = torch.zeros(2, dtype=torch.float64, device=self.dev)
        self.host_status = torch.zeros(2, 8, dtype=torch.int32).pin_memory()   # [0] after preprocess, [1] after render
        self._ev_pre = torch.cuda.Event()
        self._status_dev = L.gsb_status_device(self.geom.data_ptr(), P)        # device address of the status words
        so = self._status_dev - self.geom.data_ptr()
        self._status_t = self.geom[so:so + 32].view(torch.int32)               # [R, overflow, longest list, ...]
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
        self._status_t.zero_()        # the forward serial number lives in these words
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

    # ------------------------------------------------------------------------------------------
    def view(self, flat: torch.Tensor, name: str) -> torch.Tensor:
        k = dict(SEGMENTS)[name]
        o = self.offs[name]
        return flat[o:o + self.P * k].view(self.P, k)

    def my_views(self) -> List[int]:
        from .parallel import shard_views
        return shard_views(self.n_views, self.world_size, self.rank)

    def _cam(self) -> GsbCamera:
        cam = GsbCamera()
        cam.width, cam.height = self.W, self.H
        cam.tanfovx, cam.tanfovy, cam.scale_modifier = self.tanfovx, self.tanfovy, 1.0
        cam.sh_degree, cam.sh_coeffs = self.active_sh_degree, 16
        cam.exact_cull = 1 if self.exact_cull else 0
        cam.bg, cam.viewmatrix = self.bg.data_ptr(), self.viewmatrix.data_ptr()
        cam.projmatrix, cam.campos = self.projmatrix.data_ptr(), self.campos.data_ptr()
        return cam

    def _gauss(self, view: int) -> GsbGaussians:
        g = GsbGaussians()
        g.P, g.sh_packed, g.raw_params = self.P, 0, 1
        p = self.params
        g.means3D = self.view(p, "xyz").data_ptr()
        g.scales = self.view(p, "scaling").data_ptr()
        g.rotations = self.view(p, "rotation").data_ptr()
        g.opacities = self.view(p, "opacity").data_ptr()
        g.sh_dc = self.view(p, "f_dc").data_ptr()
        g.sh_rest = self.view(p, "f_rest").data_ptr()
        g.pose = self.poses[view].data_ptr()
        return g

    # ------------------------------------------------------------------------------------------
    def _size_binning(self, R: int) -> None:
        L = _lib.lib()
        self.cap = int(R * self.headroom) + 65536
        self.bin_bytes = L.gsb_binning_bytes(self.cap, self.W, self.H)
        self.binning = torch.empty(self.bin_bytes, dtype=torch.uint8, device=self.dev)

    def _launch_forward(self, view: int) -> None:
        """Enqueue the forward without ever waiting for the GPU: the instance count R stays on the device; the
        host only provides a capacity (sized from the counts seen so far, +50 %) and reads R back lazily."""
        L = _lib.lib()
        st = _lib.stream_ptr()
        cam, g = self._cam(), self._gauss(view)
        capturing = torch.cuda.is_current_stream_capturing()
        check(L.gsb_preprocess(ctypes.byref(cam), ctypes.byref(g), self.geom.data_ptr(), self.geom_bytes,
                               self.radii.data_ptr(), self.host_status[0].data_ptr(), st), "gsb_preprocess")
        if not capturing:
            self._fwd_count += 1
            self._polling = False
            self._ev_pre.record()
            if self.cap == 0:                               # very first forward: size the buffer from the real count
                self._ev_pre.synchronize()
                self._size_binning(int(self.host_status[0, 0]) & 0xFFFFFFFF)
        check(L.gsb_render(ctypes.byref(cam), self.P, self.geom.data_ptr(), self.binning.data_ptr(),
                           self.bin_bytes, self.cap, self.image_buf.data_ptr(), self.color.data_ptr(),
                           self.host_status[1].data_ptr(), st), "gsb_render")
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
            while (int(hs[0, 6]) & 0x7FFFFFFF) != want:
                n += 1
                if n > 20_000_000:
                    raise _lib.GsbError("graph replay: the forward's status words never arrived")
        else:
            self._ev_pre.synchronize()
        R = int(self.host_status[0, 0]) & 0xFFFFFFFF
        self.last_R = R
        if R > self.cap:
            self.overflows += 1
            self._size_binning(R)
            return False
        if R > 0.85 * self.cap:                              # grow ahead of need
            self._size_binning(R)
        return True

    def render(self, view: int) -> torch.Tensor:
        """Forward only (exact: repeated with a larger buffer in the unlikely case the capacity was exceeded)."""
        self._launch_forward(view)
        if not self._settle():
            self._launch_forward(view)
            assert self._settle()
        return self.color

    def loss_and_backward(self, view: int, gt: torch.Tensor) -> None:
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
        check(L.gsb_backward(ctypes.byref(cam), ctypes.byref(g), self.geom.data_ptr(), self.binning.data_ptr(),
                             self.cap, self.image_buf.data_ptr(), self.dL_dimg.data_ptr(), ctypes.byref(gr), st),
              "gsb_backward")

    def loss_value(self) -> torch.Tensor:
        n = 3 * self.H * self.W
        lam = self.cfg.lambda_dssim
        return (1.0 - lam) * self.sums[0] / n + lam * (1.0 - self.sums[1] / n)

    def reduce_grads(self) -> None:
        if self.world_size > 1:
            from .parallel import allreduce_sum_
            self._pg_buf[-1:].copy_(self._status_t[1:2])
            allreduce_sum_((self.grads, self._pg_buf), self.pg)

    def _step_sizes(self):
        """lr * sqrt(1-b2^t)/(1-b1^t) per tensor for the current counters (host, double)."""
        c = self.cfg
        t = max(1, self.opt_step)
        corr = (1 - 0.999 ** t) ** 0.5 / (1 - 0.9 ** t)
        lrs = self._lrs()
        out = [lrs[name] * corr for name, _ in SEGMENTS]
        if c.optim_pose:
            out.append(self.cam_sched(self.iteration) * corr)
        return out

    def _upload_step_sizes(self) -> None:
        ss = self._step_sizes()
        for i, v in enumerate(ss):
            self._step_host[i] = v
        self._step_dev.copy_(self._step_host, non_blocking=True)

    def optimizer_step(self, grad_scale: Optional[float] = None, _advance: bool = True, _dev_steps: bool = False) -> None:
        """PerPointAdam.step over the 6 Gaussian tensors + the pose table in one launch
        (param groups and LRs of scene/gaussian_model.py:203-243)."""
        c = self.cfg
        if _advance:
            self.opt_step += 1
        t = self.opt_step
        b1, b2, eps = 0.9, 0.999, 1e-15
        corr = (1 - b2 ** t) ** 0.5 / (1 - b1 ** t)
        lrs = dict(xyz=self.xyz_sched(self.iteration), f_dc=c.feature_lr * 10, f_rest=c.feature_lr / 20.0 * 10,
                   opacity=c.opacity_lr, scaling=c.scaling_lr * 10, rotation=c.rotation_lr * 10)
        gs = 1.0 / self.world_size if grad_scale is None else grad_scale
        entries = []
        for name, k in SEGMENTS:
            entries.append(dict(param=self.view(self.params, name), grad=self.view(self.grads, name),
                                exp_avg=self.view(self.exp_avg, name), exp_avg_sq=self.view(self.exp_avg_sq, name),
                                per_point_lr=self.per_point_lr if name == "xyz" else None, row_len=k,
                                step_size=lrs[name] * corr, beta1=b1, beta2=b2, eps=eps, weight_decay=0.0,
                                grad_scale=gs))
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
        return self._status_dev + 4

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
                                      self.flags.data_ptr(), self._status_dev + 4, self.pose_grad.data_ptr(),
                                      self.pose_grad.numel(), st), "gsb_peer_exchange")
        else:
            # one small SUM all-reduce carries both the gate flags (as counts) and the pose-gradient table
            # (self.pose_grad is a view of self._xch[8:]); it is also the pre-barrier of the fused kernel
            self._xch[:8].copy_(self.flags)
            self._xch[7:8].copy_(self._status_t[1:2])          # slot 7: binning overflow (summed over ranks)
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

    def _graph_iteration(self, view: int, gt: torch.Tensor, do_opt: bool) -> None:
        """Replay (capturing on first use) the CUDA graph of one iteration on `view`."""
        if do_opt:
            self.opt_step += 1
            self._upload_step_sizes()                    # stream-ordered before the replay
        for _attempt in range(2):
            key = (view, gt.data_ptr(), do_opt, self.active_sh_degree, self.cap, self.exact_cull)
            g = self._graphs.get(key)
            if g is None:
                if len(self._graphs) > 64:
                    self._graphs.clear()
                torch.cuda.synchronize()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    self._launch_forward(view)
                    self.loss_and_backward(view, gt)
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

    def _run_iteration(self, view: int, gt: torch.Tensor, do_opt: bool) -> None:
        self._launch_forward(view)
        self.loss_and_backward(view, gt)
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
        if self.use_graph and self.cap > 0:
            self._graph_iteration(view, gt, do_opt)
            return
        self._run_iteration(view, gt, do_opt)
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
            self._run_iteration(view, gt, do_opt)
            assert self._settle()

    # ---- densify / prune / opacity reset on the flat buffers (SURVEY.md section 8 row f4) -----------------------
    # Semantics of scene/gaussian_model.py: prune_points (:359-374) keeps the surviving rows of every
    # parameter AND of both Adam moments; densification_postfix (:399-418) appends rows with zero moments;
    # reset_opacity (:280-283) clamps the opacity to 0.01 (in logit space) and zeroes that tensor's moments.  The
    # optimizer's step counter is untouched by all three, as in the reference (state["step"] survives the surgery).
    def _resize(self, new_P: int, rows) -> None:
        """rows(name, old_param_view, old_m_view, old_v_view) -> (param, m, v) tensors of shape [new_P, k]."""
        if self._fused:
            raise _lib.GsbError("changing the number of Gaussians is not supported with peer-memory buffers "
                                "(exchange='fused_p2p'); use exchange='allreduce'")
        L = _lib.lib()
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
        self.geom_bytes = L.gsb_geom_bytes(new_P)
        self.geom = torch.empty(self.geom_bytes, dtype=torch.uint8, device=self.dev)
        self.radii = torch.empty(new_P, dtype=torch.int32, device=self.dev)
        self._status_dev = L.gsb_status_device(self.geom.data_ptr(), new_P)
        so = self._status_dev - self.geom.data_ptr()
        self._status_t = self.geom[so:so + 32].view(torch.int32)
        self.cap = 0                                  # the next forward sizes the binning buffer from the new count
        self._keep = None
        self._graphs.clear()
        self._status_t.zero_()
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
        self._resize(int(keep.sum()), lambda name, p, m, v: (p[keep], m[keep], v[keep]))
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

    def reset_opacity(self) -> None:
        op = self.view(self.params, "opacity")
        cur = torch.sigmoid(op)
        new = torch.min(cur, torch.full_like(cur, 0.01))
        op.copy_(torch.log(new / (1 - new)))
        self.view(self.exp_avg, "opacity").zero_()
        self.view(self.exp_avg_sq, "opacity").zero_()

    def blend_stats(self, view: int, gt: Optional[torch.Tensor] = None) -> Dict[str, int]:
        """Pair statistics of the blend kernels for one forward+backward of `view` (instrumented re-run of the same
        kernels, outside any timed region): evaluated / contributing (pixel, Gaussian) pairs."""
        L = _lib.lib()
        self.render(view)
        self.loss_and_backward(view, self.gt[view] if gt is None else gt)
        cam, _ = self._keep
        stats = torch.zeros(8, dtype=torch.int64, device=self.dev)
        check(L.gsb_blend_stats(ctypes.byref(cam), self.P, self.geom.data_ptr(), self.binning.data_ptr(), self.cap,
                                self.image_buf.data_ptr(), self.color.data_ptr(), self.dL_dimg.data_ptr(),
                                stats.data_ptr(), _lib.stream_ptr()), "gsb_blend_stats")
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
