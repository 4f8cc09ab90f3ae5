"""Drop-in for `scene.per_point_adam.PerPointAdam` (boundary B4):
scene/per_point_adam.py:17-98.  Same constructor, param-group keys
(`params, lr, betas, eps, weight_decay, per_point_lr, name`), state layout
(`state[p] = {step, exp_avg, exp_avg_sq}`) and error behaviour, but `step()` is ONE launch of the
fused sm_90a kernel (gs_adam.cu) over every tensor, with no host synchronisation."""
from __future__ import annotations

import ctypes

import torch
from torch.optim import Optimizer

from . import _lib
from ._lib import ADAM_MAX_TENSORS, GsbAdamTensor, check


def launch_adam(entries, flags, skip_ptr=None, step_sizes_dev=None):
    """entries: list of dicts(param, grad, exp_avg, exp_avg_sq, per_point_lr, step_size, beta1, beta2,
    eps, weight_decay, grad_scale, row_len).  skip_ptr: optional device address of a word that, when non-zero,
    makes the device skip the whole update (gsb_adam_step_gated).  step_sizes_dev: optional fp32 device tensor with one
    step size per entry, read by the kernel instead of the entries' `step_size` (then not needed)."""
    if step_sizes_dev is not None and len(entries) > ADAM_MAX_TENSORS:
        raise _lib.GsbError("device-side step sizes support at most one launch (8 tensors)")
    L = _lib.lib()
    if not entries:
        return
    with torch.cuda.device(entries[0]["param"].device):       # launch on the tensors' device, whatever is current
        _launch_adam_on_device(L, entries, flags, skip_ptr, step_sizes_dev)


def _launch_adam_on_device(L, entries, flags, skip_ptr, step_sizes_dev):
    for i in range(0, len(entries), ADAM_MAX_TENSORS):
        chunk = entries[i:i + ADAM_MAX_TENSORS]
        arr = (GsbAdamTensor * len(chunk))()
        for t, e in zip(arr, chunk):
            t.param, t.grad = e["param"].data_ptr(), e["grad"].data_ptr()
            t.exp_avg, t.exp_avg_sq = e["exp_avg"].data_ptr(), e["exp_avg_sq"].data_ptr()
            ppl = e.get("per_point_lr")
            t.per_point_lr = None if ppl is None else ppl.data_ptr()
            t.numel, t.row_len = e["param"].numel(), int(e.get("row_len", 1))
            t.grad_scale = float(e.get("grad_scale", 1.0))
            t.step_size = 0.0 if step_sizes_dev is not None else float(e["step_size"])
            t.beta1, t.beta2 = float(e["beta1"]), float(e["beta2"])
            t.eps, t.weight_decay = float(e["eps"]), float(e["weight_decay"])
        check(L.gsb_adam_step_ex(len(chunk), arr, flags.data_ptr(), skip_ptr,
                                 None if step_sizes_dev is None else step_sizes_dev.data_ptr(), _lib.stream_ptr()),
              "gsb_adam_step")


def _validated_multiplier(param: torch.Tensor, mult):
    """Type / device / shape checks of the optional per-row learning-rate multiplier; same exception types and
    conditions as the reference optimizer (scene/per_point_adam.py:85-92)."""
    if mult is None:
        return None, 1
    if not isinstance(mult, torch.Tensor):
        raise TypeError("per_point_lr must be a torch.Tensor")
    if mult.device != param.device:
        raise ValueError("per_point_lr must be on the same device as parameter")
    want = param.shape[:1] + (1,) * (param.dim() - 1)
    if mult.shape != want:
        raise ValueError(f"Invalid per_point_lr shape. Expected {want}, got {mult.shape}")
    return mult.float().contiguous(), param.numel() // max(1, param.shape[0])


class PerPointAdam(Optimizer):
    """Adam with an optional per-point learning-rate multiplier (see module docstring)."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0):
        if min(lr, eps, weight_decay) < 0.0:
            raise ValueError(f"Invalid learning parameters: lr={lr}, eps={eps}, weight_decay={weight_decay}")
        if any(not (0.0 <= b < 1.0) for b in betas):
            raise ValueError(f"Invalid beta parameters: {betas}")
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, per_point_lr=None))
        self._flags = None

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        work = []
        for group in self.param_groups:
            b1, b2 = group["betas"]
            for p in group["params"]:
                g = p.grad
                if g is None:
                    continue
                if g.is_sparse:
                    raise RuntimeError("PerPointAdam does not support sparse gradients")
                if not p.is_cuda:
                    raise _lib.GsbError("PerPointAdam needs CUDA parameters; there is no CPU path")
                st = self.state[p]
                if not st:                                   # lazy state, same keys as the reference
                    st["step"] = 0
                    st["exp_avg"] = torch.zeros_like(p)
                    st["exp_avg_sq"] = torch.zeros_like(p)
                st["step"] += 1
                t = st["step"]
                # old-style bias correction folded into the step size, evaluated on the host in double
                step_size = group["lr"] * ((1 - b2 ** t) ** 0.5 / (1 - b1 ** t))
                mult, row_len = _validated_multiplier(p, group.get("per_point_lr"))
                if not (p.is_contiguous() and g.is_contiguous() and p.dtype == torch.float32):
                    raise _lib.GsbError("PerPointAdam needs contiguous fp32 parameters and gradients")
                work.append(dict(param=p, grad=g, exp_avg=st["exp_avg"], exp_avg_sq=st["exp_avg_sq"], per_point_lr=mult,
                                 step_size=step_size, beta1=b1, beta2=b2, eps=group["eps"],
                                 weight_decay=group["weight_decay"], row_len=row_len))
        if work:
            dev = work[0]["param"].device
            if self._flags is None or self._flags.device != dev:
                self._flags = torch.zeros(ADAM_MAX_TENSORS, dtype=torch.int32, device=dev)
            launch_adam(work, self._flags)
        return loss
