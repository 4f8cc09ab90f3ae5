"""CPU stand-in for `scene.per_point_adam.PerPointAdam` (tests only): the reference optimizer's interface (param groups
with `lr`, `per_point_lr`, `name`; state {step, exp_avg, exp_avg_sq}) with the oracle's update
(oracle/gs_oracle.py per_point_adam_step).  instantsplat_b200.per_point_adam has no CPU path by design."""
import torch
from torch.optim import Optimizer

from oracle import gs_oracle as O


class PerPointAdam(Optimizer):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0):
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, per_point_lr=None))

    @torch.no_grad()
    def step(self, closure=None):
        for group in self.param_groups:
            b1, b2 = group["betas"]
            for p in group["params"]:
                if p.grad is None:
                    continue
                st = self.state[p]
                if not st:
                    st["step"] = 0
                    st["exp_avg"] = torch.zeros_like(p)
                    st["exp_avg_sq"] = torch.zeros_like(p)
                st["step"] += 1
                O.per_point_adam_step(p, p.grad, st["exp_avg"], st["exp_avg_sq"], st["step"], group["lr"], b1, b2,
                                      group["eps"], group["weight_decay"], per_point_lr=group.get("per_point_lr"))
