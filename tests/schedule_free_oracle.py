"""TEST INFRASTRUCTURE for Schedule-Free AdamW / SGD (``Solver.solve(..., schedule_free=...)``, the
``frl_sf_*`` kernels).

* ``RefAdamWScheduleFree`` / ``RefSGDScheduleFree``: ``torch.optim.Optimizer`` restatements of the
  schedulefree package's 1.x ``step()`` (Defazio et al. 2024, *The Road Less Scheduled*), with Adam's bias
  correction folded into lr and the package's state layout (group ``k`` / ``weight_sum`` / ``lr_max`` /
  ``train_mode`` ...; per parameter ``z`` and ``exp_avg_sq``).  ``train()`` / ``eval()`` move the
  parameters between y and x = lerp(y, z, 1 - 1/beta1) as the package does.  Meant to run in float64;
  they stand in for the package, which the project does not depend on.
* ``sf_eval_f64``: x from y and z in float64.

Never imported by the product.
"""
import math

import torch


class _RefScheduleFree(torch.optim.Optimizer):
    ADAPTIVE = False

    def _beta1(self, group):
        return group["betas"][0] if self.ADAPTIVE else group["momentum"]

    @torch.no_grad()
    def eval(self):
        for group in self.param_groups:
            if group["train_mode"]:
                beta1 = self._beta1(group)
                for p in group["params"]:
                    state = self.state[p]
                    if "z" in state:
                        p.lerp_(state["z"], 1.0 - 1.0 / beta1)       # y -> x
                group["train_mode"] = False

    @torch.no_grad()
    def train(self):
        for group in self.param_groups:
            if not group["train_mode"]:
                beta1 = self._beta1(group)
                for p in group["params"]:
                    state = self.state[p]
                    if "z" in state:
                        p.lerp_(state["z"], 1.0 - beta1)              # x -> y
                group["train_mode"] = True

    @torch.no_grad()
    def step(self, closure=None):
        for group in self.param_groups:
            if not group["train_mode"]:
                raise RuntimeError("step() in eval mode")
            k = group["k"]
            warmup = group["warmup_steps"]
            sched = (k + 1) / warmup if k < warmup else 1.0
            beta1 = self._beta1(group)
            lr = group["lr"] * sched
            if self.ADAPTIVE:
                beta2 = group["betas"][1]
                lr = lr * math.sqrt(1 - beta2 ** (k + 1))
            lr_max = group["lr_max"] = max(lr, group["lr_max"])
            weight = ((k + 1) ** group["r"]) * (lr_max ** group["weight_lr_power"])
            weight_sum = group["weight_sum"] = group["weight_sum"] + weight
            try:
                ckp1 = weight / weight_sum
            except ZeroDivisionError:
                ckp1 = 0.0
            wd = group["weight_decay"]
            for y in group["params"]:
                if y.grad is None:
                    continue
                state = self.state[y]
                if "z" not in state:
                    state["z"] = torch.clone(y, memory_format=torch.preserve_format)
                    if self.ADAPTIVE:
                        state["exp_avg_sq"] = torch.zeros_like(y, memory_format=torch.preserve_format)
                z = state["z"]
                u = y.grad.clone()
                if self.ADAPTIVE:
                    v = state["exp_avg_sq"]
                    v.mul_(beta2).addcmul_(u, u, value=1 - beta2)
                    u = u / v.sqrt().add_(group["eps"])
                if wd != 0:
                    u.add_(y, alpha=wd)
                y.lerp_(z, ckp1)
                y.add_(u, alpha=lr * (beta1 * (1 - ckp1) - 1))
                z.sub_(u, alpha=lr)
            group["k"] = k + 1


class RefAdamWScheduleFree(_RefScheduleFree):
    ADAPTIVE = True

    def __init__(self, params, lr=0.0025, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, warmup_steps=0,
                 r=0.0, weight_lr_power=2.0):
        super().__init__(params, dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay, k=0,
                                      warmup_steps=warmup_steps, train_mode=True, weight_sum=0.0, lr_max=-1.0,
                                      r=r, weight_lr_power=weight_lr_power))


class RefSGDScheduleFree(_RefScheduleFree):
    def __init__(self, params, lr=1.0, momentum=0.9, weight_decay=0.0, warmup_steps=0, r=0.0,
                 weight_lr_power=2.0):
        if not 0.0 < momentum < 1.0:
            raise ValueError("momentum %r outside (0, 1)" % (momentum,))
        super().__init__(params, dict(lr=lr, momentum=momentum, weight_decay=weight_decay, k=0,
                                      warmup_steps=warmup_steps, train_mode=True, weight_sum=0.0, lr_max=-1.0,
                                      r=r, weight_lr_power=weight_lr_power))


def sf_eval_f64(y, z, beta1):
    """x = lerp(y, z, 1 - 1/beta1) in float64."""
    y, z = y.double(), z.double()
    return y + (1.0 - 1.0 / beta1) * (z - y)
