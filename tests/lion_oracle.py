"""TEST INFRASTRUCTURE for Lion (``Solver.solve(..., lion=True)``, the ``frl_lion*`` kernels).

* ``lion_step_f64``: a float64 restatement of the rule the kernels pin (include/frl_b200.h):
  ``p *= 1 - lr*wd``; ``c = lerp(m, g, 1 - beta1)``; ``p -= lr * sign(c)``; ``m = lerp(m, g, 1 - beta2)``,
  with sign(NaN) = NaN.  ``c`` is returned too, so a caller can tell where a sign is ill-conditioned.
* ``lion_step``: the same rule in the kernel's fp32 operation order (numpy), for the CPU doubles.
* ``RefLion``: a ``torch.optim.Optimizer`` that transcribes Algorithm 2 of Chen et al. 2023
  (*Symbolic Discovery of Optimization Algorithms*) with the state layout of the published Lion
  implementations (group ``lr`` / ``betas`` / ``weight_decay``, state ``exp_avg``).  It stands in for
  lion-pytorch and timm, which the project does not depend on.
* ``LionKernelDouble``: the CPU kernel doubles plus stand-ins for ``_native.lion`` / ``lion_mt`` /
  ``dw_gemm_lion`` / ``nvls_lion`` with their call signatures, so host logic needs no GPU.

Never imported by the product.
"""
import numpy as np
import torch

from adamw_oracle import AdamWKernelDouble
from adam8_oracle import _read

f32 = np.float32


def decay_factor(lr, wd):
    """fp32(1 - lr * wd), formed in double."""
    return f32(1.0 - float(lr) * float(wd))


def _sign(x):
    return np.where(np.isnan(x), x, np.sign(x))


def lion_step_f64(p, g, m, *, lr, beta1, beta2, wd, grad_scale=1.0):
    """One Lion step in float64: (p, m, c)."""
    p, g, m = (np.asarray(x, dtype=np.float64) for x in (p, g, m))
    g = g * grad_scale
    p = p * (1.0 - lr * wd)
    c = m + (1.0 - beta1) * (g - m)
    p = p - lr * _sign(c)
    m = m + (1.0 - beta2) * (g - m)
    return p, m, c


def _fma(a, b, c):
    """fp32 a*b + c, the product exact in float64 and the sum rounded to fp32."""
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(f32)


def lion_step(p, g, m, *, lr, beta1, beta2, wd, grad_scale=1.0):
    """One Lion step in the kernel's fp32 operation order (numpy fp32 arrays): (p, m)."""
    with np.errstate(invalid="ignore", over="ignore"):
        g = (np.asarray(g, dtype=f32) * f32(grad_scale)).astype(f32)
        m = np.asarray(m, dtype=f32)
        p = (np.asarray(p, dtype=f32) * decay_factor(lr, wd)).astype(f32)
        c = _fma(f32(1.0 - beta1), (g - m).astype(f32), m)
        p = _fma(f32(-lr), _sign(c).astype(f32), p)
        m = _fma(f32(1.0 - beta2), (g - m).astype(f32), m)
    return p, m


class RefLion(torch.optim.Optimizer):
    """Lion, Algorithm 2 of Chen et al. 2023, with decoupled weight decay:
    ``update = sign(beta1*m + (1-beta1)*g)``; ``p = p - lr*(update + wd*p)``;
    ``m = beta2*m + (1-beta2)*g``.  sign(NaN) is NaN (``torch.sign`` gives 0 on the CPU)."""

    def __init__(self, params, lr=1e-4, betas=(0.9, 0.99), weight_decay=0.0):
        if not (0.0 <= betas[0] < 1.0 and 0.0 <= betas[1] < 1.0):
            raise ValueError("betas %r outside [0, 1)" % (betas,))
        super().__init__(params, dict(lr=lr, betas=tuple(betas), weight_decay=weight_decay))

    @torch.no_grad()
    def step(self, closure=None):
        for group in self.param_groups:
            lr, (beta1, beta2), wd = group["lr"], group["betas"], group["weight_decay"]
            for p in group["params"]:
                if p.grad is None:
                    continue
                state = self.state[p]
                if not state:
                    state["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                m = state["exp_avg"]
                g = p.grad
                p.mul_(1.0 - lr * wd)
                u = m * beta1 + g * (1.0 - beta1)
                p.add_(torch.where(torch.isnan(u), u, torch.sign(u)), alpha=-lr)
                m.mul_(beta2).add_(g, alpha=1.0 - beta2)


class LionKernelDouble(AdamWKernelDouble):
    """The CPU kernel doubles plus the fp32-master Lion entry points."""

    def _apply(self, p, g, m, p_lp, *, lr, beta1, beta2, wd, grad_scale=1.0, grad_scale_dev=None):
        np_, nm = lion_step(self._np(p), self._np(g), self._np(m), lr=lr, beta1=beta1, beta2=beta2, wd=wd,
                            grad_scale=self._scale(grad_scale, grad_scale_dev))
        self._store(p, np_); self._store(m, nm); self._store(p_lp, np_)

    def lion(self, p, g, m, p_lp, n, *, lr, beta1, beta2, wd, grad_scale=1.0, grad_scale_dev=None, dyn=None):
        self.calls.append(("lion", n))
        self._apply(p, g, m, p_lp, lr=lr, beta1=beta1, beta2=beta2, wd=wd, grad_scale=grad_scale,
                    grad_scale_dev=grad_scale_dev)

    def lion_mt(self, p, m, p_lp, table, *, lr, beta1, beta2, wd, grad_scale=1.0, grad_scale_dev=None, dyn=None):
        self.calls.append(("lion_mt", table.n_segs))
        for i, s in enumerate(table.slots):
            row = table._segs[i]
            g = torch.from_numpy(_read(row.g, s.numel, row.g_dtype))
            self._apply(p[s.offset:s.end], g, m[s.offset:s.end], p_lp[s.offset:s.end] if (p_lp is not None and
                        s.is_model) else None, lr=lr, beta1=beta1, beta2=beta2, wd=wd, grad_scale=grad_scale,
                        grad_scale_dev=grad_scale_dev)

    def dw_gemm_lion(self, dz, x, gw, p, m, p_lp, *, lr, beta1, beta2, wd, grad_scale=1.0, dyn=None):
        self.calls.append(("dw_gemm_lion", gw.numel()))
        torch.mm(dz.t(), x, out=gw)
        self._apply(p, gw.view(-1), m, p_lp, lr=lr, beta1=beta1, beta2=beta2, wd=wd, grad_scale=grad_scale)

    def nvls_lion(self, p, m, mc_g, mc_out, n, link, *, lr, beta1, beta2, wd, grad_scale, g_dtype, dyn=None):
        raise AssertionError("the fused NVLS step needs several GPUs")
