"""TEST INFRASTRUCTURE for Muon (K14).

* ``newton_schulz`` / ``muon_step``: a restatement of the rule in include/frl_b200.h (K14), which is
  ``torch.optim.Muon``'s: float64 accumulation with exactly the kernel's bf16 rounding points (the
  iterate, the norm, every product's output).
* ``MuonKernelDouble``: ``oracle.optim_np.KernelDouble`` plus CPU stand-ins for ``_native.adam_mt``
  and ``_native.muon_mt`` that read each gradient where the segment table points, so the host logic
  needs no GPU.  ``calls`` records (name, slot indices, clipped) per launch.

Never imported by the product.
"""
import math

import numpy as np
import torch

from frl_b200 import _native
from frl_b200.fused_optim import MUON_NS_COEFFICIENTS
from oracle.optim_np import KernelDouble
from adam8_oracle import _read


def bf16(x: torch.Tensor) -> torch.Tensor:
    return x.to(torch.bfloat16).to(torch.float64)


def _lerp32(e, x, w):
    """torch's lerp in fp32."""
    e, x, w = e.float(), x.float(), torch.tensor(w, dtype=torch.float32)
    return torch.where(w.abs() < 0.5, e + w * (x - e), x - (x - e) * (1 - w))


def newton_schulz(u: torch.Tensor, ns_coefficients=MUON_NS_COEFFICIENTS, ns_steps=5, eps=1e-7) -> torch.Tensor:
    """O = NS(u) for a 2-D ``u``, float64 with the kernel's bf16 rounding points."""
    a, b, c = ns_coefficients
    x = bf16(u.to(torch.float64))
    trans = u.shape[0] > u.shape[1]
    if trans:
        x = x.T
    nrm = bf16(x.norm().reshape(1))
    eps_bf = bf16(torch.tensor([eps], dtype=torch.float64))
    nrm = torch.where(nrm < eps_bf, eps_bf, nrm)            # NaN stays NaN
    x = bf16(x / nrm)
    for _ in range(ns_steps):
        A = bf16(x @ x.T)
        B = bf16(b * A + c * (A @ A))
        x = bf16(a * x + B @ x)
    return x.T if trans else x


def adjust_factor(shape, adjust_lr_fn) -> float:
    R, C = shape
    return 0.2 * math.sqrt(max(R, C)) if adjust_lr_fn == "match_rms_adamw" else math.sqrt(max(1, R / C))


def muon_step(p, g, buf, *, lr, wd, momentum, nesterov=True, ns_coefficients=MUON_NS_COEFFICIENTS, ns_steps=5,
              eps=1e-7, adjust_lr_fn="match_rms_adamw"):
    """One step of one matrix.  ``p`` fp32 or float64 [R, C], ``g`` the effective gradient (fp32),
    ``buf`` fp32 momentum.  Returns (new p as float64, new buf as fp32)."""
    buf = _lerp32(buf, g, 1 - momentum)
    u = _lerp32(g, buf, momentum) if nesterov else buf
    o = newton_schulz(u, ns_coefficients, ns_steps, eps)
    p = p.to(torch.float64) * (1 - lr * wd) - adjust_factor(tuple(p.shape), adjust_lr_fn) * lr * o
    return p, buf


class MuonKernelDouble(KernelDouble):
    """Host-logic double: K2-mt Adam per slot through ``KernelDouble.adam`` and K14 through
    ``muon_step``, both reading gradients through the segment table's host rows."""

    def __init__(self):
        super().__init__()

    def _rows(self, table):
        for i, s in enumerate(table.slots):
            row = table._segs[i]
            yield s, torch.from_numpy(_read(row.g, s.numel, row.g_dtype))

    def adam_mt(self, p, m, v, vmax, p_lp, table, *, grad_scale=1.0, grad_scale_dev=None, **kw):
        self.calls.append(("adam_mt", tuple(s.index for s in table.slots), grad_scale_dev is not None))
        kw.pop("dyn", None)
        for s, g in self._rows(table):
            cut = lambda t: None if t is None else t[s.offset:s.end]
            KernelDouble.adam(self, cut(p), g, cut(m), cut(v), cut(vmax), cut(p_lp), s.numel, grad_scale=grad_scale,
                              grad_scale_dev=grad_scale_dev, **kw)
            self.calls.pop()

    def grad_accumulate_mt(self, acc, table, *, w=1.0, first=False, dyn=None):
        self.calls.append(("grad_accumulate_mt", table.n_segs))
        if dyn is not None:
            w, first = float(dyn[0]), bool(dyn[1] != 0)
        for i, s in enumerate(table.slots):
            row = table._segs[i]
            base = np.zeros(s.numel, np.float32) if first else acc[s.offset:s.end].numpy().copy()
            if row.g:
                base = (base + np.float32(w) * _read(row.g, s.numel, row.g_dtype)).astype(np.float32)
            acc[s.offset:s.end] = torch.from_numpy(base)

    muon_plan_bytes = staticmethod(_native.muon_plan_bytes)
    check_muon_hyper = staticmethod(_native.check_muon_hyper)

    def muon_plan(self, shape, exp_avg_sq, workspace):
        _, scratch, ws = _native.muon_plan_bytes(shape)
        assert workspace.numel() * workspace.element_size() >= ws
        self.plans = getattr(self, "plans", 0) + 1
        return _native.MuonPlan(shape.clone(), None, None, torch.zeros(scratch // 4 + 1, dtype=torch.int32), workspace,
                                exp_avg_sq)

    def muon_mt(self, p, exp_avg, p_lp, table, plan, *, lr, wd, momentum, nesterov, ns_coefficients, ns_steps, eps,
                adjust_lr_fn, grad_scale=1.0, grad_scale_dev=None, dyn=None):
        _native.check_muon_hyper(lr=lr, wd=wd, momentum=momentum, ns_steps=ns_steps, eps=eps, adjust_lr_fn=adjust_lr_fn)
        rows = [int(r[0]) for r in plan.shape.tolist()]
        self.calls.append(("muon_mt", tuple(table.slots[i].index for i in rows), grad_scale_dev is not None))
        scale = np.float32(grad_scale) * np.float32(float(grad_scale_dev.item()) if grad_scale_dev is not None else 1.0)
        for i in rows:
            s, row = table.slots[i], table._segs[i]
            g = torch.from_numpy(_read(row.g, s.numel, row.g_dtype) * scale).view(s.shape)
            w, b = muon_step(p[s.offset:s.end].view(s.shape), g, exp_avg[s.offset:s.end].view(s.shape), lr=lr, wd=wd,
                             momentum=momentum, nesterov=nesterov, ns_coefficients=ns_coefficients,
                             ns_steps=ns_steps, eps=eps, adjust_lr_fn=adjust_lr_fn)
            p[s.offset:s.end] = w.float().reshape(-1)
            exp_avg[s.offset:s.end] = b.reshape(-1)
            if p_lp is not None:
                p_lp[s.offset:s.end] = w.reshape(-1).to(p_lp.dtype)
