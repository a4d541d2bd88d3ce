"""TEST INFRASTRUCTURE for Adafactor (K2-af).

* ``adafactor_step``: a float64 numpy restatement of one step of one tensor, written from the rule
  in include/frl_b200.h (K2-af), which is ``torch.optim.Adafactor``'s with foreach=False.
* ``AdafactorKernelDouble``: ``oracle.optim_np.KernelDouble`` plus a CPU stand-in for
  ``_native.adafactor_mt`` that reads each gradient where the segment table points, so the host
  logic (and multi-rank runs under gloo) needs no GPU.  The band table comes from the library's
  host planner.

Never imported by the product.
"""
import numpy as np
import torch

from frl_b200 import _native
from frl_b200.fused_optim import adafactor_shape
from oracle.optim_np import KernelDouble
from adam8_oracle import _read


def _lerp(e, x, w):
    return e + w * (x - e) if abs(w) < 0.5 else x - (x - e) * (1.0 - w)


def _pymax(lo, x):
    return x if x > lo else lo


def adafactor_step(p, g, state, shape, *, lr, t, beta2_decay=-0.8, eps1=2.0 ** -23, eps2=1e-3, d=1.0, wd=0.0):
    """One step of one tensor in float64.  ``p``, ``g``: flat arrays; ``state``: dict with ``row_var``
    [B, R] and ``col_var`` [B, C], or ``variance`` [numel].  Returns the new p; updates ``state``."""
    p = np.asarray(p, dtype=np.float64).copy()
    g = np.asarray(g, dtype=np.float64)
    B, R, C = adafactor_shape(shape)
    w = float(t) ** beta2_decay
    rho = min(lr, 1.0 / float(t) ** 0.5)
    with np.errstate(invalid="ignore", over="ignore"):
        alpha = _pymax(eps2, float(np.sqrt((p * p).sum())) / p.size ** 0.5) * rho
        p *= 1.0 - lr * wd
        if R:
            g3 = g.reshape(B, R, C)
            rv = state["row_var"] = _lerp(state["row_var"], (g3 * g3).sum(axis=2) / C, w)
            cv = state["col_var"] = _lerp(state["col_var"], (g3 * g3).sum(axis=1) / R, w)
            m = rv.mean(axis=1)
            den = np.where(m < eps1, eps1, m)
            vhat = (rv[:, :, None] * cv[:, None, :] / den[:, None, None]).ravel()
        else:
            vhat = state["variance"] = _lerp(state["variance"], g * g, w)
        u = 1.0 / np.sqrt(np.where(vhat < eps1 * eps1, eps1 * eps1, vhat)) * g
        denom = _pymax(1.0, float(np.sqrt((u * u).sum())) / (u.size ** 0.5 * d))
    return p + (-alpha / denom) * u


def zero_state(shape):
    B, R, C = adafactor_shape(shape)
    if R:
        return {"row_var": np.zeros((B, R)), "col_var": np.zeros((B, C))}
    return {"variance": np.zeros(C)}


class AdafactorKernelDouble(KernelDouble):
    LW_ADAPTED, LW_CLIPPED = 1, 2

    adafactor_plan = staticmethod(_native.adafactor_plan)
    adafactor_scratch_bytes = staticmethod(_native.adafactor_scratch_bytes)

    def adafactor_mt(self, p, state, p_lp, table, plan, *, lr, beta2_decay, eps1, eps2, d, wd, step,
                     grad_scale=1.0, grad_scale_dev=None, dyn=None):
        self.calls.append(("adafactor_mt", table.n_segs))
        shape_dev, off, flags, _, _, _, _ = plan
        c = float(grad_scale_dev.item()) if grad_scale_dev is not None else 1.0
        fl, offs = flags.tolist(), off.tolist()
        for i, s in enumerate(table.slots):
            if s.numel == 0:
                continue
            row = table._segs[i]
            g = _read(row.g, s.numel, row.g_dtype).astype(np.float32) * np.float32(grad_scale)
            if fl[i] & self.LW_CLIPPED:
                g = g * np.float32(c)
            B, R, C = adafactor_shape(s.shape)
            o = offs[i]
            if R:
                st = {"row_var": state[o:o + B * R].double().numpy().reshape(B, R),
                      "col_var": state[o + B * R:o + B * (R + C)].double().numpy().reshape(B, C)}
            else:
                st = {"variance": state[o:o + C].double().numpy()}
            w = adafactor_step(p[s.offset:s.end].double().numpy(), g, st, s.shape, lr=lr, t=step,
                               beta2_decay=beta2_decay, eps1=eps1, eps2=eps2, d=d, wd=wd)
            p[s.offset:s.end] = torch.from_numpy(w).float()
            flat = np.concatenate([st["row_var"].ravel(), st["col_var"].ravel()]) if R else st["variance"]
            state[o:o + flat.size] = torch.from_numpy(flat).float()
            if p_lp is not None and s.is_model:
                p_lp[s.offset:s.end] = torch.from_numpy(w).to(p_lp.dtype)
