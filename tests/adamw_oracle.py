"""TEST INFRASTRUCTURE for AdamW (``Solver.solve(..., adamw=True)``, the ``frl_adamw*`` kernels).

* ``adamw_step_f64``: a float64 restatement of the rule, torch 2.11's
  ``Adam(decoupled_weight_decay=True)`` (which ``torch.optim.AdamW`` is): the parameter is first
  scaled by ``1 - lr * wd``, then Adam's step runs with no decay term in the gradient.
* ``adamw_step``: the same rule in the kernel's fp32 order: ``p * fp32(1 - lr * wd)`` rounded on
  its own (the decay factor formed in double and rounded once), then ``oracle.optim_np.adam_step``
  with ``wd = 0``, which is this package's Adam step (lerp for m, bias corrections in double).
* ``adamw8_step``: one K2-q8 AdamW step of one tensor: decode, ``adamw_step``, encode.
* ``AdamWKernelDouble``: ``Adam8KernelDouble`` plus CPU stand-ins for the four entry points
  ``_native.adamw`` / ``adamw_mt`` / ``adamw8_mt`` / ``nvls_adamw`` with their call signatures,
  so host logic (and multi-rank runs under gloo) needs no GPU.

Never imported by the product.
"""
import numpy as np
import torch

from adam8_oracle import Adam8KernelDouble, _read, decode, encode
from oracle.optim_np import adam_step

f32 = np.float32


def decay_factor(lr, wd):
    """fp32(1 - lr * wd), formed in double: what ``param.mul_(1 - lr * weight_decay)`` multiplies by."""
    return f32(1.0 - float(lr) * float(wd))


def adamw_step_f64(p, g, m, v, vmax, *, lr, beta1, beta2, eps, wd, step):
    """One AdamW step in float64 (numpy arrays; ``vmax`` None without amsgrad)."""
    p, g, m, v = (np.asarray(x, dtype=np.float64) for x in (p, g, m, v))
    p = p * (1.0 - lr * wd)
    m = m + (1.0 - beta1) * (g - m)
    v = v * beta2 + (1.0 - beta2) * g * g
    if vmax is not None:
        vmax = np.maximum(np.asarray(vmax, dtype=np.float64), v)
    denom = np.sqrt(v if vmax is None else vmax) / np.sqrt(1.0 - beta2 ** step) + eps
    p = p - lr / (1.0 - beta1 ** step) * m / denom
    return p, m, v, vmax


def adamw_step(p, g, m, v, vmax, *, lr, beta1, beta2, eps, wd, step, grad_scale=1.0):
    """One AdamW step in the kernel's fp32 operation order (numpy fp32 arrays)."""
    p = (np.asarray(p, dtype=f32) * decay_factor(lr, wd)).astype(f32)
    return adam_step(p, g, m, v, vmax, lr=lr, beta1=beta1, beta2=beta2, eps=eps, wd=0.0, step=step,
                     grad_scale=grad_scale)


def adamw8_step(p, g, mq, ma, vq, va, *, lr, beta1, beta2, eps, wd, step, grad_scale=1.0):
    """``adam8_oracle.adam8_step`` with the AdamW rule."""
    m, v = decode(mq, ma, True), decode(vq, va, False)
    with np.errstate(invalid="ignore", over="ignore"):
        p, m, v, _ = adamw_step(p, g, m, v, None, lr=lr, beta1=beta1, beta2=beta2, eps=eps, wd=wd, step=step,
                                grad_scale=grad_scale)
    return p, encode(m, True), encode(v, False), m, v


class AdamWKernelDouble(Adam8KernelDouble):
    """The CPU kernel doubles plus the four AdamW entry points."""

    @staticmethod
    def muon_plan_bytes(shape):
        from frl_b200 import _native                   # host-side sizing, no launch
        return _native.muon_plan_bytes(shape)

    def _apply(self, p, g, m, v, vmax, p_lp, *, lr, beta1, beta2, eps, wd, step, grad_scale=1.0,
               grad_scale_dev=None):
        np_, nm, nv, nvm = adamw_step(self._np(p), self._np(g), self._np(m), self._np(v), self._np(vmax),
                                      lr=lr, beta1=beta1, beta2=beta2, eps=eps, wd=wd, step=step,
                                      grad_scale=self._scale(grad_scale, grad_scale_dev))
        self._store(p, np_); self._store(m, nm); self._store(v, nv); self._store(vmax, nvm)
        self._store(p_lp, np_)

    def adamw(self, p, g, m, v, vmax, p_lp, n, *, lr, beta1, beta2, eps, wd, step, grad_scale=1.0,
              grad_scale_dev=None, dyn=None):
        self.calls.append(("adamw", n))
        self._apply(p, g, m, v, vmax, p_lp, lr=lr, beta1=beta1, beta2=beta2, eps=eps, wd=wd, step=step,
                    grad_scale=grad_scale, grad_scale_dev=grad_scale_dev)

    def adamw_mt(self, p, m, v, vmax, p_lp, table, *, lr, beta1, beta2, eps, wd, step, grad_scale=1.0,
                 grad_scale_dev=None, dyn=None):
        self.calls.append(("adamw_mt", table.n_segs))
        cut = lambda t, s: None if t is None else t[s.offset:s.end]  # noqa: E731
        for i, s in enumerate(table.slots):
            row = table._segs[i]
            g = torch.from_numpy(_read(row.g, s.numel, row.g_dtype))
            self._apply(cut(p, s), g, cut(m, s), cut(v, s), cut(vmax, s), cut(p_lp, s) if s.is_model else None,
                        lr=lr, beta1=beta1, beta2=beta2, eps=eps, wd=wd, step=step, grad_scale=grad_scale,
                        grad_scale_dev=grad_scale_dev)

    def adamw8_mt(self, p, m_q, v_q, m_absmax, v_absmax, p_lp, table, qbase, flags, *, lr, beta1, beta2, eps, wd,
                  step, grad_scale=1.0, grad_scale_dev=None, dyn=None):
        self.calls.append(("adamw8_mt", table.n_segs))
        c = float(grad_scale_dev.item()) if grad_scale_dev is not None else 1.0
        fl = flags.tolist()
        for i, s in enumerate(table.slots):
            row = table._segs[i]
            g = _read(row.g, s.numel, row.g_dtype)
            gs = grad_scale * (c if fl[i] & self.LW_CLIPPED else 1.0)
            sl, bl = slice(s.offset, s.end), self._blocks(qbase, i, s)
            w, (mq, ma), (vq, va), _, _ = adamw8_step(
                p[sl].numpy().copy(), g, m_q[sl].numpy(), m_absmax[bl].numpy(), v_q[sl].numpy(),
                v_absmax[bl].numpy(), lr=lr, beta1=beta1, beta2=beta2, eps=eps, wd=wd, step=step, grad_scale=gs)
            p[sl] = torch.from_numpy(w)
            m_q[sl], v_q[sl] = torch.from_numpy(mq), torch.from_numpy(vq)
            m_absmax[bl], v_absmax[bl] = torch.from_numpy(ma), torch.from_numpy(va)
            if p_lp is not None and s.is_model:
                p_lp[sl] = torch.from_numpy(w).to(p_lp.dtype)

    def nvls_adamw(self, p, m, v, vmax, mc_g, mc_out, n, link, *, lr, beta1, beta2, eps, wd, step, grad_scale,
                   g_dtype, dyn=None):
        """This rank's 1/world shard of the bucket (csrc/nvls.cu's split), the gradient read at
        ``mc_g`` (already reduced) and the new weights written at ``mc_out`` in the gradient's dtype."""
        self.calls.append(("nvls_adamw", n))
        per = ((n + link.world - 1) // link.world + 7) // 8 * 8
        lo = min(link.rank * per, n)
        hi = min(lo + per, n)
        if hi <= lo:
            return
        esz = 2 if g_dtype else 4
        g = torch.from_numpy(_read(mc_g + lo * esz, hi - lo, g_dtype))
        cut = lambda t: None if t is None else t[lo:hi]  # noqa: E731
        self._apply(cut(p), g, cut(m), cut(v), cut(vmax), None, lr=lr, beta1=beta1, beta2=beta2, eps=eps, wd=wd,
                    step=step, grad_scale=grad_scale)
        w = p[lo:hi].detach().numpy()
        out = np.ctypeslib.as_array((np.ctypeslib.ctypes.c_uint8 * ((hi - lo) * esz)).from_address(mc_out + lo * esz))
        src = torch.from_numpy(w).to(torch.bfloat16).view(torch.int16).numpy() if g_dtype else w
        out[:] = np.frombuffer(np.ascontiguousarray(src).tobytes(), dtype=np.uint8)
