"""TEST INFRASTRUCTURE — numpy restatement of the torch.optim update rules the reference
selects in ``_create_optimizer`` (reference solver.py:162-188), as published in torch 2.11's
``torch/optim/{sgd,adam,rmsprop}.py`` single-tensor paths.  Computed in fp32 with the same
operation order, so it doubles as an independent check of torch.optim itself
(tests/test_oracle_pinning.py) and as the checker for the K2 kernels.

Also usable as a drop-in *test double* for the kernel entry points of
``frl_b200._native`` on CPU tensors (``KernelDouble``) so multi-rank host logic can be tested
under gloo without a GPU.  Never imported by the product.
"""
import numpy as np

f32 = np.float32


def sgd_step(p, g, buf, *, lr, mu, dampening, wd, first_step, grad_scale=1.0):
    """torch/optim/sgd.py _single_tensor_sgd: g += wd*p; buf = g (first) | mu*buf + (1-d)*g."""
    g = (g.astype(f32) * f32(grad_scale)).astype(f32)
    d_p = (g + f32(wd) * p).astype(f32)
    if mu != 0:
        if first_step:
            buf = d_p.copy()
        else:
            buf = (f32(mu) * buf + f32(1 - dampening) * d_p).astype(f32)
        d_p = buf
    p = (p + f32(-lr) * d_p).astype(f32)
    return p, buf


def adam_step(p, g, m, v, vmax, *, lr, beta1, beta2, eps, wd, step, grad_scale=1.0):
    """torch/optim/adam.py _single_tensor_adam (L2-coupled weight decay, optional amsgrad)."""
    g = (g.astype(f32) * f32(grad_scale)).astype(f32)
    g = (g + f32(wd) * p).astype(f32)
    m = (m + f32(1 - beta1) * (g - m)).astype(f32)                       # lerp_
    v = (v * f32(beta2) + f32(1 - beta2) * g * g).astype(f32)            # mul_.addcmul_
    bc1 = 1 - beta1 ** step
    bc2 = 1 - beta2 ** step
    step_size = lr / bc1
    bc2_sqrt = bc2 ** 0.5
    if vmax is not None:
        vmax = np.maximum(vmax, v)
        denom = (np.sqrt(vmax) / f32(bc2_sqrt) + f32(eps)).astype(f32)
    else:
        denom = (np.sqrt(v) / f32(bc2_sqrt) + f32(eps)).astype(f32)
    p = (p + f32(-step_size) * (m / denom)).astype(f32)                  # addcdiv_
    return p, m, v, vmax


def rmsprop_step(p, g, sq, buf, *, lr, alpha, eps, wd, mu, grad_scale=1.0):
    """torch/optim/rmsprop.py _single_tensor_rmsprop (not centered)."""
    g = (g.astype(f32) * f32(grad_scale)).astype(f32)
    g = (g + f32(wd) * p).astype(f32)
    sq = (sq * f32(alpha) + f32(1 - alpha) * g * g).astype(f32)
    avg = (np.sqrt(sq) + f32(eps)).astype(f32)
    if mu > 0:
        buf = (buf * f32(mu) + g / avg).astype(f32)
        p = (p + f32(-lr) * buf).astype(f32)
    else:
        p = (p + f32(-lr) * (g / avg)).astype(f32)
    return p, sq, buf


def clip_coef(g_model, max_norm, pre_scale=1.0):
    """torch.nn.utils.clip_grad_norm_: clamp(max_norm / (||g||_2 + 1e-6), max=1).  A NaN norm
    gives a NaN coefficient (Python's min(1.0, nan) would give 1.0)."""
    norm = float(np.sqrt(np.sum((g_model.astype(np.float64) * pre_scale) ** 2)))
    coef = max_norm / (norm + 1e-6)
    return (1.0 if coef > 1.0 else coef), norm


def bf16_round(x):
    """fp32 -> bf16 -> fp32, round-to-nearest-even (what the shadow weights hold)."""
    u = np.ascontiguousarray(x, dtype=f32).view(np.uint32).astype(np.uint64)
    r = ((u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000).astype(np.uint32)
    return r.view(f32)


class KernelDouble:
    """CPU stand-in with the call signatures of ``frl_b200._native`` (tests only)."""

    def __init__(self):
        self.calls = []

    @staticmethod
    def _np(t):
        import torch
        return None if t is None else t.detach().to(torch.float32).numpy()

    @staticmethod
    def _store(t, arr):
        import torch
        if t is not None:
            t.copy_(torch.from_numpy(np.asarray(arr, dtype=f32)).to(t.dtype))

    def _scale(self, grad_scale, grad_scale_dev):
        return grad_scale * (float(grad_scale_dev.item()) if grad_scale_dev is not None else 1.0)

    def sgd_momentum(self, p, g, buf, p_lp, n, *, lr, mu, dampening, wd, grad_scale=1.0,
                     grad_scale_dev=None, first_step=False, dyn=None):
        self.calls.append(("sgd", n))
        np_, nb = sgd_step(self._np(p), self._np(g), self._np(buf), lr=lr, mu=mu,
                           dampening=dampening, wd=wd, first_step=first_step,
                           grad_scale=self._scale(grad_scale, grad_scale_dev))
        self._store(p, np_); self._store(buf, nb); self._store(p_lp, np_)

    def adam(self, p, g, m, v, vmax, p_lp, n, *, lr, beta1, beta2, eps, wd, step, grad_scale=1.0,
             grad_scale_dev=None, dyn=None):
        self.calls.append(("adam", n))
        np_, nm, nv, nvm = adam_step(self._np(p), self._np(g), self._np(m), self._np(v),
                                     self._np(vmax), lr=lr, beta1=beta1, beta2=beta2, eps=eps,
                                     wd=wd, step=step,
                                     grad_scale=self._scale(grad_scale, grad_scale_dev))
        self._store(p, np_); self._store(m, nm); self._store(v, nv); self._store(vmax, nvm)
        self._store(p_lp, np_)

    def rmsprop(self, p, g, sq, buf, p_lp, n, *, lr, alpha, eps, wd, mu, grad_scale=1.0,
                grad_scale_dev=None, dyn=None):
        self.calls.append(("rmsprop", n))
        np_, nsq, nb = rmsprop_step(self._np(p), self._np(g), self._np(sq), self._np(buf), lr=lr,
                                    alpha=alpha, eps=eps, wd=wd, mu=mu,
                                    grad_scale=self._scale(grad_scale, grad_scale_dev))
        self._store(p, np_); self._store(sq, nsq); self._store(buf, nb); self._store(p_lp, np_)

    def reduce_scratch_bytes(self):
        return 16

    def grad_sumsq_clip(self, g, n, *, pre_scale, max_norm, out3, scratch):
        self.calls.append(("sumsq", n))
        coef, norm = clip_coef(self._np(g), max_norm, pre_scale)
        self._store(out3, [norm * norm, norm, coef])

    # K6 / K6b stand-ins (bias gradient of a linear layer written into the arena)
    def colsum(self, x, out, accumulate=False):
        self.calls.append(("colsum", x.shape[1]))
        tot = x.detach().float().sum(0)
        out.copy_((out.float() + tot if accumulate else tot).to(out.dtype))

    def drelu_colsum(self, dy, act, dz, out, accumulate=False):
        import torch
        self.calls.append(("drelu_colsum", dy.shape[1]))
        dz.copy_(torch.ops.aten.threshold_backward(dy, act, 0))     # ReLU's backward: dy unless act <= 0
        tot = dz.float().sum(0)
        out.copy_((out.float() + tot if accumulate else tot).to(out.dtype))
