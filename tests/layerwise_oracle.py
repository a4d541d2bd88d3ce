"""TEST INFRASTRUCTURE for the layer-wise adaptive updates (LARS, LAMB).

* ``lars_step`` / ``lamb_step``: a numpy restatement of ``types.LayerAdaptation`` written from
  its formulas, per tensor: element-wise arithmetic in fp32, norms in float64.
* ``LayerwiseKernelDouble``: ``oracle.optim_np.KernelDouble`` plus CPU stand-ins for
  ``_native.lars_mt`` / ``_native.lamb_mt`` that read each gradient where the segment table points,
  so multi-rank host logic runs under gloo without a GPU.
* ``LayerwiseTorch``: a plain per-parameter ``torch.optim.Optimizer`` for LARS and LAMB, the
  end-to-end oracle against stock torch.

Never imported by the product.
"""
import ctypes as C
import math

import numpy as np
import torch

from oracle.optim_np import KernelDouble

f32 = np.float32
LARS_TRUST = 1e-3


def _norm(x):
    return float(np.sqrt(np.sum(np.asarray(x, dtype=np.float64) ** 2)))


def lars_step(w, g, buf, *, lr, mu, wd, adapted, first_step, grad_scale=1.0):
    """Returns (w, buf, ratio)."""
    g = (g.astype(f32) * f32(grad_scale)).astype(f32)
    ratio = 1.0
    if adapted:
        wn, gn = _norm(w), _norm(g)
        if wn > 0 and gn > 0:
            ratio = LARS_TRUST * wn / (gn + wd * wn)
        d = (f32(ratio) * (g + f32(wd) * w)).astype(f32)
    else:
        d = g
    if mu != 0:
        buf = d.copy() if first_step else (f32(mu) * buf + d).astype(f32)
        d = buf
    return (w - f32(lr) * d).astype(f32), buf, ratio


def lamb_step(w, g, m, v, *, lr, beta1, beta2, eps, wd, step, adapted, grad_scale=1.0):
    """Returns (w, m, v, ratio)."""
    g = (g.astype(f32) * f32(grad_scale)).astype(f32)
    m = (m + f32(1 - beta1) * (g - m)).astype(f32)
    v = (v * f32(beta2) + f32(1 - beta2) * g * g).astype(f32)
    bc1 = 1 - beta1 ** step
    bc2 = 1 - beta2 ** step
    lam = wd if adapted else 0.0
    u = ((m * f32(1.0 / bc1)) / (np.sqrt(v) / f32(math.sqrt(bc2)) + f32(eps)) + f32(lam) * w).astype(f32)
    ratio = 1.0
    if adapted:
        wn, un = _norm(w), _norm(u)
        if wn > 0 and un > 0:
            ratio = wn / un
    return (w - (f32(lr) * f32(ratio)) * u).astype(f32), m, v, ratio


def _read(ptr, n, code):
    """n elements of an fp32 (code 0) or bf16 (code 1) array at address ``ptr`` (CPU memory)."""
    if code == 0:
        return np.ctypeslib.as_array((C.c_float * n).from_address(ptr)).copy()
    u = np.ctypeslib.as_array((C.c_uint16 * n).from_address(ptr)).astype(np.uint32) << 16
    return u.view(f32)


class LayerwiseKernelDouble(KernelDouble):
    LW_ADAPTED, LW_CLIPPED = 1, 2

    def layerwise_scratch_bytes(self, n_tiles, n_segs):
        return 16

    def _segments(self, table, flags, coef, grad_scale):
        fl = flags.tolist()
        c = float(coef.item()) if coef is not None else 1.0
        for i, s in enumerate(table.slots):
            row = table._segs[i]
            g = _read(row.g, s.numel, row.g_dtype)
            gs = grad_scale * (c if fl[i] & self.LW_CLIPPED else 1.0)
            yield i, s, g, gs, bool(fl[i] & self.LW_ADAPTED)

    @staticmethod
    def _put(vec, s, arr):
        if vec is not None:
            vec[s.offset:s.end] = torch.from_numpy(np.asarray(arr, dtype=f32)).to(vec.dtype)

    def lars_mt(self, p, buf, p_lp, table, flags, ratio, scratch, *, lr, mu, wd, grad_scale=1.0,
                grad_scale_dev=None, first_step=False, dyn=None):
        self.calls.append(("lars_mt", table.n_segs))
        for i, s, g, gs, adapted in self._segments(table, flags, grad_scale_dev, grad_scale):
            b = buf[s.offset:s.end].numpy() if buf is not None else None
            w, nb, r = lars_step(p[s.offset:s.end].numpy().copy(), g, b, lr=lr, mu=mu, wd=wd,
                                 adapted=adapted, first_step=first_step, grad_scale=gs)
            self._put(p, s, w); self._put(buf, s, nb)
            if p_lp is not None and s.is_model:
                self._put(p_lp, s, w)
            ratio[i] = r

    def lamb_mt(self, p, m, v, p_lp, table, flags, ratio, scratch, *, lr, beta1, beta2, eps, wd, step,
                grad_scale=1.0, grad_scale_dev=None, dyn=None):
        self.calls.append(("lamb_mt", table.n_segs))
        for i, s, g, gs, adapted in self._segments(table, flags, grad_scale_dev, grad_scale):
            w, nm, nv, r = lamb_step(p[s.offset:s.end].numpy().copy(), g, m[s.offset:s.end].numpy(),
                                     v[s.offset:s.end].numpy(), lr=lr, beta1=beta1, beta2=beta2, eps=eps,
                                     wd=wd, step=step, adapted=adapted, grad_scale=gs)
            self._put(p, s, w); self._put(m, s, nm); self._put(v, s, nv)
            if p_lp is not None and s.is_model:
                self._put(p_lp, s, w)
            ratio[i] = r


class LayerwiseTorch(torch.optim.Optimizer):
    """Per-parameter LARS / LAMB in stock torch (``mode`` "lars" or "lamb"), one step count per
    parameter like ``torch.optim.Adam``.  Parameters with 2 or more dimensions are adapted.
    ``last_ratio[p]``: the trust ratio of ``p``'s last update (1.0 where it is not adapted)."""

    def __init__(self, params, mode, lr, momentum=0.9, weight_decay=0.0, betas=(0.9, 0.999), eps=1e-8):
        assert mode in ("lars", "lamb")
        self.mode = mode
        self.last_ratio = {}
        super().__init__(params, dict(lr=lr, momentum=momentum, weight_decay=weight_decay, betas=betas,
                                      eps=eps))

    @torch.no_grad()
    def step(self, closure=None):
        for group in self.param_groups:
            lr, wd = group["lr"], group["weight_decay"]
            for p in group["params"]:
                if p.grad is None:
                    continue
                g = p.grad
                adapted = p.dim() >= 2
                st = self.state[p]
                if self.mode == "lars":
                    if adapted:
                        wn, gn = float(p.norm()), float(g.norm())
                        ratio = LARS_TRUST * wn / (gn + wd * wn) if wn > 0 and gn > 0 else 1.0
                        d = (g + wd * p) * ratio
                    else:
                        ratio, d = 1.0, g.clone()
                    mu = group["momentum"]
                    if mu != 0:
                        if "momentum_buffer" not in st:
                            st["momentum_buffer"] = d.clone()
                        else:
                            st["momentum_buffer"].mul_(mu).add_(d)
                        d = st["momentum_buffer"]
                    p.add_(d, alpha=-lr)
                    self.last_ratio[p] = ratio
                else:
                    b1, b2 = group["betas"]
                    if not st:
                        st["step"] = torch.tensor(0.0)
                        st["exp_avg"] = torch.zeros_like(p)
                        st["exp_avg_sq"] = torch.zeros_like(p)
                    st["step"] += 1
                    t = float(st["step"])
                    st["exp_avg"].lerp_(g, 1 - b1)
                    st["exp_avg_sq"].mul_(b2).addcmul_(g, g, value=1 - b2)
                    u = (st["exp_avg"] / (1 - b1 ** t)) / (st["exp_avg_sq"].sqrt() / math.sqrt(1 - b2 ** t)
                                                         + group["eps"])
                    if adapted:
                        u = u + wd * p
                    wn, un = float(p.norm()), float(u.norm())
                    ratio = wn / un if adapted and wn > 0 and un > 0 else 1.0
                    p.add_(u, alpha=-lr * ratio)
                    self.last_ratio[p] = ratio


# ---- float64 reference of one K2-lw update and its fp32 rounding envelope --------------------------
# (derivation of the constants: tests/test_gpu_layerwise_paths.py's module docstring)

U, ETA = 2.0 ** -24, 2.0 ** -150
C_LARS, C_R_LARS = 16, 8            # weights / momentum buffer; trust ratio (relative)
C_LAMB, C_R_LAMB = 24, 24           # weights, exp_avg, exp_avg_sq; trust ratio (relative, times kappa)
BETAS, LAMB_EPS = (0.9, 0.999), 1e-6


def reference_update(mode, w0, g, s0, *, adapted, lr, mu, wd, step, dtype=torch.float64):
    """One ``LayerwiseTorch`` step of one tensor in ``dtype`` from the fp32 state ``w0``, ``s0``
    (LARS: [momentum_buffer] or [], LAMB: [exp_avg, exp_avg_sq]) with effective gradient ``g``;
    ``step`` is t (LARS: 1 = first step).  Returns (w, states, ratio) as float64 / float."""
    shape = (1, w0.numel()) if adapted else (w0.numel(),)
    param = torch.nn.Parameter(w0.to(dtype).reshape(shape).clone())
    opt = LayerwiseTorch([param], mode, lr=lr, momentum=mu, weight_decay=wd, betas=BETAS, eps=LAMB_EPS)
    st = opt.state[param]
    if mode == "lars":
        names = ("momentum_buffer",) if mu else ()
        if mu and step > 1:
            st["momentum_buffer"] = s0[0].to(dtype).reshape(shape).clone()
    else:
        names = ("exp_avg", "exp_avg_sq")
        st["step"] = torch.tensor(float(step - 1))
        st["exp_avg"], st["exp_avg_sq"] = (s.to(dtype).reshape(shape).clone() for s in s0)
    param.grad = g.to(dtype).reshape(shape)
    opt.step()
    return (param.detach().flatten().double(), [st[n].flatten().double() for n in names],
            opt.last_ratio[param])


def update_envelope(mode, w0, g, s0, ref_w, ref_s, ratio, *, adapted, lr, mu, wd, step):
    """(bound on the weights, bounds on the states, kappa): c * (U * mag + ETA) per element, and the
    trust ratio's relative bound is C_R * U * kappa.  kappa = 0 where the rule takes ratio 1
    (exact), else ||mag(u)|| / ||u|| (1 for LARS)."""
    w0, g = w0.double(), g.double()
    s0 = [s.double() for s in s0]
    if mode == "lars":
        dn = float(g.norm())
        kappa = 1.0 if adapted and float(w0.norm()) > 0 and dn > 0 else 0.0
        mag = ratio * (g.abs() + (wd * w0.abs() if adapted else 0.0))
        if mu and step > 1:
            mag = mu * s0[0].abs() + mag
        c, mags, step_mag = C_LARS, ([mag] if mu else []), lr * mag
    else:
        b1, b2 = BETAS
        lam = wd if adapted else 0.0
        bc1, bc2 = 1 - b1 ** step, 1 - b2 ** step
        mag_m = s0[0].abs() + (1 - b1) * (g.abs() + s0[0].abs())
        mag_v = b2 * s0[1] + (1 - b2) * g * g
        denom = ref_s[1].sqrt() / math.sqrt(bc2) + LAMB_EPS
        u = ref_s[0] / bc1 / denom + lam * w0
        mag_u = mag_m / bc1 / denom + lam * w0.abs()
        un = float(u.norm())
        kappa = float(mag_u.norm()) / un if adapted and float(w0.norm()) > 0 and un > 0 else 0.0
        c, mags, step_mag = C_LAMB, [mag_m, mag_v], lr * ratio * (mag_u + kappa * u.abs())
    return c * (U * (ref_w.abs() + step_mag) + ETA), [c * (U * m + ETA) for m in mags], kappa


def check_update(mode, got_w, got_s, got_ratio, w0, g, s0, *, adapted, lr, mu, wd, step, what,
                 dtype=torch.float64):
    """The kernel's update of one tensor (``got_*``, fp32) from (w0, s0) with effective gradient
    ``g`` against ``reference_update`` in ``dtype`` (fp32 only where fp32 storage itself
    overflows; both sides then carry their own error, so the bounds double)."""
    from test_gpu_optim_paths import assert_within
    ref_w, ref_s, r = reference_update(mode, w0, g, s0, adapted=adapted, lr=lr, mu=mu, wd=wd, step=step,
                                       dtype=dtype)
    bw, bs, kappa = update_envelope(mode, w0, g, s0, ref_w, ref_s, r, adapted=adapted, lr=lr, mu=mu, wd=wd,
                                    step=step)
    k = 1 if dtype == torch.float64 else 2
    assert_within(got_w, ref_w, k * bw, what + " weights")
    for i, (got, ref, b) in enumerate(zip(got_s, ref_s, bs)):
        assert_within(got, ref, k * b, "%s state %d" % (what, i))
    if kappa == 0:
        assert got_ratio == 1.0, "%s: ratio %r, want exactly 1" % (what, got_ratio)
    else:
        c_r = C_R_LARS if mode == "lars" else C_R_LAMB
        assert abs(got_ratio - r) <= k * c_r * U * kappa * abs(r), \
            "%s: ratio %r, float64 %r (kappa %.3g)" % (what, got_ratio, r, kappa)
    return r
