"""TEST INFRASTRUCTURE for 8-bit block-wise Adam state (K2-q8).

* ``MAG7`` / ``MAG8``, ``encode`` / ``decode``, ``adam8_step``: a numpy restatement of the storage
  format of ``types.OptimizerState.Q8`` written from its definition (include/frl_b200.h, K2-q8):
  tables formed in float64 and rounded once to fp32, blocks of 256 elements from a tensor's
  first element, NaN-propagating absmax, IEEE fp32 ``r = |x| / absmax``, nearest entry with ties
  to the smaller index (distances compared in float64, where they are exact).
* ``Adam8KernelDouble``: ``oracle.optim_np.KernelDouble`` plus CPU stand-ins for
  ``_native.adam8_mt`` / ``q8_encode_mt`` / ``q8_decode_mt`` that read each gradient where the
  segment table points, so the host logic (and multi-rank runs under gloo) needs no GPU.

Never imported by the product.
"""
import ctypes as C

import numpy as np
import torch

from oracle.optim_np import KernelDouble, adam_step

f32 = np.float32
BLOCK = 256


def _tables():
    mag7, mag8 = [0.0], [0.0]
    for i in range(7):
        dec = [1e-6, 1e-5, 1e-4, 1e-3, 1e-2, 1e-1, 1.0][i]
        mag7 += [dec * (0.1 + 0.9 * (j + 0.5) / 2 ** i) for j in range(2 ** i)]
        mag8 += [dec * (0.1 + 0.9 * (j + 0.5) / 2 ** (i + 1)) for j in range(2 ** (i + 1))]
    assert mag7[-1] == 0.99296875
    mag7[-1] = 1.0
    mag8.append(1.0)
    return np.array(mag7, dtype=f32), np.array(mag8, dtype=f32)


MAG7, MAG8 = _tables()


def nearest(table, r):
    """Index of the entry of ``table`` nearest to each fp32 ``r`` (ties to the smaller index, NaN -> 0)."""
    r = np.asarray(r, dtype=f32)
    lo = np.searchsorted(table, r, side="right") - 1          # largest i with table[i] <= r
    lo = np.where(np.isnan(r), 0, np.clip(lo, 0, len(table) - 1))
    hi = np.minimum(lo + 1, len(table) - 1)
    rd = r.astype(np.float64)
    up = (hi > lo) & (table[hi].astype(np.float64) - rd < rd - table[lo].astype(np.float64))
    return np.where(up, hi, lo).astype(np.uint8)


def _absmax(x):
    a = np.abs(x)
    return f32(np.nan) if np.isnan(a).any() else (f32(a.max()) if a.size else f32(0))


def encode(x, signed):
    """Codes (uint8, len(x)) and per-block absmax (fp32) of one tensor's flat fp32 values."""
    x = np.asarray(x, dtype=f32).ravel()
    n_blocks = (x.size + BLOCK - 1) // BLOCK
    codes = np.zeros(x.size, dtype=np.uint8)
    amax = np.zeros(n_blocks, dtype=f32)
    table = MAG7 if signed else MAG8
    for b in range(n_blocks):
        blk = x[b * BLOCK:(b + 1) * BLOCK]
        a = _absmax(blk)
        with np.errstate(invalid="ignore", divide="ignore"):
            r = np.zeros_like(blk) if a == 0 else (np.abs(blk) / a).astype(f32)
        k = nearest(table, r)
        if signed:
            k = k | (np.signbit(blk).astype(np.uint8) << 7)
        codes[b * BLOCK:(b + 1) * BLOCK] = k
        amax[b] = a
    return codes, amax


def decode(codes, amax, signed):
    codes = np.asarray(codes, dtype=np.uint8)
    a = np.repeat(np.asarray(amax, dtype=f32), BLOCK)[:codes.size]
    with np.errstate(invalid="ignore"):
        if signed:
            y = (MAG7[codes & 0x7F] * a).astype(f32)
            return np.where(codes & 0x80, -y, y).astype(f32)
        return (MAG8[codes] * a).astype(f32)


def adam8_step(p, g, mq, ma, vq, va, *, lr, beta1, beta2, eps, wd, step, grad_scale=1.0):
    """One K2-q8 step of one tensor: decode, Adam in fp32 (oracle.optim_np.adam_step), encode.
    Returns (p, (mq, ma), (vq, va), m, v) with m, v the fp32 moments before encoding."""
    m, v = decode(mq, ma, True), decode(vq, va, False)
    with np.errstate(invalid="ignore", over="ignore"):
        p, m, v, _ = adam_step(p, g, m, v, None, lr=lr, beta1=beta1, beta2=beta2, eps=eps, wd=wd, step=step,
                               grad_scale=grad_scale)
    return p, encode(m, True), encode(v, False), m, v


def _read(ptr, n, code):
    if code == 0:
        return np.ctypeslib.as_array((C.c_float * n).from_address(ptr)).copy()
    u = np.ctypeslib.as_array((C.c_uint16 * n).from_address(ptr)).astype(np.uint32) << 16
    return u.view(f32)


class Adam8KernelDouble(KernelDouble):
    LW_ADAPTED, LW_CLIPPED = 1, 2
    Q8_EXP_AVG, Q8_EXP_AVG_SQ = 0, 1

    @staticmethod
    def _blocks(qbase, i, s):
        b0 = int(qbase[i])
        return slice(b0, b0 + (s.numel + BLOCK - 1) // BLOCK)

    def adam8_mt(self, p, m_q, v_q, m_absmax, v_absmax, p_lp, table, qbase, flags, *, lr, beta1, beta2, eps, wd,
                 step, grad_scale=1.0, grad_scale_dev=None, dyn=None):
        self.calls.append(("adam8_mt", table.n_segs))
        c = float(grad_scale_dev.item()) if grad_scale_dev is not None else 1.0
        fl = flags.tolist()
        for i, s in enumerate(table.slots):
            row = table._segs[i]
            g = _read(row.g, s.numel, row.g_dtype)
            gs = grad_scale * (c if fl[i] & self.LW_CLIPPED else 1.0)
            sl, bl = slice(s.offset, s.end), self._blocks(qbase, i, s)
            w, (mq, ma), (vq, va), _, _ = adam8_step(
                p[sl].numpy().copy(), g, m_q[sl].numpy(), m_absmax[bl].numpy(), v_q[sl].numpy(),
                v_absmax[bl].numpy(), lr=lr, beta1=beta1, beta2=beta2, eps=eps, wd=wd, step=step, grad_scale=gs)
            p[sl] = torch.from_numpy(w)
            m_q[sl], v_q[sl] = torch.from_numpy(mq), torch.from_numpy(vq)
            m_absmax[bl], v_absmax[bl] = torch.from_numpy(ma), torch.from_numpy(va)
            if p_lp is not None and s.is_model:
                p_lp[sl] = torch.from_numpy(w).to(p_lp.dtype)

    def q8_encode_mt(self, x, q, absmax, state, table, qbase):
        self.calls.append(("q8_encode_mt", table.n_segs))
        for i, s in enumerate(table.slots):
            codes, a = encode(x[s.offset:s.end].numpy(), state == self.Q8_EXP_AVG)
            q[s.offset:s.end] = torch.from_numpy(codes)
            absmax[self._blocks(qbase, i, s)] = torch.from_numpy(a)

    def q8_decode_mt(self, q, absmax, x, state, table, qbase):
        self.calls.append(("q8_decode_mt", table.n_segs))
        for i, s in enumerate(table.slots):
            x[s.offset:s.end] = torch.from_numpy(
                decode(q[s.offset:s.end].numpy(), absmax[self._blocks(qbase, i, s)].numpy(),
                       state == self.Q8_EXP_AVG))
