"""TEST INFRASTRUCTURE — numpy restatement of K5p's draws (``frl_augment_policy_images``,
include/frl_b200.h): the policy's ops, bins and signs and the random-erasing box, on K5a's
Philox4x32-10 stream (oracle/augment_np.py) at blocks 11 and above.  Never imported by the product.
"""
import math

import numpy as np

from oracle.augment_np import below, draws, uniform

OP_BLOCK, ERASE_BLOCK = 11, 15
N_OPS = 14
SIGNED = set(range(1, 10))              # ShearX .. Sharpness
NO_MAGNITUDE = {0, 12, 13}              # Identity, AutoContrast, Equalize
TRIVIAL_AUGMENT, RAND_AUGMENT = 1, 2


def policy_ops(idx, *, seed: int, epoch: int, policy: int, num_ops: int, num_bins: int, magnitude: int = 0):
    """int32 [N, num_ops, 3]: (op, bin, sign) of every op of every sample."""
    idx = np.asarray(idx, dtype=np.int64)
    out = np.zeros((idx.size, num_ops, 3), np.int32)
    for k in range(num_ops):
        r = draws(idx, seed, epoch, OP_BLOCK + k)
        op = below(r[0], N_OPS)
        b = below(r[1], num_bins) if policy == TRIVIAL_AUGMENT else np.full(idx.size, magnitude, np.int64)
        neg = (r[2] >> np.uint32(31)).astype(bool) & np.isin(op, list(SIGNED))
        b = np.where(np.isin(op, list(NO_MAGNITUDE)), 0, b)
        out[:, k, 0], out[:, k, 1], out[:, k, 2] = op, b, np.where(neg, -1, 1)
    return out


def erase_boxes(idx, *, seed: int, epoch: int, out_h: int, out_w: int, p: float, scale=(0.02, 0.33),
                ratio=(0.3, 3.3)):
    """int32 [N, 5]: (erased, top, left, h, w) of every sample."""
    idx = np.asarray(idx, dtype=np.int64)
    out = np.zeros((idx.size, 5), np.int32)
    if p <= 0.0:
        return out
    apply = uniform(draws(idx, seed, epoch, ERASE_BLOCK)[0]) < p
    lmin, lmax = math.log(ratio[0]), math.log(ratio[1])
    done = ~apply
    for t in range(10):
        r = draws(idx, seed, epoch, ERASE_BLOCK + 1 + t)
        area = float(out_h * out_w) * (scale[0] + uniform(r[0]) * (scale[1] - scale[0]))
        aspect = np.exp(lmin + uniform(r[1]) * (lmax - lmin))
        h = np.rint(np.sqrt(area * aspect)).astype(np.int64)
        w = np.rint(np.sqrt(area / aspect)).astype(np.int64)
        ok = ~done & (h < out_h) & (w < out_w)
        out[ok, 0] = 1
        out[ok, 1] = below(r[2], out_h - h + 1)[ok]
        out[ok, 2] = below(r[3], out_w - w + 1)[ok]
        out[ok, 3], out[ok, 4] = h[ok], w[ok]
        done |= ok
    return out
