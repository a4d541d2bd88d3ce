"""TEST INFRASTRUCTURE — numpy restatement of the K5a sample parameters (``frl_augment_images``,
include/frl_b200.h): Philox4x32-10 and the per-sample crop box / flip of the random resized crop,
the zero-padded random crop and the two centre crops.  Vectorised over sample indices; the
arithmetic is the header's, in float64 (the box) and uint32 / uint64 (the draws).

The random resized crop follows torchvision's ``RandomResizedCrop.get_params`` with Philox words
in place of torch's generator.  Never imported by the product.
"""
import math

import numpy as np

RRC, PAD_CROP, CENTER_RESIZE, CENTER_CROP = 0, 1, 2, 3
_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = 0x9E3779B9, 0xBB67AE85
_MASK = np.uint64(0xFFFFFFFF)
FLIP_BLOCK = 10


def philox4x32_10(ctr, key):
    """Philox4x32-10 (Salmon et al., SC'11).  ``ctr``: 4 uint32 arrays (broadcastable),
    ``key``: 2 Python ints.  Returns 4 uint32 arrays."""
    c = [np.asarray(x, dtype=np.uint64) & _MASK for x in np.broadcast_arrays(*ctr)]
    k0, k1 = int(key[0]) & 0xFFFFFFFF, int(key[1]) & 0xFFFFFFFF
    for _ in range(10):
        p0 = _M0 * c[0]
        p1 = _M1 * c[2]
        hi0, lo0 = p0 >> np.uint64(32), p0 & _MASK
        hi1, lo1 = p1 >> np.uint64(32), p1 & _MASK
        c = [hi1 ^ c[1] ^ np.uint64(k0), lo1, hi0 ^ c[3] ^ np.uint64(k1), lo0]
        k0, k1 = (k0 + _W0) & 0xFFFFFFFF, (k1 + _W1) & 0xFFFFFFFF
    return [x.astype(np.uint32) for x in c]


def draws(idx, seed: int, epoch: int, block: int):
    idx = np.asarray(idx, dtype=np.int64).astype(np.uint64)
    key = (seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
    return philox4x32_10((idx & _MASK, idx >> np.uint64(32), np.uint64(epoch), np.uint64(block)), key)


def uniform(w):
    """u(w) = (w >> 8) * 2^-24, exact in float64."""
    return (w >> np.uint32(8)).astype(np.float64) * (1.0 / 16777216.0)


def below(w, n):
    """An integer in [0, n): (uint64(w) * n) >> 32."""
    return ((w.astype(np.uint64) * np.asarray(n, dtype=np.uint64)) >> np.uint64(32)).astype(np.int64)


def sample_params(idx, *, seed: int, epoch: int, mode: int, height: int, width: int, out_h: int, out_w: int,
                  scale=(0.08, 1.0), ratio=(3.0 / 4.0, 4.0 / 3.0), pad: int = 0, eval_crop: float = 0.875,
                  flip: bool = True, with_raw: bool = False):
    """int32 [N, 5] of (top, left, h, w, flipped) per sample.  ``with_raw``: also the float64
    pre-rounding (w, h) of the accepted RRC attempt (NaN where the fallback was taken, and in the
    other modes) and a bool [N] that marks fallback samples."""
    idx = np.asarray(idx, dtype=np.int64)
    n = idx.size
    H, W = int(height), int(width)
    top = np.zeros(n, np.int64)
    left = np.zeros(n, np.int64)
    h = np.full(n, out_h, np.int64)
    w = np.full(n, out_w, np.int64)
    raw = np.full((n, 2), np.nan)
    fallback = np.zeros(n, bool)
    if mode == RRC:
        smin, smax = float(scale[0]), float(scale[1])
        lmin, lmax = math.log(ratio[0]), math.log(ratio[1])
        done = np.zeros(n, bool)
        for t in range(10):
            r = draws(idx, seed, epoch, t)
            area = float(H * W) * (smin + uniform(r[0]) * (smax - smin))
            aspect = np.exp(lmin + uniform(r[1]) * (lmax - lmin))
            sw, sh = np.sqrt(area * aspect), np.sqrt(area / aspect)
            ww, hh = np.rint(sw), np.rint(sh)
            ok = ~done & (ww > 0) & (ww <= W) & (hh > 0) & (hh <= H)
            h[ok], w[ok] = hh[ok].astype(np.int64), ww[ok].astype(np.int64)
            top[ok] = below(r[2], H - h + 1)[ok]
            left[ok] = below(r[3], W - w + 1)[ok]
            raw[ok, 0], raw[ok, 1] = sw[ok], sh[ok]
            done |= ok
        fallback = ~done
        if fallback.any():
            in_ratio = W / H
            if in_ratio < ratio[0]:
                fw, fh = W, int(np.rint(W / ratio[0]))
            elif in_ratio > ratio[1]:
                fh, fw = H, int(np.rint(H * ratio[1]))
            else:
                fw, fh = W, H
            fw, fh = max(fw, 1), max(fh, 1)
            w[fallback], h[fallback] = fw, fh
            top[fallback], left[fallback] = (H - fh) // 2, (W - fw) // 2
    elif mode == PAD_CROP:
        r = draws(idx, seed, epoch, 0)
        top = below(r[0], H + 2 * pad - out_h + 1) - pad
        left = below(r[1], W + 2 * pad - out_w + 1) - pad
    elif mode in (CENTER_RESIZE, CENTER_CROP):
        ch, cw = (int(np.rint(H * eval_crop)), int(np.rint(W * eval_crop))) if mode == CENTER_RESIZE else (out_h, out_w)
        h[:], w[:] = ch, cw
        top[:], left[:] = int(np.rint(0.5 * (H - ch))), int(np.rint(0.5 * (W - cw)))
    else:
        raise ValueError(mode)
    flipped = np.zeros(n, np.int64)
    if flip and mode in (RRC, PAD_CROP):
        flipped = (draws(idx, seed, epoch, FLIP_BLOCK)[0] >> np.uint32(31)).astype(np.int64)
    out = np.stack([top, left, h, w, flipped], 1).astype(np.int32)
    return (out, raw, fallback) if with_raw else out
