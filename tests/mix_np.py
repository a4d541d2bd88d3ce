"""numpy restatement of the pair mix of frl_augment_mix_images / frl_mix_targets, applied to the
fp32 output of frl_augment_images on the same batch (include/frl_b200.h): sample i is mixed with
sample B-1-i, every product and sum rounded to fp32 as the kernels round them."""
import numpy as np
import torch

MIXUP, CUTMIX = 1, 2


def lams(lam):
    lam32 = np.float32(lam)
    return lam32, np.float32(1.0 - float(lam32))


def mix_images(a, mode, lam, box=(0, 0, 0, 0), dtype=torch.float32):
    """a: fp32 [B, C, H, W] (K5a's fp32 output); returns the mixed batch as a torch tensor of dtype."""
    a = np.asarray(a, dtype=np.float32)
    q = a[::-1]
    if mode == MIXUP:
        lam32, lam1 = lams(lam)
        out = (lam32 * a).astype(np.float32) + (lam1 * q).astype(np.float32)
    else:
        y0, y1, x0, x1 = box
        out = a.copy()
        out[:, :, y0:y1, x0:x1] = q[:, :, y0:y1, x0:x1]
    B = a.shape[0]
    if B % 2:
        out[B // 2] = a[B // 2]          # the middle sample of an odd batch is K5a's
    return torch.from_numpy(np.ascontiguousarray(out)).to(dtype)


def mix_labels(y, n, lam):
    y = np.asarray(y, dtype=np.int64)
    lam32, lam1 = lams(lam)
    B = y.size
    out = np.zeros((B, n), np.float32)
    for i in range(B):
        yi, yj = y[i], y[B - 1 - i]
        if not (0 <= yi < n and 0 <= yj < n):
            out[i] = np.nan
            continue
        out[i, yi] = np.float32(out[i, yi] + lam32)
        out[i, yj] = np.float32(out[i, yj] + lam1)
    return out


def mix_values(t, lam):
    """t: torch fp32 / bf16 [B, ...]; returns lam * t_i + lam1 * t_j rounded once to t's dtype."""
    lam32, lam1 = lams(lam)
    a = t.float().numpy()
    out = (lam32 * a).astype(np.float32) + (lam1 * a[::-1]).astype(np.float32)
    return torch.from_numpy(np.ascontiguousarray(out)).to(t.dtype)
