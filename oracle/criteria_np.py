"""TEST INFRASTRUCTURE — numpy (float64) restatement of the loss arithmetic under the
reference's criteria (reference criteria.py:42-61, 272-287 over ``nn.MSELoss`` /
``nn.CrossEntropyLoss`` with mean reduction).  Checker for the K4 kernels; never imported by
the product."""
import numpy as np


def mse(out, tgt, mask=None):
    """mean((out - tgt)^2) over the selected entries; empty mask -> 0 (reference: inner(0, 0))."""
    out = out.astype(np.float64)
    tgt = tgt.astype(np.float64)
    d2 = (out - tgt) ** 2
    grad = np.zeros_like(out)
    if mask is None:
        n = d2.size
        return d2.mean() if n else np.nan, 2.0 * (out - tgt) / max(n, 1)
    sel = mask.astype(bool)
    sel_full = np.broadcast_to(sel.reshape(sel.shape + (1,) * (out.ndim - sel.ndim)), out.shape)
    n = int(sel_full.sum())
    if n == 0:
        return 0.0, grad
    grad[sel_full] = 2.0 * (out - tgt)[sel_full] / n
    return d2[sel_full].mean(), grad


def cross_entropy(logits, labels, mask=None, ignore_index=-100):
    """mean over selected, non-ignored rows of (logsumexp(x) - x[y]); an all-False mask gives
    log(C) with zero gradient (reference MaskedLoss: CE(out - out, tgt - tgt)), or NaN when
    ignore_index == 0, since tgt - tgt makes every label 0 and so every row is ignored."""
    x = logits.astype(np.float64)
    B, C = x.shape
    m = x.max(axis=1, keepdims=True)
    lse = (m + np.log(np.exp(x - m).sum(axis=1, keepdims=True)))[:, 0]
    sel = np.ones(B, dtype=bool) if mask is None else mask.astype(bool)
    grad = np.zeros_like(x)
    if mask is not None and sel.sum() == 0:
        return (np.nan if ignore_index == 0 else float(np.log(C))), grad
    valid = sel & (labels != ignore_index)
    n = int(valid.sum())
    if n == 0:
        return np.nan, grad
    rows = np.flatnonzero(valid)
    loss = (lse[rows] - x[rows, labels[rows]]).sum() / n
    soft = np.exp(x[rows] - lse[rows, None])
    soft[np.arange(len(rows)), labels[rows]] -= 1.0
    grad[rows] = soft / n
    return float(loss), grad


def weighted_total(losses, weights):
    """total = ((0 + w1 L1) + w2 L2) ...; sub-losses are returned weighted."""
    subs = [w * l for w, l in zip(weights, losses)]
    total = 0.0
    for s in subs:
        total = total + s
    return total, subs
