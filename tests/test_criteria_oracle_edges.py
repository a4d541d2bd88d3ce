"""The numpy oracle's criterion and clip-coefficient arithmetic against torch itself (float64, on
the CPU) at the edges where the two can part: masks that select nothing, rows that are all
ignored, and non-finite or zero gradients under global-norm clipping.  The GPU kernels are checked
against the oracle elsewhere, so an oracle that agrees with itself but not with torch would hide
the same mistake in a kernel; these cases pin it to torch."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import criteria_np, optim_np


def _same(got, want):
    """Equal up to 1e-12 relative, with NaN only where the other side has NaN."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert np.array_equal(np.isnan(got), np.isnan(want)), (got, want)
    np.testing.assert_allclose(got, want, rtol=1e-12, atol=0, equal_nan=True)


def _torch_masked_ce(x, y, mask, ignore_index):
    """The reference MaskedLoss over CrossEntropyLoss: out[mask], or out - out when the mask is
    empty.  Returns (loss, d loss / d x)."""
    xt = torch.tensor(x, dtype=torch.float64, requires_grad=True)
    yt = torch.tensor(y)
    m = None if mask is None else torch.tensor(mask)
    if mask is not None and m.sum() == 0:
        loss = F.cross_entropy(xt - xt, yt - yt, ignore_index=ignore_index)
    elif mask is not None:
        loss = F.cross_entropy(xt[m], yt[m], ignore_index=ignore_index)
    else:
        loss = F.cross_entropy(xt, yt, ignore_index=ignore_index)
    loss.backward()
    return loss.item(), xt.grad.numpy()


def _case(B=9, C=6, seed=0):
    rs = np.random.RandomState(seed)
    return rs.randn(B, C) * 3, rs.randint(1, C, size=B)


@pytest.mark.parametrize("ignore_index", [-100, 0, 3])
def test_empty_mask_cross_entropy_matches_torch(ignore_index):
    # tgt - tgt makes every label 0: with ignore_index == 0 torch ignores every row (NaN),
    # otherwise each row of out - out contributes log C
    x, y = _case()
    empty = np.zeros(len(y), dtype=bool)
    want, want_grad = _torch_masked_ce(x, y, empty, ignore_index)
    got, got_grad = criteria_np.cross_entropy(x, y, empty, ignore_index=ignore_index)
    _same(got, want)
    assert np.isnan(got) == (ignore_index == 0)
    _same(got_grad, want_grad)
    assert not np.any(got_grad)


def test_empty_mask_mse_matches_torch():
    rs = np.random.RandomState(1)
    out, tgt = rs.randn(7, 5), rs.randn(7, 5)
    ot = torch.tensor(out, requires_grad=True)
    want = F.mse_loss(ot - ot, torch.tensor(tgt) - torch.tensor(tgt))
    want.backward()
    for mask in (np.zeros(7, dtype=bool), np.zeros((7, 5), dtype=bool)):
        got, got_grad = criteria_np.mse(out, tgt, mask)
        _same(got, want.item())
        _same(got_grad, ot.grad.numpy())


@pytest.mark.parametrize("ignore_index", [-100, 0, 3])
@pytest.mark.parametrize("masked", [False, True])
def test_all_rows_ignored_matches_torch(ignore_index, masked):
    # every selected row carries ignore_index: torch's mean over no rows is NaN, gradient zero
    x, y = _case(seed=2)
    y = np.full_like(y, ignore_index)
    mask = None
    if masked:
        mask = np.zeros(len(y), dtype=bool)
        mask[[1, 4, 5]] = True
        y[~mask] = 1            # the rows the mask drops hold a real label
    want, want_grad = _torch_masked_ce(x, y, mask, ignore_index)
    got, got_grad = criteria_np.cross_entropy(x, y, mask, ignore_index=ignore_index)
    assert np.isnan(want)
    _same(got, want)
    _same(got_grad, want_grad)


@pytest.mark.parametrize("ignore_index", [-100, 0, 3])
def test_partly_ignored_masked_rows_match_torch(ignore_index):
    # the ordinary masked case next to the edges above: selected rows, some of them ignored
    x, y = _case(B=23, C=7, seed=3)
    y[::4] = ignore_index
    mask = np.random.RandomState(4).rand(len(y)) > 0.3
    want, want_grad = _torch_masked_ce(x, y, mask, ignore_index)
    got, got_grad = criteria_np.cross_entropy(x, y, mask, ignore_index=ignore_index)
    np.testing.assert_allclose(got, want, rtol=1e-12)
    np.testing.assert_allclose(got_grad, want_grad, rtol=1e-10, atol=1e-15)


def _torch_clip(g, max_norm, pre_scale, pieces=(3, 1, 7)):
    """clip_grad_norm_ over float64 tensors holding pre_scale * g, split into several tensors.
    Returns (norm, clipped gradient)."""
    g = torch.tensor(g, dtype=torch.float64) * pre_scale
    bounds = np.cumsum((0,) + pieces)
    assert bounds[-1] == g.numel()
    params = []
    for lo, hi in zip(bounds[:-1], bounds[1:]):
        p = torch.zeros(int(hi - lo), dtype=torch.float64)
        p.grad = g[lo:hi].clone()
        params.append(p)
    norm = torch.nn.utils.clip_grad_norm_(params, max_norm)
    return norm.item(), torch.cat([p.grad for p in params]).numpy()


@pytest.mark.parametrize("kind", ["nan", "inf", "-inf", "zero", "below_one", "above_one"])
@pytest.mark.parametrize("pre_scale", [1.0, 0.5])
def test_clip_coefficient_matches_clip_grad_norm(kind, pre_scale):
    g = np.random.RandomState(5).randn(11)
    max_norm = 0.7
    if kind == "nan":
        g[6] = np.nan
    elif kind in ("inf", "-inf"):
        g[2] = np.inf if kind == "inf" else -np.inf
    elif kind == "zero":
        g[:] = 0.0
    else:
        # max_norm just around the norm: the coefficient lands just below or just above 1
        norm = float(np.sqrt(np.sum((g * pre_scale) ** 2)))
        max_norm = norm * (0.999 if kind == "below_one" else 1.001)
    want_norm, want_clipped = _torch_clip(g, max_norm, pre_scale)
    coef, norm = optim_np.clip_coef(g, max_norm, pre_scale=pre_scale)
    _same(norm, want_norm)
    # the oracle's coefficient applied to the gradient is what clip_grad_norm_ leaves behind
    with np.errstate(invalid="ignore"):         # inf * 0 = NaN, as in torch
        _same(g * pre_scale * coef, want_clipped)
    if kind == "nan":
        assert np.isnan(coef) and np.all(np.isnan(want_clipped))
    elif kind in ("inf", "-inf"):
        assert coef == 0.0 and np.array_equal(np.isnan(want_clipped), np.arange(11) == 2)
    elif kind == "zero":
        assert coef == 1.0
    elif kind == "below_one":
        assert 0.99 < coef < 1.0
    else:
        assert coef == 1.0
