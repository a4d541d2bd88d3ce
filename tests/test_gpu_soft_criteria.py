"""K4 (csrc/criteria.cu) with label smoothing and probability targets, on every row branch,
against float64 torch F.cross_entropy (mean reduction): class indices with eps in {0.1, 1.0}
(ignored rows, masks), probability targets in fp32 and bf16 (unnormalised rows, masks, an empty
mask), and a ParallelCriterion of MSE and smoothed CE that now runs on the kernels.  Launch
geometry, the task scaffolding and the comparison come from test_gpu_criteria_paths.py.
Tolerances: losses 1e-5 relative; gradients that file's per-element bound, scaled by sum(q')."""
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import frl_b200  # noqa: F401
from frl_b200 import _native, criteria
from frl_b200.criteria import MaskedLoss, ParallelCriterion
from test_gpu_criteria_paths import (BF16_STORE, CE_ROWS_ONE_PASS, DEV, EPS32, _assert_close, _ce_path, _gen,
                                     _release_cached_memory, _Task)  # noqa: F401

pytestmark = pytest.mark.gpu

# (rows, C, offset) per branch: an offset of one element misaligns the view (scalar branch)
BRANCHES = {"register": (300, 1000, 0), "online": (96, 2052, 0), "scalar": (200, 1000, 1),
            "register_strided": (CE_ROWS_ONE_PASS + 76, 128, 0)}


def _logits(rows, C, seed):
    return torch.randn(rows, C, generator=_gen(seed), device=DEV) * 3.0


def _labels(rows, C, seed, ignore=-100):
    y = torch.randint(0, C, (rows,), generator=_gen(seed + 1), device=DEV)
    y[0], y[-1] = 0, C - 1
    y[3::11] = ignore
    return y


def _probs(rows, C, seed, dtype):
    q = torch.rand(rows, C, generator=_gen(seed + 2), device=DEV) ** 4
    q = q / q.sum(1, keepdim=True) * (0.5 + torch.rand(rows, 1, generator=_gen(seed + 3), device=DEV))
    return q.to(dtype)                     # rows sum to 0.5 .. 1.5: torch does not renormalise


def _ref_loss(t, x, eps):
    tgt = t.targets[0]
    tgt = tgt.double() if tgt.is_floating_point() else tgt

    def fn(a, b):
        return F.cross_entropy(a, b, ignore_index=t.inner.ignore_index, label_smoothing=eps)
    if t.mask is None:
        return fn(x, tgt)
    m = t.mask.bool()
    if not bool(m.any()):
        return fn(x - x, tgt - tgt)
    return fn(x[m], tgt[m])


def _check(t, eps, upstream):
    outs = [t.out()]
    res = criteria.fused_task_losses([t.module], outs, [t.targets], [t.weight])
    assert res is not None, "the task should be inside the kernels' domain"
    res.backward(upstream)
    got = res.detach()
    g = t.storage.grad
    grad = torch.zeros(t.shape, device=DEV) if g is None else g[t.offset:].view(t.shape).clone()
    t.storage.grad = None

    x = t.out().detach().double().requires_grad_(True)
    sub = t.weight * _ref_loss(t, x, eps)
    want = torch.stack([0.0 + sub, sub])
    (wg,) = torch.autograd.grad(want, x, grad_outputs=upstream.double(), allow_unused=True)
    wg = torch.zeros_like(x) if wg is None else wg
    _assert_close(got, want.detach(), 1e-5 * want.detach().abs(), "losses")

    tgt = t.targets[0]
    sel = torch.ones(t.shape[0], dtype=torch.bool, device=DEV) if t.mask is None else t.mask.bool()
    if tgt.is_floating_point():
        count = int(sel.sum())
        s = ((1 - eps) * tgt.double().sum(1, keepdim=True) + eps).clamp(min=1.0)
    else:
        count = int((sel & (tgt != t.inner.ignore_index)).sum())
        s = 1.0
    unit = abs(float(upstream[0]) + float(upstream[1])) * abs(t.weight) / max(count, 1)
    store = BF16_STORE if t.storage.dtype == torch.bfloat16 else 8 * EPS32
    lse = torch.logsumexp(x.detach(), dim=1, keepdim=True)
    _assert_close(grad, wg, unit * s * (store + 8 * EPS32 * (1.0 + lse.abs())), "gradient")
    return got


@pytest.mark.parametrize("branch", list(BRANCHES))
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("eps", [0.1, 1.0])
@pytest.mark.parametrize("masked", [False, True])
def test_smoothed_class_index_targets(branch, dtype, eps, masked):
    rows, C, off = BRANCHES[branch]
    ce = nn.CrossEntropyLoss(label_smoothing=eps)
    y = _labels(rows, C, 1)
    targets = (y,)
    module = ce
    if masked:
        mask = torch.rand(rows, generator=_gen(9), device=DEV) < 0.6
        targets, module = (y, mask), MaskedLoss(ce)
    t = _Task(module, _logits(rows, C, 0), dtype, targets, weight=0.7, offset=off)
    assert _ce_path(t.out(), C) == branch.split("_")[0]
    _check(t, eps, torch.tensor([1.0, 0.5], device=DEV))


@pytest.mark.parametrize("branch", list(BRANCHES))
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("tgt_dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("eps", [0.0, 0.1])
def test_probability_targets(branch, dtype, tgt_dtype, eps):
    rows, C, off = BRANCHES[branch]
    t = _Task(nn.CrossEntropyLoss(label_smoothing=eps), _logits(rows, C, 2), dtype,
              (_probs(rows, C, 3, tgt_dtype),), weight=1.3, offset=off)
    assert _ce_path(t.out(), C) == branch.split("_")[0]
    _check(t, eps, torch.tensor([1.0, -0.25], device=DEV))


@pytest.mark.parametrize("eps", [0.0, 0.1])
@pytest.mark.parametrize("empty", [False, True])
def test_masked_probability_targets(eps, empty):
    rows, C = 257, 1000
    mask = torch.zeros(rows, dtype=torch.bool, device=DEV) if empty else \
        torch.rand(rows, generator=_gen(4), device=DEV) < 0.5
    t = _Task(MaskedLoss(nn.CrossEntropyLoss(label_smoothing=eps)), _logits(rows, C, 5), torch.bfloat16,
              (_probs(rows, C, 6, torch.float32), mask))
    got = _check(t, eps, torch.tensor([1.0, 0.0], device=DEV))
    if empty:                              # eps * log C, zero gradient
        assert abs(float(got[1]) - eps * torch.log(torch.tensor(float(C))).item()) <= 1e-6


def test_empty_mask_with_smoothed_index_targets():
    rows, C = 64, 100
    mask = torch.zeros(rows, dtype=torch.bool, device=DEV)
    for ignore in (-100, 0):
        t = _Task(MaskedLoss(nn.CrossEntropyLoss(label_smoothing=0.1, ignore_index=ignore)), _logits(rows, C, 7),
                  torch.float32, (_labels(rows, C, 8, ignore), mask))
        _check(t, 0.1, torch.tensor([1.0, 0.0], device=DEV))


def test_parallel_criterion_of_mse_and_smoothed_ce_is_fused():
    B, C = 512, 1000
    crit = ParallelCriterion([nn.MSELoss(), nn.CrossEntropyLoss(label_smoothing=0.1),
                              nn.CrossEntropyLoss(label_smoothing=0.1)], [0.5, 1.0, 2.0], ["reg", "cls", "soft"])
    reg = torch.randn(B, 16, generator=_gen(10), device=DEV).requires_grad_(True)
    cls = _logits(B, C, 11).requires_grad_(True)
    soft = _logits(B, 100, 12).requires_grad_(True)
    tgts = [(torch.randn(B, 16, generator=_gen(13), device=DEV),), (_labels(B, C, 14),),
            (_probs(B, 100, 15, torch.float32),)]
    assert criteria._plan_for(list(crit.loss_modules), [reg, cls, soft], tgts) is not None
    before = _native.launch_count()
    total, split = crit([reg, cls, soft], tgts)
    assert _native.launch_count() - before == 1              # one fused forward launch
    total.backward()
    xs = [v.detach().double().requires_grad_(True) for v in (reg, cls, soft)]
    want = (0.5 * F.mse_loss(xs[0], tgts[0][0].double())
            + 1.0 * F.cross_entropy(xs[1], tgts[1][0], label_smoothing=0.1)
            + 2.0 * F.cross_entropy(xs[2], tgts[2][0].double(), label_smoothing=0.1))
    want.backward()
    assert abs(float(total) - float(want)) <= 1e-5 * abs(float(want))
    for got, ref in zip((reg, cls, soft), xs):
        torch.testing.assert_close(got.grad.double(), ref.grad, rtol=1e-4, atol=1e-7)
