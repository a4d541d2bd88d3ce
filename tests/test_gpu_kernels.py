"""Parity of the sm_90a kernels (through the C ABI) against the CPU oracle.  Bit-level
agreement is not expected for floating point (FMA contraction, reduction order); tolerances are
written at each check.  The north star's bound is 1e-5 rel (fp32) / 1e-2 (bf16)."""
import numpy as np
import pytest
import torch

import frl_b200  # noqa: F401
from frl_b200 import _native
from oracle import criteria_np, optim_np

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _dev(a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    return t if dtype is None else t.to(dtype)


SIZES = [1, 3, 4, 5, 1023, 4096, 4099, 256 * 4 * 4 * 3 + 2, (1 << 20) + 7]


# ------------------------------------------------------------------------------------------------
# K2
# ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("gdt,lp", [(torch.float32, False), (torch.bfloat16, True), (torch.float32, True)])
def test_sgd_momentum_matches_oracle(n, gdt, lp):
    rs = np.random.RandomState(n % 1000)
    p0 = rs.randn(n).astype(np.float32)
    p, buf = _dev(p0), torch.zeros(n, device=DEV)
    p_lp = torch.zeros(n, dtype=torch.bfloat16, device=DEV) if lp else None
    rp, rb = p0.copy(), np.zeros(n, np.float32)
    for step in range(3):
        g = rs.randn(n).astype(np.float32)
        gd = _dev(g, gdt)
        g_seen = gd.float().cpu().numpy()          # what the kernel reads (bf16-rounded if bf16)
        _native.sgd_momentum(p, gd, buf, p_lp, n, lr=0.05, mu=0.9, dampening=0.0, wd=1e-5,
                             grad_scale=0.5, first_step=(step == 0))
        rp, rb = optim_np.sgd_step(rp, g_seen, rb, lr=0.05, mu=0.9, dampening=0.0, wd=1e-5,
                                   first_step=(step == 0), grad_scale=0.5)
    torch.cuda.synchronize()
    np.testing.assert_allclose(p.cpu().numpy(), rp, rtol=2e-6, atol=5e-7)
    np.testing.assert_allclose(buf.cpu().numpy(), rb, rtol=2e-6, atol=5e-7)
    if lp:
        assert torch.equal(p_lp, p.to(torch.bfloat16))      # shadow = RNE(bf16) of the master


def test_sgd_without_momentum_and_with_dampening():
    n = 5001
    rs = np.random.RandomState(0)
    p0, g = rs.randn(n).astype(np.float32), rs.randn(n).astype(np.float32)
    p = _dev(p0)
    _native.sgd_momentum(p, _dev(g), None, None, n, lr=0.1, mu=0.0, dampening=0.0, wd=0.0)
    np.testing.assert_allclose(p.cpu().numpy(), p0 - np.float32(0.1) * g, rtol=1e-6, atol=1e-7)
    p, buf = _dev(p0), _dev(np.ones(n, np.float32))
    _native.sgd_momentum(p, _dev(g), buf, None, n, lr=0.1, mu=0.5, dampening=0.25, wd=0.0,
                         first_step=False)
    rp, rb = optim_np.sgd_step(p0, g, np.ones(n, np.float32), lr=0.1, mu=0.5, dampening=0.25,
                               wd=0.0, first_step=False)
    np.testing.assert_allclose(p.cpu().numpy(), rp, rtol=2e-6, atol=1e-7)
    np.testing.assert_allclose(buf.cpu().numpy(), rb, rtol=2e-6, atol=1e-7)
    with pytest.raises(_native.NativeLibraryError):
        _native.sgd_momentum(p, _dev(g), None, None, n, lr=0.1, mu=0.9, dampening=0.0, wd=0.0)


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("ams", [False, True])
@pytest.mark.parametrize("gdt,lp", [(torch.float32, False), (torch.bfloat16, True)])
def test_adam_matches_oracle(n, ams, gdt, lp):
    rs = np.random.RandomState(n % 997)
    p0 = rs.randn(n).astype(np.float32)
    p, m, v = _dev(p0), torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    vmax = torch.zeros(n, device=DEV) if ams else None
    p_lp = torch.zeros(n, dtype=torch.bfloat16, device=DEV) if lp else None
    rp, rm, rv = p0.copy(), np.zeros(n, np.float32), np.zeros(n, np.float32)
    rvm = np.zeros(n, np.float32) if ams else None
    for step in range(1, 5):
        g = (rs.randn(n) * (0.1 if step == 3 else 1.0)).astype(np.float32)
        gd = _dev(g, gdt)
        _native.adam(p, gd, m, v, vmax, p_lp, n, lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8,
                     wd=1e-5, step=step)
        rp, rm, rv, rvm = optim_np.adam_step(rp, gd.float().cpu().numpy(), rm, rv, rvm, lr=1e-3,
                                             beta1=0.9, beta2=0.999, eps=1e-8, wd=1e-5, step=step)
    np.testing.assert_allclose(p.cpu().numpy(), rp, rtol=3e-6, atol=2e-7)
    np.testing.assert_allclose(m.cpu().numpy(), rm, rtol=3e-6, atol=1e-7)
    np.testing.assert_allclose(v.cpu().numpy(), rv, rtol=3e-6, atol=1e-9)
    if ams:
        np.testing.assert_allclose(vmax.cpu().numpy(), rvm, rtol=3e-6, atol=1e-9)
    if lp:
        assert torch.equal(p_lp, p.to(torch.bfloat16))


@pytest.mark.parametrize("n", [1, 4099, (1 << 18) + 3])
@pytest.mark.parametrize("mu", [0.9, 0.0])
def test_rmsprop_matches_oracle(n, mu):
    rs = np.random.RandomState(7)
    p0 = rs.randn(n).astype(np.float32)
    p, sq = _dev(p0), torch.zeros(n, device=DEV)
    buf = torch.zeros(n, device=DEV) if mu else None
    rp, rsq, rb = p0.copy(), np.zeros(n, np.float32), np.zeros(n, np.float32)
    for step in range(4):
        g = rs.randn(n).astype(np.float32)
        _native.rmsprop(p, _dev(g), sq, buf, None, n, lr=5e-4, alpha=0.99, eps=1e-8, wd=1e-5, mu=mu)
        rp, rsq, rb = optim_np.rmsprop_step(rp, g, rsq, rb, lr=5e-4, alpha=0.99, eps=1e-8, wd=1e-5, mu=mu)
    np.testing.assert_allclose(p.cpu().numpy(), rp, rtol=5e-6, atol=2e-7)
    np.testing.assert_allclose(sq.cpu().numpy(), rsq, rtol=3e-6, atol=1e-9)


def test_update_kernels_match_torch_optim_on_cpu():
    """Against torch.optim itself (the arithmetic the reference calls), 1e-5 rel."""
    n = 70001
    rs = np.random.RandomState(11)
    p0 = rs.randn(n).astype(np.float32)
    grads = [rs.randn(n).astype(np.float32) for _ in range(6)]
    for name in ("sgd", "adam", "rmsprop"):
        ref = torch.nn.Parameter(torch.from_numpy(p0.copy()))
        opt = {"sgd": lambda: torch.optim.SGD([ref], lr=0.01, momentum=0.9, weight_decay=1e-5),
               "adam": lambda: torch.optim.Adam([ref], lr=1e-3, weight_decay=1e-5, eps=1e-8),
               "rmsprop": lambda: torch.optim.RMSprop([ref], lr=1e-3, momentum=0.9, weight_decay=1e-5)}[name]()
        p = _dev(p0)
        s0, s1 = torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
        for i, g in enumerate(grads):
            ref.grad = torch.from_numpy(g.copy())
            opt.step()
            if name == "sgd":
                _native.sgd_momentum(p, _dev(g), s0, None, n, lr=0.01, mu=0.9, dampening=0.0,
                                     wd=1e-5, first_step=(i == 0))
            elif name == "adam":
                _native.adam(p, _dev(g), s0, s1, None, None, n, lr=1e-3, beta1=0.9, beta2=0.999,
                             eps=1e-8, wd=1e-5, step=i + 1)
            else:
                _native.rmsprop(p, _dev(g), s0, s1, None, n, lr=1e-3, alpha=0.99, eps=1e-8,
                                wd=1e-5, mu=0.9)
        np.testing.assert_allclose(p.cpu().numpy(), ref.detach().numpy(), rtol=1e-5, atol=1e-6)


def test_update_at_baseline_size_properties():
    """Full MLP arena (54.7M elements): size-independent properties instead of a CPU re-run."""
    n = 54_703_144 + 24
    g = torch.randn(n, device=DEV)
    p = torch.randn(n, device=DEV)
    p_before = p.clone()
    buf = torch.zeros(n, device=DEV)
    lp = torch.empty(n, dtype=torch.bfloat16, device=DEV)
    # (1) zero gradient, no decay: parameters are a fixed point, shadow = bf16(master)
    _native.sgd_momentum(p, torch.zeros_like(g), buf, lp, n, lr=0.1, mu=0.9, dampening=0.0, wd=0.0,
                         first_step=True)
    assert torch.equal(p, p_before) and torch.equal(lp, p.to(torch.bfloat16))
    # (2) linearity: one step with scale s on g == one step on (s*g)
    p1, p2 = p_before.clone(), p_before.clone()
    b1, b2 = torch.zeros_like(p), torch.zeros_like(p)
    _native.sgd_momentum(p1, g, b1, None, n, lr=0.1, mu=0.9, dampening=0.0, wd=0.0, grad_scale=0.125,
                         first_step=True)
    _native.sgd_momentum(p2, g * 0.125, b2, None, n, lr=0.1, mu=0.9, dampening=0.0, wd=0.0,
                         first_step=True)
    assert torch.equal(p1, p2) and torch.equal(b1, b2)
    # (3) closed form against torch ops on the device, and a checksum
    want = torch.addcmul(p_before, g, torch.full_like(g, -0.1 * 0.125))
    torch.testing.assert_close(p1, want, rtol=1e-6, atol=1e-6)
    assert abs(p1.double().sum().item() - want.double().sum().item()) < 1e-3 * n ** 0.5
    # (4) device-side clip coefficient multiplies in
    coef = torch.tensor([0.5], device=DEV)
    p3, b3 = p_before.clone(), torch.zeros_like(p)
    _native.sgd_momentum(p3, g, b3, None, n, lr=0.1, mu=0.9, dampening=0.0, wd=0.0, grad_scale=0.25,
                         grad_scale_dev=coef, first_step=True)
    assert torch.equal(p3, p1)


# ------------------------------------------------------------------------------------------------
# K3
# ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n", [1, 7, 4096, 1_000_003, 54_703_144])
@pytest.mark.parametrize("dt", [torch.float32, torch.bfloat16])
def test_grad_norm_and_clip_coefficient(n, dt):
    g = (torch.randn(n, device=DEV) * 0.01).to(dt)
    out = torch.zeros(3, device=DEV)
    scratch = torch.zeros((_native.reduce_scratch_bytes() + 3) // 4, dtype=torch.int32, device=DEV)
    for _ in range(2):                 # second launch checks the ticket was reset
        _native.grad_sumsq_clip(g, n, pre_scale=0.5, max_norm=0.3, out3=out, scratch=scratch)
    coef, norm = optim_np.clip_coef(g.float().cpu().numpy(), 0.3, pre_scale=0.5)
    got = out.cpu().numpy()
    assert got[1] == pytest.approx(norm, rel=2e-5)
    assert got[2] == pytest.approx(coef, rel=2e-5)
    assert got[0] == pytest.approx(norm * norm, rel=4e-5)


# ------------------------------------------------------------------------------------------------
# K4
# ------------------------------------------------------------------------------------------------

def _run_criterion(mods, outs, tgts, weights, upstream=None):
    from frl_b200 import criteria
    outs = [o.clone().requires_grad_(True) for o in outs]
    res = criteria.fused_task_losses(mods, outs, tgts, weights)
    assert res is not None, "tasks should be inside the kernels' domain"
    if upstream is None:
        res[0].backward()
    else:
        res.backward(upstream)
    return res.detach().cpu().numpy(), [o.grad for o in outs]


@pytest.mark.parametrize("dt,tol", [(torch.float32, 2e-6), (torch.bfloat16, 1e-2)])
@pytest.mark.parametrize("B,C", [(64, 10), (4096, 1000), (33, 7), (5, 4097), (1, 1)])
def test_fused_mse_and_ce_match_oracle(dt, tol, B, C):
    rs = np.random.RandomState(B + C)
    logits = (rs.randn(B, C) * 2).astype(np.float32)
    labels = rs.randint(0, C, size=B)
    reg_o, reg_t = rs.randn(B, 3).astype(np.float32), rs.randn(B, 3).astype(np.float32)
    lo, ro = _dev(logits, dt), _dev(reg_o, dt)
    mods = [torch.nn.MSELoss(), torch.nn.CrossEntropyLoss()]
    res, grads = _run_criterion(mods, [ro, lo], [(_dev(reg_t),), (_dev(labels),)], [0.5, 2.0])
    l_mse, g_mse = criteria_np.mse(ro.float().cpu().numpy(), reg_t)
    l_ce, g_ce = criteria_np.cross_entropy(lo.float().cpu().numpy(), labels)
    total, subs = criteria_np.weighted_total([l_mse, l_ce], [0.5, 2.0])
    np.testing.assert_allclose(res, [total] + subs, rtol=max(tol, 5e-6) if dt == torch.float32 else 2e-3)
    np.testing.assert_allclose(grads[0].float().cpu().numpy(), 0.5 * g_mse, rtol=tol * 4, atol=tol * 1e-2 + 1e-9)
    np.testing.assert_allclose(grads[1].float().cpu().numpy(), 2.0 * g_ce, rtol=tol * 4, atol=tol * 1e-3 + 2e-8)


def test_fused_criterion_matches_torch_losses_exactly_in_structure():
    """Against nn.MSELoss / nn.CrossEntropyLoss on the CPU (what the reference calls)."""
    torch.manual_seed(0)
    out_a, out_b = torch.randn(256, 4), torch.randn(256, 10)
    tgt_a, tgt_b = torch.randn(256, 4), torch.randint(0, 10, (256,))
    a, b = out_a.clone().requires_grad_(True), out_b.clone().requires_grad_(True)
    want = 0.5 * torch.nn.functional.mse_loss(a, tgt_a) + 2.0 * torch.nn.functional.cross_entropy(b, tgt_b)
    want.backward()
    mods = [torch.nn.MSELoss(), torch.nn.CrossEntropyLoss()]
    res, grads = _run_criterion(mods, [out_a.to(DEV), out_b.to(DEV)],
                                [(tgt_a.to(DEV),), (tgt_b.to(DEV),)], [0.5, 2.0])
    assert res[0] == pytest.approx(want.item(), rel=1e-6)
    torch.testing.assert_close(grads[0].cpu(), a.grad, rtol=1e-5, atol=1e-8)
    torch.testing.assert_close(grads[1].cpu(), b.grad, rtol=1e-5, atol=1e-8)


def test_masked_losses_ignore_index_and_empty_mask():
    from frl_b200.criteria import MaskedLoss
    rs = np.random.RandomState(2)
    B, C = 257, 12
    logits, labels = rs.randn(B, C).astype(np.float32), rs.randint(0, C, size=B)
    labels[::7] = -100
    reg_o, reg_t = rs.randn(B, 6).astype(np.float32), rs.randn(B, 6).astype(np.float32)
    row_mask = rs.rand(B) > 0.4
    elem_mask = rs.rand(B, 6) > 0.5
    mods = [MaskedLoss(torch.nn.MSELoss()), MaskedLoss(torch.nn.CrossEntropyLoss()),
            MaskedLoss(torch.nn.MSELoss())]
    tg = [(_dev(reg_t), _dev(elem_mask)), (_dev(labels), _dev(row_mask)), (_dev(reg_t), _dev(row_mask))]
    res, grads = _run_criterion(mods, [_dev(reg_o), _dev(logits), _dev(reg_o)], tg, [1.0, 1.0, 3.0])
    l0, g0 = criteria_np.mse(reg_o, reg_t, elem_mask)
    l1, g1 = criteria_np.cross_entropy(logits, labels, row_mask)
    l2, g2 = criteria_np.mse(reg_o, reg_t, row_mask)
    np.testing.assert_allclose(res[1:], [l0, l1, 3 * l2], rtol=3e-6)
    np.testing.assert_allclose(grads[0].cpu().numpy(), g0, rtol=1e-5, atol=1e-9)
    np.testing.assert_allclose(grads[1].cpu().numpy(), g1, rtol=1e-5, atol=1e-9)
    np.testing.assert_allclose(grads[2].cpu().numpy(), 3 * g2, rtol=1e-5, atol=1e-9)
    # empty masks: reference gives 0 (MSE) / log C (CE) with zero gradients, no host sync
    none = np.zeros(B, dtype=bool)
    res, grads = _run_criterion(mods[1:], [_dev(logits), _dev(reg_o)],
                                [(_dev(labels), _dev(none)), (_dev(reg_t), _dev(none))], [1.0, 1.0])
    np.testing.assert_allclose(res, [np.log(C), np.log(C), 0.0], rtol=1e-6)
    assert all(float(g.abs().max()) == 0.0 for g in grads)
    # the module itself (used stand-alone) takes the same path
    m = MaskedLoss(torch.nn.MSELoss())
    val = m(_dev(reg_o), _dev(reg_t), _dev(row_mask))
    assert val.item() == pytest.approx(l2, rel=3e-6)


def test_arbitrary_upstream_gradient_and_nan_flag_and_sink():
    from frl_b200 import criteria
    rs = np.random.RandomState(4)
    out_a, tgt_a = rs.randn(32, 4).astype(np.float32), rs.randn(32, 4).astype(np.float32)
    out_b, tgt_b = rs.randn(32, 9).astype(np.float32), rs.randint(0, 9, size=32)
    mods = [torch.nn.MSELoss(), torch.nn.CrossEntropyLoss()]
    up = torch.tensor([0.5, 2.0, -1.0], device=DEV)
    res, grads = _run_criterion(mods, [_dev(out_a), _dev(out_b)], [(_dev(tgt_a),), (_dev(tgt_b),)],
                                [1.5, 0.25], upstream=up)
    _, g_a = criteria_np.mse(out_a, tgt_a)
    _, g_b = criteria_np.cross_entropy(out_b, tgt_b)
    np.testing.assert_allclose(grads[0].cpu().numpy(), (0.5 + 2.0) * 1.5 * g_a, rtol=1e-5, atol=1e-9)
    np.testing.assert_allclose(grads[1].cpu().numpy(), (0.5 - 1.0) * 0.25 * g_b, rtol=1e-5, atol=1e-9)
    # sink + NaN flag in pinned host memory, written by the kernel itself
    sink = torch.zeros(3, pin_memory=True)
    flag = torch.zeros(1, dtype=torch.int32, pin_memory=True)
    bad = out_b.copy()
    bad[3, 2] = np.nan
    r = criteria.fused_task_losses(mods, [_dev(out_a), _dev(bad)], [(_dev(tgt_a),), (_dev(tgt_b),)],
                                   [1.0, 1.0], sink, flag)
    torch.cuda.synchronize()
    assert np.isnan(sink[0].item()) and np.isnan(sink[2].item()) and not np.isnan(sink[1].item())
    assert flag.item() == 1 and np.isnan(r[0].item())


def test_criterion_classes_on_device_match_reference_restatement():
    """ParallelCriterion / UncertaintyWeightedCriterion on CUDA vs oracle/ref_loop on CPU."""
    from frl_b200 import criteria
    from frl_b200.types import LossType
    from oracle import ref_loop
    torch.manual_seed(1)
    outs = [torch.randn(128, 4), torch.randn(128, 10)]
    tgts = [(torch.randn(128, 4),), (torch.randint(0, 10, (128,)),)]
    mods = [torch.nn.MSELoss(), torch.nn.CrossEntropyLoss()]
    d_outs = [o.to(DEV).requires_grad_(True) for o in outs]
    d_tgts = [tuple(t.to(DEV) for t in tt) for tt in tgts]
    c_outs = [o.clone().requires_grad_(True) for o in outs]

    pc = criteria.ParallelCriterion(mods, [0.5, 2.0], ["reg", "cls"])
    total, split = pc(d_outs, d_tgts)
    want_total, want_split = ref_loop.parallel_criterion(mods, [0.5, 2.0], ["reg", "cls"], c_outs, tgts)
    assert total.item() == pytest.approx(want_total.item(), rel=1e-6)
    for k in split:
        assert split[k].item() == pytest.approx(want_split[k].item(), rel=1e-6)

    uc = criteria.UncertaintyWeightedCriterion(mods, [LossType.MSE, LossType.CrossEntropy],
                                               ["reg", "cls"], [0.5, 2.0]).to(DEV)
    total, split = uc(d_outs, d_tgts)
    total.backward()
    lv = uc.log_variance.detach().cpu().clone().requires_grad_(True)
    want_total, want_split = ref_loop.uncertainty_criterion(mods, ["mse", "crossentropy"],
                                                            ["reg", "cls"], lv, c_outs, tgts)
    want_total.backward()
    assert total.item() == pytest.approx(want_total.item(), rel=1e-6)
    torch.testing.assert_close(uc.log_variance.grad.cpu(), lv.grad, rtol=1e-5, atol=1e-8)
    torch.testing.assert_close(d_outs[1].grad.cpu(), c_outs[1].grad, rtol=1e-5, atol=1e-9)


# ------------------------------------------------------------------------------------------------
# K5
# ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n", [8, 13, 3 * 224 * 224 * 2 + 5])
def test_preproc_affine_and_cast(n):
    rs = np.random.RandomState(n % 100)
    raw = rs.randint(0, 256, size=n).astype(np.uint8)
    scale = np.array([1 / 58.4, 1 / 57.1, 1 / 57.4], np.float32)
    bias = -np.array([123.7, 116.3, 103.5], np.float32) * scale
    inner = 5
    for ddt in (torch.float32, torch.bfloat16):
        dst = torch.empty(n, dtype=ddt, device=DEV)
        _native.preproc_affine(_dev(raw), dst, inner=inner, channels=3, scale=_dev(scale), bias=_dev(bias))
        c = (np.arange(n) // inner) % 3
        want = raw.astype(np.float32) * scale[c] + bias[c]
        if ddt == torch.bfloat16:
            np.testing.assert_allclose(dst.float().cpu().numpy(), optim_np.bf16_round(want), rtol=8e-3, atol=1e-6)
        else:
            np.testing.assert_allclose(dst.cpu().numpy(), want, rtol=1e-6, atol=1e-6)
    x = rs.randn(n).astype(np.float32)
    dst = torch.empty(n, dtype=torch.bfloat16, device=DEV)
    _native.cast_scale(_dev(x), dst, 1.0)
    assert torch.equal(dst, _dev(x).to(torch.bfloat16))
    back = torch.empty(n, dtype=torch.float32, device=DEV)
    _native.cast_scale(dst, back, 2.0)
    assert torch.equal(back, dst.float() * 2)


def test_launch_counter_counts_our_kernels():
    _native.launch_count_reset()
    n = 1024
    p, g, b = torch.zeros(n, device=DEV), torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    for _ in range(3):
        _native.sgd_momentum(p, g, b, None, n, lr=0.1, mu=0.9, dampening=0.0, wd=0.0)
    assert _native.launch_count() == 3
    assert _native.lib().frl_device_arch() == 90
    assert _native.lib().frl_device_sm_count() == 132


# ------------------------------------------------------------------------------------------------
# nn.Linear gradients born in the arena (K6 and K6b themselves: test_gpu_colsum_paths.py)
# ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_linear_gradients_are_written_into_the_arena(precision, monkeypatch):
    import torch.nn as nn
    monkeypatch.setenv("FRL_B200_FUSE_RELU", "0")           # the plain per-layer path; units: see below
    from frl_b200 import fused_optim, grad_sync
    from frl_b200.arena import ParamArena
    from frl_b200.types import OptAlgorithm, OptimOpts, Precision
    torch.manual_seed(0)
    torch.backends.cuda.matmul.allow_tf32 = False

    def build():
        torch.manual_seed(0)
        return nn.Sequential(nn.Linear(40, 64), nn.ReLU(), nn.Linear(64, 64), nn.ReLU(),
                             nn.Linear(64, 8)).to(DEV)
    plain, fancy = build(), build()
    prec = Precision(precision)
    x0 = torch.randn(32, 40, device=DEV)
    results = []
    for net, direct in ((plain, False), (fancy, True)):
        arena = ParamArena(net.parameters(), device=DEV, precision=prec)
        opt = fused_optim.create_fused_optimizer(arena, OptimOpts(algo=OptAlgorithm.SGD, lr=0.05))
        pipe = grad_sync.GradBucketPipeline(arena, opt, bucket_cap_mb=0.004, eager_update=direct)
        if direct:
            assert pipe.patch_linears(net) == 3 and len(pipe.buckets) > 1
        else:
            pipe.mt_enabled = False       # reference point: autograd's gradients copied into the arena
        x = x0.to(torch.bfloat16) if prec == Precision.BF16 else x0
        for _ in range(3):
            pipe.begin_step()
            net(x).float().square().mean().backward()
            pipe.finish_step()
        torch.cuda.synchronize()
        results.append((arena.grad.float().clone(), arena.master.clone()))
        pipe.remove_hooks()
    tol = dict(rtol=2e-2, atol=2e-3) if prec == Precision.BF16 else dict(rtol=1e-5, atol=1e-7)
    torch.testing.assert_close(results[1][0], results[0][0], **tol)      # same gradients
    torch.testing.assert_close(results[1][1], results[0][1], **tol)      # same weights after 3 steps
    assert "forward" not in fancy[0].__dict__                            # unpatched again


# ------------------------------------------------------------------------------------------------
# K8 + the batched device-side input path
# ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("rows,cols,dt", [(1000, 64, torch.float32), (257, 4096, torch.float32),
                                          (64, 8, torch.int64), (33, 1024, torch.bfloat16),
                                          (500, 1, torch.int64), (77, 3, torch.float32), (50, 5, torch.uint8)])
def test_gather_rows_from_pinned_host_memory(rows, cols, dt):
    src = (torch.randn(rows, cols) * 100).to(dt).pin_memory()
    idx = torch.randint(0, rows, (123,), dtype=torch.int64)
    dst = torch.zeros(123, cols, dtype=dt, device=DEV)
    _native.gather_rows(src, idx.to(DEV), dst)
    torch.cuda.synchronize()
    assert torch.equal(dst.cpu(), src[idx])
    # out-of-range indices never read outside the dataset (clamped to row 0)
    bad = torch.tensor([rows + 5, -1], dtype=torch.int64, device=DEV)
    out = torch.zeros(2, cols, dtype=dt, device=DEV)
    _native.gather_rows(src, bad, out)
    assert torch.equal(out.cpu(), src[[0, 0]])


@pytest.mark.parametrize("sizes,tail,dt", [([64, 64, 17], (4096,), torch.bfloat16), ([5], (3,), torch.float32),
                                           ([8, 1, 30], (3, 7, 5), torch.uint8), ([4] * 150, (16,), torch.int64),
                                           ([33, 2], (), torch.float32)])
def test_window_gather_matches_index_select_of_the_concatenation(sizes, tail, dt):
    """K8w: picked rows of a list of separate device tensors == index_select on their cat (bit-exact);
    ragged batches, > 64 batches (several tables), unaligned rows, 1-D batches, rows outside the
    window left untouched."""
    torch.manual_seed(sum(sizes))
    batches = [(torch.randn(n, *tail, device=DEV) * 50).to(dt) for n in sizes]
    if dt == torch.uint8 and len(sizes) == 3:
        batches[1] = torch.cat([batches[1].new_zeros(1, *tail), batches[1]])[1:]     # odd base address
    total = sum(sizes)
    idx = torch.randint(0, total, (19,), dtype=torch.int64, device=DEV)
    idx[0], idx[1] = 0, total - 1
    got = _native.gather_window_rows(batches, idx)
    assert got.shape == (19,) + tuple(tail) and torch.equal(got, torch.cat(batches).index_select(0, idx))
    dst = torch.full((3,) + tuple(tail), 7, dtype=dt, device=DEV)
    out = _native.gather_window_rows(batches, torch.tensor([total, -1, 1 % total], device=DEV), dst)
    assert torch.equal(out[:2], torch.full_like(out[:2], 7)) and torch.equal(out[2], torch.cat(batches)[1 % total])


@pytest.mark.parametrize("rows,cols,dt,blocks", [(1000, 4096, torch.float32, 0), (257, 4096, torch.float32, 3),
                                                 (64, 8, torch.int64, 1), (33, 1024, torch.bfloat16, 2),
                                                 (300, 4096 + 8, torch.float32, 4), (40, 3 * 224 * 224, torch.uint8, 5),
                                                 (9, 20000, torch.float32, 7)])
def test_tma_gather_rows_matches_index_select(rows, cols, dt, blocks):
    """cp.async.bulk variant: rows longer than one 16 KB stage are chunked, tails are partial
    chunks, more stages than work items, every grid size."""
    src = (torch.randn(rows, cols) * 100).to(dt).pin_memory()
    n = 211
    idx = torch.randint(0, rows, (n,), dtype=torch.int64)
    dst = torch.zeros(n, cols, dtype=dt, device=DEV)
    _native.gather_rows_tma(src, idx.to(DEV), dst, max_blocks=blocks)
    torch.cuda.synchronize()
    assert torch.equal(dst.cpu(), src[idx])
    bad = torch.tensor([rows + 5, -1], dtype=torch.int64, device=DEV)
    out = torch.zeros(2, cols, dtype=dt, device=DEV)
    _native.gather_rows_tma(src, bad, out)
    assert torch.equal(out.cpu(), src[[0, 0]])


def test_tma_gather_rejects_rows_that_are_not_multiples_of_16_bytes():
    src = torch.zeros(10, 3).pin_memory()
    with pytest.raises(_native.NativeLibraryError):
        _native.gather_rows_tma(src, torch.zeros(2, dtype=torch.int64, device=DEV),
                                torch.zeros(2, 3, device=DEV))


# ------------------------------------------------------------------------------------------------
# Linear/ReLU units (FRL_B200_FUSE_RELU)
# ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_fused_linear_relu_units_match_the_unfused_modules(precision, monkeypatch):
    import torch.nn as nn
    from frl_b200 import fused_optim, grad_sync
    from frl_b200.arena import ParamArena
    from frl_b200.types import OptAlgorithm, OptimOpts, Precision
    torch.backends.cuda.matmul.allow_tf32 = False

    def build():
        torch.manual_seed(0)
        shared = nn.ReLU()
        return nn.Sequential(nn.Linear(40, 64), nn.ReLU(), nn.Linear(64, 64), nn.ReLU(inplace=True),
                             nn.Linear(64, 32), shared, nn.Linear(32, 32), shared, nn.Linear(32, 8)).to(DEV)
    prec = Precision(precision)
    x0 = torch.randn(3, 32, 40, device=DEV)               # 3-D input: units must keep leading dims
    results = []
    for fuse in ("0", "1"):
        monkeypatch.setenv("FRL_B200_FUSE_RELU", fuse)
        net = build()
        arena = ParamArena(net.parameters(), device=DEV, precision=prec)
        opt = fused_optim.create_fused_optimizer(arena, OptimOpts(algo=OptAlgorithm.SGD, lr=0.05))
        pipe = grad_sync.GradBucketPipeline(arena, opt, bucket_cap_mb=0.004, eager_update=True)
        assert pipe.patch_linears(net) == 5
        fused = [s.relu is not None for s in pipe.linear_sites]
        assert fused == ([True, True, False, False, False] if fuse == "1" else [False] * 5)  # shared ReLU: left alone
        x = x0.to(torch.bfloat16) if prec == Precision.BF16 else x0
        outs = []
        for _ in range(3):
            pipe.begin_step()
            y = net(x)
            outs.append(y.detach().float().clone())
            y.float().square().mean().backward()
            pipe.finish_step()
        torch.cuda.synchronize()
        results.append((arena.grad.float().clone(), arena.master.clone(), outs))
        pipe.remove_hooks()
        assert all("forward" not in m.__dict__ for m in net)          # everything unpatched again
    tol = dict(rtol=2e-2, atol=2e-3) if prec == Precision.BF16 else dict(rtol=1e-4, atol=1e-6)
    for a, b in zip(results[1][2], results[0][2]):
        torch.testing.assert_close(a, b, **tol)
    torch.testing.assert_close(results[1][0], results[0][0], **tol)
    torch.testing.assert_close(results[1][1], results[0][1], **tol)


# ------------------------------------------------------------------------------------------------
# K1 / K2-mt — multi-tensor forms: gradients read where autograd left them (segment tables)
# ------------------------------------------------------------------------------------------------

class _Slot:
    def __init__(self, index, offset, numel):
        self.index, self.offset, self.numel = index, offset, numel


def _mt_case(seed=0, sizes=(10, 64, 3, 9408, 4097, 8, 1, 36864, 4096 * 5 + 2, 1000)):
    """Slots at 8-aligned arena offsets (arena.py layout) + one separately allocated gradient
    tensor per slot, fp32 and bf16 mixed as in a BF16-mode run with criterion parameters."""
    from frl_b200.multi_tensor import GradSegTable
    rs = np.random.RandomState(seed)
    slots, off = [], 0
    for i, n in enumerate(sizes):
        slots.append(_Slot(i, off, n))
        off = (off + n + 7) // 8 * 8
    grads = []
    for i, s in enumerate(slots):
        g = _dev(rs.randn(s.numel).astype(np.float32), torch.bfloat16 if i % 3 == 1 else torch.float32)
        grads.append(g)
    table = GradSegTable(slots, torch.device(DEV))
    for s, g in zip(slots, grads):
        table.point(s, g.data_ptr(), g.dtype)
    table.upload()
    return slots, grads, table, off


@pytest.mark.parametrize("dst", [torch.float32, torch.bfloat16])
def test_flatten_grads_gathers_every_segment_in_one_launch(dst):
    slots, grads, table, n = _mt_case()
    arena = torch.full((n,), 7.0, dtype=dst, device=DEV)
    before = _native.launch_count()
    _native.flatten_grads(table, arena, scale=0.5)
    assert _native.launch_count() - before == 1
    torch.cuda.synchronize()
    for s, g in zip(slots, grads):
        want = (g.float() * 0.5).to(dst)
        assert torch.equal(arena[s.offset:s.offset + s.numel], want), s.index
        # the padding up to the next multiple of 4 is zero-filled, the rest of the gap untouched
        pad4 = (s.numel + 3) // 4 * 4
        assert torch.all(arena[s.offset + s.numel:s.offset + pad4] == 0)
    # pointing the same table at other tensors and uploading again is enough for the next step
    grads2 = [torch.ones_like(g) for g in grads]
    for s, g in zip(slots, grads2):
        table.point(s, g.data_ptr(), g.dtype)
    table.upload()
    _native.flatten_grads(table, arena, scale=1.0)
    torch.cuda.synchronize()
    assert all(torch.all(arena[s.offset:s.offset + s.numel] == 1) for s in slots)


@pytest.mark.parametrize("algo", ["sgd", "adam", "adam_amsgrad", "rmsprop"])
@pytest.mark.parametrize("lp", [False, True])
def test_multi_tensor_update_equals_flatten_then_flat_update(algo, lp):
    """K2-mt reads the gradients in place; the result must be BIT-identical to gathering them into
    the arena (fp32, so no rounding on the way) and running the flat K2 over it."""
    slots, grads, table, n = _mt_case(seed=3)
    rs = np.random.RandomState(9)
    p0 = rs.randn(n).astype(np.float32)
    used = np.zeros(n, bool)
    for s in slots:
        used[s.offset:s.offset + s.numel] = True
    p0[~used] = 0.0                                   # arena padding is zero
    flat_g = torch.zeros(n, device=DEV)
    _native.flatten_grads(table, flat_g, scale=1.0)

    def run(mt):
        p = _dev(p0)
        s0, s1, s2 = (torch.zeros(n, device=DEV) for _ in range(3))
        p_lp = torch.zeros(n, dtype=torch.bfloat16, device=DEV) if lp else None
        for step in range(3):
            first = step == 0
            if algo == "sgd":
                if mt:
                    _native.sgd_momentum_mt(p, s0, p_lp, table, lr=0.05, mu=0.9, dampening=0.0, wd=1e-5,
                                            grad_scale=0.5, first_step=first)
                else:
                    _native.sgd_momentum(p, flat_g, s0, p_lp, n, lr=0.05, mu=0.9, dampening=0.0, wd=1e-5,
                                         grad_scale=0.5, first_step=first)
            elif algo.startswith("adam"):
                vmax = s2 if algo == "adam_amsgrad" else None
                kw = dict(lr=1e-2, beta1=0.9, beta2=0.999, eps=1e-8, wd=1e-5, step=step + 1, grad_scale=0.5)
                if mt:
                    _native.adam_mt(p, s0, s1, vmax, p_lp, table, **kw)
                else:
                    _native.adam(p, flat_g, s0, s1, vmax, p_lp, n, **kw)
            else:
                kw = dict(lr=1e-2, alpha=0.99, eps=1e-8, wd=1e-5, mu=0.9, grad_scale=0.5)
                if mt:
                    _native.rmsprop_mt(p, s0, s1, p_lp, table, **kw)
                else:
                    _native.rmsprop(p, flat_g, s0, s1, p_lp, n, **kw)
        torch.cuda.synchronize()
        return p, s0, s1, s2, p_lp

    a, b = run(True), run(False)
    for s in slots:
        sl = slice(s.offset, s.offset + s.numel)
        for x, y in zip(a, b):
            if x is not None:
                assert torch.equal(x[sl], y[sl]), (algo, s.index)
