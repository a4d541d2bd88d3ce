"""The CPU stand-ins for K2-lw that the host-logic tests run on (``lars_step`` / ``lamb_step``, and
through them ``LayerwiseKernelDouble.lars_mt`` / ``lamb_mt``) pinned to the float64 reference and
the envelopes the GPU kernels are held to (``layerwise_oracle.check_update``; derivation in
tests/test_gpu_layerwise_paths.py): ``FusedLars`` / ``FusedLamb`` on a CPU arena, two steps at
gradient scales from 1e-30 to 1e30, a tensor with zero weights and one with a zero gradient (ratio
exactly 1), the clip coefficient on model parameters only."""
import pytest
import torch

import frl_b200  # noqa: F401
from frl_b200 import fused_optim
from frl_b200.arena import ParamArena
from frl_b200.multi_tensor import GradSegTable
from layerwise_oracle import BETAS, LAMB_EPS, LayerwiseKernelDouble, check_update

LR = {"lars": 5.0, "lamb": 1e-2}


def _weights(*shape, gen):
    return torch.randn(*shape, generator=gen).clamp_(-3, 3)


def _grad(n, gen, scale):
    mag = torch.rand(n, generator=gen, dtype=torch.float64) * 1.5 + 0.5
    sign = torch.randint(0, 2, (n,), generator=gen).double() * 2 - 1
    return (mag * sign * scale).float()


@pytest.mark.parametrize("scale", [1e-30, 1e-20, 1.0, 1e17, 1e20, 1e30])
@pytest.mark.parametrize("wd", [0.0, 1e-2], ids=["wd0", "wd"])
@pytest.mark.parametrize("mode", ["lars", "lamb"])
def test_host_double_matches_float64_within_the_kernel_envelope(monkeypatch, mode, wd, scale):
    double = LayerwiseKernelDouble()
    monkeypatch.setattr(fused_optim, "KERNELS", double)
    gen = torch.Generator().manual_seed(3)
    model = [torch.nn.Parameter(_weights(33, 17, gen=gen)), torch.nn.Parameter(_weights(5, gen=gen)),
             torch.nn.Parameter(torch.zeros(3, 4)), torch.nn.Parameter(_weights(2, 7, gen=gen))]
    crit = [torch.nn.Parameter(_weights(2, 3, gen=gen)), torch.nn.Parameter(_weights(7, gen=gen))]
    arena = ParamArena(model, crit, device="cpu")
    if mode == "lars":
        opt = fused_optim.FusedLars(arena, lr=LR[mode], momentum=0.9, weight_decay=wd)
        names, mu = ("momentum_buffer",), 0.9
    else:
        opt = fused_optim.FusedLamb(arena, lr=LR[mode], betas=BETAS, eps=LAMB_EPS, weight_decay=wd)
        names, mu = ("exp_avg", "exp_avg_sq"), 0.0
    slots = list(arena.slots)
    table = GradSegTable(slots, arena.device)
    g = arena.grad
    for s in slots:
        table.point(s, g.data_ptr() + s.offset * g.element_size(), g.dtype)
    table.upload()
    zero_grad = arena.slot_of(model[3])
    coef = torch.tensor([0.75])
    dtype = torch.float32 if mode == "lamb" and scale >= 1e30 else torch.float64   # exp_avg_sq overflows fp32
    for step in (1, 2):
        lr = LR[mode] * (1.0, 0.6)[step - 1]
        opt.hyper["lr"] = lr
        for s in slots:
            g[s.offset:s.end].copy_(_grad(s.numel, gen, scale) if s is not zero_grad else torch.zeros(s.numel))
        w0 = [arena.master[s.offset:s.end].clone() for s in slots]
        s0 = [[opt._vec[n][s.offset:s.end].clone() if n in opt._vec else torch.zeros(s.numel) for n in names]
              for s in slots]
        opt.begin_step()
        opt.apply_table(table, grad_scale=0.5, clip_coef_dev=coef)
        opt.end_step()
        ratios = opt.last_ratios(table).tolist()
        for j, s in enumerate(slots):
            check_update(mode, arena.master[s.offset:s.end], [opt._vec[n][s.offset:s.end] for n in names], ratios[j],
                         w0[j], g[s.offset:s.end].double() * 0.5 * (0.75 if s.is_model else 1.0), s0[j],
                         adapted=fused_optim.is_adapted(s), lr=lr, mu=mu, wd=wd, step=step,
                         what="step %d slot %d %s" % (step, s.index, s.shape), dtype=dtype)
        if step == 1:
            row = {s.index: j for j, s in enumerate(slots)}
            assert ratios[row[arena.slot_of(model[2]).index]] == 1.0            # ||w|| = 0
            assert ratios[row[arena.slot_of(model[1]).index]] == 1.0            # not adapted
            if mode == "lars" or wd == 0:                                      # ||g^|| = 0, ||u|| = 0
                assert ratios[row[zero_grad.index]] == 1.0
    assert [c[0] for c in double.calls] == ["%s_mt" % mode] * 2
