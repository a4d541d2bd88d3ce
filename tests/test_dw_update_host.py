"""Where K12 (the weight-gradient GEMM with the SGD update in its epilogue) enters a 1-GPU step, on
CPU tensors: with kernels that export it, each trunk Linear site whose dW GEMM qualifies launches
it once, after that site's dX, and the end-of-step update covers exactly the rest of the arena;
with kernels that do not export it, the step is what it was (one update launch over the arena).
The kernels are ``oracle.optim_np.KernelDouble``; the K12 stand-in computes the gradient with
``torch.mm`` and updates from it with the double's SGD, so both runs train to the same weights."""
import pytest
import torch
import torch.nn as nn

import frl_b200  # noqa: F401
from frl_b200 import arena_linear, fused_optim, grad_sync
from frl_b200.arena import ParamArena
from frl_b200.types import OptAlgorithm, OptimOpts, Precision
from oracle.optim_np import KernelDouble

WIDTH, ROWS = 256, 64            # the smallest trunk K12 tiles: out % 128, in % 256, rows % 64
_DX = arena_linear._DenseGemms.dx


class _Mlp(nn.Module):
    def __init__(self):
        super().__init__()
        torch.manual_seed(0)
        self.trunk = nn.Sequential(*[m for _ in range(3) for m in (nn.Linear(WIDTH, WIDTH), nn.ReLU())])
        self.head = nn.Linear(WIDTH, 8)          # 8 output rows: not a K12 shape

    def forward(self, x):
        return self.head(self.trunk(x))


class _Logged(KernelDouble):
    def __init__(self, arena):
        super().__init__()
        self.arena = arena
        self.log = []

    def _slot(self, t):
        off = (t.data_ptr() - self.arena.grad.data_ptr()) // self.arena.grad.element_size()
        return next(s.index for s in self.arena.slots if s.offset == off)

    def sgd_momentum(self, p, g, buf, p_lp, n, **kw):
        off = (g.data_ptr() - self.arena.grad.data_ptr()) // g.element_size()
        self.log.append(("sgd", off, off + n))
        super().sgd_momentum(p, g, buf, p_lp, n, **kw)


class _WithK12(_Logged):
    def dw_gemm_sgd(self, dz, x, gw, p, buf, p_lp, **kw):
        self.log.append(("k12", self._slot(gw)))
        torch.mm(dz.t(), x, out=gw)
        self.sgd_momentum(p, gw.view(-1), buf, p_lp, gw.numel(), **kw)
        self.log.pop()                   # the stand-in's own update is not a tail launch


def _run(monkeypatch, double_cls, steps=3, fused_env=None):
    if fused_env is not None:
        monkeypatch.setenv("FRL_B200_FUSED_DW_UPDATE", fused_env)
    net = _Mlp()
    arena = ParamArena(net.parameters(), device="cpu", precision=Precision.BF16)
    opt = fused_optim.create_fused_optimizer(
        arena, OptimOpts(algo=OptAlgorithm.SGD, lr=0.05, momentum=0.9, weightDecay=1e-3))
    double = double_cls(arena)
    for mod in (arena_linear, grad_sync, fused_optim):
        monkeypatch.setattr(mod, "KERNELS", double)
    pipe = grad_sync.GradBucketPipeline(arena, opt, world_size=1, eager_update=False)
    pipe.patch_linears(net)
    slot_at = {s.offset: s.index for s in arena.slots}

    def logged_dx(gemms):                # the site is the weight dX reads (its bf16 shadow)
        double.log.append(("dx", slot_at[(gemms.weight.data_ptr() - arena.lp.data_ptr()) // 2]))
        return _DX(gemms)
    monkeypatch.setattr(arena_linear._DenseGemms, "dx", logged_dx)
    net.train()
    logs = []
    for i in range(steps):
        x = torch.randn(ROWS, WIDTH, generator=torch.Generator().manual_seed(10 + i)).to(torch.bfloat16)
        x.requires_grad_(True)           # so the first layer computes a dX too
        out = net(x)
        pipe.begin_step()
        del double.log[:]
        out.float().square().mean().backward()
        pipe.finish_step()
        logs.append(list(double.log))
    trunk = [arena.slot_of(m.weight) for m in net.trunk if isinstance(m, nn.Linear)]
    return pipe, arena, trunk, logs


def test_k12_runs_once_per_trunk_site_after_its_dx_and_the_tail_takes_the_rest(monkeypatch):
    pipe, arena, trunk, logs = _run(monkeypatch, _WithK12)
    assert pipe.fused_dw_update
    trunk_idx = [s.index for s in trunk]
    for log in logs:
        k12 = [e[1] for e in log if e[0] == "k12"]
        assert sorted(k12) == sorted(trunk_idx)                 # once per trunk site
        for idx in trunk_idx:                                   # backward order: dX, then K12
            pos = log.index(("k12", idx))
            assert log[pos - 1] == ("dx", idx)
        covered = []
        for e in log:
            if e[0] == "sgd":
                covered += list(range(e[1], e[2]))
        assert len(covered) == len(set(covered))                # nothing updated twice
        want = set(range(arena.numel)) - {i for s in trunk for i in range(s.offset, s.end)}
        assert set(covered) == want                             # exactly the complement
        assert log.index(next(e for e in log if e[0] == "sgd")) > max(log.index(("k12", i)) for i in trunk_idx)


def test_without_the_export_the_step_is_unchanged(monkeypatch):
    pipe, arena, _, logs = _run(monkeypatch, _Logged)
    assert not pipe.fused_dw_update
    for log in logs:
        assert [e for e in log if e[0] != "dx"] == [("sgd", 0, arena.numel)]


@pytest.mark.parametrize("fused_env", ["0", "1"])
def test_both_paths_train_to_the_same_weights(monkeypatch, fused_env):
    _, arena_k12, _, _ = _run(monkeypatch, _WithK12, fused_env=fused_env)
    _, arena_ref, _, _ = _run(monkeypatch, _Logged)
    assert torch.equal(arena_k12.master, arena_ref.master)
    assert torch.equal(arena_k12.lp, arena_ref.lp)


def test_the_environment_switch_turns_k12_off(monkeypatch):
    pipe, arena, _, logs = _run(monkeypatch, _WithK12, steps=1, fused_env="0")
    assert not pipe.fused_dw_update
    assert [e for e in logs[0] if e[0] != "dx"] == [("sgd", 0, arena.numel)]
