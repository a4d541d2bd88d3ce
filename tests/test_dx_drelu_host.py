"""The K13 protocol on CPU tensors: which Linear+ReLU units get their dZ and bias gradient from the
dX GEMM of the site above them (``frl_dx_gemm_drelu``), and where those calls fall in the step.

The kernels are ``oracle.optim_np.KernelDouble`` with stand-ins for K12 and K13; K13's stand-in
computes what the unfused path computes (the bf16 dX GEMM, then ReLU's backward and the column
sum), so the arena's gradients must come out identical with and without the link."""
import torch
import torch.nn as nn

import frl_b200  # noqa: F401
from frl_b200 import arena_linear, fused_optim, grad_sync
from frl_b200.arena import ParamArena
from frl_b200.model import MultiTaskModel
from frl_b200.types import OptAlgorithm, OptimOpts, Precision
from oracle.optim_np import KernelDouble

WIDTH, ROWS = 256, 128           # the smallest trunk K13 tiles: rows % 128, columns % 256


def _model():
    torch.manual_seed(0)
    trunk = nn.Sequential(*[m for _ in range(3) for m in (nn.Linear(WIDTH, WIDTH), nn.ReLU())])
    return MultiTaskModel(trunk, [nn.Linear(WIDTH, 24), nn.Linear(WIDTH, 8)])


class _WithK12(KernelDouble):
    def __init__(self, names):
        super().__init__()
        self.names = names               # data_ptr of a gradient slice -> parameter name
        self.log = []

    def dw_gemm_sgd(self, dz, x, gw, p, buf, p_lp, **kw):
        self.log.append(("k12", self.names[gw.data_ptr()]))
        torch.mm(dz.t(), x, out=gw)
        self.sgd_momentum(p, gw.view(-1), buf, p_lp, gw.numel(), **kw)

    def colsum(self, x, out, accumulate=False):
        self.log.append(("colsum", self.names[out.data_ptr()]))
        super().colsum(x, out, accumulate)

    def drelu_colsum(self, dy, act, dz, out, accumulate=False):
        self.log.append(("drelu_colsum", self.names[out.data_ptr()]))
        super().drelu_colsum(dy, act, dz, out, accumulate)


class _WithK13(_WithK12):
    def dx_gemm_drelu(self, dz_up, w_up, act, dz_out, db_out, accumulate=False):
        self.log.append(("k13", self.names[db_out.data_ptr()]))
        dz_out.copy_(torch.ops.aten.threshold_backward(dz_up.matmul(w_up), act, 0))
        tot = dz_out.float().sum(0)
        db_out.copy_((db_out.float() + tot if accumulate else tot).to(db_out.dtype))


def _run(monkeypatch, double_cls, steps=2):
    net = _model()
    arena = ParamArena(net.parameters(), device="cpu", precision=Precision.BF16,
                       adjacent=arena_linear.head_layout_groups(net))
    opt = fused_optim.create_fused_optimizer(arena, OptimOpts(algo=OptAlgorithm.SGD, lr=0.05, momentum=0.9))
    double = double_cls({arena.grad_view(arena.slot_of(p)).data_ptr(): n for n, p in net.named_parameters()})
    for mod in (arena_linear, grad_sync, fused_optim):
        monkeypatch.setattr(mod, "KERNELS", double)
    pipe = grad_sync.GradBucketPipeline(arena, opt, world_size=1, eager_update=False)
    pipe.patch_linears(net)
    net.train()
    logs, grads = [], []
    for i in range(steps):
        x = torch.randn(ROWS, WIDTH, generator=torch.Generator().manual_seed(10 + i)).to(torch.bfloat16)
        out = net(x)
        pipe.begin_step()
        del double.log[:]
        sum(o.float().square().mean() for o in out).backward()
        grads.append(arena.grad.clone())
        pipe.finish_step()
        logs.append(list(double.log))
    return pipe, logs, grads


def test_three_k13_calls_replace_the_k6b_passes(monkeypatch):
    pipe, logs, grads = _run(monkeypatch, _WithK13)
    assert pipe.fused_dw_update
    for log in logs:
        assert [e for e in log if e[0] == "k13"] == [("k13", "model_base.4.bias"), ("k13", "model_base.2.bias"),
                                                    ("k13", "model_base.0.bias")]
        assert not [e for e in log if e[0] == "drelu_colsum"]
        # the heads' dY gets K13's aligned row stride, so their bias sums run per head
        assert [e for e in log if e[0] == "colsum"] == [("colsum", "additional_layers.0.bias"),
                                                       ("colsum", "additional_layers.1.bias")]
        # each K13 runs in its consumer's backward, before that consumer's K12
        assert log.index(("k13", "model_base.2.bias")) < log.index(("k12", "model_base.4.weight"))
        assert log.index(("k13", "model_base.0.bias")) < log.index(("k12", "model_base.2.weight"))
    monkeypatch.setenv("FRL_B200_FUSED_DRELU_DX", "0")
    _, logs0, grads0 = _run(monkeypatch, _WithK13)
    for log in logs0:
        assert not [e for e in log if e[0] == "k13"] and len([e for e in log if e[0] == "drelu_colsum"]) == 3
    for g, g0 in zip(grads, grads0):
        assert torch.equal(g, g0)


def test_without_the_export_the_step_keeps_k6b(monkeypatch):
    _, logs, _ = _run(monkeypatch, _WithK12)
    for log in logs:
        assert not [e for e in log if e[0] == "k13"]
        assert [e for e in log if e[0] == "drelu_colsum"] == [("drelu_colsum", "model_base.4.bias"),
                                                             ("drelu_colsum", "model_base.2.bias"),
                                                             ("drelu_colsum", "model_base.0.bias")]


def _links(net):
    arena = ParamArena(net.parameters(), device="cpu", precision=Precision.BF16)
    opt = fused_optim.create_fused_optimizer(arena, OptimOpts(algo=OptAlgorithm.SGD, lr=0.05))
    pipe = grad_sync.GradBucketPipeline(arena, opt, world_size=1, eager_update=False)
    pipe.patch_linears(net)
    return [(s.module, s.consumer.module if s.consumer is not None else None) for s in pipe.linear_sites]


def test_a_unit_feeding_a_non_linear_keeps_k6b(monkeypatch):
    monkeypatch.setattr(arena_linear, "KERNELS", KernelDouble())
    a, b = nn.Linear(WIDTH, WIDTH), nn.Linear(WIDTH, WIDTH)
    net = nn.Sequential(a, nn.ReLU(), b, nn.ReLU(), nn.Tanh())
    assert _links(net) == [(a, b), (b, None)]


def test_a_module_used_twice_is_not_linked(monkeypatch):
    monkeypatch.setattr(arena_linear, "KERNELS", KernelDouble())

    class _Twice(nn.Module):
        def __init__(self):
            super().__init__()
            self.b = nn.Linear(WIDTH, WIDTH)
            self.seq = nn.Sequential(nn.Linear(WIDTH, WIDTH), nn.ReLU(), self.b)

        def forward(self, x):
            return self.b(self.seq(x))

    net = _Twice()
    assert all(cons is None for _, cons in _links(net))


def test_the_switch_turns_the_links_off(monkeypatch):
    monkeypatch.setattr(arena_linear, "KERNELS", KernelDouble())
    monkeypatch.setenv("FRL_B200_FUSED_DRELU_DX", "0")
    a, b = nn.Linear(WIDTH, WIDTH), nn.Linear(WIDTH, WIDTH)
    assert _links(nn.Sequential(a, nn.ReLU(), b)) == [(a, None), (b, None)]
