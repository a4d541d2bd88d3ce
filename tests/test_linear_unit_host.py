"""The backward protocol of an arena ``nn.Linear`` site on CPU tensors: plain and ReLU sites, a
module applied once or twice per forward, dense and FP8 GEMMs, inside an open pipeline step and
outside one.  The kernels are ``oracle.optim_np.KernelDouble`` plus an FP8 stand-in, and every call
a site makes into the kernels or the pipeline is logged in order.

Inside a step each site writes its bias gradient (``colsum``, or ``drelu_colsum`` on a ReLU site:
store on the parameter's first touch in the step, accumulate after) and then marks its slots
ready, or defers them while another application of the module still has to run its backward.
Outside a step it returns ordinary gradients and touches neither the arena nor the pipeline."""
import pytest
import torch
import torch.nn as nn

import frl_b200  # noqa: F401
from frl_b200 import _native, arena_linear, fused_optim, grad_sync
from frl_b200.arena import ParamArena
from frl_b200.types import OptAlgorithm, OptimOpts, Precision
from oracle.optim_np import KernelDouble

_FMT = {_native.FP8_E4M3: "e4m3", _native.FP8_E5M2: "e5m2"}


class _Net(nn.Module):
    def __init__(self):
        super().__init__()
        torch.manual_seed(0)
        self.inp = nn.Linear(16, 32)                                # plain, applied once
        self.block = nn.Sequential(nn.Linear(32, 32), nn.ReLU())    # ReLU site, applied twice
        self.mid = nn.Linear(32, 32)                                # plain, applied twice
        self.head = nn.Linear(32, 16, bias=False)                   # plain, no bias

    def forward(self, x):
        h = self.block(self.block(self.inp(x)))
        return self.head(self.mid(torch.relu(self.mid(h))))


class _Recorder(KernelDouble):
    """The host double, logging the calls a Linear site makes; FP8 codes at scale 1."""

    def __init__(self, bias_of):
        super().__init__()
        self.log = []
        self._bias_of = bias_of          # data_ptr of a bias gradient slice -> parameter name

    def colsum(self, x, out, accumulate=False):
        self.log.append(("colsum", self._bias_of[out.data_ptr()], accumulate))
        super().colsum(x, out, accumulate)

    def drelu_colsum(self, dy, act, dz, out, accumulate=False):
        self.log.append(("drelu_colsum", self._bias_of[out.data_ptr()], accumulate))
        super().drelu_colsum(dy, act, dz, out, accumulate)

    def fp8_amax(self, src, amax_out):
        amax_out.fill_(float(src.float().abs().max()))

    def fp8_quantize(self, src, amax, fmt, dst=None, dst_t=None, inv_scale_out=None):
        self.log.append(("quantize", _FMT[fmt], dst is not None, dst_t is not None))
        dt = _native.FP8_DTYPE[fmt]
        codes = src.float().clamp(-torch.finfo(dt).max, torch.finfo(dt).max).to(dt)
        if dst is not None:
            dst.copy_(codes)
        if dst_t is not None:
            dst_t.copy_(codes.t())
        inv_scale_out.fill_(1.0)


def _patched(monkeypatch, precision):
    net = _Net()
    arena = ParamArena(net.parameters(), device="cpu", precision=precision)
    opt = fused_optim.create_fused_optimizer(arena, OptimOpts(algo=OptAlgorithm.SGD, lr=0.1))
    pipe = grad_sync.GradBucketPipeline(arena, opt, world_size=1, eager_update=False)
    names = {arena.slot_of(p).index: n for n, p in net.named_parameters()}
    double = _Recorder({arena.grad_view(arena.slot_of(p)).data_ptr(): n
                        for n, p in net.named_parameters() if n.endswith("bias")})
    for mod in (arena_linear, grad_sync, fused_optim):
        monkeypatch.setattr(mod, "KERNELS", double)
    for h in pipe._handles:              # the parameters' own hooks: the log holds the sites' calls only
        h.remove()
    for method in ("mark_ready", "defer_ready"):
        inner = getattr(pipe, method)

        def logged(slot, _method=method, _inner=inner):
            double.log.append((_method, names[slot.index]))
            _inner(slot)
        setattr(pipe, method, logged)
    assert pipe.patch_linears(net) == 4
    assert [s.relu is not None for s in pipe.linear_sites] == [False, True, False, False]
    assert [s.fp8 for s in pipe.linear_sites] == [precision is Precision.FP8] * 4
    net.train()
    return net, arena, pipe, double


def _input(shape, dtype):
    return torch.randn(shape, generator=torch.Generator().manual_seed(1)).to(dtype).requires_grad_(True)


_DENSE_STEP = [
    ("mark_ready", "head.weight"),
    ("colsum", "mid.bias", False), ("defer_ready", "mid.weight"), ("defer_ready", "mid.bias"),
    ("colsum", "mid.bias", True), ("mark_ready", "mid.weight"), ("mark_ready", "mid.bias"),
    ("drelu_colsum", "block.0.bias", False), ("defer_ready", "block.0.weight"), ("defer_ready", "block.0.bias"),
    ("drelu_colsum", "block.0.bias", True), ("mark_ready", "block.0.weight"), ("mark_ready", "block.0.bias"),
    ("colsum", "inp.bias", False), ("mark_ready", "inp.weight"), ("mark_ready", "inp.bias"),
]
# FP8: dZ is quantised to e5m2 after the ReLU mask (row-major copy for dX, transposed one for dW);
# the first layer's input needs no gradient, so its dZ gets the transposed copy only
_dz = ("quantize", "e5m2", True, True)
_FP8_STEP = [
    _dz, ("mark_ready", "head.weight"),
    _dz, ("colsum", "mid.bias", False), ("defer_ready", "mid.weight"), ("defer_ready", "mid.bias"),
    _dz, ("colsum", "mid.bias", True), ("mark_ready", "mid.weight"), ("mark_ready", "mid.bias"),
    ("drelu_colsum", "block.0.bias", False), _dz, ("defer_ready", "block.0.weight"), ("defer_ready", "block.0.bias"),
    ("drelu_colsum", "block.0.bias", True), _dz, ("mark_ready", "block.0.weight"), ("mark_ready", "block.0.bias"),
    ("quantize", "e5m2", False, True), ("colsum", "inp.bias", False), ("mark_ready", "inp.weight"),
    ("mark_ready", "inp.bias"),
]


@pytest.mark.parametrize("shape", [(32, 16), (2, 16, 16)])
@pytest.mark.parametrize("precision", [Precision.FP32, Precision.FP8])
def test_step_backward_writes_the_bias_gradients_and_marks_slots_in_order(monkeypatch, precision, shape):
    net, arena, pipe, double = _patched(monkeypatch, precision)
    fp8 = precision is Precision.FP8
    x = _input(shape, torch.bfloat16 if fp8 else torch.float32).detach()
    out = net(x)
    # forward: X and W quantised to e4m3, row-major for the GEMM and transposed for backward
    assert double.log == [("quantize", "e4m3", True, True)] * (2 * 6 if fp8 else 0)
    pipe.begin_step()
    del double.log[:]
    out.float().square().mean().backward()
    assert double.log == (_FP8_STEP if fp8 else _DENSE_STEP)
    if not fp8:                          # the arena holds what stock autograd computes
        ref = _Net()
        ref(x).square().mean().backward()
        for (n, p), r in zip(net.named_parameters(), ref.parameters()):
            torch.testing.assert_close(arena.grad_view(arena.slot_of(p)), r.grad, msg=n)
    pipe.finish_step()


@pytest.mark.parametrize("shape", [(32, 16), (2, 16, 16)])
def test_outside_a_step_the_sites_return_stock_gradients(monkeypatch, shape):
    net, _, _, double = _patched(monkeypatch, Precision.FP32)
    ref = _Net()
    x, xr = _input(shape, torch.float32), _input(shape, torch.float32)
    got = torch.autograd.grad(net(x).square().mean(), [x] + list(net.parameters()))
    want = torch.autograd.grad(ref(xr).square().mean(), [xr] + list(ref.parameters()))
    assert double.log == []
    for (n, _), g, w in zip([("x", None)] + list(net.named_parameters()), got, want):
        torch.testing.assert_close(g, w, msg=n)


def test_fp8_outside_a_step_and_without_a_graph(monkeypatch):
    net, _, _, double = _patched(monkeypatch, Precision.FP8)
    x = _input((32, 16), torch.bfloat16)
    with torch.no_grad():                # no graph: only the row-major copies the GEMM reads
        net(x)
    assert double.log == [("quantize", "e4m3", True, False)] * (2 * 6)
    del double.log[:]
    grads = torch.autograd.grad(net(x).float().square().mean(), [x] + list(net.parameters()))
    # no arena writes and no pipeline calls; dZ is quantised with both copies as dX and dW need them
    assert [c for c in double.log if c[0] != "quantize"] == []
    assert double.log[2 * 6:] == [("quantize", "e5m2", True, True)] * 6
    assert all(g is not None and g.shape == p.shape for g, p in zip(grads, [x] + list(net.parameters())))
