"""The FP8 training precision on the H100: K9 bit for bit against torch's float8 casts, one FP8
Linear site against fp32 arithmetic on the very operands it quantised, the headline MLP against
stock torch running the same FP8 recipe and against the fp32 CPU oracle, CUDA-graph replay,
checkpoints and the per-call bf16 fallback."""
import math
import os
import shutil
import tempfile
import types

import numpy as np
import pytest
import torch
import torch.nn as nn

import frl_b200  # noqa: F401
from frl_b200 import _native, arena_linear, synthetic
from frl_b200.solver import Solver, SolverWorkerArgs
from frl_b200.types import Device, Precision
from test_gpu_mlp_parity import BATCH, DEPTH, LR, N_CLASSES, REG_DIM, WIDTH, _batches, _oracle

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
FMTS = {"e4m3": (_native.FP8_E4M3, torch.float8_e4m3fn, 448.0), "e5m2": (_native.FP8_E5M2, torch.float8_e5m2, 57344.0)}


def _pow2_scale(amax: float, fmt_max: float) -> float:
    """2^floor(log2(fmt_max / amax)) in exact arithmetic, exponent clamped to [-126, 126]."""
    if amax == 0.0:
        return 1.0
    if not math.isfinite(amax):
        return math.nan
    ma, ea = math.frexp(amax)
    mm, em = math.frexp(fmt_max)
    return 2.0 ** max(-126, min(126, em - ea - (1 if ma > mm else 0)))


def _k9(x, fmt):
    code, _, _ = FMTS[fmt]
    sc = torch.full((2,), -1.0, device=DEV)
    q = torch.empty(x.shape, dtype=FMTS[fmt][1], device=DEV)
    qt = torch.empty(x.shape[::-1], dtype=FMTS[fmt][1], device=DEV)
    _native.fp8_amax(x, sc[:1])
    _native.fp8_quantize(x, sc[:1], code, q, qt, sc[1:])
    torch.cuda.synchronize()
    return float(sc[0]), float(sc[1]), q, qt


def _assert_codes_equal(got, want):
    gn, wn = got.float().isnan(), want.float().isnan()
    assert torch.equal(gn, wn)
    assert torch.equal(got.view(torch.uint8)[~wn], want.view(torch.uint8)[~wn])


def _check_k9(x, fmt):
    _, dt, fmax = FMTS[fmt]
    amax, inv, q, qt = _k9(x, fmt)
    want_amax = float(x.float().abs().max())
    assert (amax == want_amax) or (math.isnan(amax) and math.isnan(want_amax))
    scale = _pow2_scale(want_amax, fmax)
    if math.isnan(scale):
        assert math.isnan(inv)
    else:
        assert inv == 1.0 / scale                       # exactly the power of two
    want = (x.float() * scale).clamp(-fmax, fmax).to(dt)
    _assert_codes_equal(q, want)
    _assert_codes_equal(qt, want.t().contiguous())
    return amax, inv


@pytest.mark.parametrize("shape", [(4096, 4096), (4096, 1000), (17, 48), (1, 16), (130, 260)])
@pytest.mark.parametrize("src", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("fmt", ["e4m3", "e5m2"])
def test_k9_matches_torch_bit_for_bit(fmt, src, shape):
    g = torch.Generator().manual_seed(shape[0] * 7 + shape[1])
    x = (torch.randn(shape, generator=g) * 3.7).to(src).to(DEV)
    _check_k9(x, fmt)
    # only the row-major or only the transposed copy
    code, dt, _ = FMTS[fmt]
    sc = torch.empty(2, device=DEV)
    q = torch.empty(shape, dtype=dt, device=DEV)
    qt = torch.empty(shape[::-1], dtype=dt, device=DEV)
    _native.fp8_amax(x, sc[:1])
    _native.fp8_quantize(x, sc[:1], code, q, None, sc[1:])
    _native.fp8_quantize(x, sc[:1], code, None, qt, sc[1:])
    _, _, q2, qt2 = _k9(x, fmt)
    assert torch.equal(q.view(torch.uint8), q2.view(torch.uint8))
    assert torch.equal(qt.view(torch.uint8), qt2.view(torch.uint8))


@pytest.mark.parametrize("src", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("fmt", ["e4m3", "e5m2"])
def test_k9_special_inputs(fmt, src):
    _, _, fmax = FMTS[fmt]
    # all zeros: scale 1, zero codes
    amax, inv = _check_k9(torch.zeros(48, 64, dtype=src, device=DEV), fmt)
    assert amax == 0.0 and inv == 1.0
    # the saturation edge: amax * scale lands exactly on FP8_MAX, neighbours round to it or just below
    edge = fmax / 32.0
    x = torch.linspace(-edge, edge, 64 * 80, dtype=torch.float64).view(64, 80)
    x[0, :4] = torch.tensor([edge, -edge, edge * (1 - 2 ** -8), -edge * (1 - 2 ** -9)], dtype=torch.float64)
    x = x.to(src).to(DEV)
    amax, inv = _check_k9(x, fmt)
    assert amax == edge and inv == 1.0 / 32.0
    # just above a power-of-two boundary: the scale halves
    x[0, 0] = edge * (1 + 2 ** -7)
    _check_k9(x, fmt)
    # tiny and huge magnitudes
    _check_k9((torch.randn(32, 32) * 1e-30).to(src).to(DEV), fmt)
    _check_k9((torch.randn(32, 32) * 1e30).to(src).to(DEV), fmt)
    # one NaN: NaN amax, NaN codes everywhere, NaN inverse scale
    x = torch.randn(33, 48).to(src).to(DEV)
    x[20, 7] = float("nan")
    amax, inv, q, qt = _k9(x, fmt)
    assert math.isnan(amax) and math.isnan(inv)
    assert bool(q.float().isnan().all()) and bool(qt.float().isnan().all())
    # an infinity: no scale either
    x[20, 7] = float("inf")
    amax, inv, q, _ = _k9(x, fmt)
    assert amax == math.inf and math.isnan(inv) and bool(q.float().isnan().all())


def test_k9_amax_of_long_vectors_with_a_tail():
    for n in (1, 7, 4099, (1 << 24) + 3):
        for dt in (torch.bfloat16, torch.float32):
            x = torch.randn(n, device=DEV).to(dt)
            x[n // 2] = -9.5
            out = torch.full((1,), 123.0, device=DEV)          # zeroed by the call
            _native.fp8_amax(x, out)
            assert float(out) == float(x.float().abs().max()), (n, dt)


# ---- one site against its own operands ---------------------------------------------------------

def _dequant(x2, fmt):
    _, inv, q, _ = _k9(x2.contiguous(), fmt)
    return q.float() * inv


@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("xshape", [(256, 512), (4, 64, 512)])
def test_fp8_linear_fn_matches_fp32_on_its_dequantised_operands(relu, xshape):
    torch.manual_seed(3)
    K, N = xshape[-1], 384
    x = torch.randn(xshape, device=DEV).bfloat16().requires_grad_(True)
    w = (torch.randn(N, K, device=DEV) / K ** 0.5).bfloat16().requires_grad_(True)
    b = torch.randn(N, device=DEV).bfloat16().requires_grad_(True)
    # outside a pipeline step: ordinary grads
    site = types.SimpleNamespace(pipeline=None, relu=nn.ReLU() if relu else None)
    y = arena_linear._ArenaLinearFn.apply(x, w, b, site, True, True)
    assert y.dtype == torch.bfloat16 and y.shape == xshape[:-1] + (N,)
    dy = torch.randn(y.shape, device=DEV).bfloat16()
    y.backward(dy)

    x2 = x.detach().reshape(-1, K)
    xd, wd = _dequant(x2, "e4m3"), _dequant(w.detach(), "e4m3")
    z = xd @ wd.t() + b.detach().float()
    want_y = z.relu() if relu else z
    dz = dy.reshape(-1, N)
    if relu:
        dz = dz * (y.detach().reshape(-1, N) > 0).to(dz.dtype)
    dzd = _dequant(dz, "e5m2")
    want = {"y": want_y, "dx": dzd @ wd, "dw": dzd.t() @ xd, "db": dz.float().sum(0)}
    got = {"y": y.detach().reshape(-1, N).float(), "dx": x.grad.reshape(-1, K).float(), "dw": w.grad.float(),
           "db": b.grad.float()}
    for k in want:
        err = float((got[k] - want[k]).norm() / want[k].norm())
        print("%s relu=%s %s: relative L2 %.2e" % (xshape, relu, k, err))
        assert err <= 1e-2, (k, err)
        torch.testing.assert_close(got[k], want[k], rtol=1e-2, atol=1e-2 * float(want[k].abs().max()))


# ---- the headline MLP --------------------------------------------------------------------------

def _headline_problem(save_dir):
    ns = synthetic.api_namespace("frl_b200")
    torch.manual_seed(0)
    return ns, synthetic.make_mlp_problem(ns, save_dir, n_train=8, width=WIDTH, n_classes=N_CLASSES,
                                          reg_dim=REG_DIM, depth=DEPTH)


_RUNS = {}


def _fp8_run(algo, graph, monkeypatch):
    """Six steps of the headline MLP in FP8 through Solver.build_worker (cached per algo/graph)."""
    if (algo, graph) in _RUNS:
        return _RUNS[(algo, graph)]
    monkeypatch.setenv("FRL_B200_CUDA_GRAPH", graph)
    save_dir = tempfile.mkdtemp(prefix="frl_b200_fp8_")
    ns, problem = _headline_problem(save_dir)
    t = ns.types
    run_opts = t.RunOpts(optim=t.OptimOpts(algo=t.OptAlgorithm(algo), lr=LR[algo]), batchSize=BATCH,
                         nEpochs=1, numThreads=0, singleThreaded=True, numVisualizedSamples=0)
    args = SolverWorkerArgs(run_opts=run_opts, problem=problem, save_dir=save_dir, run_device=Device.GPU,
                            node_idx=0, node_count=1, rank=0, local_rank=0, world_size=1, group_name=None,
                            init_method="", precision=Precision.FP8)
    worker, _, _ = Solver.build_worker(args)
    worker.model.train()
    worker.criterion.train()
    sites = worker.pipeline.linear_sites
    n_fp8 = sum(s.fp8 for s in sites)
    rows, first_grads = [], None
    for i, (x, y, r) in enumerate(_batches()):
        _, total, sub, _ = worker._pass_one_minibatch(i, t.Split.TRAIN, [x.cuda()], [(y.cuda(),), (r.cuda(),)])
        rows.append([float(total.detach())] + [float(sub[n].detach()) for n in worker.criterion.loss_names])
        del total, sub
        if first_grads is None:
            torch.cuda.synchronize()
            first_grads = [worker.arena.grad_view(s).float().cpu().clone()
                           for s in sorted(worker.arena.slots, key=lambda s: s.index) if s.is_model]
    torch.cuda.synchronize()
    n_graphs = len(worker.graphed._graphs) if worker.graphed is not None else 0
    _RUNS[(algo, graph)] = (np.asarray(rows, dtype=np.float64), first_grads, n_fp8, len(sites), n_graphs)
    del worker
    torch.cuda.empty_cache()
    return _RUNS[(algo, graph)]


def _torch_quantize(t, dtype, fmax):
    """The same recipe in stock torch: power-of-two scale from the tensor's amax, on the device."""
    amax = t.float().abs().max()
    ma, ea = torch.frexp(amax)
    mm, em = math.frexp(fmax)
    k = (em - ea - (ma > mm).to(ea.dtype)).clamp(-126, 126).float()
    scale = torch.where(amax == 0, torch.ones_like(amax), torch.exp2(k))
    return (t.float() * scale).clamp(-fmax, fmax).to(dtype), (1.0 / scale).reshape(())


class _TorchFp8Linear(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, b):
        xq, sx = _torch_quantize(x, torch.float8_e4m3fn, 448.0)
        wq, sw = _torch_quantize(w, torch.float8_e4m3fn, 448.0)
        ctx.save_for_backward(xq, sx, wq, sw)
        return torch._scaled_mm(xq, wq.t(), sx, sw, bias=b, out_dtype=torch.bfloat16)

    @staticmethod
    def backward(ctx, dy):
        xq, sx, wq, sw = ctx.saved_tensors
        dq, sd = _torch_quantize(dy.contiguous(), torch.float8_e5m2, 57344.0)
        dx = torch._scaled_mm(dq, wq.t().contiguous().t(), sd, sw, out_dtype=torch.bfloat16)
        dw = torch._scaled_mm(dq.t().contiguous(), xq.t().contiguous().t(), sd, sx, out_dtype=torch.bfloat16)
        return dx, dw, dy.float().sum(0).to(dy.dtype)


class _FusedHeads(torch.autograd.Function):
    """The task heads as this repo runs them: one F.linear per head forward, and the input gradient
    as ONE GEMM over the concatenated heads (autograd sums one GEMM per head instead)."""

    @staticmethod
    def forward(ctx, x, *params):
        ctx.save_for_backward(x, *params)
        return tuple(torch.nn.functional.linear(x, params[i], params[i + 1]) for i in range(0, len(params), 2))

    @staticmethod
    def backward(ctx, *dys):
        x, *params = ctx.saved_tensors
        dx = torch.cat(dys, dim=1) @ torch.cat(params[0::2], dim=0)
        grads = []
        for dy in dys:
            grads += [dy.t() @ x, dy.float().sum(0).to(dy.dtype)]
        return (dx,) + tuple(grads)


def _stock_fp8_first_grads(fused_heads):
    """First-step gradients of the plain module in stock torch (bf16, trunk Linear layers through
    the torch FP8 recipe above), with the heads' input gradient as autograd computes it or as one
    GEMM like this repo."""
    key = ("stock", fused_heads)
    if key not in _RUNS:
        _, problem = _headline_problem("/tmp/unused")
        stock = problem.get_model().cuda().to(torch.bfloat16)
        for m in stock.model_base.modules():
            if type(m) is nn.Linear:
                m.forward = types.MethodType(lambda self, x: _TorchFp8Linear.apply(x, self.weight, self.bias), m)
        if fused_heads:
            params = [p for h in stock.additional_layers for p in (h.weight, h.bias)]
            stock.forward = lambda xs: list(_FusedHeads.apply(stock.model_base(xs), *params))
        x, y, r = _batches()[0]
        out = stock([x.cuda().to(torch.bfloat16)])
        loss = torch.nn.functional.cross_entropy(out[0].float(), y.cuda()) + \
            torch.nn.functional.mse_loss(out[1].float(), r.cuda())
        loss.backward()
        _RUNS[key] = [p.grad.float().cpu() for p in stock.parameters()]
    return _RUNS[key]


def _rel(a, b):
    return [float((x - y).norm() / y.norm()) for x, y in zip(a, b)]


@pytest.mark.parametrize("graph", ["0", "1"])
@pytest.mark.parametrize("algo", ["sgd", "adam"])
def test_headline_mlp_in_fp8(algo, graph, monkeypatch):
    rows, grads, n_fp8, n_sites, n_graphs = _fp8_run(algo, graph, monkeypatch)
    assert (n_fp8, n_sites) == (3, 5)
    want_rows, want_grads, _ = _oracle(algo)
    stock, stock_fused = _stock_fp8_first_grads(False), _stock_fp8_first_grads(True)
    same = _rel(grads, stock_fused)
    # why the comparison computes the heads' dX as this repo does: requantising dZ to e5m2 turns a
    # last-bit bf16 difference upstream into whole-code flips, layer after layer (measured: 7e-2
    # on W1 between the two stock variants)
    floor = _rel(stock_fused, stock)
    vs_oracle = _rel(grads, want_grads)
    loss_err = np.abs(rows - want_rows) / np.abs(want_rows)
    fmt = lambda v: " ".join("%.1e" % e for e in v)              # noqa: E731
    print("fp8 %s graph=%s: first-step gradients, relative L2 per tensor (W1 b1 W2 b2 W3 b3 heads)\n"
          "  vs stock torch doing the same FP8 recipe, heads' dX as one GEMM: %s\n"
          "  stock torch, heads' dX as one GEMM vs as autograd sums it:      %s\n"
          "  vs the fp32 CPU oracle:                                          %s\n"
          "  worst loss error per step vs the fp32 CPU oracle: %s"
          % (algo, graph, fmt(same), fmt(floor), fmt(vs_oracle), fmt(loss_err.max(1))))
    # measured on an H100: 0 for every tensor, i.e. bit for bit the stock recipe
    assert max(same) <= 1e-2
    assert float(loss_err.max()) <= 5e-2
    if graph == "1":
        assert n_graphs == 1


@pytest.mark.parametrize("algo", ["sgd", "adam"])
def test_cuda_graph_replay_reproduces_the_eager_fp8_run(algo, monkeypatch):
    eager = _fp8_run(algo, "0", monkeypatch)
    graphed = _fp8_run(algo, "1", monkeypatch)
    assert graphed[4] == 1
    np.testing.assert_array_equal(graphed[0], eager[0])


# ---- checkpoints and fallbacks -----------------------------------------------------------------

def _small_run_opts(ns, n_epochs, batch=32):
    t = ns.types
    return t.RunOpts(optim=t.OptimOpts(algo=t.OptAlgorithm.ADAM, lr=1e-3), batchSize=batch, nEpochs=n_epochs,
                     numThreads=0, singleThreaded=True, numVisualizedSamples=0)


def _small_problem(ns, save_dir):
    return synthetic.make_mlp_problem(ns, save_dir, n_train=128, width=64, n_classes=16, reg_dim=16, depth=2)


def _solve(ns, save_dir, n_epochs, precision, stop_after=None):
    torch.manual_seed(0)
    gen = Solver.solve(_small_run_opts(ns, n_epochs), _small_problem(ns, save_dir), group_name=None,
                       init_method="file:///tmp/unused", precision=precision)
    out = []
    for s in gen:
        out.append(s)
        if s.epoch == stop_after:
            break
    gen.close()
    return out


def _layout(blob):
    def walk(x, path=""):
        if isinstance(x, torch.Tensor):
            yield path, tuple(x.shape), x.dtype
        elif isinstance(x, dict):
            for k in sorted(x, key=str):
                yield from walk(x[k], "%s/%s" % (path, k))
        elif isinstance(x, (list, tuple)):
            for i, v in enumerate(x):
                yield from walk(v, "%s/%d" % (path, i))
        else:
            yield path, type(x).__name__, None
    return list(walk(blob))


def test_fp8_checkpoints_have_the_bf16_layout_and_resume():
    ns = synthetic.api_namespace("frl_b200")
    dirs = {p: tempfile.mkdtemp(prefix="frl_b200_fp8_ckpt_") for p in (Precision.FP8, Precision.BF16)}
    for p, d in dirs.items():
        _solve(ns, d, 6, p, stop_after=5)                   # checkpoint cadence: epoch 5
        assert os.path.exists(os.path.join(d, ".checkpoint.pth"))
    load = lambda p, name: torch.load(os.path.join(dirs[p], name), weights_only=False)   # noqa: E731
    assert _layout(load(Precision.FP8, ".checkpoint.pth")) == _layout(load(Precision.BF16, ".checkpoint.pth"))
    ckpt = load(Precision.FP8, ".checkpoint.pth")
    assert all(v.dtype == torch.float32 for v in ckpt["state_dict"].values())
    fp32_dir = tempfile.mkdtemp(prefix="frl_b200_fp8_ckpt_")
    shutil.copy(os.path.join(dirs[Precision.FP8], ".checkpoint.pth"), fp32_dir)
    # resume under FP8 and load under FP32: both continue with epoch 6 and write the final model
    for d, p in ((dirs[Precision.FP8], Precision.FP8), (fp32_dir, Precision.FP32)):
        rest = _solve(ns, d, 6, p)
        assert [s.epoch for s in rest] == [6]
        assert all(np.isfinite(v) for v in rest[0].performance[ns.Split.TRAIN].losses.values())
        final = torch.load(os.path.join(d, "final_model.pth"), weights_only=False)
        assert _layout(final["state_dict"]) == _layout(ckpt["state_dict"])


def test_ragged_minibatch_falls_back_to_bf16_gemms(monkeypatch):
    ns = synthetic.api_namespace("frl_b200")
    t = ns.types
    save_dir = tempfile.mkdtemp(prefix="frl_b200_fp8_")
    torch.manual_seed(0)
    args = SolverWorkerArgs(run_opts=_small_run_opts(ns, 1), problem=_small_problem(ns, save_dir), save_dir=save_dir,
                            run_device=Device.GPU, node_idx=0, node_count=1, rank=0, local_rank=0, world_size=1,
                            group_name=None, init_method="", precision=Precision.FP8)
    worker, _, _ = Solver.build_worker(args)
    worker.model.train()
    assert sum(s.fp8 for s in worker.pipeline.linear_sites) == 2
    calls = {"fp8": 0, "bf16": 0}
    orig = arena_linear._ArenaLinearFn.apply

    def counted(x, weight, bias, site, fp8, for_backward):
        calls["fp8" if fp8 else "bf16"] += 1
        return orig(x, weight, bias, site, fp8, for_backward)
    monkeypatch.setattr(arena_linear._ArenaLinearFn, "apply", counted)
    g = torch.Generator().manual_seed(7)
    for step, (rows, want) in enumerate(((32, {"fp8": 2, "bf16": 0}), (24, {"fp8": 2, "bf16": 2}))):
        x = torch.randn(rows, 64, generator=g).cuda()
        y = torch.randint(0, 16, (rows,), generator=g).cuda()
        r = torch.randn(rows, 16, generator=g).cuda()
        _, total, _, _ = worker._pass_one_minibatch(step, t.Split.TRAIN, [x], [(y,), (r,)])
        assert math.isfinite(float(total)) and calls == want, (rows, calls)
