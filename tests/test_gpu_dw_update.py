"""K12 on the H100: the weight-gradient GEMM dW = dZ^T X (``frl_dw_gemm``) and the same GEMM with
the SGD update in its epilogue (``frl_dw_gemm_sgd``).

* gradient: within cuBLAS's own error of a float64 dZ^T X (the summation order differs, so bit
  equality with cuBLAS is not expected), at the headline 4096^3 and at small, padded shapes;
* update: bit for bit what K2 (``frl_sgd_momentum``) computes on a copy of the pre-step state from
  the gradient K12 wrote -- first and later steps, momentum and plain SGD, an lr changed between
  CUDA-graph replays through the device-resident scalars, NaN and inf in dZ;
* wiring: every configuration K12 does not serve (a weight applied twice, FP8, fp32, clipping,
  accumulation, LARS) keeps the tail update and trains to the weights the tail update gives; a 1-GPU
  bf16 SGD MLP trains to the same weights with and without K12 within the bf16 parity bounds.
"""
import tempfile

import pytest
import torch
import torch.nn as nn

import frl_b200  # noqa: F401
from frl_b200 import _native, synthetic
from frl_b200.solver import Solver, SolverWorkerArgs
from frl_b200.types import Device, LayerAdaptation, Precision

pytestmark = pytest.mark.gpu
SGD = dict(lr=0.01, mu=0.9, dampening=0.0, wd=1e-4)


def _operands(rows, out, inp, pad=0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    dz = torch.randn(rows, out + pad, device="cuda", generator=g).to(torch.bfloat16)[:, :out]
    x = torch.randn(rows, inp, device="cuda", generator=g).to(torch.bfloat16)
    return dz, x


@pytest.mark.parametrize("rows,out,inp,pad", [(4096, 4096, 4096, 0), (64, 128, 256, 0), (192, 384, 512, 8),
                                              (1024, 1280, 768, 0)])
def test_gradient_is_within_the_cublas_error_envelope(rows, out, inp, pad):
    dz, x = _operands(rows, out, inp, pad)
    gw = torch.full((out, inp), float("nan"), device="cuda", dtype=torch.bfloat16)
    _native.dw_gemm(dz, x, gw)
    ref = dz.double().t() @ x.double()
    err_k12 = (gw.double() - ref).abs().max().item()
    err_cublas = (torch.mm(dz.t(), x).double() - ref).abs().max().item()
    assert torch.isfinite(gw).all()
    assert err_k12 <= 1.25 * err_cublas, (err_k12, err_cublas)


def _state(n, seed=1):
    g = torch.Generator(device="cuda").manual_seed(seed)
    p = torch.randn(n, device="cuda", generator=g)
    return p, torch.randn(n, device="cuda", generator=g), p.to(torch.bfloat16)


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t.view(torch.int16)


def _assert_same_bits(a, b):
    assert torch.equal(_bits(a), _bits(b))


@pytest.mark.parametrize("first_step", [True, False])
@pytest.mark.parametrize("mu", [0.9, 0.0])
@pytest.mark.parametrize("shape", [(4096, 4096, 4096), (128, 256, 512)])
def test_update_is_k2_on_the_written_gradient_bit_for_bit(first_step, mu, shape):
    rows, out, inp = shape
    dz, x = _operands(rows, out, inp)
    n = out * inp
    p, buf, lp = _state(n)
    p2, buf2, lp2 = p.clone(), buf.clone(), lp.clone()
    gw = torch.empty(out, inp, device="cuda", dtype=torch.bfloat16)
    kw = dict(SGD, mu=mu, dampening=0.1 if mu else 0.0)
    _native.dw_gemm_sgd(dz, x, gw, p, buf if mu else None, lp, first_step=first_step, **kw)
    gw_plain = torch.empty_like(gw)
    _native.dw_gemm(dz, x, gw_plain)
    _native.sgd_momentum(p2, gw.view(-1), buf2 if mu else None, lp2, n, first_step=first_step, **kw)
    _assert_same_bits(gw, gw_plain)
    _assert_same_bits(p, p2)
    _assert_same_bits(lp, lp2)
    _assert_same_bits(buf, buf2)


def test_nan_and_inf_in_dz_propagate_as_in_k2():
    dz, x = _operands(256, 256, 512)
    dz[3, 7] = float("nan")
    dz[10, 200] = float("inf")
    dz[11, 200] = float("-inf")
    n = 256 * 512
    p, buf, lp = _state(n)
    p2, buf2, lp2 = p.clone(), buf.clone(), lp.clone()
    gw = torch.empty(256, 512, device="cuda", dtype=torch.bfloat16)
    _native.dw_gemm_sgd(dz, x, gw, p, buf, lp, **SGD)
    _native.sgd_momentum(p2, gw.view(-1), buf2, lp2, n, **SGD)
    assert not torch.isfinite(gw).all()
    for a, b in ((p, p2), (buf, buf2), (lp, lp2)):
        _assert_same_bits(a, b)


def test_lr_changed_between_graph_replays_follows_the_device_scalars():
    dz, x = _operands(256, 256, 512)
    n = 256 * 512
    p, buf, lp = _state(n)
    p2, buf2, lp2 = p.clone(), buf.clone(), lp.clone()
    gw = torch.empty(256, 512, device="cuda", dtype=torch.bfloat16)
    dyn = torch.tensor([0.5, 0, 0, 0], device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):        # warm-up outside the capture: driver entry point, smem attribute
        _native.dw_gemm_sgd(dz, x, torch.empty_like(gw), p.clone(), buf.clone(), lp.clone(), dyn=dyn, **SGD)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        _native.dw_gemm_sgd(dz, x, gw, p, buf, lp, dyn=dyn, **SGD)
    for lr in (0.25, 0.125, 0.03):
        dyn[0] = lr
        graph.replay()
        _native.sgd_momentum(p2, gw.view(-1), buf2, lp2, n, dyn=dyn, **SGD)
        torch.cuda.synchronize()
        for a, b in ((p, p2), (buf, buf2), (lp, lp2)):
            _assert_same_bits(a, b)


def test_shapes_off_the_tile_are_rejected():
    dz, x = _operands(64, 128, 256)
    gw = torch.empty(128, 256, device="cuda", dtype=torch.bfloat16)
    assert _native.dw_gemm_fits(dz, x, gw)
    assert not _native.dw_gemm_fits(dz[:32], x[:32], gw)
    assert not _native.dw_gemm_fits(dz[:, :64], x, gw[:64])
    with pytest.raises(_native.NativeLibraryError):
        _native.dw_gemm(dz[:, :64], x, gw[:64])


# ---- wiring -------------------------------------------------------------------------------------

WIDTH, BATCH, STEPS = 512, 64, 5


def _mlp_run(monkeypatch, fused, precision=Precision.BF16, clip=0.0, accumulation=1,
             adaptation=LayerAdaptation.NONE, graph="1"):
    monkeypatch.setenv("FRL_B200_FUSED_DW_UPDATE", fused)
    monkeypatch.setenv("FRL_B200_CUDA_GRAPH", graph)
    ns = synthetic.api_namespace("frl_b200")
    t = ns.types
    save_dir = tempfile.mkdtemp(prefix="frl_b200_dw_")
    torch.manual_seed(0)
    problem = synthetic.make_mlp_problem(ns, save_dir, n_train=8, width=WIDTH, n_classes=100, reg_dim=64, depth=3)
    run_opts = t.RunOpts(optim=t.OptimOpts(algo=t.OptAlgorithm.SGD, lr=0.01, momentum=0.9, gradientClip=clip),
                         batchSize=BATCH, nEpochs=1, numThreads=0, singleThreaded=True, numVisualizedSamples=0)
    args = SolverWorkerArgs(run_opts=run_opts, problem=problem, save_dir=save_dir, run_device=Device.GPU,
                            node_idx=0, node_count=1, rank=0, local_rank=0, world_size=1, group_name=None,
                            init_method="", precision=precision, layer_adaptation=adaptation,
                            grad_accumulation=accumulation)
    worker, _, _ = Solver.build_worker(args)
    worker.model.train()
    worker.criterion.train()
    g = torch.Generator().manual_seed(1234)
    losses = []
    for i in range(STEPS):
        x = torch.randn(BATCH, WIDTH, generator=g).cuda()
        y = torch.randint(0, 100, (BATCH,), generator=g).cuda()
        r = torch.randn(BATCH, 64, generator=g).cuda()
        _, total, _, _ = worker._pass_one_minibatch(i, t.Split.TRAIN, [x], [(y,), (r,)])
        losses.append(float(total.detach()))
        del total
    torch.cuda.synchronize()
    return worker.pipeline, worker.arena.master.clone(), losses


@pytest.mark.parametrize("graph", ["0", "1"])
def test_bf16_sgd_mlp_with_and_without_k12(monkeypatch, graph):
    pipe, w_fused, l_fused = _mlp_run(monkeypatch, "1", graph=graph)
    assert pipe.fused_dw_update and len(pipe.dw_updated) == 3          # the three trunk weights
    pipe0, w_tail, l_tail = _mlp_run(monkeypatch, "0", graph=graph)
    assert not pipe0.fused_dw_update and not pipe0.dw_updated
    torch.testing.assert_close(torch.tensor(l_fused), torch.tensor(l_tail), rtol=1e-2, atol=0)
    rel = (w_fused - w_tail).norm() / w_tail.norm()
    assert rel < 1e-2, rel


@pytest.mark.parametrize("config", [dict(precision=Precision.FP32), dict(precision=Precision.FP8),
                                    dict(clip=1.0), dict(accumulation=2),
                                    dict(adaptation=LayerAdaptation.LARS)],
                         ids=["fp32", "fp8", "clip", "accumulation", "lars"])
def test_configurations_k12_does_not_serve_keep_the_tail_update(monkeypatch, config):
    pipe, w_on, l_on = _mlp_run(monkeypatch, "1", graph="0", **config)
    assert not pipe.fused_dw_update and not pipe.dw_updated
    _, w_off, l_off = _mlp_run(monkeypatch, "0", graph="0", **config)
    assert l_on == l_off
    assert torch.equal(w_on, w_off)


def test_a_weight_applied_twice_keeps_the_tail_update():
    from frl_b200 import fused_optim, grad_sync
    from frl_b200.arena import ParamArena
    from frl_b200.types import OptAlgorithm, OptimOpts

    torch.manual_seed(0)
    lin = nn.Linear(256, 256).cuda()
    head = nn.Linear(256, 256).cuda()
    arena = ParamArena(list(lin.parameters()) + list(head.parameters()), device="cuda", precision=Precision.BF16)
    opt = fused_optim.create_fused_optimizer(arena, OptimOpts(algo=OptAlgorithm.SGD, lr=0.1, momentum=0.9))
    pipe = grad_sync.GradBucketPipeline(arena, opt, world_size=1, eager_update=False)
    pipe.patch_linears(nn.ModuleList([lin, head]))
    assert pipe.fused_dw_update
    x = torch.randn(64, 256, device="cuda").to(torch.bfloat16)
    out = head(lin(lin(x)))
    pipe.begin_step()
    out.float().square().mean().backward()
    pipe.finish_step()
    assert pipe.dw_updated == {arena.slot_of(head.weight).index}      # lin ran twice: tail update
