"""Schedule-Free AdamW / SGD on the H100: the frl_sf_* update kernels (K2 in every instantiation, K2-mt,
grouped, SR and grouped SR) against float64, a device ``dyn`` overriding wrong by-value scalars, NaN
propagation, K2-sfx against float64, swaps that restore every byte in each precision and master mode,
and training runs through the solver (FP32, BF16 with graph replay, bf16 master weights, FP8) with the
held-out split at x, and ``<stem>.sf`` reproducing the held-out loss in ``Mode.EVAL``."""
import io
import os

import numpy as np
import pytest
import torch
import torch.nn as nn

import frl_b200  # noqa: F401
from frl_b200 import _native, fused_optim, synthetic
from frl_b200.arena import ParamArena
from frl_b200.multi_tensor import GradSegTable
from frl_b200.solver import Solver, SolverWorkerArgs
from frl_b200.types import Device, MasterWeights, Mode, OptAlgorithm, OptimOpts, Precision, RunOpts, ScheduleFree, Split
from schedule_free_oracle import sf_eval_f64
from sr_oracle import sr_arena

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _sf_f64(adaptive, y, g, z, v, *, lr, ckp1, beta1, wd, beta2=0.999, eps=1e-8):
    y, g, z = y.double(), g.double(), z.double()
    u = g
    if adaptive:
        v = v.double() * beta2 + (1 - beta2) * g * g
        u = g / (v.sqrt() + eps)
    u = u + wd * y
    y = y + ckp1 * (z - y)
    y = y + lr * (beta1 * (1 - ckp1) - 1) * u
    return y, z - lr * u, v


def _inputs(n, seed=0):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    y = torch.randn(n, device=DEV, generator=gen)
    z = y + 0.01 * torch.randn(n, device=DEV, generator=gen)
    v = torch.rand(n, device=DEV, generator=gen) * 1e-3
    g = torch.randn(n, device=DEV, generator=gen)
    return y, z, v, g


def _close(got, want, rtol=2e-6, atol=1e-6):
    torch.testing.assert_close(got.double(), want, rtol=rtol, atol=atol)


@pytest.mark.parametrize("adaptive", [True, False])
@pytest.mark.parametrize("g_dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("shadow", [False, True])
@pytest.mark.parametrize("ckp1", [1.0, 0.3, 0.7])
def test_k2_matches_float64(adaptive, g_dtype, shadow, ckp1):
    n = 50_003
    y, z, v, g = _inputs(n)
    g = g.to(g_dtype)
    lp = torch.empty(n, dtype=torch.bfloat16, device=DEV) if shadow else None
    kw = dict(lr=3e-3, ckp1=ckp1, beta1=0.9, wd=0.05)
    want_y, want_z, want_v = _sf_f64(adaptive, y, g.float(), z, v, **kw)
    if adaptive:
        _native.sf_adamw(y, g, z, v, lp, n, beta2=0.999, eps=1e-8, **kw)
        _close(v, want_v)
    else:
        _native.sf_sgd(y, g, z, lp, n, **kw)
    _close(y, want_y)
    _close(z, want_z)
    if shadow:
        assert torch.equal(lp, y.to(torch.bfloat16))


@pytest.mark.parametrize("adaptive", [True, False])
def test_k2_mt_and_grouped_match_k2(adaptive):
    sizes = [4096 * 5 + 3, 17, 70_000, 256]
    params = [nn.Parameter(torch.randn(s)) for s in sizes]
    arena = ParamArena(params, device=DEV)
    n = arena.numel
    z = arena.master * 1.01                  # the arena's zero padding stays zero in every form
    v = torch.rand(n, device=DEV) * 1e-3
    grads = [torch.randn(s, device=DEV) for s in sizes]
    table = GradSegTable(arena.slots, torch.device(DEV))
    for s, gr in zip(arena.slots, grads):
        table.point(s, gr.data_ptr(), gr.dtype)
    table.upload()
    flat = torch.zeros(n, device=DEV)
    for s, gr in zip(arena.slots, grads):
        flat[s.offset:s.end] = gr
    kw = dict(lr=1e-3, ckp1=0.25, beta1=0.9, wd=0.01)
    rule = dict(beta2=0.999, eps=1e-8) if adaptive else {}
    st = (z, v) if adaptive else (z,)
    ref = [t.clone() for t in (arena.master,) + st]
    (_native.sf_adamw if adaptive else _native.sf_sgd)(ref[0], flat, *ref[1:], None, n, **kw, **rule)
    mt = [t.clone() for t in (arena.master,) + st]
    (_native.sf_adamw_mt if adaptive else _native.sf_sgd_mt)(mt[0], *mt[1:], None, table, **kw, **rule)
    def same(a, b):                          # the slots (the flat form also moves the padding)
        return all(torch.equal(a[s.offset:s.end], b[s.offset:s.end]) for s in arena.slots)

    assert all(same(a, b) for a, b in zip(ref, mt))
    # grouped, one group whose row carries the same scalars
    rows = torch.zeros(1, _native.GROUP_DYN_COLS, device=DEV)
    y_lr = kw["lr"] * (kw["beta1"] * (1 - kw["ckp1"]) - 1)
    rows[0, :3] = torch.tensor([kw["lr"], kw["ckp1"], y_lr])
    rows[0, 4] = kw["wd"]
    groups = _native.SegGroups([0] * len(sizes), [0] * len(sizes), rows)
    gr_ = [t.clone() for t in (arena.master,) + st]
    (_native.sf_adamw_mt_grouped if adaptive else _native.sf_sgd_mt_grouped)(gr_[0], *gr_[1:], None, table, groups,
                                                                              beta1=0.9, **rule)
    assert all(same(a, b) for a, b in zip(ref, gr_))


@pytest.mark.parametrize("adaptive", [True, False])
def test_device_dyn_overrides_wrong_by_value_scalars(adaptive):
    n = 10_000
    y, z, v, g = _inputs(n, 3)
    kw = dict(lr=2e-3, ckp1=0.4, beta1=0.9, wd=0.0)
    rule = dict(beta2=0.999, eps=1e-8) if adaptive else {}
    ref = [t.clone() for t in (y, z, v)]
    fn = _native.sf_adamw if adaptive else _native.sf_sgd
    st = lambda t: (t[1], t[2]) if adaptive else (t[1],)
    fn(ref[0], g, *st(ref), None, n, **kw, **rule)
    y_lr = kw["lr"] * (kw["beta1"] * (1 - kw["ckp1"]) - 1)
    dyn = torch.tensor([kw["lr"], kw["ckp1"], y_lr, 0.0], device=DEV)
    got = [t.clone() for t in (y, z, v)]
    fn(got[0], g, *st(got), None, n, **dict(kw, lr=9.0, ckp1=0.9), **rule, dyn=dyn)
    for a, b in zip(ref, got):
        assert torch.equal(a, b)


def test_nan_reaches_the_weights():
    n = 64
    y, z, v, g = _inputs(n, 4)
    g[5] = float("nan")
    _native.sf_adamw(y, g, z, v, None, n, lr=1e-3, ckp1=0.5, beta1=0.9, beta2=0.999, eps=1e-8, wd=0.0)
    assert torch.isnan(y[5]) and torch.isnan(z[5]) and torch.isfinite(y[:5]).all()


@pytest.mark.parametrize("adaptive", [True, False])
def test_sr_forms_round_within_one_bf16_ulp_and_grouped_sr_matches(adaptive):
    sizes = [8192 + 5, 300]
    params = [nn.Parameter(torch.randn(s)) for s in sizes]
    arena = ParamArena(params, device=DEV, precision=Precision.BF16, master_weights=MasterWeights.BF16)
    n = arena.model_end
    y = arena.lp
    z = y[:n].float() * 1.5 + 0.1 * (y[:n].float() != 0)     # padding stays zero
    v = torch.zeros(n, device=DEV)             # v and g zero on the padding, which only the flat form moves
    g = torch.zeros(n, device=DEV)
    for s in arena.slots:
        g[s.offset:s.end] = torch.randn(s.numel, device=DEV)
        v[s.offset:s.end] = torch.rand(s.numel, device=DEV) * 1e-3
    kw = dict(lr=1e-3, ckp1=0.3, beta1=0.9, wd=0.01)
    rule = dict(beta2=0.999, eps=1e-8) if adaptive else {}
    # K2-sr is the fp32 rule (frl_sf_* on an fp32 copy of the bf16 weights) then the stochastic rounding of
    # K2-sr's definition (tests/sr_oracle.py), bit for bit
    y32, st32 = y[:n].float(), ((z.clone(), v.clone()) if adaptive else (z.clone(),))
    (_native.sf_adamw if adaptive else _native.sf_sgd)(y32, g, *st32, None, n, **kw, **rule)
    st = (z.clone(), v.clone()) if adaptive else (z.clone(),)
    y1 = y.clone()
    (_native.sf_adamw_sr if adaptive else _native.sf_sgd_sr)(y1[:n], g, *st, n, arena_off=0, seed=7, t=3, **kw,
                                                                **rule)
    torch.cuda.synchronize()
    assert np.array_equal(y1[:n].view(torch.int16).cpu().numpy().view(np.uint16), sr_arena(y32.cpu().numpy(), 0, 3, 7))
    assert all(torch.equal(a, b) for a, b in zip(st, st32))
    # and the fp32 rule itself against float64: z far enough from y that the lerp term is many bf16 ulps
    want_y, want_z, _ = _sf_f64(adaptive, y[:n].float(), g, z, v, **kw)
    _close(y32, want_y)
    _close(st32[0], want_z)
    table = GradSegTable(arena.slots, torch.device(DEV))
    for s in arena.slots:
        table.point(s, g.data_ptr() + s.offset * 4, g.dtype)
    table.upload()
    st2 = (z.clone(), v.clone()) if adaptive else (z.clone(),)
    y2 = y.clone()
    (_native.sf_adamw_mt_sr if adaptive else _native.sf_sgd_mt_sr)(y2, *st2, table, seed=7, t=3, **kw, **rule)
    assert torch.equal(y1[:n], y2[:n]) and all(torch.equal(a, b) for a, b in zip(st, st2))
    rows = torch.zeros(1, _native.GROUP_DYN_COLS, device=DEV)
    rows[0, :3] = torch.tensor([kw["lr"], kw["ckp1"], kw["lr"] * (0.9 * (1 - kw["ckp1"]) - 1)])
    rows[0, 4] = kw["wd"]
    rows.view(torch.int32)[0, 3] = 3
    groups = _native.SegGroups([0, 0], [0, 0], rows)
    st3 = (z.clone(), v.clone()) if adaptive else (z.clone(),)
    y3 = y.clone()
    (_native.sf_adamw_mt_grouped_sr if adaptive else _native.sf_sgd_mt_grouped_sr)(y3, *st3, table, groups, seed=7,
                                                                                  beta1=0.9, **rule)
    assert torch.equal(y1[:n], y3[:n]) and all(torch.equal(a, b) for a, b in zip(st, st3))


@pytest.mark.parametrize("y_dtype,x_dtype", [(torch.float32, torch.bfloat16), (torch.float32, torch.float32),
                                              (torch.bfloat16, torch.bfloat16), (torch.bfloat16, torch.float32)])
@pytest.mark.parametrize("beta1", [0.9, 0.5])
def test_k2_sfx_matches_float64(y_dtype, x_dtype, beta1):
    n = 100_001
    y, z, _, _ = _inputs(n, 5)
    y = y.to(y_dtype)
    want = sf_eval_f64(y.float(), z, beta1)
    x = torch.empty(n, dtype=x_dtype, device=DEV)
    _native.sf_eval_weights(y, z, x, beta1=beta1)
    if x_dtype == torch.float32:
        _close(x, want, rtol=2e-6, atol=1e-6)
    else:
        torch.testing.assert_close(x.float(), want.float().to(torch.bfloat16).float(), rtol=8e-3, atol=1e-5)
    if y_dtype == x_dtype:                    # in place
        y2 = y.clone()
        _native.sf_eval_weights(y2, z, y2, beta1=beta1)
        assert torch.equal(y2, x)


@pytest.mark.parametrize("precision,master", [(Precision.FP32, MasterWeights.FP32), (Precision.BF16, MasterWeights.FP32),
                                              (Precision.BF16, MasterWeights.BF16)])
def test_swap_restores_every_byte(precision, master):
    torch.manual_seed(0)
    net = nn.Sequential(nn.Linear(64, 64), nn.ReLU(), nn.Linear(64, 10)).to(DEV)
    arena = ParamArena(list(net.parameters()), device=DEV, precision=precision, master_weights=master)
    opt = fused_optim.FusedScheduleFreeAdamW(arena, lr=1e-2)
    for i in range(3):
        arena.grad.copy_(torch.randn(arena.numel, device=DEV).to(arena.grad.dtype))
        opt.step()
    before = [t.clone() for t in (arena.master, arena.lp) if t is not None]
    x = opt.eval_weights()
    y = (arena.lp if master is MasterWeights.BF16 else arena.master)[:arena.model_end]
    _close(x, sf_eval_f64(y.float(), opt._state("z")[:arena.model_end], 0.9))
    with opt.swapped():
        seen = (arena.lp if arena.lp is not None else arena.master)[:arena.model_end].float()
        want = x.to(torch.bfloat16).float() if arena.lp is not None else x
        assert torch.equal(seen, want)
    after = [t for t in (arena.master, arena.lp) if t is not None]
    assert all(torch.equal(a, b) for a, b in zip(before, after))


# ---- through the solver -----------------------------------------------------------------------------

def _args(tmp_path, algo, precision, master=MasterWeights.FP32, graph=False, n_epochs=2, mode=Mode.TRAIN,
          initial=None):
    ns = synthetic.api_namespace("frl_b200")
    torch.manual_seed(0)
    problem = synthetic.make_toy_problem(ns, str(tmp_path), n_train=512, n_test=128)
    opts = OptimOpts(algo=algo, lr=1e-2 if algo == OptAlgorithm.ADAM else 0.05, momentum=0.9, weightDecay=1e-4,
                     gradientClip=0.0)
    run_opts = RunOpts(optim=opts, batchSize=64, nEpochs=n_epochs, numThreads=0, singleThreaded=True,
                       numVisualizedSamples=2, mode=mode, initialModelPath=initial)
    return SolverWorkerArgs(run_opts=run_opts, problem=problem, save_dir=str(tmp_path), run_device=Device.GPU,
                            node_idx=0, node_count=1, rank=0, local_rank=0, world_size=1, group_name=None,
                            init_method="", precision=precision, graph_step=graph, master_weights=master,
                            schedule_free=ScheduleFree(warmup_steps=4) if mode == Mode.TRAIN else None)


@pytest.mark.parametrize("algo,precision,master,graph", [
    (OptAlgorithm.ADAM, Precision.FP32, MasterWeights.FP32, False),
    (OptAlgorithm.SGD, Precision.BF16, MasterWeights.FP32, True),
    (OptAlgorithm.ADAM, Precision.BF16, MasterWeights.BF16, False),
    (OptAlgorithm.SGD, Precision.FP8, MasterWeights.FP32, False),
])
def test_solver_trains_and_evaluates_held_out_at_x(tmp_path, algo, precision, master, graph):
    args = _args(tmp_path, algo, precision, master, graph)
    worker, scheduler, _ = Solver.build_worker(args)
    opt = worker.optimizer
    assert isinstance(opt, fused_optim.FusedScheduleFree) and not worker.pipeline.fused_dw_update
    results = list(worker.train(args.problem, startEpoch=0, nEpochs=2, batchSize=64, scheduler=scheduler))
    train = [r.performance[Split.TRAIN].losses for r in results]
    held = [r.performance[s].losses for r in results for s in r.performance if s != Split.TRAIN]
    assert all(np.isfinite(list(d.values())).all() for d in train + held)
    assert opt.hyper["k"] == opt._steps > 0
    # the held-out split was evaluated at x: the same split evaluated again, by hand, inside swapped()
    # reproduces the reported loss, and at y it differs
    split = [sp for sp in results[-1].performance if sp != Split.TRAIN][0]
    reported = results[-1].performance[split].losses
    y_before = (worker.arena.lp if worker.arena.bf16_master else worker.arena.master).clone()
    with opt.swapped():
        at_x = _held_out_losses(worker, args.problem, split)
    at_y = _held_out_losses(worker, args.problem, split)
    assert torch.equal(y_before, worker.arena.lp if worker.arena.bf16_master else worker.arena.master)
    for k in reported:
        assert at_x[k] == pytest.approx(reported[k], rel=1e-5, abs=1e-7), (k, at_x[k], reported[k])
    assert any(at_y[k] != pytest.approx(reported[k], rel=1e-6, abs=0) for k in reported), (at_y, reported)


def _held_out_losses(worker, problem, split):
    """The losses of ``split`` at the weights the model holds now (the worker's EVAL pass never swaps)."""
    return list(worker.eval(problem, batchSize=worker.run_opts.batchSize))[-1].performance[split].losses


def test_sf_file_evaluates_the_schedule_free_model(tmp_path):
    args = _args(tmp_path, OptAlgorithm.ADAM, Precision.FP32, n_epochs=1)
    held = list(Solver._run_solver_worker(args))[-1]
    # what the parent writes to <stem>.sf travels in the optimizer-state bytes
    blob = torch.load(io.BytesIO(held.optimizerStateBuffer), weights_only=False)
    path = os.path.join(str(tmp_path), "final_model.pth.sf")
    torch.save({"epoch": 1, "state_dict": blob.pop(fused_optim.SF_STATE_KEY)}, path)
    assert blob["param_groups"][0]["train_mode"] is True and "z" in blob["state"][0]
    ev = _args(tmp_path, OptAlgorithm.ADAM, Precision.FP32, mode=Mode.EVAL, initial=path)
    out = list(Solver._run_solver_worker(ev))[-1]
    split = [s for s in held.performance if s != Split.TRAIN][0]
    want, got = held.performance[split].losses, out.performance[split].losses
    for k in want:
        assert got[k] == pytest.approx(want[k], rel=1e-5, abs=1e-7), k
