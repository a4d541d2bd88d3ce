"""Lion (``Solver.solve(..., lion=True)``, the ``frl_lion*`` kernels) on the device.

* every K2 instantiation ({fp32, bf16 gradient} x {shadow off, on} x {host scale, device clip
  coefficient}), K2-mt, K2-sr and K2-mt-sr, and K12 / K12-sr, against the float64 restatement
  (tests/lion_oracle.py).  A sign may differ only where |c| is within a few ulps of zero; those
  elements are counted and bounded;
* bit-for-bit equality across paths: frl_lion == frl_lion_mt, frl_dw_gemm_lion == frl_dw_gemm +
  frl_lion, and the SR pair the same way;
* NaN propagation, a captured graph that follows an lr change through ``dyn``;
* through Solver.build_worker: the width-512 MLP against a ``RefLion`` loop, a resume bit for bit,
  graph replay, FP8, accumulation with clipping, EMA, bf16 master weights, a channels_last ResNet,
  and the optimizer state's size.
"""
import logging
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

import frl_b200  # noqa: F401
from frl_b200 import _native, fused_optim, synthetic
from frl_b200.multi_tensor import GradSegTable
from frl_b200.solver import Solver, SolverWorkerArgs
from frl_b200.types import Device, MasterWeights, OptAlgorithm, Precision, Split
from lion_oracle import RefLion, decay_factor, lion_step_f64
from sr_oracle import sr_arena

pytestmark = pytest.mark.gpu
DEV = "cuda"
SEED = 0x1234_5678_9ABC_DEF0
HYPER = dict(lr=1e-3, beta1=0.9, beta2=0.99, wd=0.1)
EPS32 = float(np.finfo(np.float32).eps)


def _inputs(n, gdt, seed):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    p = torch.randn(n, device=DEV, generator=gen) * 0.5
    g = (torch.randn(n, device=DEV, generator=gen) * 0.1).to(gdt)
    m = torch.randn(n, device=DEV, generator=gen) * 0.05
    return p, g, m


def _check_against_f64(p0, g, m0, p, m, *, gscale, h=HYPER):
    """The kernel's p and m against the float64 rule.  Away from a sign flip the weight is within a
    few fp32 roundings of |p| + lr (the decay product, the update's FMA, c's lerp cannot flip the
    sign there); m within a few roundings of |m| + |g|.  Flips are allowed only where |c| is within
    4 ulps of |m| + |g| of zero, and counted."""
    p64, m64, c64 = lion_step_f64(p0.double().cpu().numpy(), g.double().cpu().numpy() * gscale,
                                  m0.double().cpu().numpy(), **h)
    p, m = p.double().cpu().numpy(), m.double().cpu().numpy()
    g64 = np.abs(g.double().cpu().numpy() * gscale)
    near = np.abs(c64) <= 4 * EPS32 * (np.abs(m0.double().cpu().numpy()) + g64)
    err_p = np.abs(p - p64)
    ok_p = err_p <= 3 * EPS32 * (np.abs(p64) + h["lr"])
    flips = ~ok_p
    assert np.all(near[flips]), int((flips & ~near).sum())
    assert flips.sum() <= max(4, 1e-4 * p.size), int(flips.sum())
    assert np.all(np.abs(m - m64) <= 4 * EPS32 * (np.abs(m64) + g64 + 1e-30))
    return int(flips.sum())


@pytest.mark.parametrize("gdt", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("shadow", [False, True])
@pytest.mark.parametrize("coef", [False, True])
@pytest.mark.parametrize("n", [4099, 3 * 132 * 8 * 4096 + 3])
def test_k2_every_instantiation_against_float64(gdt, shadow, coef, n):
    p, g, m = _inputs(n, gdt, n + 2 * shadow + coef)
    p0, m0 = p.clone(), m.clone()
    lp = torch.empty(n, device=DEV, dtype=torch.bfloat16) if shadow else None
    cdev = torch.tensor([0.75], device=DEV) if coef else None
    _native.lion(p, g, m, lp, n, **HYPER, grad_scale=0.5, grad_scale_dev=cdev)
    torch.cuda.synchronize()
    _check_against_f64(p0, g, m0, p, m, gscale=0.5 * (0.75 if coef else 1.0))
    if shadow:
        assert torch.equal(lp, p.to(torch.bfloat16))


def _table(layout, gen, gdts=(torch.float32, torch.bfloat16)):
    class _Slot:
        def __init__(self, i, off, n):
            self.index, self.offset, self.numel, self.shape, self.is_model = i, off, n, (n,), True
            self.end = off + n

    slots, off = [], 0
    for i, n in enumerate(layout):
        slots.append(_Slot(i, off, n))
        off = (off + n + 7) // 8 * 8
    table = GradSegTable(slots, torch.device(DEV))
    grads = []
    for i, s in enumerate(slots):
        gd = (torch.randn(s.numel, device=DEV, generator=gen) * 0.1).to(gdts[i % len(gdts)])
        grads.append(gd)
        table.point(s, gd.data_ptr(), gd.dtype)
    table.upload()
    return slots, table, grads, off


def _zero_padding(slots, *vecs):
    """The arena keeps each slice's padding (up to a multiple of 8) at zero, in weights and state; the
    segment-table kernels update it with a zero gradient, which leaves it zero under Lion."""
    keep = torch.zeros(vecs[0].numel(), dtype=torch.bool, device=DEV)
    for s in slots:
        keep[s.offset:s.end] = True
    for v in vecs:
        v[~keep] = 0


MT_LAYOUT = [3, 4096 * 4 + 5, 17, 40000, 8]


def test_k2_mt_against_float64_and_equal_to_k2():
    gen = torch.Generator(device=DEV).manual_seed(5)
    slots, table, grads, total = _table(MT_LAYOUT, gen)
    p = torch.randn(total, device=DEV, generator=gen) * 0.5
    m = torch.randn(total, device=DEV, generator=gen) * 0.05
    _zero_padding(slots, p, m)
    lp = torch.zeros(total, device=DEV, dtype=torch.bfloat16)
    p0, m0 = p.clone(), m.clone()
    p2, m2, lp2 = p.clone(), m.clone(), lp.clone()
    _native.lion_mt(p, m, lp, table, **HYPER, grad_scale=0.5)
    for s, gd in zip(slots, grads):
        _native.lion(p2[s.offset:s.end], gd, m2[s.offset:s.end], lp2[s.offset:s.end], s.numel, **HYPER,
                     grad_scale=0.5)
    torch.cuda.synchronize()
    assert torch.equal(p, p2) and torch.equal(m, m2) and torch.equal(lp, lp2)      # frl_lion == frl_lion_mt
    for s, gd in zip(slots, grads):
        sl = slice(s.offset, s.end)
        _check_against_f64(p0[sl], gd, m0[sl], p[sl], m[sl], gscale=0.5)


@pytest.mark.parametrize("gdt", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("n, off", [(4099, 8), (70001, 4096)])
def test_k2_sr_is_the_fp32_rule_then_the_rounding(gdt, n, off):
    p, g, m = _inputs(n, gdt, n)
    w = p.to(torch.bfloat16)
    p32, m32 = w.float(), m.clone()
    _native.lion(p32, g, m32, None, n, **HYPER, grad_scale=0.5)
    _native.lion_sr(w, g, m, n, arena_off=off, seed=SEED, t=11, **HYPER, grad_scale=0.5)
    torch.cuda.synchronize()
    assert np.array_equal(w.view(torch.int16).cpu().numpy().view(np.uint16), sr_arena(p32.cpu().numpy(), off, 11, SEED))
    assert torch.equal(m, m32)


def test_k2_mt_sr_is_the_fp32_rule_then_the_rounding():
    gen = torch.Generator(device=DEV).manual_seed(9)
    slots, table, grads, total = _table(MT_LAYOUT, gen)
    w = (torch.randn(total, device=DEV, generator=gen) * 0.5).to(torch.bfloat16)
    m = torch.randn(total, device=DEV, generator=gen) * 0.05
    _zero_padding(slots, w, m)
    p32, m32 = w.float(), m.clone()
    _native.lion_mt(p32, m32, None, table, **HYPER)
    _native.lion_mt_sr(w, m, table, seed=SEED, t=4, **HYPER)
    torch.cuda.synchronize()
    assert torch.equal(m, m32)
    got = w.view(torch.int16).cpu().numpy().view(np.uint16)
    for s in slots:
        assert np.array_equal(got[s.offset:s.end], sr_arena(p32[s.offset:s.end].cpu().numpy(), s.offset, 4, SEED))


# K12 at 4096^2 and at shapes of its tile table (one tile, several k-blocks, a partial wave)
K12_SHAPES = [(4096, 4096, 4096), (128, 256, 64), (256, 512, 192), (384, 768, 256), (1024, 1024, 512)]


@pytest.mark.parametrize("out, inp, rows", K12_SHAPES)
@pytest.mark.parametrize("dyn_mode", [False, True])
def test_k12_lion_equals_dw_gemm_then_k2_and_follows_float64(out, inp, rows, dyn_mode):
    """With dyn the by-value lr and decay are wrong on purpose: LionRule::patch must take dyn's."""
    gen = torch.Generator(device=DEV).manual_seed(out + inp + rows)
    dz = torch.randn(rows, out, device=DEV, generator=gen).to(torch.bfloat16)
    x = torch.randn(rows, inp, device=DEV, generator=gen).to(torch.bfloat16)
    p = torch.randn(out * inp, device=DEV, generator=gen) * 0.05
    m = torch.randn(out * inp, device=DEV, generator=gen) * 1e-2
    p0, m0 = p.clone(), m.clone()
    gw_ref, p_ref, m_ref = torch.empty(out, inp, device=DEV, dtype=torch.bfloat16), p.clone(), m.clone()
    lp_ref = torch.empty(out * inp, device=DEV, dtype=torch.bfloat16)
    _native.dw_gemm(dz, x, gw_ref)
    _native.lion(p_ref, gw_ref.view(-1), m_ref, lp_ref, out * inp, **HYPER, grad_scale=0.25)
    gw, lp = torch.empty_like(gw_ref), torch.empty_like(lp_ref)
    kw, dyn = dict(HYPER), None
    if dyn_mode:
        dyn = torch.tensor([HYPER["lr"], float(decay_factor(HYPER["lr"], HYPER["wd"])), 0.0, 0.0], device=DEV)
        kw["lr"], kw["wd"] = 7.0, 0.5
    _native.dw_gemm_lion(dz, x, gw, p, m, lp, **kw, grad_scale=0.25, dyn=dyn)
    torch.cuda.synchronize()
    assert torch.equal(gw, gw_ref) and torch.equal(p, p_ref) and torch.equal(m, m_ref) and torch.equal(lp, lp_ref)
    _check_against_f64(p0, gw.view(-1), m0, p, m, gscale=0.25)


@pytest.mark.parametrize("out, inp, rows", K12_SHAPES[1:])
@pytest.mark.parametrize("dyn_mode", [False, True])
def test_k12_lion_sr_equals_dw_gemm_then_k2_sr(out, inp, rows, dyn_mode):
    """With dyn the by-value lr, decay and update count are wrong on purpose: dyn must win."""
    gen = torch.Generator(device=DEV).manual_seed(out + inp + rows + 1)
    dz = torch.randn(rows, out, device=DEV, generator=gen).to(torch.bfloat16)
    x = torch.randn(rows, inp, device=DEV, generator=gen).to(torch.bfloat16)
    w = (torch.randn(out * inp, device=DEV, generator=gen) * 0.05).to(torch.bfloat16)
    m = torch.randn(out * inp, device=DEV, generator=gen) * 1e-3
    off, t = 4096 + 8, 9
    dyn = None
    if dyn_mode:
        dyn = torch.tensor([HYPER["lr"], float(decay_factor(HYPER["lr"], HYPER["wd"])), 0.0, 0.0])
        dyn.view(torch.int32)[3] = t
        dyn = dyn.to(DEV)
    gw_ref, w_ref, m_ref = torch.empty(out, inp, device=DEV, dtype=torch.bfloat16), w.clone(), m.clone()
    _native.dw_gemm(dz, x, gw_ref)
    _native.lion_sr(w_ref, gw_ref.view(-1), m_ref, out * inp, arena_off=off, seed=SEED, t=t, **HYPER, grad_scale=0.5)
    kw = dict(HYPER)
    if dyn_mode:
        kw["lr"], kw["wd"] = 7.0, 0.5
    gw = torch.empty_like(gw_ref)
    _native.dw_gemm_lion_sr(dz, x, gw, w, m, arena_off=off, seed=SEED, t=1 if dyn_mode else t, **kw,
                            grad_scale=0.5, dyn=dyn)
    torch.cuda.synchronize()
    assert torch.equal(gw, gw_ref)
    assert torch.equal(w.view(torch.int16), w_ref.view(torch.int16)) and torch.equal(m, m_ref)


def test_nan_and_inf_reach_the_weight():
    n = 4099
    p, g, m = _inputs(n, torch.float32, 3)
    g[[5, 700]] = float("nan")
    g[900] = float("inf")
    _native.lion(p, g, m, None, n, **HYPER)
    torch.cuda.synchronize()
    assert torch.isnan(p[5]) and torch.isnan(p[700]) and torch.isnan(m[5])
    assert torch.isinf(m[900]) and torch.isfinite(p[900])                   # sign(+inf) = 1
    bad = torch.zeros(n, dtype=torch.bool, device=DEV)
    bad[[5, 700, 900]] = True
    assert torch.isfinite(p[~bad]).all() and torch.isfinite(m[~bad]).all()


def test_captured_graph_follows_an_lr_change_through_dyn():
    n = 70001
    p, g, m = _inputs(n, torch.bfloat16, 4)
    dyn = torch.zeros(4, device=DEV)
    s = torch.cuda.Stream()
    graph = torch.cuda.CUDAGraph()
    p_ref, m_ref = p.clone(), m.clone()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            _native.lion(p, g, m, None, n, lr=99.0, beta1=0.9, beta2=0.99, wd=0.1, dyn=dyn)
    for lr in (1e-3, 3e-4, 1e-4):
        dyn.copy_(torch.tensor([lr, float(decay_factor(lr, 0.1)), 0.0, 0.0]))
        graph.replay()
        _native.lion(p_ref, g, m_ref, None, n, lr=lr, beta1=0.9, beta2=0.99, wd=0.1)
    torch.cuda.synchronize()
    assert torch.equal(p, p_ref) and torch.equal(m, m_ref)


# ---- through Solver.build_worker ------------------------------------------------------------------------

def _worker(lion=True, seed=0, lr=1e-4, precision=Precision.BF16, graph=False, master=MasterWeights.FP32,
            algo=OptAlgorithm.SGD, **kw):
    ns = synthetic.api_namespace("frl_b200")
    t = ns.types
    save_dir = tempfile.mkdtemp(prefix="frl_b200_lion_")
    torch.manual_seed(seed)
    problem = synthetic.make_mlp_problem(ns, save_dir, n_train=8, width=512, n_classes=100, reg_dim=16, depth=3)
    run_opts = t.RunOpts(optim=t.OptimOpts(algo=algo, lr=lr, momentum=0.9, weightDecay=0.1),
                         batchSize=256, nEpochs=1, numThreads=0, singleThreaded=True, numVisualizedSamples=0)
    args = SolverWorkerArgs(run_opts=run_opts, problem=problem, save_dir=save_dir, run_device=Device.GPU,
                            node_idx=0, node_count=1, rank=0, local_rank=0, world_size=1, group_name=None,
                            init_method="", precision=precision, graph_step=graph, master_weights=master,
                            lion=lion, **kw)
    worker, _, _ = Solver.build_worker(args)
    worker.model.train()
    worker.criterion.train()
    return worker


def _batches(n, width=512, seed=1234):
    gen = torch.Generator().manual_seed(seed)
    w = torch.randn(width, 100, generator=gen) / width ** 0.5
    out = []
    for _ in range(n):
        x = torch.randn(256, width, generator=gen)
        out.append((x, (x @ w).argmax(1), torch.randn(256, 16, generator=gen) * 0.1 + x[:, :16]))
    return out


def _train(worker, batches, start=0):
    rows = []
    for i, (x, y, r) in enumerate(batches, start):
        _, total, _, _ = worker._pass_one_minibatch(i, Split.TRAIN, [x.cuda()], [(y.cuda(),), (r.cuda(),)])
        rows.append(float(total.detach()))
        del total
    torch.cuda.synchronize()
    return rows


def _params(worker):
    return list(worker.model.parameters()) + list(worker.criterion.parameters())


def _gap(a, b, p0):
    """Largest over the parameters of ||a - b|| / ||b - p0||: how far apart two runs' updates are."""
    return max(((x - y).norm() / (y - q).norm().clamp_min(1e-30)).item() for x, y, q in zip(a, b, p0))


def _weights(worker):
    with worker.arena.exported(cpu=False):
        return [p.detach().float().clone() for p in _params(worker)]


def test_solver_mlp_tracks_a_ref_lion_loop():
    """Precision.FP32, width-512 MLP, batch 256, 20 steps: the Solver with lion=True against stock
    autograd + ``RefLion`` with the same hyper-parameters.  The two differ in rounding order, and a
    sign flip where c is near zero moves an element by 2 lr, so the runs drift apart a little; they
    must stay far closer to each other than an SGD-momentum run is to the Lion reference.  Measured
    on an H100 80GB HBM3 (700 W, seed 0, this test): the largest per-parameter update gap to RefLion
    is 0.154 of the update, the SGD run's is 1.00.  Bound: 0.25, and a quarter of the SGD gap."""
    from oracle import ref_loop
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        batches = _batches(20)
        w = _worker(precision=Precision.FP32)
        assert type(w.optimizer) is fused_optim.FusedLion and not w.pipeline.fused_dw_update
        p0 = _weights(w)
        ns = synthetic.api_namespace("frl_b200")
        ref_problem = synthetic.make_mlp_problem(ns, tempfile.mkdtemp(prefix="frl_b200_lion_ref_"), n_train=8,
                                                 width=512, n_classes=100, reg_dim=16, depth=3)
        ref = ref_problem.get_model().cuda()
        ref.load_state_dict(w.model.state_dict())
        crit = ref_problem.get_criterion().cuda()
        crit.load_state_dict(w.criterion.state_dict())
        mods, weights, names = list(crit.loss_modules), list(crit.loss_weights), list(crit.loss_names)
        params = list(ref.parameters()) + list(crit.parameters())
        opt = RefLion(params, lr=1e-4, betas=(0.9, 0.99), weight_decay=0.1)
        ref.train()
        crit.train()
        got = _train(w, batches)
        want = []
        for x, y, r in batches:
            opt.zero_grad()
            total, _ = ref_loop.parallel_criterion(mods, weights, names, ref([x.cuda()]), [(y.cuda(),), (r.cuda(),)])
            total.backward()
            want.append(total.item())
            opt.step()
        torch.cuda.synchronize()
        sgd = _worker(lion=False, precision=Precision.FP32)
        _train(sgd, batches)
        theirs = [p.detach().float() for p in params]
        gap_ref = _gap(_weights(w), theirs, p0)
        gap_sgd = _gap(_weights(sgd), theirs, p0)
        print("gap to RefLion %.3e, SGD run to RefLion %.3e, last rows %r %r" % (gap_ref, gap_sgd, got[-1], want[-1]))
        assert gap_ref < 0.25 and gap_ref < 0.25 * gap_sgd, (gap_ref, gap_sgd)
        assert abs(got[-1] - want[-1]) < 0.1 * abs(want[0] - want[-1]), (got[-1], want[-1])
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def test_k12_lion_is_taken_and_resume_continues_bit_for_bit():
    batches = _batches(10)
    for master in (MasterWeights.FP32, MasterWeights.BF16):
        x = _worker(master=master)
        assert x.pipeline.fused_dw_update
        _train(x, batches[:5])
        assert x.pipeline.dw_updated, "no slot was updated inside its dW GEMM"
        saved = _weights(x)
        sd = x.optimizer.state_dict()
        assert set(sd["param_groups"][0]) >= {"lr", "betas", "weight_decay"}
        assert all(set(e) == {"exp_avg"} and e["exp_avg"].is_contiguous() for e in sd["state"].values())
        rows_x = _train(x, batches[5:], 5)
        y = _worker(master=master, seed=7)
        y.arena.load_master_from_params(list(zip(_params(y), saved)))
        y.optimizer.load_state_dict(sd)
        rows_y = _train(y, batches[5:], 5)
        assert rows_x == rows_y and torch.equal(x.arena.lp, y.arena.lp), master
        assert torch.equal(x.optimizer._state("exp_avg"), y.optimizer._state("exp_avg"))


def test_graph_replay_gives_the_eager_bytes():
    batches = _batches(8)
    eager, graphed = _worker(), _worker(graph=True)
    a, b = _train(eager, batches), _train(graphed, batches)
    assert graphed.graphed is not None and graphed.optimizer._dyn is not None
    assert a == b
    assert torch.equal(eager.arena.lp, graphed.arena.lp) and torch.equal(eager.arena.master, graphed.arena.master)


def test_state_is_four_bytes_per_arena_element_against_adamws_eight():
    lion, adamw = _worker(), _worker(lion=False, algo=OptAlgorithm.ADAM, adamw=True)
    _train(lion, _batches(1))
    _train(adamw, _batches(1))
    nbytes = lambda w: sum(v.numel() * v.element_size() for v in w.optimizer._vec.values())   # noqa: E731
    assert set(lion.optimizer._vec) == {"exp_avg"} and nbytes(lion) == 4 * lion.arena.numel
    assert nbytes(adamw) == 8 * adamw.arena.numel == 2 * nbytes(lion)


@pytest.mark.parametrize("combo", ["accumulation_clip", "fp8", "ema", "bf16_master", "graph"])
def test_solver_loop_in_combination(combo, tmp_path):
    ns = synthetic.api_namespace("frl_b200")
    t = ns.types
    torch.manual_seed(0)
    problem = synthetic.make_mlp_problem(ns, str(tmp_path), n_train=2048, width=512, n_classes=100, reg_dim=16,
                                         depth=3)
    run_opts = t.RunOpts(optim=t.OptimOpts(algo=t.OptAlgorithm.SGD, lr=1e-4, momentum=0.9, weightDecay=0.1,
                                           gradientClip=1.0 if combo == "accumulation_clip" else 0.0),
                         batchSize=256, nEpochs=2, numThreads=0, singleThreaded=True, numVisualizedSamples=0)
    kw = dict(precision=Precision.FP8 if combo == "fp8" else Precision.BF16,
              grad_accumulation=2 if combo == "accumulation_clip" else 1, ema_decay=0.9 if combo == "ema" else 0.0,
              master_weights=MasterWeights.BF16 if combo == "bf16_master" else MasterWeights.FP32,
              graph_step=combo == "graph")
    args = SolverWorkerArgs(run_opts=run_opts, problem=problem, save_dir=str(tmp_path), run_device=Device.GPU,
                            node_idx=0, node_count=1, rank=0, local_rank=0, world_size=1, group_name=None,
                            init_method="", lion=True, **kw)
    rows = [frac.performance[t.Split.TRAIN].losses for frac in Solver._run_solver_worker(args)]
    totals = [sum(float(v) for v in r.values()) for r in rows]
    assert all(np.isfinite(totals)) and totals[-1] < totals[0], totals


def test_channels_last_resnet_trains(tmp_path):
    ns = synthetic.api_namespace("frl_b200")
    t = ns.types
    torch.manual_seed(0)
    problem = synthetic.make_resnet_problem(ns, str(tmp_path), "resnet18", image=64, n_train=128)
    run_opts = t.RunOpts(optim=t.OptimOpts(algo=t.OptAlgorithm.SGD, lr=1e-4, momentum=0.9, weightDecay=0.1),
                         batchSize=32, nEpochs=2, numThreads=0, singleThreaded=True, numVisualizedSamples=0)
    args = SolverWorkerArgs(run_opts=run_opts, problem=problem, save_dir=str(tmp_path), run_device=Device.GPU,
                            node_idx=0, node_count=1, rank=0, local_rank=0, world_size=1, group_name=None,
                            init_method="", precision=Precision.BF16, channels_last=True, lion=True)
    rows = [frac.performance[t.Split.TRAIN].losses for frac in Solver._run_solver_worker(args)]
    totals = [sum(float(v) for v in r.values()) for r in rows]
    assert all(np.isfinite(totals)), totals


@pytest.mark.parametrize("master, kernels", [
    (MasterWeights.FP32, "frl_dw_gemm_lion, K12, for the trunk's weights, frl_lion / frl_lion_mt, K2 / K2-mt for "
                         "the rest"),
    (MasterWeights.BF16, "frl_dw_gemm_lion_sr, K12, for the trunk's weights, frl_lion_sr / frl_lion_mt_sr, K2-sr "
                         "for the rest")])
def test_info_line_names_lion_and_its_kernels(caplog, master, kernels):
    with caplog.at_level(logging.INFO):
        _worker(master=master)
    want = "optimizer lion, betas (0.9, 0.99), decoupled weight decay 0.1 (%s) |" % kernels
    assert any(want in r.getMessage() for r in caplog.records), [r.getMessage() for r in caplog.records][-5:]


def test_two_ranks_agree_and_match_one_gpu_at_the_global_batch():
    """tests/run_lion_mp.py: over gloo with both ranks on GPU 0 when only one GPU is visible (the K7
    arm reported as not run), over NCCL where two or more GPUs are visible."""
    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    backend = "nccl" if torch.cuda.device_count() >= 2 else "gloo"
    res = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nproc-per-node", "2",
                          os.path.join(repo, "tests", "run_lion_mp.py"), "--backend", backend],
                         capture_output=True, text=True, timeout=600, cwd=repo)
    print(res.stdout[-2000:])
    assert res.returncode == 0 and res.stdout.count("LION_MP_OK") == 2, res.stdout[-3000:] + res.stderr[-3000:]
    assert "LION_K7" in res.stdout
