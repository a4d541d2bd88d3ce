"""K2-lw (LARS, LAMB) on the H100: the kernels against the numpy restatement, determinism, NaN
containment, and the headline MLP through ``Solver.build_worker`` against stock torch running the
per-parameter oracle (``tests/layerwise_oracle.py``)."""
import tempfile

import numpy as np
import pytest
import torch
import torch.nn as nn

import frl_b200  # noqa: F401
from frl_b200 import fused_optim, synthetic
from frl_b200.arena import ParamArena
from frl_b200.multi_tensor import GradSegTable
from frl_b200.solver import Solver, SolverWorkerArgs
from frl_b200.types import Device, LayerAdaptation, OptAlgorithm, OptimOpts, Precision
from layerwise_oracle import LayerwiseTorch, lamb_step, lars_step

pytestmark = pytest.mark.gpu

# smaller than a tile, numel % 4 != 0, several tiles with a ragged end, 1-D, and one 4096 x 4096
SHAPES = [(3,), (5, 7), (13,), (33, 17), (300, 70), (4096, 4096), (1000,), (2, 3, 3, 3)]


def _setup(precision, seed=0):
    torch.manual_seed(seed)
    params = [nn.Parameter(torch.randn(*s, device="cuda") * 0.1) for s in SHAPES[:-1]]
    crit = [nn.Parameter(torch.randn(*SHAPES[-1], device="cuda") * 0.1)]   # criterion parameter: never clipped
    arena = ParamArena(params, crit, device="cuda", precision=precision)
    g = torch.Generator().manual_seed(seed + 1)
    grads, table = [], GradSegTable(arena.slots, arena.device)
    table.grads = []                                       # the tensors the table points at
    for i, s in enumerate(arena.slots):
        v = torch.randn(s.numel, generator=g) * 10.0 ** (i % 3 - 1)
        if i % 2 == 0:                                     # in the arena
            dst = arena.grad[s.offset:s.end]
            dst.copy_(v.to(dst.dtype))
            grads.append(dst.float().cpu().numpy())
            table.point(s, dst.data_ptr(), dst.dtype)
            table.grads.append(dst)
        else:                                              # outside the arena (autograd-allocated)
            dt = torch.bfloat16 if i % 4 == 1 else torch.float32
            ext = v.to(dt).cuda()
            grads.append(ext.float().cpu().numpy())
            table.point(s, ext.data_ptr(), dt)
            table.grads.append(ext)
    table.upload()
    return arena, table, grads


def _state(opt, name, s):
    return opt._vec[name][s.offset:s.end].cpu().numpy()


@pytest.mark.parametrize("dyn", [False, True])
@pytest.mark.parametrize("precision", [Precision.FP32, Precision.BF16])
@pytest.mark.parametrize("mode", ["lars", "lamb"])
def test_kernels_match_the_restatement(mode, precision, dyn):
    arena, table, grads = _setup(precision)
    if mode == "lars":
        opt = fused_optim.FusedLars(arena, lr=0.1, momentum=0.9, weight_decay=1e-2)
    else:
        opt = fused_optim.FusedLamb(arena, lr=0.01, weight_decay=1e-2, eps=1e-6)
    if dyn:
        opt.enable_dynamic_scalars()
    coef = torch.tensor([0.75], device="cuda")
    w = [arena.master[s.offset:s.end].cpu().numpy().copy() for s in arena.slots]
    st = {k: [np.zeros(s.numel, np.float32) for s in arena.slots] for k in ("buf", "m", "v")}
    for step in (1, 2, 3):
        opt.begin_step()
        if dyn:
            # the launch's by-value scalars are wrong on purpose: only the device block is right
            lr, opt.hyper["lr"] = opt.hyper["lr"], 123.0
            opt._steps += 7 if mode == "lamb" else 0          # LAMB's by-value bias corrections
            opt.apply_table(table, grad_scale=0.5, clip_coef_dev=coef)
            opt.hyper["lr"] = lr
            opt._steps -= 7 if mode == "lamb" else 0
        else:
            opt.apply_table(table, grad_scale=0.5, clip_coef_dev=coef)
        opt.end_step()
        ratios = opt.last_ratios(table).cpu().numpy()
        for i, s in enumerate(arena.slots):
            gs = 0.5 * (0.75 if s.is_model else 1.0)
            adapted = len(s.shape) >= 2
            if mode == "lars":
                w[i], st["buf"][i], r = lars_step(w[i], grads[i], st["buf"][i], lr=0.1, mu=0.9, wd=1e-2,
                                                  adapted=adapted, first_step=step == 1, grad_scale=gs)
                np.testing.assert_allclose(_state(opt, "momentum_buffer", s), st["buf"][i], rtol=1e-5, atol=1e-9)
            else:
                w[i], st["m"][i], st["v"][i], r = lamb_step(w[i], grads[i], st["m"][i], st["v"][i], lr=0.01,
                                                            beta1=0.9, beta2=0.999, eps=1e-6, wd=1e-2, step=step,
                                                            adapted=adapted, grad_scale=gs)
                np.testing.assert_allclose(_state(opt, "exp_avg", s), st["m"][i], rtol=1e-5, atol=1e-9)
                np.testing.assert_allclose(_state(opt, "exp_avg_sq", s), st["v"][i], rtol=1e-5, atol=1e-12)
            assert abs(ratios[i] - r) <= 1e-5 * abs(r), (step, s.shape, ratios[i], r)
            got = arena.master[s.offset:s.end].cpu().numpy()
            np.testing.assert_allclose(got, w[i], rtol=1e-5, atol=1e-7)
            w[i] = got.copy()          # compare each step from the kernel's own weights
            if arena.lp is not None and s.is_model:
                assert torch.equal(arena.lp[s.offset:s.end].cpu(), torch.from_numpy(got).to(torch.bfloat16))


@pytest.mark.parametrize("mode", ["lars", "lamb"])
def test_two_launches_are_bitwise_equal_and_nan_stays_in_its_tensor(mode):
    outs = []
    for rep in range(3):
        arena, table, _ = _setup(Precision.BF16)
        opt = (fused_optim.FusedLars(arena, lr=0.1, momentum=0.9, weight_decay=1e-2) if mode == "lars"
               else fused_optim.FusedLamb(arena, lr=0.01, weight_decay=1e-2))
        if rep == 2:                                       # NaN in the 4096 x 4096 gradient
            table.grads[5][12345] = float("nan")
        for _ in range(2):
            opt.begin_step(); opt.apply_table(table); opt.end_step()
        outs.append((arena.master.clone(), opt.last_ratios(table).clone(), arena.lp.clone()))
    (p0, r0, l0), (p1, r1, l1), (p2, _, _) = outs
    assert torch.equal(p0, p1) and torch.equal(r0, r1) and torch.equal(l0, l1)
    bad = arena.slots[5]
    for s in arena.slots:
        finite = bool(torch.isfinite(p2[s.offset:s.end]).all())
        assert finite == (s is not bad), s.shape


# ---- end to end: the headline MLP ---------------------------------------------------------------

WIDTH, N_CLASSES, REG_DIM, DEPTH, BATCH, STEPS = 4096, 1000, 64, 3, 64, 6
LR = {"lars": 0.5, "lamb": 1e-3}


def _opts(mode):
    if mode == "lars":
        return OptimOpts(algo=OptAlgorithm.SGD, lr=LR[mode], weightDecay=1e-4)
    return OptimOpts(algo=OptAlgorithm.ADAM, lr=LR[mode], weightDecay=1e-2)


def _batches():
    g = torch.Generator().manual_seed(1234)
    return [(torch.randn(BATCH, WIDTH, generator=g), torch.randint(0, N_CLASSES, (BATCH,), generator=g),
             torch.randn(BATCH, REG_DIM, generator=g)) for _ in range(STEPS)]


_ORACLE = {}


def _oracle(mode):
    """Stock fp32 torch on the GPU (TF32 off) with the per-parameter LARS / LAMB oracle."""
    if mode in _ORACLE:
        return _ORACLE[mode]
    from oracle import ref_loop
    torch.backends.cuda.matmul.allow_tf32 = False
    ns = synthetic.api_namespace("frl_b200")
    torch.manual_seed(0)
    problem = synthetic.make_mlp_problem(ns, "/tmp/unused", n_train=8, width=WIDTH, n_classes=N_CLASSES,
                                         reg_dim=REG_DIM, depth=DEPTH)
    model, crit = problem.get_model().cuda(), problem.get_criterion()
    mods, weights, names = list(crit.loss_modules), list(crit.loss_weights), list(crit.loss_names)
    o = _opts(mode)
    opt = LayerwiseTorch(model.parameters(), mode, lr=o.lr, momentum=o.momentum, weight_decay=o.weightDecay,
                         eps=o.epsilon)
    rows = []
    for x, y, r in _batches():
        _, total, sub = ref_loop.reference_minibatch(
            model, lambda out, t: ref_loop.parallel_criterion(mods, weights, names, out, t), opt,
            list(model.parameters()), 0.0, [x.cuda()], [(y.cuda(),), (r.cuda(),)])
        rows.append([total.item()] + [sub[n].item() for n in names])
    _ORACLE[mode] = np.asarray(rows, dtype=np.float64)
    return _ORACLE[mode]


def _run(mode, precision, graph):
    ns = synthetic.api_namespace("frl_b200")
    t = ns.types
    save_dir = tempfile.mkdtemp(prefix="frl_b200_lw_")
    torch.manual_seed(0)
    problem = synthetic.make_mlp_problem(ns, save_dir, n_train=8, width=WIDTH, n_classes=N_CLASSES,
                                         reg_dim=REG_DIM, depth=DEPTH)
    run_opts = t.RunOpts(optim=_opts(mode), batchSize=BATCH, nEpochs=1, numThreads=0, singleThreaded=True,
                         numVisualizedSamples=0)
    args = SolverWorkerArgs(run_opts=run_opts, problem=problem, save_dir=save_dir, run_device=Device.GPU,
                            node_idx=0, node_count=1, rank=0, local_rank=0, world_size=1, group_name=None,
                            init_method="", precision=precision, graph_step=graph,
                            layer_adaptation=LayerAdaptation(mode))
    worker, _, _ = Solver.build_worker(args)
    worker.model.train()
    worker.criterion.train()
    assert type(worker.optimizer) is (fused_optim.FusedLars if mode == "lars" else fused_optim.FusedLamb)
    assert not worker.pipeline.eager
    rows = []
    for i, (x, y, r) in enumerate(_batches()):
        _, total, sub, _ = worker._pass_one_minibatch(i, t.Split.TRAIN, [x.cuda()], [(y.cuda(),), (r.cuda(),)])
        rows.append([float(total.detach())] + [float(sub[n].detach()) for n in worker.criterion.loss_names])
        del total, sub
    torch.cuda.synchronize()
    if graph:
        assert worker.graphed is not None and len(worker.graphed._graphs) == 1
    return np.asarray(rows, dtype=np.float64)


@pytest.mark.parametrize("mode", ["lars", "lamb"])
def test_headline_mlp_matches_stock_torch_and_graph_replay_is_exact(mode):
    want = _oracle(mode)
    eager = _run(mode, Precision.FP32, False)
    graphed = _run(mode, Precision.FP32, True)
    print(mode, "losses (total, per task) per step:\n", eager, "\noracle:\n", want)
    np.testing.assert_allclose(eager[:1], want[:1], rtol=1e-5, atol=0)
    np.testing.assert_allclose(eager[1:], want[1:], rtol=1e-3, atol=0)
    assert np.array_equal(graphed, eager)
    assert not np.array_equal(eager[0], eager[-1])            # the model actually trained


@pytest.mark.parametrize("mode", ["lars", "lamb"])
def test_headline_mlp_bf16_within_the_bf16_parity_bounds(mode):
    want = _oracle(mode)
    rows = _run(mode, Precision.BF16, True)
    np.testing.assert_allclose(rows[:1], want[:1], rtol=1e-2, atol=0)
    # the existing bf16 parity bounds: 1e-2 on the SGD rule, 3e-2 on the Adam rule
    np.testing.assert_allclose(rows[1:], want[1:], rtol=1e-2 if mode == "lars" else 3e-2, atol=0)


@pytest.mark.parametrize("mode", ["lars", "lamb"])
def test_checkpoint_resumes_bit_identically_and_loads_under_torch(mode):
    def fresh():
        arena, table, _ = _setup(Precision.BF16)
        opt = (fused_optim.FusedLars(arena, lr=0.1, momentum=0.9, weight_decay=1e-2) if mode == "lars"
               else fused_optim.FusedLamb(arena, lr=0.01, weight_decay=1e-2))
        return arena, table, opt

    a, ta, oa = fresh()
    for _ in range(4):
        oa.begin_step(); oa.apply_table(ta); oa.end_step()
    b, tb, ob = fresh()
    for _ in range(2):
        ob.begin_step(); ob.apply_table(tb); ob.end_step()
    sd = ob.state_dict()
    master = b.master.clone()
    c, tc, oc = fresh()
    c.master.copy_(master)
    c.refresh_shadow()
    oc.load_state_dict(sd)
    for _ in range(2):
        oc.begin_step(); oc.apply_table(tc); oc.end_step()
    assert torch.equal(c.master, a.master) and torch.equal(c.lp, a.lp)
    assert all(torch.equal(oc._vec[k], oa._vec[k]) for k in oa._vec)
    params = [nn.Parameter(torch.zeros(s.shape, device="cuda")) for s in sorted(b.slots, key=lambda s: s.index)]
    stock = torch.optim.SGD(params, lr=0.1, momentum=0.9) if mode == "lars" else torch.optim.Adam(params, lr=0.01)
    stock.load_state_dict(sd)
    name = "momentum_buffer" if mode == "lars" else "exp_avg"
    s5 = sorted(b.slots, key=lambda s: s.index)[5]
    assert torch.equal(stock.state_dict()["state"][5][name].flatten(), ob._vec[name][s5.offset:s5.end])


@pytest.mark.parametrize("mode", ["lars", "lamb"])
def test_parameter_without_gradient_is_left_untouched(mode):
    """One GPU, real kernels: a step in which only the first layer gets a gradient updates that
    layer through a table of the slots that did (as torch.optim skips the others), and leaves the
    other slots' weights and state bit for bit as they were."""
    from frl_b200 import grad_sync

    def net():
        torch.manual_seed(3)
        return nn.Sequential(nn.Linear(64, 48), nn.ReLU(), nn.Linear(48, 40), nn.ReLU(), nn.Linear(40, 8)).cuda()

    mine, ref = net(), net()
    arena = ParamArena(mine.parameters(), device="cuda")
    o = _opts(mode)
    opt = fused_optim.create_fused_optimizer(arena, o, LayerAdaptation(mode))
    pipe = grad_sync.GradBucketPipeline(arena, opt)
    ref_opt = LayerwiseTorch(ref.parameters(), mode, lr=o.lr, momentum=o.momentum, weight_decay=o.weightDecay,
                             eps=o.epsilon)
    x = torch.randn(32, 64, device="cuda")
    pipe.begin_step(); mine(x).square().mean().backward(); pipe.finish_step()
    ref_opt.zero_grad(); ref(x).square().mean().backward(); ref_opt.step()
    torch.cuda.synchronize()
    before = {k: v.clone() for k, v in opt._vec.items()}
    rest = [p.detach().clone() for p in list(mine.parameters())[2:]]
    pipe.begin_step(); mine[0](x).square().mean().backward(); pipe.finish_step()       # layer 0 only
    ref_opt.zero_grad(); ref[0](x).square().mean().backward(); ref_opt.step()
    torch.cuda.synchronize()
    for a, b in zip(mine.parameters(), ref.parameters()):
        torch.testing.assert_close(a.detach(), b.detach(), rtol=1e-5, atol=1e-7)
    for a, b in zip(list(mine.parameters())[2:], rest):
        assert torch.equal(a.detach(), b)
    s = arena.slot_of(mine[2].weight)
    for k, v in opt._vec.items():
        assert torch.equal(v[s.offset:], before[k][s.offset:]), k


def test_resnet_problem_under_lars_matches_stock_torch():
    """A small ResNet Problem, LARS, 3 steps, one GPU: convolution gradients (allocated by cuDNN) are
    read in place through the segment table, BatchNorm parameters keep ratio 1, and the losses follow
    stock torch running the per-parameter oracle on the same GPU."""
    from oracle import ref_loop
    ns = synthetic.api_namespace("frl_b200")
    t = ns.types
    batch, steps = 16, 3
    old = (torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic,
           torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic = False, True
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    g = torch.Generator().manual_seed(7)
    data = [(torch.randn(batch, 3, 32, 32, generator=g), torch.randint(0, 1000, (batch,), generator=g))
            for _ in range(steps)]
    o = OptimOpts(algo=OptAlgorithm.SGD, lr=0.5, weightDecay=1e-4)
    try:
        torch.manual_seed(0)
        ref_problem = synthetic.make_resnet_problem(ns, "/tmp/unused", image=32, n_train=2)
        ref_model, crit = ref_problem.get_model().cuda(), ref_problem.get_criterion()
        mods, weights, names = list(crit.loss_modules), list(crit.loss_weights), list(crit.loss_names)
        ref_opt = LayerwiseTorch(ref_model.parameters(), "lars", lr=o.lr, momentum=o.momentum,
                                 weight_decay=o.weightDecay)
        ref_model.train()
        want = []
        for x, y in data:
            _, total, _ = ref_loop.reference_minibatch(
                ref_model, lambda out, tg: ref_loop.parallel_criterion(mods, weights, names, out, tg), ref_opt,
                list(ref_model.parameters()), 0.0, [x.cuda()], [(y.cuda(),)])
            want.append(total.item())
        save_dir = tempfile.mkdtemp(prefix="frl_b200_lw_resnet_")
        torch.manual_seed(0)
        problem = synthetic.make_resnet_problem(ns, save_dir, image=32, n_train=2)
        run_opts = t.RunOpts(optim=o, batchSize=batch, nEpochs=1, numThreads=0, singleThreaded=True,
                             numVisualizedSamples=0)
        args = SolverWorkerArgs(run_opts=run_opts, problem=problem, save_dir=save_dir, run_device=Device.GPU,
                                node_idx=0, node_count=1, rank=0, local_rank=0, world_size=1, group_name=None,
                                init_method="", precision=Precision.FP32, graph_step=False,
                                layer_adaptation=LayerAdaptation.LARS)
        worker, _, _ = Solver.build_worker(args)
        torch.backends.cudnn.benchmark = False
        worker.model.train()
        worker.criterion.train()
        got, in_place = [], None
        for i, (x, y) in enumerate(data):
            _, total, _, _ = worker._pass_one_minibatch(i, t.Split.TRAIN, [x.cuda()], [(y.cuda(),)])
            got.append(float(total.detach()))
            del total
            if in_place is None:       # where the update read each gradient in the first step
                table = worker.pipeline.tables.whole()
                lo = worker.arena.grad.data_ptr()
                hi = lo + worker.arena.grad.numel() * worker.arena.grad.element_size()
                in_place = {s.index: not (lo <= table._segs[k].g < hi) for k, s in enumerate(table.slots)}
        torch.cuda.synchronize()
    finally:
        (torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic,
         torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32) = old
    model = worker.model
    convs = [m for m in model.modules() if isinstance(m, nn.Conv2d)]
    bns = [m for m in model.modules() if isinstance(m, nn.BatchNorm2d)]
    slot = worker.arena.slot_of
    assert convs and bns and all(in_place[slot(m.weight).index] for m in convs)
    ratios = worker.optimizer.last_ratios(table).cpu()
    row = {s.index: k for k, s in enumerate(table.slots)}
    assert all(float(ratios[row[slot(m.weight).index]]) != 1.0 for m in convs)
    assert all(float(ratios[row[slot(p).index]]) == 1.0 for m in bns for p in (m.weight, m.bias))
    print("resnet lars losses", got, "oracle", want)
    np.testing.assert_allclose(got[:1], want[:1], rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(got[1:], want[1:], rtol=1e-3, atol=1e-5)


def test_two_gpus_match_one_gpu_at_double_the_batch():
    """>= 2 GPUs only: NCCL all-reduce per bucket, then one K2-lw update over the all-reduced arena,
    against one GPU at the global batch with the same kernels (tests/run_layerwise_mp.py)."""
    import os
    import subprocess
    import sys
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    script = os.path.join(os.path.dirname(__file__), "run_layerwise_mp.py")
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                          "--master-addr", "127.0.0.1", "--master-port", "29541", script],
                         capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
    assert out.stdout.count("LAYERWISE_MP_OK") == 2
