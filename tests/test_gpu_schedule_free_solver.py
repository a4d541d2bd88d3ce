"""Schedule-Free AdamW / SGD through ``Solver.build_worker`` on the H100: the width-512 MLP against a
restatement autograd loop (FP32 tight, BF16 as a bounded per-parameter update gap), held-out losses at x
against the restatement's after ``eval()``, a bit-for-bit resume with fp32 and with bf16 master weights,
graph replay that follows an lr change, accumulation with clipping, FP8, bf16 master weights, two param
groups, a channels_last ResNet, and two ranks against one GPU (``tests/run_schedule_free_mp.py``)."""
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

import frl_b200  # noqa: F401
from frl_b200 import fused_optim, synthetic
from frl_b200.solver import Solver, SolverWorkerArgs
from frl_b200.types import Device, MasterWeights, OptAlgorithm, Precision, ScheduleFree, Split
from schedule_free_oracle import RefAdamWScheduleFree, RefSGDScheduleFree

pytestmark = pytest.mark.gpu
LR = {OptAlgorithm.ADAM: 1e-3, OptAlgorithm.SGD: 1e-2}


def _worker(algo=OptAlgorithm.ADAM, seed=0, precision=Precision.FP32, graph=False, master=MasterWeights.FP32,
            schedule_free=ScheduleFree(warmup_steps=3), **kw):
    ns = synthetic.api_namespace("frl_b200")
    t = ns.types
    save_dir = tempfile.mkdtemp(prefix="frl_b200_sf_")
    torch.manual_seed(seed)
    problem = synthetic.make_mlp_problem(ns, save_dir, n_train=8, width=512, n_classes=100, reg_dim=16, depth=3)
    run_opts = t.RunOpts(optim=t.OptimOpts(algo=algo, lr=LR[algo], momentum=0.9, weightDecay=0.1),
                         batchSize=256, nEpochs=1, numThreads=0, singleThreaded=True, numVisualizedSamples=0)
    args = SolverWorkerArgs(run_opts=run_opts, problem=problem, save_dir=save_dir, run_device=Device.GPU,
                            node_idx=0, node_count=1, rank=0, local_rank=0, world_size=1, group_name=None,
                            init_method="", precision=precision, graph_step=graph, master_weights=master,
                            schedule_free=schedule_free, **kw)
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


def _weights(worker):
    with worker.arena.exported(cpu=False):
        return [p.detach().float().clone() for p in _params(worker)]


def _gap(a, b, p0):
    """Largest over the parameters of ||a - b|| / ||b - p0||: how far apart two runs' updates are."""
    return max(((x - y).norm() / (y - q).norm().clamp_min(1e-30)).item() for x, y, q in zip(a, b, p0))


def _loss(model, crit, x, y, r):
    from oracle import ref_loop
    mods, weights, names = list(crit.loss_modules), list(crit.loss_weights), list(crit.loss_names)
    with torch.no_grad():
        total, _ = ref_loop.parallel_criterion(mods, weights, names, model([x.cuda()]), [(y.cuda(),), (r.cuda(),)])
    return float(total)


def _reference(worker, algo, batches):
    """The stock autograd loop with the restatement optimizer from ``worker``'s initial weights."""
    from oracle import ref_loop
    ns = synthetic.api_namespace("frl_b200")
    problem = synthetic.make_mlp_problem(ns, tempfile.mkdtemp(prefix="frl_b200_sf_ref_"), n_train=8, width=512,
                                         n_classes=100, reg_dim=16, depth=3)
    ref = problem.get_model().cuda()
    ref.load_state_dict(worker.model.state_dict())
    crit = problem.get_criterion().cuda()
    crit.load_state_dict(worker.criterion.state_dict())
    params = list(ref.parameters()) + list(crit.parameters())
    if algo == OptAlgorithm.ADAM:
        opt = RefAdamWScheduleFree(params, lr=LR[algo], weight_decay=0.1, warmup_steps=3)
    else:
        opt = RefSGDScheduleFree(params, lr=LR[algo], momentum=0.9, weight_decay=0.1, warmup_steps=3)
    ref.train()
    crit.train()
    mods, weights, names = list(crit.loss_modules), list(crit.loss_weights), list(crit.loss_names)
    rows = []
    for x, y, r in batches:
        opt.zero_grad()
        total, _ = ref_loop.parallel_criterion(mods, weights, names, ref([x.cuda()]), [(y.cuda(),), (r.cuda(),)])
        total.backward()
        rows.append(total.item())
        opt.step()
    torch.cuda.synchronize()
    return ref, crit, opt, params, rows


@pytest.mark.parametrize("algo", [OptAlgorithm.ADAM, OptAlgorithm.SGD])
def test_fp32_mlp_and_its_held_out_loss_at_x_follow_the_restatement(algo):
    """Precision.FP32, no TF32, width-512 MLP, batch 256, 20 steps, warm-up 3: the Solver against stock
    autograd + the restatement.  They differ only in rounding order: the loss rows agree to the tolerance of
    the FP32 SGD / Adam parity (tests/test_gpu_mlp_parity.py: rtol 1e-5 / 1e-3; Adam's normalised step
    amplifies the reordering), and so does the loss of a held-out batch at x (the Solver inside
    ``swapped()``, the restatement after ``eval()``)."""
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        batches = _batches(21)
        train, held = batches[:20], batches[20]
        w = _worker(algo)
        assert isinstance(w.optimizer, fused_optim.FusedScheduleFree) and not w.pipeline.fused_dw_update
        p0 = _weights(w)
        ref, crit, opt, params, want_rows = _reference(w, algo, train)
        rows = _train(w, train)
        rtol = 1e-3 if algo == OptAlgorithm.ADAM else 1e-5
        print("update gap to the restatement %.3e" % _gap(_weights(w), [p.detach().float() for p in params], p0))
        np.testing.assert_allclose(rows, want_rows, rtol=rtol, atol=0)
        assert w.optimizer.hyper["k"] == opt.param_groups[0]["k"] == 20
        w.model.eval()
        w.criterion.eval()
        ref.eval()
        crit.eval()
        at_y = _loss(w.model, w.criterion, *held)
        with w.optimizer.swapped():
            at_x = _loss(w.model, w.criterion, *held)
        opt.eval()
        want = _loss(ref, crit, *held)
        print("held-out loss at x %.6f, restatement %.6f, at y %.6f" % (at_x, want, at_y))
        assert at_x == pytest.approx(want, rel=rtol) and at_x != at_y
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def test_bf16_mlp_stays_within_a_bounded_gap_of_the_restatement():
    """Precision.BF16: bf16 forward / backward and gradients, so the runs drift apart (in FP32 the AdamW
    restatement's reordering alone leaves a 0.20 update gap after 20 steps).  Measured on an H100 80GB HBM3
    (700 W, seed 0, this test): the largest per-parameter update gap to the restatement is 0.43 of the
    update, a plain AdamW run's 1.43.  Bound: 0.6, and under half the plain AdamW gap."""
    batches = _batches(20)
    w = _worker(precision=Precision.BF16)
    p0 = _weights(w)
    params = _reference(w, OptAlgorithm.ADAM, batches)[3]
    _train(w, batches)
    plain = _worker(precision=Precision.BF16, schedule_free=None, adamw=True)
    _train(plain, batches)
    theirs = [p.detach().float() for p in params]
    gap, gap_plain = _gap(_weights(w), theirs, p0), _gap(_weights(plain), theirs, p0)
    print("bf16 update gap to the restatement %.3e, plain AdamW's %.3e" % (gap, gap_plain))
    assert gap < 0.6 and gap < 0.5 * gap_plain, (gap, gap_plain)


@pytest.mark.parametrize("master", [MasterWeights.FP32, MasterWeights.BF16])
@pytest.mark.parametrize("algo", [OptAlgorithm.ADAM, OptAlgorithm.SGD])
def test_resume_continues_bit_for_bit(master, algo):
    batches = _batches(10)
    x = _worker(algo, precision=Precision.BF16, master=master)
    _train(x, batches[:5])
    saved = _weights(x)
    sd = x.optimizer.state_dict()
    assert sd["param_groups"][0]["k"] == 5 and sd["param_groups"][0]["train_mode"] is True
    assert all(e["z"].is_contiguous() for e in sd["state"].values())
    rows_x = _train(x, batches[5:], 5)
    y = _worker(algo, precision=Precision.BF16, master=master, seed=7)
    y.arena.load_master_from_params(list(zip(_params(y), saved)))
    y.optimizer.load_state_dict(sd)
    assert y.optimizer._steps == 5
    rows_y = _train(y, batches[5:], 5)
    assert rows_x == rows_y and torch.equal(x.arena.lp, y.arena.lp), master
    assert torch.equal(x.arena.master, y.arena.master)
    for name in x.optimizer._vec:
        assert torch.equal(x.optimizer._state(name), y.optimizer._state(name)), name


@pytest.mark.parametrize("groups", [False, True])
def test_graph_replay_follows_an_lr_change_and_gives_the_eager_bytes(groups):
    batches = _batches(10)
    eager = _worker(precision=Precision.BF16, no_decay_1d=groups)
    graphed = _worker(precision=Precision.BF16, graph=True, no_decay_1d=groups)
    assert graphed.optimizer.grouped == groups
    a, b = _train(eager, batches[:5]), _train(graphed, batches[:5])
    for w in (eager, graphed):                   # what the per-epoch scheduler does
        for g in w.optimizer.param_groups:
            g["lr"] *= 0.1
    a += _train(eager, batches[5:], 5)
    b += _train(graphed, batches[5:], 5)
    assert graphed.graphed is not None and graphed.optimizer._dyn is not None
    assert a == b
    assert torch.equal(eager.arena.lp, graphed.arena.lp) and torch.equal(eager.arena.master, graphed.arena.master)
    assert torch.equal(eager.optimizer._state("z"), graphed.optimizer._state("z"))
    assert [g["lr_max"] for g in eager.optimizer.param_groups] == [g["lr_max"] for g in graphed.optimizer.param_groups]


@pytest.mark.parametrize("combo", ["accumulation_clip", "fp8", "bf16_master", "graph", "groups"])
def test_solver_loop_in_combination(combo, tmp_path):
    ns = synthetic.api_namespace("frl_b200")
    t = ns.types
    torch.manual_seed(0)
    problem = synthetic.make_mlp_problem(ns, str(tmp_path), n_train=2048, width=512, n_classes=100, reg_dim=16,
                                         depth=3)
    run_opts = t.RunOpts(optim=t.OptimOpts(algo=t.OptAlgorithm.ADAM, lr=1e-3, weightDecay=0.1,
                                           gradientClip=1.0 if combo == "accumulation_clip" else 0.0),
                         batchSize=256, nEpochs=2, numThreads=0, singleThreaded=True, numVisualizedSamples=0)
    kw = dict(precision=Precision.FP8 if combo == "fp8" else Precision.BF16,
              grad_accumulation=2 if combo == "accumulation_clip" else 1,
              master_weights=MasterWeights.BF16 if combo == "bf16_master" else MasterWeights.FP32,
              graph_step=combo == "graph", no_decay_1d=combo == "groups")
    args = SolverWorkerArgs(run_opts=run_opts, problem=problem, save_dir=str(tmp_path), run_device=Device.GPU,
                            node_idx=0, node_count=1, rank=0, local_rank=0, world_size=1, group_name=None,
                            init_method="", schedule_free=ScheduleFree(warmup_steps=2), **kw)
    rows = [frac.performance[t.Split.TRAIN].losses for frac in Solver._run_solver_worker(args)]
    totals = [sum(float(v) for v in r.values()) for r in rows]
    assert all(np.isfinite(totals)) and totals[-1] < totals[0], totals


def test_accumulation_counts_updates():
    batches = _batches(6)
    w = _worker(precision=Precision.BF16, grad_accumulation=2)
    for i, (x, y, r) in enumerate(batches):
        w.pipeline.set_microbatch(first=i % 2 == 0, closes=i % 2 == 1)
        w._pass_one_minibatch(i, Split.TRAIN, [x.cuda()], [(y.cuda(),), (r.cuda(),)])
    torch.cuda.synchronize()
    assert w.optimizer.hyper["k"] == w.optimizer._steps == 3


def test_channels_last_resnet_trains_and_evaluates_at_x(tmp_path):
    ns = synthetic.api_namespace("frl_b200")
    t = ns.types
    torch.manual_seed(0)
    problem = synthetic.make_resnet_problem(ns, str(tmp_path), "resnet18", image=64, n_train=128)
    run_opts = t.RunOpts(optim=t.OptimOpts(algo=t.OptAlgorithm.SGD, lr=1e-2, momentum=0.9, weightDecay=1e-4),
                         batchSize=32, nEpochs=2, numThreads=0, singleThreaded=True, numVisualizedSamples=0)
    args = SolverWorkerArgs(run_opts=run_opts, problem=problem, save_dir=str(tmp_path), run_device=Device.GPU,
                            node_idx=0, node_count=1, rank=0, local_rank=0, world_size=1, group_name=None,
                            init_method="", precision=Precision.BF16, channels_last=True,
                            schedule_free=ScheduleFree())
    rows = [frac.performance for frac in Solver._run_solver_worker(args)]
    totals = [sum(float(v) for v in p[s].losses.values()) for p in rows for s in p]
    assert all(np.isfinite(totals)), totals


def test_two_ranks_agree_and_match_one_gpu_at_the_global_batch():
    """tests/run_schedule_free_mp.py: over gloo with both ranks on GPU 0 when only one GPU is visible,
    over NCCL where two or more GPUs are visible."""
    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    backend = "nccl" if torch.cuda.device_count() >= 2 else "gloo"
    res = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nproc-per-node", "2",
                          os.path.join(repo, "tests", "run_schedule_free_mp.py"), "--backend", backend],
                         capture_output=True, text=True, timeout=600, cwd=repo)
    print(res.stdout[-2000:])
    assert res.returncode == 0 and res.stdout.count("SF_MP_OK") == 2, res.stdout[-3000:] + res.stderr[-3000:]
