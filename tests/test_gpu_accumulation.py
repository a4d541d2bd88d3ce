"""Gradient accumulation on the H100: K10 (``frl_grad_accumulate_mt``) against numpy, and whole runs
through ``LocalSolver.solve`` with k microbatches per update against one batch of their rows."""
import collections
import logging
import os
import random
import shutil
import tempfile

import numpy as np
import pytest
import torch

import frl_b200  # noqa: F401
from frl_b200 import _native, synthetic
from frl_b200.device_loader import DeviceBatchLoader
from frl_b200.grad_sync import accumulation_plan
from frl_b200.local_solver import LocalSolver
from frl_b200.multi_tensor import GradSegTable
from frl_b200.solver import Solver, SolverWorkerArgs
from frl_b200.types import Device, LayerAdaptation, OptAlgorithm, OptimOpts, Precision, Split

pytestmark = pytest.mark.gpu

# ---- K10 against numpy -------------------------------------------------------------------------

Slot = collections.namedtuple("Slot", "index offset numel end")
SENTINEL = -7.25
# (numel, where the gradient lies): odd tails, a zero-length segment, NULL segments, several tiles
SPECS = [(3, "arena_bf16"), (35, "f32"), (0, "f32"), (13, "null"), (561, "bf16"), (20483, "arena_bf16"),
         (70001, "f32"), (1, "null"), (9, "arena_f32"), (4096 * 3 + 5, "bf16")]


def _mixed_table(seed=0):
    slots, off = [], 0
    for i, (n, _) in enumerate(SPECS):
        off += 8                                           # a gap before every segment
        slots.append(Slot(i, off, n, off + n))
        off += (n + 7) // 8 * 8
    total = off + 8
    g = torch.Generator().manual_seed(seed)
    arena_bf16 = torch.zeros(total, dtype=torch.bfloat16, device="cuda")
    arena_f32 = torch.zeros(total, dtype=torch.float32, device="cuda")
    table = GradSegTable(slots, torch.device("cuda"))
    keep, grads = [], []
    for s, (n, where) in zip(slots, SPECS):
        v = torch.randn(n, generator=g) * 3
        if where == "null":
            table.point(s, 0, torch.float32)
            grads.append(None)
            continue
        if where.startswith("arena"):
            buf = arena_bf16 if where == "arena_bf16" else arena_f32
            t = buf[s.offset:s.end]
            t.copy_(v.to(t.dtype))
        else:
            t = v.to(torch.bfloat16 if where == "bf16" else torch.float32).cuda()
        keep.append(t)
        table.point(s, t.data_ptr() if n else 0, t.dtype)
        grads.append(t.float().cpu().numpy())
    table.upload()
    table.keep = keep + [arena_bf16, arena_f32]
    return table, slots, grads, total


def _expect(acc, slots, grads, w, first):
    """float64 value of every element after one pass, and the exact fp32 result where it is exact."""
    out = acc.astype(np.float64)
    for s, g in zip(slots, grads):
        base = np.zeros(s.numel) if first else acc[s.offset:s.end].astype(np.float64)
        if g is None:
            out[s.offset:s.end] = base
        else:
            out[s.offset:s.end] = np.float64(np.float32(w)) * g.astype(np.float64) + base
    return out


@pytest.mark.parametrize("w", [1.0, 0.5, 0.37])
def test_k10_matches_numpy(w):
    table, slots, grads, total = _mixed_table()
    acc = torch.full((total,), SENTINEL, dtype=torch.float32, device="cuda")
    before = _native.launch_count()
    for p, first in enumerate((True, False, False)):
        host = acc.cpu().numpy()
        want = _expect(host, slots, grads, w, first)
        _native.grad_accumulate_mt(acc, table, w=w, first=first)
        got = acc.cpu().numpy()
        if w in (1.0, 0.5):                    # w * g is exact: fmaf == one rounding of the sum
            assert np.array_equal(got, want.astype(np.float32)), p
        else:
            ulp = np.spacing(np.abs(got).astype(np.float32)).astype(np.float64)
            assert np.all(np.abs(got.astype(np.float64) - want) <= ulp), p
        inside = np.zeros(total, bool)
        for s in slots:
            inside[s.offset:s.end] = True
        assert np.all(got[~inside] == SENTINEL)                 # gaps and padding untouched
        for s, g in zip(slots, grads):
            if g is None:
                assert np.all(got[s.offset:s.end] == (0.0 if first else host[s.offset:s.end]))
    assert _native.launch_count() - before == 3


def test_k10_dyn_overrides_and_graph_replay_equals_eager():
    table, slots, grads, total = _mixed_table(1)
    positions = [(1.0, True), (1.0, False), (0.5, False), (0.37, True), (0.25, False)]
    eager = torch.full((total,), SENTINEL, dtype=torch.float32, device="cuda")
    via_dyn = eager.clone()
    dyn = torch.zeros(2, dtype=torch.float32, device="cuda")
    for w, first in positions:
        _native.grad_accumulate_mt(eager, table, w=w, first=first)
        dyn.copy_(torch.tensor([w, 1.0 if first else 0.0]))
        _native.grad_accumulate_mt(via_dyn, table, w=123.0, first=not first, dyn=dyn)   # by-value args ignored
        assert torch.equal(eager, via_dyn)
    replayed = torch.full((total,), SENTINEL, dtype=torch.float32, device="cuda")
    graph_dyn = torch.zeros(2, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        _native.grad_accumulate_mt(replayed, table, dyn=graph_dyn)
    replayed.fill_(SENTINEL)
    for w, first in positions:
        graph_dyn.copy_(torch.tensor([w, 1.0 if first else 0.0]))
        graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(replayed, eager)


# ---- end to end through LocalSolver.solve --------------------------------------------------------

SEED = 11
N_TRAIN = 600                  # batch 16: 38 microbatches, the last of 8 rows -> last group 16 + 8 = 24


def _opts(kind):
    clip = 0.05 if kind.endswith("_clip") else 0.0
    if kind.startswith(("sgd", "lars")):
        return OptimOpts(algo=OptAlgorithm.SGD, lr=0.05, momentum=0.9, weightDecay=1e-4, gradientClip=clip)
    return OptimOpts(algo=OptAlgorithm.ADAM, lr=1e-3, weightDecay=1e-4, gradientClip=clip)


def _solve(kind, batch, k, *, precision=Precision.FP32, graph=False, n_epochs=1, problem_fn=None, save_dir=None,
           **solve_kw):
    ns = synthetic.api_namespace("frl_b200")
    save_dir = save_dir or tempfile.mkdtemp(prefix="frl_b200_accum_")
    torch.manual_seed(SEED)
    if problem_fn is None:
        problem = synthetic.make_mlp_problem(ns, save_dir, n_train=N_TRAIN, n_test=0, width=128, n_classes=10,
                                             reg_dim=8, depth=2)
    else:
        problem = problem_fn(ns, save_dir)
    run_opts = ns.types.RunOpts(optim=_opts(kind), batchSize=batch, nEpochs=n_epochs, numThreads=0,
                                singleThreaded=True, numVisualizedSamples=0)
    la = {"lars": LayerAdaptation.LARS, "lamb": LayerAdaptation.LAMB}.get(kind.split("_")[0], LayerAdaptation.NONE)
    captured = {}
    orig = Solver.build_worker.__func__

    def spy(cls, args):
        worker, sched, ckpt = orig(cls, args)
        captured["worker"] = worker
        return worker, sched, ckpt

    Solver.build_worker = classmethod(spy)
    try:
        torch.manual_seed(SEED)
        random.seed(SEED)            # the loop's random sample picks decide how many gather launches run
        LocalSolver.solve(run_opts, problem, precision=precision, graph=graph, layer_adaptation=la,
                          grad_accumulation=k, **solve_kw)
    finally:
        Solver.build_worker = classmethod(orig)
    final = torch.load(os.path.join(save_dir, "final_model.pth"), weights_only=False)
    return captured["worker"], final


def _compare(a, b, rtol=1e-5, atol=1e-7):
    for name, v in a["state_dict"].items():
        np.testing.assert_allclose(v.float().numpy(), b["state_dict"][name].float().numpy(), rtol=rtol, atol=atol,
                                   err_msg=name)
    sa, sb = a["optimizer"]["state"], b["optimizer"]["state"]
    assert sa.keys() == sb.keys()
    for i in sa:
        for key, v in sa[i].items():
            if torch.is_tensor(v):
                np.testing.assert_allclose(v.float().numpy(), sb[i][key].float().numpy(), rtol=rtol, atol=atol,
                                           err_msg="%s %s" % (i, key))


@pytest.mark.parametrize("kind", ["sgd", "adam", "sgd_clip", "adam_clip", "lars", "lamb"])
def test_four_microbatches_equal_one_batch_of_their_rows(kind):
    w_acc, acc = _solve(kind, 16, 4)
    w_big, big = _solve(kind, 64, 1)
    assert w_acc.optimizer._steps == w_big.optimizer._steps == 10           # 9 full groups + the ragged one
    _compare(acc, big)
    if kind.startswith(("adam", "lamb")):
        assert float(acc["optimizer"]["state"][0]["step"]) == 10
    rows = [r for _, split, r in w_acc.loss_history if split.name == "TRAIN"]
    assert rows[0].shape[0] == 38 and [r for _, _, r in w_big.loss_history][0].shape[0] == 10


def test_graph_replay_matches_eager_launches_bit_for_bit():
    w_eager, eager = _solve("adam", 16, 4, n_epochs=2)
    w_graph, graphed = _solve("adam", 16, 4, graph=True, n_epochs=2)
    assert w_graph.graphed is not None and len(w_graph.graphed._graphs) == 1     # one per batch signature
    for name, v in eager["state_dict"].items():
        assert torch.equal(v, graphed["state_dict"][name]), name
    _compare(eager, graphed, rtol=0, atol=0)


def test_k1_keyword_is_todays_path(caplog):
    with caplog.at_level(logging.INFO):
        w_kw, kw = _solve("sgd", 32, 1)
    assert w_kw.pipeline.acc is None
    assert any("gradient accumulation none" in r.getMessage() for r in caplog.records)
    before = _native.launch_count()
    w_plain, plain = _solve("sgd", 32, None)
    n_plain = _native.launch_count() - before
    before = _native.launch_count()
    w_again, _ = _solve("sgd", 32, 1)
    assert _native.launch_count() - before == n_plain
    assert w_again.optimizer._steps == w_plain.optimizer._steps == 19       # 600 rows / 32, one update each
    for name, v in plain["state_dict"].items():
        assert torch.equal(v, kw["state_dict"][name]), name


def test_info_line_names_the_accumulator(caplog):
    with caplog.at_level(logging.INFO):
        w, _ = _solve("sgd", 16, 4)
    mib = w.pipeline.acc.numel() * 4 / 2 ** 20
    assert any("gradient accumulation 4 microbatches per update (K10, fp32 accumulator %.1f MiB)" % mib
               in r.getMessage() for r in caplog.records)


@pytest.mark.parametrize("precision,tol", [(Precision.BF16, 1e-2), (Precision.FP8, 5e-2)])
def test_low_precision_losses_follow_fp32(precision, tol):
    def mlp(ns, d):            # 6 updates of 2 microbatches; a width the FP8 path takes
        return synthetic.make_mlp_problem(ns, d, n_train=12 * 64, n_test=0, width=256, n_classes=16, reg_dim=16,
                                          depth=2)
    w32, _ = _solve("adam", 64, 2, problem_fn=mlp)
    wlp, _ = _solve("adam", 64, 2, problem_fn=mlp, precision=precision)
    assert w32.optimizer._steps == wlp.optimizer._steps == 6
    a = np.concatenate([r for _, _, r in w32.loss_history])
    b = np.concatenate([r for _, _, r in wlp.loss_history])
    np.testing.assert_allclose(b, a, rtol=tol, atol=tol)


# ---- autograd-allocated gradients, BatchNorm, ignore_index: against stock torch accumulation ------

def _against_torch(problem_fn, batch, k, optim, batches_fn, graph=False):
    """The worker at ``batch`` rows x ``k`` per update against stock fp32 torch doing the same
    per-microbatch forward and ``.grad`` accumulation of ``loss * n_i / N``, then ``SGD.step()``.
    Returns (worker, worker losses, torch losses, where each slot's gradient was read after the
    first microbatch: True = in place, outside the arena)."""
    from oracle import ref_loop
    ns = synthetic.api_namespace("frl_b200")
    t = ns.types
    save_dir = tempfile.mkdtemp(prefix="frl_b200_accum_ref_")
    problem = problem_fn(ns, save_dir)
    run_opts = t.RunOpts(optim=optim, batchSize=batch, nEpochs=1, numThreads=0, singleThreaded=True,
                         numVisualizedSamples=0)
    args = SolverWorkerArgs(run_opts=run_opts, problem=problem, save_dir=save_dir, run_device=Device.GPU,
                            node_idx=0, node_count=1, rank=0, local_rank=0, world_size=1, group_name=None,
                            init_method="", precision=Precision.FP32, graph_step=graph, grad_accumulation=k)
    torch.manual_seed(0)
    worker, _, _ = Solver.build_worker(args)
    torch.backends.cudnn.benchmark = False
    worker.model.train()
    worker.criterion.train()
    batches = batches_fn(worker, problem)
    rows = [d[0].shape[0] for d, _ in batches]
    plan = accumulation_plan(len(batches), k, batch, sum(rows))
    got, in_place = [], None
    for i, (mb, (data, target)) in enumerate(zip(plan, batches)):
        worker.pipeline.set_microbatch(first=mb.first, closes=mb.closes, weight=mb.weight,
                                       group_scale=batch / mb.group_rows)
        _, total, _, _ = worker._pass_one_minibatch(i, t.Split.TRAIN, data, target)
        got.append(float(total.detach()))
        del total
        if in_place is None:
            table = worker.pipeline.tables.whole()
            lo = worker.arena.grad.data_ptr()
            hi = lo + worker.arena.grad.numel() * worker.arena.grad.element_size()
            in_place = {s.index: not (lo <= (table._segs[j].g or 0) < hi) for j, s in enumerate(table.slots)}
    torch.cuda.synchronize()
    assert worker.optimizer._steps == sum(mb.closes for mb in plan)

    torch.manual_seed(0)
    ref_problem = problem_fn(ns, tempfile.mkdtemp(prefix="frl_b200_accum_ref_"))
    ref = ref_problem.get_model().cuda()
    crit = ref_problem.get_criterion()
    mods, weights, names = list(crit.loss_modules), list(crit.loss_weights), list(crit.loss_names)
    opt = torch.optim.SGD(ref.parameters(), lr=optim.lr, momentum=optim.momentum, weight_decay=optim.weightDecay)
    ref.train()
    want = []
    opt.zero_grad()
    for mb, (data, target) in zip(plan, batches):
        total, _ = ref_loop.parallel_criterion(mods, weights, names, ref(data), target)
        (total * (mb.rows / mb.group_rows)).backward()
        want.append(total.item())
        if mb.closes:
            opt.step()
            opt.zero_grad()
    return worker, np.asarray(got), np.asarray(want), in_place


@pytest.fixture()
def exact_cudnn():
    old = (torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic,
           torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic = False, True
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    (torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic,
     torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32) = old


@pytest.mark.parametrize("graph", [False, True])
def test_resnet_with_batchnorm_matches_stock_torch_accumulation(exact_cudnn, graph):
    """k = 2 over 8-row microbatches, the last one of 4 rows: convolution and BatchNorm gradients are
    allocated by cuDNN and read in place by K10 (kept alive by the captured graph when replayed),
    BatchNorm statistics move per microbatch as in stock torch."""
    g = torch.Generator().manual_seed(7)
    rows = [8] * 7 + [4]
    data = [(torch.randn(n, 3, 32, 32, generator=g), torch.randint(0, 1000, (n,), generator=g)) for n in rows]

    def problem_fn(ns, d):
        return synthetic.make_resnet_problem(ns, d, image=32, n_train=2)

    def batches_fn(worker, problem):
        return [([x.cuda()], [(y.cuda(),)]) for x, y in data]

    o = OptimOpts(algo=OptAlgorithm.SGD, lr=0.05, momentum=0.9, weightDecay=1e-4)
    worker, got, want, in_place = _against_torch(problem_fn, 8, 2, o, batches_fn, graph=graph)
    convs = [m for m in worker.model.modules() if isinstance(m, torch.nn.Conv2d)]
    bns = [m for m in worker.model.modules() if isinstance(m, torch.nn.BatchNorm2d)]
    slot = worker.arena.slot_of
    assert convs and bns and all(in_place[slot(m.weight).index] for m in convs)
    if graph:
        assert worker.graphed is not None and len(worker.graphed._graphs) == 1
    print("resnet k=2 losses", got.tolist(), "torch", want.tolist())
    np.testing.assert_allclose(got[:2], want[:2], rtol=1e-5, atol=1e-6)       # before any update
    np.testing.assert_allclose(got[2:], want[2:], rtol=1e-3, atol=1e-5)


def test_text_problem_with_ignore_index_matches_stock_torch_accumulation():
    """Cross-entropy with ignore_index = 0 over padded lines served by the device loader, k = 2: the
    update is the row-weighted mean of the per-microbatch means, exactly what stock torch's
    accumulation of ``loss * n_i / N`` computes."""
    def problem_fn(ns, d):
        for name in ("train.txt", "test.txt"):
            synthetic.write_text_corpus(os.path.join(d, name), 100, 3, seq_len=16)
        return synthetic.make_text_problem(ns, d, os.path.join(d, "train.txt"), os.path.join(d, "test.txt"),
                                           seq_len=16, device_batches=True)

    def batches_fn(worker, problem):
        torch.manual_seed(1)
        loader = DeviceBatchLoader(problem.datasets[0], batch_size=16, sampler=None, device=torch.device("cuda", 0))
        # the loader's device slots are reused: keep copies
        return [([t.clone() for t in d], [tuple(x.clone() for x in h) for h in tg]) for d, tg, _ in loader]

    o = OptimOpts(algo=OptAlgorithm.SGD, lr=0.5, momentum=0.9, weightDecay=1e-4)
    worker, got, want, _ = _against_torch(problem_fn, 16, 2, o, batches_fn)
    assert len(got) >= 4
    print("text k=2 losses", got.tolist(), "torch", want.tolist())
    np.testing.assert_allclose(got[:2], want[:2], rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(got[2:], want[2:], rtol=1e-3, atol=1e-5)


# ---- resume ------------------------------------------------------------------------------------

def test_resumed_run_is_bit_exact(monkeypatch):
    """4 epochs in one run against 2 epochs plus a resume for 2 more, k = 3 over 38 microbatches per
    epoch (not a multiple of 3).  The test reseeds torch's global RNG at the start of every epoch, so
    the single-process sampler's permutation depends only on the epoch (as ScaffoldSampler's does)."""
    from frl_b200.solver_worker import SolverWorker
    orig = SolverWorker._pass_one_epoch

    def seeded(self, *a, **kw):
        torch.manual_seed(1000 + self.cur_epoch)
        return orig(self, *a, **kw)

    monkeypatch.setattr(SolverWorker, "_pass_one_epoch", seeded)
    _, whole = _solve("adam", 16, 3, n_epochs=4)
    save_dir = tempfile.mkdtemp(prefix="frl_b200_accum_resume_")
    _solve("adam", 16, 3, n_epochs=2, save_dir=save_dir)
    shutil.copy(os.path.join(save_dir, "final_model.pth"), os.path.join(save_dir, ".checkpoint.pth"))
    w, resumed = _solve("adam", 16, 3, n_epochs=4, save_dir=save_dir)
    assert resumed["epoch"] == whole["epoch"] == 4
    assert float(resumed["optimizer"]["state"][0]["step"]) == float(whole["optimizer"]["state"][0]["step"]) == 4 * 13
    _compare(whole, resumed, rtol=0, atol=0)
    for name, v in whole["state_dict"].items():
        assert torch.equal(v, resumed["state_dict"][name]), name


# ---- refusals and two GPUs -----------------------------------------------------------------------

def test_gradnorm_criterion_refuses_accumulation():
    ns = synthetic.api_namespace("frl_b200")
    save_dir = tempfile.mkdtemp(prefix="frl_b200_accum_gn_")
    problem = synthetic.make_toy_problem(ns, save_dir, criterion_kind="gradnorm")
    run_opts = ns.types.RunOpts(optim=OptimOpts(algo=OptAlgorithm.SGD), batchSize=16, nEpochs=1, numThreads=0,
                                singleThreaded=True)
    args = SolverWorkerArgs(run_opts=run_opts, problem=problem, save_dir=save_dir, run_device=Device.GPU,
                            node_idx=0, node_count=1, rank=0, local_rank=0, world_size=1, group_name=None,
                            init_method="", grad_accumulation=2)
    with pytest.raises(ValueError, match="GradNormWeightedCriterion"):
        Solver.build_worker(args)
    worker, _, _ = Solver.build_worker(args._replace(grad_accumulation=1))    # k = 1 stays allowed
    assert worker.pipeline.acc is None


@pytest.mark.parametrize("backend", ["nccl", "gloo"])
def test_two_ranks_accumulating_equal_two_ranks_at_the_group_batch(backend):
    """2 ranks at 16 rows x 2 per update against 2 ranks at 32 rows, with the real kernels
    (tests/run_accum_mp.py): over NCCL with one GPU per rank (needs 2 GPUs), and over gloo with both
    ranks on GPU 0, which runs the same world > 1 accumulation path on a one-GPU machine."""
    import subprocess
    import sys
    if backend == "nccl" and torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    script = os.path.join(os.path.dirname(__file__), "run_accum_mp.py")
    port = "29543" if backend == "nccl" else "29544"
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                          "--master-addr", "127.0.0.1", "--master-port", port, script, "--backend", backend],
                         capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
    assert out.stdout.count("ACCUM_MP_OK") == 2
