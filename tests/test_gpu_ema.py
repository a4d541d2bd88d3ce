"""Weight EMA on the H100: K11 (``frl_weight_ema``) against torch's lerp, the solver's EMA against
stock torch's ``AveragedModel``, and whole runs through ``LocalSolver.solve``: the EMA leaves
training untouched, resumes bit for bit, and its saved file evaluates to the held-out losses the
run reported."""
import logging
import math
import os
import random
import shutil
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch
from torch.optim.swa_utils import AveragedModel, get_ema_multi_avg_fn

import frl_b200  # noqa: F401
from frl_b200 import _native, synthetic
from frl_b200.local_solver import LocalSolver
from frl_b200.solver import Solver, SolverWorkerArgs
from frl_b200.types import Device, Mode, OptAlgorithm, OptimOpts, Precision, Split

pytestmark = pytest.mark.gpu


# ---- K11 against torch -------------------------------------------------------------------------

@pytest.mark.parametrize("n", [0, 1, 3, 4, 4097, (1 << 20) + 3])
def test_k11_matches_torch_lerp_bit_for_bit(n):
    """Bit-exact against ``torch.lerp`` and ``torch._foreach_lerp_`` (what ``AveragedModel`` calls)
    with the same fp32 weight: K11 writes each branch of torch's formula as the fmaf nvcc contracts
    torch's own kernel into."""
    g = torch.Generator(device="cuda").manual_seed(n)
    for w in (1e-4, 0.3, 0.5, 0.7, 1.0):
        ema = torch.randn(n, device="cuda", generator=g)
        p = torch.randn(n, device="cuda", generator=g) * 3
        want = torch.lerp(ema, p, w)
        foreach = [ema.clone()]
        torch._foreach_lerp_(foreach, [p], w)
        before = _native.launch_count()
        _native.weight_ema(ema, p, w)
        assert _native.launch_count() - before == (1 if n else 0)
        torch.cuda.synchronize()
        assert torch.equal(ema, want), (n, w)
        assert torch.equal(ema, foreach[0]), (n, w)


def test_k11_argument_errors_launch_nothing():
    a = torch.zeros(64, device="cuda")
    before = _native.launch_count()
    for ema, p, w in ((a[1:9], a[16:24], 0.5), (a[:8], a[17:25], 0.5), (a[:8], a[8:16], 1.5),
                      (a[:8], a[8:16], -0.25), (a[:8], a[8:16], math.nan)):
        with pytest.raises(_native.NativeLibraryError):
            _native.weight_ema(ema, p, w)
    assert _native.launch_count() == before


def test_k11_replays_from_a_cuda_graph():
    n = 4097
    ema, p = torch.randn(n, device="cuda"), torch.randn(n, device="cuda")
    want = ema.clone()
    for _ in range(3):
        want = torch.lerp(want, p, 0.25)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    start = ema.clone()
    with torch.cuda.graph(graph):
        _native.weight_ema(ema, p, 0.25)
    ema.copy_(start)
    for _ in range(3):
        graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(ema, want)


# ---- against stock torch: AveragedModel(..., use_buffers=True) -----------------------------------

@pytest.fixture()
def exact_cudnn():
    old = (torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic,
           torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic = False, True
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    (torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic,
     torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32) = old


def _against_torch(problem_fn, optim, decay, train, held_out):
    """The worker (fp32, one GPU) over ``train`` batches with a weight EMA, against stock fp32 torch
    (the same model, ``torch.optim``, ``AveragedModel(..., use_buffers=True)`` updated after every
    ``step()``).  Returns the worker's EMA state dict, the averaged module's, and both held-out
    losses per batch (the worker's from its EMA swapped in)."""
    from oracle import ref_loop
    ns = synthetic.api_namespace("frl_b200")
    t = ns.types
    save_dir = tempfile.mkdtemp(prefix="frl_b200_ema_ref_")
    problem = problem_fn(ns, save_dir)
    run_opts = t.RunOpts(optim=optim, batchSize=train[0][0][0].shape[0], nEpochs=1, numThreads=0,
                         singleThreaded=True, numVisualizedSamples=0)
    args = SolverWorkerArgs(run_opts=run_opts, problem=problem, save_dir=save_dir, run_device=Device.GPU,
                            node_idx=0, node_count=1, rank=0, local_rank=0, world_size=1, group_name=None,
                            init_method="", precision=Precision.FP32, ema_decay=decay)
    torch.manual_seed(0)
    worker, _, _ = Solver.build_worker(args)
    torch.backends.cudnn.benchmark = False
    worker.model.train()
    worker.criterion.train()
    for i, (data, target) in enumerate(train):
        _, total, _, _ = worker._pass_one_minibatch(i, t.Split.TRAIN, data, target)
        del total
    assert worker.ema.updates == len(train)
    worker.model.eval()
    worker.criterion.eval()
    got = []
    with torch.no_grad(), worker.ema.swapped():
        for i, (data, target) in enumerate(held_out):
            _, total, _, _ = worker._pass_one_minibatch(i, t.Split.TEST, data, target)
            got.append(float(total))
    mine = worker.ema.state_dict()["state_dict"]
    live = {k: v.detach().cpu().clone() for k, v in worker.model.state_dict().items()}

    torch.manual_seed(0)
    ref_problem = problem_fn(ns, tempfile.mkdtemp(prefix="frl_b200_ema_ref_"))
    ref = ref_problem.get_model().cuda()
    crit = ref_problem.get_criterion()
    mods, weights, names = list(crit.loss_modules), list(crit.loss_weights), list(crit.loss_names)
    if optim.algo == OptAlgorithm.SGD:
        opt = torch.optim.SGD(ref.parameters(), lr=optim.lr, momentum=optim.momentum, weight_decay=optim.weightDecay)
    else:
        opt = torch.optim.Adam(ref.parameters(), lr=optim.lr, weight_decay=optim.weightDecay, eps=optim.epsilon)
    avg = AveragedModel(ref, multi_avg_fn=get_ema_multi_avg_fn(decay), use_buffers=True)
    ref.train()
    for data, target in train:
        total, _ = ref_loop.parallel_criterion(mods, weights, names, ref(data), target)
        opt.zero_grad()
        total.backward()
        opt.step()
        avg.update_parameters(ref)
    avg.module.eval()
    want = []
    with torch.no_grad():
        for data, target in held_out:
            want.append(float(ref_loop.parallel_criterion(mods, weights, names, avg.module(data), target)[0]))
    theirs = {k: v.detach().cpu() for k, v in avg.module.state_dict().items()}
    ref_live = {k: v.detach().cpu() for k, v in ref.state_dict().items()}
    return mine, theirs, np.asarray(got), np.asarray(want), live, ref_live


def _mlp_batches(n, rows, seed):
    g = torch.Generator().manual_seed(seed)
    return [([torch.randn(rows, 128, generator=g).cuda()],
             [(torch.randint(0, 10, (rows,), generator=g).cuda(),), (torch.randn(rows, 8, generator=g).cuda(),)])
            for _ in range(n)]


def _mlp(ns, d):
    return synthetic.make_mlp_problem(ns, d, n_train=64, n_test=0, width=128, n_classes=10, reg_dim=8, depth=2)


@pytest.mark.parametrize("algo", ["sgd", "adam"])
def test_mlp_ema_matches_averaged_model(algo):
    if algo == "sgd":
        o = OptimOpts(algo=OptAlgorithm.SGD, lr=0.05, momentum=0.9, weightDecay=1e-4)
    else:
        o = OptimOpts(algo=OptAlgorithm.ADAM, lr=1e-3, weightDecay=1e-4)
    mine, theirs, got, want, _, _ = _against_torch(_mlp, o, 0.8, _mlp_batches(8, 16, 1), _mlp_batches(3, 16, 2))
    assert list(mine) == list(theirs)
    print("mlp %s held-out losses" % algo, got.tolist(), "torch", want.tolist())
    for k, v in theirs.items():
        d = (mine[k] - v).abs()
        print("  %-24s max %.2e median %.2e" % (k, float(d.max()), float(d.flatten().median())))
        if algo == "sgd":
            np.testing.assert_allclose(mine[k].numpy(), v.numpy(), rtol=1e-4, atol=1e-6, err_msg=k)
        else:
            # Adam's first steps are lr * sign(g): a gradient entry at rounding level can take either
            # sign on two code paths, which moves that weight by up to 2 lr (test_gpu_mlp_parity)
            assert float(d.flatten().median()) <= 1e-6 and float(d.max()) <= 4 * o.lr, k
    np.testing.assert_allclose(got, want, rtol=1e-4 if algo == "sgd" else 1e-3)


def test_resnet_with_batchnorm_ema_matches_averaged_model(exact_cudnn):
    g = torch.Generator().manual_seed(7)

    def batches(n, rows):
        return [([torch.randn(rows, 3, 32, 32, generator=g).cuda()], [(torch.randint(0, 1000, (rows,), generator=g).cuda(),)])
                for _ in range(n)]

    def problem_fn(ns, d):
        return synthetic.make_resnet_problem(ns, d, image=32, n_train=2)

    o = OptimOpts(algo=OptAlgorithm.SGD, lr=1e-3, momentum=0.9, weightDecay=1e-4)
    mine, theirs, got, want, live, ref_live = _against_torch(problem_fn, o, 0.7, batches(5, 8), batches(2, 8))
    assert list(mine) == list(theirs)
    assert any("running_mean" in k for k in theirs)
    print("resnet held-out losses", got.tolist(), "torch", want.tolist())
    for k, v in theirs.items():
        if v.is_floating_point():
            # the live ResNet weights already differ from stock torch's (cuDNN's convolution
            # gradients are not this path's); the average of the trajectory may differ by as much
            d_ema = float((mine[k] - v).abs().max())
            d_live = float((live[k] - ref_live[k]).abs().max())
            print("  %-40s ema %.2e live %.2e" % (k, d_ema, d_live))
            assert d_ema <= 2 * d_live + 1e-6, (k, d_ema, d_live)
        else:
            # num_batches_tracked is copied from the live model (torch lerps it in floats and truncates)
            assert torch.equal(mine[k], ref_live[k]), k
    np.testing.assert_allclose(got, want, rtol=1e-3, atol=1e-5)


# ---- whole runs through LocalSolver.solve --------------------------------------------------------

SEED = 11
N_TRAIN, N_TEST = 600, 64      # batch 16: 38 training microbatches, 4 held-out batches


def _solve(ema_decay, *, k=1, precision=Precision.FP32, graph=False, n_epochs=1, save_dir=None, algo="adam",
           mode=Mode.TRAIN, initial=None):
    ns = synthetic.api_namespace("frl_b200")
    save_dir = save_dir or tempfile.mkdtemp(prefix="frl_b200_ema_")
    torch.manual_seed(SEED)
    problem = synthetic.make_mlp_problem(ns, save_dir, n_train=N_TRAIN, n_test=N_TEST, width=128, n_classes=10,
                                         reg_dim=8, depth=2)
    if algo == "sgd":
        o = OptimOpts(algo=OptAlgorithm.SGD, lr=0.05, momentum=0.9, weightDecay=1e-4)
    else:
        o = OptimOpts(algo=OptAlgorithm.ADAM, lr=1e-3, weightDecay=1e-4)
    run_opts = ns.types.RunOpts(optim=o, batchSize=16, nEpochs=n_epochs, numThreads=0, singleThreaded=True,
                                numVisualizedSamples=0, mode=mode, initialModelPath=initial)
    captured = {}
    orig = Solver.build_worker.__func__

    def spy(cls, args):
        worker, sched, ckpt = orig(cls, args)
        captured["worker"] = worker
        return worker, sched, ckpt

    Solver.build_worker = classmethod(spy)
    try:
        torch.manual_seed(SEED)
        random.seed(SEED)
        last = LocalSolver.solve(run_opts, problem, precision=precision, graph=graph, grad_accumulation=k,
                                 ema_decay=ema_decay)
    finally:
        Solver.build_worker = classmethod(orig)
    return captured["worker"], last, save_dir


def _load(save_dir, name):
    return torch.load(os.path.join(save_dir, name), weights_only=False)


def _train_rows(worker):
    return [r for _, split, r in worker.loss_history if split == Split.TRAIN]


@pytest.mark.parametrize("k", [1, 3])
@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("precision", [Precision.FP32, Precision.BF16])
def test_ema_does_not_perturb_training(precision, graph, k):
    """Two epochs, the held-out split evaluated with the EMA in between: training losses and the
    final live weights are bit-identical to the same run without an EMA."""
    w_off, _, d_off = _solve(0.0, k=k, precision=precision, graph=graph, n_epochs=2)
    w_on, _, d_on = _solve(0.99, k=k, precision=precision, graph=graph, n_epochs=2)
    assert w_off.ema is None and w_on.ema is not None
    if graph:
        assert w_on.graphed is not None and w_on.graphed._graphs
    a, b = _train_rows(w_off), _train_rows(w_on)
    assert len(a) == len(b) == 2 and a[0].shape[0] == 38
    for x, y in zip(a, b):
        assert np.array_equal(x, y)
    off, on = _load(d_off, "final_model.pth"), _load(d_on, "final_model.pth")
    assert list(off) == list(on)
    for name, v in off["state_dict"].items():
        assert torch.equal(v, on["state_dict"][name]), name
    assert not os.path.exists(os.path.join(d_off, "final_model.pth.ema"))
    blob = _load(d_on, "final_model.pth.ema")
    assert list(blob) == ["epoch", "decay", "updates", "state_dict"]
    assert blob["updates"] == 2 * (38 if k == 1 else 13) == w_on.optimizer._steps
    assert list(blob["state_dict"]) == list(on["state_dict"])


def test_resumed_run_is_bit_exact(monkeypatch):
    """4 epochs in one run against 2 epochs plus a resume for 2 more (k = 3, 13 updates per epoch),
    with the main checkpoint and its EMA file copied to the resume names."""
    from frl_b200.solver_worker import SolverWorker
    orig = SolverWorker._pass_one_epoch

    def seeded(self, *a, **kw):
        torch.manual_seed(1000 + self.cur_epoch)
        return orig(self, *a, **kw)

    monkeypatch.setattr(SolverWorker, "_pass_one_epoch", seeded)
    _, _, d_whole = _solve(0.9, k=3, n_epochs=4)
    save_dir = tempfile.mkdtemp(prefix="frl_b200_ema_resume_")
    _solve(0.9, k=3, n_epochs=2, save_dir=save_dir)
    for src, dst in (("final_model.pth", ".checkpoint.pth"), ("final_model.pth.ema", ".checkpoint.pth.ema")):
        shutil.copy(os.path.join(save_dir, src), os.path.join(save_dir, dst))
    w, _, _ = _solve(0.9, k=3, n_epochs=4, save_dir=save_dir)
    whole, resumed = _load(d_whole, "final_model.pth.ema"), _load(save_dir, "final_model.pth.ema")
    assert resumed["epoch"] == whole["epoch"] == 4
    assert resumed["updates"] == whole["updates"] == 4 * 13
    for name, v in whole["state_dict"].items():
        assert torch.equal(v, resumed["state_dict"][name]), name
    live_whole, live_resumed = _load(d_whole, "final_model.pth"), _load(save_dir, "final_model.pth")
    for name, v in live_whole["state_dict"].items():
        assert torch.equal(v, live_resumed["state_dict"][name]), name


def test_saved_ema_evaluates_to_the_reported_held_out_losses():
    w, last, save_dir = _solve(0.9, n_epochs=2, algo="sgd")
    reported = last.performance[Split.TEST].losses
    path = os.path.join(save_dir, "final_model.pth.ema")
    _, evaluated, _ = _solve(0.9, mode=Mode.EVAL, initial=path, algo="sgd",
                             save_dir=tempfile.mkdtemp(prefix="frl_b200_ema_eval_"))
    got = evaluated.performance[Split.TEST].losses
    assert reported.keys() == got.keys()
    for name, v in reported.items():
        # the held-out batches come in another order: the same per-batch losses, summed differently
        assert math.isclose(got[name], v, rel_tol=1e-5), (name, got[name], v)
    # ... and they are the EMA's, not the live model's
    live = _solve(0.9, mode=Mode.EVAL, initial=os.path.join(save_dir, "final_model.pth"), algo="sgd",
                  save_dir=tempfile.mkdtemp(prefix="frl_b200_ema_eval_"))[1].performance[Split.TEST].losses
    assert any(not math.isclose(live[name], v, rel_tol=1e-6) for name, v in reported.items())


def test_info_line_names_the_ema(caplog):
    with caplog.at_level(logging.INFO):
        w, _, _ = _solve(0.9)
    mib = w.ema.nbytes / 2 ** 20
    assert any("weight EMA decay 0.9, one K11 launch per update (%.1f MiB), held-out splits evaluated with it"
               % mib in r.getMessage() for r in caplog.records)
    caplog.clear()
    with caplog.at_level(logging.INFO):
        _solve(0.0)
    assert any("| weight EMA none" in r.getMessage() for r in caplog.records)


def test_two_ranks_keep_identical_emas():
    """tests/run_ema_mp.py: two ranks over gloo, both on GPU 0, eager per-bucket updates."""
    script = os.path.join(os.path.dirname(__file__), "run_ema_mp.py")
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                          "--master-addr", "127.0.0.1", "--master-port", "29547", script],
                         capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
    assert out.stdout.count("EMA_MP_OK") == 2
