"""Gradient accumulation on the host: resolving and validating the switch, the group arithmetic,
the pipeline's accumulate-then-update path against one large batch (1 and 2 ranks over gloo) with
the kernels replaced by a CPU double, and K10's argument checks."""
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn as nn

import frl_b200  # noqa: F401
from frl_b200 import fused_optim, grad_sync, synthetic
from frl_b200.arena import ParamArena
from frl_b200.grad_sync import accumulation_plan
from frl_b200.solver import Solver, SolverWorkerArgs, resolve_grad_accumulation
from frl_b200.types import LayerAdaptation, Mode, OptAlgorithm, OptimOpts
from layerwise_oracle import LayerwiseKernelDouble, _read

f32 = np.float32


class AccumKernelDouble(LayerwiseKernelDouble):
    """Adds a CPU stand-in for ``_native.grad_accumulate_mt`` (K10)."""

    def grad_accumulate_mt(self, acc, table, *, w=1.0, first=False, dyn=None):
        self.calls.append(("grad_accumulate_mt", table.n_segs))
        if dyn is not None:
            w, first = float(dyn[0]), bool(dyn[1] != 0)
        for i, s in enumerate(table.slots):
            row = table._segs[i]
            base = np.zeros(s.numel, f32) if first else acc[s.offset:s.end].numpy().copy()
            if row.g:
                base = (base + f32(w) * _read(row.g, s.numel, row.g_dtype)).astype(f32)
            acc[s.offset:s.end] = torch.from_numpy(base)


@pytest.fixture()
def double(monkeypatch):
    d = AccumKernelDouble()
    monkeypatch.setattr(fused_optim, "KERNELS", d)
    monkeypatch.setattr(grad_sync, "KERNELS", d)
    return d


# ---- the switch --------------------------------------------------------------------------------

def test_resolution_keyword_beats_environment(monkeypatch):
    monkeypatch.delenv("FRL_B200_GRAD_ACCUM", raising=False)
    assert resolve_grad_accumulation() == 1
    monkeypatch.setenv("FRL_B200_GRAD_ACCUM", "4")
    assert resolve_grad_accumulation() == 4
    assert resolve_grad_accumulation(2) == 2
    assert SolverWorkerArgs._field_defaults["grad_accumulation"] == 1
    assert SolverWorkerArgs._fields[-1] == "grad_accumulation"


def _toy(tmp_path, mode=Mode.TRAIN, **kw):
    ns = synthetic.api_namespace("frl_b200")
    problem = synthetic.make_toy_problem(ns, str(tmp_path), n_train=8, n_test=0)
    run_opts = ns.types.RunOpts(optim=OptimOpts(algo=OptAlgorithm.SGD), batchSize=4, nEpochs=1,
                                singleThreaded=True, mode=mode, **kw)
    return problem, run_opts


@pytest.mark.parametrize("bad", [0, -2, 2.5, True, "3"])
def test_bad_keyword_values_raise_before_any_rank_starts(tmp_path, monkeypatch, bad):
    monkeypatch.delenv("FRL_B200_GRAD_ACCUM", raising=False)
    problem, run_opts = _toy(tmp_path)
    with pytest.raises(ValueError, match=repr(bad).replace(".", r"\.")):
        next(Solver.solve(run_opts, problem, group_name=None, init_method="", grad_accumulation=bad))


@pytest.mark.parametrize("raw", ["0", "-1", "two", "2.5", ""])
def test_bad_environment_values_raise_before_any_rank_starts(tmp_path, monkeypatch, raw):
    monkeypatch.setenv("FRL_B200_GRAD_ACCUM", raw)
    problem, run_opts = _toy(tmp_path)
    with pytest.raises(ValueError, match="gradient accumulation"):
        next(Solver.solve(run_opts, problem, group_name=None, init_method=""))


def test_eval_mode_ignores_the_setting(tmp_path, monkeypatch):
    monkeypatch.setenv("FRL_B200_GRAD_ACCUM", "two")
    problem, run_opts = _toy(tmp_path, mode=Mode.EVAL, cpuonly=True)
    # no ValueError: EVAL never resolves the switch and stops at the missing device instead
    with pytest.raises(RuntimeError, match="no CPU path"):
        next(Solver.solve(run_opts, problem, group_name=None, init_method="", grad_accumulation=0))


# ---- group arithmetic --------------------------------------------------------------------------

@pytest.mark.parametrize("n_batches,k,closing,groups", [
    (10, 4, [3, 7, 9], [(0, 4), (4, 8), (8, 10)]),
    (3, 4, [2], [(0, 3)]),
    (8, 4, [3, 7], [(0, 4), (4, 8)]),
    (5, 1, [0, 1, 2, 3, 4], [(0, 1), (1, 2), (2, 3), (3, 4), (4, 5)]),
])
def test_group_plan(n_batches, k, closing, groups):
    B = 16
    n_samples = (n_batches - 1) * B + 8                  # ragged last microbatch of 8 rows
    plan = accumulation_plan(n_batches, k, B, n_samples)
    assert len(plan) == n_batches
    assert [j for j, mb in enumerate(plan) if mb.closes] == closing
    assert [j for j, mb in enumerate(plan) if mb.first] == [lo for lo, _ in groups]
    for lo, hi in groups:
        rows = [B] * (hi - lo)
        if hi == n_batches:
            rows[-1] = 8
        for j in range(lo, hi):
            assert plan[j].rows == rows[j - lo]
            assert plan[j].weight == rows[j - lo] / B
            assert plan[j].group_rows == sum(rows)
    # full last microbatch: every weight is exactly 1
    assert all(mb.weight == 1.0 for mb in accumulation_plan(n_batches, k, B, n_batches * B))


def test_plan_rejects_inconsistent_sizes():
    with pytest.raises(ValueError):
        accumulation_plan(3, 2, 16, 100)
    assert accumulation_plan(0, 3, 16, 0) == []


# ---- the pipeline over a small model -----------------------------------------------------------

class _Net(nn.Module):
    def __init__(self, seed):
        super().__init__()
        torch.manual_seed(seed)
        self.body = nn.Sequential(nn.Linear(7, 5), nn.ReLU(), nn.Linear(5, 3), nn.ReLU(), nn.Linear(3, 2))
        self.unused = nn.Linear(2, 2)              # never in the forward: keeps weights and state

    def forward(self, x):
        return self.body(x)


def _opts(algo, clip):
    if algo == "sgd" or algo == "lars":
        return OptimOpts(algo=OptAlgorithm.SGD, lr=0.05, momentum=0.9, weightDecay=1e-2, gradientClip=clip)
    return OptimOpts(algo=OptAlgorithm.ADAM, lr=0.01, weightDecay=1e-2, gradientClip=clip)


def _make(seed, algo, clip, k, world=1):
    net = _Net(seed)
    arena = ParamArena(net.parameters(), device="cpu")
    la = LayerAdaptation.LARS if algo == "lars" else LayerAdaptation.NONE
    opt = fused_optim.create_fused_optimizer(arena, _opts(algo, clip), la)
    kw = dict(bucket_cap_mb=0.0001, first_bucket_mb=0.00005) if world > 1 else {}
    pipe = grad_sync.GradBucketPipeline(arena, opt, world_size=world, clip_norm=clip, accumulation=k, **kw)
    return net, arena, opt, pipe


def _run_groups(net, pipe, xs, k, B):
    """Train over the rows ``xs`` in microbatches of B, k per update (as the solver worker does)."""
    n = xs.shape[0]
    n_batches = (n + B - 1) // B
    for j, mb in enumerate(accumulation_plan(n_batches, k, B, n)):
        pipe.set_microbatch(first=mb.first, closes=mb.closes, weight=mb.weight, group_scale=B / mb.group_rows)
        pipe.begin_step()
        net(xs[j * B:(j + 1) * B]).square().mean().backward()
        pipe.finish_step()


@pytest.mark.parametrize("algo,clip", [("sgd", 0.0), ("sgd", 0.05), ("adam", 0.0), ("adam", 0.05),
                                       ("lars", 0.0), ("lars", 0.05)])
def test_three_microbatches_equal_one_batch_of_their_rows(double, algo, clip):
    g = torch.Generator().manual_seed(5)
    xs = torch.randn(44, 7, generator=g)            # groups of 24 and 20 rows (8 + 8 + 4)
    net, arena, opt, pipe = _make(1, algo, clip, k=3)
    assert pipe.acc is not None and pipe.acc.numel() == arena.numel and not pipe.eager
    ref, ref_arena, ref_opt, ref_pipe = _make(1, algo, clip, k=1)
    assert ref_pipe.acc is None and ref_pipe.accumulator_bytes == 0
    unused = [p.detach().clone() for p in net.unused.parameters()]
    _run_groups(net, pipe, xs, 3, 8)
    ref_pipe.set_microbatch(first=True, closes=True)                   # no-op at k = 1
    for lo, hi in ((0, 24), (24, 44)):
        ref_pipe.begin_step()
        ref(xs[lo:hi]).square().mean().backward()
        ref_pipe.finish_step()
    assert opt._steps == ref_opt._steps == 2
    for a, b in zip(net.parameters(), ref.parameters()):
        np.testing.assert_allclose(a.detach().numpy(), b.detach().numpy(), rtol=2e-5, atol=1e-7)
    for name, vec in ref_opt._vec.items():
        np.testing.assert_allclose(opt._vec[name].numpy(), vec.numpy(), rtol=2e-5, atol=1e-7)
    # a parameter that never got a gradient keeps its weights and its state
    for a, b in zip(net.unused.parameters(), unused):
        assert torch.equal(a.detach(), b)
    for p in net.unused.parameters():
        s = arena.slot_of(p)
        for vec in opt._vec.values():
            assert not vec[s.offset:s.end].any()
    assert sum(1 for c in double.calls if c[0] == "grad_accumulate_mt") == 6


def test_parameter_with_gradients_in_some_microbatches_only(double):
    """A slot that misses a microbatch's gradient counts it as zero: the same as one batch whose
    loss only reaches it through the rows of the other microbatches."""
    g = torch.Generator().manual_seed(7)
    xs = torch.randn(16, 7, generator=g)
    net, arena, opt, pipe = _make(2, "sgd", 0.0, k=2)
    ref = _Net(2)
    ref_opt = torch.optim.SGD(ref.parameters(), lr=0.05, momentum=0.9, weight_decay=1e-2)
    for j, mb in enumerate(accumulation_plan(2, 2, 8, 16)):
        pipe.set_microbatch(first=mb.first, closes=mb.closes, weight=mb.weight, group_scale=8 / mb.group_rows)
        pipe.begin_step()
        x = xs[j * 8:(j + 1) * 8]
        out = net.body(x) if j == 0 else net.body[0](x)           # layers 2 and 4 miss microbatch 1
        out.square().mean().backward()
        pipe.finish_step()
    ref_opt.zero_grad()
    (ref.body(xs[:8]).square().mean() * 0.5 + ref.body[0](xs[8:]).square().mean() * 0.5).backward()
    ref_opt.step()
    for a, b in zip(net.body.parameters(), ref.body.parameters()):
        np.testing.assert_allclose(a.detach().numpy(), b.detach().numpy(), rtol=2e-5, atol=1e-7)


def test_without_a_position_every_microbatch_is_its_own_group(double):
    """A caller that never calls set_microbatch() (a benchmark driving the worker directly) gets one
    update per microbatch at weight 1 — the device block agrees with the by-value defaults."""
    g = torch.Generator().manual_seed(9)
    xs = torch.randn(24, 7, generator=g)
    net, arena, opt, pipe = _make(4, "adam", 0.0, k=3)
    ref, _, ref_opt, ref_pipe = _make(4, "adam", 0.0, k=1)
    assert pipe._acc_dyn.tolist() == [1.0, 1.0]
    for m, p in ((net, pipe), (ref, ref_pipe)):
        for j in range(3):
            p.begin_step(); m(xs[j * 8:(j + 1) * 8]).square().mean().backward(); p.finish_step()
    assert opt._steps == ref_opt._steps == 3
    for a, b in zip(net.parameters(), ref.parameters()):
        np.testing.assert_allclose(a.detach().numpy(), b.detach().numpy(), rtol=2e-5, atol=1e-7)


# ---- two ranks over gloo -----------------------------------------------------------------------

def _rank_main(rank, world, port, algo, out_dir):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    d = AccumKernelDouble()
    fused_optim.KERNELS = d
    grad_sync.KERNELS = d
    net, arena, opt, pipe = _make(20, algo, 0.0, k=2, world=world)
    assert not pipe.eager and pipe.nvls is None and len(pipe.buckets) > 1
    g = torch.Generator().manual_seed(99)
    for _ in range(2):                                        # 2 groups of 2 microbatches
        for j in range(2):
            x = torch.randn(4 * world, 7, generator=g)
            pipe.set_microbatch(first=j == 0, closes=j == 1, weight=1.0, group_scale=4 / 8)
            pipe.begin_step()
            (net(x[rank::world]).square().mean() + 0 * net.unused(net(x[rank::world])).sum()).backward()
            pipe.finish_step()
    torch.save([p.detach().clone() for p in net.parameters()], os.path.join(out_dir, f"r{rank}.pt"))
    dist.destroy_process_group()


@pytest.mark.parametrize("algo", ["sgd", "adam", "lars"])
def test_two_ranks_accumulating_equal_one_rank_at_the_global_group(tmp_path, algo):
    world = 2
    port = 33500 + (os.getpid() % 2000)
    mp.spawn(_rank_main, args=(world, port, algo, str(tmp_path)), nprocs=world, join=True)
    r0, r1 = torch.load(tmp_path / "r0.pt"), torch.load(tmp_path / "r1.pt")
    for a, b in zip(r0, r1):
        assert torch.equal(a, b)
    ref = _Net(20)
    la = LayerAdaptation.LARS if algo == "lars" else LayerAdaptation.NONE
    arena = ParamArena(ref.parameters(), device="cpu")
    d = AccumKernelDouble()
    old = fused_optim.KERNELS, grad_sync.KERNELS
    fused_optim.KERNELS = grad_sync.KERNELS = d
    try:
        opt = fused_optim.create_fused_optimizer(arena, _opts(algo, 0.0), la)
        pipe = grad_sync.GradBucketPipeline(arena, opt)
        g = torch.Generator().manual_seed(99)
        for _ in range(2):
            x = torch.cat([torch.randn(4 * world, 7, generator=g) for _ in range(2)])
            pipe.begin_step()
            (ref(x).square().mean() + 0 * ref.unused(ref(x)).sum()).backward()
            pipe.finish_step()
    finally:
        fused_optim.KERNELS, grad_sync.KERNELS = old
    for a, b in zip(r0, ref.parameters()):
        np.testing.assert_allclose(a.numpy(), b.detach().numpy(), rtol=2e-5, atol=1e-7)


# ---- K10 argument checks -----------------------------------------------------------------------

def test_grad_accumulate_rejects_bad_arguments_before_any_launch():
    from frl_b200 import _native
    lib = _native.lib()
    ok = 1 << 20                           # 16-byte aligned, never dereferenced: every call below fails a check
    before = lib.frl_launch_count()

    def acc(**kw):
        a = dict(acc=ok, segs=ok, pre=ok, tseg=ok, nt=4, dyn=None)
        a.update(kw)
        return lib.frl_grad_accumulate_mt(a["acc"], a["segs"], a["pre"], a["tseg"], a["nt"], 1.0, 1, a["dyn"], None)

    bad = [acc(acc=None), acc(acc=ok + 4), acc(acc=ok + 8), acc(segs=None), acc(pre=None), acc(tseg=None),
           acc(nt=-1), acc(dyn=ok + 2), acc(acc=None, nt=0)]
    assert all(rc < 0 for rc in bad), bad
    assert lib.frl_launch_count() == before
    assert acc(segs=None, pre=None, tseg=None, nt=0) == 0          # nothing to do, nothing launched
    assert lib.frl_launch_count() == before
