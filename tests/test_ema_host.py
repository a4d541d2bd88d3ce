"""Weight EMA on the host: resolving and validating the switch, where the K11 launch sits in the
end-of-step sequence of ``GradBucketPipeline`` (every configuration of ``test_pipeline_launches``,
one rank and two ranks over gloo, with a CPU double of K11), ``WeightEMA``'s swap and state
round trip, K11's argument checks, and what ``Solver._save_checkpoint`` writes."""
import io
import math
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn as nn
from torch.optim.swa_utils import AveragedModel, get_ema_multi_avg_fn

import frl_b200  # noqa: F401
from frl_b200 import ema as ema_mod, fused_optim, grad_sync, multi_tensor, synthetic
from frl_b200.arena import ParamArena
from frl_b200.ema import EMA_STATE_KEY, WeightEMA
from frl_b200.grad_sync import accumulation_plan
from frl_b200.solver import Solver, SolverWorkerArgs, resolve_ema_decay
from frl_b200.solver_worker import FractionalEpochSplitPerformanceSummary, FractionalPerformanceSummary, SingleSample
from frl_b200.types import Mode, OptAlgorithm, OptimOpts, Precision, Split
from test_pipeline_launches import (B, DEFERRED, EXPECTED, EXPECTED_2RANKS, N_MB, N_ROWS, OPTS, RecordingDouble,
                                    _CONFIGS_2RANKS, _in_place, _key, _Net)

DECAY = 0.75          # large steps, so that a misplaced or missing update shows in the values


# ---- the switch --------------------------------------------------------------------------------

def test_resolution_keyword_beats_environment(monkeypatch):
    monkeypatch.delenv("FRL_B200_EMA_DECAY", raising=False)
    assert resolve_ema_decay() == 0.0
    monkeypatch.setenv("FRL_B200_EMA_DECAY", "0.999")
    assert resolve_ema_decay() == 0.999
    assert resolve_ema_decay(0.5) == 0.5
    assert resolve_ema_decay(0) == 0.0
    assert SolverWorkerArgs._field_defaults["ema_decay"] == 0.0
    assert SolverWorkerArgs._fields[-2:] == ("ema_decay", "grad_accumulation")


def _toy(tmp_path, mode=Mode.TRAIN, **kw):
    ns = synthetic.api_namespace("frl_b200")
    problem = synthetic.make_toy_problem(ns, str(tmp_path), n_train=8, n_test=0)
    run_opts = ns.types.RunOpts(optim=OptimOpts(algo=OptAlgorithm.SGD), batchSize=4, nEpochs=1,
                                singleThreaded=True, mode=mode, **kw)
    return problem, run_opts


@pytest.mark.parametrize("bad", [True, -0.1, 1.0, 1, 2.5, float("nan"), float("inf"), "0.9"])
def test_bad_keyword_values_raise_before_any_rank_starts(tmp_path, monkeypatch, bad):
    monkeypatch.delenv("FRL_B200_EMA_DECAY", raising=False)
    problem, run_opts = _toy(tmp_path)
    with pytest.raises(ValueError, match="ema_decay=%s" % repr(bad).replace(".", r"\.")):
        next(Solver.solve(run_opts, problem, group_name=None, init_method="", ema_decay=bad))


@pytest.mark.parametrize("raw", ["abc", "", "1", "1.0", "-0.5", "nan"])
def test_bad_environment_values_raise_before_any_rank_starts(tmp_path, monkeypatch, raw):
    monkeypatch.setenv("FRL_B200_EMA_DECAY", raw)
    problem, run_opts = _toy(tmp_path)
    with pytest.raises(ValueError, match="EMA decay"):
        next(Solver.solve(run_opts, problem, group_name=None, init_method=""))


def test_eval_mode_ignores_the_setting(tmp_path, monkeypatch):
    monkeypatch.setenv("FRL_B200_EMA_DECAY", "abc")
    problem, run_opts = _toy(tmp_path, mode=Mode.EVAL, cpuonly=True)
    # no ValueError: EVAL never resolves the switch and stops at the missing device instead
    with pytest.raises(RuntimeError, match="no CPU path"):
        next(Solver.solve(run_opts, problem, group_name=None, init_method="", ema_decay=2.0))


# ---- where K11 runs ----------------------------------------------------------------------------

class EmaRecordingDouble(RecordingDouble):
    """``RecordingDouble`` plus K11 (``weight_ema``) as ``torch.lerp`` in fp32, logged as
    ``ema lo:hi xW``; ``end_step`` lines mark where the optimizer counted an update."""

    def weight_ema(self, ema, p, w):
        self.log.append("ema 0:%d x%g" % (ema.numel(), w))
        ema.lerp_(p[:ema.numel()], float(np.float32(w)))          # the kernel rounds w to fp32


def _run_ema(double, opt, clip, k, in_place, defer, skip, xs, decay, rank=0, world=1):
    """``test_pipeline_launches._run`` with a weight EMA (``decay`` > 0) and markers in the log:
    ``mb j`` where microbatch j starts, ``tail`` where a deferred step's run_tail() starts.  Returns
    (log, parameters, EMA vector or None, the torch AveragedModel's model parameters)."""
    net = _Net()
    arena = ParamArena(net.model_params(), [net.extra], device="cpu")
    optim_opts, la = OPTS[opt]
    optimizer = fused_optim.create_fused_optimizer(arena, optim_opts, la)
    end_step = optimizer.end_step

    def logged_end_step():
        double.log.append("end_step")
        end_step()

    optimizer.end_step = logged_end_step
    ema = WeightEMA(arena, net, decay) if decay else None
    kw = dict(bucket_cap_mb=0.0001, first_bucket_mb=0.00005) if world > 1 else {}
    pipe = grad_sync.GradBucketPipeline(arena, optimizer, world_size=world, clip_norm=clip, accumulation=k,
                                        ema=ema, **kw)
    pipe.mt_enabled = in_place
    double.pipe, double.log = pipe, []
    ref = AveragedModel(nn.Sequential(net.l0, net.l1, net.l2), multi_avg_fn=get_ema_multi_avg_fn(decay or 0.5),
                        use_buffers=True)
    for j, mb in enumerate(accumulation_plan(N_MB, k, B, N_ROWS)):
        double.log.append("mb %d" % j)
        pipe.set_microbatch(first=mb.first, closes=mb.closes, weight=mb.weight, group_scale=B / mb.group_rows)
        pipe.begin_step()
        net.loss(xs[j * B * world:(j + 1) * B * world][rank::world], skip).backward()
        if defer:
            pipe.finish_step(defer_tail=True)
            refs, tables = pipe.detach_grad_refs()
            double.log.append("tail")
            pipe.run_tail(refs, tables, pipe.last_ready)
        else:
            pipe.finish_step()
        if mb.closes:
            ref.update_parameters(nn.Sequential(net.l0, net.l1, net.l2))
    pipe.remove_hooks()
    return (double.log, [p.detach().clone() for p in net.parameters()],
            None if ema is None else ema.ema.clone(), [p.detach().clone() for p in ref.module.parameters()])


def _kernels(log):
    return [e for e in log if not (e.startswith(("mb ", "ema ")) or e in ("end_step", "tail"))]


def _check_positions(log, defer, n_updates, n_model):
    """Every end_step outside a capture is followed by exactly one K11 over the model range, every
    K11 follows an end_step, none is in a captured part, and there are ``n_updates`` of them."""
    captured = False
    emas = 0
    for i, e in enumerate(log):
        if e.startswith("mb "):
            captured = defer
        elif e == "tail":
            captured = False
        elif e.startswith("ema "):
            assert not captured, log
            assert log[i - 1] == "end_step", log
            assert e.startswith("ema 0:%d " % n_model), e
            emas += 1
        elif e == "end_step" and not captured:
            assert log[i + 1].startswith("ema "), log
    assert emas == n_updates, log


@pytest.fixture()
def double(monkeypatch):
    d = EmaRecordingDouble()
    monkeypatch.setattr(fused_optim, "KERNELS", d)
    monkeypatch.setattr(grad_sync, "KERNELS", d)
    monkeypatch.setattr(ema_mod, "KERNELS", d)
    monkeypatch.setattr(multi_tensor, "grad_usable_in_place", _in_place)
    return d


def _ema_by_slot(arena_like_net, vec):
    """The EMA vector cut into the model parameters' shapes (arena order = parameter order here)."""
    out, off = [], 0
    for p in arena_like_net:
        out.append(vec[off:off + p.numel()].view(p.shape))
        off = (off + p.numel() + 7) // 8 * 8
    return out


@pytest.mark.parametrize("in_place", [True, False], ids=["in-place", "arena"])
@pytest.mark.parametrize("k", [1, 3])
@pytest.mark.parametrize("skip", [False, True], ids=["all", "partial"])
@pytest.mark.parametrize("clip", [0.0, 0.05], ids=["noclip", "clip"])
@pytest.mark.parametrize("opt", list(OPTS))
def test_one_rank_k11_follows_every_update(double, opt, clip, skip, k, in_place):
    key = _key(opt, clip, skip, k, in_place)
    xs = torch.randn(N_ROWS, 7, generator=torch.Generator().manual_seed(11))
    n_updates = N_MB if k == 1 else 2                  # k = 3: a group of three, then a group of one
    for defer in (False, True):
        want = DEFERRED[key] * N_MB if (defer and key in DEFERRED) else EXPECTED[key] * (N_MB if k == 1 else 1)
        off_log, off_params, off_ema, _ = _run_ema(double, opt, clip, k, in_place, defer, skip, xs, 0.0)
        assert off_ema is None and not any(e.startswith("ema ") for e in off_log)
        assert _kernels(off_log) == want                # EMA off: today's launches
        log, params, vec, ref = _run_ema(double, opt, clip, k, in_place, defer, skip, xs, DECAY)
        assert _kernels(log) == want                    # the EMA adds K11 and nothing else
        n_model = double.pipe.arena.model_end
        _check_positions(log, defer, n_updates, n_model)
        if k == 3:                                      # nothing on the microbatches that do not close a group
            for j in (0, 1):
                seg = log[log.index("mb %d" % j):log.index("mb %d" % (j + 1))]
                assert not any(e.startswith("ema ") for e in seg), seg
        for a, b in zip(params, off_params):
            assert torch.equal(a, b)                    # training is untouched
        # against torch's AveragedModel over the same live weights (criterion parameter excluded);
        # a captured step with an unused parameter updates twice (see test_pipeline_launches) and
        # both are averaged as one, after the second
        for mine, theirs in zip(_ema_by_slot(list(_Net().model_params()), vec), ref):
            torch.testing.assert_close(mine, theirs, rtol=0, atol=0)


def _rank_main(rank, world, port, out_dir):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    d = EmaRecordingDouble()
    fused_optim.KERNELS = grad_sync.KERNELS = ema_mod.KERNELS = d
    multi_tensor.grad_usable_in_place = _in_place
    all_reduce = dist.all_reduce

    def logged_all_reduce(t, *args, **kw):
        d.log.append("all_reduce %s" % d._range(t, t.numel()))
        return all_reduce(t, *args, **kw)

    dist.all_reduce = logged_all_reduce
    xs = torch.randn(B * N_MB * world, 7, generator=torch.Generator().manual_seed(12))
    out = {}
    for opt, clip, k, in_place in _CONFIGS_2RANKS:
        key = _key(opt, clip, False, k, in_place)
        out[key] = [_run_ema(d, opt, clip, k, in_place, defer, False, xs, DECAY, rank, world)[:3]
                    for defer in (False, True)]
        out[key].append(d.pipe.arena.model_end)
    torch.save(out, os.path.join(out_dir, f"r{rank}.pt"))
    dist.destroy_process_group()


def test_two_rank_k11_follows_every_update(tmp_path):
    world = 2
    port = 37600 + (os.getpid() % 2000)
    mp.spawn(_rank_main, args=(world, port, str(tmp_path)), nprocs=world, join=True)
    r0, r1 = torch.load(tmp_path / "r0.pt"), torch.load(tmp_path / "r1.pt")
    assert sorted(r0) == sorted(EXPECTED_2RANKS)
    for key, want in EXPECTED_2RANKS.items():
        k1 = " k1 " in key
        n_model = r0[key][2]
        for defer, ((log0, p0, e0), (log1, p1, e1)) in enumerate(zip(r0[key][:2], r1[key][:2])):
            assert _kernels(log0) == _kernels(log1) == want * (N_MB if k1 else 1), key
            for log in (log0, log1):
                _check_positions(log, bool(defer), N_MB if k1 else 2, n_model)
            assert torch.equal(e0, e1), key                  # every rank keeps the same EMA
            for a, b in zip(p0, p1):
                assert torch.equal(a, b), key
        assert torch.equal(r0[key][0][2], r0[key][1][2]), key     # finish_step == the hand-over


def test_pipeline_refuses_ema_with_the_fused_nvls_step():
    net = _Net()
    arena = ParamArena(net.model_params(), [net.extra], device="cpu")
    opt = fused_optim.create_fused_optimizer(arena, OPTS["sgd"][0])

    class Link:                            # enough of a link for the constructor to pick K7
        pass

    with pytest.raises(ValueError, match="NVLS"):
        grad_sync.GradBucketPipeline(arena, opt, world_size=2, nvls_link=Link(), ema=WeightEMA(arena, net, 0.5))


# ---- WeightEMA ---------------------------------------------------------------------------------

class _BNNet(nn.Module):
    def __init__(self):
        super().__init__()
        torch.manual_seed(4)
        self.lin = nn.Linear(6, 5)
        self.bn = nn.BatchNorm1d(5)
        self.head = nn.Linear(5, 3)

    def forward(self, x):
        return self.head(self.bn(self.lin(x)))


@pytest.mark.parametrize("precision", [Precision.FP32, Precision.BF16])
def test_swap_restores_every_bit_also_when_the_block_raises(double, precision):
    net = _BNNet()
    arena = ParamArena(net.parameters(), device="cpu", precision=precision)
    ema = WeightEMA(arena, net, 0.9)
    ema.update()
    with torch.no_grad():
        arena.master.add_(torch.randn(arena.numel, generator=torch.Generator().manual_seed(1)))
        arena.refresh_shadow()
        net.bn.running_mean.add_(1.0)
        net.bn.num_batches_tracked.add_(3)
    ema.update()
    live = (arena.master.clone(), None if arena.lp is None else arena.lp.clone(),
            [b.clone() for b in net.buffers()])
    averaged = ema.ema.clone()
    with pytest.raises(KeyError):
        with ema.swapped():
            assert torch.equal(arena.master[:arena.model_end], averaged)
            if arena.lp is not None:
                assert torch.equal(arena.lp[:arena.model_end], averaged.to(torch.bfloat16))
            with pytest.raises(RuntimeError):
                ema.update()
            raise KeyError("split failed")
    assert torch.equal(arena.master, live[0])
    if arena.lp is not None:
        assert torch.equal(arena.lp, live[1])
    for b, want in zip(net.buffers(), live[2]):
        assert torch.equal(b, want)
    assert torch.equal(ema.ema, averaged)


def test_buffers_follow_averaged_model_and_state_round_trips(double):
    net = _BNNet()
    arena = ParamArena(net.parameters(), device="cpu")
    ema = WeightEMA(arena, net, 0.8)
    ref = AveragedModel(net, multi_avg_fn=get_ema_multi_avg_fn(0.8), use_buffers=True)
    g = torch.Generator().manual_seed(2)
    net.train()
    for _ in range(3):
        with torch.no_grad():
            net(torch.randn(16, 6, generator=g))            # moves the BatchNorm statistics
            for p in net.parameters():                      # arena views: the padding stays zero
                p.add_(torch.randn(p.shape, generator=g) * 0.1)
        ema.update()
        ref.update_parameters(net)
    blob = ema.state_dict()
    assert sorted(blob) == ["decay", "state_dict", "updates"] and blob["updates"] == 3
    assert list(blob["state_dict"]) == list(net.state_dict())
    for name, v in ref.module.state_dict().items():
        if v.is_floating_point():
            assert torch.equal(blob["state_dict"][name], v), name
    assert int(blob["state_dict"]["bn.num_batches_tracked"]) == 3      # copied, not averaged
    other = WeightEMA(arena, net, 0.8)
    other.load_state_dict(blob)
    assert other.updates == 3 and torch.equal(other.ema, ema.ema)
    for (_, _, a), (_, _, b) in zip(other.buffers, ema.buffers):
        assert torch.equal(a, b)


def test_weight_ema_rejects_bad_arguments_before_any_launch():
    from frl_b200 import _native
    lib = _native.lib()
    ok = 1 << 20                           # 16-byte aligned, never dereferenced: every call below fails a check
    before = lib.frl_launch_count()
    bad = [lib.frl_weight_ema(ok + 4, ok, 8, 0.5, None), lib.frl_weight_ema(ok, ok + 8, 8, 0.5, None),
           lib.frl_weight_ema(ok, ok, -1, 0.5, None), lib.frl_weight_ema(ok, ok, 8, -0.1, None),
           lib.frl_weight_ema(ok, ok, 8, 1.5, None), lib.frl_weight_ema(ok, ok, 8, math.nan, None),
           lib.frl_weight_ema(None, ok, 8, 0.5, None)]
    assert bad == [-2, -2, -1, -1, -1, -1, -1], bad
    assert lib.frl_launch_count() == before
    assert lib.frl_weight_ema(ok, ok, 0, 0.5, None) == 0                 # nothing to do, nothing launched
    assert lib.frl_launch_count() == before


# ---- checkpoint transport ----------------------------------------------------------------------

def _fractional(net, with_ema):
    state = {"state": {}, "param_groups": [{"lr": 0.1, "params": [0, 1]}]}
    if with_ema:
        state[EMA_STATE_KEY] = {"decay": 0.99, "updates": 7,
                                "state_dict": {k: v + 1 for k, v in net.state_dict().items()}}
    model_buf, optim_buf = io.BytesIO(), io.BytesIO()
    torch.save(net, model_buf)
    torch.save(state, optim_buf)
    sample = SingleSample(data=[torch.zeros(4)], target=[], meta={}, output=[torch.ones(2)], metric={})
    perf = {Split.TEST: FractionalEpochSplitPerformanceSummary(nSamples=1, losses={}, metrics={}, samples=[],
                                                                  worstSamples=[], testIO=[sample, sample])}
    return [FractionalPerformanceSummary(epoch=3, modelBuffer=model_buf.getvalue(),
                                         optimizerStateBuffer=optim_buf.getvalue(), performance=perf)]


def test_save_checkpoint_writes_the_ema_file_and_keeps_the_main_checkpoint(tmp_path):
    ns = synthetic.api_namespace("frl_b200")
    problem = synthetic.make_toy_problem(ns, str(tmp_path), n_train=8, n_test=0)
    run_opts = ns.types.RunOpts(optim=OptimOpts(algo=OptAlgorithm.SGD), batchSize=4, nEpochs=3)
    net = nn.Sequential(nn.Linear(4, 3), nn.BatchNorm1d(3))
    plain_dir, ema_dir = tmp_path / "plain", tmp_path / "ema"
    plain_dir.mkdir()
    ema_dir.mkdir()
    Solver._save_checkpoint(3, str(plain_dir), run_opts, problem, _fractional(net, False), "final_model.pth")
    Solver._save_checkpoint(3, str(ema_dir), run_opts, problem, _fractional(net, True), "final_model.pth")
    assert sorted(os.listdir(ema_dir)) == sorted(os.listdir(plain_dir) + ["final_model.pth.ema"])
    plain = torch.load(plain_dir / "final_model.pth", weights_only=False)
    main = torch.load(ema_dir / "final_model.pth", weights_only=False)
    assert list(main) == list(plain) and main["optimizer"] == plain["optimizer"] and main["epoch"] == 3
    for k, v in plain["state_dict"].items():
        assert torch.equal(main["state_dict"][k], v)
    blob = torch.load(ema_dir / "final_model.pth.ema", weights_only=False)
    assert list(blob) == ["epoch", "decay", "updates", "state_dict"]
    assert (blob["epoch"], blob["decay"], blob["updates"]) == (3, 0.99, 7)
    assert list(blob["state_dict"]) == list(main["state_dict"])
    for k, v in main["state_dict"].items():
        assert torch.equal(blob["state_dict"][k], v + 1)
    np.testing.assert_array_equal(torch.load(ema_dir / "final_model.pth.test_data")["test_input"][0].numpy(),
                                  torch.zeros(2, 4).numpy())


def test_resume_uses_the_ema_file_only_at_the_checkpoints_epoch(double, tmp_path):
    """A ``.checkpoint.pth.ema`` of another epoch than the checkpoint (a later run without an EMA
    overwrote the checkpoint, or a save stopped between the two files) is not resumed from."""
    from frl_b200.solver import load_ema_checkpoint
    net = _BNNet()
    arena = ParamArena(net.parameters(), device="cpu")
    saved = WeightEMA(arena, net, 0.9)
    saved.update()
    with torch.no_grad():
        for p in net.parameters():
            p.add_(1.0)
    saved.update()
    path = str(tmp_path / ".checkpoint.pth.ema")
    torch.save(dict({"epoch": 4}, **saved.state_dict()), path)
    assert not load_ema_checkpoint(WeightEMA(arena, net, 0.9), str(tmp_path / "missing.ema"), 4)
    stale = WeightEMA(arena, net, 0.9)
    assert not load_ema_checkpoint(stale, path, 5)
    assert stale.updates == 0 and torch.equal(stale.ema, arena.master[:arena.model_end])
    fresh = WeightEMA(arena, net, 0.9)
    assert load_ema_checkpoint(fresh, path, 4)
    assert fresh.updates == 2 and torch.equal(fresh.ema, saved.ema)
