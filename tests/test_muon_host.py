"""Muon (K14) on the host: the restatement against CPU ``torch.optim.Muon``, which slots Muon takes,
the switch and its refusals, the pipeline's launch sequence and the torch-format state dict, with
the kernels replaced by a CPU double."""
import os
import zlib

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn as nn

import frl_b200  # noqa: F401
from frl_b200 import _native, fused_optim, grad_sync, synthetic
from frl_b200.arena import ParamArena
from frl_b200.solver import Solver, SolverWorkerArgs, resolve_muon
from frl_b200.types import LayerAdaptation, Mode, OptAlgorithm, OptimizerState, OptimOpts
import muon_oracle as mo
from muon_oracle import MuonKernelDouble


@pytest.fixture()
def double(monkeypatch):
    d = MuonKernelDouble()
    monkeypatch.setattr(fused_optim, "KERNELS", d)
    monkeypatch.setattr(grad_sync, "KERNELS", d)
    return d


def _rel(a, b):
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


# ---- the restatement -----------------------------------------------------------------------------

@pytest.mark.parametrize("shape", [(24, 80), (80, 24), (1, 64), (48, 48)])
@pytest.mark.parametrize("kind", ["random", "lowrank", "zero"])
@pytest.mark.parametrize("nesterov", [True, False])
@pytest.mark.parametrize("adjust", ["match_rms_adamw", "original"])
def test_restatement_follows_torch_muon(shape, kind, nesterov, adjust):
    gen = torch.Generator().manual_seed(zlib.crc32(repr((shape, kind, nesterov, adjust)).encode()))
    p0 = torch.randn(shape, generator=gen)
    param = nn.Parameter(p0.clone())
    ref = torch.optim.Muon([param], lr=0.02, weight_decay=0.1, momentum=0.9, nesterov=nesterov, adjust_lr_fn=adjust)
    p, buf = p0.double(), torch.zeros(shape)
    for _ in range(3):
        if kind == "lowrank":
            g = torch.randn(shape[0], 2, generator=gen) @ torch.randn(2, shape[1], generator=gen)
        else:
            g = torch.randn(shape, generator=gen) * (kind == "random")
        param.grad = g.clone()
        ref.step()
        p, buf = mo.muon_step(p, g, buf, lr=0.02, wd=0.1, momentum=0.9, nesterov=nesterov, adjust_lr_fn=adjust)
    want = param.detach().double() - p0.double()
    got = p - p0.double()
    assert _rel(got, want) < 3e-2
    torch.testing.assert_close(buf, ref.state[param]["momentum_buffer"], rtol=1e-6, atol=1e-7)


# ---- which parameters ----------------------------------------------------------------------------

def _model_slots(model):
    arena = ParamArena(model.parameters(), device="cpu")
    opt = fused_optim.FusedMuon(arena, lr=0.01)
    return [tuple(p.shape) for p in opt.muon_params], opt


def test_muon_slots_of_the_benchmark_models(tmp_path):
    ns = synthetic.api_namespace("frl_b200")
    mlp = synthetic.make_mlp_problem(ns, str(tmp_path), n_train=8, width=4096).get_model()
    got, opt = _model_slots(mlp)
    assert sorted(got) == sorted([(4096, 4096)] * 3 + [(1000, 4096), (64, 4096)])
    # the Gram workspace: A and B, [m, m] bf16, per matrix
    assert opt.workspace_bytes == 2 * 2 * (3 * 4096 * 4096 + 1000 * 1000 + 64 * 64)
    resnet = synthetic.make_resnet_problem(ns, str(tmp_path), config="resnet18", image=32, n_train=4).get_model()
    got, _ = _model_slots(resnet)
    assert got == [tuple(p.shape) for p in resnet.parameters() if p.ndim == 2] and len(got) >= 1
    assert all(len(s) == 2 and s[1] == 512 for s in got)         # the task heads behind the trunk
    train, test = os.path.join(tmp_path, "train.txt"), os.path.join(tmp_path, "test.txt")
    synthetic.write_text_corpus(train, 16, 0)
    synthetic.write_text_corpus(test, 4, 1)
    text = synthetic.make_text_problem(ns, str(tmp_path), train, test).get_model()
    got, _ = _model_slots(text)
    assert sorted(got) == sorted([(256, 64), (128, 64), (256, 128)])


def test_workspace_is_sized_at_construction_and_shared_by_every_table(double):
    net = nn.Sequential(nn.Linear(30, 40), nn.Linear(40, 7))
    arena = ParamArena(net.parameters(), device="cpu")
    opt = fused_optim.FusedMuon(arena, lr=0.01)
    assert opt.workspace_bytes == _native.muon_plan_bytes(torch.tensor([[0, 0, 40, 30], [0, 0, 7, 40]]))[2] > 0
    from frl_b200.multi_tensor import GradSegTable
    grads = [torch.randn(s.shape) for s in arena.slots]
    for slots in (arena.slots, arena.slots[2:]):
        table = GradSegTable(slots, arena.device)
        for s in slots:
            table.point(s, grads[s.index].data_ptr(), torch.float32)
        table.upload()
        opt.begin_step(); opt.apply_table(table); opt.end_step()
    assert double.plans == 2 and opt._workspace.numel() * 4 >= opt.workspace_bytes


@pytest.mark.parametrize("bad", [dict(ns_steps=0), dict(ns_steps=100), dict(momentum=-0.5),
                                 dict(adjust_lr_fn="bogus")])
def test_bad_muon_group_is_refused_before_any_launch(double, bad):
    _, arena, opt = _stepped(double)
    before = arena.master.clone()
    opt.muon_group.update(bad)
    from frl_b200.multi_tensor import GradSegTable
    table = GradSegTable(arena.slots, arena.device)
    grads = [torch.randn(s.shape) for s in arena.slots]
    for s, g in zip(arena.slots, grads):
        table.point(s, g.data_ptr(), g.dtype)
    table.upload()
    double.calls.clear()
    with pytest.raises(_native.NativeLibraryError, match="Muon"):
        opt.apply_table(table)
    assert double.calls == [] and torch.equal(arena.master, before)


def test_muon_takes_the_models_matrices():
    net = nn.Sequential(nn.Embedding(10, 6), nn.Linear(6, 8), nn.BatchNorm1d(8), nn.Conv1d(8, 4, 3), nn.Linear(4, 2))
    crit = nn.Linear(3, 3)                                 # criterion parameters stay with Adam
    arena = ParamArena(net.parameters(), crit.parameters(), device="cpu")
    opt = fused_optim.FusedMuon(arena, lr=0.01)
    want = [p for p in net.parameters() if p.ndim == 2]
    assert [id(p) for p in opt.muon_params] == [id(p) for p in want]
    assert len(opt.adam_params) == len(arena.all_params) - len(want)
    assert all(id(p) not in {id(q) for q in want} for p in opt.adam_params)
    assert opt.param_groups[0]["params"] == opt.muon_params and opt.param_groups[1]["params"] == opt.adam_params
    assert opt.needs_whole_tensors


def test_muon_group_hyper_parameters():
    arena = ParamArena(nn.Linear(4, 3).parameters(), device="cpu")
    opts = OptimOpts(algo=OptAlgorithm.ADAM, lr=0.03, weightDecay=0.01, momentum=0.8, epsilon=1e-6)
    opt = fused_optim.create_fused_optimizer(arena, opts, muon=True)
    m, a = opt.param_groups
    assert set(m) - {"params"} == set(torch.optim.Muon([nn.Parameter(torch.zeros(2, 2))]).defaults)
    assert (m["lr"], m["weight_decay"], m["momentum"], m["nesterov"], m["ns_steps"], m["eps"], m["adjust_lr_fn"]) == \
        (0.03, 0.01, 0.8, True, 5, 1e-7, "match_rms_adamw")
    assert m["ns_coefficients"] == (3.4445, -4.7750, 2.0315)
    assert (a["lr"], a["weight_decay"], a["eps"], a["amsgrad"]) == (0.03, 0.01, 1e-6, False)
    assert type(fused_optim.create_fused_optimizer(arena, opts)) is fused_optim.FusedAdam


# ---- the switch ----------------------------------------------------------------------------------

def test_resolution(monkeypatch):
    monkeypatch.delenv("FRL_B200_MUON", raising=False)
    assert resolve_muon() is False
    monkeypatch.setenv("FRL_B200_MUON", "1")
    assert resolve_muon() is True and resolve_muon(False) is False
    for bad in ("yes", "2", "true"):
        monkeypatch.setenv("FRL_B200_MUON", bad)
        with pytest.raises(ValueError, match="FRL_B200_MUON"):
            resolve_muon()


def test_worker_args_field():
    assert SolverWorkerArgs._field_defaults["muon"] is False
    f = SolverWorkerArgs._fields
    assert f.index("muon") < f.index("optimizer_state") and f[-2:] == ("ema_decay", "grad_accumulation")


def _problem(tmp_path, opts, **kw):
    ns = synthetic.api_namespace("frl_b200")
    problem = synthetic.make_toy_problem(ns, str(tmp_path), n_train=8, n_test=0)
    return problem, ns.types.RunOpts(optim=opts, batchSize=4, nEpochs=1, singleThreaded=True, **kw)


@pytest.mark.parametrize("algo,amsgrad,la,st,af", [
    (OptAlgorithm.SGD, False, LayerAdaptation.NONE, OptimizerState.FP32, False),
    (OptAlgorithm.ADAM, True, LayerAdaptation.NONE, OptimizerState.FP32, False),
    (OptAlgorithm.ADAM, False, LayerAdaptation.LAMB, OptimizerState.FP32, False),
    (OptAlgorithm.ADAM, False, LayerAdaptation.NONE, OptimizerState.Q8, False),
    (OptAlgorithm.ADAM, False, LayerAdaptation.NONE, OptimizerState.FP32, True)])
def test_refused_combinations_name_the_values(tmp_path, algo, amsgrad, la, st, af):
    opts = OptimOpts(algo=algo, amsgrad=amsgrad)
    with pytest.raises(ValueError, match="muon") as e:
        fused_optim.check_muon(opts, la, st, af, True)
    assert algo.value in str(e.value) and la.value in str(e.value) and st.value in str(e.value)
    fused_optim.check_muon(opts, la, st, af, False)
    problem, run_opts = _problem(tmp_path, opts)
    with pytest.raises(ValueError, match="muon"):               # before any rank or device is touched
        next(Solver.solve(run_opts, problem, group_name=None, init_method="", layer_adaptation=la,
                          optimizer_state=st, adafactor=False, muon=True) if not af else
             Solver.solve(run_opts, problem, group_name=None, init_method="", adafactor=True, muon=True))


def test_eval_ignores_the_option(tmp_path, monkeypatch):
    monkeypatch.setenv("FRL_B200_MUON", "bogus")
    problem, run_opts = _problem(tmp_path, OptimOpts(algo=OptAlgorithm.SGD), mode=Mode.EVAL, cpuonly=True)
    with pytest.raises(RuntimeError, match="H100"):
        next(Solver.solve(run_opts, problem, group_name=None, init_method="", muon=True))


# ---- the pipeline --------------------------------------------------------------------------------

class _Net(nn.Module):
    def __init__(self):
        super().__init__()
        torch.manual_seed(3)
        self.l0, self.l1 = nn.Linear(7, 6), nn.Linear(6, 2)

    def loss(self, x):
        return self.l1(self.l0(x).relu()).square().mean()


@pytest.mark.parametrize("clip", [0.0, 0.5])
@pytest.mark.parametrize("k", [1, 2])
def test_one_adam_launch_and_one_muon_launch_after_backward(double, clip, k):
    """The launches, and the weights against torch.optim.Muon + torch.optim.Adam fed the same
    (clipped, microbatch-mean) gradient: the double restates K14, so the gap is the restatement's."""
    net = _Net()
    ref = _Net()
    arena = ParamArena(net.parameters(), device="cpu")
    opt = fused_optim.create_fused_optimizer(arena, OptimOpts(algo=OptAlgorithm.ADAM, lr=0.02, momentum=0.9),
                                             muon=True)
    pipe = grad_sync.GradBucketPipeline(arena, opt, world_size=1, clip_norm=clip, accumulation=k)
    rp = list(ref.parameters())
    ref_m = torch.optim.Muon([rp[0], rp[2]], lr=0.02, weight_decay=0.0, momentum=0.9, adjust_lr_fn="match_rms_adamw")
    ref_a = torch.optim.Adam([rp[1], rp[3]], lr=0.02)
    xs = torch.randn(4 * k, 5, 7, generator=torch.Generator().manual_seed(1))
    for step in range(4):
        double.calls.clear()
        for j in range(k):
            pipe.set_microbatch(first=j == 0, closes=j == k - 1, weight=1.0, group_scale=1.0 / k)
            pipe.begin_step()
            net.loss(xs[(step % 2) * k + j]).backward()
            pipe.finish_step()
        kinds = [c for c in double.calls if c[0] in ("adam_mt", "muon_mt", "adam")]
        assert kinds == [("adam_mt", (1, 3), clip > 0), ("muon_mt", (0, 2), clip > 0)], double.calls
        ref_m.zero_grad(); ref_a.zero_grad()
        (sum(ref.loss(xs[(step % 2) * k + j]) for j in range(k)) / k).backward()
        if clip:
            torch.nn.utils.clip_grad_norm_(rp, clip)
        ref_m.step(); ref_a.step()
    pipe.remove_hooks()
    for i in (1, 3):                                        # Adam: fp32 arithmetic on both sides
        torch.testing.assert_close(arena.master_view(arena.slots[i]), rp[i].detach(), rtol=1e-5, atol=1e-6)
    for i in (0, 2):                                        # Muon: the restatement's bf16 rounding
        p0 = list(_Net().parameters())[i].detach()
        assert _rel(arena.master_view(arena.slots[i]) - p0, rp[i].detach() - p0) < 3e-2


# ---- state dict ----------------------------------------------------------------------------------

def _stepped(double, seed=0):
    torch.manual_seed(seed)
    net = nn.Sequential(nn.Linear(5, 4), nn.Linear(4, 3))
    arena = ParamArena(net.parameters(), device="cpu")
    opt = fused_optim.FusedMuon(arena, lr=0.01, weight_decay=0.01)
    from frl_b200.multi_tensor import GradSegTable
    table = GradSegTable(arena.slots, arena.device)
    grads = [torch.randn(s.shape) for s in arena.slots]
    for s, g in zip(arena.slots, grads):
        table.point(s, g.data_ptr(), g.dtype)
    table.upload()
    opt.begin_step(); opt.apply_table(table); opt.end_step()
    return net, arena, opt


def test_state_dict_round_trips_through_torch_muon_and_adam(double):
    net, arena, opt = _stepped(double)
    sd = opt.state_dict()
    assert [g["params"] for g in sd["param_groups"]] == [[0, 1], [2, 3]]
    assert set(sd["state"][0]) == {"momentum_buffer"} and set(sd["state"][2]) == {"step", "exp_avg", "exp_avg_sq"}
    muon_sd, adam_sd = fused_optim.split_muon_state_dict(sd)
    w = [p for p in net.parameters()]
    m = torch.optim.Muon([w[0], w[2]], lr=0.5)
    a = torch.optim.Adam([w[1], w[3]], lr=0.5)
    m.load_state_dict(muon_sd)
    a.load_state_dict(adam_sd)
    assert m.param_groups[0]["lr"] == 0.01 and a.param_groups[0]["lr"] == 0.01
    torch.testing.assert_close(m.state[w[0]]["momentum_buffer"], sd["state"][0]["momentum_buffer"])
    torch.testing.assert_close(a.state[w[3]]["exp_avg_sq"], sd["state"][3]["exp_avg_sq"])
    _, _, other = _stepped(double, seed=1)
    other.load_state_dict(fused_optim.join_muon_state_dict(m.state_dict(), a.state_dict()))
    assert torch.equal(other._state("exp_avg"), opt._state("exp_avg"))
    assert torch.equal(other._state("exp_avg_sq")[arena.slots[1].offset:arena.slots[1].end],
                       opt._state("exp_avg_sq")[arena.slots[1].offset:arena.slots[1].end])
    assert other._steps == 1


def test_adam_only_state_dict_is_refused(double):
    _, arena, opt = _stepped(double)
    adam = fused_optim.FusedAdam(arena, lr=0.01)
    with pytest.raises(ValueError, match="two param groups"):
        opt.load_state_dict(adam.state_dict())
    with pytest.raises(ValueError, match="groups"):
        adam.load_state_dict(opt.state_dict())


# ---- world_size 2 over gloo ----------------------------------------------------------------------

def _gloo_net(seed):
    torch.manual_seed(seed)
    return nn.Sequential(nn.Linear(7, 30), nn.ReLU(), nn.Linear(30, 5), nn.ReLU(), nn.Linear(5, 1))


def _gloo_opt(net):
    arena = ParamArena(net.parameters(), device="cpu")
    return arena, fused_optim.create_fused_optimizer(arena, OptimOpts(algo=OptAlgorithm.ADAM, lr=0.01,
                                                                      weightDecay=1e-2, momentum=0.9), muon=True)


def _rank_main(rank, world, port, clip, out_dir):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    d = MuonKernelDouble()
    fused_optim.KERNELS = d
    grad_sync.KERNELS = d
    net = _gloo_net(10 + rank)
    arena, opt = _gloo_opt(net)
    pipe = grad_sync.GradBucketPipeline(arena, opt, world_size=world, clip_norm=clip,
                                        bucket_cap_mb=0.001, first_bucket_mb=0.0005,
                                        eager_update=True, nvls_link=object())
    assert not pipe.eager and pipe.nvls is None and len(pipe.buckets) > 1
    pipe.broadcast_parameters(src=0)
    g = torch.Generator().manual_seed(99)
    for _ in range(3):
        x = torch.randn(8 * world, 7, generator=g)
        d.calls.clear()
        pipe.begin_step()
        net(x[rank::world]).square().mean().backward()
        pipe.finish_step()
        assert [c[0] for c in d.calls if c[0] in ("adam_mt", "muon_mt")] == ["adam_mt", "muon_mt"]
    torch.save([p.detach().clone() for p in net.parameters()], os.path.join(out_dir, f"r{rank}.pt"))
    dist.destroy_process_group()


def _single_rank(world, clip):
    d = MuonKernelDouble()
    net = _gloo_net(10)
    saved = fused_optim.KERNELS, grad_sync.KERNELS
    fused_optim.KERNELS = grad_sync.KERNELS = d
    try:
        arena, opt = _gloo_opt(net)
        pipe = grad_sync.GradBucketPipeline(arena, opt, clip_norm=clip)
        g = torch.Generator().manual_seed(99)
        for _ in range(3):
            x = torch.randn(8 * world, 7, generator=g)
            pipe.begin_step(); net(x).square().mean().backward(); pipe.finish_step()
    finally:
        fused_optim.KERNELS, grad_sync.KERNELS = saved
    return [p.detach().clone() for p in net.parameters()]


@pytest.mark.parametrize("clip", [0.0, 0.01])
def test_two_ranks_at_half_batch_equal_one_rank_at_full_batch(tmp_path, clip):
    """Every rank runs the same Newton-Schulz on the same all-reduced gradient: the ranks agree bit
    for bit, and with one rank at the full batch up to the order of the gradient sums (the bf16
    rounding inside NS can turn a last-bit difference into one bf16 step, so the Muon matrices are
    held to the restatement's relative bound)."""
    world = 2
    port = 37500 + (os.getpid() % 2000)
    mp.spawn(_rank_main, args=(world, port, clip, str(tmp_path)), nprocs=world, join=True)
    r0, r1 = torch.load(tmp_path / "r0.pt"), torch.load(tmp_path / "r1.pt")
    for a, b in zip(r0, r1):
        assert torch.equal(a, b)
    p0 = [p.detach() for p in _gloo_net(10).parameters()]
    for a, b, q in zip(r0, _single_rank(world, clip), p0):
        if a.ndim == 2:
            assert _rel(a - q, b - q) < 3e-2
        else:
            np.testing.assert_allclose(a.numpy(), b.numpy(), rtol=1e-5, atol=1e-6)
