"""Param groups on the host: hook and switch resolution and ``FRL_B200_NO_DECAY_1D``, the canonical
order, every refusal (from the factory and from ``Solver.solve`` before a rank starts), the worker-args
position, the per-group ``dyn`` rows, the state dict against ``torch.optim`` built with the same groups
in both directions, the scheduler's per-group lr, and the launch sequence on recording fakes."""
import types

import numpy as np
import pytest
import torch
import torch.nn as nn

import frl_b200  # noqa: F401
from frl_b200 import _native, fused_optim, grad_sync, solver, synthetic
from frl_b200.arena import ParamArena
from frl_b200.lr_scheduler import WarmupMultiStepLR
from frl_b200.solver import SolverWorkerArgs, resolve_no_decay_1d
from frl_b200.types import LayerAdaptation, MasterWeights, OptAlgorithm, OptimizerState, OptimOpts, Precision, RunOpts

SGD = OptimOpts(algo=OptAlgorithm.SGD, lr=1e-2, momentum=0.9, weightDecay=0.1)
ADAM = OptimOpts(algo=OptAlgorithm.ADAM, lr=1e-3, weightDecay=0.1)


def _model(seed=0):
    torch.manual_seed(seed)
    net = nn.Sequential(nn.Linear(6, 5), nn.LayerNorm(5), nn.ReLU(), nn.Linear(5, 3))
    extra = nn.Parameter(torch.tensor([0.5, -1.0]))
    return net, extra


def _arena(net, extra, precision=Precision.FP32, master=MasterWeights.FP32):
    return ParamArena(list(net.parameters()), [extra], device="cpu", precision=precision, master_weights=master)


def _crit(extra):
    m = nn.Module()
    m.extra = extra
    return m


# ---- resolution ------------------------------------------------------------------------------------

def test_no_decay_1d_and_the_environment_variable(monkeypatch):
    monkeypatch.delenv("FRL_B200_NO_DECAY_1D", raising=False)
    assert resolve_no_decay_1d() is False
    assert resolve_no_decay_1d(True) is True and resolve_no_decay_1d(False) is False
    monkeypatch.setenv("FRL_B200_NO_DECAY_1D", "1")
    assert resolve_no_decay_1d() is True and resolve_no_decay_1d(False) is False
    for bad in ("2", "true", "", "yes"):
        monkeypatch.setenv("FRL_B200_NO_DECAY_1D", bad)
        with pytest.raises(ValueError, match="FRL_B200_NO_DECAY_1D"):
            resolve_no_decay_1d()


def test_canonical_order_hook_groups_then_the_default_group():
    net, extra = _model()
    w0, b0, ln_w, ln_b, w1, b1 = net.parameters()
    groups = fused_optim.resolve_param_groups(net, [extra], [{"params": [w1], "lr": 0.5},
                                                             {"params": [b0, ln_b], "weight_decay": 0}])
    assert [[id(p) for p in g["params"]] for g in groups] == [
        [id(w1)], [id(b0), id(ln_b)], [id(w0), id(ln_w), id(b1), id(extra)]]
    assert groups[0] == {"params": [w1], "lr": 0.5} and groups[1]["weight_decay"] == 0.0
    assert set(groups[2]) == {"params"}                    # OptimOpts' lr / weightDecay
    # a hook covering every model parameter: the default group still holds the criterion parameters
    full = fused_optim.resolve_param_groups(net, [extra], [{"params": list(net.parameters())}])
    assert [len(g["params"]) for g in full] == [6, 1]
    assert fused_optim.resolve_param_groups(net, [extra], None) is None


def test_the_switch_is_the_ndim_le_1_hook():
    net, extra = _model()
    via_switch = solver.problem_param_groups(types.SimpleNamespace(), net, _crit(extra), True)
    hook = [{"params": [p for p in net.parameters() if p.ndim <= 1], "weight_decay": 0.0}]
    via_hook = fused_optim.resolve_param_groups(net, [extra], hook)
    assert [[id(p) for p in g["params"]] for g in via_switch] == [[id(p) for p in g["params"]] for g in via_hook]
    assert [{k: v for k, v in g.items() if k != "params"} for g in via_switch] == [{"weight_decay": 0.0}, {}]
    flat = nn.Sequential(nn.Linear(4, 4, bias=False))        # nothing with ndim <= 1: the group is omitted
    assert fused_optim.no_decay_1d_groups(flat) == []
    assert len(solver.problem_param_groups(types.SimpleNamespace(), flat, nn.Module(), True)) == 1


@pytest.mark.parametrize("bad,msg", [
    (lambda net, extra: [{"params": [net[0].weight], "momentum": 0.5}], "key 'momentum'"),
    (lambda net, extra: [{"params": [net[0].weight], "betas": (0.9, 0.9)}], "key 'betas'"),
    (lambda net, extra: [{"params": []}], "param group 0 is empty"),
    (lambda net, extra: [{"params": [net[0].weight, net[0].weight]}], "already holds"),
    (lambda net, extra: [{"params": [net[0].weight]}, {"params": [net[0].weight]}], "already holds"),
    (lambda net, extra: [{"params": [nn.Parameter(torch.zeros(2))]}], "not in model.parameters"),
    (lambda net, extra: [{"params": [extra]}], "criterion parameter"),
    (lambda net, extra: [{"lr": 0.1}], "'params' key"),
])
def test_malformed_groups_are_refused(bad, msg):
    net, extra = _model()
    with pytest.raises(ValueError, match=msg):
        fused_optim.resolve_param_groups(net, [extra], bad(net, extra))


def test_hook_and_switch_together_are_refused():
    net, extra = _model()

    class P:
        def get_param_groups(self, model):
            return [{"params": [model[0].weight], "lr": 0.1}]
    with pytest.raises(ValueError, match="no_decay_1d cannot be combined"):
        solver.problem_param_groups(P(), net, _crit(extra), True)
    assert len(solver.problem_param_groups(P(), net, _crit(extra), False)) == 2


REFUSED = [   # (opts, layer adaptation, optimizer state, adafactor, muon, message)
    (SGD, LayerAdaptation.LARS, OptimizerState.FP32, False, False, "layer adaptation lars"),
    (ADAM, LayerAdaptation.LAMB, OptimizerState.FP32, False, False, "layer adaptation lamb"),
    (ADAM, LayerAdaptation.NONE, OptimizerState.Q8, False, False, "optimizer state 8bit"),
    (ADAM, LayerAdaptation.NONE, OptimizerState.FP32, True, False, "adafactor"),
    (ADAM, LayerAdaptation.NONE, OptimizerState.FP32, False, True, "muon"),
]


@pytest.mark.parametrize("opts,la,state,adafactor,muon,msg", REFUSED)
def test_refusals_in_the_factory(opts, la, state, adafactor, muon, msg):
    net, extra = _model()
    arena = _arena(net, extra)
    groups = fused_optim.resolve_param_groups(net, [extra], fused_optim.no_decay_1d_groups(net))
    with pytest.raises(ValueError, match="param groups .* cannot be combined with %s" % msg):
        fused_optim.create_fused_optimizer(arena, opts, la, state, adafactor, muon, param_groups=groups)


@pytest.mark.parametrize("opts,la,state,adafactor,muon,msg", REFUSED)
def test_refusals_before_a_rank_starts(tmp_path, opts, la, state, adafactor, muon, msg):
    ns = synthetic.api_namespace("frl_b200")
    problem = synthetic.make_toy_problem(ns, str(tmp_path), n_train=16, n_test=8)
    run_opts = RunOpts(optim=opts, batchSize=8, nEpochs=1, cpuonly=True)
    with pytest.raises(ValueError, match="param groups .* cannot be combined with %s" % msg):
        next(iter(solver.Solver.solve(run_opts, problem, group_name="g", init_method="", layer_adaptation=la,
                                      optimizer_state=state, adafactor=adafactor, muon=muon, no_decay_1d=True)))


def test_a_malformed_hook_is_refused_before_a_rank_starts_and_the_rng_is_kept(tmp_path):
    ns = synthetic.api_namespace("frl_b200")
    problem = synthetic.make_toy_problem(ns, str(tmp_path), n_train=16, n_test=8)
    problem.__class__ = type("Hooked", (type(problem),),
                             {"get_param_groups": lambda self, model: [{"params": [], "lr": 0.1}]})
    run_opts = RunOpts(optim=SGD, batchSize=8, nEpochs=1, cpuonly=True)
    torch.manual_seed(3)
    before = torch.random.get_rng_state()
    with pytest.raises(ValueError, match="param group 0 is empty"):
        next(iter(solver.Solver.solve(run_opts, problem, group_name="g", init_method="")))
    assert torch.equal(torch.random.get_rng_state(), before)
    problem.__class__ = type("Hooked", (type(problem),),
                             {"get_param_groups": lambda self, model: [{"params": [next(model.parameters())],
                                                                        "lr": 0.1}]})
    with pytest.raises(RuntimeError, match="H100 GPUs only"):             # the first thing after the checks
        next(iter(solver.Solver.solve(run_opts, problem, group_name="g", init_method="", no_decay_1d=False)))
    with pytest.raises(RuntimeError, match="H100 GPUs only"):
        next(iter(solver.Solver.solve(run_opts, synthetic.make_toy_problem(ns, str(tmp_path), n_train=16,
                                                                           n_test=8),
                                      group_name="g", init_method="", no_decay_1d=True)))


def test_worker_args_field():
    f = SolverWorkerArgs._fields
    assert f.index("no_decay_1d") == f.index("layer_adaptation") + 1 == f.index("lion") - 1
    assert f.index("lion") == f.index("muon") - 1 and f.index("adamw") == f.index("muon") + 1
    assert f.index("channels_last") == f.index("adamw") + 1 and f.index("master_weights") == f.index("channels_last") + 1
    assert f[-5:] == ("master_weights", "optimizer_state", "adafactor", "ema_decay", "grad_accumulation")
    assert SolverWorkerArgs._field_defaults["no_decay_1d"] is None


# ---- dyn rows, state dict, scheduler -----------------------------------------------------------------

def _grouped(kind, sr=False, precision=Precision.FP32):
    net, extra = _model()
    w0 = net[0].weight
    hook = [{"params": [w0], "lr": 0.5 * (1e-2 if kind != "adam" else 1e-3)},
            {"params": [p for p in net.parameters() if p.ndim <= 1], "weight_decay": 0.0}]
    groups = fused_optim.resolve_param_groups(net, [extra], hook)
    arena = _arena(net, extra, Precision.BF16 if sr else precision, MasterWeights.BF16 if sr else MasterWeights.FP32)
    if kind == "sgd":
        opt = fused_optim.FusedSGD(arena, lr=1e-2, momentum=0.9, weight_decay=0.1, param_groups=groups)
    elif kind == "lion":
        opt = fused_optim.FusedLion(arena, lr=1e-2, betas=(0.9, 0.99), weight_decay=0.1, param_groups=groups)
    elif kind == "rmsprop":
        opt = fused_optim.FusedRMSprop(arena, lr=1e-2, momentum=0.9, weight_decay=0.1, param_groups=groups)
    else:
        opt = fused_optim.FusedAdam(arena, lr=1e-3, weight_decay=0.1, adamw=(kind == "adamw"), param_groups=groups)
    return net, extra, groups, opt


@pytest.mark.parametrize("kind", ["sgd", "adam", "adamw", "rmsprop", "lion"])
def test_dyn_rows_per_group(kind):
    _, _, groups, opt = _grouped(kind)
    assert opt.grouped and opt.needs_whole_tensors and opt._dyn.shape == (3, _native.GROUP_DYN_COLS)
    opt._steps = 4
    opt.refresh_dynamic_scalars()
    rows = opt._dyn.numpy()
    for gi, h in enumerate(opt.param_groups):
        lr, wd = float(h["lr"]), float(h["weight_decay"])
        if kind in ("adam", "adamw"):
            bc1, bc2 = 1 - 0.9 ** 5, 1 - 0.999 ** 5
            want = [-(lr / bc1), bc2 ** 0.5, np.float32(1 - lr * wd) if kind == "adamw" else 0.0]
        elif kind == "lion":
            want = [lr, np.float32(1 - lr * wd), 0.0]
        else:
            want = [lr, 0.0, 0.0]
        assert np.array_equal(rows[gi, :3], np.float32(want)), (gi, rows[gi])
        assert rows[gi].view(np.uint32)[3] == 5                      # the update count, uint32 bits
        assert rows[gi, 4] == np.float32(wd) and not rows[gi, 5:].any()
        # columns 0-3 are the rule's ungrouped dyn for this group's lr / wd
        assert np.array_equal(rows[gi, :len(opt._dyn_row(h))], np.float32(opt._dyn_row(h)))
    assert [h["lr"] for h in opt.param_groups][1:] == [opt.defaults["lr"]] * 2
    assert opt.param_groups[1]["weight_decay"] == 0.0 and opt.param_groups[0]["weight_decay"] == 0.1


def test_one_group_keeps_todays_optimizer():
    net, extra = _model()
    arena = _arena(net, extra)
    opt = fused_optim.create_fused_optimizer(arena, SGD)
    assert not opt.grouped and not opt.needs_whole_tensors and opt._dyn is None
    sd = opt.state_dict()
    assert sd["param_groups"][0]["params"] == list(range(len(arena.all_params)))


TORCH = {
    "sgd": lambda g: torch.optim.SGD(g, lr=1e-2, momentum=0.9, weight_decay=0.1),
    "adam": lambda g: torch.optim.Adam(g, lr=1e-3, weight_decay=0.1),
    "adamw": lambda g: torch.optim.AdamW(g, lr=1e-3, weight_decay=0.1),
    "rmsprop": lambda g: torch.optim.RMSprop(g, lr=1e-2, momentum=0.9, weight_decay=0.1),
}


@pytest.mark.parametrize("kind", sorted(TORCH))
def test_state_dict_against_torch_optim_both_directions(kind):
    net, extra, groups, opt = _grouped(kind)
    ref_net, ref_extra = _model()
    ref_params = dict(zip(map(id, list(net.parameters()) + [extra]), list(ref_net.parameters()) + [ref_extra]))
    ref = TORCH[kind]([dict(g, params=[ref_params[id(p)] for p in g["params"]]) for g in groups])
    for p in ref_params.values():
        p.grad = torch.randn_like(p)
    ref.step()
    theirs = ref.state_dict()
    opt.load_state_dict(theirs)
    mine = opt.state_dict()
    assert [{k: v for k, v in g.items()} for g in mine["param_groups"]] == theirs["param_groups"]
    assert sorted(mine["state"]) == sorted(theirs["state"])
    for i, entry in theirs["state"].items():
        assert set(mine["state"][i]) == set(entry)
        for k, v in entry.items():
            assert torch.equal(mine["state"][i][k].float(), v.float()), (i, k)
    ref2 = TORCH[kind]([dict(g, params=[ref_params[id(p)] for p in g["params"]]) for g in groups])
    ref2.load_state_dict(mine)                                        # and back into torch.optim
    assert ref2.state_dict()["param_groups"] == theirs["param_groups"]
    bad = dict(theirs, param_groups=theirs["param_groups"][:2])
    with pytest.raises(ValueError, match=r"2 param groups of \[1, 4\] params; this optimizer has 3 of \[1, 4, 2\]"):
        opt.load_state_dict(bad)


def test_lion_state_dict_against_ref_lion():
    from lion_oracle import RefLion
    net, extra, groups, opt = _grouped("lion")
    ref_net, ref_extra = _model()
    ref_params = dict(zip(map(id, list(net.parameters()) + [extra]), list(ref_net.parameters()) + [ref_extra]))
    ref = RefLion([dict(g, params=[ref_params[id(p)] for p in g["params"]]) for g in groups], lr=1e-2,
                  betas=(0.9, 0.99), weight_decay=0.1)
    for p in ref_params.values():
        p.grad = torch.randn_like(p)
    ref.step()
    opt.load_state_dict(ref.state_dict())
    mine = opt.state_dict()
    assert [g["params"] for g in mine["param_groups"]] == [[0], [1, 2, 3, 4], [5, 6]]
    assert [g["lr"] for g in mine["param_groups"]] == [5e-3, 1e-2, 1e-2]
    ref.load_state_dict(mine)


def test_bf16_master_keys_live_in_the_first_group():
    _, _, _, opt = _grouped("sgd", sr=True)
    sd = opt.state_dict()
    assert "sr_seed" in sd["param_groups"][0] and "sr_updates" in sd["param_groups"][0]
    assert all("sr_seed" not in g for g in sd["param_groups"][1:])


def test_scheduler_sets_each_group_as_torch_does():
    net, extra, groups, opt = _grouped("sgd")
    ref_net, ref_extra = _model()
    ref_params = dict(zip(map(id, list(net.parameters()) + [extra]), list(ref_net.parameters()) + [ref_extra]))
    ref = TORCH["sgd"]([dict(g, params=[ref_params[id(p)] for p in g["params"]]) for g in groups])
    mine = WarmupMultiStepLR(opt, [3, 6], gamma=0.1, warmup_factor=1e-3, warmup_iters=5)
    theirs = WarmupMultiStepLR(ref, [3, 6], gamma=0.1, warmup_factor=1e-3, warmup_iters=5)
    for _ in range(8):
        assert [g["lr"] for g in opt.param_groups] == [g["lr"] for g in ref.param_groups]
        mine.step()
        theirs.step()
    opt.refresh_dynamic_scalars() if opt._dyn is not None else None
    assert np.array_equal(opt._dyn.numpy()[:, 0], np.float32([g["lr"] for g in ref.param_groups]))


# ---- the launch sequence ----------------------------------------------------------------------------

class _Recorder:
    """``_native`` with the update entry points recorded instead of launched."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        real = getattr(_native, name)
        if not callable(real) or name[0].isupper() or name in ("dtype_code",):
            return real

        def rec(*a, **kw):
            self.calls.append((name, a, kw))
        return rec


def test_one_grouped_table_launch_after_backward_and_k12_with_its_group_row(monkeypatch):
    rec = _Recorder()
    for mod in (fused_optim, grad_sync):
        monkeypatch.setattr(mod, "KERNELS", rec)
    _, _, _, opt = _grouped("sgd", precision=Precision.BF16)
    pipe = grad_sync.GradBucketPipeline(opt.arena, opt, eager_update=True)
    assert pipe.whole_tensors and not pipe.eager
    slot = next(s for s in opt.arena.slots if s.param is opt.param_groups[2]["params"][0])   # net[3].weight
    pipe.fused_dw_update = True
    pipe.begin_step()
    pipe.update_in_dw_gemm(slot, None, None, None)
    name, _, kw = rec.calls[-1]
    assert name == "dw_gemm_sgd" and kw["lr"] == 1e-2 and kw["wd"] == 0.1
    assert kw["dyn"].data_ptr() == opt._dyn[2].data_ptr() != opt._dyn[0].data_ptr()
    for s in opt.arena.slots:
        pipe.mark_ready(s)
    pipe.finish_step()
    launches = [c for c in rec.calls if c[0].startswith(("sgd", "dw_gemm"))]
    assert [c[0] for c in launches] == ["dw_gemm_sgd", "sgd_momentum_mt_grouped"]
    _, args, kw = launches[-1]
    table, groups = args[3], args[4]
    assert [s.index for s in table.slots] == [s.index for s in opt.arena.slots if s is not slot]   # K12's slot
    assert groups.seg_group.tolist() == [opt._group_of[id(s.param)] for s in table.slots]
    assert groups.seg_flags.tolist() == [_native.LW_CLIPPED if s.is_model else 0 for s in table.slots]
    assert opt._steps == 1


def test_a_failed_capture_keeps_the_group_rows_and_later_steps_follow_the_schedule(monkeypatch):
    """graph_step's fallback after a failed capture: an ungrouped optimizer drops its dyn block, a
    grouped one keeps its rows (its tables and K12 read them), and the next steps upload them afresh."""
    from frl_b200 import graph_step
    monkeypatch.setattr(graph_step, "_Captured", lambda *a: (_ for _ in ()).throw(RuntimeError("no capture")))
    monkeypatch.setattr(graph_step.torch.cuda, "synchronize", lambda *a: None)
    for kind, grouped in (("adam", True), ("adam", False)):
        if grouped:
            _, _, _, opt = _grouped(kind)
        else:
            net, extra = _model()
            opt = fused_optim.create_fused_optimizer(_arena(net, extra), ADAM)
            opt.enable_dynamic_scalars()
        opt._steps = 2
        worker = types.SimpleNamespace(optimizer=opt, pipeline=types.SimpleNamespace(_step_open=True))
        stepper = graph_step.GraphedTrainStep(worker)
        data, target = [torch.zeros(2, 3)], [(torch.zeros(2),)]
        for _ in range(graph_step.GraphedTrainStep.WARMUP_STEPS + 1):
            assert stepper.ready_for(data, target) is None
        assert not stepper.enabled
        if not grouped:
            assert opt._dyn is None
            continue
        rows = opt._dyn
        assert rows is not None
        for g in opt.param_groups:
            g["lr"] *= 0.1                       # the per-epoch schedule moves every group
        opt.begin_step()
        assert opt._dyn is rows
        want = opt._group_rows()
        assert np.array_equal(rows.numpy().view(np.uint32), want.view(np.uint32))
        assert rows.numpy().view(np.uint32)[0, 3] == 3
        opt.end_step()


def test_a_one_group_optimizer_names_both_counts_when_loading_a_grouped_dict():
    _, _, _, grouped = _grouped("sgd")
    net, extra = _model()
    plain = fused_optim.create_fused_optimizer(_arena(net, extra), SGD)
    with pytest.raises(ValueError, match=r"3 param groups of \[1, 4, 2\] params; this optimizer has 1 of \[7\]"):
        plain.load_state_dict(grouped.state_dict())


def test_info_field_says_none_for_a_single_resolved_group():
    net, extra = _model()
    one = fused_optim.resolve_param_groups(net, [extra], [{"params": list(net.parameters()) + [], "lr": 0.1}])
    arena = _arena(net, extra)
    single = fused_optim.create_fused_optimizer(arena, SGD, param_groups=[{"params": arena.all_params}])
    assert not single.grouped and solver.describe_param_groups(single) == "none"
    assert len(one) == 2
    _, _, _, grouped = _grouped("sgd")
    assert solver.describe_param_groups(grouped).startswith("3: 1 tensors, lr 0.005, wd 0.1")
