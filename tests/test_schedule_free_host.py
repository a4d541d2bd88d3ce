"""Schedule-Free AdamW / SGD on the host: the restatements (and the mean-of-z property), the switch and
its environment variables, the refusals (also from ``Solver.solve``, before a rank starts), the
worker-args field, the ``dyn`` values and group rows against the double arithmetic, the state dict
against the restatement's, foreign state dicts, the entry points' argument checks without a GPU, and
the one-GPU launch sequence (no K12) on CPU kernel doubles."""
import math

import numpy as np
import pytest
import torch
import torch.nn as nn

import frl_b200  # noqa: F401
from frl_b200 import _native, arena_linear, fused_optim, grad_sync, solver, synthetic
from frl_b200.arena import ParamArena
from frl_b200.solver import SolverWorkerArgs, resolve_schedule_free
from frl_b200.types import (LayerAdaptation, OptAlgorithm, OptimizerState, OptimOpts, Precision, RunOpts,
                            ScheduleFree)
from lion_oracle import LionKernelDouble
from schedule_free_oracle import RefAdamWScheduleFree, RefSGDScheduleFree, sf_eval_f64

ADAM = OptimOpts(algo=OptAlgorithm.ADAM, lr=1e-3, weightDecay=0.01, epsilon=1e-8)
SGD = OptimOpts(algo=OptAlgorithm.SGD, lr=0.1, momentum=0.9, weightDecay=1e-4)


class SFKernelDouble(LionKernelDouble):
    """The CPU kernel doubles plus the flat Schedule-Free entry points and K2-sfx, in float64."""

    GROUP_DYN_COLS = _native.GROUP_DYN_COLS

    def _sf(self, adaptive, y, g, z, v, p_lp, *, lr, ckp1, beta1, wd, beta2=0.0, eps=0.0, grad_scale=1.0,
            grad_scale_dev=None):
        yd, zd = y.double(), z.double()
        u = g.double() * self._scale(grad_scale, grad_scale_dev)
        if adaptive:
            vd = v.double() * beta2 + (1 - beta2) * u * u
            v.copy_(vd)
            u = u / (vd.sqrt() + eps)
        u = u + wd * yd
        yd = yd + ckp1 * (zd - yd)
        yd = yd + lr * (beta1 * (1 - ckp1) - 1) * u
        z.copy_(zd - lr * u)
        y.copy_(yd)
        if p_lp is not None:
            p_lp.copy_(y)

    def sf_adamw(self, y, g, z, v, p_lp, n, *, lr, ckp1, beta1, beta2, eps, wd, grad_scale=1.0,
                 grad_scale_dev=None, dyn=None):
        self.calls.append(("sf_adamw", n))
        self._sf(True, y, g, z, v, p_lp, lr=lr, ckp1=ckp1, beta1=beta1, beta2=beta2, eps=eps, wd=wd,
                 grad_scale=grad_scale, grad_scale_dev=grad_scale_dev)

    def sf_sgd(self, y, g, z, p_lp, n, *, lr, ckp1, beta1, wd, grad_scale=1.0, grad_scale_dev=None, dyn=None):
        self.calls.append(("sf_sgd", n))
        self._sf(False, y, g, z, None, p_lp, lr=lr, ckp1=ckp1, beta1=beta1, wd=wd, grad_scale=grad_scale,
                 grad_scale_dev=grad_scale_dev)

    def sf_eval_weights(self, y, z, x, *, beta1):
        self.calls.append(("sf_eval_weights", y.numel()))
        x.copy_(sf_eval_f64(y, z, beta1))


def _arena(seed=0, precision=Precision.FP32):
    torch.manual_seed(seed)
    net = nn.Sequential(nn.Linear(6, 5), nn.ReLU(), nn.Linear(5, 3))
    extra = nn.Parameter(torch.tensor([0.5, -1.0]))
    return net, extra, ParamArena(list(net.parameters()), [extra], device="cpu", precision=precision)


@pytest.fixture()
def double(monkeypatch):
    d = SFKernelDouble()
    for mod in (fused_optim, grad_sync, arena_linear):
        monkeypatch.setattr(mod, "KERNELS", d)
    return d


# ---- the restatements ------------------------------------------------------------------------------

@pytest.mark.parametrize("momentum", [0.9, 0.5])
def test_sgd_restatement_evaluates_at_the_mean_of_z(momentum):
    torch.manual_seed(1)
    p = nn.Parameter(torch.randn(7, dtype=torch.float64))
    opt = RefSGDScheduleFree([p], lr=0.05, momentum=momentum)
    zs = []
    for t in range(6):
        p.grad = torch.randn(7, dtype=torch.float64)
        opt.step()
        zs.append(opt.state[p]["z"].clone())
        opt.eval()
        torch.testing.assert_close(p.detach(), torch.stack(zs).mean(0), rtol=1e-12, atol=1e-12)
        opt.train()


def test_adamw_restatement_first_step_and_modes():
    torch.manual_seed(2)
    p = nn.Parameter(torch.randn(5, dtype=torch.float64))
    y0 = p.detach().clone()
    opt = RefAdamWScheduleFree([p], lr=1e-2, weight_decay=0.1)
    g = torch.randn(5, dtype=torch.float64)
    p.grad = g.clone()
    opt.step()
    # k = 0: ckp1 = 1, so y = z_1 + lr*(beta1*0 - 1)*u ... and z_1 = y0 - lr*u
    lr = 1e-2 * math.sqrt(1 - 0.999)
    u = g / (torch.sqrt(0.001 * g * g) + 1e-8) + 0.1 * y0
    torch.testing.assert_close(opt.state[p]["z"], y0 - lr * u)
    torch.testing.assert_close(p.detach(), y0 - lr * u)
    opt.eval()
    torch.testing.assert_close(p.detach(), opt.state[p]["z"])      # x = z after one update
    opt.train()
    assert opt.param_groups[0]["k"] == 1 and opt.param_groups[0]["lr_max"] == pytest.approx(lr)


# ---- the switch, the refusals, the field -------------------------------------------------------------

def test_resolve_schedule_free_and_the_environment_variables(monkeypatch):
    monkeypatch.delenv("FRL_B200_SCHEDULE_FREE", raising=False)
    monkeypatch.delenv("FRL_B200_SCHEDULE_FREE_WARMUP", raising=False)
    assert resolve_schedule_free() is None
    assert resolve_schedule_free(True) == ScheduleFree(0, 0.0, 2.0)
    assert resolve_schedule_free(False) is None
    assert resolve_schedule_free(ScheduleFree(warmup_steps=5, r=1.0)) == ScheduleFree(5, 1.0, 2.0)
    monkeypatch.setenv("FRL_B200_SCHEDULE_FREE", "1")
    assert resolve_schedule_free() == ScheduleFree()
    assert resolve_schedule_free(False) is None                      # the keyword wins
    monkeypatch.setenv("FRL_B200_SCHEDULE_FREE_WARMUP", "100")
    assert resolve_schedule_free() == ScheduleFree(warmup_steps=100)
    for bad in ("-1", "2.5", "x", ""):
        monkeypatch.setenv("FRL_B200_SCHEDULE_FREE_WARMUP", bad)
        with pytest.raises(ValueError, match="FRL_B200_SCHEDULE_FREE_WARMUP"):
            resolve_schedule_free()
    for bad in ("2", "true", "yes", ""):
        monkeypatch.setenv("FRL_B200_SCHEDULE_FREE", bad)
        with pytest.raises(ValueError, match="FRL_B200_SCHEDULE_FREE must be 0 or 1"):
            resolve_schedule_free()
    for bad in ("1", 1, ScheduleFree(warmup_steps=-1), ScheduleFree(warmup_steps=1.5), ScheduleFree(r=float("nan"))):
        with pytest.raises(ValueError, match="schedule_free"):
            resolve_schedule_free(bad)


def test_the_factory_builds_the_two_rules():
    _, _, arena = _arena()
    a = fused_optim.create_fused_optimizer(arena, ADAM, schedule_free=ScheduleFree(warmup_steps=3))
    assert type(a) is fused_optim.FusedScheduleFreeAdamW
    assert a.hyper["betas"] == (0.9, 0.999) and a.hyper["eps"] == ADAM.epsilon and a.hyper["warmup_steps"] == 3
    s = fused_optim.create_fused_optimizer(arena, SGD, schedule_free=True)
    assert type(s) is fused_optim.FusedScheduleFreeSGD and s.beta1 == 0.9 and s.hyper["weight_decay"] == 1e-4
    assert type(fused_optim.create_fused_optimizer(arena, SGD)) is fused_optim.FusedSGD


REFUSED = [   # (opts, la, state, adafactor, muon, adamw, lion, ema, message)
    (ADAM._replace(algo=OptAlgorithm.RMSPROP), LayerAdaptation.NONE, OptimizerState.FP32, 0, 0, 0, 0, 0,
     "optimizer 'rmsprop'"),
    (ADAM._replace(amsgrad=True), LayerAdaptation.NONE, OptimizerState.FP32, 0, 0, 0, 0, 0, "amsgrad"),
    (SGD._replace(momentum=0.0), LayerAdaptation.NONE, OptimizerState.FP32, 0, 0, 0, 0, 0, "sgd momentum 0.0"),
    (SGD._replace(momentum=1.0), LayerAdaptation.NONE, OptimizerState.FP32, 0, 0, 0, 0, 0, "sgd momentum 1.0"),
    (SGD, LayerAdaptation.LARS, OptimizerState.FP32, 0, 0, 0, 0, 0, "layer adaptation 'lars'"),
    (ADAM, LayerAdaptation.LAMB, OptimizerState.FP32, 0, 0, 0, 0, 0, "layer adaptation 'lamb'"),
    (ADAM, LayerAdaptation.NONE, OptimizerState.Q8, 0, 0, 0, 0, 0, "optimizer state '8bit'"),
    (ADAM, LayerAdaptation.NONE, OptimizerState.FP32, 1, 0, 0, 0, 0, "adafactor"),
    (ADAM, LayerAdaptation.NONE, OptimizerState.FP32, 0, 1, 0, 0, 0, "muon"),
    (ADAM, LayerAdaptation.NONE, OptimizerState.FP32, 0, 0, 1, 0, 0, "adamw"),
    (SGD, LayerAdaptation.NONE, OptimizerState.FP32, 0, 0, 0, 1, 0, "lion"),
    (ADAM, LayerAdaptation.NONE, OptimizerState.FP32, 0, 0, 0, 0, 1, "a weight EMA"),
]


@pytest.mark.parametrize("opts,la,state,adafactor,muon,adamw,lion,ema,msg", REFUSED)
def test_refusals(opts, la, state, adafactor, muon, adamw, lion, ema, msg):
    with pytest.raises(ValueError, match="schedule_free cannot be combined with " + msg):
        fused_optim.check_schedule_free(opts, la, state, bool(adafactor), bool(muon), bool(adamw), bool(lion),
                                        bool(ema), ScheduleFree())
    fused_optim.check_schedule_free(opts, la, state, bool(adafactor), bool(muon), bool(adamw), bool(lion), bool(ema),
                                    None)


def _problem(tmp_path):
    return synthetic.make_toy_problem(synthetic.api_namespace("frl_b200"), str(tmp_path), n_train=16, n_test=8)


@pytest.mark.parametrize("opts,kw,msg", [
    (ADAM._replace(algo=OptAlgorithm.RMSPROP), {}, "optimizer 'rmsprop'"),
    (ADAM._replace(amsgrad=True), {}, "amsgrad"),
    (SGD._replace(momentum=0.0), {}, "sgd momentum"),
    (SGD, {"layer_adaptation": LayerAdaptation.LARS}, "layer adaptation 'lars'"),
    (ADAM, {"optimizer_state": OptimizerState.Q8}, "optimizer state '8bit'"),
    (ADAM, {"adamw": True}, "adamw"),
    (SGD, {"lion": True}, "lion"),
    (ADAM, {"ema_decay": 0.99}, "a weight EMA"),
])
def test_refusals_before_a_rank_starts(tmp_path, opts, kw, msg):
    run_opts = RunOpts(optim=opts, batchSize=8, nEpochs=1, cpuonly=True)
    with pytest.raises(ValueError, match="schedule_free cannot be combined with " + msg):
        next(iter(solver.Solver.solve(run_opts, _problem(tmp_path), group_name="g", init_method="",
                                      schedule_free=True, **kw)))


def test_allowed_run_gets_past_the_checks(tmp_path, monkeypatch):
    run_opts = RunOpts(optim=ADAM, batchSize=8, nEpochs=1, cpuonly=True)
    with pytest.raises(RuntimeError, match="H100 GPUs only"):             # the first thing after the checks
        next(iter(solver.Solver.solve(run_opts, _problem(tmp_path), group_name="g", init_method="",
                                      schedule_free=True, no_decay_1d=True)))
    monkeypatch.setenv("FRL_B200_SCHEDULE_FREE", "maybe")
    with pytest.raises(ValueError, match="FRL_B200_SCHEDULE_FREE"):
        next(iter(solver.Solver.solve(run_opts, _problem(tmp_path), group_name="g", init_method="")))


def test_worker_args_field():
    f = SolverWorkerArgs._fields
    assert f.index("schedule_free") == f.index("layer_adaptation") - 1
    assert f[-5:] == ("master_weights", "optimizer_state", "adafactor", "ema_decay", "grad_accumulation")
    assert f.index("layer_adaptation") == len(f) - 11
    assert SolverWorkerArgs._field_defaults["schedule_free"] is None


# ---- dyn values and group rows -----------------------------------------------------------------------

def _double_scalars(lr, k, warmup, beta1, beta2, lr_max, weight_sum, r=0.0, power=2.0):
    lr_t = lr * ((k + 1) / warmup if k < warmup else 1.0)
    if beta2 is not None:
        lr_t *= math.sqrt(1 - beta2 ** (k + 1))
    lr_max = max(lr_max, lr_t)
    weight = (k + 1) ** r * lr_max ** power
    weight_sum += weight
    ckp1 = weight / weight_sum if weight_sum else 0.0
    return lr_t, ckp1, lr_t * (beta1 * (1 - ckp1) - 1), lr_max, weight_sum


@pytest.mark.parametrize("adaptive", [True, False])
def test_dyn_and_group_rows_follow_the_double_arithmetic(double, adaptive):
    net, extra, arena = _arena()
    groups = [{"params": [net[0].bias, net[2].bias], "weight_decay": 0.0, "lr": 0.5},
              {"params": [net[0].weight, net[2].weight, extra]}]
    cls = fused_optim.FusedScheduleFreeAdamW if adaptive else fused_optim.FusedScheduleFreeSGD
    opt = cls(arena, lr=0.1, weight_decay=0.01, warmup_steps=3, param_groups=groups)
    beta2 = 0.999 if adaptive else None
    state = [(g["lr"], -1.0, 0.0) for g in opt.param_groups]
    for k in range(7):
        if k == 4:                             # a scheduler drop, and lr = 0 in one group
            opt.param_groups[0]["lr"] = 0.0
            opt.param_groups[1]["lr"] *= 0.1
        rows = opt._group_rows()
        for gi, g in enumerate(opt.param_groups):
            _, lr_max, ws = state[gi]
            want = _double_scalars(g["lr"], k, 3, 0.9, beta2, lr_max, ws)
            assert tuple(rows[gi, :3]) == tuple(np.float32(w) for w in want[:3])
            assert rows[gi, 4] == np.float32(g["weight_decay"]) and rows.view(np.uint32)[gi, 3] == k + 1
            state[gi] = (g["lr"], want[3], want[4])
        for p in arena.all_params:
            p.grad = torch.randn(p.shape)
        opt.begin_step()
        opt.end_step()
        for gi, g in enumerate(opt.param_groups):
            assert g["k"] == k + 1 and g["lr_max"] == state[gi][1] and g["weight_sum"] == state[gi][2]


def test_ungrouped_dyn_block_is_lr_ckp1_y_lr(double):
    _, _, arena = _arena()
    opt = fused_optim.FusedScheduleFreeSGD(arena, lr=0.2, momentum=0.8)
    opt.enable_dynamic_scalars()
    lr, ckp1, y_lr = _double_scalars(0.2, 0, 0, 0.8, None, -1.0, 0.0)[:3]
    assert opt._dyn.tolist() == [np.float32(lr), np.float32(ckp1), np.float32(y_lr), 0.0]
    assert ckp1 == 1.0 and y_lr == -0.2


# ---- steps and the state dict against the restatement ------------------------------------------------

def _grads(net, extra, seed, arena=None):
    gen = torch.Generator().manual_seed(seed)
    for p in list(net.parameters()) + [extra]:
        p.grad = torch.randn(p.shape, generator=gen)
    if arena is not None:                    # where the update reads them
        for s in arena.slots:
            arena.grad[s.offset:s.end].copy_(s.param.grad.reshape(-1))


@pytest.mark.parametrize("adaptive", [True, False])
def test_steps_state_dict_and_x_follow_the_restatement(double, adaptive):
    net, extra, arena = _arena()
    ref_params = [p.detach().clone().double().requires_grad_(True) for p in arena.all_params]
    if adaptive:
        ref = RefAdamWScheduleFree(ref_params, lr=1e-2, weight_decay=0.1, warmup_steps=2)
        opt = fused_optim.FusedScheduleFreeAdamW(arena, lr=1e-2, weight_decay=0.1, warmup_steps=2)
    else:
        ref = RefSGDScheduleFree(ref_params, lr=0.1, momentum=0.9, weight_decay=0.1, warmup_steps=2)
        opt = fused_optim.FusedScheduleFreeSGD(arena, lr=0.1, momentum=0.9, weight_decay=0.1, warmup_steps=2)
    assert opt.state_dict()["state"] == {}
    for step in range(4):
        _grads(net, extra, step, arena)
        for r, p in zip(ref_params, arena.all_params):
            r.grad = p.grad.double()
        ref.step()
        opt.step()
        for r, p in zip(ref_params, arena.all_params):
            torch.testing.assert_close(p.detach().double(), r.detach(), rtol=1e-5, atol=1e-6)
    sd, want = opt.state_dict(), ref.state_dict()
    mine = {k: v for k, v in sd["param_groups"][0].items() if k != "params"}
    theirs = {k: v for k, v in want["param_groups"][0].items() if k not in ("params", "foreach")}
    assert set(mine) == set(theirs)
    for k in theirs:
        assert mine[k] == pytest.approx(theirs[k]), k
    assert sorted(sd["state"]) == sorted(want["state"])
    for i in want["state"]:
        assert set(sd["state"][i]) == set(want["state"][i])
        for k in want["state"][i]:
            torch.testing.assert_close(sd["state"][i][k].double(), want["state"][i][k], rtol=1e-5, atol=1e-6)
    # x: the swapped weights (FP32 arena: in place) and the export
    ref.eval()
    n_model = len(list(net.parameters()))
    with opt.swapped():
        for r, p in zip(ref_params[:n_model], list(net.parameters())):
            torch.testing.assert_close(p.detach().double(), r.detach(), rtol=1e-5, atol=1e-6)
    ref.train()
    for r, p in zip(ref_params, arena.all_params):
        torch.testing.assert_close(p.detach().double(), r.detach(), rtol=1e-5, atol=1e-6)
    # a resume from the state dict continues with the same scalars
    net2, extra2, arena2 = _arena()
    opt2 = type(opt)(arena2, lr=1.0)
    opt2.load_state_dict(sd)
    assert opt2._steps == 4 and opt2.hyper["k"] == 4 and opt2._group_rows().tobytes() == opt._group_rows().tobytes()


def test_swap_restores_y_bit_for_bit_also_when_the_block_raises(double):
    net, extra, arena = _arena()
    opt = fused_optim.FusedScheduleFreeSGD(arena, lr=0.1, momentum=0.9)
    with opt.swapped():                       # before the first update x is y: nothing to do
        pass
    for step in range(3):
        _grads(net, extra, step, arena)
        opt.step()
    before = arena.master.clone()
    with pytest.raises(KeyError):
        with opt.swapped():
            assert not torch.equal(arena.master, before)
            raise KeyError("split failed")
    assert torch.equal(arena.master, before)
    with pytest.raises(RuntimeError, match="inside swapped"):
        with opt.swapped():
            opt.begin_step()


def test_foreign_state_dicts_are_refused_with_their_keys(double):
    net, extra, arena = _arena()
    sgd = fused_optim.FusedSGD(arena, lr=0.1, momentum=0.9)
    _grads(net, extra, 0, arena)
    sgd.step()
    sf = fused_optim.FusedScheduleFreeSGD(arena, lr=0.1)
    with pytest.raises(ValueError, match="momentum_buffer"):
        sf.load_state_dict(sgd.state_dict())
    with pytest.raises(ValueError, match="param group keys"):
        sf.load_state_dict(fused_optim.FusedSGD(arena, lr=0.1).state_dict())     # empty state
    adamw = fused_optim.FusedScheduleFreeAdamW(arena, lr=1e-3)
    with pytest.raises(ValueError, match="betas"):
        adamw.load_state_dict(sf.state_dict())
    sd = sf.state_dict()
    sd["param_groups"][0]["a_newer_key"] = 1           # tolerated
    fused_optim.FusedScheduleFreeSGD(arena, lr=0.1).load_state_dict(sd)


# ---- the entry points' argument checks ---------------------------------------------------------------

def test_entry_points_refuse_bad_arguments_before_any_launch():
    lib = _native.lib()
    ok = 1 << 20
    before = lib.frl_launch_count()
    cases = [
        ("frl_sf_adamw", "null z", lambda: lib.frl_sf_adamw(ok, ok, None, ok, None, 64, 1e-3, 1.0, 0.9, 0.999, 1e-8, 0.0,
                                                    1.0, None, None, 0, None)),
        ("frl_sf_adamw", "null exp_avg_sq", lambda: lib.frl_sf_adamw(ok, ok, ok, None, None, 64, 1e-3, 1.0, 0.9, 0.999,
                                                             1e-8, 0.0, 1.0, None, None, 0, None)),
        ("frl_sf_adamw", "beta1 1 outside (0, 1)", lambda: lib.frl_sf_adamw(ok, ok, ok, ok, None, 64, 1e-3, 1.0, 1.0,
                                                                    0.999, 1e-8, 0.0, 1.0, None, None, 0, None)),
        ("frl_sf_adamw", "g_dtype", lambda: lib.frl_sf_adamw(ok, ok, ok, ok, None, 64, 1e-3, 1.0, 0.9, 0.999, 1e-8, 0.0,
                                                     1.0, None, None, 7, None)),
        ("frl_sf_sgd", "null z", lambda: lib.frl_sf_sgd(ok, ok, None, None, 64, 0.1, 1.0, 0.9, 0.0, 1.0, None, None, 0,
                                                None)),
        ("frl_sf_sgd", "beta1 0 outside", lambda: lib.frl_sf_sgd(ok, ok, ok, None, 64, 0.1, 1.0, 0.0, 0.0, 1.0, None, None,
                                                         0, None)),
        ("frl_sf_adamw_mt", "null exp_avg_sq", lambda: lib.frl_sf_adamw_mt(ok, ok, None, None, ok, ok, ok, 4, 1e-3, 1.0,
                                                                   0.9, 0.999, 1e-8, 0.0, 1.0, None, None, None)),
        ("frl_sf_sgd_mt", "null p", lambda: lib.frl_sf_sgd_mt(None, ok, None, ok, ok, ok, 4, 0.1, 1.0, 0.9, 0.0, 1.0,
                                                      None, None, None)),
        ("frl_sf_adamw_mt_grouped", "n_groups 0", lambda: lib.frl_sf_adamw_mt_grouped(
            ok, ok, ok, None, ok, ok, ok, 4, ok, ok, ok, 0, 0.9, 0.999, 1e-8, 1.0, None, None)),
        ("frl_sf_sgd_mt_grouped", "beta1", lambda: lib.frl_sf_sgd_mt_grouped(
            ok, ok, None, ok, ok, ok, 4, ok, ok, ok, 1, 1.5, 1.0, None, None)),
        ("frl_sf_adamw_sr", "update count", lambda: lib.frl_sf_adamw_sr(ok, ok, ok, ok, 64, 0, 1, 0, 1e-3, 1.0, 0.9,
                                                                0.999, 1e-8, 0.0, 1.0, None, None, 0, None)),
        ("frl_sf_sgd_sr", "multiple of 4", lambda: lib.frl_sf_sgd_sr(ok, ok, ok, 64, 2, 1, 1, 0.1, 1.0, 0.9, 0.0, 1.0,
                                                             None, None, 0, None)),
        ("frl_sf_adamw_mt_sr", "null z", lambda: lib.frl_sf_adamw_mt_sr(ok, None, ok, ok, ok, ok, 4, 1, 1, 1e-3, 1.0, 0.9,
                                                                0.999, 1e-8, 0.0, 1.0, None, None, None)),
        ("frl_sf_sgd_mt_sr", "update count", lambda: lib.frl_sf_sgd_mt_sr(ok, ok, ok, ok, ok, 4, 1, 1 << 32, 0.1, 1.0,
                                                                  0.9, 0.0, 1.0, None, None, None)),
        ("frl_sf_adamw_mt_grouped_sr", "null exp_avg_sq", lambda: lib.frl_sf_adamw_mt_grouped_sr(
            ok, ok, None, ok, ok, ok, 4, ok, ok, ok, 1, 1, 0.9, 0.999, 1e-8, 1.0, None, None)),
        ("frl_sf_sgd_mt_grouped_sr", "null seg_group", lambda: lib.frl_sf_sgd_mt_grouped_sr(
            ok, ok, ok, ok, ok, 4, None, ok, ok, 1, 1, 0.9, 1.0, None, None)),
        ("frl_sf_eval_weights", "beta1", lambda: lib.frl_sf_eval_weights(ok, 0, ok, ok, 1, 64, 1.0, None)),
        ("frl_sf_eval_weights", "in place needs", lambda: lib.frl_sf_eval_weights(ok, 0, ok, ok, 1, 64, 0.9, None)),
        ("frl_sf_eval_weights", "x_dtype 7", lambda: lib.frl_sf_eval_weights(ok, 0, ok, ok + 64, 7, 64, 0.9, None)),
        ("frl_sf_eval_weights", "null y / z / x", lambda: lib.frl_sf_eval_weights(ok, 0, None, ok + 64, 1, 64, 0.9,
                                                                          None)),
        ("frl_sf_eval_weights", "aligned", lambda: lib.frl_sf_eval_weights(ok, 0, ok + 4, ok + 64, 1, 64, 0.9, None)),
    ]
    for name, want, call in cases:
        assert call() != 0, (name, want)
        msg = lib.frl_last_error().decode()
        assert msg.startswith(name + ":") and want in msg, (name, want, msg)
    assert lib.frl_launch_count() == before                  # every refusal came before a launch


# ---- the one-GPU launch sequence: no K12 ---------------------------------------------------------------

WIDTH, ROWS = 256, 64            # the smallest trunk K12 tiles


def test_no_k12_and_no_k7_under_schedule_free(monkeypatch):
    torch.manual_seed(0)
    net = nn.Sequential(nn.Linear(WIDTH, WIDTH), nn.ReLU(), nn.Linear(WIDTH, WIDTH), nn.ReLU(), nn.Linear(WIDTH, 8))
    arena = ParamArena(net.parameters(), device="cpu", precision=Precision.BF16)
    opt = fused_optim.create_fused_optimizer(arena, SGD, schedule_free=True)
    d = SFKernelDouble()
    for mod in (arena_linear, grad_sync, fused_optim):
        monkeypatch.setattr(mod, "KERNELS", d)
    pipe = grad_sync.GradBucketPipeline(arena, opt, world_size=1, eager_update=False)
    assert not pipe.fused_dw_update
    pipe.patch_linears(net)
    for i in range(2):
        x = torch.randn(ROWS, WIDTH, generator=torch.Generator().manual_seed(i)).to(torch.bfloat16)
        out = net(x)
        pipe.begin_step()
        del d.calls[:]
        out.float().square().mean().backward()
        pipe.finish_step()
        names = {c[0] for c in d.calls}
        assert "sf_sgd" in names and not any(n.startswith(("dw_gemm", "nvls")) for n in names), names
    assert opt.hyper["k"] == 2
    with pytest.raises(RuntimeError, match="no fused NVLS step"):
        opt._launch_nvls(0, 8, 1.0)
