"""Lion on the host: the switch and ``FRL_B200_LION``, the refusals (also from ``Solver.solve``,
before a rank starts), the worker-args field, the ``dyn`` block, the state-dict format against
``RefLion``, the entry points' argument checks, the float64 restatement against ``RefLion``, and
the one-GPU launch sequence with K12-Lion on the fake kernels."""
import numpy as np
import pytest
import torch
import torch.nn as nn

import frl_b200  # noqa: F401
from frl_b200 import _native, arena_linear, fused_optim, grad_sync, solver, synthetic
from frl_b200.arena import ParamArena
from frl_b200.solver import SolverWorkerArgs, resolve_lion
from frl_b200.types import LayerAdaptation, OptAlgorithm, OptimizerState, OptimOpts, Precision, RunOpts
from lion_oracle import LionKernelDouble, RefLion, decay_factor, lion_step, lion_step_f64

SGD = OptimOpts(algo=OptAlgorithm.SGD, lr=1e-3, momentum=0.9, weightDecay=0.1)


def _arena(seed=0, precision=Precision.FP32):
    torch.manual_seed(seed)
    net = nn.Sequential(nn.Linear(6, 5), nn.ReLU(), nn.Linear(5, 3))
    extra = nn.Parameter(torch.tensor([0.5, -1.0]))
    return net, extra, ParamArena(list(net.parameters()), [extra], device="cpu", precision=precision)


@pytest.fixture()
def double(monkeypatch):
    d = LionKernelDouble()
    for mod in (fused_optim, grad_sync, arena_linear):
        monkeypatch.setattr(mod, "KERNELS", d)
    return d


# ---- the switch and the refusals -------------------------------------------------------------------

def test_resolve_lion_and_the_environment_variable(monkeypatch):
    monkeypatch.delenv("FRL_B200_LION", raising=False)
    assert resolve_lion() is False
    assert resolve_lion(True) is True and resolve_lion(False) is False
    monkeypatch.setenv("FRL_B200_LION", "1")
    assert resolve_lion() is True and resolve_lion(False) is False       # the keyword wins
    monkeypatch.setenv("FRL_B200_LION", "0")
    assert resolve_lion() is False
    for bad in ("2", "true", "yes", "-1", ""):
        monkeypatch.setenv("FRL_B200_LION", bad)
        with pytest.raises(ValueError, match="FRL_B200_LION"):
            resolve_lion()


@pytest.mark.parametrize("momentum", [0.9, 0.0])
def test_the_factory_builds_lion_from_sgd(momentum):
    _, _, arena = _arena()
    opt = fused_optim.create_fused_optimizer(arena, SGD._replace(momentum=momentum), lion=True)
    assert type(opt) is fused_optim.FusedLion
    assert opt.hyper["betas"] == (momentum, 0.99) and opt.hyper["lr"] == SGD.lr
    assert opt.hyper["weight_decay"] == SGD.weightDecay
    assert type(fused_optim.create_fused_optimizer(arena, SGD)) is fused_optim.FusedSGD


REFUSED = [   # (opts, layer adaptation, optimizer state, adafactor, muon, adamw, message)
    (SGD._replace(algo=OptAlgorithm.ADAM), LayerAdaptation.NONE, OptimizerState.FP32, False, False, False,
     "lion cannot be combined with optimizer 'adam'"),
    (SGD._replace(algo=OptAlgorithm.RMSPROP), LayerAdaptation.NONE, OptimizerState.FP32, False, False, False,
     "lion cannot be combined with optimizer 'rmsprop'"),
    (SGD, LayerAdaptation.LARS, OptimizerState.FP32, False, False, False, "layer adaptation 'lars'"),
    (SGD, LayerAdaptation.NONE, OptimizerState.FP32, True, False, False, "adafactor cannot be combined"),
    (SGD, LayerAdaptation.NONE, OptimizerState.FP32, False, True, False, "muon cannot be combined"),
    (SGD, LayerAdaptation.NONE, OptimizerState.FP32, False, False, True, "adamw cannot be combined"),
    (SGD, LayerAdaptation.NONE, OptimizerState.Q8, False, False, False, "8-bit state needs adam"),
]


@pytest.mark.parametrize("opts,la,state,adafactor,muon,adamw,msg", REFUSED)
def test_refusals_in_the_factory(opts, la, state, adafactor, muon, adamw, msg):
    _, _, arena = _arena()
    with pytest.raises(ValueError, match=msg):
        fused_optim.create_fused_optimizer(arena, opts, la, state, adafactor, muon, adamw, True)


@pytest.mark.parametrize("opts,la,state,adafactor,muon,adamw,msg", REFUSED)
def test_refusals_before_a_rank_starts(tmp_path, opts, la, state, adafactor, muon, adamw, msg):
    ns = synthetic.api_namespace("frl_b200")
    problem = synthetic.make_toy_problem(ns, str(tmp_path), n_train=16, n_test=8)
    run_opts = RunOpts(optim=opts, batchSize=8, nEpochs=1, cpuonly=True)
    with pytest.raises(ValueError, match=msg):
        next(iter(solver.Solver.solve(run_opts, problem, group_name="g", init_method="", layer_adaptation=la,
                                      optimizer_state=state, adafactor=adafactor, muon=muon, adamw=adamw,
                                      lion=True)))


def test_allowed_run_gets_past_the_checks(tmp_path):
    ns = synthetic.api_namespace("frl_b200")
    problem = synthetic.make_toy_problem(ns, str(tmp_path), n_train=16, n_test=8)
    run_opts = RunOpts(optim=SGD, batchSize=8, nEpochs=1, cpuonly=True)
    with pytest.raises(RuntimeError, match="H100 GPUs only"):             # the first thing after the checks
        next(iter(solver.Solver.solve(run_opts, problem, group_name="g", init_method="", lion=True)))


def test_worker_args_field():
    f = SolverWorkerArgs._fields
    assert f.index("lion") == f.index("muon") - 1
    assert f[-5:] == ("master_weights", "optimizer_state", "adafactor", "ema_decay", "grad_accumulation")
    assert SolverWorkerArgs._field_defaults["lion"] is False


# ---- dyn and the state dict ------------------------------------------------------------------------

def test_dyn_values_are_lr_and_the_decay_factor():
    _, _, arena = _arena()
    for lr, wd in ((1e-3, 0.1), (3e-4, 1.0), (1e-4, 0.0)):
        opt = fused_optim.FusedLion(arena, lr=lr, weight_decay=wd)
        assert opt._dyn_values() == (lr, float(decay_factor(lr, wd)))
        opt.enable_dynamic_scalars()
        assert opt._dyn[0].item() == np.float32(lr) and opt._dyn[1].item() == decay_factor(lr, wd)


def _grads(net, extra, seed):
    gen = torch.Generator().manual_seed(seed)
    for p in list(net.parameters()) + [extra]:
        p.grad = torch.randn(p.shape, generator=gen)


def test_steps_and_state_dict_follow_ref_lion(double):
    net, extra, arena = _arena()
    ref_params = [p.detach().clone().double().requires_grad_(True) for p in arena.all_params]
    ref = RefLion(ref_params, lr=1e-2, betas=(0.9, 0.99), weight_decay=0.1)
    opt = fused_optim.FusedLion(arena, lr=1e-2, betas=(0.9, 0.99), weight_decay=0.1)
    for step in range(3):
        _grads(net, extra, step)
        for s in arena.slots:
            arena.grad[s.offset:s.end].copy_(s.param.grad.reshape(-1))
        for q, p in zip(ref_params, arena.all_params):
            q.grad = p.grad.double()
        opt.step()
        ref.step()
    sd, rsd = opt.state_dict(), ref.state_dict()
    assert set(sd["param_groups"][0]) == set(rsd["param_groups"][0])
    assert sd["param_groups"][0]["betas"] == rsd["param_groups"][0]["betas"]
    assert sorted(sd["state"]) == sorted(rsd["state"])
    for i, entry in sd["state"].items():
        assert set(entry) == {"exp_avg"} and entry["exp_avg"].is_contiguous()
        np.testing.assert_allclose(entry["exp_avg"].double(), rsd["state"][i]["exp_avg"], rtol=1e-5, atol=1e-6)
    for s in arena.slots:
        np.testing.assert_allclose(s.param.detach().double(), ref_params[s.index].detach(), atol=1e-5)
    # RefLion's state dict loads back, its betas honoured
    other = fused_optim.FusedLion(_arena()[2], lr=5.0, betas=(0.5, 0.5))
    rsd32 = {"state": {i: {"exp_avg": e["exp_avg"].float()} for i, e in rsd["state"].items()},
             "param_groups": rsd["param_groups"]}
    other.load_state_dict(rsd32)
    assert other.hyper["betas"] == (0.9, 0.99) and other.hyper["lr"] == 1e-2


def test_foreign_state_dicts_are_refused_with_their_keys(double):
    net, extra, arena = _arena()
    sgd = torch.optim.SGD(list(net.parameters()) + [extra], lr=0.1, momentum=0.9)
    adam = torch.optim.Adam(list(net.parameters()) + [extra], lr=0.1)
    _grads(net, extra, 0)
    sgd.step()
    adam.step()
    opt = fused_optim.FusedLion(arena, lr=1e-3)
    with pytest.raises(ValueError, match="momentum_buffer"):
        opt.load_state_dict(sgd.state_dict())
    with pytest.raises(ValueError, match="exp_avg_sq"):
        opt.load_state_dict(adam.state_dict())


@pytest.mark.parametrize("make", [
    lambda ps: torch.optim.SGD(ps, lr=0.1),                    # momentum 0: no momentum_buffer
    lambda ps: torch.optim.SGD(ps, lr=0.1, momentum=0.9),      # before its first step: empty state
    lambda ps: torch.optim.RMSprop(ps, lr=0.1),
])
def test_foreign_param_groups_are_refused_even_with_empty_state(double, make):
    net, extra, arena = _arena()
    other = make(list(net.parameters()) + [extra])
    _grads(net, extra, 0)
    if isinstance(other, torch.optim.SGD) and other.defaults["momentum"] == 0.0:
        other.step()
    opt = fused_optim.FusedLion(arena, lr=1e-3, betas=(0.8, 0.9))
    with pytest.raises(ValueError, match="param group keys"):
        opt.load_state_dict(other.state_dict())
    assert opt.hyper["betas"] == (0.8, 0.9) and "momentum" not in opt.hyper       # nothing was copied


# ---- the entry points' argument checks -------------------------------------------------------------

def test_entry_points_refuse_bad_arguments_before_any_launch():
    lib = _native.lib()
    ok = 1 << 20
    before = lib.frl_launch_count()
    cases = [
        ("frl_lion", "null exp_avg", lambda: lib.frl_lion(ok, ok, None, None, 64, 1e-3, 0.9, 0.99, 0.1, 1.0, None, None, 0,
                                                  None)),
        ("frl_lion", "betas", lambda: lib.frl_lion(ok, ok, ok, None, 64, 1e-3, 1.0, 0.99, 0.1, 1.0, None, None, 0, None)),
        ("frl_lion", "betas", lambda: lib.frl_lion(ok, ok, ok, None, 64, 1e-3, 0.9, -0.1, 0.1, 1.0, None, None, 0, None)),
        ("frl_lion", "g_dtype", lambda: lib.frl_lion(ok, ok, ok, None, 64, 1e-3, 0.9, 0.99, 0.1, 1.0, None, None, 7, None)),
        ("frl_lion_mt", "null exp_avg", lambda: lib.frl_lion_mt(ok, None, None, ok, ok, ok, 4, 1e-3, 0.9, 0.99, 0.1, 1.0,
                                                        None, None, None)),
        ("frl_lion_mt", "betas", lambda: lib.frl_lion_mt(ok, ok, None, ok, ok, ok, 4, 1e-3, 0.9, 1.5, 0.1, 1.0, None, None,
                                                 None)),
        ("frl_lion_mt", "null p", lambda: lib.frl_lion_mt(None, ok, None, ok, ok, ok, 4, 1e-3, 0.9, 0.99, 0.1, 1.0, None,
                                                  None, None)),
        ("frl_lion_sr", "null exp_avg", lambda: lib.frl_lion_sr(ok, ok, None, 64, 0, 1, 1, 1e-3, 0.9, 0.99, 0.1, 1.0, None,
                                                        None, 0, None)),
        ("frl_lion_sr", "update count", lambda: lib.frl_lion_sr(ok, ok, ok, 64, 0, 1, 0, 1e-3, 0.9, 0.99, 0.1, 1.0, None,
                                                        None, 0, None)),
        ("frl_lion_sr", "multiple of 4", lambda: lib.frl_lion_sr(ok, ok, ok, 64, 2, 1, 1, 1e-3, 0.9, 0.99, 0.1, 1.0, None,
                                                         None, 0, None)),
        ("frl_lion_mt_sr", "betas", lambda: lib.frl_lion_mt_sr(ok, ok, ok, ok, ok, 4, 1, 1, 1e-3, 0.9, 1.0, 0.1, 1.0, None,
                                                       None, None)),
        ("frl_lion_mt_sr", "update count", lambda: lib.frl_lion_mt_sr(ok, ok, ok, ok, ok, 4, 1, 1 << 32, 1e-3, 0.9, 0.99,
                                                              0.1, 1.0, None, None, None)),
        ("frl_nvls_lion", "null exp_avg", lambda: lib.frl_nvls_lion(ok, None, ok, ok, 64, 0, 2, ok, 0, ok, 8, 1e-3, 0.9,
                                                            0.99, 0.1, 1.0, None, 0, 0, None)),
        ("frl_nvls_lion", "rank/world", lambda: lib.frl_nvls_lion(ok, ok, ok, ok, 64, 0, 1, ok, 0, ok, 8, 1e-3, 0.9, 0.99,
                                                          0.1, 1.0, None, 0, 0, None)),
        ("frl_dw_gemm_lion", "null exp_avg", lambda: lib.frl_dw_gemm_lion(ok, 256, ok, 256, 64, 128, 256, ok, ok, None,
                                                                  None, 1e-3, 0.9, 0.99, 0.1, 1.0, None, None)),
        ("frl_dw_gemm_lion", "null master", lambda: lib.frl_dw_gemm_lion(ok, 256, ok, 256, 64, 128, 256, ok, None, ok,
                                                                 None, 1e-3, 0.9, 0.99, 0.1, 1.0, None, None)),
        ("frl_dw_gemm_lion", "multiple of the 128x256x32 tile",
         lambda: lib.frl_dw_gemm_lion(ok, 256, ok, 256, 64, 100, 256, ok, ok, ok, None, 1e-3, 0.9, 0.99, 0.1, 1.0, None,
                              None)),
        ("frl_dw_gemm_lion", "multiple of the 128x256x32 tile",
         lambda: lib.frl_dw_gemm_lion(ok, 256, ok, 256, 48, 128, 200, ok, ok, ok, None, 1e-3, 0.9, 0.99, 0.1, 1.0, None,
                              None)),
        ("frl_dw_gemm_lion", "betas", lambda: lib.frl_dw_gemm_lion(ok, 256, ok, 256, 64, 128, 256, ok, ok, ok, None, 1e-3,
                                                           -0.5, 0.99, 0.1, 1.0, None, None)),
        ("frl_dw_gemm_lion_sr", "null weights", lambda: lib.frl_dw_gemm_lion_sr(ok, 256, ok, 256, 64, 128, 256, ok, None,
                                                                        ok, 0, 1, 1, 1e-3, 0.9, 0.99, 0.1, 1.0,
                                                                        None, None)),
        ("frl_dw_gemm_lion_sr", "update count", lambda: lib.frl_dw_gemm_lion_sr(ok, 256, ok, 256, 64, 128, 256, ok, ok, ok,
                                                                        0, 1, 0, 1e-3, 0.9, 0.99, 0.1, 1.0, None,
                                                                        None)),
        ("frl_dw_gemm_lion_sr", "multiple of the 128x256x32 tile",
         lambda: lib.frl_dw_gemm_lion_sr(ok, 256, ok, 256, 64, 128, 100, ok, ok, ok, 0, 1, 1, 1e-3, 0.9, 0.99, 0.1, 1.0,
                                 None, None)),
    ]
    for name, want, call in cases:
        assert call() != 0, (name, want)
        msg = lib.frl_last_error().decode()
        assert msg.startswith(name + ":") and want in msg, (name, want, msg)
    assert lib.frl_launch_count() == before                  # every refusal came before a launch


@pytest.mark.parametrize("call,want", [
    (lambda lib, ok: lib.frl_lion(ok, ok, None, None, 64, 1e-3, 0.9, 0.99, 0.1, 1.0, None, None, 0, None),
     "frl_lion: null exp_avg"),
    (lambda lib, ok: lib.frl_lion(ok, ok, ok, None, 64, 1e-3, 1.0, 0.99, 0.1, 1.0, None, None, 0, None),
     "frl_lion: betas (1, 0.99) outside [0, 1)"),
    (lambda lib, ok: lib.frl_dw_gemm_lion(ok, 256, ok, 256, 64, 100, 256, ok, ok, ok, None, 1e-3, 0.9, 0.99,
                                          0.1, 1.0, None, None), "is not a multiple of the 128x256x32 tile"),
])
def test_refusal_messages(call, want):
    lib = _native.lib()
    assert call(lib, 1 << 20) != 0
    assert want in lib.frl_last_error().decode()


# ---- the restatement against RefLion, in float64 -----------------------------------------------------

@pytest.mark.parametrize("beta1,beta2,wd", [(0.9, 0.99, 0.1), (0.0, 0.99, 0.0), (0.95, 0.98, 1.0)])
def test_restatement_equals_ref_lion_in_float64(beta1, beta2, wd):
    rs = np.random.RandomState(1)
    p0 = rs.randn(1000)
    p = torch.tensor(p0, requires_grad=True)
    ref = RefLion([p], lr=1e-2, betas=(beta1, beta2), weight_decay=wd)
    pp, mm = p0.copy(), np.zeros(1000)
    for _ in range(5):
        g = rs.randn(1000)
        p.grad = torch.tensor(g)
        ref.step()
        pp, mm, _ = lion_step_f64(pp, g, mm, lr=1e-2, beta1=beta1, beta2=beta2, wd=wd)
    np.testing.assert_allclose(pp, p.detach().numpy(), rtol=0, atol=1e-14)
    np.testing.assert_allclose(mm, ref.state[p]["exp_avg"].numpy(), rtol=1e-13, atol=1e-15)


def test_nan_reaches_the_weight_in_every_restatement():
    g = np.array([1.0, np.nan, -1.0])
    p, m, _ = lion_step_f64(np.ones(3), g, np.zeros(3), lr=0.1, beta1=0.9, beta2=0.99, wd=0.0)
    assert np.isnan(p[1]) and np.isnan(m[1]) and p[0] == 0.9 and p[2] == 1.1
    p32, m32 = lion_step(np.ones(3, np.float32), g, np.zeros(3, np.float32), lr=0.1, beta1=0.9, beta2=0.99, wd=0.0)
    assert np.isnan(p32[1]) and np.isnan(m32[1])
    t = torch.ones(3, requires_grad=True)
    t.grad = torch.tensor(g, dtype=torch.float32)
    RefLion([t], lr=0.1).step()
    assert torch.isnan(t[1]) and not torch.isnan(t[0])


# ---- the one-GPU launch sequence with K12 (fake kernels) ---------------------------------------------

WIDTH, ROWS = 256, 64            # the smallest trunk K12 tiles


class _Mlp(nn.Module):
    def __init__(self):
        super().__init__()
        torch.manual_seed(0)
        self.trunk = nn.Sequential(*[m for _ in range(2) for m in (nn.Linear(WIDTH, WIDTH), nn.ReLU())])
        self.head = nn.Linear(WIDTH, 8)          # 8 output rows: not a K12 shape

    def forward(self, x):
        return self.head(self.trunk(x))


def _run(monkeypatch, steps=2, clip=0.0, accumulation=1, kernels=None):
    net = _Mlp()
    arena = ParamArena(net.parameters(), device="cpu", precision=Precision.BF16)
    opt = fused_optim.create_fused_optimizer(arena, SGD, lion=True)
    double = kernels or LionKernelDouble()
    for mod in (arena_linear, grad_sync, fused_optim):
        monkeypatch.setattr(mod, "KERNELS", double)
    pipe = grad_sync.GradBucketPipeline(arena, opt, world_size=1, eager_update=False, clip_norm=clip,
                                        accumulation=accumulation)
    pipe.patch_linears(net)
    net.train()
    logs = []
    for i in range(steps):
        for k in range(accumulation):
            x = torch.randn(ROWS, WIDTH, generator=torch.Generator().manual_seed(10 + i * 7 + k)).to(torch.bfloat16)
            out = net(x)
            if accumulation > 1:
                pipe.set_microbatch(first=k == 0, closes=k == accumulation - 1)
            pipe.begin_step()
            del double.calls[:]
            out.float().square().mean().backward()
            pipe.finish_step()
        logs.append([c for c in double.calls if c[0] in ("lion", "lion_mt", "dw_gemm_lion")])
    trunk = [arena.slot_of(m.weight) for m in net.trunk if isinstance(m, nn.Linear)]
    return pipe, arena, trunk, logs


def test_k12_lion_on_one_gpu_and_the_tail_takes_the_rest(monkeypatch):
    pipe, arena, trunk, logs = _run(monkeypatch)
    assert pipe.fused_dw_update
    trunk_elems = sum(s.numel for s in trunk)
    for log in logs:
        k12 = [c for c in log if c[0] == "dw_gemm_lion"]
        assert sorted(n for _, n in k12) == sorted(s.numel for s in trunk)
        tail = [c for c in log if c[0] == "lion"]
        assert tail and sum(n for _, n in tail) == arena.numel - trunk_elems
        assert log.index(tail[0]) > max(log.index(c) for c in k12)


def test_k12_lion_trains_to_the_same_weights_as_the_tail_alone(monkeypatch):
    _, arena_k12, _, _ = _run(monkeypatch)
    monkeypatch.setenv("FRL_B200_FUSED_DW_UPDATE", "0")
    pipe, arena_ref, _, logs = _run(monkeypatch)
    assert not pipe.fused_dw_update
    assert all(c[0] == "lion" for log in logs for c in log)
    assert torch.equal(arena_k12.master, arena_ref.master) and torch.equal(arena_k12.lp, arena_ref.lp)


def test_no_k12_under_clipping(monkeypatch):
    pipe, _, _, logs = _run(monkeypatch, clip=1.0)
    assert not pipe.fused_dw_update
    assert all(log and all(c[0] == "lion" for c in log) for log in logs)


def test_no_k12_under_accumulation(monkeypatch):
    pipe, _, _, _ = _run(monkeypatch, steps=0, accumulation=2)
    assert not pipe.fused_dw_update
