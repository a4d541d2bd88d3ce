"""Bf16 master weights with stochastic rounding, without a GPU: the numpy restatement of the rounding
against hand-worked bit patterns and its exact expectation, the option's parsing and refusals,
``SolverWorkerArgs``' field order and the new symbols of the library."""
import ctypes

import numpy as np
import pytest
import torch

import frl_b200  # noqa: F401
from frl_b200 import _native, fused_optim, solver, synthetic
from frl_b200.arena import ParamArena
from frl_b200.solver import SolverWorkerArgs, resolve_master_weights
from frl_b200.types import (LayerAdaptation, MasterWeights, OptAlgorithm, OptimizerState, OptimOpts, Precision,
                            RunOpts)
from sr_oracle import bf16_to_f32, sr_bits, sr_round

F = lambda bits: np.uint32(bits).view(np.float32)     # noqa: E731


def test_hand_worked_patterns():
    # 1 + 2^-9 (0x3F804000): half an ulp of bf16 above 1.0 -> rounds up iff r >= 0xC000
    x = F(0x3F804000)
    assert sr_round([x], [0xBFFF])[0] == 0x3F80
    assert sr_round([x], [0xC000])[0] == 0x3F81
    # negative values round the magnitude: -(1 + 2^-9)
    assert sr_round([-x], [0xBFFF])[0] == 0xBF80
    assert sr_round([-x], [0xC000])[0] == 0xBF81
    # exact bf16 values never change, whatever r is
    for v in (0.0, -0.0, 1.0, -2.5, 65536.0):
        b = np.float32(v).view(np.uint32) >> 16
        assert np.all(sr_round(np.full(4, v, np.float32), [0, 1, 0x8000, 0xFFFF]) == b)
    # NaN stays NaN as 0x7FC0, also a negative NaN whose carry could reach the sign bit
    assert sr_round([F(0x7FFFFFFF)], [0xFFFF])[0] == 0x7FC0
    assert sr_round([F(0xFFFFFFFF)], [0xFFFF])[0] == 0x7FC0
    assert sr_round([np.float32("nan")], [0])[0] == 0x7FC0
    # +-inf stay inf
    assert sr_round([np.float32("inf")], [0xFFFF])[0] == 0x7F80
    assert sr_round([np.float32("-inf")], [0xFFFF])[0] == 0xFF80
    # the largest finite fp32 rounds to inf only by the same carry
    assert sr_round([F(0x7F7FFFFF)], [0])[0] == 0x7F7F
    assert sr_round([F(0x7F7FFFFF)], [1])[0] == 0x7F80
    assert sr_round([F(0xFF7FFFFF)], [1])[0] == 0xFF80


def test_expectation_over_every_r_is_exact():
    rng = np.random.default_rng(0)
    xs = np.concatenate([rng.standard_normal(40) * 10.0 ** rng.integers(-6, 6, 40),
                         [1e-39, -3e-40, 1.0 + 2 ** -20]]).astype(np.float32)
    r = np.arange(65536, dtype=np.uint32)
    for x in xs:
        got = bf16_to_f32(sr_round(np.full(65536, x, np.float32), r)).astype(np.float64).mean()
        assert got == np.float64(x), (x, got)


def test_draws_depend_on_index_update_and_seed_only():
    a = sr_bits(np.arange(0, 64), 7, 123)
    assert np.array_equal(a[16:32], sr_bits(np.arange(16, 32), 7, 123))        # any split of the range
    assert not np.array_equal(a, sr_bits(np.arange(0, 64), 8, 123))
    assert not np.array_equal(a, sr_bits(np.arange(0, 64), 7, 124))
    assert a.max() <= 0xFFFF


def test_resolve_master_weights(monkeypatch):
    monkeypatch.delenv(solver.MASTER_WEIGHTS_ENV, raising=False)
    assert resolve_master_weights() is MasterWeights.FP32
    assert resolve_master_weights(MasterWeights.BF16) is MasterWeights.BF16
    assert resolve_master_weights("bf16") is MasterWeights.BF16
    monkeypatch.setenv(solver.MASTER_WEIGHTS_ENV, "BF16")
    assert resolve_master_weights() is MasterWeights.BF16
    monkeypatch.setenv(solver.MASTER_WEIGHTS_ENV, "fp16")
    with pytest.raises(ValueError, match=solver.MASTER_WEIGHTS_ENV):
        resolve_master_weights()


@pytest.mark.parametrize("kw, match", [
    (dict(precision=Precision.FP32), "precision fp32"),
    (dict(layer_adaptation=LayerAdaptation.LARS), "layer adaptation lars"),
    (dict(layer_adaptation=LayerAdaptation.LAMB), "layer adaptation lamb"),
    (dict(adafactor=True), "adafactor"),
    (dict(muon=True), "muon"),
    (dict(optimizer_state=OptimizerState.Q8), "optimizer state 8bit"),
])
def test_refusals(kw, match):
    args = dict(precision=Precision.BF16, layer_adaptation=LayerAdaptation.NONE, optimizer_state=OptimizerState.FP32,
                adafactor=False, muon=False)
    args.update(kw)
    with pytest.raises(ValueError, match="master_weights=bf16 cannot be combined with " + match):
        fused_optim.check_master_weights(MasterWeights.BF16, **args)
    fused_optim.check_master_weights(MasterWeights.FP32, **args)        # fp32 master: anything goes


@pytest.mark.parametrize("prec", [Precision.BF16, Precision.FP8])
def test_allowed_combinations(prec):
    fused_optim.check_master_weights(MasterWeights.BF16, prec, LayerAdaptation.NONE, OptimizerState.FP32,
                                     False, False)


def test_solve_refuses_before_a_rank_starts(tmp_path):
    ns = synthetic.api_namespace("frl_b200")
    problem = synthetic.make_toy_problem(ns, str(tmp_path), n_train=16, n_test=8)
    run_opts = RunOpts(optim=OptimOpts(algo=OptAlgorithm.SGD, lr=0.1), batchSize=8, nEpochs=1, cpuonly=True)
    with pytest.raises(ValueError, match="precision fp32"):
        next(iter(solver.Solver.solve(run_opts, problem, group_name="g", init_method="", precision=Precision.FP32,
                                      master_weights=MasterWeights.BF16)))


def test_worker_args_field_order():
    f = SolverWorkerArgs._fields
    assert f.index("master_weights") == f.index("channels_last") + 1
    assert f[-5:] == ("master_weights", "optimizer_state", "adafactor", "ema_decay", "grad_accumulation")
    assert SolverWorkerArgs.__new__.__defaults__[f.index("master_weights") - len(f)] is MasterWeights.FP32


def test_arena_on_cpu_has_no_model_master():
    torch.manual_seed(0)
    model = torch.nn.Sequential(torch.nn.Linear(5, 3), torch.nn.Linear(3, 2))
    crit = torch.nn.Parameter(torch.randn(3))
    want = [p.detach().clone() for p in model.parameters()] + [crit.detach().clone()]
    a = ParamArena(model.parameters(), [crit], device="cpu", precision=Precision.BF16,
                   master_weights=MasterWeights.BF16)
    assert a.master.numel() == a.numel - a.model_end and a.master_base == a.model_end
    for s, w in zip(a.slots, want):
        if s.is_model:
            assert torch.equal(s.param.data, w.to(torch.bfloat16))
            with pytest.raises(ValueError):
                a.master_view(s)
        else:
            assert torch.equal(s.param.data, w)
    with a.exported():
        for s, w in zip(a.slots, want):
            assert s.param.dtype == torch.float32
            assert torch.equal(s.param.data, w.to(torch.bfloat16).float() if s.is_model else w)
    with pytest.raises(ValueError, match="bf16-storage precision"):
        ParamArena(torch.nn.Linear(2, 2).parameters(), device="cpu", precision=Precision.FP32,
                   master_weights=MasterWeights.BF16)


def test_new_symbols_are_exported():
    handle = ctypes.CDLL(_native.LIB_PATH)
    for base in ("sgd_momentum", "adam", "adamw", "rmsprop"):
        for suffix in ("_sr", "_mt_sr"):
            assert hasattr(handle, "frl_" + base + suffix)
    assert hasattr(handle, "frl_weight_ema_bf16")
    lib = _native.lib()
    assert lib.frl_abi_version() == 1
    # argument errors come back without a GPU
    assert lib.frl_adam_sr(None, None, None, None, None, 16, 0, 1, 0.1, 0.9, 0.999, 1e-8, 0.0, 0, 1.0,
                           None, None, 0, None) < 0
    assert b"frl_adam_sr" in lib.frl_last_error()
    assert lib.frl_sgd_momentum_sr(None, None, None, 16, 2, 1, 1, 0.1, 0.0, 0.0, 0.0, 1.0, None, None, 0, 0,
                                   None) < 0
