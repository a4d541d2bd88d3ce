"""AdamW on the host: the switch, the refusals, the worker-args field, the ``dyn`` block, the
state-dict format against CPU ``torch.optim.AdamW``, the CPU doubles against float64 torch, the
entry points' argument checks, and the pipeline's launch sequences (Adam's, with every Adam
launch replaced by its AdamW form) on one rank and on two gloo ranks."""
import itertools
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import frl_b200  # noqa: F401
from frl_b200 import _native, fused_optim, grad_sync, multi_tensor
from frl_b200.arena import ParamArena
from frl_b200.grad_sync import accumulation_plan
from frl_b200.solver import SolverWorkerArgs, resolve_adamw
from frl_b200.types import LayerAdaptation, OptAlgorithm, OptimizerState, OptimOpts
from adamw_oracle import AdamWKernelDouble, adamw_step, decay_factor
from oracle.optim_np import KernelDouble
import test_pipeline_launches as tpl

f32 = np.float32
ADAM = OptimOpts(algo=OptAlgorithm.ADAM, lr=0.01, weightDecay=1e-2)


@pytest.fixture()
def double(monkeypatch):
    d = AdamWKernelDouble()
    monkeypatch.setattr(fused_optim, "KERNELS", d)
    monkeypatch.setattr(grad_sync, "KERNELS", d)
    return d


def _arena(seed=0):
    torch.manual_seed(seed)
    net = torch.nn.Sequential(torch.nn.Linear(6, 5), torch.nn.ReLU(), torch.nn.Linear(5, 3))
    extra = torch.nn.Parameter(torch.tensor([0.5, -1.0]))
    return net, extra, ParamArena(list(net.parameters()), [extra], device="cpu")


# ---- the switch ------------------------------------------------------------------------------------

def test_resolve_adamw_and_the_environment_variable(monkeypatch):
    monkeypatch.delenv("FRL_B200_ADAMW", raising=False)
    assert resolve_adamw() is False
    assert resolve_adamw(True) is True and resolve_adamw(False) is False
    monkeypatch.setenv("FRL_B200_ADAMW", "1")
    assert resolve_adamw() is True
    assert resolve_adamw(False) is False                 # the keyword wins
    monkeypatch.setenv("FRL_B200_ADAMW", "0")
    assert resolve_adamw() is False
    for bad in ("2", "true", "yes", "-1", ""):
        monkeypatch.setenv("FRL_B200_ADAMW", bad)
        with pytest.raises(ValueError, match="FRL_B200_ADAMW"):
            resolve_adamw()


ACCEPTED = [(False, OptimizerState.FP32, False), (True, OptimizerState.FP32, False),
            (False, OptimizerState.Q8, False), (False, OptimizerState.FP32, True)]   # (amsgrad, state, muon)


@pytest.mark.parametrize("amsgrad,state,muon", ACCEPTED)
def test_check_adamw_accepts_every_adam_form_and_the_factory_picks_it(double, amsgrad, state, muon):
    opts = ADAM._replace(amsgrad=amsgrad)
    fused_optim.check_adamw(opts, LayerAdaptation.NONE, state, False, True)
    _, _, arena = _arena()
    opt = fused_optim.create_fused_optimizer(arena, opts, LayerAdaptation.NONE, state, False, muon, True)
    want = fused_optim.FusedMuon if muon else fused_optim.FusedAdam8bit if state is OptimizerState.Q8 \
        else fused_optim.FusedAdam
    assert type(opt) is want and opt.adamw is True
    assert opt.hyper["decoupled_weight_decay"] is True and opt.hyper["amsgrad"] is amsgrad
    off = fused_optim.create_fused_optimizer(arena, opts, LayerAdaptation.NONE, state, False, muon)
    assert type(off) is want and off.adamw is False and off.hyper["decoupled_weight_decay"] is False


REFUSED = [
    (OptimOpts(algo=OptAlgorithm.SGD, lr=0.1), LayerAdaptation.NONE, OptimizerState.FP32, False, "'sgd'"),
    (OptimOpts(algo=OptAlgorithm.RMSPROP, lr=0.1), LayerAdaptation.NONE, OptimizerState.FP32, False, "'rmsprop'"),
    (OptimOpts(algo=OptAlgorithm.SGD, lr=0.1), LayerAdaptation.LARS, OptimizerState.FP32, False, "'lars'"),
    (ADAM, LayerAdaptation.LAMB, OptimizerState.FP32, False, "'lamb'"),
    (ADAM, LayerAdaptation.NONE, OptimizerState.FP32, True, "adafactor"),
]


@pytest.mark.parametrize("opts,la,state,adafactor,named", REFUSED)
def test_check_adamw_refuses_and_names_the_combination(opts, la, state, adafactor, named):
    with pytest.raises(ValueError, match="adamw cannot be combined") as e:
        fused_optim.check_adamw(opts, la, state, adafactor, True)
    assert named in str(e.value)
    fused_optim.check_adamw(opts, la, state, adafactor, False)          # off: nothing to refuse
    _, _, arena = _arena()
    if not adafactor and la is LayerAdaptation.NONE:
        with pytest.raises(ValueError, match="adamw"):
            fused_optim.create_fused_optimizer(arena, opts, la, state, False, False, True)


def test_q8_with_amsgrad_stays_refused():
    with pytest.raises(ValueError, match="8-bit state"):
        fused_optim.check_optimizer_state(ADAM._replace(amsgrad=True), LayerAdaptation.NONE, OptimizerState.Q8)
    _, _, arena = _arena()
    with pytest.raises(ValueError):
        fused_optim.create_fused_optimizer(arena, ADAM._replace(amsgrad=True), LayerAdaptation.NONE,
                                           OptimizerState.Q8, False, False, True)


def test_worker_args_field_sits_after_muon_and_the_pinned_tail_holds():
    f = SolverWorkerArgs._fields
    assert f.index("adamw") == f.index("muon") + 1
    assert f.index("adamw") < f.index("optimizer_state")
    assert SolverWorkerArgs._field_defaults["adamw"] is False
    assert f[f.index("optimizer_state") + 1] == "adafactor"
    assert f[-2:] == ("ema_decay", "grad_accumulation")
    assert f.index("adafactor") == f.index("optimizer_state") + 1 == len(f) - 3


# ---- dyn ---------------------------------------------------------------------------------------------

def test_dyn_values_carry_the_decay_factor_third():
    _, _, arena = _arena()
    for lr, wd in ((0.01, 1e-2), (3e-4, 0.1), (1e-3, 0.0)):
        opt = fused_optim.FusedAdam(arena, lr=lr, weight_decay=wd, adamw=True)
        adam = fused_optim.FusedAdam(arena, lr=lr, weight_decay=wd)
        vals = opt._dyn_values()
        assert len(vals) == 3 and vals[:2] == adam._dyn_values()
        assert vals[2] == float(f32(1.0 - lr * wd)) == float(decay_factor(lr, wd))
        opt.enable_dynamic_scalars()
        assert opt._dyn[2].item() == vals[2] and opt._dyn[3].item() == 0.0
    muon = fused_optim.FusedMuon(arena, lr=0.02, weight_decay=0.1, adamw=True)
    vals = muon._dyn_values()
    assert len(vals) == 4 and vals[2] == float(f32(1.0 - 0.02 * 0.1)) and vals[3] == 0.02
    muon.enable_dynamic_scalars()
    assert muon._muon_dyn()[2].item() == pytest.approx(0.02)           # K14's dyn[2]: the Muon lr
    plain = fused_optim.FusedMuon(arena, lr=0.02, weight_decay=0.1)
    plain.enable_dynamic_scalars()
    assert plain._muon_dyn() is plain._dyn and len(plain._dyn_values()) == 3


# ---- state dicts against CPU torch.optim.AdamW ----------------------------------------------------------

def _train(opt, params, steps=3, seed=5):
    gen = torch.Generator().manual_seed(seed)
    for _ in range(steps):
        for q in params:
            q.grad = torch.randn(q.shape, generator=gen)
        if isinstance(opt, fused_optim.FusedArenaOptimizer):
            for s in opt.arena.slots:
                opt.arena.grad[s.offset:s.end] = s.param.grad.flatten()
        opt.step()


@pytest.mark.parametrize("amsgrad", [False, True])
def test_state_dict_is_torch_adamw_format_in_both_directions(double, amsgrad):
    net, extra, arena = _arena()
    opt = fused_optim.FusedAdam(arena, lr=0.01, weight_decay=0.05, amsgrad=amsgrad, adamw=True)
    params = list(net.parameters()) + [extra]
    _train(opt, params)
    sd = opt.state_dict()
    ref_params = [torch.nn.Parameter(p.detach().clone()) for p in params]
    ref = torch.optim.AdamW(ref_params, lr=0.01, weight_decay=0.05, amsgrad=amsgrad)
    _train(ref, ref_params)
    rsd = ref.state_dict()
    assert sd["param_groups"][0].keys() == rsd["param_groups"][0].keys()
    assert sd["param_groups"][0]["decoupled_weight_decay"] is True
    assert sd["state"].keys() == rsd["state"].keys()
    for k in sd["state"]:
        assert sd["state"][k].keys() == rsd["state"][k].keys()
    ref.load_state_dict(sd)                                   # ours -> torch.optim.AdamW
    assert ref.param_groups[0]["decoupled_weight_decay"] is True
    for k, entry in sd["state"].items():
        for name, t in entry.items():
            assert torch.equal(ref.state[ref_params[k]][name], t)
    back = fused_optim.FusedAdam(arena, lr=1.0, weight_decay=0.0, amsgrad=amsgrad, adamw=True)
    back.load_state_dict(rsd)                                 # torch.optim.AdamW -> ours
    assert back._steps == 3 and back.hyper["lr"] == 0.01 and back.hyper["weight_decay"] == 0.05
    for s in arena.slots:
        for name in rsd["state"][s.index]:
            if name != "step":
                assert torch.equal(back._vec[name][s.offset:s.end].view(s.shape), rsd["state"][s.index][name])


def test_adamw_loads_an_adam_state_dict_and_keeps_reporting_its_rule(double):
    net, extra, arena = _arena()
    adam = fused_optim.FusedAdam(arena, lr=0.01, weight_decay=0.05)
    _train(adam, list(net.parameters()) + [extra])
    sd = adam.state_dict()
    assert sd["param_groups"][0]["decoupled_weight_decay"] is False
    opt = fused_optim.FusedAdam(arena, lr=0.5, weight_decay=0.0, adamw=True)
    opt.load_state_dict(sd)
    assert opt.hyper["decoupled_weight_decay"] is True and opt.state_dict()["param_groups"][0][
        "decoupled_weight_decay"] is True
    assert opt._steps == 3 and opt.hyper["weight_decay"] == 0.05
    for name in ("exp_avg", "exp_avg_sq"):
        assert torch.equal(opt._vec[name], adam._vec[name])


def test_adamw8_state_dict_is_torch_adamw_format(double):
    net, extra, arena = _arena()
    opt = fused_optim.FusedAdam8bit(arena, lr=0.01, weight_decay=0.05, adamw=True)
    _train(opt, list(net.parameters()) + [extra])
    assert ("adamw8_mt", len(arena.slots)) in double.calls and not any(c[0] == "adam8_mt" for c in double.calls)
    sd = opt.state_dict()
    assert sd["param_groups"][0]["decoupled_weight_decay"] is True
    ref = torch.optim.AdamW([torch.nn.Parameter(p.detach().clone()) for p in arena.all_params], lr=0.01)
    ref.load_state_dict(sd)
    back = fused_optim.FusedAdam8bit(arena, lr=1.0, adamw=True)
    back.load_state_dict(ref.state_dict())
    assert back.hyper["decoupled_weight_decay"] is True
    for n in ("exp_avg", "exp_avg_sq"):
        assert torch.equal(back.codes[n], opt.codes[n]) and torch.equal(back.absmax[n], opt.absmax[n])


def test_muon_adamw_group_splits_into_torch_adamw_and_joins_back():
    net, extra, arena = _arena()
    opt = fused_optim.FusedMuon(arena, lr=0.02, weight_decay=0.1, adamw=True)
    for s in arena.slots:
        opt._state("exp_avg")[s.offset:s.end] = torch.randn(s.numel)
        opt._state("exp_avg_sq")[s.offset:s.end] = torch.rand(s.numel)
    opt._steps = 2
    sd = opt.state_dict()
    muon_sd, adamw_sd = fused_optim.split_muon_state_dict(sd)
    assert adamw_sd["param_groups"][0]["decoupled_weight_decay"] is True
    ref = torch.optim.AdamW([torch.nn.Parameter(p.detach().clone()) for p in opt.adam_params], lr=0.02)
    ref.load_state_dict(adamw_sd)
    assert ref.state_dict()["param_groups"][0].keys() == adamw_sd["param_groups"][0].keys()
    joined = fused_optim.join_muon_state_dict(muon_sd, ref.state_dict())
    back = fused_optim.FusedMuon(arena, lr=1.0, adamw=True)
    back.load_state_dict(joined)
    assert back.hyper["decoupled_weight_decay"] is True and back._steps == 2
    for n in ("exp_avg", "exp_avg_sq"):
        for s in arena.slots:
            if n == "exp_avg" or not fused_optim.is_muon_slot(s):
                assert torch.equal(back._vec[n][s.offset:s.end], opt._vec[n][s.offset:s.end])


# ---- the doubles against float64 torch ----------------------------------------------------------------

@pytest.mark.parametrize("amsgrad", [False, True])
def test_doubles_match_float64_torch_adamw(amsgrad):
    gen = torch.Generator().manual_seed(7)
    n = 257
    p = torch.randn(n, generator=gen).clamp(-3, 3)
    m, v = torch.zeros(n), torch.zeros(n)
    vmax = torch.zeros(n) if amsgrad else None
    ref_p = torch.nn.Parameter(p.double().clone())
    ref = torch.optim.AdamW([ref_p], lr=0.01, weight_decay=0.1, amsgrad=amsgrad, foreach=False)
    d = AdamWKernelDouble()
    for step in range(1, 6):
        g = (torch.rand(n, generator=gen) * 1.5 + 0.5) * (torch.randint(0, 2, (n,), generator=gen) * 2 - 1)
        lr = 0.01 * (1.0, 0.6, 0.3, 0.8, 0.45)[step - 1]
        ref.param_groups[0]["lr"] = lr
        ref_p.data.copy_(p.double())                          # every step from the double's fp32 state
        st = ref.state[ref_p]
        if step > 1:
            st["exp_avg"].copy_(m.double()); st["exp_avg_sq"].copy_(v.double())
            if amsgrad:
                st["max_exp_avg_sq"].copy_(vmax.double())
        ref_p.grad = (g * 0.5).double()
        p0 = p.double().clone()
        ref.step()
        d.adamw(p, g, m, v, vmax, None, n, lr=lr, beta1=0.9, beta2=0.999, eps=1e-8, wd=0.1, step=step,
                grad_scale=0.5)
        pairs = [(p, ref_p.detach()), (m, st["exp_avg"]), (v, st["exp_avg_sq"])]
        if amsgrad:
            pairs.append((vmax, st["max_exp_avg_sq"]))
        # fp32 envelope: 26 roundings of the magnitudes the weight is formed from (|p0| and the
        # step, at most lr / (1 - beta1^t) * |m| / denom <= 10 lr here), relative for the moments
        bound = 26 * 2.0 ** -24 * (p0.abs() + ref_p.detach().abs() + 10 * lr)
        assert ((p.double() - ref_p.detach()).abs() <= bound).all(), step
        for got, want in pairs[1:]:
            np.testing.assert_allclose(got.double().numpy(), want.numpy(), rtol=2e-6, atol=2e-7)


def test_wd_zero_gives_the_adam_doubles_bytes():
    gen = torch.Generator().manual_seed(9)
    n = 300
    base = [torch.randn(n, generator=gen) for _ in range(2)] + [torch.rand(n, generator=gen) * 0.01]
    for amsgrad in (False, True):
        a = [t.clone() for t in base] + ([torch.rand(n, generator=gen) * 0.01] if amsgrad else [None])
        w = [None if t is None else t.clone() for t in a]
        g = torch.randn(n, generator=gen).to(torch.bfloat16)
        lp_a, lp_w = torch.zeros(n, dtype=torch.bfloat16), torch.zeros(n, dtype=torch.bfloat16)
        kw = dict(lr=3e-3, beta1=0.9, beta2=0.999, eps=1e-8, wd=0.0, step=4, grad_scale=0.7)
        KernelDouble().adam(a[0], g, a[1], a[2], a[3], lp_a, n, **kw)
        AdamWKernelDouble().adamw(w[0], g, w[1], w[2], w[3], lp_w, n, **kw)
        for x, y in zip(a + [lp_a], w + [lp_w]):
            if x is not None:
                assert torch.equal(x.view(torch.int16 if x.dtype == torch.bfloat16 else torch.int32),
                                   y.view(torch.int16 if y.dtype == torch.bfloat16 else torch.int32))


def test_fp32_double_rounds_the_decay_on_its_own():
    p = np.array([1.0000001, -2.5, 3.0e-3], dtype=f32)
    z = np.zeros(3, dtype=f32)
    got, _, _, _ = adamw_step(p, z, z, z, None, lr=0.1, beta1=0.9, beta2=0.999, eps=1e-8, wd=0.3, step=1)
    assert np.array_equal(got, (p * f32(1.0 - 0.1 * 0.3)).astype(f32))


# ---- entry points: every argument check before any launch ----------------------------------------------

def test_entry_points_refuse_bad_arguments_and_name_themselves():
    lib = _native.lib()
    ok = 1 << 20
    before = lib.frl_launch_count()

    def last():
        return lib.frl_last_error().decode()

    cases = []
    cases.append(("frl_adamw", lib.frl_adamw(ok, ok, None, ok, None, None, 64, 0.1, 0.9, 0.999, 1e-8, 0.1, 1, 1.0,
                                             None, None, 0, None)))
    cases.append(("frl_adamw", lib.frl_adamw(ok, ok, ok, ok, None, None, 64, 0.1, 0.9, 0.999, 1e-8, 0.1, 0, 1.0,
                                             None, None, 0, None)))
    cases.append(("frl_adamw", lib.frl_adamw(ok + 4, ok, ok, ok, None, None, 64, 0.1, 0.9, 0.999, 1e-8, 0.1, 1,
                                             1.0, None, None, 0, None)))
    cases.append(("frl_adamw", lib.frl_adamw(ok, ok, ok, ok, None, None, 64, 0.1, 0.9, 0.999, 1e-8, 0.1, 1, 1.0,
                                             None, None, 7, None)))
    cases.append(("frl_adamw_mt", lib.frl_adamw_mt(ok, None, ok, None, None, ok, ok, ok, 4, 0.1, 0.9, 0.999, 1e-8,
                                                   0.1, 1, 1.0, None, None, None)))
    cases.append(("frl_adamw_mt", lib.frl_adamw_mt(ok, ok, ok, None, None, None, ok, ok, 4, 0.1, 0.9, 0.999, 1e-8,
                                                   0.1, 1, 1.0, None, None, None)))
    cases.append(("frl_adamw_mt", lib.frl_adamw_mt(ok, ok, ok, None, None, ok, ok, ok, 4, 0.1, 0.9, 0.999, 1e-8,
                                                   0.1, 0, 1.0, None, None, None)))

    def adamw8(**kw):
        a = dict(p=ok, mq=ok, vq=ok, ma=ok, va=ok, lp=None, segs=ok, nt=4, ns=2, qb=ok, fl=ok, step=1)
        a.update(kw)
        return lib.frl_adamw8_mt(a["p"], a["mq"], a["vq"], a["ma"], a["va"], a["lp"], a["segs"], ok, ok, a["nt"],
                                 a["ns"], a["qb"], a["fl"], 0.1, 0.9, 0.999, 1e-8, 0.1, a["step"], 1.0, None, None,
                                 None)

    for kw in (dict(p=None), dict(mq=None), dict(fl=None), dict(segs=None), dict(step=0), dict(p=ok + 4),
               dict(lp=ok + 2), dict(nt=-1), dict(nt=4, ns=0)):
        cases.append(("frl_adamw8_mt", adamw8(**kw)))
        cases[-1] += (last(),)
    for name, rc, *msg in cases:
        assert rc < 0, (name, rc)
    for name, rc, *msg in cases:
        if msg:
            assert name in msg[0], msg

    def nvls(**kw):
        a = dict(p=ok, m=ok, v=ok, n=64, rank=0, world=2, step=1, blocks=4, g_dtype=0)
        a.update(kw)
        return lib.frl_nvls_adamw(a["p"], a["m"], a["v"], None, ok, ok, a["n"], a["rank"], a["world"], ok, 0, ok,
                                  a["blocks"], 0.1, 0.9, 0.999, 1e-8, 0.1, a["step"], 1.0, None, a["g_dtype"], 0,
                                  None)

    for kw in (dict(m=None), dict(step=0), dict(world=1), dict(rank=2), dict(n=12), dict(p=ok + 4),
               dict(blocks=0), dict(g_dtype=7)):
        rc = nvls(**kw)
        assert rc < 0 and "frl_nvls_adamw" in last(), (kw, rc, last())
    # each of the flat / mt forms names itself too
    assert lib.frl_adamw(ok, ok, None, ok, None, None, 64, 0.1, 0.9, 0.999, 1e-8, 0.1, 1, 1.0, None, None, 0,
                         None) < 0 and "frl_adamw:" in last()
    assert lib.frl_adamw_mt(ok, None, ok, None, None, ok, ok, ok, 4, 0.1, 0.9, 0.999, 1e-8, 0.1, 1, 1.0, None, None,
                            None) < 0 and "frl_adamw_mt" in last()
    assert lib.frl_launch_count() == before
    assert adamw8(nt=0, ns=0) == 0 and lib.frl_launch_count() == before


# ---- GradBucketPipeline launch sequences ------------------------------------------------------------------

class AdamWRecordingDouble(tpl.RecordingDouble, AdamWKernelDouble):
    """``test_pipeline_launches.RecordingDouble`` with the AdamW entry points logged."""

    def adamw(self, p, g, m, v, vmax, p_lp, n, **kw):
        self._log("adamw", self._range(g, n), kw["grad_scale"], kw.get("grad_scale_dev"))
        AdamWKernelDouble.adamw(self, p, g, m, v, vmax, p_lp, n, **kw)

    def adamw_mt(self, p, m, v, vmax, p_lp, table, **kw):
        self._log("adamw_mt", self._slots(table), kw["grad_scale"])
        AdamWKernelDouble.adamw_mt(self, p, m, v, vmax, p_lp, table, **kw)


def _as_adamw(lines):
    out = []
    for line in lines:
        head, _, rest = line.partition(" ")
        out.append({"adam": "adamw", "adam_mt": "adamw_mt"}.get(head, head) + " " + rest)
    return out


def _adamw_factory(orig):
    def create(arena, optim_opts, la=LayerAdaptation.NONE, *a):
        return orig(arena, optim_opts, la, OptimizerState.FP32, False, False, True)
    return create


def _torch_adamw_reference(clip, k, xs):
    net = tpl._Net()
    params = net.model_params() + [net.extra]
    o = tpl.OPTS["adam"][0]
    ref = torch.optim.AdamW(params, lr=o.lr, weight_decay=o.weightDecay, eps=o.epsilon)
    lo = 0
    for j, mb in enumerate(accumulation_plan(tpl.N_MB, k, tpl.B, tpl.N_ROWS)):
        if mb.closes:
            hi = j * tpl.B + mb.rows
            ref.zero_grad()
            net.loss(xs[lo:hi], False).backward()
            if clip:
                torch.nn.utils.clip_grad_norm_(net.model_params(), clip)
            ref.step()
            lo = hi
    return [p.detach().clone() for p in net.parameters()]


@pytest.mark.parametrize("in_place", [True, False], ids=["in-place", "arena"])
@pytest.mark.parametrize("k", [1, 3])
@pytest.mark.parametrize("clip", [0.0, tpl.CLIP], ids=["noclip", "clip"])
def test_one_rank_launch_sequence_is_adams_with_adamw_kernels(monkeypatch, clip, k, in_place):
    d = AdamWRecordingDouble()
    monkeypatch.setattr(fused_optim, "KERNELS", d)
    monkeypatch.setattr(grad_sync, "KERNELS", d)
    monkeypatch.setattr(multi_tensor, "grad_usable_in_place", tpl._in_place)
    monkeypatch.setattr(fused_optim, "create_fused_optimizer", _adamw_factory(fused_optim.create_fused_optimizer))
    key = tpl._key("adam", clip, False, k, in_place)
    want = _as_adamw(tpl.EXPECTED[key]) * (tpl.N_MB if k == 1 else 1)
    assert want != tpl.EXPECTED[key] * (tpl.N_MB if k == 1 else 1)
    xs = torch.randn(tpl.N_ROWS, 7, generator=torch.Generator().manual_seed(11))
    log, params = tpl._run(d, "adam", clip, k, in_place, False, False, xs)
    assert log == want
    for a, b in zip(params, _torch_adamw_reference(clip, k, xs)):
        np.testing.assert_allclose(a.numpy(), b.numpy(), rtol=1e-4, atol=1e-6)
    log, deferred = tpl._run(d, "adam", clip, k, in_place, True, False, xs)
    assert log == want
    for a, b in zip(deferred, params):
        assert torch.equal(a, b)


_CONFIGS_2RANKS = list(itertools.product((0.0, tpl.CLIP), (1, 3), (True, False)))


def _rank_main(rank, world, port, out_dir):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    d = AdamWRecordingDouble()
    fused_optim.KERNELS = grad_sync.KERNELS = d
    fused_optim.create_fused_optimizer = _adamw_factory(fused_optim.create_fused_optimizer)
    multi_tensor.grad_usable_in_place = tpl._in_place
    all_reduce = dist.all_reduce

    def logged_all_reduce(t, *args, **kw):
        d.log.append("all_reduce %s" % d._range(t, t.numel()))
        return all_reduce(t, *args, **kw)

    dist.all_reduce = logged_all_reduce
    xs = torch.randn(tpl.N_ROWS * world, 7, generator=torch.Generator().manual_seed(12))
    out = {}
    for clip, k, in_place in _CONFIGS_2RANKS:
        out[tpl._key("adam", clip, False, k, in_place)] = [
            tpl._run(d, "adam", clip, k, in_place, defer, False, xs, rank, world) for defer in (False, True)]
    torch.save(out, os.path.join(out_dir, f"r{rank}.pt"))
    dist.destroy_process_group()


def test_two_rank_launch_sequences_are_adams_with_adamw_kernels(tmp_path):
    world = 2
    port = 37600 + (os.getpid() % 2000)
    mp.spawn(_rank_main, args=(world, port, str(tmp_path)), nprocs=world, join=True)
    r0, r1 = torch.load(tmp_path / "r0.pt"), torch.load(tmp_path / "r1.pt")
    keys = [tpl._key("adam", c, False, k, i) for c, k, i in _CONFIGS_2RANKS]
    assert sorted(r0) == sorted(keys)
    for key in keys:
        want = _as_adamw(tpl.EXPECTED_2RANKS[key]) * (tpl.N_MB if " k1 " in key else 1)
        assert any(line.startswith("adamw") for line in want)
        for (log0, p0), (log1, p1) in zip(r0[key], r1[key]):
            assert log0 == log1 == want, key
            for a, b in zip(p0, p1):
                assert torch.equal(a, b), key
        for a, b in zip(r0[key][0][1], r0[key][1][1]):
            assert torch.equal(a, b), key
