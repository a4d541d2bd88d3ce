"""AdamW (the ``frl_adamw*`` kernels) on the GPU, by the method of ``test_gpu_optim_paths.py``.

Reference.  ``torch.optim.AdamW(foreach=False)`` on float64 copies, fed exactly the gradient the
kernel reads (bf16-rounded when the gradient is bf16, times ``grad_scale`` and the device clip
coefficient), every step started from the kernel's own fp32 state.

Tolerance: the fp32 envelope of ``test_gpu_optim_paths``,

    |got - ref| <= c * (U * mag + ETA),    U = 2^-24,  ETA = 2^-150,

with ``mag`` the float64 sum of the magnitudes of the terms a value is formed from.  For AdamW
the gradient carries no decay term, so mag(g) = |g|, and the weights' magnitude is
|p0| + |ref| + lr * (magnitude of the step's update).  ``c`` counts the fp32 roundings on the
longest chain:

    AdamW 26 = Adam's 24 (gradient 3; exp_avg 3; exp_avg_sq 10, halved by sqrt to 5, sqrt,
               / bc2_sqrt, bc2_sqrt, + eps 4; m / denom 1; step_size and the fma 2; headroom)
             + 1 for the decay factor's conversion fp32(1 - lr * wd)
             + 1 for its product p * decay, rounded on its own before the update's fma.

The decay's two roundings are relative to |p0|, which the weights' magnitude holds.

Second reference: ``torch.optim.AdamW`` in its default form (foreach, fp32) on the same GPU, from
the same fp32 state and fp32 gradient, 2^20 + 3 elements over 4 steps, weights and every state
vector.  Measured on an H100 80GB HBM3 (SXM, 700 W power limit) with torch 2.11:

    rule               elements differing   largest distance   in units of U * mag
    AdamW                     772435              1035 ulps              3.678
    AdamW, amsgrad           1536282              1035 ulps              3.678

As for Adam, the ulp counts come from weights that cancel to far below their terms; against the
magnitude of the terms torch's fp32 result is within 4 roundings of the kernel's.  The test pins
these distances rounded up to a half unit (``DISTANCE_TO_FP32_TORCH``).
"""
import json
import math
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

import frl_b200  # noqa: F401
from frl_b200 import _native, fused_optim, synthetic
from frl_b200.multi_tensor import GradSegTable
from frl_b200.solver import Solver, SolverWorkerArgs
from frl_b200.types import Device, OptAlgorithm, OptimizerState, OptimOpts, Precision, Split
from test_gpu_optim_paths import (ETA, LR_SCALE, SCALE, SENTINEL, U, _assert_sentinels, _grad, _MtCase, _padded,
                                  _three_waves, _ulps, _weights, assert_shadow, assert_within)
import test_gpu_adam8 as a8

pytestmark = pytest.mark.gpu
DEV = "cuda"
C_ADAMW = 26
HP = dict(beta1=0.9, beta2=0.999, eps=1e-8)
BASE_LR = 1e-2
WD = 0.1
VARIANTS = {"adamw": False, "adamw_amsgrad": True}
STATES = {False: ("exp_avg", "exp_avg_sq"), True: ("exp_avg", "exp_avg_sq", "max_exp_avg_sq")}
# largest |kernel - fp32 torch.optim.AdamW (foreach)| / (U * mag + ETA), as measured (module docstring)
DISTANCE_TO_FP32_TORCH = {"adamw": 4.0, "adamw_amsgrad": 4.0}


def _kw(lr, wd, step):
    return dict(lr=lr, wd=wd, step=step, **HP)


def launch_flat(ams, p, g, states, lp, n, *, lr, wd, step, coef=None, dyn=None, adamw=True):
    gs, gs_dev = (SCALE, None) if coef is None else (0.5, coef)
    s = list(states) + [None] * 3
    (_native.adamw if adamw else _native.adam)(p, g, s[0], s[1], s[2] if ams else None, lp, n, grad_scale=gs,
                                               grad_scale_dev=gs_dev, dyn=dyn, **_kw(lr, wd, step))


def launch_mt(ams, p, states, lp, table, *, lr, wd, step, coef=None, dyn=None, adamw=True):
    gs, gs_dev = (SCALE, None) if coef is None else (0.5, coef)
    s = list(states) + [None] * 3
    (_native.adamw_mt if adamw else _native.adam_mt)(p, s[0], s[1], s[2] if ams else None, lp, table,
                                                     grad_scale=gs, grad_scale_dev=gs_dev, dyn=dyn,
                                                     **_kw(lr, wd, step))


def reference_step(ams, p, g, states, *, lr, wd, step, dtype=torch.float64, foreach=False):
    param = torch.nn.Parameter(p.to(dtype, copy=True))
    opt = torch.optim.AdamW([param], lr=lr, weight_decay=wd, betas=(HP["beta1"], HP["beta2"]), eps=HP["eps"],
                            amsgrad=ams, foreach=foreach)
    st = opt.state[param]
    for name, s in zip(STATES[ams], states):
        st[name] = s.to(dtype, copy=True)
    st["step"] = torch.tensor(float(step - 1))
    param.grad = g.to(dtype)
    opt.step()
    return param.detach(), [opt.state[param][name] for name in STATES[ams]]


def envelope(ams, p0, g, s0, ref_p, ref_s, *, lr, step):
    b1, b2 = HP["beta1"], HP["beta2"]
    mag_g = g.abs()
    mag_m = s0[0].abs() + (1 - b1) * (mag_g + s0[0].abs())
    mag_v = b2 * s0[1].abs() + (1 - b2) * mag_g * mag_g
    mags = [mag_m, mag_v] + ([torch.maximum(s0[2].abs(), mag_v)] if ams else [])
    denom = ref_s[-1].sqrt() / math.sqrt(1 - b2 ** step) + HP["eps"]
    step_mag = lr / (1 - b1 ** step) * mag_m / denom
    return [C_ADAMW * (U * (p0.abs() + ref_p.abs() + step_mag) + ETA)] + [C_ADAMW * (U * m + ETA) for m in mags]


def check_step(ams, got_p, got_s, p0, g, s0, *, lr, wd, step, what):
    ref_p, ref_s = reference_step(ams, p0, g, s0, lr=lr, wd=wd, step=step)
    bounds = envelope(ams, p0.double(), g.double(), [s.double() for s in s0], ref_p, ref_s, lr=lr, step=step)
    assert_within(got_p, ref_p, bounds[0], what + " weights")
    for name, got, ref, b in zip(STATES[ams], got_s, ref_s, bounds[1:]):
        assert_within(got, ref, b, "%s %s" % (what, name))


# ---- K2: every instantiation against float64 torch.optim.AdamW ------------------------------------------

LENGTHS = [1, 3, 4096, 4099, 4096 + 2500 + 2, "three_waves"]


@pytest.mark.parametrize("length", LENGTHS)
@pytest.mark.parametrize("lp", [False, True], ids=["no_shadow", "shadow"])
@pytest.mark.parametrize("gdt", [torch.float32, torch.bfloat16], ids=["g_f32", "g_bf16"])
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_flat_adamw_matches_float64_torch_adamw(variant, gdt, lp, length):
    ams = VARIANTS[variant]
    i = LENGTHS.index(length)
    n = _three_waves() if length == "three_waves" else length
    coef = torch.tensor([0.75], device=DEV) if i % 2 else None
    gen = torch.Generator(device=DEV).manual_seed(2000 + i)
    pbuf, p = _padded(n, torch.float32, SENTINEL)
    p.copy_(_weights(n, gen))
    sbufs = [_padded(n, torch.float32, SENTINEL) for _ in STATES[ams]]
    states = [s for _, s in sbufs]
    for s in states:
        s.zero_()
    lbuf, shadow = _padded(n, torch.bfloat16, SENTINEL) if lp else (None, None)
    gbuf, g = _padded(n, gdt, float("nan"))
    for step in range(1, 5):
        lr = BASE_LR * LR_SCALE[step - 1]
        g.copy_(_grad(n, gen))
        p0, s0 = p.clone(), [s.clone() for s in states]
        launch_flat(ams, p, g, states, shadow, n, lr=lr, wd=WD, step=step, coef=coef)
        check_step(ams, p, states, p0, g.double() * SCALE, s0, lr=lr, wd=WD, step=step,
                   what="n=%d step %d" % (n, step))
        if lp:
            assert_shadow(shadow, p, "step %d" % step)
    for name, buf in [("weights", pbuf), ("shadow", lbuf)] + list(zip(STATES[ams], (b for b, _ in sbufs))):
        if buf is not None:
            _assert_sentinels(buf, n, name)


# ---- K2-mt: every instantiation -----------------------------------------------------------------------

@pytest.mark.parametrize("lp", [False, True], ids=["no_shadow", "shadow"])
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_mt_adamw_matches_float64_torch_adamw(variant, lp):
    ams = VARIANTS[variant]
    case = _MtCase("adam_amsgrad" if ams else "adam", lp, seed=23)
    coef = torch.tensor([0.75], device=DEV)
    idx = case.idx
    for step in range(1, 5):
        lr = BASE_LR * LR_SCALE[step - 1]
        g = case.new_grads()
        p0, s0 = case.p[idx].clone(), [s[idx].clone() for s in case.states]
        launch_mt(ams, case.p, case.states, case.shadow, case.table, lr=lr, wd=WD, step=step, coef=coef)
        check_step(ams, case.p[idx], [s[idx] for s in case.states], p0, g, s0, lr=lr, wd=WD, step=step,
                   what="mt step %d" % step)
        if lp:
            assert_shadow(case.shadow[idx], case.p[idx], "mt step %d" % step)
        case.assert_pad_and_outside("mt step %d" % step)


# ---- dyn and CUDA-graph replay ------------------------------------------------------------------------------

def _dyn(lr, wd, step):
    b1, b2 = HP["beta1"], HP["beta2"]
    return torch.tensor([-(lr / (1 - b1 ** step)), (1 - b2 ** step) ** 0.5, 1.0 - lr * wd, 0.0],
                        dtype=torch.float32, device=DEV)


@pytest.mark.parametrize("form", ["flat", "mt"])
def test_dyn_block_and_graph_replay_equal_by_value_launches(form):
    """A wrong by-value lr / step / wd with a correct ``dyn`` == the by-value launch; one launch captured
    in a CUDA graph, replayed over 5 steps with lr changing and the block uploaded before each replay,
    == eager launches.  Bit for bit."""
    n = 4096 * 3 + 5
    gen = torch.Generator(device=DEV).manual_seed(4)
    p_a = _weights(n, gen)
    g = _grad(n, gen)
    table = None
    if form == "mt":
        from test_gpu_optim_paths import _Slot
        slots = [_Slot(0, 0, n)]
        table = GradSegTable(slots, torch.device(DEV))
        table.point(slots[0], g.data_ptr(), g.dtype)
        table.upload()

    def launch(p, states, *, lr, wd, step, dyn=None):
        if form == "flat":
            launch_flat(True, p, g, states, None, n, lr=lr, wd=wd, step=step, dyn=dyn)
        else:
            launch_mt(True, p, states, None, table, lr=lr, wd=wd, step=step, dyn=dyn)

    s_a = [torch.zeros(n, device=DEV) for _ in range(3)]
    p_b, s_b = p_a.clone(), [s.clone() for s in s_a]
    p_c, s_c = p_a.clone(), [s.clone() for s in s_a]
    dyn = torch.zeros(4, device=DEV)
    stream = torch.cuda.Stream()
    graph = None
    for step in range(1, 6):
        lr = BASE_LR * LR_SCALE[step - 1]
        launch(p_a, s_a, lr=lr, wd=WD, step=step)
        launch(p_b, s_b, lr=123.0, wd=0.7, step=99, dyn=_dyn(lr, WD, step))
        dyn.copy_(_dyn(lr, WD, step))
        if graph is None:
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph, stream=stream):
                launch(p_c, s_c, lr=7.0, wd=0.5, step=50, dyn=dyn)
        graph.replay()
    torch.cuda.synchronize()
    for a, b, c in zip([p_a] + s_a, [p_b] + s_b, [p_c] + s_c):
        assert torch.equal(a, b) and torch.equal(a, c)


# ---- against fp32 torch.optim.AdamW (foreach) ----------------------------------------------------------------

@pytest.mark.parametrize("variant", list(VARIANTS))
def test_distance_to_fp32_torch_adamw(variant):
    ams = VARIANTS[variant]
    n = (1 << 20) + 3
    gen = torch.Generator(device=DEV).manual_seed(3)
    p = _weights(n, gen)
    states = [torch.zeros(n, device=DEV) for _ in STATES[ams]]
    worst, differ, worst_env = 0, 0, 0.0
    for step in range(1, 5):
        lr = BASE_LR * LR_SCALE[step - 1]
        g = _grad(n, gen)
        p0, s0 = p.clone(), [s.clone() for s in states]
        launch_flat(ams, p, g, states, None, n, lr=lr, wd=WD, step=step)
        g32 = g * SCALE
        ref_p, ref_s = reference_step(ams, p0, g32, s0, lr=lr, wd=WD, step=step, dtype=torch.float32, foreach=True)
        bounds = envelope(ams, p0.double(), g32.double(), [s.double() for s in s0], ref_p.double(),
                          [s.double() for s in ref_s], lr=lr, step=step)
        for got, ref, b in zip([p] + states, [ref_p] + ref_s, bounds):
            worst = max(worst, int(_ulps(got, ref).max()))
            differ += int((got != ref).sum())
            worst_env = max(worst_env, float(((got.double() - ref.double()).abs() / (b / C_ADAMW)).max()))
    print("fp32 torch.optim.AdamW (foreach) vs kernel: %s max %d ulps, %d elements differ, max |diff| / (U mag + "
          "ETA) %.3f" % (variant, worst, differ, worst_env))
    assert worst_env <= DISTANCE_TO_FP32_TORCH[variant], (variant, worst_env)


# ---- wd = 0: AdamW's bytes are Adam's ----------------------------------------------------------------------

def test_wd_zero_gives_adams_bytes_on_k2_k2mt_and_k2q8():
    n = 4096 * 2 + 7
    for ams in (False, True):
        for gdt in (torch.float32, torch.bfloat16):
            gen = torch.Generator(device=DEV).manual_seed(8)
            p = _weights(n, gen)
            g = _grad(n, gen).to(gdt)
            runs = []
            for adamw in (False, True):
                q, st = p.clone(), [torch.zeros(n, device=DEV) for _ in STATES[ams]]
                lp = torch.zeros(n, dtype=torch.bfloat16, device=DEV)
                for step in range(1, 4):
                    launch_flat(ams, q, g, st, lp, n, lr=1e-2, wd=0.0, step=step, adamw=adamw)
                runs.append([q, lp] + st)
            for a, b in zip(*runs):
                assert torch.equal(a.view(torch.int16 if a.dtype == torch.bfloat16 else torch.int32),
                                   b.view(torch.int16 if b.dtype == torch.bfloat16 else torch.int32))
    for ams in (False, True):
        runs = []
        for adamw in (False, True):
            case = _MtCase("adam_amsgrad" if ams else "adam", True, seed=29)
            for step in range(1, 4):
                case.new_grads()
                launch_mt(ams, case.p, case.states, case.shadow, case.table, lr=1e-2, wd=0.0, step=step,
                          adamw=adamw)
            runs.append(case.vectors())
        for a, b in zip(*runs):
            assert torch.equal(a, b)
    runs = []
    for fn in (_native.adam8_mt, _native.adamw8_mt):
        case = a8._Case(torch.bfloat16, True, seed=31)
        for step in range(1, 4):
            fn(case.p, case.codes["m"], case.codes["v"], case.absmax["m"], case.absmax["v"], case.shadow, case.table,
               case.qbase, case.flags, lr=1e-2, wd=0.0, step=step, grad_scale=0.5, **HP)
            case.new_grads()
        runs.append(case.snapshot())
    for a, b in zip(*runs):
        assert torch.equal(a, b)


# ---- K2-q8: decode -> AdamW -> encode ----------------------------------------------------------------------

@pytest.mark.parametrize("gdt", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("lp", [False, True])
def test_q8_adamw_equals_adamw_mt_from_the_decoded_state_and_float64_adamw(gdt, lp):
    """Each step: K2-q8 AdamW against (a) ``frl_adamw_mt`` from the decoded fp32 moments, bit for bit in
    the weights, and the codes of its new moments; (b) float64 ``torch.optim.AdamW`` from the decoded
    state, within the envelope."""
    case = a8._Case(gdt, lp, seed=41)
    coef = torch.tensor([0.6], device=DEV)
    for step in range(1, 4):
        lr = 1e-2 * LR_SCALE[step - 1]
        m0, v0 = case.decoded()
        p0 = case.p.clone()
        p_mt, m_mt, v_mt = p0.clone(), m0.clone(), v0.clone()
        lp_mt = case.shadow.clone() if lp else None
        # frl_adamw_mt with the same scales: model slots take the clip coefficient, others do not
        model = [s for s in case.slots if s.is_model]
        other = [s for s in case.slots if not s.is_model]
        for slots, c in ((model, coef), (other, None)):
            t = GradSegTable(slots, torch.device(DEV))
            for s in slots:
                t.point(s, case.grads[s.index].data_ptr(), case.grads[s.index].dtype)
            t.upload()
            _native.adamw_mt(p_mt, m_mt, v_mt, None, lp_mt, t, lr=lr, wd=WD, step=step, grad_scale=0.5,
                             grad_scale_dev=c, **HP)
        _native.adamw8_mt(case.p, case.codes["m"], case.codes["v"], case.absmax["m"], case.absmax["v"], case.shadow,
                          case.table, case.qbase, case.flags, lr=lr, wd=WD, step=step, grad_scale=0.5,
                          grad_scale_dev=coef, **HP)
        torch.cuda.synchronize()
        assert torch.equal(case.p, p_mt), step
        if lp:
            assert torch.equal(case.shadow, lp_mt), step
        want_m = torch.zeros(case.n, dtype=torch.uint8, device=DEV)
        want_ma = torch.zeros_like(case.absmax["m"])
        _native.q8_encode_mt(m_mt, want_m, want_ma, _native.Q8_EXP_AVG, case.table, case.qbase)
        assert torch.equal(want_m, case.codes["m"]) and torch.equal(want_ma, case.absmax["m"]), step
        want_v = torch.zeros(case.n, dtype=torch.uint8, device=DEV)
        want_va = torch.zeros_like(case.absmax["v"])
        _native.q8_encode_mt(v_mt, want_v, want_va, _native.Q8_EXP_AVG_SQ, case.table, case.qbase)
        assert torch.equal(want_v, case.codes["v"]) and torch.equal(want_va, case.absmax["v"]), step
        g_eff = case.g_eff(0.5 * 0.6, 0.5)
        idx = torch.cat([torch.arange(s.offset, s.end, device=DEV) for s in case.slots])
        check_step(False, case.p[idx], [m_mt[idx], v_mt[idx]], p0[idx], g_eff[idx], [m0[idx], v0[idx]], lr=lr,
                   wd=WD, step=step, what="q8 step %d" % step)
        case.new_grads()


# ---- every new instantiation is launched ----------------------------------------------------------------------

FLAT = sorted("frl::AdamWRule<%s>,frl::%s,%d,%s" % (a, gv, ns, lp) for a, ns in (("false", 2), ("true", 3))
              for gv in ("f32x4", "bf16x4") for lp in ("false", "true"))
MT = sorted("frl::AdamWRule<%s>,%d,%s" % (a, ns, lp) for a, ns in (("false", 2), ("true", 3))
            for lp in ("false", "true"))
Q8 = sorted("frl::AdamWRule<false>,%s" % lp for lp in ("false", "true"))


def test_every_adamw_instantiation_is_launched():
    """Every new K2, K2-mt and K2-q8 instantiation launches, the K2 and K2-mt ones each checked
    against float64.  The profiler runs in a process of its own (tests/run_adamw_instantiations.py),
    so this process never starts a profiling session: one that ended here would hide kernels from
    later sessions, such as the one in test_gpu_optim_paths.py."""
    script = os.path.join(os.path.dirname(os.path.abspath(__file__)), "run_adamw_instantiations.py")
    res = subprocess.run([sys.executable, script], capture_output=True, text=True, timeout=600)
    assert res.returncode == 0 and "ADAMW_INSTANTIATIONS_OK" in res.stdout, res.stdout[-3000:] + res.stderr[-3000:]
    line = [ln for ln in res.stdout.splitlines() if ln.startswith("INSTANTIATIONS ")][-1]
    seen = json.loads(line[len("INSTANTIATIONS "):])
    print(seen)
    assert seen["flat"] == FLAT and len(FLAT) == 8
    assert seen["mt"] == MT and len(MT) == 4
    assert seen["q8"] == Q8 and len(Q8) == 2


# ---- through Solver.build_worker ------------------------------------------------------------------------------

def _worker(precision=Precision.FP32, seed=0, lr=1e-3, wd=0.1, adamw=True, graph=False, **kw):
    ns = synthetic.api_namespace("frl_b200")
    t = ns.types
    save_dir = tempfile.mkdtemp(prefix="frl_b200_adamw_")
    torch.manual_seed(seed)
    problem = synthetic.make_mlp_problem(ns, save_dir, n_train=8, width=512, n_classes=100, reg_dim=16, depth=3)
    run_opts = t.RunOpts(optim=t.OptimOpts(algo=t.OptAlgorithm.ADAM, lr=lr, weightDecay=wd, momentum=0.95),
                         batchSize=256, nEpochs=1, numThreads=0, singleThreaded=True, numVisualizedSamples=0)
    args = SolverWorkerArgs(run_opts=run_opts, problem=problem, save_dir=save_dir, run_device=Device.GPU,
                            node_idx=0, node_count=1, rank=0, local_rank=0, world_size=1, group_name=None,
                            init_method="", precision=precision, adamw=adamw, graph_step=graph, **kw)
    worker, _, _ = Solver.build_worker(args)
    worker.model.train()
    worker.criterion.train()
    return worker, problem


def _batches(n, width=512, seed=1234):
    gen = torch.Generator().manual_seed(seed)
    w = torch.randn(width, 100, generator=gen) / width ** 0.5
    out = []
    for _ in range(n):
        x = torch.randn(256, width, generator=gen)
        out.append((x, (x @ w).argmax(1), torch.randn(256, 16, generator=gen) * 0.1 + x[:, :16]))
    return out


def _train(worker, batches, start=0, lrs=None):
    rows = []
    for i, (x, y, r) in enumerate(batches, start):
        if lrs is not None:
            worker.optimizer.hyper["lr"] = lrs[i % len(lrs)]
        _, total, _, _ = worker._pass_one_minibatch(i, Split.TRAIN, [x.cuda()], [(y.cuda(),), (r.cuda(),)])
        rows.append(float(total.detach()))
        del total
    torch.cuda.synchronize()
    return rows


def _params(worker):
    return [p.detach().float().clone() for p in list(worker.model.parameters()) + list(worker.criterion.parameters())]


def _gap(a, b, p0):
    return max(((x - y).norm() / (y - q).norm().clamp_min(1e-30)).item() for x, y, q in zip(a, b, p0))


def _torch_loop(worker, problem, batches, make_opts):
    from oracle import ref_loop
    ns = synthetic.api_namespace("frl_b200")
    ref_problem = synthetic.make_mlp_problem(ns, tempfile.mkdtemp(prefix="frl_b200_adamw_ref_"), n_train=8,
                                             width=512, n_classes=100, reg_dim=16, depth=3)
    ref = ref_problem.get_model().cuda()
    ref.load_state_dict(worker.model.state_dict())
    crit = ref_problem.get_criterion().cuda()
    crit.load_state_dict(worker.criterion.state_dict())
    mods, weights, names = list(crit.loss_modules), list(crit.loss_weights), list(crit.loss_names)
    params = list(ref.parameters()) + list(crit.parameters())
    opts = make_opts(ref, params)
    ref.train()
    crit.train()
    rows = []
    for x, y, r in batches:
        for o in opts:
            o.zero_grad()
        total, _ = ref_loop.parallel_criterion(mods, weights, names, ref([x.cuda()]), [(y.cuda(),), (r.cuda(),)])
        total.backward()
        rows.append(total.item())
        for o in opts:
            o.step()
    torch.cuda.synchronize()
    return rows, [p.detach().float() for p in params]


def test_solver_matches_a_torch_adamw_loop():
    """FP32 width-512 MLP, batch 256, lr 1e-3, weight decay 0.1, 30 steps: the Solver with adamw=True
    against autograd + ``torch.optim.AdamW``, and an Adam run (L2-coupled decay) for contrast.
    Measured on an H100 (seed 0): the largest per-parameter update gap to torch is 0.022 of the
    update, the Adam run's is 7.7, and the last loss rows agree to 2e-5 relative.  The bound, 0.05,
    is twice the measured gap."""
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        batches = _batches(30)
        w, problem = _worker()
        assert type(w.optimizer) is fused_optim.FusedAdam and w.optimizer.adamw
        p0 = _params(w)
        want, theirs = _torch_loop(w, problem, batches,
                                   lambda m, ps: [torch.optim.AdamW(ps, lr=1e-3, weight_decay=0.1)])
        got = _train(w, batches)
        adam, _ = _worker(adamw=False)
        _train(adam, batches)
        gap_torch, gap_adam = _gap(_params(w), theirs, p0), _gap(_params(adam), theirs, p0)
        print("AdamW: update gap to torch.optim.AdamW %.3e, an Adam run's %.3e, last rows %r %r"
              % (gap_torch, gap_adam, got[-1], want[-1]))
        assert gap_torch < 0.1 * gap_adam and gap_torch < 0.05, (gap_torch, gap_adam)
        assert abs(got[-1] - want[-1]) < 0.05 * abs(want[0] - want[-1]), (got[-1], want[-1])
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def test_graph_replay_equals_eager_while_lr_changes_every_step():
    batches = _batches(8)
    lrs = [1e-3 * s for s in LR_SCALE]
    eager, _ = _worker(graph=False)
    graphed, _ = _worker(graph=True)
    a, b = _train(eager, batches, lrs=lrs), _train(graphed, batches, lrs=lrs)
    assert graphed.graphed is not None and graphed.optimizer._dyn is not None
    assert a == b and a[0] != a[-1]
    assert torch.equal(eager.arena.master, graphed.arena.master)
    for k, v in graphed.optimizer._vec.items():
        assert torch.equal(v, eager.optimizer._vec[k]), k


def test_checkpoint_resume_continues_bit_for_bit_and_torch_adamw_state_resumes():
    batches = _batches(12)
    a, _ = _worker()
    _train(a, batches[:6])
    model_sd = {k: v.detach().clone() for k, v in a.model.state_dict().items()}
    opt_sd = a.optimizer.state_dict()
    assert opt_sd["param_groups"][0]["decoupled_weight_decay"] is True
    rows_a = _train(a, batches[6:], 6)
    b, _ = _worker(seed=7)
    b.model.load_state_dict(model_sd)
    b.optimizer.load_state_dict(opt_sd)
    rows_b = _train(b, batches[6:], 6)
    assert rows_a == rows_b and torch.equal(a.arena.master, b.arena.master)
    for k in ("exp_avg", "exp_avg_sq"):
        assert torch.equal(a.optimizer._vec[k], b.optimizer._vec[k])
    # a torch.optim.AdamW state dict: moments and step load, and the run continues with AdamW
    params = [torch.nn.Parameter(p.detach().clone()) for p in list(a.model.parameters()) +
              list(a.criterion.parameters())]
    stock = torch.optim.AdamW(params, lr=1e-3, weight_decay=0.1)
    stock.load_state_dict(opt_sd)
    for p in params:
        p.grad = torch.randn_like(p) * 1e-2
    stock.step()
    c, _ = _worker(seed=3)
    c.optimizer.load_state_dict(stock.state_dict())
    assert c.optimizer._steps == 7 and c.optimizer.hyper["decoupled_weight_decay"] is True
    for i, s in enumerate(sorted(c.arena.slots, key=lambda s: s.index)):
        st = stock.state_dict()["state"][i]
        assert torch.equal(c.optimizer._vec["exp_avg"][s.offset:s.end], st["exp_avg"].flatten())
    rows = _train(c, _batches(2, seed=5))
    assert all(np.isfinite(rows))


@pytest.mark.parametrize("combo", ["q8", "accumulation_clip", "fp8", "ema"])
def test_solver_loop_with_adamw_in_combination(combo, tmp_path):
    """The solver's own loop (epochs, schedule, checkpoints) with adamw=True: the losses stay finite
    and fall, the optimizer runs the AdamW rule, and its checkpoint says so."""
    ns = synthetic.api_namespace("frl_b200")
    t = ns.types
    torch.manual_seed(0)
    problem = synthetic.make_mlp_problem(ns, str(tmp_path), n_train=2048, width=512, n_classes=100, reg_dim=16,
                                         depth=3)
    run_opts = t.RunOpts(optim=t.OptimOpts(algo=t.OptAlgorithm.ADAM, lr=1e-3, weightDecay=0.05,
                                           gradientClip=1.0 if combo == "accumulation_clip" else 0.0),
                         batchSize=256, nEpochs=2, numThreads=0, singleThreaded=True, numVisualizedSamples=0)
    kw = dict(precision=Precision.FP8 if combo == "fp8" else Precision.BF16,
              grad_accumulation=2 if combo == "accumulation_clip" else 1, ema_decay=0.9 if combo == "ema" else 0.0,
              optimizer_state=OptimizerState.Q8 if combo == "q8" else OptimizerState.FP32)
    args = SolverWorkerArgs(run_opts=run_opts, problem=problem, save_dir=str(tmp_path), run_device=Device.GPU,
                            node_idx=0, node_count=1, rank=0, local_rank=0, world_size=1, group_name=None,
                            init_method="", adamw=True, **kw)
    worker, _, _ = Solver.build_worker(args)
    assert worker.optimizer.adamw and type(worker.optimizer) is (
        fused_optim.FusedAdam8bit if combo == "q8" else fused_optim.FusedAdam)
    del worker
    _native.launch_count_reset()
    rows = []
    for frac in Solver._run_solver_worker(args):
        rows.append(frac.performance[t.Split.TRAIN].losses)
    totals = [sum(float(v) for v in r.values()) for r in rows]
    assert all(torch.isfinite(torch.tensor(totals))) and totals[-1] < totals[0], totals


def test_muon_with_adamw_matches_torch_muon_and_adamw():
    """Muon for the 2-D model weights with AdamW for the rest against ``torch.optim.Muon`` +
    ``torch.optim.AdamW``: the Newton-Schulz products round to bf16 in their own order on each side, so
    the runs drift a little (the Muon + Adam test allows 0.2 of an update; the same here).  Measured on
    an H100 (seed 0): 0.081 of the update, last loss rows within 1e-5 relative."""
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        batches = _batches(30)
        w, problem = _worker(wd=0.1, muon=True)
        assert type(w.optimizer) is fused_optim.FusedMuon and w.optimizer.adamw
        p0 = _params(w)

        def make(model, params):
            mats = [p for p in model.parameters() if p.ndim == 2]
            rest = [p for p in params if all(p is not q for q in mats)]
            return [torch.optim.Muon(mats, lr=1e-3, weight_decay=0.1, momentum=0.95, adjust_lr_fn="match_rms_adamw"),
                    torch.optim.AdamW(rest, lr=1e-3, weight_decay=0.1)]

        want, theirs = _torch_loop(w, problem, batches, make)
        got = _train(w, batches)
        gap = _gap(_params(w), theirs, p0)
        print("Muon + AdamW: update gap to torch.optim.Muon + AdamW %.3e, last rows %r %r" % (gap, got[-1], want[-1]))
        assert gap < 0.2, gap
        assert abs(got[-1] - want[-1]) < 0.1 * abs(want[0] - want[-1]), (got[-1], want[-1])
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def test_two_ranks_agree_and_match_one_gpu_at_the_global_batch():
    """tests/run_adamw_mp.py: over gloo with both ranks on GPU 0 when only one GPU is visible (K7 arm
    reported as not run), over NCCL with the K7 arm where two or more GPUs are visible."""
    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    backend = "nccl" if torch.cuda.device_count() >= 2 else "gloo"
    res = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nproc-per-node", "2",
                          os.path.join(repo, "tests", "run_adamw_mp.py"), "--backend", backend],
                         capture_output=True, text=True, timeout=600, cwd=repo)
    print(res.stdout[-2000:])
    assert res.returncode == 0 and res.stdout.count("ADAMW_MP_OK") == 2, res.stdout[-3000:] + res.stderr[-3000:]
    assert "ADAMW_K7" in res.stdout
