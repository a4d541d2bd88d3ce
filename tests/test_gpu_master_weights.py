"""Bf16 master weights with stochastic rounding (types.MasterWeights.BF16) on the device.

* every K2-sr / K2-mt-sr instantiation equals the fp32 form of the same rule (K2 / K2-mt, whose rules
  the optimizer-path tests hold against float64 torch.optim) on the widened bf16 weights, followed by
  the numpy restatement of the rounding (tests/sr_oracle.py), bit for bit: weights and state;
* K11 on bf16 weights equals K11 on the same weights widened to fp32;
* the rounding is unbiased: 1000 SGD updates of 0.1 ulp move the weights as far as an fp32 master
  does, where round-to-nearest leaves them where they were;
* through Solver.build_worker: bf16 against fp32 master weights (SGD, Adam), graph replay, resume,
  EMA with a held-out swap, accumulation with clipping, FP8, a channels_last ResNet, and the memory
  the option saves.
"""
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

import frl_b200  # noqa: F401
from frl_b200 import _native, synthetic
from frl_b200.multi_tensor import GradSegTable
from frl_b200.solver import Solver, SolverWorkerArgs
from frl_b200.types import Device, MasterWeights, OptAlgorithm, Precision, Split
from sr_oracle import sr_arena

pytestmark = pytest.mark.gpu
DEV = "cuda"
SEED = 0x1234_5678_9ABC_DEF0

# the update rules of the SR kernels, each with the state it keeps
RULES = ["sgd", "sgd_momentum", "adam", "adam_amsgrad", "adamw", "rmsprop", "rmsprop_momentum"]


def _states(rule, n, gen):
    names = {"sgd": [], "sgd_momentum": ["buf"], "adam": ["m", "v"], "adam_amsgrad": ["m", "v", "vmax"],
             "adamw": ["m", "v"], "rmsprop": ["sq"], "rmsprop_momentum": ["sq", "buf"]}[rule]
    out = {}
    for k in names:
        x = torch.rand(n, device=DEV, generator=gen) * 0.01
        out[k] = x + 1e-4 if k in ("v", "vmax", "sq") else x - 0.005
    return out


def _hyper(rule, t):
    if rule.startswith("sgd"):
        return dict(lr=0.05, mu=0.9 if rule == "sgd_momentum" else 0.0, dampening=0.1, wd=1e-3, first_step=False)
    if rule.startswith("adam"):
        return dict(lr=3e-3, beta1=0.9, beta2=0.999, eps=1e-8, wd=1e-2, step=t)
    return dict(lr=1e-3, alpha=0.99, eps=1e-8, wd=1e-3, mu=0.9 if rule == "rmsprop_momentum" else 0.0)


def _flat_fp32(rule, p, g, st, n, **kw):
    if rule.startswith("sgd"):
        _native.sgd_momentum(p, g, st.get("buf"), None, n, **kw)
    elif rule.startswith("adam"):
        getattr(_native, "adamw" if rule == "adamw" else "adam")(p, g, st["m"], st["v"], st.get("vmax"), None, n, **kw)
    else:
        _native.rmsprop(p, g, st["sq"], st.get("buf"), None, n, **kw)


def _flat_sr(rule, w, g, st, n, off, t, **kw):
    if rule.startswith("sgd"):
        _native.sgd_momentum_sr(w, g, st.get("buf"), n, arena_off=off, seed=SEED, t=t, **kw)
    elif rule.startswith("adam"):
        getattr(_native, "adamw_sr" if rule == "adamw" else "adam_sr")(w, g, st["m"], st["v"], st.get("vmax"), n,
                                                                       arena_off=off, seed=SEED, **kw)
    else:
        _native.rmsprop_sr(w, g, st["sq"], st.get("buf"), n, arena_off=off, seed=SEED, t=t, **kw)


def _dyn_block(rule, kw, t):
    """The dyn block the optimizer uploads (the by-value scalars, then t's bits at dyn[3])."""
    if rule.startswith("adam"):
        bc1, bc2 = 1 - kw["beta1"] ** t, 1 - kw["beta2"] ** t
        vals = [-(kw["lr"] / bc1), bc2 ** 0.5, float(np.float32(1 - kw["lr"] * kw["wd"])) if rule == "adamw" else 0.0]
    else:
        vals = [kw["lr"], 0.0, 0.0]
    d = torch.tensor(vals + [0.0], dtype=torch.float32)
    d.view(torch.int32)[3] = t
    return d.to(DEV)


@pytest.mark.parametrize("rule", RULES)
@pytest.mark.parametrize("gdt", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("n, off, mode", [(4099, 8, "plain"), (70001, 4096, "coef"), (5, 0, "dyn"),
                                          (3 * 132 * 8 * 4096 + 3, 1 << 20, "plain")])
def test_flat_sr_equals_fp32_rule_then_numpy_sr(rule, gdt, n, off, mode):
    gen = torch.Generator(device=DEV).manual_seed(n + len(rule))
    t = 37
    w = (torch.randn(n, device=DEV, generator=gen) * 0.5).to(torch.bfloat16)
    g = (torch.randn(n, device=DEV, generator=gen) * 0.1).to(gdt)
    st = _states(rule, n, gen)
    kw = _hyper(rule, t)
    coef = torch.tensor([0.75], device=DEV) if mode == "coef" else None
    dyn = _dyn_block(rule, kw, t) if mode == "dyn" else None
    p32, st32 = w.float(), {k: v.clone() for k, v in st.items()}
    _flat_fp32(rule, p32, g, st32, n, grad_scale=0.5, grad_scale_dev=coef, dyn=dyn, **kw)
    kw_sr, t_arg = dict(kw), t
    if mode == "dyn":            # the by-value update count is wrong on purpose: dyn[3] must win
        t_arg = 1
        if "step" in kw_sr:
            kw_sr["step"] = 1
    _flat_sr(rule, w, g, st, n, off, t_arg, grad_scale=0.5, grad_scale_dev=coef, dyn=dyn, **kw_sr)
    torch.cuda.synchronize()
    want = sr_arena(p32.cpu().numpy(), off, t, SEED)
    got = w.view(torch.int16).cpu().numpy().view(np.uint16)
    assert np.array_equal(got, want), (rule, int((got != want).sum()))
    for k in st:
        assert torch.equal(st[k], st32[k]), k


MT_LAYOUT = [(3, True), (4096 * 4 + 5, True), (17, False), (40000, True), (8, True)]


@pytest.mark.parametrize("rule", RULES)
@pytest.mark.parametrize("dyn_mode", [False, True])
def test_mt_sr_equals_fp32_mt_then_numpy_sr(rule, dyn_mode):
    gen = torch.Generator(device=DEV).manual_seed(len(rule) + 100 * dyn_mode)

    class _Slot:
        def __init__(self, i, off, n):
            self.index, self.offset, self.numel, self.shape, self.is_model = i, off, n, (n,), True
            self.end = off + n

    slots, off = [], 0
    for i, (n, listed) in enumerate(MT_LAYOUT):
        slots.append((_Slot(i, off, n), listed))
        off = (off + n + 7) // 8 * 8
    total = off
    listed = [s for s, keep in slots if keep]
    table = GradSegTable(listed, torch.device(DEV))
    grads = []
    for i, s in enumerate(listed):
        gd = torch.randn(s.numel, device=DEV, generator=gen) * 0.1
        gd = gd.to(torch.bfloat16) if i % 2 else gd
        grads.append(gd)
        table.point(s, gd.data_ptr(), gd.dtype)
    table.upload()
    w = (torch.randn(total, device=DEV, generator=gen) * 0.5).to(torch.bfloat16)
    w0 = w.clone()
    st = _states(rule, total, gen)
    t = 5
    kw = _hyper(rule, t)
    dyn = _dyn_block(rule, kw, t) if dyn_mode else None
    p32, st32 = w.float(), {k: v.clone() for k, v in st.items()}
    if rule.startswith("sgd"):
        _native.sgd_momentum_mt(p32, st32.get("buf"), None, table, dyn=dyn, **kw)
        _native.sgd_momentum_mt_sr(w, st.get("buf"), table, seed=SEED, t=1 if dyn_mode else t, dyn=dyn, **kw)
    elif rule.startswith("adam"):
        name = "adamw" if rule == "adamw" else "adam"
        getattr(_native, name + "_mt")(p32, st32["m"], st32["v"], st32.get("vmax"), None, table, dyn=dyn, **kw)
        getattr(_native, name + "_mt_sr")(w, st["m"], st["v"], st.get("vmax"), table, seed=SEED, dyn=dyn, **kw)
    else:
        _native.rmsprop_mt(p32, st32["sq"], st32.get("buf"), None, table, dyn=dyn, **kw)
        _native.rmsprop_mt_sr(w, st["sq"], st.get("buf"), table, seed=SEED, t=1 if dyn_mode else t, dyn=dyn, **kw)
    torch.cuda.synchronize()
    want = w0.view(torch.int16).cpu().numpy().view(np.uint16).copy()
    x = p32.cpu().numpy()
    for s in listed:
        lo, hi = s.offset, (s.end + 3) // 4 * 4
        want[lo:hi] = sr_arena(x[lo:hi], lo, t, SEED)
    got = w.view(torch.int16).cpu().numpy().view(np.uint16)
    assert np.array_equal(got, want), (rule, int((got != want).sum()))
    for k in st:
        assert torch.equal(st[k], st32[k]), k


@pytest.mark.parametrize("n", [3, 4096 * 5 + 2, 1 << 20])
@pytest.mark.parametrize("w", [1.0, 0.1, 0.7])
def test_k11_bf16_equals_k11_on_the_widened_weights(n, w):
    gen = torch.Generator(device=DEV).manual_seed(n)
    p = torch.randn(n, device=DEV, generator=gen).to(torch.bfloat16)
    ema = torch.randn(n, device=DEV, generator=gen)
    e0, ref = ema.double(), ema.clone()
    _native.weight_ema(ref, p.float(), w)
    _native.weight_ema_bf16(ema, p, w)
    assert torch.equal(ema, ref)
    # the float64 lerp restatement, to the one fp32 rounding of the fused multiply-add
    want = e0 + w * (p.double() - e0)
    tol = 2.0 ** -23 * 2 * torch.maximum(e0.abs(), p.double().abs())
    assert torch.all((ema.double() - want).abs() <= tol)


def test_sr_is_unbiased_where_round_to_nearest_stalls():
    """Weights 1.0 (bf16 ulp 2^-7), a constant update of 0.1 ulp per SGD step, 1000 steps."""
    n, steps = 1 << 16, 1000
    lr = 2.0 ** -7 * 0.1
    g = torch.ones(n, device=DEV)
    w = torch.ones(n, device=DEV, dtype=torch.bfloat16)
    m = torch.ones(n, device=DEV)
    rn = torch.ones(n, device=DEV, dtype=torch.bfloat16)
    for t in range(1, steps + 1):
        _native.sgd_momentum_sr(w, g, None, n, arena_off=0, seed=SEED, t=t, lr=-lr, mu=0.0, dampening=0.0, wd=0.0)
        _native.sgd_momentum(m, g, None, None, n, lr=-lr, mu=0.0, dampening=0.0, wd=0.0)
        rn = (rn.float() + lr).to(torch.bfloat16)
    torch.cuda.synchronize()
    drift_fp32 = (m.double() - 1).mean().item()
    drift_sr = (w.double() - 1).mean().item()
    # each step's rounding error has mean 0 and |error| < 1 ulp, so the per-element error after
    # 1000 steps has sd <= sqrt(1000) / 2 ulp; the mean of 2^16 independent ones <= that / 256
    sd = (steps ** 0.5 / 2) * 2.0 ** -7 / 256
    assert abs(drift_sr - drift_fp32) < 6 * sd, (drift_sr, drift_fp32, sd)
    assert drift_fp32 > 0.7
    assert torch.all(rn == 1.0)            # round to nearest: every 0.1-ulp update is lost


# ---- through Solver.build_worker ------------------------------------------------------------------------------

def _worker(algo=OptAlgorithm.SGD, master=MasterWeights.BF16, precision=Precision.BF16, seed=0, lr=None,
            graph=False, **kw):
    ns = synthetic.api_namespace("frl_b200")
    t = ns.types
    save_dir = tempfile.mkdtemp(prefix="frl_b200_mw_")
    torch.manual_seed(seed)
    problem = synthetic.make_mlp_problem(ns, save_dir, n_train=8, width=512, n_classes=100, reg_dim=16, depth=3)
    lr = lr if lr is not None else (0.05 if algo == OptAlgorithm.SGD else 1e-3)
    run_opts = t.RunOpts(optim=t.OptimOpts(algo=algo, lr=lr, momentum=0.9, weightDecay=1e-4),
                         batchSize=256, nEpochs=1, numThreads=0, singleThreaded=True, numVisualizedSamples=0)
    args = SolverWorkerArgs(run_opts=run_opts, problem=problem, save_dir=save_dir, run_device=Device.GPU,
                            node_idx=0, node_count=1, rank=0, local_rank=0, world_size=1, group_name=None,
                            init_method="", precision=precision, graph_step=graph, master_weights=master, **kw)
    worker, _, _ = Solver.build_worker(args)
    worker.model.train()
    worker.criterion.train()
    return worker


def _batches(n, width=512, seed=1234):
    gen = torch.Generator().manual_seed(seed)
    w = torch.randn(width, 100, generator=gen) / width ** 0.5
    out = []
    for _ in range(n):
        x = torch.randn(256, width, generator=gen)
        out.append((x, (x @ w).argmax(1), torch.randn(256, 16, generator=gen) * 0.1 + x[:, :16]))
    return out


def _train(worker, batches, start=0):
    rows = []
    for i, (x, y, r) in enumerate(batches, start):
        _, total, _, _ = worker._pass_one_minibatch(i, Split.TRAIN, [x.cuda()], [(y.cuda(),), (r.cuda(),)])
        rows.append(float(total.detach()))
        del total
    torch.cuda.synchronize()
    return rows


def _weights(worker):
    with worker.arena.exported(cpu=False):
        return [p.detach().clone() for p in list(worker.model.parameters()) + list(worker.criterion.parameters())]


@pytest.mark.parametrize("algo", [OptAlgorithm.SGD, OptAlgorithm.ADAM])
def test_bf16_master_tracks_fp32_master(algo):
    """Width-512 MLP, 20 steps in BF16.  The update gap of a tensor is the distance between the two
    runs' weights over how far the fp32-master run moved it; measured on an H100, the largest was
    0.53 (SGD, whose 20 small steps are a few bf16 ulps) and 0.23 (Adam), over the whole model 0.39
    and 0.19, and the final losses agreed to 3e-5 relative.  Stated tolerances: 0.75 per tensor, 0.5
    over the model, 1e-3 relative on the loss."""
    batches = _batches(20)
    a, b = _worker(algo, MasterWeights.FP32), _worker(algo, MasterWeights.BF16)
    assert b.arena.bf16_master and not a.arena.bf16_master
    assert b.pipeline.fused_dw_update == (algo == OptAlgorithm.SGD)       # K12 SR for SGD
    w0 = _weights(a)
    la, lb = _train(a, batches), _train(b, batches)
    wa, wb = _weights(a), _weights(b)
    gaps = [((x - y).norm() / (x - q).norm().clamp_min(1e-30)).item() for x, y, q in zip(wa, wb, w0)]
    whole = (torch.cat([(x - y).flatten() for x, y in zip(wa, wb)]).norm()
             / torch.cat([(x - q).flatten() for x, q in zip(wa, w0)]).norm()).item()
    print("update gaps per tensor", [round(g, 3) for g in gaps], "whole model %.3f" % whole,
          "losses", la[-1], lb[-1])
    assert max(gaps) < 0.75 and whole < 0.5, (gaps, whole)
    assert abs(la[-1] - lb[-1]) <= 1e-3 * abs(la[-1]), (la[-1], lb[-1])
    assert lb[-1] < lb[0]


def test_graph_replay_and_resume_give_identical_bytes():
    batches = _batches(10)
    eager, graphed = _worker(OptAlgorithm.ADAM), _worker(OptAlgorithm.ADAM, graph=True)
    a, b = _train(eager, batches), _train(graphed, batches)
    assert graphed.graphed is not None and graphed.optimizer._dyn is not None
    assert a == b
    assert torch.equal(eager.arena.lp, graphed.arena.lp) and torch.equal(eager.arena.master, graphed.arena.master)
    for k, v in graphed.optimizer._vec.items():
        assert torch.equal(v, eager.optimizer._vec[k]), k
    # resume: model state + optimizer state dict (seed and update count in the param group)
    for algo in (OptAlgorithm.SGD, OptAlgorithm.ADAM):
        x = _worker(algo)
        _train(x, batches[:5])
        saved = _weights(x)
        opt_sd = x.optimizer.state_dict()
        assert opt_sd["param_groups"][0]["sr_updates"] == 5 and "sr_seed" in opt_sd["param_groups"][0]
        rows_x = _train(x, batches[5:], 5)
        y = _worker(algo, seed=7)
        y.arena.load_master_from_params(list(zip(list(y.model.parameters()) + list(y.criterion.parameters()),
                                                 saved)))
        y.optimizer.load_state_dict(opt_sd)
        assert y.optimizer._steps == 5
        rows_y = _train(y, batches[5:], 5)
        assert rows_x == rows_y and torch.equal(x.arena.lp, y.arena.lp), algo
        # the same files load into an fp32-master run, and its state dict stays torch's
        z = _worker(algo, MasterWeights.FP32, seed=3)
        z.optimizer.load_state_dict(opt_sd)
        assert "sr_seed" not in z.optimizer.state_dict()["param_groups"][0]


_MEMORY_ARM = r"""
import sys, torch
sys.path.insert(0, {tests!r})
import test_gpu_master_weights as t
from frl_b200.types import MasterWeights, OptAlgorithm
w = t._worker(OptAlgorithm.ADAM, MasterWeights({master!r}))
torch.cuda.synchronize()
print("ARM", torch.cuda.memory_allocated(), w.arena.model_end, w.arena.numel)
"""


def test_memory_falls_by_four_bytes_per_model_parameter():
    """Device memory after the build, each arm in a fresh process (nothing left over from other tests)."""
    tests = os.path.dirname(os.path.abspath(__file__))
    got = {}
    for master in ("fp32", "bf16"):
        res = subprocess.run([sys.executable, "-c", _MEMORY_ARM.format(tests=tests, master=master)],
                             capture_output=True, text=True, timeout=300, cwd=os.path.dirname(tests))
        line = [x for x in res.stdout.splitlines() if x.startswith("ARM")]
        assert res.returncode == 0 and line, res.stderr[-3000:]
        got[master] = [int(v) for v in line[0].split()[1:]]
    (m_fp32, n, numel), (m_bf16, n2, _) = got["fp32"], got["bf16"]
    assert n2 == n
    # 4 B per model parameter, seen through the caching allocator's 512-byte rounding of each block
    blk = lambda nbytes: (nbytes + 511) // 512 * 512        # noqa: E731
    assert m_fp32 - m_bf16 == blk(4 * numel) - blk(4 * (numel - n)), (m_fp32, m_bf16, n)


def test_ema_swap_restores_the_bf16_weights_bit_for_bit():
    w = _worker(OptAlgorithm.ADAM, ema_decay=0.9)
    _train(w, _batches(4))
    ema = w.pipeline.ema
    assert ema.bf16 and ema.updates == 4
    before = w.arena.lp.clone()
    with ema.swapped():
        assert torch.equal(w.arena.lp[:ema.n], ema.ema.to(torch.bfloat16))
    assert torch.equal(w.arena.lp, before)
    sd = ema.state_dict()
    assert all(v.dtype == torch.float32 for v in sd["state_dict"].values() if v.is_floating_point())
    assert torch.equal(w.arena.lp, before)
    # the file holds the fp32 EMA itself, so a resumed EMA continues bit for bit
    other = _worker(OptAlgorithm.ADAM, ema_decay=0.9, seed=3).pipeline.ema
    other.load_state_dict(sd)
    assert torch.equal(other.ema, ema.ema) and other.updates == ema.updates


@pytest.mark.parametrize("combo", ["accumulation_clip", "fp8", "ema", "rmsprop"])
def test_solver_loop_in_combination(combo, tmp_path):
    ns = synthetic.api_namespace("frl_b200")
    t = ns.types
    torch.manual_seed(0)
    problem = synthetic.make_mlp_problem(ns, str(tmp_path), n_train=2048, width=512, n_classes=100, reg_dim=16,
                                         depth=3)
    algo = t.OptAlgorithm.RMSPROP if combo == "rmsprop" else t.OptAlgorithm.ADAM
    run_opts = t.RunOpts(optim=t.OptimOpts(algo=algo, lr=1e-3 if combo != "rmsprop" else 1e-4,
                                           gradientClip=1.0 if combo == "accumulation_clip" else 0.0),
                         batchSize=256, nEpochs=2, numThreads=0, singleThreaded=True, numVisualizedSamples=0)
    kw = dict(precision=Precision.FP8 if combo == "fp8" else Precision.BF16,
              grad_accumulation=2 if combo == "accumulation_clip" else 1, ema_decay=0.9 if combo == "ema" else 0.0)
    args = SolverWorkerArgs(run_opts=run_opts, problem=problem, save_dir=str(tmp_path), run_device=Device.GPU,
                            node_idx=0, node_count=1, rank=0, local_rank=0, world_size=1, group_name=None,
                            init_method="", master_weights=MasterWeights.BF16, **kw)
    rows = [frac.performance[t.Split.TRAIN].losses for frac in Solver._run_solver_worker(args)]
    totals = [sum(float(v) for v in r.values()) for r in rows]
    assert all(np.isfinite(totals)) and totals[-1] < totals[0], totals


def test_channels_last_resnet_trains(tmp_path):
    ns = synthetic.api_namespace("frl_b200")
    t = ns.types
    torch.manual_seed(0)
    torch.manual_seed(0)
    problem = synthetic.make_resnet_problem(ns, str(tmp_path), "resnet18", image=64, n_train=128)
    run_opts = t.RunOpts(optim=t.OptimOpts(algo=t.OptAlgorithm.SGD, lr=0.05, momentum=0.9), batchSize=32, nEpochs=2,
                         numThreads=0, singleThreaded=True, numVisualizedSamples=0)
    args = SolverWorkerArgs(run_opts=run_opts, problem=problem, save_dir=str(tmp_path), run_device=Device.GPU,
                            node_idx=0, node_count=1, rank=0, local_rank=0, world_size=1, group_name=None,
                            init_method="", precision=Precision.BF16, channels_last=True,
                            master_weights=MasterWeights.BF16)
    captured = {}
    orig = Solver.build_worker.__func__

    def spy(cls, a):
        out = orig(cls, a)
        captured["worker"], captured["w0"] = out[0], _weights(out[0])
        return out

    Solver.build_worker = classmethod(spy)
    try:
        rows = [frac.performance[t.Split.TRAIN].losses for frac in Solver._run_solver_worker(args)]
    finally:
        Solver.build_worker = classmethod(orig)
    totals = [sum(float(v) for v in r.values()) for r in rows]
    assert all(np.isfinite(totals)), totals
    w, w0 = captured["worker"], captured["w0"]
    assert w.arena.bf16_master and w.arena.n_channels_last > 0
    # every conv weight moved under the SR update, and it moved by more than a rounding step
    moved = [(a.float() - b.float()).abs().max().item() for a, b in zip(w0, _weights(w))]
    assert sum(m > 0 for m in moved) >= 0.9 * len(moved), moved


# ---- criterion parameters: fp32 master beside the bf16 model weights ---------------------------------------

class _Crit(torch.nn.Module):
    """Two criterion parameters after a 2-layer model: they keep an fp32 master under MasterWeights.BF16."""

    def __init__(self):
        super().__init__()
        self.s = torch.nn.Parameter(torch.randn(5))
        self.t = torch.nn.Parameter(torch.randn(3, 3))


def _crit_case(algo, seed=0):
    from frl_b200 import fused_optim
    from frl_b200.arena import ParamArena
    from frl_b200.types import OptimOpts
    torch.manual_seed(seed)
    net = torch.nn.Sequential(torch.nn.Linear(64, 40), torch.nn.Linear(40, 7)).to(DEV)
    crit = _Crit().to(DEV)
    arena = ParamArena(net.parameters(), crit.parameters(), device=DEV, precision=Precision.BF16,
                       master_weights=MasterWeights.BF16)
    opts = OptimOpts(algo=algo, lr=0.05 if algo == OptAlgorithm.SGD else 1e-2, momentum=0.9, weightDecay=1e-3)
    opt = fused_optim.create_fused_optimizer(arena, opts)
    return arena, opt


@pytest.mark.parametrize("algo", [OptAlgorithm.SGD, OptAlgorithm.ADAM])
@pytest.mark.parametrize("path", ["table", "table_graph", "range", "range_clip"])
def test_criterion_slots_follow_the_fp32_rule_and_model_slots_the_sr_rule(algo, path):
    """Three updates through the optimizer's own paths: criterion slots against the fp32 K2-mt kernel on
    a full-size fp32 copy (the oracle), model slots against fp32 K2-mt on the widened bf16 weights
    followed by the numpy rounding.  ``range``: apply_range over the whole arena, split at model_end;
    ``range_clip`` with a device clip coefficient (criterion slots unclipped); ``table_graph``: the
    segment-table update captured after an eager step and replayed (the by-value scalars frozen at
    capture, the device-resident ones current)."""
    arena, opt = _crit_case(algo)
    n, me = arena.numel, arena.model_end
    assert arena.master.numel() == n - me > 0
    gen = torch.Generator(device=DEV).manual_seed(1)
    # criterion gradients fp32 but bf16-exact: apply_range reads them from the bf16 gradient arena
    grads = {s.index: (torch.randn(s.numel, device=DEV, generator=gen) * 0.1).to(torch.bfloat16).to(
        torch.bfloat16 if s.is_model else torch.float32) for s in arena.slots}
    table = GradSegTable(arena.slots, torch.device(DEV))
    for s in arena.slots:
        table.point(s, grads[s.index].data_ptr(), grads[s.index].dtype)
        arena.grad[s.offset:s.end].copy_(grads[s.index])           # what apply_range reads
    table.upload()
    # oracle state: fp32 weights of every slot, the optimizer's state vectors
    p32 = torch.zeros(n, device=DEV)
    p32[:me] = arena.lp[:me].float()
    p32[me:] = arena.master
    names = ("momentum_buffer",) if algo == OptAlgorithm.SGD else ("exp_avg", "exp_avg_sq")
    ref_state = {k: torch.zeros(n, device=DEV) for k in names}
    coef = torch.tensor([0.5], device=DEV) if path == "range_clip" else None
    h = opt.hyper
    graph = None
    if path == "table_graph":
        opt.enable_dynamic_scalars()
    for step in range(1, 5):
        t = step
        opt.begin_step()
        if path == "table" or (path == "table_graph" and step == 1):
            # table_graph: one eager step first, as the solver's loop runs eager steps before it captures;
            # state vectors created inside a capture would belong to the graph's pool and be re-zeroed
            opt.apply_table(table)
        elif path == "table_graph":
            if graph is None:
                opt._sr_split(table)      # built with the table, before any capture, as the pipeline does
                torch.cuda.synchronize()
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph):
                    opt.apply_table(table)
            graph.replay()
        else:
            opt.apply_range(0, n, clip_coef_dev=coef)
        opt.end_step()
        # oracle: fp32 K2-mt over each half, the model half's gradient clipped
        for part in ("model", "crit"):
            slots = [s for s in arena.slots if s.is_model == (part == "model")]
            sub = GradSegTable(slots, torch.device(DEV))
            for s in slots:
                sub.point(s, grads[s.index].data_ptr(), grads[s.index].dtype)
            sub.upload()
            gs = 0.5 if (coef is not None and part == "model") else 1.0
            if algo == OptAlgorithm.SGD:
                _native.sgd_momentum_mt(p32, ref_state["momentum_buffer"], None, sub, lr=h["lr"], mu=h["momentum"],
                                        dampening=h["dampening"], wd=h["weight_decay"], grad_scale=gs,
                                        first_step=(step == 1))
            else:
                _native.adam_mt(p32, ref_state["exp_avg"], ref_state["exp_avg_sq"], None, None, sub, lr=h["lr"],
                                beta1=h["betas"][0], beta2=h["betas"][1], eps=h["eps"], wd=h["weight_decay"], step=t,
                                grad_scale=gs)
        torch.cuda.synchronize()
        # the model range: round the oracle's fp32 result as the SR kernels do, then continue from it
        x = p32[:me].cpu().numpy()
        want = np.zeros(me, dtype=np.uint16)
        for s in arena.slots:
            if s.is_model:
                lo, hi = s.offset, (s.end + 3) // 4 * 4
                want[lo:hi] = sr_arena(x[lo:hi], lo, t, opt.sr_seed)
        got = arena.lp[:me].view(torch.int16).cpu().numpy().view(np.uint16)
        assert np.array_equal(got, want), (path, step, int((got != want).sum()))
        p32[:me] = arena.lp[:me].float()
        assert torch.equal(arena.master, p32[me:]), (path, step)
        for k in names:
            assert torch.equal(opt._state(k), ref_state[k]), (path, step, k)
    # export and load of criterion slots: their fp32 master, not a bf16 view
    with arena.exported(cpu=False):
        crit_vals = [s.param.detach().clone() for s in arena.slots if not s.is_model]
    assert all(v.dtype == torch.float32 for v in crit_vals)
    assert torch.equal(torch.cat([v.flatten() for v in crit_vals]),
                       torch.cat([arena.master_view(s).flatten() for s in arena.slots if not s.is_model]))
    arena.load_master_from_params([(s.param, v + 1) for s, v in zip([s for s in arena.slots if not s.is_model],
                                                                      crit_vals)])
    assert torch.equal(arena.master_view([s for s in arena.slots if not s.is_model][0]), crit_vals[0] + 1)


@pytest.mark.parametrize("clip", [0.0, 1.0])
def test_solver_with_an_uncertainty_criterion_eager_equals_graph(clip, tmp_path):
    """A toy Problem whose criterion learns its task weights: with bf16 master weights its parameters
    train on their fp32 master, and eager and graph-replayed runs give identical bytes."""
    ns = synthetic.api_namespace("frl_b200")
    t = ns.types
    out = []
    for graph in (False, True):
        torch.manual_seed(0)
        problem = synthetic.make_toy_problem(ns, str(tmp_path), n_train=64, n_test=0, criterion_kind="uncertainty")
        run_opts = t.RunOpts(optim=t.OptimOpts(algo=t.OptAlgorithm.ADAM, lr=1e-2, gradientClip=clip), batchSize=16,
                             nEpochs=1, numThreads=0, singleThreaded=True, numVisualizedSamples=0)
        args = SolverWorkerArgs(run_opts=run_opts, problem=problem, save_dir=str(tmp_path), run_device=Device.GPU,
                                node_idx=0, node_count=1, rank=0, local_rank=0, world_size=1, group_name=None,
                                init_method="", precision=Precision.BF16, graph_step=graph,
                                master_weights=MasterWeights.BF16)
        worker, _, _ = Solver.build_worker(args)
        worker.model.train()
        worker.criterion.train()
        crit0 = worker.arena.master.clone()
        assert crit0.numel() > 0
        gen = torch.Generator().manual_seed(9)
        for i in range(6):
            x = torch.randn(16, 64, generator=gen).cuda()
            y_reg, y_cls = torch.randn(16, 4, generator=gen).cuda(), torch.randint(0, 10, (16,), generator=gen).cuda()
            worker._pass_one_minibatch(i, Split.TRAIN, [x], [(y_reg,), (y_cls,)])
        torch.cuda.synchronize()
        assert not torch.equal(worker.arena.master, crit0)             # the criterion's weights trained
        out.append((worker.arena.lp.clone(), worker.arena.master.clone(), graph and worker.graphed is not None))
    assert out[1][2]
    assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1])


def test_two_ranks_agree_and_match_one_gpu_at_the_global_batch():
    """tests/run_master_weights_mp.py: over gloo with both ranks on GPU 0 when only one GPU is visible
    (the NCCL arm reported as not run), over NCCL where two or more GPUs are visible."""
    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    backend = "nccl" if torch.cuda.device_count() >= 2 else "gloo"
    res = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nproc-per-node", "2",
                          os.path.join(repo, "tests", "run_master_weights_mp.py"), "--backend", backend],
                         capture_output=True, text=True, timeout=600, cwd=repo)
    print(res.stdout[-2000:])
    assert res.returncode == 0 and res.stdout.count("MASTER_WEIGHTS_MP_OK") == 2, res.stdout[-3000:] + res.stderr[-3000:]
    assert "MASTER_WEIGHTS_NCCL" in res.stdout


@pytest.mark.parametrize("out, inp, rows", [(128, 256, 64), (256, 512, 192), (384, 768, 256), (1024, 1024, 512)])
@pytest.mark.parametrize("mu, dyn_mode", [(0.0, False), (0.9, False), (0.9, True)])
def test_k12_sr_equals_dw_gemm_then_k2_sr(out, inp, rows, mu, dyn_mode):
    """frl_dw_gemm_sgd_sr against frl_dw_gemm followed by frl_sgd_momentum_sr over the slice (bf16
    gradient), bit for bit: gradient, weights and momentum, at a non-zero arena offset; with dyn the
    by-value lr and update count are wrong on purpose."""
    gen = torch.Generator(device=DEV).manual_seed(out + inp + rows)
    dz = torch.randn(rows, out, device=DEV, generator=gen).to(torch.bfloat16)
    x = torch.randn(rows, inp, device=DEV, generator=gen).to(torch.bfloat16)
    w = (torch.randn(out * inp, device=DEV, generator=gen) * 0.05).to(torch.bfloat16)
    buf = torch.randn(out * inp, device=DEV, generator=gen) * 1e-3
    off, t = 4096 + 8, 9
    kw = dict(lr=0.05, mu=mu, dampening=0.0, wd=1e-4, grad_scale=0.5, first_step=False)
    dyn = None
    if dyn_mode:
        dyn = torch.tensor([0.05, 0.0, 0.0, 0.0])
        dyn.view(torch.int32)[3] = t
        dyn = dyn.to(DEV)
    gw_ref, w_ref, buf_ref = torch.empty(out, inp, device=DEV, dtype=torch.bfloat16), w.clone(), buf.clone()
    _native.dw_gemm(dz, x, gw_ref)
    _native.sgd_momentum_sr(w_ref, gw_ref.view(-1), buf_ref if mu else None, out * inp, arena_off=off, seed=SEED,
                            t=t, dyn=dyn, **kw)
    gw = torch.empty(out, inp, device=DEV, dtype=torch.bfloat16)
    if dyn_mode:
        kw["lr"] = 7.0
    _native.dw_gemm_sgd_sr(dz, x, gw, w, buf if mu else None, arena_off=off, seed=SEED, t=1 if dyn_mode else t,
                           dyn=dyn, **kw)
    torch.cuda.synchronize()
    assert torch.equal(gw, gw_ref)
    assert torch.equal(w.view(torch.int16), w_ref.view(torch.int16))
    assert torch.equal(buf, buf_ref)


def test_k12_sr_is_taken_on_one_gpu_with_sgd():
    w = _worker(OptAlgorithm.SGD)
    assert w.pipeline.fused_dw_update
    _train(w, _batches(2))
    assert w.pipeline.dw_updated, "no slot was updated inside its dW GEMM"
