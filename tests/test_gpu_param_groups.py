"""Param groups on the H100: every grouped instantiation (K2-mt grouped, K2-mt-sr grouped) against the
ungrouped kernel run segment by segment with that segment's group's lr / wd (which the existing suites
check against float64 torch.optim), one group bit-equal to the ungrouped kernel, a captured graph
following per-group lr changes through the rows, and the Solver with ``no_decay_1d`` and a hook against
a ``torch.optim`` loop with the same groups, K12 with a trunk weight in a non-default group, resume and
graph replay bit for bit."""
import tempfile
import zlib

import numpy as np
import pytest
import torch

import frl_b200  # noqa: F401
from frl_b200 import _native, fused_optim, synthetic
from frl_b200.multi_tensor import GradSegTable
from frl_b200.solver import Solver, SolverWorkerArgs
from frl_b200.types import Device, MasterWeights, OptAlgorithm, Precision, Split

pytestmark = pytest.mark.gpu
DEV = "cuda"
SEED = 0x1234_5678_9ABC_DEF0
LAYOUT = [3, 4096 * 4 + 5, 17, 40000, 8, 4096]
GROUP_OF = [0, 1, 2, 1, 0, 2]            # segment -> group
LR_WD = [(1e-3, 0.1), (5e-4, 0.0), (2e-3, 0.05)]
STEP = 3

RULES = {   # name -> (states, ungrouped flat form, grouped form, kwargs of both without lr / wd)
    "sgd": (1, "sgd_momentum", dict(mu=0.9, dampening=0.0)),
    "sgd0": (0, "sgd_momentum", dict(mu=0.0, dampening=0.0)),
    "adam": (2, "adam", dict(beta1=0.9, beta2=0.999, eps=1e-8)),
    "adam_ams": (3, "adam", dict(beta1=0.9, beta2=0.999, eps=1e-8)),
    "adamw": (2, "adamw", dict(beta1=0.9, beta2=0.999, eps=1e-8)),
    "adamw_ams": (3, "adamw", dict(beta1=0.9, beta2=0.999, eps=1e-8)),
    "rmsprop": (2, "rmsprop", dict(alpha=0.99, eps=1e-8, mu=0.9)),
    "rmsprop0": (1, "rmsprop", dict(alpha=0.99, eps=1e-8, mu=0.0)),
    "lion": (1, "lion", dict(beta1=0.9, beta2=0.99)),
}


def _rows(base, kw):
    rows = np.zeros((len(LR_WD), _native.GROUP_DYN_COLS), dtype=np.float32)
    for gi, (lr, wd) in enumerate(LR_WD):
        if base in ("adam", "adamw"):
            bc1, bc2 = 1 - kw["beta1"] ** STEP, 1 - kw["beta2"] ** STEP
            vals = [-(lr / bc1), bc2 ** 0.5] + ([np.float32(1 - lr * wd)] if base == "adamw" else [])
        elif base == "lion":
            vals = [lr, np.float32(1 - lr * wd)]
        else:
            vals = [lr]
        rows[gi, :len(vals)] = vals
        rows[gi, 4] = wd
    rows.view(np.uint32)[:, 3] = STEP
    return torch.from_numpy(rows).to(DEV)


class _Slot:
    def __init__(self, i, off, n, is_model):
        self.index, self.offset, self.numel, self.shape, self.is_model = i, off, n, (n,), is_model
        self.end = off + n


def _table(gen):
    slots, off = [], 0
    for i, n in enumerate(LAYOUT):
        slots.append(_Slot(i, off, n, is_model=i != 2))            # segment 2: a criterion parameter
        off = (off + n + 7) // 8 * 8
    table = GradSegTable(slots, torch.device(DEV))
    grads = []
    for i, s in enumerate(slots):
        gd = (torch.randn(s.numel, device=DEV, generator=gen) * 0.1).to((torch.float32, torch.bfloat16)[i % 2])
        grads.append(gd)
        table.point(s, gd.data_ptr(), gd.dtype)
    table.upload()
    return slots, table, grads, off


def _flat_call(name, base, p, g, st, lp, n, lr, wd, kw, gscale, coef, sr, off):
    """The ungrouped K2 (or K2-sr) form over one segment."""
    fn = getattr(_native, base + ("_sr" if sr else ""))
    extra = dict(grad_scale=gscale, grad_scale_dev=coef)
    if base == "sgd_momentum":
        args = (p, g, st[0] if kw["mu"] else None)
        extra.update(lr=lr, wd=wd, first_step=False, **kw)
    elif base in ("adam", "adamw"):
        args = (p, g, st[0], st[1], st[2] if len(st) > 2 else None)
        extra.update(lr=lr, wd=wd, step=STEP, **kw)
    elif base == "rmsprop":
        args = (p, g, st[0], st[1] if kw["mu"] else None)
        extra.update(lr=lr, wd=wd, **kw)
    else:
        args = (p, g, st[0])
        extra.update(lr=lr, wd=wd, **kw)
    if sr:
        extra.update(arena_off=off, seed=SEED)
        if base not in ("adam", "adamw"):
            extra["t"] = STEP
        fn(*args, n, **extra)
    else:
        fn(*args, lp, n, **extra)


def _grouped_call(base, p, st, lp, table, groups, kw, gscale, coef, sr):
    fn = getattr(_native, base + "_mt_grouped" + ("_sr" if sr else ""))
    extra = dict(grad_scale=gscale, grad_scale_dev=coef, **kw)
    if base == "sgd_momentum":
        args = (p, st[0] if kw["mu"] else None)
        extra["first_step"] = False
    elif base in ("adam", "adamw"):
        args = (p, st[0], st[1], st[2] if len(st) > 2 else None)
    elif base == "rmsprop":
        args = (p, st[0], st[1] if kw["mu"] else None)
    else:
        args = (p, st[0])
    if sr:
        fn(*args, table, groups, seed=SEED, **extra)
    else:
        fn(*args, lp, table, groups, **extra)


def _zero_padding(slots, vecs):
    keep = torch.zeros(vecs[0].numel(), dtype=torch.bool, device=DEV)
    for s in slots:
        keep[s.offset:s.end] = True
    for v in vecs:
        v[~keep] = 0


@pytest.mark.parametrize("rule", sorted(RULES))
@pytest.mark.parametrize("shadow", [False, True])
@pytest.mark.parametrize("coef", [False, True])
@pytest.mark.parametrize("sr", [False, True])
def test_grouped_equals_the_ungrouped_kernel_per_segment(rule, shadow, coef, sr):
    """fp32 and bf16 gradients (alternating segments), a criterion segment (no FRL_LW_CLIPPED), three
    groups: each segment must come out bit for bit as the ungrouped kernel leaves it with its group's
    lr / wd and, on a model segment only, the clip coefficient.  The reference shares the rule functors
    of optim_rules.cuh with the code under test, so this checks the row, flag and segment selection;
    the rules themselves are checked against float64 torch.optim by the ungrouped kernels' suites, and
    against an independent float64 restatement below (test_grouped_sgd_and_adamw_against_float64)."""
    if sr and shadow:
        pytest.skip("the SR forms have no shadow: the bf16 vector is the weights")
    n_states, base, kw = RULES[rule]
    gen = torch.Generator(device=DEV).manual_seed(zlib.crc32(repr((rule, shadow, coef, sr)).encode()))
    slots, table, grads, total = _table(gen)
    p = torch.randn(total, device=DEV, generator=gen) * 0.5
    st = [torch.rand(total, device=DEV, generator=gen) * 0.05 for _ in range(n_states)]
    if sr:
        p = p.to(torch.bfloat16)
    _zero_padding(slots, [p] + st)
    lp = torch.zeros(total, device=DEV, dtype=torch.bfloat16) if shadow else None
    cdev = torch.tensor([0.75], device=DEV) if coef else None
    p2, st2, lp2 = p.clone(), [s.clone() for s in st], (lp.clone() if shadow else None)
    groups = _native.SegGroups(GROUP_OF, [_native.LW_CLIPPED if s.is_model else 0 for s in slots], _rows(base, kw))
    _grouped_call(base, p, st, lp, table, groups, kw, 0.5, cdev, sr)
    for s, gd, gi in zip(slots, grads, GROUP_OF):
        lr, wd = LR_WD[gi]
        sl = slice(s.offset, s.end)
        _flat_call(rule, base, p2[sl], gd, [x[sl] for x in st2], lp2[sl] if shadow else None, s.numel, lr, wd, kw,
                   0.5, cdev if s.is_model else None, sr, s.offset)
    torch.cuda.synchronize()
    assert torch.equal(p.view(torch.int16) if sr else p, p2.view(torch.int16) if sr else p2)
    for a, b in zip(st, st2):
        assert torch.equal(a, b)
    if shadow:
        assert torch.equal(lp, lp2)


@pytest.mark.parametrize("rule", ["sgd", "adamw"])
def test_grouped_sgd_and_adamw_against_float64(rule):
    """An independent float64 restatement of torch's SGD-momentum and AdamW, per element, with each
    segment's own lr / wd and the clip coefficient on model segments only: within a few fp32 roundings."""
    n_states, base, kw = RULES[rule]
    gen = torch.Generator(device=DEV).manual_seed(21)
    slots, table, grads, total = _table(gen)
    p = torch.randn(total, device=DEV, generator=gen) * 0.5
    st = [torch.rand(total, device=DEV, generator=gen) * 0.05 for _ in range(n_states)]
    _zero_padding(slots, [p] + st)
    p0, st0 = p.double().cpu(), [x.double().cpu() for x in st]
    coef = 0.75
    groups = _native.SegGroups(GROUP_OF, [_native.LW_CLIPPED if s.is_model else 0 for s in slots], _rows(base, kw))
    _grouped_call(base, p, st, None, table, groups, kw, 0.5, torch.tensor([coef], device=DEV), False)
    torch.cuda.synchronize()
    eps = float(np.finfo(np.float32).eps)
    for s, gd, gi in zip(slots, grads, GROUP_OF):
        lr, wd = LR_WD[gi]
        sl = slice(s.offset, s.end)
        g = gd.double().cpu() * 0.5 * (coef if s.is_model else 1.0)
        w = p0[sl]
        if rule == "sgd":
            d = g + wd * w
            buf = 0.9 * st0[0][sl] + d
            want_w, want_s = w - lr * buf, [buf]
            scale = [0.9 * st0[0][sl].abs() + g.abs() + wd * w.abs()]      # the summands' magnitudes
        else:
            w = w * (1 - lr * wd)
            m = st0[0][sl] + (1 - 0.9) * (g - st0[0][sl])
            v = 0.999 * st0[1][sl] + (1 - 0.999) * g * g
            bc1, bc2 = 1 - 0.9 ** STEP, 1 - 0.999 ** STEP
            want_w = w - (lr / bc1) * m / (v.sqrt() / bc2 ** 0.5 + 1e-8)
            want_s = [m, v]
            scale = [st0[0][sl].abs() + g.abs(), 0.999 * st0[1][sl] + g * g]
        got_w = p[sl].double().cpu()
        assert torch.all((got_w - want_w).abs() <= 8 * eps * (want_w.abs() + (want_w - p0[sl]).abs() + 1e-12)), gi
        for got, want, mag in zip(st, want_s, scale):
            got = got[sl].double().cpu()
            assert torch.all((got - want).abs() <= 8 * eps * (mag + 1e-30)), gi


@pytest.mark.parametrize("lion", [False, True])
@pytest.mark.parametrize("sr", [False, True])
def test_k12_with_a_later_group_row_equals_dw_gemm_then_grouped_k2_mt(lion, sr):
    """K12 given group 2's row as its dyn (and that group's lr / wd by value, as the optimizer passes
    them) against dw_gemm + the grouped K2-mt over a one-slot table whose slot is in group 2."""
    out, inp, rows_n = 384, 768, 256
    gen = torch.Generator(device=DEV).manual_seed(31 + 2 * lion + sr)
    dz = torch.randn(rows_n, out, device=DEV, generator=gen).to(torch.bfloat16)
    x = torch.randn(rows_n, inp, device=DEV, generator=gen).to(torch.bfloat16)
    n = out * inp
    p = torch.randn(n, device=DEV, generator=gen) * 0.05
    m = torch.randn(n, device=DEV, generator=gen) * 1e-2
    w = p.to(torch.bfloat16)
    base = "lion" if lion else "sgd_momentum"
    kw = dict(beta1=0.9, beta2=0.99) if lion else dict(mu=0.9, dampening=0.0)
    rows = _rows(base, kw)
    lr, wd = LR_WD[2]
    gw_ref = torch.empty(out, inp, device=DEV, dtype=torch.bfloat16)
    _native.dw_gemm(dz, x, gw_ref)

    class _S:
        index, offset, numel, shape, is_model, end = 0, 0, n, (n,), True, n
    table = GradSegTable([_S()], torch.device(DEV))
    table.point(_S(), gw_ref.data_ptr(), gw_ref.dtype)
    table.upload()
    groups = _native.SegGroups([2], [_native.LW_CLIPPED], rows)
    p_ref, m_ref, w_ref = p.clone(), m.clone(), w.clone()
    lp_ref = torch.empty(n, device=DEV, dtype=torch.bfloat16)
    gw, lp = torch.empty_like(gw_ref), torch.empty_like(lp_ref)
    by_value = dict(lr=lr, wd=wd, beta1=0.9, beta2=0.99) if lion else dict(lr=lr, wd=wd, mu=0.9, dampening=0.0,
                                                                           first_step=False)
    if sr:
        _grouped_call(base, w_ref, [m_ref], None, table, groups, kw, 0.25, None, True)
        fn = _native.dw_gemm_lion_sr if lion else _native.dw_gemm_sgd_sr
        fn(dz, x, gw, w, m, arena_off=0, seed=SEED, t=STEP, **by_value, grad_scale=0.25, dyn=rows[2])
    else:
        _grouped_call(base, p_ref, [m_ref], lp_ref, table, groups, kw, 0.25, None, False)
        fn = _native.dw_gemm_lion if lion else _native.dw_gemm_sgd
        fn(dz, x, gw, p, m, lp, **by_value, grad_scale=0.25, dyn=rows[2])
    torch.cuda.synchronize()
    assert torch.equal(gw, gw_ref) and torch.equal(m, m_ref)
    if sr:
        assert torch.equal(w.view(torch.int16), w_ref.view(torch.int16))
    else:
        assert torch.equal(p, p_ref) and torch.equal(lp, lp_ref)


def test_two_ranks_agree_and_match_one_gpu_at_the_global_batch():
    """tests/run_param_groups_mp.py: over gloo with both ranks on GPU 0 when only one GPU is visible (the
    NCCL run reported as not run), over NCCL where two or more GPUs are visible."""
    import os
    import subprocess
    import sys
    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    backend = "nccl" if torch.cuda.device_count() >= 2 else "gloo"
    res = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nproc-per-node", "2",
                          os.path.join(repo, "tests", "run_param_groups_mp.py"), "--backend", backend],
                         capture_output=True, text=True, timeout=600, cwd=repo)
    print(res.stdout[-3000:])
    assert res.returncode == 0 and res.stdout.count("PARAM_GROUPS_MP_OK") == 2, res.stdout[-3000:] + res.stderr[-3000:]
    assert "PARAM_GROUPS_NCCL" in res.stdout


def test_one_group_is_bit_equal_to_the_ungrouped_mt_kernel():
    gen = torch.Generator(device=DEV).manual_seed(11)
    slots, table, grads, total = _table(gen)
    p = torch.randn(total, device=DEV, generator=gen) * 0.5
    m, v = (torch.rand(total, device=DEV, generator=gen) * 0.05 for _ in range(2))
    _zero_padding(slots, [p, m, v])
    p2, m2, v2 = p.clone(), m.clone(), v.clone()
    kw = dict(beta1=0.9, beta2=0.999, eps=1e-8)
    rows = _rows("adamw", kw)[:1].contiguous()
    lr, wd = LR_WD[0]
    _native.adamw_mt_grouped(p, m, v, None, None, table, _native.SegGroups([0] * len(slots), [0] * len(slots), rows),
                             **kw, grad_scale=0.5)
    _native.adamw_mt(p2, m2, v2, None, None, table, lr=lr, wd=wd, step=STEP, **kw, grad_scale=0.5)
    torch.cuda.synchronize()
    assert torch.equal(p, p2) and torch.equal(m, m2) and torch.equal(v, v2)


def test_group_index_out_of_range_is_refused_before_a_launch():
    with pytest.raises(_native.NativeLibraryError, match=r"group indices \[3\] outside \[0, 3\)"):
        _native.SegGroups([0, 3], [0, 0], torch.zeros(3, _native.GROUP_DYN_COLS, device=DEV))


def test_a_captured_graph_follows_per_group_lr_changes_through_the_rows():
    gen = torch.Generator(device=DEV).manual_seed(13)
    slots, table, grads, total = _table(gen)
    p = torch.randn(total, device=DEV, generator=gen) * 0.5
    buf = torch.zeros(total, device=DEV)
    _zero_padding(slots, [p])
    rows = _rows("sgd_momentum", dict(mu=0.9))
    groups = _native.SegGroups(GROUP_OF, [0] * len(slots), rows)
    p_ref, buf_ref = p.clone(), buf.clone()
    graph = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        _native.sgd_momentum_mt_grouped(p.clone(), buf.clone(), None, table, groups, mu=0.9, dampening=0.0)
        torch.cuda.synchronize()
        with torch.cuda.graph(graph, stream=side):
            _native.sgd_momentum_mt_grouped(p, buf, None, table, groups, mu=0.9, dampening=0.0)
    for k in range(3):
        new = rows.clone()
        new[:, 0] *= 0.5 ** k
        new[1, 0] *= 3.0                                   # one group moves on its own
        rows.copy_(new)
        graph.replay()
        for s, gd, gi in zip(slots, grads, GROUP_OF):
            sl = slice(s.offset, s.end)
            _native.sgd_momentum(p_ref[sl], gd, buf_ref[sl], None, s.numel, lr=float(new[gi, 0]), mu=0.9,
                                 dampening=0.0, wd=float(new[gi, 4]))
        torch.cuda.synchronize()
        assert torch.equal(p, p_ref) and torch.equal(buf, buf_ref), k


# ---- through Solver.build_worker ------------------------------------------------------------------------

def _hook(model):
    """1-D parameters without decay, the last two 2-D parameters (the heads) at 2x lr, and the first
    trunk weight in the LAST group at half the lr, so K12 runs with a row other than row 0."""
    params = list(model.parameters())
    mats = [p for p in params if p.ndim == 2]
    return [{"params": [p for p in params if p.ndim <= 1], "weight_decay": 0.0},
            {"params": mats[-2:], "lr": 2e-3},
            {"params": [mats[0]], "lr": 0.5e-3}]


def _worker(algo=OptAlgorithm.SGD, precision=Precision.FP32, hook=True, no_decay=None, seed=0, graph=False,
            lr=1e-3, **kw):
    ns = synthetic.api_namespace("frl_b200")
    t = ns.types
    save_dir = tempfile.mkdtemp(prefix="frl_b200_groups_")
    torch.manual_seed(seed)
    problem = synthetic.make_mlp_problem(ns, save_dir, n_train=8, width=512, n_classes=100, reg_dim=16, depth=3)
    if hook:
        problem.__class__ = type("Hooked", (type(problem),), {"get_param_groups": lambda self, m: _hook(m)})
    run_opts = t.RunOpts(optim=t.OptimOpts(algo=algo, lr=lr, momentum=0.9, weightDecay=0.1),
                         batchSize=256, nEpochs=1, numThreads=0, singleThreaded=True, numVisualizedSamples=0)
    args = SolverWorkerArgs(run_opts=run_opts, problem=problem, save_dir=save_dir, run_device=Device.GPU,
                            node_idx=0, node_count=1, rank=0, local_rank=0, world_size=1, group_name=None,
                            init_method="", precision=precision, graph_step=graph, no_decay_1d=no_decay, **kw)
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


def _params(worker):
    return list(worker.model.parameters()) + list(worker.criterion.parameters())


def _weights(worker):
    with worker.arena.exported(cpu=False):
        return [p.detach().float().clone() for p in _params(worker)]


def _gap(a, b, p0):
    return max(((x - y).norm() / (y - q).norm().clamp_min(1e-30)).item() for x, y, q in zip(a, b, p0))


TORCH = {
    "sgd": (OptAlgorithm.SGD, {}, lambda g: torch.optim.SGD(g, lr=1e-3, momentum=0.9, weight_decay=0.1)),
    "adam": (OptAlgorithm.ADAM, {}, lambda g: torch.optim.Adam(g, lr=1e-3, weight_decay=0.1)),
    "adamw": (OptAlgorithm.ADAM, {"adamw": True}, lambda g: torch.optim.AdamW(g, lr=1e-3, weight_decay=0.1)),
    "rmsprop": (OptAlgorithm.RMSPROP, {}, lambda g: torch.optim.RMSprop(g, lr=1e-3, momentum=0.9, weight_decay=0.1)),
    "lion": (OptAlgorithm.SGD, {"lion": True}, None),
}


@pytest.mark.parametrize("kind", sorted(TORCH))
@pytest.mark.parametrize("mode", ["hook", "no_decay_1d"])
def test_solver_mlp_tracks_torch_optim_with_the_same_groups(kind, mode):
    """FP32, TF32 off, 10 steps: the Solver against stock autograd + torch.optim (Lion: RefLion) built
    with the Solver's canonical groups.  The runs differ in rounding order only, so the largest
    per-parameter update gap must be far below the gap to the same Solver run without groups, or, where
    that run differs from the groups' only by lr*wd*p on the 1-D parameters (AdamW with no_decay_1d:
    measured on an H100 80GB HBM3 at 700 W, gap 1.5e-2 against 4.3e-2 without groups; Adam normalises
    near-zero gradients, which magnifies rounding-order differences), below 0.05 of the update.  Every
    other case measured 0 to 6e-3 against 0.19 to 27 without groups."""
    from lion_oracle import RefLion
    from oracle import ref_loop
    algo, kw, make = TORCH[kind]
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        batches = _batches(10)
        lr = 1e-4 if kind == "lion" else 1e-3
        w = _worker(algo, hook=mode == "hook", no_decay=mode == "no_decay_1d", lr=lr, **kw)
        assert w.optimizer.grouped and w.pipeline.whole_tensors and not w.pipeline.eager
        p0 = _weights(w)
        ns = synthetic.api_namespace("frl_b200")
        ref_problem = synthetic.make_mlp_problem(ns, tempfile.mkdtemp(prefix="frl_b200_groups_ref_"), n_train=8,
                                                 width=512, n_classes=100, reg_dim=16, depth=3)
        ref = ref_problem.get_model().cuda()
        ref.load_state_dict(w.model.state_dict())
        crit = ref_problem.get_criterion().cuda()
        crit.load_state_dict(w.criterion.state_dict())
        mine = dict(zip(map(id, _params(w)), list(ref.parameters()) + list(crit.parameters())))
        groups = [dict({k: v for k, v in g.items() if k in ("lr", "weight_decay")},
                       params=[mine[id(p)] for p in g["params"]]) for g in w.optimizer.param_groups]
        opt = (RefLion(groups, lr=lr, betas=(0.9, 0.99), weight_decay=0.1) if kind == "lion" else make(groups))
        mods, weights, names = list(crit.loss_modules), list(crit.loss_weights), list(crit.loss_names)
        _train(w, batches)
        for x, y, r in batches:
            opt.zero_grad()
            total, _ = ref_loop.parallel_criterion(mods, weights, names, ref([x.cuda()]), [(y.cuda(),), (r.cuda(),)])
            total.backward()
            opt.step()
        torch.cuda.synchronize()
        plain = _worker(algo, hook=False, lr=lr, **kw)
        _train(plain, batches)
        theirs = [p.detach().float() for p in list(ref.parameters()) + list(crit.parameters())]
        gap, gap_plain = _gap(_weights(w), theirs, p0), _gap(_weights(plain), theirs, p0)
        print("%s %s: gap %.3e, without groups %.3e" % (kind, mode, gap, gap_plain))
        assert gap < 0.1 * gap_plain or (kind == "adamw" and mode == "no_decay_1d" and gap < 0.05), (gap, gap_plain)
        if mode == "no_decay_1d" and kind == "sgd":
            # a 1-D parameter is untouched by decay: same update as with wd 0 in torch
            for a, b in zip(_weights(w), theirs):
                if a.dim() <= 1:
                    assert torch.allclose(a, b, rtol=1e-4, atol=1e-6)
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


@pytest.mark.parametrize("master", [MasterWeights.FP32, MasterWeights.BF16])
@pytest.mark.parametrize("lion", [False, True])
def test_k12_with_a_grouped_trunk_weight_resume_and_graph_replay(master, lion):
    batches = _batches(10)
    x = _worker(precision=Precision.BF16, master_weights=master, lion=lion, lr=1e-4 if lion else 1e-3)
    assert x.pipeline.fused_dw_update and x.optimizer.grouped
    _train(x, batches[:5])
    first = x.arena.slots[[id(s.param) for s in x.arena.slots].index(id(_hook(x.model)[2]["params"][0]))]
    assert first.index in x.pipeline.dw_updated, "the grouped trunk weight did not go through K12"
    saved = _weights(x)
    sd = x.optimizer.state_dict()
    assert len(sd["param_groups"]) == 4 and sd["param_groups"][2]["lr"] == 0.5e-3
    assert x.optimizer._group_of[id(first.param)] == 2
    rows_x = _train(x, batches[5:], 5)
    y = _worker(precision=Precision.BF16, master_weights=master, lion=lion, lr=1e-4 if lion else 1e-3, seed=7)
    y.arena.load_master_from_params(list(zip(_params(y), saved)))
    y.optimizer.load_state_dict(sd)
    rows_y = _train(y, batches[5:], 5)
    assert rows_x == rows_y and torch.equal(x.arena.lp, y.arena.lp)
    eager = _worker(precision=Precision.BF16, master_weights=master, lion=lion, lr=1e-4 if lion else 1e-3)
    graphed = _worker(precision=Precision.BF16, master_weights=master, lion=lion, lr=1e-4 if lion else 1e-3,
                      graph=True)
    a = _train(eager, batches[:5])
    b = _train(graphed, batches[:5])
    for wk in (eager, graphed):                  # a schedule step between replays: every group's lr moves
        for g in wk.optimizer.param_groups:
            g["lr"] *= 0.5
    a += _train(eager, batches[5:], 5)
    b += _train(graphed, batches[5:], 5)
    assert graphed.graphed is not None and a == b
    assert torch.equal(eager.arena.lp, graphed.arena.lp)


@pytest.mark.parametrize("combo", ["accumulation_clip", "fp8", "ema", "bf16_master", "graph", "adamw"])
def test_solver_loop_in_combination(combo, tmp_path):
    ns = synthetic.api_namespace("frl_b200")
    t = ns.types
    torch.manual_seed(0)
    problem = synthetic.make_mlp_problem(ns, str(tmp_path), n_train=2048, width=512, n_classes=100, reg_dim=16,
                                         depth=3)
    run_opts = t.RunOpts(optim=t.OptimOpts(algo=t.OptAlgorithm.ADAM if combo == "adamw" else t.OptAlgorithm.SGD,
                                           lr=1e-3, momentum=0.9, weightDecay=0.1,
                                           gradientClip=1.0 if combo == "accumulation_clip" else 0.0),
                         batchSize=256, nEpochs=2, numThreads=0, singleThreaded=True, numVisualizedSamples=0)
    kw = dict(precision=Precision.FP8 if combo == "fp8" else Precision.BF16,
              grad_accumulation=2 if combo == "accumulation_clip" else 1, ema_decay=0.9 if combo == "ema" else 0.0,
              master_weights=MasterWeights.BF16 if combo == "bf16_master" else MasterWeights.FP32,
              graph_step=combo == "graph", adamw=combo == "adamw")
    args = SolverWorkerArgs(run_opts=run_opts, problem=problem, save_dir=str(tmp_path), run_device=Device.GPU,
                            node_idx=0, node_count=1, rank=0, local_rank=0, world_size=1, group_name=None,
                            init_method="", no_decay_1d=True, **kw)
    rows = [frac.performance[t.Split.TRAIN].losses for frac in Solver._run_solver_worker(args)]
    totals = [sum(float(v) for v in r.values()) for r in rows]
    assert all(np.isfinite(totals)) and totals[-1] < totals[0], totals


def test_channels_last_resnet_trains(tmp_path):
    ns = synthetic.api_namespace("frl_b200")
    t = ns.types
    torch.manual_seed(0)
    problem = synthetic.make_resnet_problem(ns, str(tmp_path), "resnet18", image=64, n_train=128)
    run_opts = t.RunOpts(optim=t.OptimOpts(algo=t.OptAlgorithm.SGD, lr=1e-3, momentum=0.9, weightDecay=0.1),
                         batchSize=32, nEpochs=2, numThreads=0, singleThreaded=True, numVisualizedSamples=0)
    args = SolverWorkerArgs(run_opts=run_opts, problem=problem, save_dir=str(tmp_path), run_device=Device.GPU,
                            node_idx=0, node_count=1, rank=0, local_rank=0, world_size=1, group_name=None,
                            init_method="", precision=Precision.BF16, channels_last=True, no_decay_1d=True)
    rows = [frac.performance[t.Split.TRAIN].losses for frac in Solver._run_solver_worker(args)]
    totals = [sum(float(v) for v in r.values()) for r in rows]
    assert all(np.isfinite(totals)), totals
