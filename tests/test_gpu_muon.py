"""K14 (Muon) on the H100, against the restatement in ``muon_oracle`` and torch's own Newton-Schulz.

Bounds: relative Frobenius error 3e-2.  The restatement agrees with
``torch.optim._muon._zeropower_via_newtonschulz`` on CPU bf16 tensors to 1.2e-2 (float64
accumulation) and 1.7e-2 (fp32 accumulation) over random, low-rank and tiny gradients: every
product rounds to bf16, and Newton-Schulz amplifies the rounding of small singular values.  The
kernel accumulates in fp32 in its own order, so it is held to the same bound against both.
"""
import pytest
import torch
import torch.nn as nn

import frl_b200  # noqa: F401
from frl_b200 import fused_optim
from frl_b200.arena import ParamArena
from frl_b200.multi_tensor import GradSegTable
from frl_b200.types import Precision
import muon_oracle as mo

pytestmark = pytest.mark.gpu
DEV = "cuda"
NS_SHAPES = ((4096, 4096), (1000, 4096), (64, 4096), (4096, 1000), (300, 700), (1, 512))
TOL = 3e-2


def _rel(got, want):
    return ((got.double() - want.double()).norm() / want.double().norm().clamp_min(1e-30)).item()


def _grad(shape, kind, gen):
    if kind == "lowrank":
        r = 8
        g = torch.randn(shape[0], r, generator=gen) @ torch.randn(r, shape[1], generator=gen)
        return g + 1e-3 * torch.randn(shape, generator=gen)
    return torch.randn(shape, generator=gen)


class _Case:
    """Muon matrices (plus one bias for the Adam half) in a real arena, gradients read in place."""

    def __init__(self, shapes, *, shadow=True, gdt=torch.float32, seed=0, lr=0.02, wd=0.01, momentum=0.95,
                 nesterov=True, adjust="match_rms_adamw"):
        gen = self.gen = torch.Generator().manual_seed(seed)
        self.params = [nn.Parameter(torch.randn(sh, generator=gen) * 0.02) for sh in shapes]
        self.params.append(nn.Parameter(torch.randn(17, generator=gen)))
        self.arena = ParamArena(self.params, device=DEV, precision=Precision.BF16 if shadow else Precision.FP32)
        self.opt = fused_optim.FusedMuon(self.arena, lr=lr, weight_decay=wd, momentum=momentum, nesterov=nesterov,
                                         adjust_lr_fn=adjust)
        self.table = GradSegTable(self.arena.slots, self.arena.device)
        self.gdt = gdt

    def point(self, grads):
        self.grads = [g.to(self.gdt).to(DEV).contiguous() for g in grads]
        for s, g in zip(self.arena.slots, self.grads):
            self.table.point(s, g.data_ptr(), g.dtype)
        self.table.upload()

    def step(self, gs=1.0, coef=None):
        self.opt.begin_step()
        self.opt.apply_table(self.table, grad_scale=gs, clip_coef_dev=coef)
        self.opt.end_step()

    def master(self, i):
        s = self.arena.slots[i]
        return self.arena.master[s.offset:s.end].view(s.shape)


@pytest.mark.parametrize("shape", NS_SHAPES)
@pytest.mark.parametrize("kind", ["normal", "lowrank"])
def test_newton_schulz_alone(shape, kind):
    """momentum 0, no nesterov, lr 1, wd 0, weights 0: the update is -adj * O."""
    case = _Case([shape], shadow=False, lr=1.0, wd=0.0, momentum=0.0, nesterov=False, adjust="original")
    case.arena.master.zero_()
    g = _grad(shape, kind, case.gen)
    case.point([g, torch.zeros(17)])
    case.step()
    torch.cuda.synchronize()
    got = -case.master(0) / mo.adjust_factor(shape, "original")
    want = mo.newton_schulz(g)
    assert _rel(got.cpu(), want) < TOL
    from torch.optim._muon import _zeropower_via_newtonschulz
    ref = _zeropower_via_newtonschulz(g.to(DEV), mo.MUON_NS_COEFFICIENTS, 5, 1e-7)
    assert _rel(got, ref) < TOL


def _full_check(case, steps, gs=1.0, coef=None, edit=None):
    h = case.opt.muon_group
    ref_p = [case.master(i).detach().cpu().double() for i in range(len(case.params) - 1)]
    ref_b = [torch.zeros(p.shape) for p in ref_p]
    for t in range(steps):
        grads = [torch.randn(p.shape, generator=case.gen) * 0.1 for p in case.params]
        if edit is not None:
            edit(grads)
        case.point(grads)
        case.step(gs, None if coef is None else torch.tensor([coef], device=DEV))
        for i in range(len(ref_p)):
            g = case.grads[i].float().cpu() * torch.tensor(gs, dtype=torch.float32) * \
                torch.tensor(1.0 if coef is None else coef, dtype=torch.float32)
            ref_p[i], ref_b[i] = mo.muon_step(ref_p[i], g, ref_b[i], lr=h["lr"], wd=h["weight_decay"],
                                              momentum=h["momentum"], nesterov=h["nesterov"],
                                              adjust_lr_fn=h["adjust_lr_fn"])
    torch.cuda.synchronize()
    return ref_p, ref_b


@pytest.mark.parametrize("gdt", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("shadow", [True, False])
def test_full_update_against_restatement(gdt, shadow):
    shapes = ((300, 700), (700, 300), (1, 512), (256, 256))
    case = _Case(shapes, shadow=shadow, gdt=gdt, seed=1)
    p0 = [case.master(i).detach().cpu().double() for i in range(len(shapes))]
    ref_p, ref_b = _full_check(case, 3, gs=0.5, coef=0.75)
    for i, sh in enumerate(shapes):
        got = case.master(i).cpu().double()
        assert _rel(got - p0[i], ref_p[i] - p0[i]) < TOL, sh
        s = case.arena.slots[i]
        buf = case.opt._state("exp_avg")[s.offset:s.end].view(sh).cpu()
        torch.testing.assert_close(buf, ref_b[i], rtol=1e-5, atol=1e-7)
        if shadow:
            assert torch.equal(case.arena.lp[s.offset:s.end].view(sh), case.master(i).to(torch.bfloat16))


def test_zero_gradient_only_decays_and_nan_poisons_its_matrix():
    case = _Case(((64, 96), (96, 64)), seed=2, lr=0.1, wd=0.5)
    p0 = [case.master(i).clone() for i in range(2)]
    case.point([torch.zeros(64, 96), torch.zeros(96, 64), torch.zeros(17)])
    case.step()
    torch.cuda.synchronize()
    decay = torch.tensor(1 - 0.1 * 0.5, dtype=torch.float32).item()
    for i in range(2):
        torch.testing.assert_close(case.master(i), p0[i] * decay, rtol=1e-6, atol=0)
    g = torch.randn(64, 96, generator=case.gen)
    g[3, 5] = float("nan")
    case.point([g, torch.randn(96, 64, generator=case.gen), torch.zeros(17)])
    case.step()
    torch.cuda.synchronize()
    assert torch.isnan(case.master(0)).all()
    assert torch.isfinite(case.master(1)).all()


def test_two_launches_give_the_same_bytes_and_graph_replay_takes_lr_from_dyn():
    shapes = ((1000, 4096), (300, 700))

    def run(graph):
        case = _Case(shapes, seed=3)
        grads = [torch.randn(p.shape, generator=case.gen) for p in case.params]
        case.point(grads)
        case.opt.enable_dynamic_scalars()
        if graph:
            case.step()                                   # warm-up: plans, workspace
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                g = torch.cuda.CUDAGraph()
                case.opt.begin_step()
                with torch.cuda.graph(g, stream=s):
                    case.opt.apply_table(case.table)
                case.opt.end_step()
            torch.cuda.current_stream().wait_stream(s)
            case.opt._steps -= 1                          # the capture ran no update
            for lr in (0.02, 0.05, 0.01):
                for grp in case.opt.param_groups:
                    grp["lr"] = lr
                case.opt.begin_step()
                g.replay()
                case.opt.end_step()
        else:
            for lr in (0.02, 0.02, 0.05, 0.01):
                for grp in case.opt.param_groups:
                    grp["lr"] = lr
                case.step()
        torch.cuda.synchronize()
        return case.arena.master.clone(), case.opt._state("exp_avg").clone()

    a, b = run(False), run(False)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    c = run(True)
    assert torch.equal(a[0], c[0]) and torch.equal(a[1], c[1])


def test_state_dict_moves_to_torch_muon_and_back():
    case = _Case(((64, 96), (96, 64)), seed=4)
    case.point([torch.randn(p.shape, generator=case.gen) for p in case.params])
    case.step()
    sd = case.opt.state_dict()
    muon_sd, adam_sd = fused_optim.split_muon_state_dict(sd)
    ps = [nn.Parameter(case.master(i).clone()) for i in range(2)]
    m = torch.optim.Muon(ps, lr=0.02, adjust_lr_fn="match_rms_adamw")
    m.load_state_dict(muon_sd)
    a = torch.optim.Adam([nn.Parameter(torch.zeros(17, device=DEV))], lr=0.02)
    a.load_state_dict(adam_sd)
    back = fused_optim.join_muon_state_dict(m.state_dict(), a.state_dict())
    other = _Case(((64, 96), (96, 64)), seed=5)
    other.opt.load_state_dict(back)
    assert torch.equal(other.opt._state("exp_avg"), case.opt._state("exp_avg"))


# ---- through the solver ----------------------------------------------------------------------------

def _worker(precision, seed=0, lr=1e-3, muon=True, **kw):
    import tempfile

    from frl_b200 import synthetic
    from frl_b200.solver import Solver, SolverWorkerArgs
    from frl_b200.types import Device
    ns = synthetic.api_namespace("frl_b200")
    t = ns.types
    save_dir = tempfile.mkdtemp(prefix="frl_b200_muon_")
    torch.manual_seed(seed)
    problem = synthetic.make_mlp_problem(ns, save_dir, n_train=8, width=512, n_classes=100, reg_dim=16, depth=3)
    run_opts = t.RunOpts(optim=t.OptimOpts(algo=t.OptAlgorithm.ADAM, lr=lr, weightDecay=1e-5, momentum=0.95),
                         batchSize=256, nEpochs=1, numThreads=0, singleThreaded=True, numVisualizedSamples=0)
    args = SolverWorkerArgs(run_opts=run_opts, problem=problem, save_dir=save_dir, run_device=Device.GPU,
                            node_idx=0, node_count=1, rank=0, local_rank=0, world_size=1, group_name=None,
                            init_method="", precision=precision, muon=muon, **kw)
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
    from frl_b200.types import Split
    rows = []
    for i, (x, y, r) in enumerate(batches, start):
        _, total, _, _ = worker._pass_one_minibatch(i, Split.TRAIN, [x.cuda()], [(y.cuda(),), (r.cuda(),)])
        rows.append(float(total.detach()))
        del total
    torch.cuda.synchronize()
    return rows


def _params(worker):
    return [p.detach().float().clone() for p in list(worker.model.parameters()) + list(worker.criterion.parameters())]


def _gap(a, b, p0):
    """Largest over the parameters of ||a - b|| / ||b - p0||: how far apart two runs' updates are."""
    return max(((x - y).norm() / (y - q).norm().clamp_min(1e-30)).item() for x, y, q in zip(a, b, p0))


def test_solver_matches_a_torch_muon_and_adam_loop():
    """Precision.FP32, width-512 MLP, batch 256, 40 steps: the Solver with muon=True against stock
    autograd + torch.optim.Muon (the 2-D model weights) + torch.optim.Adam (the rest) with the same
    hyper-parameters.  Both round every Newton-Schulz product to bf16 in their own order, so the two
    runs drift apart a little; they must stay far closer to each other than a Muon run is to an Adam
    run.  Measured on an H100 (seed 0, this test): the largest per-parameter update gap to torch is
    0.103 of the update, an Adam run's is 2.03, and the last loss rows agree to 3e-5 relative.
    TOL_RUN = 0.2 is twice the measured gap and a tenth of the Adam gap, so the test separates the
    two optimizers."""
    import tempfile

    from frl_b200 import synthetic
    from oracle import ref_loop
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        batches = _batches(40)
        w = _worker(Precision.FP32)
        assert type(w.optimizer) is fused_optim.FusedMuon
        p0 = _params(w)
        ns = synthetic.api_namespace("frl_b200")
        ref_problem = synthetic.make_mlp_problem(ns, tempfile.mkdtemp(prefix="frl_b200_muon_ref_"), n_train=8,
                                                 width=512, n_classes=100, reg_dim=16, depth=3)
        ref = ref_problem.get_model().cuda()
        ref.load_state_dict(w.model.state_dict())
        crit = ref_problem.get_criterion().cuda()
        crit.load_state_dict(w.criterion.state_dict())
        mods, weights, names = list(crit.loss_modules), list(crit.loss_weights), list(crit.loss_names)
        params = list(ref.parameters()) + list(crit.parameters())
        mats = [p for p in ref.parameters() if p.ndim == 2]
        rest = [p for p in params if all(p is not q for q in mats)]
        om = torch.optim.Muon(mats, lr=1e-3, weight_decay=1e-5, momentum=0.95, adjust_lr_fn="match_rms_adamw")
        oa = torch.optim.Adam(rest, lr=1e-3, weight_decay=1e-5)
        ref.train()
        crit.train()
        got = _train(w, batches)
        want = []
        for x, y, r in batches:
            om.zero_grad()
            oa.zero_grad()
            total, _ = ref_loop.parallel_criterion(mods, weights, names, ref([x.cuda()]), [(y.cuda(),), (r.cuda(),)])
            total.backward()
            want.append(total.item())
            om.step()
            oa.step()
        torch.cuda.synchronize()
        adam = _worker(Precision.FP32, muon=False)
        _train(adam, batches)
        mine, theirs = _params(w), [p.detach().float() for p in params]
        gap_torch = _gap(mine, theirs, p0)
        gap_adam = _gap(_params(adam), theirs, p0)
        print("gap to torch %.3e, Adam run to torch %.3e, last rows %r %r" % (gap_torch, gap_adam, got[-1], want[-1]))
        assert gap_torch < TOL_RUN and gap_torch < 0.1 * gap_adam, (gap_torch, gap_adam)
        assert abs(got[-1] - want[-1]) < 0.1 * abs(want[0] - want[-1]), (got[-1], want[-1])
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


TOL_RUN = 0.2


def test_checkpoint_resume_continues_bit_for_bit():
    batches = _batches(12)
    a = _worker(Precision.FP32)
    _train(a, batches[:6])
    model_sd = {k: v.detach().clone() for k, v in a.model.state_dict().items()}
    opt_sd = a.optimizer.state_dict()
    rows_a = _train(a, batches[6:], 6)
    b = _worker(Precision.FP32, seed=7)
    b.model.load_state_dict(model_sd)
    b.optimizer.load_state_dict(opt_sd)
    rows_b = _train(b, batches[6:], 6)
    assert rows_a == rows_b
    assert torch.equal(a.arena.master, b.arena.master)
    assert torch.equal(a.optimizer._state("exp_avg"), b.optimizer._state("exp_avg"))


@pytest.mark.parametrize("combo", ["graph", "fp8", "accumulation", "ema"])
def test_solver_loop_with_muon_in_combination(combo, tmp_path):
    """The solver's own loop (epochs, schedule, checkpoints) with muon=True: the losses stay finite
    and fall, and the update ran through K14."""
    from frl_b200 import _native, synthetic
    from frl_b200.solver import Solver, SolverWorkerArgs
    from frl_b200.types import Device
    ns = synthetic.api_namespace("frl_b200")
    t = ns.types
    torch.manual_seed(0)
    problem = synthetic.make_mlp_problem(ns, str(tmp_path), n_train=2048, width=512, n_classes=100, reg_dim=16,
                                         depth=3)
    run_opts = t.RunOpts(optim=t.OptimOpts(algo=t.OptAlgorithm.ADAM, lr=1e-3, weightDecay=1e-5, momentum=0.95,
                                           gradientClip=1.0 if combo == "accumulation" else 0.0),
                         batchSize=256, nEpochs=2, numThreads=0, singleThreaded=True, numVisualizedSamples=0)
    kw = dict(graph_step=combo == "graph", precision=Precision.FP8 if combo == "fp8" else Precision.BF16,
              grad_accumulation=2 if combo == "accumulation" else 1, ema_decay=0.9 if combo == "ema" else 0.0)
    args = SolverWorkerArgs(run_opts=run_opts, problem=problem, save_dir=str(tmp_path), run_device=Device.GPU,
                            node_idx=0, node_count=1, rank=0, local_rank=0, world_size=1, group_name=None,
                            init_method="", muon=True, **kw)
    rows = []
    for frac in Solver._run_solver_worker(args):
        rows.append(frac.performance[t.Split.TRAIN].losses)
    totals = [sum(float(v) for v in r.values()) for r in rows]
    assert all(torch.isfinite(torch.tensor(totals))) and totals[-1] < totals[0], totals


def test_two_ranks_on_one_gpu_equal_one_rank_at_the_double_batch():
    """tests/run_muon_mp.py over gloo, both ranks on GPU 0 (NCCL needs one GPU per rank)."""
    import os
    import subprocess
    import sys
    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    backend = "nccl" if torch.cuda.device_count() >= 2 else "gloo"
    res = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nproc-per-node", "2",
                          os.path.join(repo, "tests", "run_muon_mp.py"), "--backend", backend],
                         capture_output=True, text=True, timeout=600, cwd=repo)
    assert res.returncode == 0 and res.stdout.count("MUON_MP_OK") == 2, res.stdout[-3000:] + res.stderr[-3000:]
