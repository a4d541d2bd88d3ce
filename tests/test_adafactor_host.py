"""Adafactor (K2-af) on the host: the float64 restatement against ``torch.optim.Adafactor``, the
switch and its refusals, the pipeline's launch sequence, torch-format state in both directions,
unused parameters and argument checks of the C entry point, with the kernel replaced by a CPU
double."""
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn as nn

import frl_b200  # noqa: F401
from frl_b200 import _native, fused_optim, grad_sync, synthetic
from frl_b200.arena import ParamArena
from frl_b200.solver import Solver, SolverWorkerArgs, resolve_adafactor
from frl_b200.types import LayerAdaptation, Mode, OptAlgorithm, OptimizerState, OptimOpts
import adafactor_oracle as af
from adafactor_oracle import AdafactorKernelDouble

SHAPES = ((37, 130), (1, 64), (64, 1), (8, 4, 3, 3), (6, 5, 1, 1), (1000,), ())
EPS1 = 2.0 ** -23


@pytest.fixture()
def double(monkeypatch):
    d = AdafactorKernelDouble()
    monkeypatch.setattr(fused_optim, "KERNELS", d)
    monkeypatch.setattr(grad_sync, "KERNELS", d)
    return d


def _net(seed=0):
    torch.manual_seed(seed)
    return nn.Sequential(nn.Linear(7, 30), nn.ReLU(), nn.Linear(30, 5), nn.ReLU(), nn.Linear(5, 1))


def _opts(**kw):
    kw.setdefault("algo", OptAlgorithm.ADAM)
    return OptimOpts(lr=0.01, weightDecay=1e-2, **kw)


def _make(net):
    arena = ParamArena(net.parameters(), device="cpu")
    return arena, fused_optim.create_fused_optimizer(arena, _opts(), adafactor=True)


# ---- the restatement -----------------------------------------------------------------------------

@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("lr", [1e-2, 0.8])          # below and above 1/sqrt(t) for t <= 5
def test_restatement_equals_torch_adafactor_in_float64(shape, lr):
    gen = torch.Generator().manual_seed(len(shape) * 31 + int(lr * 10))
    p0 = torch.randn(shape, generator=gen, dtype=torch.float64)
    param = nn.Parameter(p0.clone())
    ref = torch.optim.Adafactor([param], lr=lr, weight_decay=0.1, eps=(EPS1, 1e-3), foreach=False)
    p, st = p0.numpy().ravel().copy(), af.zero_state(shape)
    for t in range(1, 6):
        g = torch.randn(shape, generator=gen, dtype=torch.float64) * 10.0 ** (t - 3)
        param.grad = g.clone()
        ref.step()
        p = af.adafactor_step(p, g.numpy().ravel(), st, shape, lr=lr, t=t, wd=0.1)
        np.testing.assert_allclose(p, param.detach().numpy().ravel(), rtol=1e-10, atol=1e-12)   # float64 rounding of the two orders
        s = ref.state[param]
        for k, v in st.items():
            np.testing.assert_allclose(v.ravel(), s[k].numpy().ravel(), rtol=1e-12, atol=0)


# ---- the switch ----------------------------------------------------------------------------------

def test_resolution(monkeypatch):
    monkeypatch.delenv("FRL_B200_ADAFACTOR", raising=False)
    assert resolve_adafactor() is False
    monkeypatch.setenv("FRL_B200_ADAFACTOR", "1")
    assert resolve_adafactor() is True
    assert resolve_adafactor(False) is False
    monkeypatch.setenv("FRL_B200_ADAFACTOR", "0")
    assert resolve_adafactor() is False and resolve_adafactor(True) is True
    for bad in ("yes", "2", "true"):
        monkeypatch.setenv("FRL_B200_ADAFACTOR", bad)
        with pytest.raises(ValueError, match="FRL_B200_ADAFACTOR"):
            resolve_adafactor()


def test_worker_args_field_order():
    f = SolverWorkerArgs._fields
    assert f[-2:] == ("ema_decay", "grad_accumulation")
    assert f.index("adafactor") == f.index("optimizer_state") + 1 == len(f) - 3
    assert SolverWorkerArgs._field_defaults["adafactor"] is False


def _problem(tmp_path, opts, **kw):
    ns = synthetic.api_namespace("frl_b200")
    problem = synthetic.make_toy_problem(ns, str(tmp_path), n_train=8, n_test=0)
    return problem, ns.types.RunOpts(optim=opts, batchSize=4, nEpochs=1, singleThreaded=True, **kw)


@pytest.mark.parametrize("algo,amsgrad,la,st", [
    (OptAlgorithm.SGD, False, LayerAdaptation.NONE, OptimizerState.FP32),
    (OptAlgorithm.RMSPROP, False, LayerAdaptation.NONE, OptimizerState.FP32),
    (OptAlgorithm.ADAM, True, LayerAdaptation.NONE, OptimizerState.FP32),
    (OptAlgorithm.SGD, False, LayerAdaptation.LARS, OptimizerState.FP32),
    (OptAlgorithm.ADAM, False, LayerAdaptation.LAMB, OptimizerState.FP32),
    (OptAlgorithm.ADAM, False, LayerAdaptation.NONE, OptimizerState.Q8)])
def test_refused_combinations_name_the_values(tmp_path, algo, amsgrad, la, st):
    opts = OptimOpts(algo=algo, amsgrad=amsgrad)
    with pytest.raises(ValueError, match="adafactor") as e:
        fused_optim.check_adafactor(opts, la, st, True)
    assert algo.value in str(e.value) and la.value in str(e.value) and st.value in str(e.value)
    assert ("amsgrad" in str(e.value).split("(")[0]) == amsgrad
    fused_optim.check_adafactor(opts, la, st, False)
    problem, run_opts = _problem(tmp_path, opts)
    with pytest.raises(ValueError, match="adafactor"):          # before any rank or device is touched
        next(Solver.solve(run_opts, problem, group_name=None, init_method="", layer_adaptation=la,
                          optimizer_state=st, adafactor=True))


def test_eval_ignores_the_option(tmp_path, monkeypatch):
    monkeypatch.setenv("FRL_B200_ADAFACTOR", "bogus")
    problem, run_opts = _problem(tmp_path, OptimOpts(algo=OptAlgorithm.SGD), mode=Mode.EVAL, cpuonly=True)
    with pytest.raises(RuntimeError, match="H100"):              # got past the option to the device check
        next(Solver.solve(run_opts, problem, group_name=None, init_method="", adafactor=True))


def test_built_optimizer_and_state_layout(double):
    arena, opt = _make(_net())
    assert type(opt) is fused_optim.FusedAdafactor and opt.needs_whole_tensors
    assert type(fused_optim.create_fused_optimizer(arena, _opts())) is fused_optim.FusedAdam
    assert set(opt.hyper) - {"params"} == set(torch.optim.Adafactor([nn.Parameter(torch.zeros(1))]).defaults)
    assert opt.hyper["eps"] == (None, 1e-3) and opt.hyper["beta2_decay"] == -0.8 and opt.hyper["d"] == 1.0
    assert opt.hyper["weight_decay"] == 1e-2 and opt.hyper["lr"] == 0.01
    want = sum(s.shape[0] + s.shape[1] if len(s.shape) == 2 else s.numel for s in arena.slots)
    assert opt.state_bytes == 4 * want and opt.fp32_state_bytes == 8 * arena.numel
    assert fused_optim.adafactor_shape((8, 4, 3, 3)) == (32, 3, 3)
    assert fused_optim.adafactor_shape(()) == (1, 0, 1) and fused_optim.adafactor_shape((5,)) == (1, 0, 5)


def _oracle_steps(ref, xs, lr=0.01, wd=1e-2):
    st, t = {}, 0
    for t, x in enumerate(xs, 1):
        for p in ref.parameters():
            p.grad = None
        ref(x).square().mean().backward()
        with torch.no_grad():
            for p in ref.parameters():
                s = st.setdefault(id(p), af.zero_state(p.shape))
                w = af.adafactor_step(p.detach().numpy().ravel(), p.grad.float().numpy().ravel(), s, p.shape, lr=lr,
                                      t=t, wd=wd)
                p.copy_(torch.from_numpy(w).float().view(p.shape))
                for k in s:                                     # the state is kept in fp32
                    s[k] = s[k].astype(np.float32).astype(np.float64)
    return st


def test_pipeline_launches_one_table_update_and_follows_the_restatement(double):
    net, ref = _net(1), _net(1)
    arena, opt = _make(net)
    pipe = grad_sync.GradBucketPipeline(arena, opt, eager_update=True)
    assert not pipe.eager and pipe.has_tail and pipe.nvls is None and not pipe.fused_dw_update
    xs = [torch.randn(16, 7) for _ in range(3)]
    for x in xs:
        double.calls.clear()
        pipe.begin_step(); net(x).square().mean().backward(); pipe.finish_step()
        assert double.calls == [("adafactor_mt", len(arena.slots))]
    st = _oracle_steps(ref, xs)
    for a, b in zip(net.parameters(), ref.parameters()):
        assert torch.equal(a, b)
        views = opt._slot_state(arena.slot_of(a))
        for k, v in st[id(b)].items():
            assert np.array_equal(views[k].numpy().ravel(), v.astype(np.float32).ravel())


def test_state_dict_is_torch_format_in_both_directions_and_resume_is_exact(double):
    net = _net(2)
    arena, opt = _make(net)
    pipe = grad_sync.GradBucketPipeline(arena, opt)
    x = torch.randn(16, 7)
    for _ in range(3):
        pipe.begin_step(); net(x).square().mean().backward(); pipe.finish_step()
    sd = opt.state_dict()
    stock = torch.optim.Adafactor(_net(2).parameters(), lr=0.01, weight_decay=1e-2)
    y = torch.randn(16, 7)
    m = _net(2)
    m(y).square().mean().backward()
    stock2 = torch.optim.Adafactor(m.parameters(), lr=0.01, weight_decay=1e-2)
    stock2.step()
    torch_sd = stock2.state_dict()
    for i, p in enumerate(net.parameters()):
        e, te = sd["state"][i], torch_sd["state"][i]
        assert set(e) == set(te)
        for k in e:
            assert e[k].shape == te[k].shape and e[k].dtype == te[k].dtype, (i, k)
        assert e["step"].dim() == 0 and float(e["step"]) == 3.0
    assert sd["param_groups"][0].keys() == torch_sd["param_groups"][0].keys()
    stock.load_state_dict(sd)
    # resume: a second optimizer loaded from the state dict continues bit for bit
    net2 = _net(2)
    with torch.no_grad():
        for a, b in zip(net2.parameters(), net.parameters()):
            a.copy_(b)
    arena2, opt2 = _make(net2)
    opt2.load_state_dict(sd)
    assert opt2._steps == 3 and torch.equal(opt2.state_buf, opt.state_buf)
    pipe2 = grad_sync.GradBucketPipeline(arena2, opt2)
    for p_, mm in ((pipe, net), (pipe2, net2)):
        p_.begin_step(); mm(x).square().mean().backward(); p_.finish_step()
    for a, b in zip(net.parameters(), net2.parameters()):
        assert torch.equal(a, b)
    # torch.optim.Adafactor -> fused
    arena3, opt3 = _make(_net(5))
    opt3.load_state_dict(torch_sd)
    assert opt3._steps == 1
    for i, s in enumerate(sorted(arena3.slots, key=lambda s: s.index)):
        for k, v in opt3._slot_state(s).items():
            assert torch.equal(v, torch_sd["state"][i][k])
    adam = torch.optim.Adam(m.parameters(), lr=0.01)
    adam.step()
    with pytest.raises(ValueError, match="exp_avg"):
        opt3.load_state_dict(adam.state_dict())


def test_unused_parameter_and_its_state_stay_untouched(double):
    net = _net(3)
    arena, opt = _make(net)
    pipe = grad_sync.GradBucketPipeline(arena, opt)
    x = torch.randn(8, 7)
    pipe.begin_step(); net(x).square().mean().backward(); pipe.finish_step()
    before = {s.index: {k: v.clone() for k, v in opt._slot_state(s).items()} for s in arena.slots}
    w = [p.detach().clone() for p in net.parameters()]
    pipe.begin_step(); net[0](x).square().mean().backward(); pipe.finish_step()      # only layer 0
    assert not torch.equal(net[0].weight.detach(), w[0])
    for a, b in zip(list(net.parameters())[2:], w[2:]):
        assert torch.equal(a.detach(), b)
    for p in list(net.parameters())[2:]:
        s = arena.slot_of(p)
        for k, v in opt._slot_state(s).items():
            assert torch.equal(v, before[s.index][k]), (s.index, k)
    for k, v in opt._slot_state(arena.slot_of(net[0].weight)).items():
        assert not torch.equal(v, before[arena.slot_of(net[0].weight).index][k]), k
    assert ("adafactor_mt", 2) in double.calls


def test_refuses_partial_tensors_and_the_flat_launchers(double):
    arena, opt = _make(_net())
    s = arena.slots[0]
    with pytest.raises(ValueError, match="whole tensors"):
        opt.apply_range(s.offset, s.end - 1)
    for call in (lambda: opt._launch(0, 8, 1.0, None), lambda: opt._launch_mt(None, 1.0),
                 lambda: opt._launch_nvls(0, 8, 1.0)):
        with pytest.raises(RuntimeError):
            call()


def test_plan_covers_every_element_once():
    shape = torch.tensor([fused_optim.adafactor_shape(s) for s in SHAPES + ((300, 2100),)], dtype=torch.int64)
    work, seg_info = _native.adafactor_plan(shape)
    assert seg_info[0, 0] == 0 and seg_info[-1, 1] == work.shape[0]
    assert torch.equal(seg_info[1:, 0], seg_info[:-1, 1])
    for i, (b, r, c) in enumerate(shape.tolist()):
        rows = work[seg_info[i, 0]:seg_info[i, 1]]
        assert (rows[:, 0] == i).all()
        if r:
            assert rows.shape[0] == b * -(-r // 64) * -(-c // 1024)
        else:
            assert rows[:, 2].tolist() == list(range(0, c, 16 * 1024))
    assert _native.adafactor_scratch_bytes(shape) > 0
    with pytest.raises(_native.NativeLibraryError):
        _native.adafactor_plan(torch.tensor([[1, 2, 0]], dtype=torch.int64))


def test_kernel_entry_point_rejects_bad_arguments_before_any_launch():
    lib = _native.lib()
    ok = 1 << 20                           # 16-byte aligned, never dereferenced: every call below fails a check
    before = lib.frl_launch_count()

    def call(**kw):
        a = dict(p=ok, st=ok, segs=ok, ns=2, shape=ok, off=ok, fl=ok, work=ok, nw=4, info=ok, scratch=ok, lr=0.01,
                 b2=-0.8, e1=EPS1, e2=1e-3, d=1.0, wd=0.0, step=1)
        a.update(kw)
        return lib.frl_adafactor_mt(a["p"], a["st"], None, a["segs"], a["ns"], a["shape"], a["off"], a["fl"],
                                    a["work"], a["nw"], a["info"], a["scratch"], a["lr"], a["b2"], a["e1"], a["e2"],
                                    a["d"], a["wd"], a["step"], 1.0, None, None, None)

    bad = [call(p=None), call(st=None), call(segs=None), call(shape=None), call(off=None), call(fl=None),
           call(work=None), call(info=None), call(scratch=None), call(scratch=ok + 8), call(step=0), call(lr=-1.0),
           call(b2=0.5), call(d=0.5), call(e2=-1.0), call(wd=-1.0), call(nw=-1), call(nw=4, ns=0)]
    assert all(rc < 0 for rc in bad), bad
    assert lib.frl_launch_count() == before
    assert call(nw=0, ns=0) == 0                                 # nothing to do, nothing launched


# ---- world_size 2 over gloo ----------------------------------------------------------------------

def _rank_main(rank, world, port, clip, out_dir):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    d = AdafactorKernelDouble()
    fused_optim.KERNELS = d
    grad_sync.KERNELS = d
    net = _net(10 + rank)
    arena, opt = _make(net)
    pipe = grad_sync.GradBucketPipeline(arena, opt, world_size=world, clip_norm=clip,
                                        bucket_cap_mb=0.001, first_bucket_mb=0.0005,
                                        eager_update=True, nvls_link=object())
    # whole-tensor updates: no eager per-bucket update, no fused NVLS step, no tail split
    assert not pipe.eager and pipe.nvls is None and not pipe._row_split and len(pipe.buckets) > 1
    pipe.broadcast_parameters(src=0)
    g = torch.Generator().manual_seed(99)
    for _ in range(3):
        x = torch.randn(8 * world, 7, generator=g)
        d.calls.clear()
        pipe.begin_step()
        net(x[rank::world]).square().mean().backward()
        pipe.finish_step()
        assert [c for c in d.calls if c[0] != "sumsq"] == [("adafactor_mt", len(arena.slots))]
    torch.save([p.detach().clone() for p in net.parameters()], os.path.join(out_dir, f"r{rank}.pt"))
    dist.destroy_process_group()


def _single_rank(world, clip):
    d = AdafactorKernelDouble()
    net = _net(10)
    saved = fused_optim.KERNELS, grad_sync.KERNELS
    fused_optim.KERNELS = grad_sync.KERNELS = d
    try:
        arena, opt = _make(net)
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
    world = 2
    port = 35500 + (os.getpid() % 2000)
    mp.spawn(_rank_main, args=(world, port, clip, str(tmp_path)), nprocs=world, join=True)
    r0, r1 = torch.load(tmp_path / "r0.pt"), torch.load(tmp_path / "r1.pt")
    for a, b in zip(r0, r1):
        assert torch.equal(a, b)
    for a, b in zip(r0, _single_rank(world, clip)):
        np.testing.assert_allclose(a.numpy(), b.numpy(), rtol=1e-5, atol=1e-6)


def test_zero_element_tensors_plan_no_work_and_keep_torch_state_shapes():
    assert fused_optim.adafactor_kernel_shape((0, 7)) == (1, 0, 0)
    assert fused_optim.adafactor_kernel_shape((3, 0, 2)) == (1, 0, 0)
    assert fused_optim.adafactor_kernel_shape((0,)) == (1, 0, 0)
    assert fused_optim.adafactor_state_elems((0, 7)) == 7 and fused_optim.adafactor_state_elems((0,)) == 0
    shape = torch.tensor([(1, 0, 0), (1, 4, 5), (1, 0, 0)], dtype=torch.int64)
    work, seg_info = _native.adafactor_plan(shape)
    assert work.shape[0] == 1 and seg_info[0, 0] == seg_info[0, 1] == 0 and seg_info[2, 0] == seg_info[2, 1] == 1
