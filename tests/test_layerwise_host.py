"""Layer-wise adaptation (LARS, LAMB) on the host: the enum and its switches, the combinations that
are refused, which tensors adapt, torch-format state, the restatement's properties, and the
pipeline's whole-tensor path (1 and 2 ranks over gloo) with the kernels replaced by a CPU double."""
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn as nn

import frl_b200  # noqa: F401
from frl_b200 import fused_optim, grad_sync, synthetic
from frl_b200.arena import ParamArena
from frl_b200.multi_tensor import GradSegTable
from frl_b200.solver import Solver, resolve_layer_adaptation
from frl_b200.types import LayerAdaptation, OptAlgorithm, OptimOpts
from layerwise_oracle import LayerwiseKernelDouble, LayerwiseTorch, lamb_step, lars_step

LA = LayerAdaptation


@pytest.fixture()
def double(monkeypatch):
    d = LayerwiseKernelDouble()
    monkeypatch.setattr(fused_optim, "KERNELS", d)
    monkeypatch.setattr(grad_sync, "KERNELS", d)
    return d


def _net(seed=0):
    torch.manual_seed(seed)
    return nn.Sequential(nn.Linear(7, 5), nn.ReLU(), nn.Linear(5, 3), nn.ReLU(), nn.Linear(3, 2))


def _opts(mode, **kw):
    if mode == "lars":
        return OptimOpts(algo=OptAlgorithm.SGD, lr=0.05, weightDecay=1e-2, **kw)
    return OptimOpts(algo=OptAlgorithm.ADAM, lr=0.01, weightDecay=1e-2, **kw)


def _torch_oracle(params, mode):
    o = _opts(mode)
    return LayerwiseTorch(params, mode, lr=o.lr, momentum=o.momentum, weight_decay=o.weightDecay, eps=o.epsilon)


def test_enum_values_and_resolution(monkeypatch):
    assert [e.value for e in LA] == ["none", "lars", "lamb"]
    monkeypatch.delenv("FRL_B200_LAYER_ADAPTATION", raising=False)
    assert resolve_layer_adaptation() is LA.NONE
    monkeypatch.setenv("FRL_B200_LAYER_ADAPTATION", "LAMB")
    assert resolve_layer_adaptation() is LA.LAMB
    assert resolve_layer_adaptation(LA.LARS) is LA.LARS
    monkeypatch.setenv("FRL_B200_LAYER_ADAPTATION", "adamw")
    with pytest.raises(ValueError):
        resolve_layer_adaptation()


@pytest.mark.parametrize("algo,amsgrad,la", [
    (OptAlgorithm.ADAM, False, LA.LARS), (OptAlgorithm.RMSPROP, False, LA.LARS),
    (OptAlgorithm.SGD, False, LA.LAMB), (OptAlgorithm.RMSPROP, False, LA.LAMB),
    (OptAlgorithm.ADAM, True, LA.LAMB)])
def test_refused_combinations_name_both_values(tmp_path, algo, amsgrad, la):
    opts = OptimOpts(algo=algo, amsgrad=amsgrad)
    with pytest.raises(ValueError, match=la.value) as e:
        fused_optim.check_layer_adaptation(opts, la)
    assert algo.value in str(e.value)
    ns = synthetic.api_namespace("frl_b200")
    problem = synthetic.make_toy_problem(ns, str(tmp_path), n_train=8, n_test=0)
    run_opts = ns.types.RunOpts(optim=opts, batchSize=4, nEpochs=1, singleThreaded=True)
    with pytest.raises(ValueError, match=la.value):          # before any rank or device is touched
        next(Solver.solve(run_opts, problem, group_name=None, init_method="", layer_adaptation=la))


def test_accepted_combinations_build_the_layerwise_optimizers(double):
    arena = ParamArena(_net().parameters(), device="cpu")
    assert type(fused_optim.create_fused_optimizer(arena, _opts("lars"), LA.LARS)) is fused_optim.FusedLars
    lamb = fused_optim.create_fused_optimizer(arena, _opts("lamb"), LA.LAMB)
    assert type(lamb) is fused_optim.FusedLamb and lamb.needs_whole_tensors
    plain = fused_optim.create_fused_optimizer(arena, _opts("lamb"))
    assert type(plain) is fused_optim.FusedAdam and not plain.needs_whole_tensors


def _flags(double, model_params, crit_params=()):
    arena = ParamArena(model_params, crit_params, device="cpu")
    opt = fused_optim.create_fused_optimizer(arena, _opts("lars"), LA.LARS)
    table = GradSegTable(arena.slots, arena.device)
    flags = opt._lw_buffers(table)[0].tolist()
    return {id(s.param): f for s, f in zip(table.slots, flags)}


def test_which_tensors_adapt(double, tmp_path):
    ns = synthetic.api_namespace("frl_b200")
    # headline MLP structure (narrow): trunk and head weights adapt, biases and criterion
    # parameters do not; only model parameters take the clip coefficient
    mlp = synthetic.make_mlp_problem(ns, str(tmp_path), n_train=4, width=32, n_classes=10, reg_dim=4)
    model = mlp.get_model()
    log_var = nn.Parameter(torch.zeros(2))
    fl = _flags(double, model.parameters(), [log_var])
    linears = [m for m in model.modules() if isinstance(m, nn.Linear)]
    assert len(linears) == 5
    for m in linears:
        assert fl[id(m.weight)] == 3 and fl[id(m.bias)] == 2
    assert fl[id(log_var)] == 0
    # ResNet: convolutions adapt, BatchNorm does not
    net = synthetic.make_resnet_problem(ns, str(tmp_path), image=32, n_train=2).get_model()
    fl = _flags(double, net.parameters())
    convs = [m for m in net.modules() if isinstance(m, nn.Conv2d)]
    bns = [m for m in net.modules() if isinstance(m, nn.BatchNorm2d)]
    assert convs and bns
    assert all(fl[id(m.weight)] & 1 for m in convs)
    assert not any(fl[id(m.weight)] & 1 or fl[id(m.bias)] & 1 for m in bns)
    # text: the embedding adapts
    for name in ("a.txt", "b.txt"):
        synthetic.write_text_corpus(str(tmp_path / name), 16, 0)
    text = synthetic.make_text_problem(ns, str(tmp_path), str(tmp_path / "a.txt"), str(tmp_path / "b.txt"))
    tm = text.get_model()
    embs = [m for m in tm.modules() if isinstance(m, nn.Embedding)]
    assert len(embs) == 1 and _flags(double, tm.parameters())[id(embs[0].weight)] & 1


@pytest.mark.parametrize("mode", ["lars", "lamb"])
def test_pipeline_follows_the_torch_oracle_and_state_is_torch_format(double, mode):
    net, ref = _net(1), _net(1)
    arena = ParamArena(net.parameters(), device="cpu")
    opt = fused_optim.create_fused_optimizer(arena, _opts(mode), LA(mode))
    pipe = grad_sync.GradBucketPipeline(arena, opt)
    assert not pipe.eager and pipe.has_tail
    ref_opt = _torch_oracle(ref.parameters(), mode)
    x = torch.randn(16, 7)
    for _ in range(4):
        pipe.begin_step(); net(x).square().mean().backward(); pipe.finish_step()
        ref_opt.zero_grad(); ref(x).square().mean().backward(); ref_opt.step()
    for a, b in zip(net.parameters(), ref.parameters()):
        np.testing.assert_allclose(a.detach().numpy(), b.detach().numpy(), rtol=1e-5, atol=1e-7)
    assert ("%s_mt" % mode, len(arena.slots)) in double.calls
    # the state dict is torch.optim.SGD's / Adam's and loads there
    sd = opt.state_dict()
    stock = (torch.optim.SGD(_net(1).parameters(), lr=0.05, momentum=0.9) if mode == "lars"
             else torch.optim.Adam(_net(1).parameters(), lr=0.01))
    stock.load_state_dict(sd)
    names = ("momentum_buffer",) if mode == "lars" else ("exp_avg", "exp_avg_sq")
    for i, p in enumerate(ref.parameters()):
        for n in names:
            np.testing.assert_allclose(stock.state_dict()["state"][i][n].numpy(),
                                       ref_opt.state[p][n].numpy(), rtol=1e-5, atol=1e-8)
    # and a resumed optimizer continues the trajectory
    net2 = _net(1)
    with torch.no_grad():
        for a, b in zip(net2.parameters(), net.parameters()):
            a.copy_(b)
    arena2 = ParamArena(net2.parameters(), device="cpu")
    opt2 = fused_optim.create_fused_optimizer(arena2, _opts(mode), LA(mode))
    opt2.load_state_dict(sd)
    pipe2 = grad_sync.GradBucketPipeline(arena2, opt2)
    for p_, m in ((pipe, net), (pipe2, net2)):
        p_.begin_step(); m(x).square().mean().backward(); p_.finish_step()
    for a, b in zip(net.parameters(), net2.parameters()):
        assert torch.equal(a, b)


def test_adam_checkpoint_resumes_under_lamb(double):
    net = _net(4)
    stock = torch.optim.Adam(net.parameters(), lr=0.01, weight_decay=1e-2)
    x = torch.randn(8, 7)
    for _ in range(2):
        stock.zero_grad(); net(x).square().mean().backward(); stock.step()
    arena = ParamArena(net.parameters(), device="cpu")
    lamb = fused_optim.create_fused_optimizer(arena, _opts("lamb"), LA.LAMB)
    lamb.load_state_dict(stock.state_dict())
    assert lamb._steps == 2
    for i, s in enumerate(sorted(arena.slots, key=lambda s: s.index)):
        assert torch.equal(lamb._vec["exp_avg"][s.offset:s.end].view(s.shape), stock.state_dict()["state"][i]["exp_avg"])


@pytest.mark.parametrize("mode", ["lars", "lamb"])
def test_unused_parameter_and_its_state_stay_untouched(double, mode):
    net, ref = _net(3), _net(3)
    arena = ParamArena(net.parameters(), device="cpu")
    opt = fused_optim.create_fused_optimizer(arena, _opts(mode), LA(mode))
    pipe = grad_sync.GradBucketPipeline(arena, opt)
    ref_opt = _torch_oracle(ref.parameters(), mode)
    x = torch.randn(8, 7)
    pipe.begin_step(); net(x).square().mean().backward(); pipe.finish_step()
    ref_opt.zero_grad(); ref(x).square().mean().backward(); ref_opt.step()
    state_before = {k: v.clone() for k, v in opt._vec.items()}
    w2 = [p.detach().clone() for p in list(net.parameters())[2:]]
    pipe.begin_step(); net[0](x).square().mean().backward(); pipe.finish_step()      # only layer 0
    ref_opt.zero_grad(); ref[0](x).square().mean().backward(); ref_opt.step()
    for a, b in zip(net.parameters(), ref.parameters()):
        np.testing.assert_allclose(a.detach().numpy(), b.detach().numpy(), rtol=1e-5, atol=1e-7)
    for a, b in zip(list(net.parameters())[2:], w2):
        assert torch.equal(a.detach(), b)
    s = arena.slot_of(net[2].weight)
    for k, v in opt._vec.items():
        assert torch.equal(v[s.offset:], state_before[k][s.offset:])


def test_restatement_ratio_is_one_for_zero_weight_or_gradient_and_nan_propagates():
    rs = np.random.RandomState(0)
    w, g = rs.randn(6, 5).astype(np.float32), rs.randn(6, 5).astype(np.float32)
    z = np.zeros_like(w)
    assert lars_step(z, g, None, lr=0.1, mu=0.0, wd=0.1, adapted=True, first_step=True)[2] == 1.0
    assert lars_step(w, z, None, lr=0.1, mu=0.0, wd=0.1, adapted=True, first_step=True)[2] == 1.0
    kw = dict(lr=0.1, beta1=0.9, beta2=0.999, eps=1e-8, wd=0.1, step=1, adapted=True)
    assert lamb_step(z, g, z, z, **kw)[3] == 1.0
    assert lamb_step(w, z, z, z, **dict(kw, wd=0.0))[3] == 1.0          # u == 0
    assert lars_step(w, g, None, lr=0.1, mu=0.0, wd=0.1, adapted=True, first_step=True)[2] != 1.0
    for bad in (np.nan, np.inf):
        gb = g.copy()
        gb[1, 2] = bad
        assert not np.isfinite(lars_step(w, gb, None, lr=0.1, mu=0.9, wd=0.1, adapted=True,
                                         first_step=True)[0]).all()
        assert not np.isfinite(lamb_step(w, gb, z, z, **kw)[0]).all()


# ---- world_size 2 over gloo ---------------------------------------------------------------------

def _rank_main(rank, world, port, mode, clip, out_dir):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    d = LayerwiseKernelDouble()
    fused_optim.KERNELS = d
    grad_sync.KERNELS = d
    net = _net(10 + rank)
    arena = ParamArena(net.parameters(), device="cpu")
    opt = fused_optim.create_fused_optimizer(arena, _opts(mode), LA(mode))
    pipe = grad_sync.GradBucketPipeline(arena, opt, world_size=world, clip_norm=clip,
                                        bucket_cap_mb=0.0001, first_bucket_mb=0.00005,
                                        eager_update=True, nvls_link=object())
    # whole-tensor updates: no eager per-bucket update, no fused NVLS step, no tail split
    assert not pipe.eager and pipe.nvls is None and not pipe._row_split and len(pipe.buckets) > 1
    pipe.broadcast_parameters(src=0)
    g = torch.Generator().manual_seed(99)
    for _ in range(3):
        x = torch.randn(8 * world, 7, generator=g)
        pipe.begin_step()
        net(x[rank::world]).square().mean().backward()
        pipe.finish_step()
    torch.save([p.detach().clone() for p in net.parameters()], os.path.join(out_dir, f"r{rank}.pt"))
    dist.destroy_process_group()


@pytest.mark.parametrize("mode,clip", [("lars", 0.0), ("lamb", 0.0), ("lars", 0.01)])
def test_two_ranks_at_half_batch_equal_one_rank_at_full_batch(tmp_path, mode, clip):
    world = 2
    port = 31500 + (os.getpid() % 2000)
    mp.spawn(_rank_main, args=(world, port, mode, clip, str(tmp_path)), nprocs=world, join=True)
    r0, r1 = torch.load(tmp_path / "r0.pt"), torch.load(tmp_path / "r1.pt")
    for a, b in zip(r0, r1):
        assert torch.equal(a, b)
    ref = _net(10)
    ref_opt = _torch_oracle(ref.parameters(), mode)
    g = torch.Generator().manual_seed(99)
    for _ in range(3):
        x = torch.randn(8 * world, 7, generator=g)
        ref_opt.zero_grad()
        ref(x).square().mean().backward()
        if clip:
            torch.nn.utils.clip_grad_norm_(ref.parameters(), clip)
        ref_opt.step()
    for a, b in zip(r0, ref.parameters()):
        np.testing.assert_allclose(a.numpy(), b.detach().numpy(), rtol=2e-5, atol=1e-7)


def test_kernel_entry_points_reject_bad_arguments_before_any_launch():
    from frl_b200 import _native
    lib = _native.lib()
    ok = 1 << 20                           # 16-byte aligned, never dereferenced: every call below fails a check
    before = lib.frl_launch_count()

    def lars(**kw):
        a = dict(p=ok, buf=ok, lp=None, segs=ok, pre=ok, tseg=ok, nt=4, ns=2, fl=ok, r=ok, sc=ok, mu=0.9)
        a.update(kw)
        return lib.frl_lars_mt(a["p"], a["buf"], a["lp"], a["segs"], a["pre"], a["tseg"], a["nt"], a["ns"],
                               a["fl"], a["r"], a["sc"], 0.1, a["mu"], 0.0, 1.0, None, None, 1, None)

    def lamb(**kw):
        a = dict(p=ok, m=ok, v=ok, lp=None, segs=ok, fl=ok, r=ok, sc=ok, step=1)
        a.update(kw)
        return lib.frl_lamb_mt(a["p"], a["m"], a["v"], a["lp"], a["segs"], ok, ok, 4, 2, a["fl"], a["r"], a["sc"],
                               0.1, 0.9, 0.999, 1e-8, 0.0, a["step"], 1.0, None, None, None)

    bad = [lars(p=None), lars(segs=None), lars(fl=None), lars(r=None), lars(sc=None), lars(buf=None),
           lars(p=ok + 4), lars(buf=ok + 8), lars(lp=ok + 2), lars(sc=ok + 4), lars(nt=-1), lars(nt=4, ns=0),
           lamb(m=None), lamb(v=None), lamb(step=0), lamb(p=ok + 4), lamb(r=None), lamb(fl=None)]
    assert all(rc < 0 for rc in bad), bad
    assert lib.frl_launch_count() == before
    assert lars(buf=None, mu=0.0, nt=0, ns=0) == 0            # nothing to do, nothing launched
    assert _native.layerwise_scratch_bytes(5, 3) >= 5 * 8 + 3 * 4


def test_layerwise_optimizers_refuse_partial_tensors_and_the_flat_launchers(double):
    arena = ParamArena(_net().parameters(), device="cpu")
    for mode in ("lars", "lamb"):
        opt = fused_optim.create_fused_optimizer(arena, _opts(mode), LA(mode))
        s = arena.slots[0]
        with pytest.raises(ValueError, match="whole tensors"):
            opt.apply_range(s.offset, s.end - 1)
        for call in (lambda: opt._launch(0, 8, 1.0, None), lambda: opt._launch_mt(None, 1.0),
                     lambda: opt._launch_nvls(0, 8, 1.0)):
            with pytest.raises(RuntimeError):
                call()
