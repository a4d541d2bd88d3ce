"""8-bit block-wise Adam state (K2-q8) on the host: the tables and the round trip of the format, the
enum and its switches, the refused combinations, the pipeline's launch sequence, torch-format state
in both directions, unused parameters, argument checks of the C entry points, and two ranks over
gloo against one rank at the global batch, with the kernels replaced by a CPU double."""
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
from frl_b200.solver import Solver, resolve_optimizer_state
from frl_b200.types import LayerAdaptation, OptAlgorithm, OptimizerState, OptimOpts
import adam8_oracle as q8
from adam8_oracle import Adam8KernelDouble

OS = OptimizerState
KW = dict(beta1=0.9, beta2=0.999, eps=1e-8, wd=1e-2)


@pytest.fixture()
def double(monkeypatch):
    d = Adam8KernelDouble()
    monkeypatch.setattr(fused_optim, "KERNELS", d)
    monkeypatch.setattr(grad_sync, "KERNELS", d)
    return d


def _net(seed=0):
    torch.manual_seed(seed)
    # 300 x 7 weight: two blocks, the second one short; 5-element bias: one short block
    return nn.Sequential(nn.Linear(7, 300), nn.ReLU(), nn.Linear(300, 5), nn.ReLU(), nn.Linear(5, 2))


def _opts(**kw):
    return OptimOpts(algo=OptAlgorithm.ADAM, lr=0.01, weightDecay=1e-2, **kw)


def _make(net):
    arena = ParamArena(net.parameters(), device="cpu")
    return arena, fused_optim.create_fused_optimizer(arena, _opts(), optimizer_state=OS.Q8)


# ---- the format ----------------------------------------------------------------------------------

def test_tables_are_sorted_hold_zero_and_one_and_agree_everywhere():
    mag7, mag8 = fused_optim.q8_tables()
    assert mag7.dtype == mag8.dtype == np.float32 and len(mag7) == 128 and len(mag8) == 256
    for t in (mag7, mag8):
        assert (np.diff(t) > 0).all() and t[0] == 0.0 and t[-1] == 1.0
    assert np.array_equal(mag7, q8.MAG7) and np.array_equal(mag8, q8.MAG8)
    d7, d8 = _native.q8_device_tables()            # the tables compiled into the library
    assert np.array_equal(d7.numpy(), mag7) and np.array_equal(d8.numpy(), mag8)
    assert fused_optim.Q8_BLOCK == _native.Q8_BLOCK == q8.BLOCK == 256


@pytest.mark.parametrize("signed", [True, False])
def test_decode_then_encode_returns_the_same_bytes(signed):
    rs = np.random.RandomState(0)
    cases = [rs.randn(1000).astype(np.float32) * 1e-3,
             (rs.randn(777) * np.exp(rs.randn(777) * 8)).astype(np.float32),
             np.zeros(300, np.float32), np.array([3.5], np.float32), np.array([-2.0], np.float32),
             np.array([-0.0, 0.0, -0.0], np.float32), np.array([0.0, 1e-40, -1e-38], np.float32)]
    for x in cases:
        x = x if signed else np.abs(x)
        c, a = q8.encode(x, signed)
        y = q8.decode(c, a, signed)
        c2, a2 = q8.encode(y, signed)
        assert np.array_equal(c, c2) and np.array_equal(a.view(np.uint32), a2.view(np.uint32))
        assert np.array_equal(q8.decode(c2, a2, signed).view(np.uint32), y.view(np.uint32))
    # the element that sets the absmax encodes exactly; a zero block decodes to zeros; -0.0 keeps its sign
    c, a = q8.encode(np.array([0.25, -1.0, 0.5], np.float32), True)
    assert q8.decode(c, a, True)[1] == -1.0 and a[0] == 1.0
    c, a = q8.encode(np.array([-0.0, 0.0], np.float32), True)
    assert a[0] == 0 and list(c) == [0x80, 0] and np.signbit(q8.decode(c, a, True)[0])


def test_nearest_entry_ties_go_to_the_smaller_index_and_nan_propagates_to_absmax():
    t = q8.MAG8
    mid = np.float32((np.float64(t[10]) + np.float64(t[11])) / 2)
    if np.float64(mid) == (np.float64(t[10]) + np.float64(t[11])) / 2:
        assert q8.nearest(t, mid) == 10
    assert q8.nearest(t, np.nextafter(t[10], np.float32(1))) == 10
    assert q8.nearest(t, np.float32(np.nan)) == 0
    _, a = q8.encode(np.array([1.0, np.nan, 2.0], np.float32), True)
    assert np.isnan(a[0])


# ---- options -------------------------------------------------------------------------------------

def test_enum_values_and_resolution(monkeypatch):
    assert [e.value for e in OS] == ["fp32", "8bit"]
    monkeypatch.delenv("FRL_B200_OPTIMIZER_STATE", raising=False)
    assert resolve_optimizer_state() is OS.FP32
    monkeypatch.setenv("FRL_B200_OPTIMIZER_STATE", "8BIT")
    assert resolve_optimizer_state() is OS.Q8
    assert resolve_optimizer_state(OS.FP32) is OS.FP32
    assert resolve_optimizer_state("8bit") is OS.Q8
    monkeypatch.setenv("FRL_B200_OPTIMIZER_STATE", "4bit")
    with pytest.raises(ValueError):
        resolve_optimizer_state()


@pytest.mark.parametrize("algo,amsgrad,la", [
    (OptAlgorithm.SGD, False, LayerAdaptation.NONE), (OptAlgorithm.RMSPROP, False, LayerAdaptation.NONE),
    (OptAlgorithm.ADAM, True, LayerAdaptation.NONE), (OptAlgorithm.ADAM, False, LayerAdaptation.LAMB)])
def test_refused_combinations_name_the_values(tmp_path, algo, amsgrad, la):
    opts = OptimOpts(algo=algo, amsgrad=amsgrad)
    with pytest.raises(ValueError, match="8bit") as e:
        fused_optim.check_optimizer_state(opts, la, OS.Q8)
    assert algo.value in str(e.value) and la.value in str(e.value)
    ns = synthetic.api_namespace("frl_b200")
    problem = synthetic.make_toy_problem(ns, str(tmp_path), n_train=8, n_test=0)
    run_opts = ns.types.RunOpts(optim=opts, batchSize=4, nEpochs=1, singleThreaded=True)
    with pytest.raises(ValueError, match="8bit"):          # before any rank or device is touched
        next(Solver.solve(run_opts, problem, group_name=None, init_method="", layer_adaptation=la,
                          optimizer_state=OS.Q8))


def test_accepted_combination_builds_the_8bit_optimizer(double):
    arena, opt = _make(_net())
    assert type(opt) is fused_optim.FusedAdam8bit and opt.needs_whole_tensors
    assert type(fused_optim.create_fused_optimizer(arena, _opts())) is fused_optim.FusedAdam
    n_blocks = sum((s.numel + 255) // 256 for s in arena.slots)
    assert opt.q8_blocks == n_blocks and opt.state_bytes == 2 * arena.numel + 2 * 4 * n_blocks
    assert opt.fp32_state_bytes == 8 * arena.numel and not opt._vec
    bases, total = fused_optim.q8_block_bases(arena.slots)
    assert total == n_blocks and [bases[s.index] for s in arena.slots] == \
        list(np.cumsum([0] + [(s.numel + 255) // 256 for s in arena.slots])[:-1])


# ---- the pipeline --------------------------------------------------------------------------------

def _oracle_steps(ref, xs, lr=0.01):
    """The restatement applied per parameter to stock autograd gradients."""
    st = {}
    for t, x in enumerate(xs, 1):
        for p in ref.parameters():
            p.grad = None
        ref(x).square().mean().backward()
        with torch.no_grad():
            for p in ref.parameters():
                n = p.numel()
                nb = (n + 255) // 256
                mq, ma, vq, va = st.get(id(p), (np.zeros(n, np.uint8), np.zeros(nb, np.float32),
                                                np.zeros(n, np.uint8), np.zeros(nb, np.float32)))
                w, (mq, ma), (vq, va), _, _ = q8.adam8_step(p.detach().numpy().ravel().copy(),
                                                            p.grad.numpy().ravel(), mq, ma, vq, va, lr=lr,
                                                            step=t, **KW)
                st[id(p)] = (mq, ma, vq, va)
                p.copy_(torch.from_numpy(w).view(p.shape))
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
        assert double.calls == [("adam8_mt", len(arena.slots))]
    st = _oracle_steps(ref, xs)
    for a, b in zip(net.parameters(), ref.parameters()):
        assert torch.equal(a, b)
        s = arena.slot_of(a)
        mq, ma, vq, va = st[id(b)]
        assert np.array_equal(opt.codes["exp_avg"][s.offset:s.end].numpy(), mq)
        assert np.array_equal(opt.codes["exp_avg_sq"][s.offset:s.end].numpy(), vq)
        b0 = opt._qbase[s.index]
        assert np.array_equal(opt.absmax["exp_avg"][b0:b0 + len(ma)].numpy(), ma)
        assert np.array_equal(opt.absmax["exp_avg_sq"][b0:b0 + len(va)].numpy(), va)
    assert not (opt.codes["exp_avg"][arena.slots[0].end:arena.slots[1].offset] != 0).any()     # padding


def test_state_dict_is_torch_adam_format_in_both_directions_and_resume_is_exact(double):
    net = _net(2)
    arena, opt = _make(net)
    pipe = grad_sync.GradBucketPipeline(arena, opt)
    x = torch.randn(16, 7)
    for _ in range(3):
        pipe.begin_step(); net(x).square().mean().backward(); pipe.finish_step()
    sd = opt.state_dict()
    assert not opt._vec and set(sd["state"][0]) == {"step", "exp_avg", "exp_avg_sq"}
    assert float(sd["state"][0]["step"]) == 3.0
    stock = torch.optim.Adam(_net(2).parameters(), lr=0.01)
    stock.load_state_dict(sd)                                   # loads into torch.optim.Adam
    for i, s in enumerate(sorted(arena.slots, key=lambda s: s.index)):
        want = q8.decode(opt.codes["exp_avg"][s.offset:s.end].numpy(),
                         opt.absmax["exp_avg"][opt._qbase[s.index]:].numpy(), True)
        assert np.array_equal(stock.state_dict()["state"][i]["exp_avg"].numpy().ravel(), want)
    # resume: a second optimizer loaded from the state dict continues bit for bit
    net2 = _net(2)
    with torch.no_grad():
        for a, b in zip(net2.parameters(), net.parameters()):
            a.copy_(b)
    arena2, opt2 = _make(net2)
    opt2.load_state_dict(sd)
    assert opt2._steps == 3 and not opt2._vec
    for n in ("exp_avg", "exp_avg_sq"):
        assert torch.equal(opt2.codes[n], opt.codes[n]) and torch.equal(opt2.absmax[n], opt.absmax[n])
    pipe2 = grad_sync.GradBucketPipeline(arena2, opt2)
    for p_, m in ((pipe, net), (pipe2, net2)):
        p_.begin_step(); m(x).square().mean().backward(); p_.finish_step()
    for a, b in zip(net.parameters(), net2.parameters()):
        assert torch.equal(a, b)
    # torch.optim.Adam -> 8-bit: the moments are encoded
    ref = _net(5)
    adam = torch.optim.Adam(ref.parameters(), lr=0.01)
    for _ in range(2):
        adam.zero_grad(); ref(x).square().mean().backward(); adam.step()
    arena3, opt3 = _make(_net(5))
    opt3.load_state_dict(adam.state_dict())
    assert opt3._steps == 2
    for i, s in enumerate(sorted(arena3.slots, key=lambda s: s.index)):
        c, a = q8.encode(adam.state_dict()["state"][i]["exp_avg_sq"].numpy(), False)
        assert np.array_equal(opt3.codes["exp_avg_sq"][s.offset:s.end].numpy(), c)
    amsgrad = torch.optim.Adam(_net(5).parameters(), lr=0.01, amsgrad=True).state_dict()
    with pytest.raises(ValueError, match="amsgrad"):
        opt3.load_state_dict(amsgrad)


def test_unused_parameter_and_its_state_stay_untouched(double):
    net = _net(3)
    arena, opt = _make(net)
    pipe = grad_sync.GradBucketPipeline(arena, opt)
    x = torch.randn(8, 7)
    pipe.begin_step(); net(x).square().mean().backward(); pipe.finish_step()
    before = {k: (opt.codes[k].clone(), opt.absmax[k].clone()) for k in opt.codes}
    w = [p.detach().clone() for p in net.parameters()]
    pipe.begin_step(); net[0](x).square().mean().backward(); pipe.finish_step()      # only layer 0
    s0, s2 = arena.slot_of(net[0].bias), arena.slot_of(net[2].weight)
    assert not torch.equal(net[0].weight.detach(), w[0])
    for a, b in zip(list(net.parameters())[2:], w[2:]):
        assert torch.equal(a.detach(), b)
    for k, (c, a) in before.items():
        assert torch.equal(opt.codes[k][s2.offset:], c[s2.offset:])
        assert torch.equal(opt.absmax[k][opt._qbase[s2.index]:], a[opt._qbase[s2.index]:])
        assert not torch.equal(opt.codes[k][:s0.end], c[:s0.end])
    assert ("adam8_mt", 2) in double.calls


def test_refuses_partial_tensors_and_the_flat_launchers(double):
    arena, opt = _make(_net())
    s = arena.slots[0]
    with pytest.raises(ValueError, match="whole tensors"):
        opt.apply_range(s.offset, s.end - 1)
    for call in (lambda: opt._launch(0, 8, 1.0, None), lambda: opt._launch_mt(None, 1.0),
                 lambda: opt._launch_nvls(0, 8, 1.0)):
        with pytest.raises(RuntimeError):
            call()


def test_kernel_entry_points_reject_bad_arguments_before_any_launch():
    lib = _native.lib()
    ok = 1 << 20                           # 16-byte aligned, never dereferenced: every call below fails a check
    before = lib.frl_launch_count()

    def adam8(**kw):
        a = dict(p=ok, mq=ok, vq=ok, ma=ok, va=ok, lp=None, segs=ok, nt=4, ns=2, qb=ok, fl=ok, step=1)
        a.update(kw)
        return lib.frl_adam8_mt(a["p"], a["mq"], a["vq"], a["ma"], a["va"], a["lp"], a["segs"], ok, ok, a["nt"],
                                a["ns"], a["qb"], a["fl"], 0.1, 0.9, 0.999, 1e-8, 0.0, a["step"], 1.0, None, None,
                                None)

    def conv(fn, **kw):
        a = dict(x=ok, q=ok, am=ok, state=0, segs=ok, nt=4, ns=2, qb=ok)
        a.update(kw)
        return fn(a["x"], a["q"], a["am"], a["state"], a["segs"], ok, ok, a["nt"], a["ns"], a["qb"], None)

    bad = [adam8(p=None), adam8(mq=None), adam8(va=None), adam8(segs=None), adam8(qb=None), adam8(fl=None),
           adam8(step=0), adam8(p=ok + 4), adam8(mq=ok + 4), adam8(lp=ok + 2), adam8(nt=-1), adam8(nt=4, ns=0)]
    for fn in (lib.frl_q8_encode_mt, lib.frl_q8_decode_mt):
        bad += [conv(fn, x=None), conv(fn, q=None), conv(fn, am=None), conv(fn, qb=None), conv(fn, state=2),
                conv(fn, x=ok + 4), conv(fn, nt=-1)]
    assert all(rc < 0 for rc in bad), bad
    assert lib.frl_launch_count() == before
    assert adam8(nt=0, ns=0) == 0                                # nothing to do, nothing launched


# ---- world_size 2 over gloo ----------------------------------------------------------------------

def _rank_main(rank, world, port, clip, out_dir):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    d = Adam8KernelDouble()
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
        assert [c for c in d.calls if c[0] != "sumsq"] == [("adam8_mt", len(arena.slots))]
    torch.save([p.detach().clone() for p in net.parameters()], os.path.join(out_dir, f"r{rank}.pt"))
    dist.destroy_process_group()


def _single_rank(world, clip):
    d = Adam8KernelDouble()
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
    port = 33500 + (os.getpid() % 2000)
    mp.spawn(_rank_main, args=(world, port, clip, str(tmp_path)), nprocs=world, join=True)
    r0, r1 = torch.load(tmp_path / "r0.pt"), torch.load(tmp_path / "r1.pt")
    for a, b in zip(r0, r1):
        assert torch.equal(a, b)
    for a, b in zip(r0, _single_rank(world, clip)):
        np.testing.assert_allclose(a.numpy(), b.numpy(), rtol=1e-5, atol=1e-6)
