"""channels_last training, host side: the arena layout (``ParamArena.slot_view``), which gradients the
kernels read in place, contiguous state dicts and checkpoints with loads across layouts on a CPU
arena, the switch (``FRL_B200_CHANNELS_LAST``) and its refusals, the ``SolverWorkerArgs`` field
positions, and a numpy restatement of K5 into channels_last (``frl_preproc_affine_nhwc``)."""
import copy

import numpy as np
import pytest
import torch
import torch.nn as nn

import frl_b200  # noqa: F401
from frl_b200 import fused_optim, solver
from frl_b200.arena import ParamArena
from frl_b200.ema import WeightEMA
from frl_b200.multi_tensor import same_element_order
from frl_b200.solver import CHANNELS_LAST_ENV, SolverWorkerArgs, check_channels_last, resolve_channels_last

CL = torch.channels_last


def _net(seed=0):
    torch.manual_seed(seed)
    return nn.Sequential(nn.Conv2d(3, 8, 3), nn.BatchNorm2d(8), nn.Conv2d(8, 16, 1), nn.Conv2d(1, 4, 3),
                         nn.Conv2d(16, 6, (2, 5)), nn.Flatten(), nn.Linear(20, 7))


def _arena(net, channels_last):
    return ParamArena(net.parameters(), device=torch.device("cpu"), channels_last=channels_last)


# ---- layout ------------------------------------------------------------------------------------------

def test_slot_view_gives_4d_parameters_channels_last_strides():
    net = _net()
    values = [p.detach().clone() for p in net.parameters()]
    arena = _arena(net, True)
    base = arena.master.data_ptr()
    for s, p, v in zip(arena.slots, net.parameters(), values):
        assert p.data_ptr() == base + 4 * s.offset
        assert torch.equal(p.detach(), v)                     # same values, other element order
        if p.dim() == 4:
            assert s.memory_format is CL
            assert p.stride() == torch.empty(s.shape, memory_format=CL).stride()
            # the slice holds (O, kh, kw, I)
            assert torch.equal(arena.master[s.offset:s.end], v.permute(0, 2, 3, 1).reshape(-1))
        else:
            assert s.memory_format is torch.contiguous_format and p.is_contiguous()
            assert torch.equal(arena.master[s.offset:s.end], v.reshape(-1))
        assert ParamArena.slot_view(arena.grad, s).stride() == p.stride()
    assert arena.n_channels_last == 4


def test_switch_off_keeps_the_contiguous_layout():
    net_a, net_b = _net(), _net()
    a, b = _arena(net_a, False), ParamArena(net_b.parameters(), device=torch.device("cpu"))
    assert torch.equal(a.master, b.master) and a.n_channels_last == 0
    assert all(p.is_contiguous() for p in net_a.parameters())


def test_1x1_and_single_input_channel_weights_have_one_element_order():
    net = _net()
    arena = _arena(net, True)
    conv3, conv1x1, conv_i1, conv_rect = (arena.slot_of(m.weight) for m in (net[0], net[2], net[3], net[4]))
    for s in (conv1x1, conv_i1):
        # the same elements in the same order in both layouts: both gradients are read in place
        assert same_element_order(torch.empty(s.shape), s)
        assert same_element_order(torch.empty(s.shape, memory_format=CL), s)
        assert torch.equal(arena.master[s.offset:s.end], net[2 if s is conv1x1 else 3].weight.detach()
                           .contiguous().reshape(-1))
    for s in (conv3, conv_rect):
        assert same_element_order(torch.empty(s.shape, memory_format=CL), s)
        assert not same_element_order(torch.empty(s.shape), s)                 # NCHW dW: copied
        assert not same_element_order(torch.empty(s.shape, memory_format=CL).transpose(2, 3), s) \
            or s.shape[2] == s.shape[3]
    lin = arena.slot_of(net[6].weight)
    assert same_element_order(torch.empty(lin.shape), lin)
    assert not same_element_order(torch.empty(lin.shape[::-1]).t(), lin)
    nchw = _arena(_net(), False)
    s = nchw.slot_of(nchw.all_params[0])
    assert not same_element_order(torch.empty(s.shape, memory_format=CL), s)   # channels_last dW, NCHW slot


# ---- checkpoints ---------------------------------------------------------------------------------------

def _fill(arena, opt, names, seed):
    """The same logical state in any layout: every state vector set through slot views."""
    g = torch.Generator().manual_seed(seed)
    for name in names:
        vec = opt._state(name)
        for s in arena.slots:
            ParamArena.slot_view(vec, s).copy_(torch.randn(s.shape, generator=g))
    opt._steps = 3


def _all_contiguous(obj):
    if torch.is_tensor(obj):
        return obj.is_contiguous()
    if isinstance(obj, dict):
        return all(_all_contiguous(v) for v in obj.values())
    if isinstance(obj, (list, tuple)):
        return all(_all_contiguous(v) for v in obj)
    return True


def _same_sd(a, b):
    assert a["param_groups"] == b["param_groups"]
    assert a["state"].keys() == b["state"].keys()
    for k in a["state"]:
        for name, v in a["state"][k].items():
            w = b["state"][k][name]
            assert v.shape == w.shape and v.stride() == w.stride() and v.dtype == w.dtype
            assert torch.equal(v, w), (k, name)


@pytest.mark.parametrize("kind", ["sgd", "adam"])
def test_state_dicts_are_contiguous_and_load_across_layouts(kind):
    def make(cl):
        net = _net()
        arena = _arena(net, cl)
        if kind == "sgd":
            return net, arena, fused_optim.FusedSGD(arena, lr=0.1, momentum=0.9), ("momentum_buffer",), torch.optim.SGD
        return net, arena, fused_optim.FusedAdam(arena, lr=1e-3), ("exp_avg", "exp_avg_sq"), torch.optim.Adam

    net_c, ar_c, opt_c, names, stock = make(False)
    net_l, ar_l, opt_l, _, _ = make(True)
    _fill(ar_c, opt_c, names, 1)
    _fill(ar_l, opt_l, names, 1)
    sd_c, sd_l = opt_c.state_dict(), opt_l.state_dict()
    assert _all_contiguous(sd_l)
    _same_sd(sd_c, sd_l)                                     # the files are the same
    # NCHW -> NHWC and NHWC -> NCHW
    _, ar2, opt2, _, _ = make(True)
    opt2.load_state_dict(copy.deepcopy(sd_c))
    for n in names:
        assert torch.equal(opt2._state(n), opt_l._state(n))
    _, ar3, opt3, _, _ = make(False)
    opt3.load_state_dict(copy.deepcopy(sd_l))
    for n in names:
        assert torch.equal(opt3._state(n), opt_c._state(n))
    # to and from torch.optim
    params = [nn.Parameter(p.detach().clone()) for p in net_l.parameters()]
    t = stock(params, lr=0.1)
    t.load_state_dict(copy.deepcopy(sd_l))
    _, ar4, opt4, _, _ = make(True)
    opt4.load_state_dict(t.state_dict())
    for n in names:
        assert torch.equal(opt4._state(n), opt_l._state(n))


def test_exported_weights_and_ema_files_are_contiguous_and_load_across_layouts():
    net_c, net_l = _net(), _net()
    ar_c, ar_l = _arena(net_c, False), _arena(net_l, True)
    with ar_l.exported(cpu=True, module=net_l):
        sd_l = {k: v.clone() for k, v in net_l.state_dict().items()}
        assert all(p.is_contiguous() for p in net_l.parameters())
    with ar_c.exported(cpu=True, module=net_c):
        sd_c = {k: v.clone() for k, v in net_c.state_dict().items()}
    for k in sd_c:
        assert sd_l[k].stride() == sd_c[k].stride() and torch.equal(sd_l[k], sd_c[k]), k
    # EMA: averaged values written contiguous, read back into either layout
    ema_c, ema_l = WeightEMA(ar_c, net_c, 0.9), WeightEMA(ar_l, net_l, 0.9)
    g = torch.Generator().manual_seed(2)
    for s_c, s_l in zip(ar_c.slots, ar_l.slots):
        v = torch.randn(s_c.shape, generator=g)
        ParamArena.slot_view(ema_c.ema, s_c).copy_(v)
        ParamArena.slot_view(ema_l.ema, s_l).copy_(v)
    ema_c.updates = ema_l.updates = 4
    blob_c, blob_l = ema_c.state_dict(), ema_l.state_dict()
    assert _all_contiguous(blob_l["state_dict"])
    for k, v in blob_c["state_dict"].items():
        assert torch.equal(v, blob_l["state_dict"][k]) and v.stride() == blob_l["state_dict"][k].stride(), k
    other_l = WeightEMA(_arena(n1 := _net(1), True), n1, 0.9)
    other_l.load_state_dict(blob_c)                                   # NCHW file -> NHWC run
    assert torch.equal(other_l.ema, ema_l.ema) and other_l.updates == 4
    other_c = WeightEMA(_arena(n2 := _net(1), False), n2, 0.9)
    other_c.load_state_dict(blob_l)                                   # NHWC file -> NCHW run
    assert torch.equal(other_c.ema, ema_c.ema)


# ---- the switch ------------------------------------------------------------------------------------------

def test_env_parsing(monkeypatch):
    monkeypatch.delenv(CHANNELS_LAST_ENV, raising=False)
    assert resolve_channels_last() is False
    assert resolve_channels_last(True) is True and resolve_channels_last(False) is False
    monkeypatch.setenv(CHANNELS_LAST_ENV, "1")
    assert resolve_channels_last() is True and resolve_channels_last(False) is False
    monkeypatch.setenv(CHANNELS_LAST_ENV, " 0 ")
    assert resolve_channels_last() is False
    for bad in ("2", "yes", "true", ""):
        monkeypatch.setenv(CHANNELS_LAST_ENV, bad)
        with pytest.raises(ValueError, match=CHANNELS_LAST_ENV):
            resolve_channels_last()


def test_adafactor_is_refused_before_a_rank_starts(ns, monkeypatch, tmp_path):
    from frl_b200 import synthetic
    check_channels_last(True, False)
    check_channels_last(False, True)
    with pytest.raises(ValueError, match="adafactor.*channels_last"):
        check_channels_last(True, True)
    t = ns.types
    run_opts = t.RunOpts(optim=t.OptimOpts(algo=t.OptAlgorithm.ADAM), batchSize=8, nEpochs=1, numThreads=0,
                         singleThreaded=True)
    problem = synthetic.make_toy_problem(ns, str(tmp_path), n_train=16, n_test=0)
    monkeypatch.setattr(solver, "_cuda_device_count_without_poisoning_fork",
                        lambda: pytest.fail("a rank was about to start"))
    with pytest.raises(ValueError, match="adafactor.*channels_last"):
        list(solver.Solver.solve(run_opts, problem, group_name=None, init_method="file:///tmp/unused",
                                 adafactor=True, channels_last=True))
    monkeypatch.setenv(CHANNELS_LAST_ENV, "1")
    with pytest.raises(ValueError, match="adafactor.*channels_last"):
        list(solver.Solver.solve(run_opts, problem, group_name=None, init_method="file:///tmp/unused",
                                 adafactor=True))
    monkeypatch.setenv(CHANNELS_LAST_ENV, "on")
    with pytest.raises(ValueError, match=CHANNELS_LAST_ENV):
        list(solver.Solver.solve(run_opts, problem, group_name=None, init_method="file:///tmp/unused"))


def test_solver_worker_args_field_positions():
    f = SolverWorkerArgs._fields
    assert f.index("channels_last") == f.index("adamw") + 1
    assert f[-4:] == ("optimizer_state", "adafactor", "ema_decay", "grad_accumulation")
    assert SolverWorkerArgs._field_defaults["channels_last"] is None


def test_local_solver_takes_the_keyword():
    import inspect
    from frl_b200.local_solver import LocalSolver
    assert "channels_last" in inspect.signature(LocalSolver.solve).parameters
    assert "channels_last" in inspect.signature(solver.Solver.solve).parameters


# ---- K5 into channels_last, restated -------------------------------------------------------------------------

def k5_nhwc_np(src, scale, bias, out_dtype):
    """What ``frl_preproc_affine_nhwc`` writes, as the [B, H, W, C] array of its memory: K5's fp32
    per-channel ``fma(x, scale[c], bias[c])`` (a missing scale is 1, a missing bias 0; ``x * 1`` with
    neither), rounded once to ``out_dtype`` (float32, or bfloat16 as torch rounds)."""
    x = np.asarray(src, dtype=np.float32)
    C = x.shape[1]
    if scale is None and bias is None:
        y = x * np.float32(1.0)
    else:
        sc = np.ones(C, np.float32) if scale is None else np.asarray(scale, np.float32)
        bi = np.zeros(C, np.float32) if bias is None else np.asarray(bias, np.float32)
        # one rounding of the exact x*sc + bi, as fmaf
        y = (x.astype(np.float64) * sc[None, :, None, None].astype(np.float64)
             + bi[None, :, None, None].astype(np.float64)).astype(np.float32)
    y = np.ascontiguousarray(y.transpose(0, 2, 3, 1))
    if out_dtype == torch.bfloat16:
        return torch.from_numpy(y).to(torch.bfloat16)
    return torch.from_numpy(y)


def _k5_nchw_np(src, scale, bias):
    x = np.asarray(src, dtype=np.float32)
    C = x.shape[1]
    out = np.empty_like(x)
    for c in range(C):
        s = np.float64(1.0 if scale is None else scale[c])
        b = np.float64(0.0 if bias is None else bias[c])
        out[:, c] = (x[:, c].astype(np.float64) * s + b).astype(np.float32) if (scale is not None or bias is not None) \
            else x[:, c]
    return out


@pytest.mark.parametrize("C", [1, 3, 4])
@pytest.mark.parametrize("hw", [(5, 7), (4, 8)])
def test_k5_nhwc_restatement_is_k5_permuted(C, hw):
    g = np.random.default_rng(C)
    src = g.integers(0, 256, (3, C) + hw).astype(np.uint8)
    scale = [float(np.float32(1 / (255 * (0.2 + 0.1 * c)))) for c in range(C)]
    bias = [float(np.float32(-0.4 - 0.1 * c)) for c in range(C)]
    for sc, bi in ((scale, bias), (None, bias), (scale, None), (None, None)):
        want = _k5_nchw_np(src, sc, bi)
        got = k5_nhwc_np(src, sc, bi, torch.float32).numpy()
        assert np.array_equal(got, want.transpose(0, 2, 3, 1))
        got16 = k5_nhwc_np(src, sc, bi, torch.bfloat16)
        assert torch.equal(got16, torch.from_numpy(want).to(torch.bfloat16).permute(0, 2, 3, 1).contiguous())
