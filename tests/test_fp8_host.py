"""The FP8 training precision on the host: the enum and its environment switch, argument checks of
the K9 entry points (no GPU needed: they fail before any launch) and which Linear sites an FP8 run
puts on the FP8 tensor cores."""
import os
import tempfile

import torch
import torch.nn as nn

import frl_b200  # noqa: F401
from frl_b200 import _native, arena_linear, fused_optim, grad_sync, synthetic
from frl_b200.arena import ParamArena
from frl_b200.solver import resolve_precision
from frl_b200.types import OptAlgorithm, OptimOpts, Precision
from oracle.optim_np import KernelDouble


def test_fp8_precision_resolves_from_the_enum_and_the_environment(monkeypatch):
    assert Precision("fp8") is Precision.FP8
    monkeypatch.setenv("FRL_B200_PRECISION", "fp8")
    assert resolve_precision() is Precision.FP8
    monkeypatch.setenv("FRL_B200_PRECISION", "FP8")
    assert resolve_precision() is Precision.FP8
    assert resolve_precision(Precision.BF16) is Precision.BF16
    assert [p.bf16_storage for p in Precision] == [False, True, True]


def test_fp8_arena_is_laid_out_like_bf16():
    def net():
        torch.manual_seed(0)
        return nn.Sequential(nn.Linear(32, 48), nn.ReLU(), nn.Linear(48, 5))
    a16 = ParamArena(net().parameters(), device="cpu", precision=Precision.BF16)
    a8 = ParamArena(net().parameters(), device="cpu", precision=Precision.FP8)
    assert a8.grad.dtype == a16.grad.dtype == torch.bfloat16
    assert a8.master.dtype == torch.float32 and a8.lp.dtype == torch.bfloat16
    assert [(s.offset, s.numel, s.uses_lp) for s in a8.slots] == [(s.offset, s.numel, s.uses_lp) for s in a16.slots]
    assert torch.equal(a8.lp, a16.lp) and torch.equal(a8.master, a16.master)


def test_fp8_entry_points_reject_bad_arguments_before_any_launch():
    lib = _native.lib()
    ok = 1 << 20                           # 16-byte aligned, never dereferenced: every call below fails a check
    bad_cases = [
        ("frl_fp8_amax", lambda: lib.frl_fp8_amax(None, 16, _native.BF16, ok, None)),
        ("frl_fp8_amax", lambda: lib.frl_fp8_amax(ok, 16, _native.BF16, None, None)),
        ("frl_fp8_amax", lambda: lib.frl_fp8_amax(ok, 0, _native.BF16, ok, None)),
        ("frl_fp8_amax", lambda: lib.frl_fp8_amax(ok, 16, _native.U8, ok, None)),
        ("frl_fp8_amax", lambda: lib.frl_fp8_amax(ok + 2, 16, _native.BF16, ok, None)),
        ("frl_fp8_quantize", lambda: lib.frl_fp8_quantize(None, 16, 16, _native.BF16, ok, 0, ok, ok, ok, None)),
        ("frl_fp8_quantize", lambda: lib.frl_fp8_quantize(ok, 16, 16, _native.BF16, None, 0, ok, ok, ok, None)),
        ("frl_fp8_quantize", lambda: lib.frl_fp8_quantize(ok, 16, 16, _native.BF16, ok, 0, ok, ok, None, None)),
        ("frl_fp8_quantize", lambda: lib.frl_fp8_quantize(ok, 16, 16, _native.BF16, ok, 0, None, None, ok, None)),
        ("frl_fp8_quantize", lambda: lib.frl_fp8_quantize(ok, 0, 16, _native.BF16, ok, 0, ok, ok, ok, None)),
        ("frl_fp8_quantize", lambda: lib.frl_fp8_quantize(ok, 16, -1, _native.BF16, ok, 0, ok, ok, ok, None)),
        ("frl_fp8_quantize", lambda: lib.frl_fp8_quantize(ok, 16, 16, _native.I64, ok, 0, ok, ok, ok, None)),
        ("frl_fp8_quantize", lambda: lib.frl_fp8_quantize(ok, 16, 16, _native.BF16, ok, 2, ok, ok, ok, None)),
        ("frl_fp8_quantize", lambda: lib.frl_fp8_quantize(ok + 8, 16, 16, _native.BF16, ok, 0, ok, ok, ok, None)),
        ("frl_fp8_quantize", lambda: lib.frl_fp8_quantize(ok, 16, 16, _native.BF16, ok, 1, ok, ok + 4, ok, None)),
        ("frl_fp8_quantize", lambda: lib.frl_fp8_quantize(ok, 16, 16, _native.BF16, ok + 1, 1, ok, None, ok, None)),
    ]
    for name, call in bad_cases:
        lib.frl_launch_count_reset()
        rc = call()
        assert rc < 0, name
        assert name.encode() in lib.frl_last_error()
        assert lib.frl_launch_count() == 0


def test_site_rule_as_a_pure_function():
    q = arena_linear.fp8_site_qualifies
    assert q(True, 4096, 4096)
    assert not q(True, 4096, 1000 + 64)          # the headline MLP's fused heads
    assert not q(True, 4096, 1000) and q(True, 4096, 64)
    assert not q(False, 4096, 4096)              # weight not in the bf16 shadow
    assert not q(True, 24, 32) and not q(True, 32, 40)
    c = arena_linear.fp8_call_qualifies
    assert c(torch.empty(64, 32, dtype=torch.bfloat16)) and c(torch.empty(4, 8, 32, dtype=torch.bfloat16))
    assert c(torch.empty(16, 32)) and not c(torch.empty(16, 32, dtype=torch.float16))
    assert not c(torch.empty(17, 32, dtype=torch.bfloat16)) and not c(torch.empty(0, 32, dtype=torch.bfloat16))
    assert not c(torch.empty(3, 4, 32, dtype=torch.bfloat16))            # 12 rows
    flat = torch.empty(16 * 32 + 8, dtype=torch.bfloat16)
    unaligned = flat[1:1 + 16 * 32].view(16, 32)
    assert unaligned.data_ptr() % 16 != 0 and not c(unaligned)
    assert c(torch.empty(16, 64, dtype=torch.bfloat16)[:, 1:33])       # not contiguous: copied first


def _fp8_flags(model, precision=Precision.FP8, monkeypatch=None):
    """{module: site.fp8} of the Linear sites ``patch_linears`` makes for ``model`` (CPU tensors,
    kernels replaced by the host double: only the bookkeeping runs)."""
    arena = ParamArena(model.parameters(), device="cpu", precision=precision,
                       adjacent=arena_linear.head_layout_groups(model))
    opt = fused_optim.create_fused_optimizer(arena, OptimOpts(algo=OptAlgorithm.SGD, lr=0.1))
    pipe = grad_sync.GradBucketPipeline(arena, opt, world_size=1, eager_update=False)
    monkeypatch.setattr(arena_linear, "KERNELS", KernelDouble())
    monkeypatch.setattr(grad_sync, "KERNELS", KernelDouble())
    pipe.patch_linears(model)
    flags = {s.module: s.fp8 for s in pipe.linear_sites}
    pipe.unpatch_linears()
    return flags


def test_headline_mlp_runs_its_three_trunk_layers_in_fp8(monkeypatch):
    ns = synthetic.api_namespace("frl_b200")
    problem = synthetic.make_mlp_problem(ns, tempfile.mkdtemp(prefix="frl_b200_fp8_"), n_train=8, width=4096,
                                         n_classes=1000, reg_dim=64, depth=3)
    model = problem.get_model()
    flags = _fp8_flags(model, monkeypatch=monkeypatch)
    trunk = [m for m in model.model_base.modules() if type(m) is nn.Linear]
    heads = list(model.additional_layers)
    assert len(trunk) == 3 and len(heads) == 2 and len(flags) == 5
    assert all(flags[m] for m in trunk)
    assert not any(flags[h] for h in heads)      # fused into one [1064, 4096] unit that stays bf16
    assert not any(_fp8_flags(problem.get_model(), Precision.BF16, monkeypatch).values())


def test_text_problem_and_odd_widths(monkeypatch, tmp_path):
    ns = synthetic.api_namespace("frl_b200")
    train, test = os.path.join(tmp_path, "train.txt"), os.path.join(tmp_path, "test.txt")
    synthetic.write_text_corpus(train, 64, 0)
    synthetic.write_text_corpus(test, 16, 1)
    torch.manual_seed(0)
    model = synthetic.make_text_problem(ns, str(tmp_path), train, test).get_model()
    flags = _fp8_flags(model, monkeypatch=monkeypatch)
    assert sorted((m.in_features, m.out_features, f) for m, f in flags.items()) == [(64, 128, True), (128, 256, True)]

    odd = nn.Sequential(nn.Linear(24, 32), nn.ReLU(), nn.Linear(32, 40), nn.Linear(40, 48), nn.Linear(48, 16))
    flags = _fp8_flags(odd, monkeypatch=monkeypatch)
    assert [flags[m] for m in odd if type(m) is nn.Linear] == [False, False, False, True]
    frozen = nn.Sequential(nn.Linear(32, 32), nn.Linear(32, 32))
    frozen[0].weight.requires_grad_(False)       # not in the arena: stock nn.Linear
    flags = _fp8_flags(frozen, monkeypatch=monkeypatch)
    assert list(flags.values()) == [True] and frozen[1] in flags
