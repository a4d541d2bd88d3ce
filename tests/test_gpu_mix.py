"""Mixup / CutMix on the device (frl_augment_mix_images, frl_mix_targets, BatchMix): images bit
for bit against the numpy restatement (tests/mix_np.py) applied to K5a's fp32 output on the same
batch, the odd middle sample and unmixed batches against K5a, resnet50x4's four target fields,
loader reproducibility, and Solver.solve over the mixing ResNet with smoothed labels."""
import logging
import tempfile

import numpy as np
import pytest
import torch
import torch.nn as nn

import frl_b200  # noqa: F401
import mix_np as M
from frl_b200 import _native, criteria, synthetic
from frl_b200.device_loader import DeviceBatchLoader
from frl_b200.solver import Solver
from frl_b200.transform import BatchMix
from frl_b200.types import Precision, Split

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
SC, BI = synthetic.U8_CHANNEL_AFFINE


def _inputs(B, H=72, W=80, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(0, 256, (B, 3, H, W), generator=g, dtype=torch.uint8).to(DEV)
    idx = torch.randint(0, 1 << 40, (B,), generator=g).to(DEV)
    return x, idx


def _kw(**over):
    kw = dict(seed=11, epoch=3, mode=_native.AUG_RRC, scale=torch.tensor(SC, device=DEV),
              bias=torch.tensor(BI, device=DEV), flip=True)
    kw.update(over)
    return kw


def _k5a(x, idx, out_hw, dtype, **over):
    out = torch.empty((x.shape[0], 3) + out_hw, dtype=dtype, device=DEV)
    params = torch.full((x.shape[0], 5), -7, dtype=torch.int32, device=DEV)
    _native.augment_images(x, idx, out, params_out=params, **_kw(**over))
    return out, params


def _mixed(x, idx, out_hw, dtype, mix_mode, lam, box, **over):
    out = torch.full((x.shape[0], 3) + out_hw, float("nan"), dtype=dtype, device=DEV)
    params = torch.full((x.shape[0], 5), -7, dtype=torch.int32, device=DEV)
    _native.augment_mix_images(x, idx, out, mix_mode=mix_mode, lam=lam, box=box, params_out=params, **_kw(**over))
    return out, params


def _bits(t):
    return t.cpu().view(torch.int16) if t.dtype == torch.bfloat16 else t.cpu().view(torch.int32)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("B", [32, 33])
@pytest.mark.parametrize("mode,lam,box", [(M.MIXUP, 0.3141, (0, 0, 0, 0)), (M.MIXUP, 0.9, (0, 0, 0, 0)),
                                          (M.CUTMIX, 0.75, (8, 40, 20, 52)), (M.CUTMIX, 0.0, (0, 56, 0, 64)),
                                          (M.CUTMIX, 1.0, (5, 5, 0, 64))])
def test_images_equal_the_numpy_restatement(dtype, B, mode, lam, box):
    x, idx = _inputs(B)
    a32, p_ref = _k5a(x, idx, (56, 64), torch.float32)
    got, p = _mixed(x, idx, (56, 64), dtype, mode, lam, box)
    torch.cuda.synchronize()
    assert torch.equal(p.cpu(), p_ref.cpu())
    want = M.mix_images(a32.cpu().numpy(), mode, lam, box, dtype)
    assert torch.equal(_bits(got), _bits(want))
    if B % 2:                                    # the middle sample is K5a's, bit for bit
        k5a, _ = _k5a(x, idx, (56, 64), dtype)
        assert torch.equal(_bits(got[B // 2]), _bits(k5a[B // 2]))


def test_pad_crop_mode_and_single_sample():
    x, idx = _inputs(7, 32, 32, seed=3)
    a32, _ = _k5a(x, idx, (32, 32), torch.float32, mode=_native.AUG_PAD_CROP, pad=4)
    got, _ = _mixed(x, idx, (32, 32), torch.float32, M.MIXUP, 0.6, (0, 0, 0, 0), mode=_native.AUG_PAD_CROP, pad=4)
    assert torch.equal(_bits(got), _bits(M.mix_images(a32.cpu().numpy(), M.MIXUP, 0.6)))
    x1, i1 = x[:1].contiguous(), idx[:1].contiguous()
    one, _ = _mixed(x1, i1, (24, 24), torch.bfloat16, M.CUTMIX, 0.5, (0, 12, 0, 24))
    k5a, _ = _k5a(x1, i1, (24, 24), torch.bfloat16)
    assert torch.equal(_bits(one), _bits(k5a))


def test_targets_of_resnet50x4_fields():
    B = 33
    g = torch.Generator().manual_seed(5)
    fields = {"y_cls": torch.randint(0, 1000, (B,), generator=g), "y_cls2": torch.randint(0, 100, (B,), generator=g),
              "y_reg": torch.randn(B, 10, generator=g), "y_reg2": torch.randn(B, 4, generator=g)}
    fields["y_cls"][4] = fields["y_cls"][B - 5]            # the same class on both sides of a pair
    for lam in (0.3141, 1.0, 0.0):
        for name, n in (("y_cls", 1000), ("y_cls2", 100)):
            dst = torch.full((B, n), -1.0, device=DEV)
            _native.mix_targets(fields[name].to(DEV), dst, lam, n)
            want = M.mix_labels(fields[name].numpy(), n, lam)
            assert np.array_equal(dst.cpu().numpy(), want, equal_nan=True), (name, lam)
        for name in ("y_reg", "y_reg2"):
            for dt in (torch.float32, torch.bfloat16):
                src = fields[name].to(dt).to(DEV)
                dst = torch.empty_like(src)
                _native.mix_targets(src, dst, lam)
                assert torch.equal(_bits(dst), _bits(M.mix_values(src.cpu(), lam))), (name, dt, lam)
    bad = fields["y_cls2"].clone()
    bad[2] = 100
    dst = torch.empty(B, 100, device=DEV)
    _native.mix_targets(bad.to(DEV), dst, 0.4, 100)
    nan_rows = torch.isnan(dst.cpu()).any(1)
    assert nan_rows.tolist() == [i in (2, B - 3) for i in range(B)]
    assert torch.isnan(dst.cpu()[nan_rows]).all()


def _mixing_problem(ns, folder, prob=1.0, n_train=64, n_test=16, config="resnet50x4"):
    p = synthetic.make_resnet_problem(ns, folder, config, uint8=True, augment="rrc", stored_image=40, image=32,
                                      n_train=n_train, n_test=n_test, mixup_alpha=0.8, cutmix_alpha=1.0,
                                      label_smoothing=0.1)
    p.datasets[0].device_transform.mix.prob = prob
    return p


def _epoch(loader, seed):
    torch.manual_seed(seed)
    return [(d[0].cpu(), [h[0].cpu() for h in tg], m["index"].cpu()) for d, tg, m in loader]


def _same(a, b):
    assert len(a) == len(b)
    for (x0, t0, i0), (x1, t1, i1) in zip(a, b):
        assert torch.equal(i0, i1) and torch.equal(_bits(x0), _bits(x1))
        assert all(torch.equal(u, v) for u, v in zip(t0, t1))


def test_unmixed_batches_are_k5a_with_one_hot_targets(ns):
    train = _mixing_problem(ns, tempfile.mkdtemp(prefix="frl_b200_mix_"), prob=0.0).datasets[0]
    ld = DeviceBatchLoader(train, batch_size=16, sampler=None, device=DEV, out_dtype=torch.bfloat16)
    ld.set_epoch(1)
    for x, tg, ids in _epoch(ld, 0):
        aug = train.device_transform
        direct = aug.augment(train.pinned_fields["x"][ids].to(DEV), ids.to(DEV), Split.TRAIN, torch.bfloat16)
        assert torch.equal(_bits(direct), _bits(x))
        for (name, n), t in zip((("y_cls", 1000), ("y_cls2", 100)), tg[:2]):
            want = torch.nn.functional.one_hot(torch.as_tensor(train.pinned_fields[name][ids]), n).float()
            assert t.dtype == torch.float32 and torch.equal(t, want)
        assert torch.equal(tg[2], torch.as_tensor(train.pinned_fields["y_reg"][ids]))


def test_loader_epochs_reproduce(ns):
    folder = tempfile.mkdtemp(prefix="frl_b200_mix_")
    train = _mixing_problem(ns, folder).datasets[0]
    ld = DeviceBatchLoader(train, batch_size=16, sampler=None, device=DEV, out_dtype=torch.bfloat16)
    ld.set_epoch(1)
    first = _epoch(ld, 0)
    ld.set_epoch(1)
    _same(first, _epoch(ld, 0))
    ld.set_epoch(2)
    second = _epoch(ld, 1)
    fresh = DeviceBatchLoader(_mixing_problem(ns, folder).datasets[0], batch_size=16, sampler=None, device=DEV,
                              out_dtype=torch.bfloat16)
    fresh.set_epoch(2)
    _same(second, _epoch(fresh, 1))
    # every batch is mixed: class targets are probability rows, and at least one is not one-hot
    for _, tg, _ in first + second:
        assert tg[0].shape == (16, 1000) and torch.allclose(tg[0].sum(1), torch.ones(16))
    assert any(bool((tg[0].max(1).values < 1).any()) for _, tg, _ in first)


def test_solve_mixing_resnet_with_label_smoothing(ns, caplog):
    folder = tempfile.mkdtemp(prefix="frl_b200_mix_")
    problem = _mixing_problem(ns, folder, n_train=64, n_test=16, config="resnet18")
    t = ns.types
    run_opts = t.RunOpts(optim=t.OptimOpts(algo=t.OptAlgorithm("sgd"), lr=0.01), batchSize=16, nEpochs=2,
                         numThreads=0, singleThreaded=True, numVisualizedSamples=0)
    captured = {}
    orig = Solver.build_worker.__func__

    def spy(cls, args):
        worker, sched, ckpt = orig(cls, args)
        captured["worker"] = worker
        return worker, sched, ckpt

    Solver.build_worker = classmethod(spy)
    criteria._path_logged.clear()              # the path line is logged once per process
    try:
        torch.manual_seed(0)
        with caplog.at_level(logging.INFO):
            list(Solver.solve(run_opts, problem, group_name=None, init_method="file:///tmp/unused",
                              precision=Precision.BF16))
    finally:
        Solver.build_worker = classmethod(orig)
    text = "\n".join(r.getMessage() for r in caplog.records)
    assert "fused kernels" in text and "composed torch ops" not in text
    hist = captured["worker"].loss_history
    assert {(e, s) for e, s, _ in hist} == {(1, Split.TEST), (1, Split.TRAIN), (2, Split.TEST), (2, Split.TRAIN)}
    assert all(v.size > 0 and np.isfinite(v).all() for _, _, v in hist)


class _ComposedCE(nn.CrossEntropyLoss):
    """Fails _classify's exact-type check, so the criterion composes torch ops for it."""


def test_fp32_first_minibatch_loss_matches_the_composed_path(ns):
    problem = _mixing_problem(ns, tempfile.mkdtemp(prefix="frl_b200_mix_"))
    train = problem.datasets[0]
    ld = DeviceBatchLoader(train, batch_size=16, sampler=None, device=DEV, out_dtype=torch.float32)
    ld.set_epoch(1)
    torch.manual_seed(0)
    data, target, _ = next(iter(ld))
    torch.manual_seed(0)
    model = problem.get_model().to(DEV)
    with torch.no_grad():
        out = model(data)
    fused = problem.get_criterion()
    composed = problem.get_criterion()
    composed.loss_modules = nn.ModuleList([_ComposedCE(label_smoothing=m.label_smoothing)
                                           if isinstance(m, nn.CrossEntropyLoss) else m
                                           for m in composed.loss_modules])
    assert criteria._plan_for(list(fused.loss_modules), list(out), target) is not None
    assert criteria._plan_for(list(composed.loss_modules), list(out), target) is None
    a, _ = fused(list(out), target)
    b, _ = composed(list(out), target)
    assert torch.isfinite(a) and abs(float(a) - float(b)) <= 1e-5 * abs(float(b))
