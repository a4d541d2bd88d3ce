"""Mixup / CutMix and soft-target cross-entropy without a GPU: BatchMix's arguments and draws,
the argument errors of frl_augment_mix_images, frl_mix_targets and of the criteria's new checks,
the criteria's routing of smoothed / probability targets, and the synthetic Problem's wiring."""
import ctypes

import numpy as np
import pytest
import scipy.stats
import torch
import torch.nn as nn

import frl_b200  # noqa: F401
from frl_b200 import _native, criteria, synthetic
from frl_b200.criteria import MaskedLoss
from frl_b200.transform import BatchMix, DeviceImageAugment

_FAKE = 1 << 20          # never dereferenced: every case below fails before any launch


# ---- BatchMix -----------------------------------------------------------------------------------

@pytest.mark.parametrize("kw", [
    dict(mixup_alpha=-0.1), dict(cutmix_alpha=-1.0), dict(mixup_alpha=float("nan")),
    dict(mixup_alpha=0.0, cutmix_alpha=0.0),
    dict(prob=1.5), dict(prob=-0.1), dict(switch_prob=2.0),
    dict(classes={"y": 1}), dict(classes={"y": 2.5}), dict(classes={"y": True}),
], ids=lambda kw: ",".join("%s=%s" % kv for kv in kw.items()))
def test_batch_mix_rejects_bad_arguments(kw):
    args = dict(classes={"y": 10}, mixup_alpha=0.2)
    args.update(kw)
    with pytest.raises(ValueError):
        BatchMix(**args)


def test_device_image_augment_takes_only_a_batch_mix():
    with pytest.raises(ValueError, match="mix"):
        DeviceImageAugment("x", ["y"], mix={"mixup_alpha": 0.2})
    aug = DeviceImageAugment("x", ["y"], mix=BatchMix({"y": 10}, mixup_alpha=0.2))
    aug.ordinal = 5
    aug.set_epoch(2)
    assert aug.ordinal == 0 and aug.epoch == 2


def _draws(mix, n, **kw):
    args = dict(seed=7, epoch=1, rank=0, out_h=224, out_w=224)
    args.update(kw)
    return [mix.draw(ordinal=k, **args) for k in range(n)]


def test_mixup_lambda_follows_the_beta_law():
    for alpha in (0.2, 0.8, 1.0):
        mix = BatchMix({"y": 10}, mixup_alpha=alpha)
        d = _draws(mix, 4000)
        assert {m for m, _, _ in d} == {BatchMix.MIXUP} and all(b == (0, 0, 0, 0) for _, _, b in d)
        lam = np.array([l for _, l, _ in d])
        assert scipy.stats.kstest(lam, scipy.stats.beta(alpha, alpha).cdf).pvalue > 1e-3


def test_cutmix_boxes_lie_inside_and_set_lambda():
    mix = BatchMix({"y": 10}, cutmix_alpha=1.0)
    for H, W in ((224, 224), (32, 48), (7, 5)):
        for mode, lam, (y0, y1, x0, x1) in _draws(mix, 2000, out_h=H, out_w=W):
            assert mode == BatchMix.CUTMIX
            assert 0 <= y0 <= y1 <= H and 0 <= x0 <= x1 <= W
            assert lam == 1.0 - (y1 - y0) * (x1 - x0) / float(H * W)
    # clipping only shrinks the box, so the reset lambda is at least the drawn one on average
    lam = np.array([l for _, l, _ in _draws(mix, 4000, out_h=1000, out_w=1000)])
    assert (lam >= 0).all() and (lam <= 1).all() and lam.mean() > 0.5


def test_switch_and_prob():
    mix = BatchMix({"y": 10}, mixup_alpha=0.8, cutmix_alpha=1.0, prob=0.75, switch_prob=0.5)
    modes = np.array([m for m, _, _ in _draws(mix, 8000)])
    assert abs((modes == BatchMix.NONE).mean() - 0.25) < 0.03
    assert abs((modes == BatchMix.CUTMIX).mean() - 0.375) < 0.03
    none = [(l, b) for m, l, b in _draws(mix, 200) if m == BatchMix.NONE]
    assert none and all(l == 1.0 and b == (0, 0, 0, 0) for l, b in none)


def test_draws_depend_only_on_seed_epoch_rank_and_ordinal():
    mix = BatchMix({"y": 10}, mixup_alpha=0.8, cutmix_alpha=1.0)
    state = np.random.get_state()
    torch_state = torch.get_rng_state()
    base = _draws(mix, 64)
    assert _draws(BatchMix({"z": 3}, mixup_alpha=0.8, cutmix_alpha=1.0), 64) == base
    np.random.seed(123)
    torch.manual_seed(5)
    assert _draws(mix, 64) == base
    for kw in (dict(seed=8), dict(epoch=2), dict(rank=1), dict(seed=7 + (1 << 32))):
        assert sum(a != b for a, b in zip(_draws(mix, 64, **kw), base)) > 56, kw
    np.random.set_state(state)
    torch.set_rng_state(torch_state)
    assert mix.draw(7, 1, 0, 10, 224, 224) == base[10]


# ---- argument errors without a GPU --------------------------------------------------------------

def _mix_call(**kw):
    args = dict(src=_FAKE, batch=4, channels=3, height=32, width=32, idx=_FAKE, seed=0, epoch=0,
                mode=_native.AUG_RRC, smin=0.08, smax=1.0, rmin=0.75, rmax=4 / 3, eval_crop=0.875, pad=4,
                flip=1, scale=None, bias=None, dst=_FAKE, dst_dtype=_native.F32, out_h=24, out_w=24,
                params_out=None, mix_mode=_native.MIX_CUTMIX, lam=0.5, y0=2, y1=10, x0=0, x1=24, stream=None)
    args.update(kw)
    lib = _native.lib()
    rc = lib.frl_augment_mix_images(*args.values())
    return rc, lib.frl_last_error()


@pytest.mark.parametrize("kw", [
    dict(src=None), dict(idx=None), dict(dst=None), dict(dst_dtype=_native.U8), dict(mode=4),
    dict(channels=5), dict(smin=0.0), dict(epoch=-1), dict(batch=-1), dict(out_h=0),
    dict(mix_mode=0), dict(mix_mode=3), dict(lam=-0.1), dict(lam=1.5), dict(lam=float("nan")),
    dict(y0=-1), dict(y1=25), dict(y0=11, y1=10), dict(x1=25), dict(x0=5, x1=4),
], ids=lambda kw: ",".join("%s=%s" % kv for kv in kw.items()))
def test_augment_mix_images_rejects_bad_arguments(kw):
    rc, msg = _mix_call(**kw)
    assert rc < 0
    assert b"frl_augment_mix_images" in msg


def test_augment_mix_images_empty_batch_and_mixup_box():
    assert _mix_call(batch=0, src=None, idx=None, dst=None)[0] == 0
    # Mixup ignores the box
    assert _mix_call(batch=0, src=None, idx=None, dst=None, mix_mode=_native.MIX_MIXUP, y0=-5, y1=99)[0] == 0


def _targets_call(**kw):
    args = dict(src=_FAKE, src_dtype=_native.I64, batch=4, inner=1, n_classes=10, lam=0.3, dst=_FAKE, stream=None)
    args.update(kw)
    lib = _native.lib()
    return lib.frl_mix_targets(*args.values()), lib.frl_last_error()


@pytest.mark.parametrize("kw", [
    dict(src=None), dict(dst=None), dict(batch=-1), dict(lam=1.01), dict(lam=-1.0),
    dict(n_classes=1), dict(n_classes=0), dict(inner=2), dict(src_dtype=_native.U8),
    dict(src_dtype=_native.F32, inner=0), dict(src_dtype=9),
], ids=lambda kw: ",".join("%s=%s" % kv for kv in kw.items()))
def test_mix_targets_rejects_bad_arguments(kw):
    rc, msg = _targets_call(**kw)
    assert rc < 0
    assert b"frl_mix_targets" in msg


def test_mix_targets_empty_batch_is_a_no_op():
    assert _targets_call(batch=0, src=None, dst=None)[0] == 0
    assert _targets_call(batch=0, src=None, dst=None, src_dtype=_native.BF16, inner=7, n_classes=0)[0] == 0


def _task(**kw):
    d = _native.TaskDesc()
    d.kind, d.out_dtype, d.tgt_dtype, d.ignore_index = _native.LOSS_CE, _native.F32, _native.I64, -100
    d.out, d.tgt, d.dout = _FAKE, _FAKE, _FAKE
    d.rows, d.cols, d.mask_inner, d.weight = 8, 10, 1, 1.0
    for k, v in kw.items():
        setattr(d, k, v)
    return d


@pytest.mark.parametrize("kw", [
    dict(label_smoothing=-0.1), dict(label_smoothing=1.5), dict(label_smoothing=float("nan")),
    dict(kind=_native.LOSS_MSE, tgt_dtype=_native.F32, label_smoothing=0.1),
    dict(kind=_native.LOSS_CE_PROB, tgt_dtype=_native.I64),
    dict(kind=_native.LOSS_CE_PROB, tgt_dtype=_native.U8),
    dict(kind=_native.LOSS_CE_PROB, tgt_dtype=_native.F32, mask=_FAKE, mask_inner=1),
    dict(kind=3),
], ids=lambda kw: ",".join("%s=%s" % kv for kv in kw.items()))
def test_criteria_reject_bad_soft_tasks(kw):
    lib = _native.lib()
    arr = _native.make_task_array([_task(**kw)])
    rc = lib.frl_criteria_forward(arr, 1, _FAKE, _FAKE, _FAKE, None, None, _FAKE, None)
    assert rc < 0 and b"frl_criteria_forward" in lib.frl_last_error()
    rc = lib.frl_criteria_backward(arr, 1, _FAKE, _FAKE, _FAKE, None)
    assert rc < 0 and b"frl_criteria_backward" in lib.frl_last_error()


def test_task_desc_keeps_its_layout():
    assert ctypes.sizeof(_native.TaskDesc) == 80
    assert _native.TaskDesc.label_smoothing.offset == 76


# ---- criteria routing (meta tensors stand in for device tensors) --------------------------------

class _Cuda:
    """Just enough of a CUDA tensor for _plan_for's checks."""

    def __init__(self, shape, dtype):
        self.shape, self.dtype, self.is_cuda, self.requires_grad = torch.Size(shape), dtype, True, False

    def dim(self):
        return len(self.shape)

    def is_floating_point(self):
        return self.dtype.is_floating_point

    def reshape(self, *s):
        return self


@pytest.mark.parametrize("ls", [0.0, 0.1, 1.0])
def test_smoothed_and_probability_targets_take_the_kernels(ls):
    ce = nn.CrossEntropyLoss(label_smoothing=ls)
    out = _Cuda((8, 10), torch.bfloat16)
    plan = criteria._plan_for([ce], [out], [(_Cuda((8,), torch.int64),)])
    assert plan.tasks[0].kind == _native.LOSS_CE and plan.tasks[0].label_smoothing == ls
    for dt in (torch.float32, torch.bfloat16):
        plan = criteria._plan_for([ce], [out], [(_Cuda((8, 10), dt),)])
        assert plan.tasks[0].kind == _native.LOSS_CE_PROB and plan.tasks[0].label_smoothing == ls
    plan = criteria._plan_for([MaskedLoss(ce)], [out], [(_Cuda((8, 10), torch.float32), _Cuda((8,), torch.bool))])
    assert plan.tasks[0].kind == _native.LOSS_CE_PROB and plan.tasks[0].masked
    # a smoothed head no longer takes its MSE neighbour off the kernels
    plan = criteria._plan_for([nn.MSELoss(), ce], [_Cuda((8, 4), torch.float32), out],
                              [(_Cuda((8, 4), torch.float32),), (_Cuda((8, 10), torch.float32),)])
    assert [t.kind for t in plan.tasks] == [_native.LOSS_MSE, _native.LOSS_CE_PROB]


def test_weighted_and_per_position_soft_targets_stay_composed():
    out = _Cuda((8, 10), torch.float32)
    assert criteria._plan_for([nn.CrossEntropyLoss(weight=torch.ones(10))], [out], [(_Cuda((8,), torch.int64),)]) is None
    per_pos = _Cuda((8, 10, 5), torch.float32)
    assert criteria._plan_for([nn.CrossEntropyLoss()], [per_pos], [(_Cuda((8, 10, 5), torch.float32),)]) is None
    assert criteria._plan_for([nn.CrossEntropyLoss()], [out], [(_Cuda((8, 10), torch.float16),)]) is None
    assert criteria._plan_for([nn.CrossEntropyLoss()], [out], [(_Cuda((8, 9), torch.float32),)]) is None

    class Sub(nn.CrossEntropyLoss):
        pass
    assert criteria._plan_for([Sub(label_smoothing=0.1)], [out], [(_Cuda((8,), torch.int64),)]) is None


# ---- the synthetic Problem ----------------------------------------------------------------------

def test_mixing_resnet_problem_wiring(ns, tmp_path):
    prob = synthetic.make_resnet_problem(ns, str(tmp_path), "resnet50x4", uint8=True, augment="rrc",
                                         stored_image=40, image=32, n_train=4, n_test=2, mixup_alpha=0.8,
                                         cutmix_alpha=1.0, label_smoothing=0.1)
    aug = prob.datasets[0].device_transform
    assert isinstance(aug.mix, BatchMix)
    assert aug.mix.classes == {"y_cls": 1000, "y_cls2": 100}
    assert (aug.mix.mixup_alpha, aug.mix.cutmix_alpha) == (0.8, 1.0)
    crit = prob.get_criterion()
    smoothing = [getattr(m, "label_smoothing", None) for m in crit.loss_modules]
    assert smoothing == [0.1, 0.1, None, None]
    plain = synthetic.make_resnet_problem(ns, str(tmp_path), "resnet18", uint8=True, augment="rrc",
                                          stored_image=40, image=32, n_train=4, n_test=2)
    assert plain.datasets[0].device_transform.mix is None
    assert plain.get_criterion().loss_modules[0].label_smoothing == 0.0
    with pytest.raises(ValueError, match="augment"):
        synthetic.make_resnet_problem(ns, str(tmp_path), uint8=True, image=32, mixup_alpha=0.2)


def test_classification_error_uses_the_dominant_class(ns):
    _, Cls = synthetic._task_classes(ns)
    task = Cls(4, 3, 1.0)
    out = torch.tensor([[0.0, 2.0, 1.0], [3.0, 0.0, 0.0]])
    soft = torch.tensor([[0.1, 0.7, 0.2], [0.4, 0.6, 0.0]])
    assert task.compute_batch_metrics(None, (soft,), out)["cls_err"].tolist() == [0.0, 1.0]
    assert task.compute_batch_metrics(None, (torch.tensor([1, 0]),), out)["cls_err"].tolist() == [0.0, 0.0]
