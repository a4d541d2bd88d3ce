"""Image augmentation without a GPU: argument checks of frl_augment_images (K5a) and of
DeviceImageAugment, the numpy restatement of the sample parameters, the loader/transform
plumbing and the augmenting ResNet Problem's per-sample (evaluation) path."""
import numpy as np
import pytest
import torch

import frl_b200  # noqa: F401
from frl_b200 import _native, synthetic
from frl_b200.device_loader import DeviceBatchLoader
from frl_b200.transform import DeviceBatchTransform, DeviceImageAugment
from frl_b200.types import Split
from oracle import augment_np as A

_FAKE = 1 << 20          # never dereferenced: every case below fails before any launch


def _call(**kw):
    args = dict(src=_FAKE, batch=4, channels=3, height=32, width=32, idx=_FAKE, seed=0, epoch=0,
                mode=_native.AUG_RRC, smin=0.08, smax=1.0, rmin=0.75, rmax=4 / 3, eval_crop=0.875, pad=4,
                flip=1, scale=None, bias=None, dst=_FAKE, dst_dtype=_native.F32, out_h=24, out_w=24,
                params_out=None, stream=None)
    args.update(kw)
    lib = _native.lib()
    rc = lib.frl_augment_images(*args.values())
    return rc, lib.frl_last_error()


@pytest.mark.parametrize("kw", [
    dict(src=None), dict(idx=None), dict(dst=None),
    dict(dst_dtype=_native.U8), dict(dst_dtype=7),
    dict(mode=4), dict(mode=-1),
    dict(out_h=0), dict(out_w=0),
    dict(channels=5), dict(channels=0),
    dict(smin=0.9, smax=0.5), dict(smin=0.0),
    dict(rmin=0.0), dict(rmin=-1.0), dict(rmin=2.0, rmax=1.0),
    dict(pad=-1),
    dict(mode=_native.AUG_PAD_CROP, pad=0, out_h=33),
    dict(mode=_native.AUG_CENTER_RESIZE, eval_crop=0.0),
    dict(mode=_native.AUG_CENTER_RESIZE, eval_crop=1.5),
    dict(height=0), dict(batch=-1), dict(epoch=-1),
], ids=lambda kw: ",".join("%s=%s" % kv for kv in kw.items()))
def test_augment_images_rejects_bad_arguments(kw):
    rc, msg = _call(**kw)
    assert rc < 0
    assert b"frl_augment_images" in msg


def test_augment_images_empty_batch_is_a_no_op():
    assert _call(batch=0, src=None, idx=None, dst=None)[0] == 0


@pytest.mark.parametrize("kw", [
    dict(mode="flip"), dict(out_size=0), dict(out_size=(8, 0)),
    dict(crop_scale=(0.9, 0.1)), dict(crop_scale=(0.0, 1.0)), dict(crop_scale=3),
    dict(crop_ratio=(0.0, 1.0)), dict(crop_ratio=(2.0, 1.0)),
    dict(pad=-1), dict(pad=1.5), dict(eval_crop=0.0), dict(eval_crop=1.2),
    dict(seed=-1), dict(seed=2 ** 64),
    dict(mean=(0.5,) * 3), dict(mean=(0.5,) * 3, std=(0.0, 1.0, 1.0)), dict(mean=(0.5,) * 5, std=(1.0,) * 5),
    dict(mean=(0.5,), std=(0.5,), scale=(1.0,)), dict(scale=(1.0,) * 5), dict(scale=(1.0,), bias=(0.0, 0.0)),
])
def test_device_image_augment_rejects_bad_arguments(kw):
    name = next(iter(kw))
    with pytest.raises(ValueError, match=name.split("_")[0] if name != "mean" else "mean|std"):
        DeviceImageAugment("x", ["y"], **kw)


def test_device_image_augment_checks_the_image_shape():
    aug = DeviceImageAugment("x", ["y"], mode="pad_crop", out_size=32, pad=4, mean=(0.5,) * 3, std=(0.25,) * 3)
    aug.check_image(3, 32, 32)
    aug.check_image(3, 24, 24)
    with pytest.raises(ValueError, match="out_size"):
        aug.check_image(3, 23, 24)
    with pytest.raises(ValueError, match="channels"):
        aug.check_image(5, 32, 32)
    with pytest.raises(ValueError, match="scale"):
        aug.check_image(1, 32, 32)
    assert aug.scale == pytest.approx([1 / (255 * 0.25)] * 3) and aug.bias == pytest.approx([-2.0] * 3)
    assert aug.needs_index and aug.epoch == 0
    aug.set_epoch(3)
    assert aug.epoch == 3
    with pytest.raises(ValueError, match="index"):
        aug.apply({"x": torch.zeros(1, 3, 32, 32, dtype=torch.uint8)}, Split.TRAIN, torch.float32)


def test_existing_transforms_keep_the_plain_apply():
    assert DeviceBatchTransform.needs_index is False
    DeviceBatchTransform.set_epoch(None, 1)               # a no-op on the base class
    assert hasattr(DeviceBatchLoader, "set_epoch")


# ---- the numpy restatement ---------------------------------------------------------------------

def test_philox_known_answers():
    # Random123's published known-answer vectors of philox4x32_10
    got = [int(w[()]) for w in A.philox4x32_10((0, 0, 0, 0), (0, 0))]
    assert got == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]
    f = 0xFFFFFFFF
    got = [int(w[()]) for w in A.philox4x32_10((f, f, f, f), (f, f))]
    assert got == [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]
    got = [int(w[()]) for w in A.philox4x32_10((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344),
                                               (0xA4093822, 0x299F31D0))]
    assert got == [0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1]


@pytest.mark.parametrize("H,W", [(256, 256), (17, 23), (72, 72), (1, 1), (3, 200)])
def test_rrc_boxes_lie_inside_the_image(H, W):
    idx = np.arange(20000)
    for epoch in (0, 1, 7):
        p = A.sample_params(idx, seed=5, epoch=epoch, mode=A.RRC, height=H, width=W, out_h=8, out_w=8)
        top, left, h, w = p[:, 0], p[:, 1], p[:, 2], p[:, 3]
        assert (h >= 1).all() and (w >= 1).all()
        assert (top >= 0).all() and (left >= 0).all()
        assert (top + h <= H).all() and (left + w <= W).all()


def test_rrc_area_and_aspect_follow_the_ranges():
    p, raw, fb = A.sample_params(np.arange(50000), seed=1, epoch=0, mode=A.RRC, height=512, width=512,
                                 out_h=8, out_w=8, with_raw=True)
    ok = ~fb
    assert ok.mean() > 0.9
    area = raw[ok, 0] * raw[ok, 1] / (512 * 512)
    aspect = raw[ok, 0] / raw[ok, 1]
    assert area.min() >= 0.08 - 1e-9 and area.max() <= 1.0 + 1e-9
    assert aspect.min() >= 0.75 - 1e-9 and aspect.max() <= 4 / 3 + 1e-9


def test_rrc_fallback_is_the_ratio_clamped_centre_crop():
    # a 10x100 image cannot hold any box of aspect in [0.5, 2] and area share >= 0.9
    p, raw, fb = A.sample_params(np.arange(1000), seed=0, epoch=0, mode=A.RRC, height=10, width=100,
                                 out_h=8, out_w=8, scale=(0.9, 1.0), ratio=(0.5, 2.0), with_raw=True)
    assert fb.all() and np.isnan(raw).all()
    # r = W/H = 10 > rmax = 2: h = H, w = round(H * rmax), centred
    assert (p[:, :4] == [0, 40, 10, 20]).all()
    # and the other side: a tall image, r < rmin
    p, _, fb = A.sample_params(np.arange(100), seed=0, epoch=0, mode=A.RRC, height=100, width=10,
                               out_h=8, out_w=8, scale=(0.9, 1.0), ratio=(0.5, 2.0), with_raw=True)
    assert fb.all() and (p[:, :4] == [40, 0, 20, 10]).all()
    # a square image where every box fits: the fallback is never taken
    _, _, fb = A.sample_params(np.arange(1000), seed=0, epoch=0, mode=A.RRC, height=64, width=64,
                               out_h=8, out_w=8, scale=(0.5, 0.5), ratio=(1.0, 1.0), with_raw=True)
    assert not fb.any()


def test_pad_crop_offsets_cover_the_padded_range():
    H, S, p = 32, 32, 4
    params = A.sample_params(np.arange(100000), seed=3, epoch=2, mode=A.PAD_CROP, height=H, width=H,
                             out_h=S, out_w=S, pad=p)
    for col in (0, 1):
        assert set(params[:, col].tolist()) == set(range(-p, H + p - S + 1))
    assert (params[:, 2] == S).all() and (params[:, 3] == S).all()
    # 17 x 23 -> 8 x 5, pad 2
    params = A.sample_params(np.arange(20000), seed=3, epoch=0, mode=A.PAD_CROP, height=17, width=23,
                             out_h=8, out_w=5, pad=2)
    assert set(params[:, 0].tolist()) == set(range(-2, 17 + 2 - 8 + 1))
    assert set(params[:, 1].tolist()) == set(range(-2, 23 + 2 - 5 + 1))


def test_flip_rate_is_one_half():
    for mode in (A.RRC, A.PAD_CROP):
        p = A.sample_params(np.arange(100000), seed=0, epoch=1, mode=mode, height=40, width=40, out_h=32,
                            out_w=32, pad=4)
        assert abs(p[:, 4].mean() - 0.5) <= 0.01
        off = A.sample_params(np.arange(1000), seed=0, epoch=1, mode=mode, height=40, width=40, out_h=32,
                              out_w=32, pad=4, flip=False)
        assert (off[:, 4] == 0).all()


def test_centre_modes_are_deterministic():
    for mode in (A.CENTER_RESIZE, A.CENTER_CROP):
        a = A.sample_params(np.arange(50), seed=0, epoch=1, mode=mode, height=256, width=200, out_h=224,
                            out_w=180)
        b = A.sample_params(np.arange(50) + 7, seed=9, epoch=4, mode=mode, height=256, width=200, out_h=224,
                            out_w=180)
        assert (a == b).all() and (a[:, 4] == 0).all()
    a = A.sample_params([0], seed=0, epoch=0, mode=A.CENTER_RESIZE, height=256, width=256, out_h=224, out_w=224)
    assert a[0].tolist() == [16, 16, 224, 224, 0]


def test_draws_depend_on_seed_epoch_and_index_only():
    kw = dict(mode=A.RRC, height=64, width=64, out_h=32, out_w=32)
    base = A.sample_params(np.arange(512), seed=1, epoch=1, **kw)
    perm = np.random.RandomState(0).permutation(512)
    assert (A.sample_params(perm, seed=1, epoch=1, **kw) == base[perm]).all()
    assert (A.sample_params(np.arange(512), seed=1, epoch=2, **kw) != base).any(1).mean() > 0.9
    assert (A.sample_params(np.arange(512), seed=2, epoch=1, **kw) != base).any(1).mean() > 0.9
    big = np.arange(512, dtype=np.int64) + (1 << 33)
    assert (A.sample_params(big, seed=1, epoch=1, **kw) != base).any(1).mean() > 0.9


# ---- the augmenting Problem --------------------------------------------------------------------

def test_augmenting_resnet_problem(ns, tmp_path):
    prob = synthetic.make_resnet_problem(ns, str(tmp_path), uint8=True, augment="rrc", stored_image=72, image=64,
                                         n_train=4, n_test=3)
    train, test = prob.datasets
    assert isinstance(train.device_transform, DeviceImageAugment)
    assert tuple(train.pinned_fields["x"].shape) == (4, 3, 72, 72)
    with pytest.raises(RuntimeError, match="device path only"):
        train[0]
    data, target, meta = test[1]
    x = data[0]
    assert tuple(x.shape) == (3, 64, 64) and x.dtype == torch.float32
    # the centre crop: round(72 * 0.875) = 63 -> top = left = round(4.5) = 4, resized to 64
    raw = torch.from_numpy(test.get_raw_item(1)["x"]).float()
    want = torch.nn.functional.interpolate(raw[None, :, 4:67, 4:67], size=(64, 64), mode="bilinear",
                                           align_corners=False)[0]
    sc, bi = synthetic.U8_CHANNEL_AFFINE
    want = want * torch.tensor(sc).view(-1, 1, 1) + torch.tensor(bi).view(-1, 1, 1)
    torch.testing.assert_close(x, want)
    pc = synthetic.make_resnet_problem(ns, str(tmp_path), uint8=True, augment="pad_crop", stored_image=32,
                                       image=32, n_train=2, n_test=2)
    assert pc.datasets[0].device_transform.mode == "pad_crop" and pc.datasets[0].device_transform.pad == 4
    assert tuple(pc.datasets[1][0][0][0].shape) == (3, 32, 32)


def test_augment_arguments_of_make_resnet_problem(ns, tmp_path):
    with pytest.raises(ValueError, match="uint8"):
        synthetic.make_resnet_problem(ns, str(tmp_path), augment="rrc", image=32)
    with pytest.raises(ValueError, match="augment"):
        synthetic.make_resnet_problem(ns, str(tmp_path), uint8=True, augment="mixup", image=32)
    with pytest.raises(ValueError, match="stored_image"):
        synthetic.make_resnet_problem(ns, str(tmp_path), uint8=True, image=32, stored_image=40)
    with pytest.raises(ValueError, match="out_size"):
        synthetic.make_resnet_problem(ns, str(tmp_path), uint8=True, augment="pad_crop", image=48,
                                      stored_image=32)
