"""K5p (policy + random erasing) without a GPU: argument validation in Python and C, the magnitude
tables against torchvision's, the numpy restatement of the draws on fixed keys, and the
shared-memory refusal."""
import numpy as np
import pytest
import torch

import frl_b200  # noqa: F401
from frl_b200 import _native
from frl_b200.transform import (POLICY_OPS, BatchMix, DeviceImageAugment, RandAugment, RandomErasing,
                                TrivialAugmentWide)
import policy_np


def test_policy_records_validate():
    assert TrivialAugmentWide().num_magnitude_bins == 31
    ra = RandAugment()
    assert (ra.num_ops, ra.magnitude, ra.num_magnitude_bins) == (2, 9, 31)
    for bad in (dict(num_ops=0), dict(num_ops=5), dict(num_ops=1.5), dict(magnitude=31), dict(magnitude=-1),
                dict(num_magnitude_bins=1), dict(num_ops=True)):
        with pytest.raises(ValueError):
            RandAugment(**bad)
    with pytest.raises(ValueError, match="num_magnitude_bins"):
        TrivialAugmentWide(num_magnitude_bins=1)
    er = RandomErasing()
    assert (er.p, er.scale, er.ratio, er.value) == (0.5, (0.02, 0.33), (0.3, 3.3), [0.0])
    assert RandomErasing(value="random").random
    for bad in (dict(p=1.5), dict(p=-0.1), dict(scale=(0.5, 0.2)), dict(scale=(0.1, 1.5)), dict(ratio=(0.0, 1.0)),
                dict(value="noise"), dict(value=[0.0] * 5), dict(value=float("nan"))):
        with pytest.raises(ValueError):
            RandomErasing(**bad)


def test_device_augment_validates_policy_and_erasing():
    with pytest.raises(ValueError, match="policy must be"):
        DeviceImageAugment("x", ["y"], policy="ta_wide")
    with pytest.raises(ValueError, match="erasing must be"):
        DeviceImageAugment("x", ["y"], erasing=0.25)
    aug = DeviceImageAugment("x", ["y"], out_size=32, policy=TrivialAugmentWide())
    aug.check_image(3, 40, 40)
    aug.check_image(1, 40, 40)
    for c in (2, 4):
        with pytest.raises(ValueError, match="1- or 3-channel"):
            aug.check_image(c, 40, 40)
    er = DeviceImageAugment("x", ["y"], out_size=32, erasing=RandomErasing(value=(0.1, 0.2)))
    with pytest.raises(ValueError, match="2 entries for 3-channel"):
        er.check_image(3, 40, 40)
    er.check_image(2, 40, 40)


def test_shared_memory_refusal():
    # 3 x 256 x 256 fits, the first square size over the budget does not
    assert 3 * 256 * 256 <= _native.POLICY_SMEM_BYTES
    side = int((_native.POLICY_SMEM_BYTES // 3) ** 0.5) + 1
    DeviceImageAugment("x", ["y"], out_size=256, policy=RandAugment()).check_image(3, 300, 300)
    with pytest.raises(ValueError, match="does not fit one CTA's shared memory"):
        DeviceImageAugment("x", ["y"], out_size=side, policy=RandAugment()).check_image(3, 300, 300)
    # the C library refuses the same size before touching any pointer, and accepts the budget itself
    lib = _native.lib()
    args = lambda oh, ow: (None, 4, 3, 300, 300, None, 0, 0, _native.AUG_RRC, 0.08, 1.0, 0.75, 4 / 3, 0, 1,  # noqa
                           _native.POLICY_TRIVIAL_AUGMENT, 1, 0, 31, None, 0.0, 0.02, 0.33, 0.3, 3.3, 0, None, None,
                           None, None, _native.F32, oh, ow, None, None, None)
    assert lib.frl_augment_policy_images(*args(side, side)) == -1
    assert b"shared memory" in lib.frl_last_error()
    # batch 0 after every check passes: returns 0 without a launch
    ok = list(args(256, 256))
    ok[1] = 0
    assert lib.frl_augment_policy_images(*ok) == 0


def test_c_argument_errors_are_reported_without_a_gpu():
    lib = _native.lib()

    def call(name="frl_augment_policy_images", **kw):
        a = dict(src=None, batch=4, C=3, H=40, W=40, idx=None, seed=0, epoch=0, mode=_native.AUG_RRC, smin=0.08,
                 smax=1.0, rmin=0.75, rmax=4 / 3, pad=0, flip=1, policy=_native.POLICY_RAND_AUGMENT, num_ops=2,
                 magnitude=9, num_bins=31, mags=None, ep=0.0, esmin=0.02, esmax=0.33, ermin=0.3, ermax=3.3, er=0,
                 ev=None, sc=None, bi=None, dst=None, dtype=_native.F32, oh=32, ow=32, po=None, pol=None)
        a.update(kw)
        rc = getattr(lib, name)(*a.values(), None)
        return rc, lib.frl_last_error().decode()

    cases = [(dict(mode=_native.AUG_CENTER_RESIZE), "mode must be"), (dict(C=4), "1 or 3 channels"),
             (dict(policy=7), "unknown policy"), (dict(num_ops=5), "num_ops must be in"),
             (dict(policy=_native.POLICY_TRIVIAL_AUGMENT, num_ops=2), "one op"),
             (dict(magnitude=31), "magnitude must be"), (dict(num_bins=1), "num_bins"),
             (dict(ep=1.5), "erase_p"), (dict(ep=0.5, esmin=0.5, esmax=0.2), "erase scale"),
             (dict(ep=0.5, ermin=0.0), "erase ratio"), (dict(policy=0, C=4), "1 to 3 channels"),
             (dict(dtype=_native.U8), "dst dtype")]
    for kw, msg in cases:
        rc, err = call(**kw)
        assert rc < 0 and msg in err, (kw, rc, err)
    rc = lib.frl_mix_images(None, _native.F32, 4, 3, 8, 8, 3, 0.5, 0, 0, 0, 0, None)
    assert rc < 0 and b"mix_mode" in lib.frl_last_error()
    rc = lib.frl_mix_images_nhwc(None, _native.F32, 4, 3, 8, 8, _native.MIX_CUTMIX, 0.5, 0, 9, 0, 4, None)
    assert rc < 0 and b"CutMix box" in lib.frl_last_error()


@pytest.mark.parametrize("size", [(224, 224), (32, 32), (160, 96), (256, 300)])
def test_magnitude_tables_equal_torchvision(size):
    tv = pytest.importorskip("torchvision.transforms.v2")
    h, w = size
    for ours, theirs in ((TrivialAugmentWide(), tv.TrivialAugmentWide()), (RandAugment(), tv.RandAugment()),
                         (TrivialAugmentWide(num_magnitude_bins=11), tv.TrivialAugmentWide(num_magnitude_bins=11))):
        table = ours.magnitudes(h, w)
        assert table.dtype == torch.float32 and table.shape == (14, ours.num_magnitude_bins)
        names = list(theirs._AUGMENTATION_SPACE)
        assert tuple(names) == POLICY_OPS
        for k, name in enumerate(names):
            fn, _ = theirs._AUGMENTATION_SPACE[name]
            ref = fn(ours.num_magnitude_bins, h, w)
            if ref is None:
                assert not table[k].any(), name
            else:
                assert torch.equal(table[k], ref.float()), name


def test_restated_draws_pinned():
    idx = np.array([0, 1, 7, 123456789012, 2 ** 40 + 5])
    ta = policy_np.policy_ops(idx, seed=1234, epoch=3, policy=policy_np.TRIVIAL_AUGMENT, num_ops=1, num_bins=31)
    ra = policy_np.policy_ops(idx, seed=1234, epoch=3, policy=policy_np.RAND_AUGMENT, num_ops=3, num_bins=31,
                              magnitude=9)
    er = policy_np.erase_boxes(idx, seed=1234, epoch=3, out_h=224, out_w=224, p=0.75)
    # the restatement's own invariants
    for t in (ta, ra):
        assert ((t[..., 0] >= 0) & (t[..., 0] < 14)).all()
        assert (t[..., 2][~np.isin(t[..., 0], list(policy_np.SIGNED))] == 1).all()
        assert (t[..., 1][np.isin(t[..., 0], list(policy_np.NO_MAGNITUDE))] == 0).all()
    assert (ra[..., 1][~np.isin(ra[..., 0], list(policy_np.NO_MAGNITUDE))] == 9).all()
    ok = er[:, 0] == 1
    assert ((er[ok, 1] + er[ok, 3] <= 224) & (er[ok, 2] + er[ok, 4] <= 224)).all()
    # pinned values on fixed keys (a change of the draw algorithm changes these)
    assert ta.reshape(-1, 3).tolist() == PINNED_TA
    assert ra[:, :, 0].tolist() == PINNED_RA_OPS
    assert er.tolist() == PINNED_ERASE
    # TrivialAugmentWide's op k = 0 is RandAugment's first op: the same block
    assert (ta[:, 0, 0] == ra[:, 0, 0]).all()


def test_restated_draws_cover_the_space():
    idx = np.arange(20000)
    ta = policy_np.policy_ops(idx, seed=5, epoch=1, policy=policy_np.TRIVIAL_AUGMENT, num_ops=1, num_bins=31)[:, 0]
    seen = {tuple(r) for r in ta.tolist()}
    want = {(0, 0, 1), (12, 0, 1), (13, 0, 1)} | {(o, b, 1) for o in (10, 11) for b in range(31)} | \
        {(o, b, s) for o in range(1, 10) for b in range(31) for s in (-1, 1)}
    assert seen == want
    counts = np.bincount(ta[:, 0], minlength=14) / len(idx)
    assert np.all(np.abs(counts - 1 / 14) < 0.01)
    er = policy_np.erase_boxes(idx, seed=5, epoch=1, out_h=64, out_w=64, p=0.5)
    assert abs(er[:, 0].mean() - 0.5) < 0.02


def test_mix_over_a_policy_batch_uses_frl_mix_images(monkeypatch):
    calls = []
    aug = DeviceImageAugment("x", ["y"], out_size=8, policy=TrivialAugmentWide(),
                             mix=BatchMix({"y": 4}, cutmix_alpha=1.0))
    monkeypatch.setattr(aug, "augment_policy", lambda x, index, out_dtype: calls.append("k5p") or x.float())
    monkeypatch.setattr(aug, "mix_targets", lambda raw, lam: [])
    monkeypatch.setattr(_native, "mix_images", lambda out, **kw: calls.append(("mix", kw["mix_mode"])))
    from frl_b200.types import Split
    x = torch.zeros(4, 3, 8, 8, dtype=torch.uint8)
    aug.apply({"x": x, "y": torch.zeros(4, dtype=torch.int64)}, Split.TRAIN, torch.float32,
              index=torch.arange(4))
    assert calls == ["k5p", ("mix", BatchMix.CUTMIX)]


PINNED_TA = [[5, 22, -1], [0, 0, 1], [4, 21, -1], [8, 8, -1], [12, 0, 1]]
PINNED_RA_OPS = [[5, 2, 13], [0, 4, 8], [4, 9, 12], [8, 4, 7], [12, 4, 13]]
PINNED_ERASE = [[1, 105, 28, 43, 89], [0, 0, 0, 0, 0], [1, 130, 46, 55, 156], [1, 25, 98, 46, 99], [1, 123, 18, 65, 195]]
