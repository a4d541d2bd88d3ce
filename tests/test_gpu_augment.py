"""K5a (frl_augment_images) and DeviceImageAugment on the GPU: the drawn boxes against the numpy
restatement (oracle/augment_np.py), the pixels against torchvision's functional transforms, the
fused normalisation against K5, independence of batch size / order, and the batched loader and
Solver.solve over an augmenting ResNet Problem."""
import logging
import tempfile

import numpy as np
import pytest
import torch
import torchvision.transforms.v2.functional as TF
from torchvision.transforms import InterpolationMode

import frl_b200  # noqa: F401
from frl_b200 import _native, synthetic
from frl_b200.device_loader import DeviceBatchLoader
from frl_b200.solver import Solver
from frl_b200.transform import DeviceBatchTransform
from frl_b200.types import Precision, Split
from oracle import augment_np as A

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


def _images(n, c, h, w, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (n, c, h, w), generator=g, dtype=torch.uint8)


def _run(x, idx, out_hw, *, mode, seed=0, epoch=0, pad=0, dtype=torch.float32, scale=None, bias=None, **kw):
    """K5a on the host tensors ``x`` [B, C, H, W] / ``idx`` [B]; returns (out, params) on the host."""
    xd = x.to(DEV).contiguous()
    idx_d = torch.as_tensor(idx, dtype=torch.int64).to(DEV)
    out = torch.full((x.shape[0], x.shape[1]) + tuple(out_hw), float("nan"), dtype=dtype, device=DEV)
    params = torch.full((x.shape[0], 5), -7, dtype=torch.int32, device=DEV)
    _native.augment_images(xd, idx_d, out, seed=seed, epoch=epoch, mode=mode, pad=pad, scale=scale, bias=bias,
                           params_out=params, **kw)
    torch.cuda.synchronize()
    return out.cpu(), params.cpu().numpy()


def _near_tie(raw):
    frac = raw - np.floor(raw)
    return (np.abs(frac - 0.5) < 1e-6).any(1)


# ---- 1. parameters against the restatement -----------------------------------------------------

@pytest.mark.parametrize("mode", [A.RRC, A.PAD_CROP])
def test_params_equal_the_numpy_restatement(mode):
    B = 4096
    H, W, out, pad = (256, 256, 224, 0) if mode == A.RRC else (40, 40, 32, 4)
    x = torch.zeros(B, 1, H, W, dtype=torch.uint8)
    idx = np.random.RandomState(1).randint(0, 1 << 40, size=B)
    ties = 0
    for epoch in (0, 1, 2):
        _, got = _run(x, idx, (out, out), mode=mode, seed=0x123456789ABC, epoch=epoch, pad=pad)
        want, raw, _ = A.sample_params(idx, seed=0x123456789ABC, epoch=epoch, mode=mode, height=H, width=W,
                                       out_h=out, out_w=out, pad=pad, with_raw=True)
        exempt = _near_tie(raw)
        ties += int(exempt.sum())
        bad = np.nonzero((got != want).any(1) & ~exempt)[0]
        assert bad.size == 0, (epoch, bad[:5], got[bad[:5]], want[bad[:5]])
    assert ties <= 3


def test_params_of_small_and_odd_images():
    for (H, W, oh, ow), ratio, scale in (((17, 23, 8, 5), (3 / 4, 4 / 3), (0.08, 1.0)),
                                         ((10, 100, 8, 8), (0.5, 2.0), (0.9, 1.0)),       # always the fallback
                                         ((1, 1, 3, 3), (3 / 4, 4 / 3), (0.08, 1.0))):
        idx = np.arange(2048)
        x = torch.zeros(idx.size, 1, H, W, dtype=torch.uint8)
        _, got = _run(x, idx, (oh, ow), mode=A.RRC, seed=7, epoch=3, scale_range=scale, ratio_range=ratio)
        want, raw, _ = A.sample_params(idx, seed=7, epoch=3, mode=A.RRC, height=H, width=W, out_h=oh, out_w=ow,
                                       scale=scale, ratio=ratio, with_raw=True)
        ok = ~_near_tie(raw)
        assert (got[ok] == want[ok]).all(), (H, W)


# ---- 2. pixels against torchvision ---------------------------------------------------------------

SHAPES = [  # C, H, W, out_h, out_w, mode, pad
    (3, 256, 256, 224, 224, A.RRC, 0),
    (3, 40, 40, 32, 32, A.PAD_CROP, 4),
    (1, 17, 23, 8, 5, A.RRC, 0),
    (4, 17, 23, 8, 5, A.PAD_CROP, 2),
    (4, 64, 48, 40, 40, A.RRC, 0),
    (1, 32, 32, 32, 32, A.PAD_CROP, 4),
]


def _torchvision(x, p, out_hw):
    top, left, h, w, flipped = (int(v) for v in p)
    y = TF.resized_crop(x.float(), top, left, h, w, list(out_hw), interpolation=InterpolationMode.BILINEAR,
                        antialias=False)
    return y.flip(-1) if flipped else y


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "C%d_%dx%d_to_%dx%d_mode%d" % s[:6])
def test_pixels_match_torchvision(shape):
    C, H, W, oh, ow, mode, pad = shape
    n = 48
    x = _images(n, C, H, W, seed=C * 1000 + H)
    idx = np.arange(n) * 977 + 5
    got, params = _run(x, idx, (oh, ow), mode=mode, seed=11, epoch=1, pad=pad)
    assert params[:, 4].min() == 0 and params[:, 4].max() == 1          # both flip states seen
    for b in range(n):
        want = _torchvision(x[b], params[b], (oh, ow))
        if mode == A.PAD_CROP or tuple(params[b, 2:4]) == (oh, ow):
            assert torch.equal(got[b], want), b                      # an exact copy, zero fill included
        else:
            torch.testing.assert_close(got[b], want, atol=1e-3, rtol=0)


def test_box_the_size_of_the_output_is_copied_bit_for_bit():
    x = _images(64, 3, 48, 48, seed=3)
    got, params = _run(x, np.arange(64), (48, 48), mode=A.RRC, scale_range=(1.0, 1.0), ratio_range=(1.0, 1.0))
    assert (params[:, :4] == [0, 0, 48, 48]).all()
    want = torch.stack([x[b].float().flip(-1) if params[b, 4] else x[b].float() for b in range(64)])
    assert torch.equal(got, want)


# ---- 3. normalisation ----------------------------------------------------------------------------

@pytest.mark.parametrize("mode", [A.RRC, A.PAD_CROP, A.CENTER_RESIZE])
def test_fused_affine_equals_k5_after_k5a(mode):
    C, H, oh = 3, 72, 64
    x = _images(32, C, H, H, seed=5)
    sc = torch.tensor([1 / (255 * 0.229), 1 / (255 * 0.224), 1 / (255 * 0.225)], device=DEV)
    bi = torch.tensor([-0.485 / 0.229, -0.456 / 0.224, -0.406 / 0.225], device=DEV)
    idx = np.arange(32) + 100
    kw = dict(mode=mode, seed=2, epoch=4, pad=4)
    plain, p0 = _run(x, idx, (oh, oh), **kw)
    fused, p1 = _run(x, idx, (oh, oh), scale=sc, bias=bi, **kw)
    fused16, p2 = _run(x, idx, (oh, oh), scale=sc, bias=bi, dtype=torch.bfloat16, **kw)
    assert (p0 == p1).all() and (p0 == p2).all()
    k5 = torch.empty(plain.shape, device=DEV)
    _native.preproc_affine(plain.to(DEV), k5, inner=oh * oh, channels=C, scale=sc, bias=bi)
    assert torch.equal(fused, k5.cpu())
    assert torch.equal(fused16.view(torch.int16), fused.to(torch.bfloat16).view(torch.int16))


# ---- 4. independence -----------------------------------------------------------------------------

@pytest.mark.parametrize("mode", [A.RRC, A.PAD_CROP])
def test_same_sample_same_image_in_any_batch(mode):
    N = 256
    x = _images(N, 3, 40, 40, seed=9)
    kw = dict(mode=mode, seed=3, epoch=2, pad=4, dtype=torch.bfloat16)
    full, pfull = _run(x, np.arange(N), (32, 32), **kw)
    rs = np.random.RandomState(0)
    for size in (1, 7, 256):
        rows = rs.permutation(N)[:size]
        got, p = _run(x[rows], rows, (32, 32), **kw)
        assert torch.equal(got.view(torch.int16), full[rows].view(torch.int16)), size
        assert (p == pfull[rows]).all()
    for other in (dict(kw, epoch=3), dict(kw, seed=4)):
        _, p = _run(x, np.arange(N), (32, 32), **other)
        assert (p != pfull).any(1).mean() > 0.5


def test_centre_crop_is_fixed_and_matches_torchvision():
    x = _images(16, 3, 256, 240, seed=1)
    idx = np.arange(16)
    a, pa = _run(x, idx, (200, 200), mode=A.CENTER_RESIZE, epoch=1, flip=True)
    b, pb = _run(x, idx, (200, 200), mode=A.CENTER_RESIZE, epoch=9, seed=5, flip=True)
    assert torch.equal(a, b) and (pa == pb).all() and (pa[:, 4] == 0).all()
    ch, cw = round(256 * 0.875), round(240 * 0.875)
    for i in range(16):
        want = TF.resize(TF.center_crop(x[i].float(), [ch, cw]), [200, 200],
                         interpolation=InterpolationMode.BILINEAR, antialias=False)
        torch.testing.assert_close(a[i], want, atol=1e-3, rtol=0)
    c, pc = _run(x, idx, (224, 224), mode=A.CENTER_CROP, epoch=2, flip=True)
    for i in range(16):
        assert torch.equal(c[i], TF.center_crop(x[i].float(), [224, 224]))


# ---- 5. loader and loop --------------------------------------------------------------------------

def _augmenting_problem(ns, folder, n_train=64, n_test=32):
    return synthetic.make_resnet_problem(ns, folder, "resnet18", uint8=True, augment="rrc", stored_image=72,
                                         image=64, n_train=n_train, n_test=n_test)


def _epoch(loader, seed):
    torch.manual_seed(seed)
    return [(d[0].cpu(), m["index"].cpu()) for d, _, m in loader]


def test_loader_epoch_is_what_a_resumed_run_sees(ns):
    folder = tempfile.mkdtemp(prefix="frl_b200_aug_")
    train = _augmenting_problem(ns, folder).datasets[0]
    ld = DeviceBatchLoader(train, batch_size=16, sampler=None, device=DEV, out_dtype=torch.bfloat16)
    ld.set_epoch(1)
    first = _epoch(ld, 0)
    ld.set_epoch(2)
    second = _epoch(ld, 1)
    fresh_train = _augmenting_problem(ns, folder).datasets[0]
    fresh = DeviceBatchLoader(fresh_train, batch_size=16, sampler=None, device=DEV, out_dtype=torch.bfloat16)
    fresh.set_epoch(2)
    again = _epoch(fresh, 1)
    assert len(second) == len(again) == 4
    for (x0, i0), (x1, i1) in zip(second, again):
        assert torch.equal(i0, i1) and torch.equal(x0.view(torch.int16), x1.view(torch.int16))
    # keyed by sample: the same index in epoch 1 got another box
    pos1 = {int(i): (b, k) for b, (_, ids) in enumerate(first) for k, i in enumerate(ids)}
    differ = 0
    for x2, ids in second:
        for k, i in enumerate(ids):
            b, k1 = pos1[int(i)]
            differ += not torch.equal(x2[k], first[b][0][k1])
    assert differ > 48
    # and each batch is the transform applied to its indices
    x2, ids = second[0]
    direct = train.device_transform.augment(train.pinned_fields["x"][ids].to(DEV), ids.to(DEV), Split.TRAIN,
                                            torch.bfloat16)
    assert torch.equal(direct.cpu().view(torch.int16), x2.view(torch.int16))


def test_solve_augmenting_resnet_on_the_device_path(ns, caplog):
    folder = tempfile.mkdtemp(prefix="frl_b200_aug_")
    problem = _augmenting_problem(ns, folder)
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
    try:
        torch.manual_seed(0)
        with caplog.at_level(logging.INFO):
            list(Solver.solve(run_opts, problem, group_name=None, init_method="file:///tmp/unused",
                              precision=Precision.BF16))
    finally:
        Solver.build_worker = classmethod(orig)
    text = "\n".join(r.getMessage() for r in caplog.records)
    assert "per-sample DataLoader" not in text
    assert "input path for split training: batched device loader" in text
    assert "input path for split testing: batched device loader" in text
    hist = captured["worker"].loss_history
    assert {(e, s) for e, s, _ in hist} == {(1, Split.TEST), (1, Split.TRAIN), (2, Split.TEST), (2, Split.TRAIN)}
    assert all(v.size > 0 and np.isfinite(v).all() for _, _, v in hist)
    assert problem.datasets[0].device_transform.epoch == 2


def test_existing_transforms_are_called_without_index(ns):
    calls = []

    class Recording(DeviceBatchTransform):
        def apply(self, raw, split, out_dtype):           # no index parameter: must not receive one
            calls.append(split)
            return [raw["x"].to(out_dtype)], [(raw["y_reg"],), (raw["y_cls"],)]

    problem = synthetic.make_toy_problem(ns, tempfile.mkdtemp(), n_train=64, n_test=16, pinned=True)
    ds = problem.datasets[0]
    plain = DeviceBatchLoader(ds, batch_size=16, sampler=None, device=DEV)
    plain.set_epoch(3)                                     # forwarded to the base class's no-op
    n = sum(1 for _ in plain)
    ds.device_transform = Recording()
    rec = DeviceBatchLoader(ds, batch_size=16, sampler=None, device=DEV)
    rec.set_epoch(1)
    assert sum(1 for _ in rec) == n == 4 and calls == [Split.TRAIN] * 4
