"""K5p on the GPU (``frl_augment_policy_images``, ``frl_mix_images``): every (op, bin, sign) of
TrivialAugmentWide against torchvision v2's own ``_apply_image_or_video_transform`` on the float-path
crop, RandAugment chains, layouts and dtypes, draw stability, random erasing, mixing over policy
images, and a short channels_last ``Solver.solve`` of the augmenting resnet18 Problem.

Exactness: a pixel may differ from torchvision only where a float64 restatement of the op puts the
quantity being decided within 1e-3 of a rounding, floor or truncation boundary (the source
coordinate of a geometric op, the blur of Sharpness, the value before the cast of a colour op);
such excused pixels are counted and bounded at 0.1 %."""
import logging
import math
import tempfile

import numpy as np
import pytest
import torch

import frl_b200  # noqa: F401
import policy_np
from frl_b200 import _native, criteria, synthetic
from frl_b200.device_loader import DeviceBatchLoader
from frl_b200.solver import Solver
from frl_b200.transform import POLICY_OPS, BatchMix, RandAugment, RandomErasing, TrivialAugmentWide
from frl_b200.types import Precision, Split

tv = pytest.importorskip("torchvision.transforms.v2")
TF = pytest.importorskip("torchvision.transforms.v2.functional")

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
SEED = 17
NEAR = 1e-3


def _inputs(B, H=80, W=80, seed=0):
    g = torch.Generator().manual_seed(seed)
    # smooth images with some flat regions, so colour statistics and equalize see real histograms
    base = torch.randint(0, 256, (B, 3, H // 8, W // 8), generator=g).float()
    x = torch.nn.functional.interpolate(base, size=(H, W), mode="bilinear", align_corners=False)
    x = (x + torch.randint(-20, 21, (B, 3, H, W), generator=g)).clamp(0, 255).to(torch.uint8)
    idx = torch.randint(0, 1 << 40, (B,), generator=g)
    return x.to(DEV), idx.to(DEV)


def _run(x, idx, out_hw=(64, 64), *, policy=None, erasing=None, dtype=torch.float32, epoch=1, nhwc=False,
         scale=None, bias=None, mode=_native.AUG_RRC):
    B = x.shape[0]
    out = torch.empty((B, x.shape[1]) + out_hw, dtype=dtype, device=DEV,
                      memory_format=torch.channels_last if nhwc else torch.contiguous_format)
    n_ops = 0 if policy is None else policy.num_ops
    params = torch.full((B, 5), -7, dtype=torch.int32, device=DEV)
    pol_out = torch.full((B, 3 * n_ops + 5), -7, dtype=torch.int32, device=DEV)
    ev = None
    if erasing is not None and not erasing.random:
        ev = torch.tensor(erasing.values(x.shape[1]), dtype=torch.float32, device=DEV)
    _native.augment_policy_images(
        x, idx, out, seed=SEED, epoch=epoch, mode=mode, pad=4, flip=True,
        policy=_native.POLICY_NONE if policy is None else policy.native, num_ops=1 if policy is None else n_ops,
        magnitude=0 if policy is None else policy.magnitude,
        mags=None if policy is None else policy.magnitudes(*out_hw).to(DEV),
        erase_p=0.0 if erasing is None else erasing.p, erase_scale=(0.02, 0.33) if erasing is None else erasing.scale,
        erase_ratio=(0.3, 3.3) if erasing is None else erasing.ratio,
        erase_random=erasing is not None and erasing.random, erase_value=ev,
        scale=None if scale is None else torch.tensor(scale, device=DEV),
        bias=None if bias is None else torch.tensor(bias, device=DEV), params_out=params, policy_out=pol_out)
    return out, params.cpu(), pol_out.cpu()


def _crop(x, box, out_hw):
    """The float-path crop torchvision makes on a CUDA tensor, rounded to uint8, flipped."""
    top, left, h, w, flipped = (int(v) for v in box)
    c = TF.resized_crop(x.float(), top, left, h, w, list(out_hw), antialias=False).round_().to(torch.uint8)
    return c.flip(-1) if flipped else c


# ---- float64 restatement: where does an op decide near a boundary? ------------------------------------------

def _near_int(v):
    return np.abs(v - np.rint(v)) < NEAR


def _near_half(v):
    return np.abs(v - np.floor(v) - 0.5) < NEAR


def _affine_src(op, m, H, W):
    """float64 source (x, y) of every output pixel of an index-map op (torchvision's formula)."""
    if op in ("ShearX", "ShearY"):
        sh = math.degrees(math.atan(m))
        shear = [sh, 0.0] if op == "ShearX" else [0.0, sh]
        mat = TF._geometry._get_inverse_affine_matrix([-0.5 * W, -0.5 * H], 0.0, [0.0, 0.0], 1.0, shear)
    elif op in ("TranslateX", "TranslateY"):
        t = [float(int(m)), 0.0] if op == "TranslateX" else [0.0, float(int(m))]
        mat = TF._geometry._get_inverse_affine_matrix([0.0, 0.0], 0.0, t, 1.0, [0.0, 0.0])
    else:
        mat = TF._geometry._get_inverse_affine_matrix([0.0, 0.0], -(m % 360), [0.0, 0.0], 1.0, [0.0, 0.0])
    ys, xs = np.meshgrid(np.arange(H) - (H - 1) / 2, np.arange(W) - (W - 1) / 2, indexing="ij")
    sx = mat[0] * xs + mat[1] * ys + mat[2] + (W - 1) / 2
    sy = mat[3] * xs + mat[4] * ys + mat[5] + (H - 1) / 2
    return sx, sy


def _near_mask(img, op, m):
    """bool [H, W]: pixels whose float64 restatement decides within 1e-3 of a boundary."""
    a = img.cpu().numpy().astype(np.float64)
    C, H, W = a.shape
    near = np.zeros((H, W), bool)
    if op in ("ShearX", "ShearY", "TranslateX", "TranslateY", "Rotate"):
        sx, sy = _affine_src(op, m, H, W)
        return _near_half(sx) | _near_half(sy)
    f = 1.0 + m
    gray = (0.2989 * a[0] + 0.587 * a[1] + 0.114 * a[2]) if C == 3 else a[0]
    if op == "Brightness":
        near = _near_int(a * f).any(0)
    elif op == "Color" and C == 3:
        g = np.floor(gray)
        near = _near_int(gray) | _near_int(a * f + (1 - f) * g).any(0)
    elif op == "Contrast":
        mean = np.floor(gray).mean() if C == 3 else gray.mean()
        near = (_near_int(gray) if C == 3 else near) | _near_int(a * f + (1 - f) * mean).any(0)
    elif op == "Sharpness" and H > 2 and W > 2:
        k = np.full((3, 3), 1 / 13)
        k[1, 1] = 5 / 13
        inner = np.zeros((C, H - 2, W - 2))
        for dy in range(3):
            for dx in range(3):
                inner += k[dy, dx] * a[:, dy:dy + H - 2, dx:dx + W - 2]
        v = a[:, 1:-1, 1:-1] + (1 - f) * (np.rint(inner) - a[:, 1:-1, 1:-1])
        near[1:-1, 1:-1] = (_near_half(inner) | _near_int(v)).any(0)
    elif op == "AutoContrast":
        lo, hi = a.min((1, 2), keepdims=True), a.max((1, 2), keepdims=True)
        v = np.where(hi > lo, (a - lo) / np.where(hi > lo, (hi - lo) / 255.0, 1.0), a)
        near = (_near_int(v) & (hi > lo)).any(0)
    return near


def _oracle(crop, ops, mags_table, tvpol):
    """torchvision's chain on the crop; returns the image and the OR of each op's near mask."""
    img = crop
    near = np.zeros(crop.shape[1:], bool)
    for op, b, sign in ops:
        name = POLICY_OPS[op]
        m = float(mags_table[op, b]) * sign if op not in (0, 12, 13) else 0.0
        near |= _near_mask(img, name, m)
        img = tvpol._apply_image_or_video_transform(img, name, m, interpolation=tv.InterpolationMode.NEAREST,
                                                    fill=tvpol._fill)
    return img, near


def test_trivial_augment_every_op_bin_and_sign_equals_torchvision():
    pol, tvpol = TrivialAugmentWide(), tv.TrivialAugmentWide()
    mags = pol.magnitudes(64, 64)
    want = {(0, 0, 1), (12, 0, 1), (13, 0, 1)} | {(o, b, 1) for o in (10, 11) for b in range(31)} | \
        {(o, b, s) for o in range(1, 10) for b in range(31) for s in (-1, 1)}
    seen, per_op = set(), {}
    excused = total = 0
    x, idx = _inputs(1024)
    xc = x.cpu()
    for epoch in range(1, 13):
        out, params, pol_out = _run(x, idx, policy=pol, epoch=epoch)
        got = out.cpu()
        assert torch.equal(got, got.round()) and got.min() >= 0 and got.max() <= 255
        got = got.to(torch.uint8)
        for s in range(x.shape[0]):
            key = tuple(pol_out[s, :3].tolist())
            if key in seen and per_op.get(key[0], 0) >= 40:
                continue
            seen.add(key)
            per_op[key[0]] = per_op.get(key[0], 0) + 1
            ref, near = _oracle(_crop(xc[s], params[s], (64, 64)), [key], mags, tvpol)
            diff = (ref != got[s]).any(0).numpy()
            assert not (diff & ~near).any(), (POLICY_OPS[key[0]], key, int((diff & ~near).sum()))
            excused += int(diff.sum())
            total += diff.size
        if seen >= want:
            break
    assert seen == want, f"not covered after {epoch} epochs: {sorted(want - seen)[:10]}"
    print(f"TrivialAugmentWide: {len(seen)} (op, bin, sign) covered in {epoch} epochs; "
          f"excused pixels {excused} of {total} ({100.0 * excused / total:.4f} %)")
    assert excused <= 1e-3 * total


@pytest.mark.parametrize("num_ops", [2, 3])
def test_rand_augment_chains_equal_torchvision(num_ops):
    pol = RandAugment(num_ops=num_ops)
    tvpol = tv.RandAugment(num_ops=num_ops)
    mags = pol.magnitudes(64, 64)
    x, idx = _inputs(384, seed=num_ops)
    out, params, pol_out = _run(x, idx, policy=pol)
    got = out.cpu().to(torch.uint8)
    xc = x.cpu()
    exact = flagged = flagged_diff = 0
    for s in range(x.shape[0]):
        ops = [tuple(pol_out[s, 3 * k:3 * k + 3].tolist()) for k in range(num_ops)]
        ref, near = _oracle(_crop(xc[s], params[s], (64, 64)), ops, mags, tvpol)
        same = torch.equal(ref, got[s])
        if not near.any():
            assert same, (s, ops)
            exact += 1
        else:
            flagged += 1
            flagged_diff += not same
    print(f"RandAugment({num_ops}, 9): {exact} samples without an excused pixel, all exact; {flagged} with "
          f"near-boundary decisions, {flagged_diff} of them differ")
    assert flagged_diff <= 0.05 * x.shape[0]


def test_policy_out_and_params_follow_the_restatement_and_k5a():
    x, idx = _inputs(256)
    er = RandomErasing(p=0.6)
    for pol in (TrivialAugmentWide(), RandAugment(num_ops=3)):
        _, params, pol_out = _run(x, idx, policy=pol, erasing=er, epoch=4)
        want = policy_np.policy_ops(idx.cpu().numpy(), seed=SEED, epoch=4, policy=pol.native, num_ops=pol.num_ops,
                                    num_bins=31, magnitude=pol.magnitude)
        assert pol_out[:, :3 * pol.num_ops].numpy().tolist() == want.reshape(256, -1).tolist()
        boxes = policy_np.erase_boxes(idx.cpu().numpy(), seed=SEED, epoch=4, out_h=64, out_w=64, p=0.6)
        assert pol_out[:, 3 * pol.num_ops:].numpy().tolist() == boxes.tolist()
        # the crop box and flip are K5a's, with or without the policy
        k5a = torch.empty((256, 3, 64, 64), device=DEV)
        p5 = torch.empty((256, 5), dtype=torch.int32, device=DEV)
        _native.augment_images(x, idx, k5a, seed=SEED, epoch=4, mode=_native.AUG_RRC, pad=4, flip=True,
                               params_out=p5)
        assert torch.equal(params, p5.cpu())
        _, params_off, _ = _run(x, idx, epoch=4)
        assert torch.equal(params, params_off)


@pytest.mark.parametrize("mode", [_native.AUG_RRC, _native.AUG_PAD_CROP])
def test_layouts_dtypes_and_batch_independence(mode):
    x, idx = _inputs(96, H=72, W=72)
    pol, er = RandAugment(num_ops=2), RandomErasing(p=0.7, value="random")
    sc, bi = synthetic.U8_CHANNEL_AFFINE
    kw = dict(policy=pol, erasing=er, scale=sc, bias=bi, mode=mode)
    hw = (64, 64)
    f32, _, _ = _run(x, idx, hw, **kw)
    f32_nhwc, _, _ = _run(x, idx, hw, nhwc=True, **kw)
    assert f32_nhwc.is_contiguous(memory_format=torch.channels_last)
    assert torch.equal(f32.cpu().view(torch.int32), f32_nhwc.contiguous().cpu().view(torch.int32))
    for nhwc in (False, True):
        bf, _, _ = _run(x, idx, hw, dtype=torch.bfloat16, nhwc=nhwc, **kw)
        assert torch.equal(bf.contiguous().cpu().view(torch.int16), f32.to(torch.bfloat16).cpu().view(torch.int16))
    # a sample's image does not depend on its batch or its place in it
    perm = torch.randperm(96, generator=torch.Generator().manual_seed(3))[:40].to(DEV)
    sub, _, _ = _run(x[perm].contiguous(), idx[perm].contiguous(), hw, **kw)
    assert torch.equal(sub.cpu(), f32.cpu()[perm.cpu()])


def test_erasing():
    x, idx = _inputs(512)
    pol = TrivialAugmentWide()
    base, _, _ = _run(x, idx, policy=pol)
    p0, _, _ = _run(x, idx, policy=pol, erasing=RandomErasing(p=0.0))
    assert torch.equal(base.cpu().view(torch.int32), p0.cpu().view(torch.int32))
    zero, _, pol_out = _run(x, idx, policy=pol, erasing=RandomErasing(p=1.0, value=0))
    boxes = pol_out[:, 3:]
    mask = torch.zeros(512, 1, 64, 64, dtype=torch.bool)
    for s, (e, t, l, h, w) in enumerate(boxes.tolist()):
        if e:
            mask[s, :, t:t + h, l:l + w] = True
    assert boxes[:, 0].float().mean() > 0.9
    mask = mask.expand(-1, 3, -1, -1)
    z, b = zero.cpu(), base.cpu()
    assert (z[mask] == 0).all() and torch.equal(z[~mask], b[~mask])
    rnd, _, pol_out_r = _run(x, idx, policy=pol, erasing=RandomErasing(p=1.0, value="random"))
    assert torch.equal(pol_out_r, pol_out)
    vals = rnd.cpu()[mask].double()
    n = vals.numel()
    assert n > 100000
    assert abs(vals.mean().item()) < 5.0 / math.sqrt(n)
    assert abs(vals.std().item() - 1.0) < 5.0 * math.sqrt(2.0 / n)
    assert torch.equal(rnd.cpu()[~mask], b[~mask])


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("nhwc", [False, True])
def test_mixing_policy_images(dtype, nhwc):
    x, idx = _inputs(33)
    sc, bi = synthetic.U8_CHANNEL_AFFINE
    kw = dict(policy=TrivialAugmentWide(), erasing=RandomErasing(p=0.5), scale=sc, bias=bi, dtype=dtype, nhwc=nhwc)
    plain = _run(x, idx, **kw)[0].contiguous().cpu().float()
    flip = torch.arange(32, -1, -1)
    for mode, lam, box in ((BatchMix.CUTMIX, 0.75, (8, 40, 20, 52)), (BatchMix.MIXUP, 0.3141, (0, 0, 0, 0))):
        out = _run(x, idx, **kw)[0]
        _native.mix_images(out, mix_mode=mode, lam=lam, box=box)
        got = out.contiguous().cpu().float()
        q = plain[flip]
        if mode == BatchMix.CUTMIX:
            y0, y1, x0, x1 = box
            want = plain.clone()
            want[:, :, y0:y1, x0:x1] = q[:, :, y0:y1, x0:x1]
            want[16] = plain[16]
            assert torch.equal(got, want)
        else:
            lam1 = np.float32(1.0 - lam)
            want = (np.float32(lam) * plain.numpy()).astype(np.float32) + (lam1 * q.numpy()).astype(np.float32)
            want = torch.from_numpy(want.astype(np.float32))
            want[16] = plain[16]
            want = want.to(dtype).float()
            ulp = torch.where(want == 0, torch.zeros_like(want),
                              want.abs() * (2.0 ** -7 if dtype == torch.bfloat16 else 2.0 ** -23))
            assert ((got - want).abs() <= ulp + 1e-30).all()


@pytest.fixture(scope="module")
def ns():
    return synthetic.api_namespace("frl_b200")


def _policy_problem(ns, folder, n_train=64, n_test=16):
    return synthetic.make_resnet_problem(ns, folder, "resnet18", uint8=True, augment="rrc", stored_image=40,
                                         image=32, n_train=n_train, n_test=n_test, mixup_alpha=0.8,
                                         policy="ta_wide", random_erasing=0.25)


def _epoch(loader, seed):
    torch.manual_seed(seed)
    return [(d[0].cpu(), [h[0].cpu() for h in tg], m["index"].cpu()) for d, tg, m in loader]


def test_loader_epochs_reproduce_and_resume(ns):
    folder = tempfile.mkdtemp(prefix="frl_b200_policy_")
    train = _policy_problem(ns, folder).datasets[0]
    aug = train.device_transform
    assert aug.policy is not None and aug.erasing is not None
    aug.memory_format = torch.channels_last
    ld = DeviceBatchLoader(train, batch_size=16, sampler=None, device=DEV, out_dtype=torch.bfloat16)
    ld.set_epoch(1)
    first = _epoch(ld, 0)
    fresh_train = _policy_problem(ns, folder).datasets[0]
    fresh_train.device_transform.memory_format = torch.channels_last
    fresh = DeviceBatchLoader(fresh_train, batch_size=16, sampler=None, device=DEV, out_dtype=torch.bfloat16)
    fresh.set_epoch(1)
    again = _epoch(fresh, 0)
    assert len(first) == len(again)
    for (x0, t0, i0), (x1, t1, i1) in zip(first, again):
        assert torch.equal(i0, i1) and torch.equal(x0.view(torch.int16), x1.view(torch.int16))
        assert all(torch.equal(u, v) for u, v in zip(t0, t1))


def test_solve_resnet18_channels_last_with_policy_erasing_and_mixup(ns, caplog):
    folder = tempfile.mkdtemp(prefix="frl_b200_policy_")
    problem = _policy_problem(ns, folder)
    t = ns.types
    run_opts = t.RunOpts(optim=t.OptimOpts(algo=t.OptAlgorithm("sgd"), lr=0.01), batchSize=16, nEpochs=2,
                         numThreads=0, singleThreaded=True, numVisualizedSamples=0)
    captured = {}
    orig = Solver.build_worker.__func__
    calls = {"k5p": 0}
    aug = problem.datasets[0].device_transform
    orig_policy = aug.augment_policy

    def counted(*a, **k):
        calls["k5p"] += 1
        return orig_policy(*a, **k)

    aug.augment_policy = counted

    def spy(cls, args):
        worker, sched, ckpt = orig(cls, args)
        captured["worker"] = worker
        return worker, sched, ckpt

    Solver.build_worker = classmethod(spy)
    criteria._path_logged.clear()
    try:
        torch.manual_seed(0)
        with caplog.at_level(logging.INFO):
            list(Solver.solve(run_opts, problem, group_name=None, init_method="file:///tmp/unused",
                              precision=Precision.BF16, channels_last=True))
    finally:
        Solver.build_worker = classmethod(orig)
    hist = captured["worker"].loss_history
    assert {(e, s) for e, s, _ in hist} == {(1, Split.TEST), (1, Split.TRAIN), (2, Split.TEST), (2, Split.TRAIN)}
    assert all(v.size > 0 and np.isfinite(v).all() for _, _, v in hist)
    assert calls["k5p"] >= 8          # 64 samples / 16 per batch, two epochs, on the batched device path
