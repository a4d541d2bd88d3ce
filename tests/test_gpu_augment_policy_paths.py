"""K5p (``frl_augment_policy_images`` and its ``_nhwc`` form, csrc/augment_policy.cu) at every output
geometry, channel count and crop mode it serves: TrivialAugmentWide and RandAugment pixels against
torchvision, NHWC / bf16 / channel-affine outputs against the fp32 NCHW output, and random-erasing
values against a float64 restatement of the header's Box-Muller.

Reference.  A sample's crop is torchvision's float-path crop rounded to uint8 and flipped (``_crop``
of test_gpu_augment_policy.py, on CPU tensors).  Each op is torchvision 0.26's own
``_apply_image_or_video_transform`` on that uint8 tensor (NEAREST, fill 0) at the magnitude that
torchvision's ``_AUGMENTATION_SPACE`` gives for the output's height and width, not at the package's
table, so a wrong TranslateX / TranslateY scale fails here.  The geometric ops stay on CPU tensors
because the kernel reproduces torch's CPU ``grid_sample`` roundings.

Exactness.  A pixel may differ from torchvision only where it is tainted.  A pixel is tainted when a
float64 restatement of an op puts the quantity that op decides within 1e-3 of a rounding, floor or
truncation boundary (``_near_mask`` of test_gpu_augment_policy.py).  It is also tainted when an
earlier tainted pixel reaches it: a geometric op moves the taint with the pixels, Sharpness spreads
it to the 3x3 neighbourhood, and a statistics op (Contrast, AutoContrast, Equalize) spreads it to the
whole image.  Every differing pixel is an excused pixel.  Excused pixels after the ops are bounded
at 0.1 % of the pixels compared per geometry and policy.

The crop is K5a's fp32 bilinear blend.  It agrees with torch's to an ulp or so, not bit for bit
(test_gpu_augment.py holds it to 1e-3), so its rounding to uint8 can differ where the value sits
that close to a half.  A crop pixel may differ from ``_crop`` only where the blend, restated in
float64 with the header's fp32 weights, is within 1e-3 of a half.  Such pixels are counted, and
torchvision's chain then starts from K5p's crop, so every op is compared on the same input.  Tiny
crops have weights near 1/2 and hit these ties often (0.9 % of the pixels at 3x3x7), so the 0.1 %
bound is on the ops alone.

Measured on an H100 80GB HBM3 at a 700 W power limit: excused pixels after the ops, of the pixels
compared, with the crop's excused pixels in brackets.

    geometry               TrivialAugmentWide            RandAugment (12 settings)
    3x48x80   RRC 96x96      2 of  2 392 320  (503)        0 of 1 105 920  (189)
    3x80x48   RRC 96x96      2 of    706 560  (114)        0 of 1 105 920  (180)
    1x37x53   RRC 45x60      0 of    360 824    (5)      223 of   564 768   (17)
    3x32x32   pad 4          0 of    188 416    (0)        0 of   294 912    (0)
    1x28x28   pad 2          0 of    144 256    (0)        0 of   225 792    (0)
    3x3x7     RRC 5x9        0 of      3 864   (34)        2 of     8 064   (61)
    1x2x9     RRC 4x12       0 of      3 312    (3)        0 of     6 912   (11)
    3x224x224 RRC 256x256   56 of 31 259 648  (166)        0 of 3 612 672   (23)
    3x256x292 RRC 288x320    0 of  1 719 296    (2)        0 of 1 794 048    (2)
    1x473x474 RRC 512x512  125 of  5 156 646    (5)        0 of 5 380 848   (18)

Inputs.  Smooth images, as in test_gpu_augment_policy.py, alternate with adversarial ones: a
constant image (Equalize's step == 0, AutoContrast's hi == lo), a two-level image, an image with
one constant channel, an image saturated at 0 and 255 (the Brightness clamp), a ramp that holds
every value 0..255 (each Solarize threshold 255*m that is an integer, compared with >=), and a
constant background with a few darker specks (Equalize's step == 0 on a large image).

Layouts.  The NHWC output equals the NCHW output permuted, the bf16 output equals the fp32 output
rounded to bf16, and with ``scale`` / ``bias`` the output equals fmaf(u8, scale[c], bias[c]).  The
last is restated as u8 * scale + bias in float64 and then rounded to fp32 once.  The product has at
most 8 + 24 significant bits and the sum spans fewer than 53, so float64 holds it exactly and the
single rounding is fmaf's.  All three are compared bit for bit.

Random erasing.  Element e = (c*h + y)*w + x of a sample's box takes block 32 + e/4, pair
j = (e/2) % 2: u1 = ((w_2j >> 8) + 1) 2^-24, u2 = (w_2j+1 >> 8) 2^-24, both exact in fp32.  The
kernel computes r = sqrtf(-2 logf(u1)) and r * (cos or sin)(2 pi u2) through sincospif.  CUDA's
logf and sincospif are within 1 ulp, so within 2^-23 relative.  Doubling is exact, and sqrtf
rounds correctly (no fast math), so r is within 2^-24 (halved log error) + 2^-24 (rounding)
= 2 * 2^-24 relative.  The cosine or sine adds 2 * 2^-24 relative, and the product's rounding adds
2^-24.  So |value - restated| <= 5 * 2^-24 * r, up to second-order terms and the restatement's own
float64 error.  The test allows 6 * 2^-24 * (r + 1).  It also checks that this bound rejects a
channel offset of c*w instead of c*h, channels that share values, a transposed box, and u1 without
its +1; the last moves r by about 2^-24 / (u1 r), far outside the bound when u1 is small.
"""
from typing import NamedTuple

import numpy as np
import pytest
import torch

import frl_b200  # noqa: F401
import policy_np
from frl_b200 import _native, synthetic
from frl_b200.transform import POLICY_OPS, RandAugment, RandomErasing, TrivialAugmentWide
from oracle import augment_np
from test_gpu_augment_policy import _crop, _near_half, _near_mask

tv = pytest.importorskip("torchvision.transforms.v2")

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
SEED = 29
EPOCH = 3
EXCUSED_SHARE = 1e-3
GEOMETRIC = {1, 2, 3, 4, 5}                 # ShearX .. Rotate
STATISTICS = {8, 12, 13}                    # Contrast, AutoContrast, Equalize
SHARPNESS = 9


class Geo(NamedTuple):
    C: int
    oh: int
    ow: int
    sh: int                  # source image
    sw: int
    mode: int = _native.AUG_RRC
    pad: int = 0
    per_key: int = 8         # TrivialAugmentWide samples per (op, sign); 0: one per (op, bin, sign)
    ra_batch: int = 24       # RandAugment samples per setting

    def __str__(self):
        crop = f"pad{self.pad}" if self.mode == _native.AUG_PAD_CROP else f"rrc{self.sh}x{self.sw}"
        return f"{self.C}x{self.oh}x{self.ow}-{crop}"


PAD = _native.AUG_PAD_CROP
G48x80 = Geo(3, 48, 80, 96, 96, per_key=0)
G80x48 = Geo(3, 80, 48, 96, 96)
G37x53 = Geo(1, 37, 53, 45, 60)
G32PAD = Geo(3, 32, 32, 32, 32, PAD, 4)
G28PAD = Geo(1, 28, 28, 28, 28, PAD, 2)
G3x7 = Geo(3, 3, 7, 5, 9, ra_batch=32)
G2x9 = Geo(1, 2, 9, 4, 12, ra_batch=32)
G224 = Geo(3, 224, 224, 256, 256, per_key=0, ra_batch=6)
G_CEIL = Geo(3, 256, 292, 288, 320, per_key=1, ra_batch=2)     # 224 256 B: FRL_AUGMENT_POLICY_SMEM_BYTES
G473 = Geo(1, 473, 474, 512, 512, per_key=1, ra_batch=2)
GEOS = [G48x80, G80x48, G37x53, G32PAD, G28PAD, G3x7, G2x9, G224, G_CEIL, G473]

# RandAugment (num_magnitude_bins, magnitude, num_ops): magnitude 0, the default 9 and the last bin
RA_SETTINGS = [(nb, m, k) for nb in (31, 11) for m in (0, 9, nb - 1) for k in (1, 4)]


def test_geometries_reach_the_shared_memory_ceiling():
    assert G_CEIL.C * G_CEIL.oh * G_CEIL.ow == _native.POLICY_SMEM_BYTES == 224256
    assert G473.C * G473.oh * G473.ow <= _native.POLICY_SMEM_BYTES
    assert G224.C * G224.oh * G224.ow > 48 * 1024


# ---- inputs ---------------------------------------------------------------------------------------------------

N_KINDS = 8


def _images(B, C, H, W, seed):
    """uint8 [B, C, H, W] on the CPU; sample s is of kind s % 8 (see the module docstring)."""
    g = torch.Generator().manual_seed(seed)
    base = torch.randint(0, 256, (B, C, max(H // 8, 1), max(W // 8, 1)), generator=g).float()
    smooth = torch.nn.functional.interpolate(base, size=(H, W), mode="bilinear", align_corners=False)
    smooth = (smooth + torch.randint(-20, 21, (B, C, H, W), generator=g)).clamp(0, 255)
    level = torch.randint(0, 256, (B, 2), generator=g)
    blocks = torch.nn.functional.interpolate(torch.randint(0, 2, (B, 1, max(H // 4, 1), max(W // 4, 1)),
                                                           generator=g).float(), size=(H, W), mode="nearest")
    ramp = torch.arange(H * W).view(H, W) % 256
    x = smooth.clone()
    for s in range(B):
        kind, k = s % N_KINDS, s // N_KINDS
        lo, hi = sorted(level[s].tolist())
        lo, hi = (254, 255) if lo == 255 else (lo, max(hi, lo + 1))
        if kind == 1:                                   # constant: 0, 255 or a random level
            x[s] = (0, 255, lo)[k % 3]
        elif kind == 2:                                 # two levels
            x[s] = lo + (hi - lo) * blocks[s]
        elif kind == 3:                                 # one constant channel
            x[s, k % C] = lo
        elif kind == 4:                                 # saturated at 0 and 255
            x[s] = (smooth[s] * 3.0 - 300.0).clamp(0, 255)
        elif kind == 5:                                 # every value, channels shifted
            x[s] = torch.stack([(ramp + 85 * c) % 256 for c in range(C)])
        elif kind == 6:                                 # a background and a few darker specks
            bg = 128 + hi % 128
            x[s] = bg
            n = min(64, max(H * W // 8, 1))
            pos = torch.randperm(H * W, generator=g)[:n]
            x[s].view(C, -1)[:, pos] = torch.randint(0, bg, (C, n), generator=g).float()
    return x.to(torch.uint8)


def _indices(n, seed):
    return torch.from_numpy(np.random.default_rng(seed).integers(0, 1 << 40, size=n))


def _run(geo, x, idx, *, policy=None, erasing=None, dtype=torch.float32, nhwc=False, scale=None, bias=None,
         epoch=EPOCH):
    """K5p on ``x`` / ``idx`` (device tensors); returns (out, params, policy_out), the last two on the CPU."""
    B = x.shape[0]
    hw = (geo.oh, geo.ow)
    out = torch.empty((B, geo.C) + hw, dtype=dtype, device=DEV,
                      memory_format=torch.channels_last if nhwc else torch.contiguous_format)
    n_ops = 0 if policy is None else policy.num_ops
    params = torch.full((B, 5), -7, dtype=torch.int32, device=DEV)
    pol_out = torch.full((B, 3 * n_ops + 5), -7, dtype=torch.int32, device=DEV)
    ev = None
    if erasing is not None and not erasing.random:
        ev = torch.tensor(erasing.values(geo.C), dtype=torch.float32, device=DEV)
    _native.augment_policy_images(
        x, idx, out, seed=SEED, epoch=epoch, mode=geo.mode, pad=geo.pad, flip=True,
        policy=_native.POLICY_NONE if policy is None else policy.native, num_ops=max(n_ops, 1),
        magnitude=0 if policy is None else policy.magnitude,
        mags=None if policy is None else policy.magnitudes(*hw).to(DEV),
        erase_p=0.0 if erasing is None else erasing.p, erase_scale=(0.02, 0.33) if erasing is None else erasing.scale,
        erase_ratio=(0.3, 3.3) if erasing is None else erasing.ratio,
        erase_random=erasing is not None and erasing.random, erase_value=ev,
        scale=None if scale is None else torch.tensor(scale, device=DEV),
        bias=None if bias is None else torch.tensor(bias, device=DEV), params_out=params, policy_out=pol_out)
    return out, params.cpu(), pol_out.cpu()


def _affine(C):
    sc, bi = synthetic.U8_CHANNEL_AFFINE
    return tuple(sc[:C]), tuple(bi[:C])


# ---- the torchvision reference ---------------------------------------------------------------------------------

def _tv_table(tvpol, num_bins, H, W):
    """fp32 [14, num_bins]: torchvision's own magnitudes for an H x W image (0 for no magnitude)."""
    rows = []
    for name in POLICY_OPS:
        m = tvpol._AUGMENTATION_SPACE[name][0](num_bins, H, W)
        rows.append(torch.zeros(num_bins) if m is None else m.float())
    return torch.stack(rows)


def _dilate(t):
    H, W = t.shape
    p = np.pad(t, 1)
    return np.logical_or.reduce([p[dy:dy + H, dx:dx + W] for dy in range(3) for dx in range(3)])


def _chain(crop, ops, table, tvpol):
    """torchvision's ops on the uint8 crop, and the bool [H, W] taint (see the module docstring)."""
    img = crop
    taint = np.zeros(crop.shape[1:], bool)
    for op, b, sign in ops:
        name = POLICY_OPS[op]
        m = float(table[op, b]) * sign
        near = _near_mask(img, name, m)
        if taint.any():
            if op in GEOMETRIC:
                t = torch.from_numpy(taint.astype(np.uint8))[None]
                taint = tvpol._apply_image_or_video_transform(t, name, m, interpolation=tv.InterpolationMode.NEAREST,
                                                              fill=tvpol._fill)[0].numpy().astype(bool)
            elif op == SHARPNESS:
                taint = _dilate(taint)
            elif op in STATISTICS:
                taint[:] = True
        taint = taint | near
        img = tvpol._apply_image_or_video_transform(img, name, m, interpolation=tv.InterpolationMode.NEAREST,
                                                    fill=tvpol._fill)
    return img, taint


def _crop_near(img, box, hw):
    """bool [oh, ow]: pixels whose crop value lies within 1e-3 of a half.  The source index and the
    weights are the header's fp32 ones; the blend is in float64."""
    top, left, h, w, flipped = (int(v) for v in box)
    a = img.numpy().astype(np.float64)
    C, H, W = a.shape

    def axis(out, crop, start, size):
        s = np.float32(crop) / np.float32(out)
        src = np.maximum((float(s) * (np.arange(out) + 0.5) - 0.5).astype(np.float32), np.float32(0.0))
        i0 = np.minimum(src.astype(np.int64), crop - 1)
        l1 = src - i0.astype(np.float32)
        taps = [start + i0, start + np.minimum(i0 + 1, crop - 1)]
        return [(np.clip(t, 0, size - 1), (t >= 0) & (t < size)) for t in taps], \
            (np.float32(1.0) - l1).astype(np.float64), l1.astype(np.float64)

    (ry0, ry1), hy0, ly = axis(hw[0], h, top, H)
    (cx0, cx1), hx0, lx = axis(hw[1], w, left, W)

    def tap(ry, cx):
        (r, rv), (c, cv) = ry, cx
        return a[:, r][:, :, c] * (rv[:, None] & cv[None, :])

    v = hy0[:, None] * (hx0 * tap(ry0, cx0) + lx * tap(ry0, cx1)) + \
        ly[:, None] * (hx0 * tap(ry1, cx0) + lx * tap(ry1, cx1))
    if flipped:
        v = v[..., ::-1]
    return _near_half(v).any(0)


def _compare(geo, x, idx, out, crop, params, pol_out, pol, tvpol, kinds, tally):
    """Every sample of a K5p fp32 NCHW output (no scale / bias) against torchvision's chain.  ``crop``
    is K5p's output without a policy: where it differs from ``_crop`` (only within 1e-3 of a half is
    allowed) torchvision's chain starts from K5p's crop, so each op is compared on the same input."""
    B, n_ops = x.shape[0], pol.num_ops
    hw = (geo.oh, geo.ow)
    idx_np = idx.numpy()
    want_ops = policy_np.policy_ops(idx_np, seed=SEED, epoch=EPOCH, policy=pol.native, num_ops=n_ops,
                                    num_bins=pol.num_magnitude_bins, magnitude=pol.magnitude)
    assert pol_out[:, :3 * n_ops].numpy().tolist() == want_ops.reshape(B, -1).tolist()
    want_box = augment_np.sample_params(idx_np, seed=SEED, epoch=EPOCH, mode=geo.mode, height=geo.sh,
                                        width=geo.sw, out_h=geo.oh, out_w=geo.ow, pad=geo.pad)
    assert params.numpy().tolist() == want_box.tolist()
    got, crop = out.cpu(), crop.cpu()
    for t in (got, crop):
        assert torch.equal(t, t.round()) and t.min() >= 0 and t.max() <= 255
    got, crop = got.to(torch.uint8), crop.to(torch.uint8)
    table = _tv_table(tvpol, pol.num_magnitude_bins, *hw)
    for s in range(B):
        what = f"{geo}: sample {s} ({KIND_NAMES[kinds[s]]} image)"
        start = _crop(x[s], params[s], hw)
        cdiff = (start != crop[s]).any(0).numpy()
        if cdiff.any():
            bad = cdiff & ~_crop_near(x[s], params[s], hw)
            assert not bad.any(), f"{what}: {int(bad.sum())} crop pixels differ from torchvision's crop"
            tally[1] += int(cdiff.sum())
            start = crop[s]
        ops = [tuple(pol_out[s, 3 * k:3 * k + 3].tolist()) for k in range(n_ops)]
        ref, taint = _chain(start, ops, table, tvpol)
        diff = (ref != got[s]).any(0).numpy()
        bad = diff & ~taint
        if bad.any():
            y, xx = np.argwhere(bad)[0]
            raise AssertionError(
                f"{what}, ops {[(POLICY_OPS[o], b, g) for o, b, g in ops]}: {int(bad.sum())} pixels differ from "
                f"torchvision, first at (y={y}, x={xx}): got {got[s, :, y, xx].tolist()}, "
                f"torchvision {ref[:, y, xx].tolist()}")
        tally[0] += int(diff.sum())
        tally[2] += diff.size


KIND_NAMES = ("smooth", "constant", "two-level", "one constant channel", "saturated", "ramp", "specks", "smooth")


def _pick(keys_of, want, per_key, seed, num_bins=31):
    """Dataset indices whose TrivialAugmentWide draw at EPOCH hits every key of ``want``, ``per_key``
    times each (one each for per_key 0); keys_of maps an (op, bin, sign) row to its key."""
    cand = _indices(1 << 18, seed).numpy()
    rows = policy_np.policy_ops(cand, seed=SEED, epoch=EPOCH, policy=policy_np.TRIVIAL_AUGMENT, num_ops=1,
                                num_bins=num_bins)[:, 0]
    need = {k: max(per_key, 1) for k in want}
    total = sum(need.values())
    picked = []
    for i, r in zip(cand.tolist(), rows.tolist()):
        k = keys_of(tuple(r))
        if need.get(k, 0) > 0:
            need[k] -= 1
            picked.append(i)
            if len(picked) == total:
                break
    assert not any(need.values()), "candidate indices do not cover every key"
    return torch.tensor(picked, dtype=torch.int64)


EVERY_OP_BIN_SIGN = {(0, 0, 1), (12, 0, 1), (13, 0, 1)} | {(o, b, 1) for o in (10, 11) for b in range(31)} | \
    {(o, b, s) for o in range(1, 10) for b in range(31) for s in (-1, 1)}
EVERY_OP_SIGN = {(o, 1) for o in (0, 10, 11, 12, 13)} | {(o, s) for o in range(1, 10) for s in (-1, 1)}


def _report(what, geo, tally):
    ops, crop, total = tally
    print(f"{what} {geo}: excused pixels {ops} after the ops ({100.0 * ops / max(total, 1):.4f} %) and {crop} "
          f"in the crop, of {total}")
    assert ops <= EXCUSED_SHARE * total, (what, str(geo), ops, total)


# ---- 1. pixels against torchvision ----------------------------------------------------------------------------

@pytest.mark.parametrize("geo", GEOS, ids=str)
def test_magnitude_tables_equal_torchvisions(geo):
    for pol, tvpol in ((TrivialAugmentWide(), tv.TrivialAugmentWide()), (RandAugment(), tv.RandAugment()),
                       (RandAugment(num_magnitude_bins=11), tv.RandAugment(num_magnitude_bins=11))):
        mine = pol.magnitudes(geo.oh, geo.ow)
        theirs = _tv_table(tvpol, pol.num_magnitude_bins, geo.oh, geo.ow)
        assert torch.equal(mine, theirs), (pol, str(geo), (mine != theirs).nonzero().tolist()[:6])


@pytest.mark.parametrize("geo", GEOS, ids=str)
def test_trivial_augment_equals_torchvision(geo):
    pol, tvpol = TrivialAugmentWide(), tv.TrivialAugmentWide()
    if geo.per_key == 0:
        idx = _pick(lambda r: r, EVERY_OP_BIN_SIGN, 0, seed=geo.oh * 1000 + geo.ow)
    else:
        idx = _pick(lambda r: (r[0], r[2]), EVERY_OP_SIGN, geo.per_key, seed=geo.oh * 1000 + geo.ow)
    x = _images(idx.numel(), geo.C, geo.sh, geo.sw, seed=geo.oh + geo.ow)
    out, params, pol_out = _run(geo, x.to(DEV), idx.to(DEV), policy=pol)
    crop, _, _ = _run(geo, x.to(DEV), idx.to(DEV))
    tally = [0, 0, 0]
    _compare(geo, x, idx, out, crop, params, pol_out, pol, tvpol, np.arange(idx.numel()) % N_KINDS, tally)
    got = {tuple(r) for r in pol_out[:, :3].tolist()}
    if geo.per_key == 0:
        assert got == EVERY_OP_BIN_SIGN
    else:
        assert {(o, s) for o, _, s in got} == EVERY_OP_SIGN
    _report("TrivialAugmentWide", geo, tally)


@pytest.mark.parametrize("geo", GEOS, ids=str)
def test_rand_augment_equals_torchvision(geo):
    tally = [0, 0, 0]
    for j, (nb, mag, n_ops) in enumerate(RA_SETTINGS):
        pol = RandAugment(num_ops=n_ops, magnitude=mag, num_magnitude_bins=nb)
        tvpol = tv.RandAugment(num_ops=n_ops, magnitude=mag, num_magnitude_bins=nb)
        B = geo.ra_batch
        idx = _indices(B, seed=1000 * j + geo.oh)
        # rotate the image kinds through the settings, so small batches still see every kind
        rows = (torch.arange(B) + j) % (B + N_KINDS)
        x = _images(B + N_KINDS, geo.C, geo.sh, geo.sw, seed=j)[rows].contiguous()
        out, params, pol_out = _run(geo, x.to(DEV), idx.to(DEV), policy=pol)
        crop, _, _ = _run(geo, x.to(DEV), idx.to(DEV))
        _compare(geo, x, idx, out, crop, params, pol_out, pol, tvpol, rows.numpy() % N_KINDS, tally)
    _report("RandAugment", geo, tally)


# ---- 2. layouts and dtypes ------------------------------------------------------------------------------------

@pytest.mark.parametrize("geo", [G48x80, G80x48, G37x53, G28PAD, G224, G_CEIL], ids=str)
def test_nhwc_bf16_and_channel_affine_are_exact(geo):
    B = {G224: 24, G_CEIL: 8}.get(geo, 96)
    x = _images(B, geo.C, geo.sh, geo.sw, seed=7).to(DEV)
    idx = _indices(B, seed=8).to(DEV)
    sc, bi = _affine(geo.C)
    for pol in (TrivialAugmentWide(), RandAugment(num_ops=4)):
        u8, _, _ = _run(geo, x, idx, policy=pol)
        aff, _, _ = _run(geo, x, idx, policy=pol, scale=sc, bias=bi)
        sc32, bi32 = (torch.tensor(v, dtype=torch.float32, device=DEV).double().view(1, -1, 1, 1) for v in (sc, bi))
        want = (u8.double() * sc32 + bi32).float()
        assert torch.equal(aff.view(torch.int32), want.view(torch.int32)), (str(geo), pol)
        kw = dict(policy=pol, erasing=RandomErasing(p=0.7, value="random"), scale=sc, bias=bi)
        f32, _, _ = _run(geo, x, idx, **kw)
        f32_nhwc, _, _ = _run(geo, x, idx, nhwc=True, **kw)
        assert f32_nhwc.is_contiguous(memory_format=torch.channels_last)
        assert torch.equal(f32.view(torch.int32), f32_nhwc.contiguous().view(torch.int32)), (str(geo), pol)
        for nhwc in (False, True):
            bf, _, _ = _run(geo, x, idx, dtype=torch.bfloat16, nhwc=nhwc, **kw)
            assert torch.equal(bf.contiguous().view(torch.int16), f32.to(torch.bfloat16).view(torch.int16)), \
                (str(geo), pol, nhwc)


# ---- 3. random-erasing values ---------------------------------------------------------------------------------

ERASE_GEOS = [G48x80, G80x48, G37x53]
ULP24 = 2.0 ** -24
ERASE_BOUND = 6.0                            # in units of 2^-24 * (r + 1)


def _box_muller(i, C, h, w, *, channel_stride=None, shared=False, transposed=False, u1_plus_one=True):
    """float64 (value, r) [C, h, w] of the header's erasing values for the sample with index i.
    The keywords restate wrong mappings, so the test can show that its bound rejects them."""
    c, y, x = np.meshgrid(np.arange(C), np.arange(h), np.arange(w), indexing="ij")
    cs = h if channel_stride is None else channel_stride
    if shared:
        c = np.zeros_like(c)
    e = ((c * cs + x) * h + y) if transposed else ((c * cs + y) * w + x)
    e = e.astype(np.uint64)
    i = np.uint64(i)
    words = np.stack(augment_np.philox4x32_10(
        (i & np.uint64(0xFFFFFFFF), i >> np.uint64(32), np.uint64(EPOCH), np.uint64(32) + e // np.uint64(4)),
        (SEED & 0xFFFFFFFF, SEED >> 32)))
    j = ((e // np.uint64(2)) % np.uint64(2)).astype(np.int64)
    wa = np.take_along_axis(words, (2 * j)[None], 0)[0]
    wb = np.take_along_axis(words, (2 * j + 1)[None], 0)[0]
    u1 = ((wa >> np.uint32(8)).astype(np.float64) + (1.0 if u1_plus_one else 0.0)) * ULP24
    u2 = (wb >> np.uint32(8)).astype(np.float64) * ULP24
    with np.errstate(divide="ignore"):
        r = np.sqrt(-2.0 * np.log(u1))
    val = np.where(e % np.uint64(2) == 0, r * np.cos(2.0 * np.pi * u2), r * np.sin(2.0 * np.pi * u2))
    return val, r


@pytest.mark.parametrize("nhwc", [False, True], ids=["nchw", "nhwc"])
@pytest.mark.parametrize("geo", ERASE_GEOS, ids=str)
def test_random_erasing_values_equal_box_muller(geo, nhwc):
    B = 192
    x = _images(B, geo.C, geo.sh, geo.sw, seed=11).to(DEV)
    idx = _indices(B, seed=12)
    pol = TrivialAugmentWide()
    base, _, _ = _run(geo, x, idx.to(DEV), policy=pol, nhwc=nhwc)
    out, _, pol_out = _run(geo, x, idx.to(DEV), policy=pol, erasing=RandomErasing(p=1.0, value="random"), nhwc=nhwc)
    boxes = pol_out[:, 3:]
    want_boxes = policy_np.erase_boxes(idx.numpy(), seed=SEED, epoch=EPOCH, out_h=geo.oh, out_w=geo.ow, p=1.0)
    assert boxes.numpy().tolist() == want_boxes.tolist()
    assert boxes[:, 0].float().mean() > 0.9
    assert (boxes[:, 3] != boxes[:, 4]).float().mean() > 0.5          # mostly non-square boxes
    got_all, base = out.cpu().double(), base.cpu()
    mask = torch.zeros(B, 1, geo.oh, geo.ow, dtype=torch.bool)
    wrong = {"channel stride w": 0, "shared channels": 0, "transposed": 0, "u1 without +1": 0}
    n = 0
    for s, (e, t, l, h, w) in enumerate(boxes.tolist()):
        if not e:
            continue
        mask[s, :, t:t + h, l:l + w] = True
        got = got_all[s, :, t:t + h, l:l + w].numpy()
        want, r = _box_muller(int(idx[s]), geo.C, h, w)
        bound = ERASE_BOUND * ULP24 * (r + 1.0)
        err = np.abs(got - want)
        assert (err <= bound).all(), (str(geo), s, (h, w), float((err / (ULP24 * (r + 1.0))).max()))
        n += got.size
        alts = {"transposed": dict(transposed=True), "u1 without +1": dict(u1_plus_one=False)}
        if geo.C > 1:
            alts.update({"channel stride w": dict(channel_stride=w), "shared channels": dict(shared=True)})
        for name, kw in alts.items():
            alt, _ = _box_muller(int(idx[s]), geo.C, h, w, **kw)
            wrong[name] += int((~(np.abs(got - alt) <= bound)).sum())
    mask = mask.expand(-1, geo.C, -1, -1)
    assert torch.equal(out.cpu()[~mask].view(torch.int32), base[~mask].view(torch.int32))
    print(f"erasing {geo} {'nhwc' if nhwc else 'nchw'}: {n} values within {ERASE_BOUND} * 2^-24 * (r + 1); "
          f"values the wrong restatements would put outside it: {wrong}")
    assert n > 50000
    assert wrong["transposed"] > 0.5 * n and wrong["u1 without +1"] > 0
    if geo.C > 1:
        assert wrong["shared channels"] > 0.3 * n and wrong["channel stride w"] > 0.3 * n


@pytest.mark.parametrize("nhwc", [False, True], ids=["nchw", "nhwc"])
@pytest.mark.parametrize("geo", ERASE_GEOS, ids=str)
def test_constant_erasing_value_per_channel_lands_exactly(geo, nhwc):
    B = 64
    x = _images(B, geo.C, geo.sh, geo.sw, seed=13).to(DEV)
    idx = _indices(B, seed=14).to(DEV)
    sc, bi = _affine(geo.C)
    values = [0.3125, -1.7, 2.640625][:geo.C]
    kw = dict(policy=RandAugment(num_ops=2), scale=sc, bias=bi, nhwc=nhwc)
    base, _, _ = _run(geo, x, idx, **kw)
    out, _, pol_out = _run(geo, x, idx, erasing=RandomErasing(p=1.0, value=values), **kw)
    mask = torch.zeros(B, 1, geo.oh, geo.ow, dtype=torch.bool)
    for s, (e, t, l, h, w) in enumerate(pol_out[:, 3 * 2:].tolist()):
        if e:
            mask[s, :, t:t + h, l:l + w] = True
    assert mask.any()
    got, base = out.cpu(), base.cpu()
    for c, v in enumerate(values):
        inside = got[:, c][mask[:, 0]]
        assert torch.equal(inside, torch.full_like(inside, np.float32(v).item()))
    mask = mask.expand(-1, geo.C, -1, -1)
    assert torch.equal(got[~mask].view(torch.int32), base[~mask].view(torch.int32))
