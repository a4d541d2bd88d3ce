"""Per-sample transform API (reference transform.py:20-44) plus its batched device-side twin.

``MultifieldTransform`` is the reference contract: a raw record (dict of ndarrays) becomes
``(Sample(data, target), meta)`` and ``__call__`` flattens that to the triple the DataLoader
collates.  ``DeviceBatchTransform`` is the H100 addition: the same arithmetic applied to a
whole batch after the raw bytes reached HBM, through the ``frl_preproc_affine`` kernel.
``DeviceImageAugment`` is a ready-made one for image Problems: crop, resize, flip and normalise in
one ``frl_augment_images`` pass, optionally with Mixup / CutMix of the batch (``BatchMix``) in the
same pass.
"""
import math
from abc import ABC, abstractmethod
from typing import Any, Dict, Generic, List, NamedTuple, Optional, Sequence, Tuple, TypeVar, Union

import numpy as np
import torch
from torch import Tensor

from .types import Split

SampleMetaT = TypeVar("SampleMetaT", bound=NamedTuple)


class Sample(NamedTuple):
    data: Sequence[Tensor]
    target: Sequence[Union[Tensor, Tuple[Tensor, ...]]]


class MultifieldTransform(ABC, Generic[SampleMetaT]):
    def __call__(self, data: Dict[str, np.ndarray], split: Split
                 ) -> Tuple[Sequence[Tensor], Sequence[Tensor], Dict[str, Any]]:
        sample, meta = self.transform(data, split)
        # default_collate handles dicts/lists/tensors only: drop unset meta fields
        kept = {k: v for k, v in meta._asdict().items() if v is not None}
        return sample.data, sample.target, kept

    @abstractmethod
    def transform(self, data: Dict[str, np.ndarray], split: Split
                  ) -> Tuple[Sample, SampleMetaT]:
        ...


class DeviceBatchTransform(ABC):
    """Batched, on-device counterpart of ``MultifieldTransform`` (extension).

    Pairs with a dataset whose raw fields sit in pinned host memory (``pinned_fields``): the
    loop's ``DeviceBatchLoader`` pulls the rows of a batch into HBM and calls ``apply`` once per
    batch with the device copies; ``apply`` must return ``(data, target)`` equal to what the
    per-sample transform + ``default_collate`` would have produced (floating outputs in
    ``out_dtype``).  ``meta`` returns the collated meta dict (tensors on any device / lists).
    """

    #: fp32 fields ``apply`` is happy to receive already rounded to bfloat16 when ``out_dtype`` is
    #: bfloat16 (typically the model inputs).  The host input path may then ship them over PCIe in
    #: bf16 (``FRL_B200_INPUT_WIRE=bf16``); targets and anything exact must not be listed.
    bf16_wire_fields: Sequence[str] = ()

    #: True: ``apply`` is also given ``index=`` (device int64 [B], the dataset row of each sample),
    #: e.g. to key per-sample random draws to the sample rather than to its place in the batch.
    needs_index: bool = False

    #: the layout image batches should come out in; the loop sets ``torch.channels_last`` when the
    #: run is channels_last (``Solver.solve(..., channels_last=True)``).  A transform that writes
    #: 4-D image fields in that layout says so with ``honours_memory_format = True``; any other
    #: keeps returning what it did, and the first convolution converts.
    memory_format: torch.memory_format = torch.contiguous_format
    honours_memory_format: bool = False

    @abstractmethod
    def apply(self, raw: Dict[str, Tensor], split: Split, out_dtype
              ) -> Tuple[List[Tensor], List[Tuple[Tensor, ...]]]:
        ...

    def meta(self, raw: Dict[str, Tensor], index: Tensor) -> Dict[str, Any]:
        return {"index": index.clone()}

    def set_epoch(self, epoch: int) -> None:
        """Called at the start of every split of every epoch (1-based, the loop's epoch)."""


def _pair(name: str, value) -> Tuple[float, float]:
    try:
        lo, hi = (float(v) for v in value)
    except (TypeError, ValueError):
        raise ValueError(f"{name} must be a pair of numbers, got {value!r}") from None
    if not (0.0 < lo <= hi and math.isfinite(hi)):
        raise ValueError(f"{name} must satisfy 0 < {name}[0] <= {name}[1], got {value!r}")
    return lo, hi


class BatchMix:
    """Mixup (Zhang et al. 2018) and CutMix (Yun et al. 2019) of a training batch, applied by
    ``DeviceImageAugment(..., mix=BatchMix(...))`` in the augmentation pass itself.

    Sample i is mixed with sample B-1-i of the same batch, images and every target field with the
    same lambda: a class-index field named in ``classes`` ({field: number of classes}) becomes fp32
    probabilities [B, n] (lam at y_i, 1 - lam at y_j); a floating field becomes
    lam * t_i + (1 - lam) * t_j.  A batch is mixed with probability ``prob``, by CutMix with
    probability ``switch_prob`` when both alphas are > 0 (else by the one whose alpha is > 0).  An
    unmixed training batch still gets one-hot fp32 class targets, so a split's target shapes never
    change.  Label smoothing stays with the loss: ``nn.CrossEntropyLoss(label_smoothing=eps)``.
    """

    NONE, MIXUP, CUTMIX = 0, 1, 2

    def __init__(self, classes: Dict[str, int], mixup_alpha: float = 0.0, cutmix_alpha: float = 0.0,
                 prob: float = 1.0, switch_prob: float = 0.5) -> None:
        for name, v in (("mixup_alpha", mixup_alpha), ("cutmix_alpha", cutmix_alpha)):
            if not (isinstance(v, (int, float)) and math.isfinite(v) and v >= 0.0):
                raise ValueError(f"{name} must be a finite number >= 0, got {v!r}")
        if mixup_alpha == 0.0 and cutmix_alpha == 0.0:
            raise ValueError("mixup_alpha and cutmix_alpha are both 0: nothing to mix")
        for name, v in (("prob", prob), ("switch_prob", switch_prob)):
            if not (isinstance(v, (int, float)) and 0.0 <= v <= 1.0):
                raise ValueError(f"{name} must be in [0, 1], got {v!r}")
        self.classes = {}
        for field, n in dict(classes).items():
            if isinstance(n, bool) or int(n) != n or n < 2:
                raise ValueError(f"classes[{field!r}] must be an integer >= 2, got {n!r}")
            self.classes[field] = int(n)
        self.mixup_alpha = float(mixup_alpha)
        self.cutmix_alpha = float(cutmix_alpha)
        self.prob = float(prob)
        self.switch_prob = float(switch_prob)

    def draw(self, seed: int, epoch: int, rank: int, ordinal: int, out_h: int, out_w: int
             ) -> Tuple[int, float, Tuple[int, int, int, int]]:
        """(mode, lam, (y0, y1, x0, x1)) of one batch: a pure function of its arguments, from a
        Philox generator keyed by (seed, epoch, rank, ordinal); no global RNG is touched.  The box
        is CutMix's, on the out_h x out_w output ((0, 0, 0, 0) otherwise); a CutMix lam is
        1 - box area / image area."""
        key = [int(seed) & 0xFFFFFFFF, int(seed) >> 32, int(epoch), int(rank), int(ordinal)]
        rng = np.random.Generator(np.random.Philox(np.random.SeedSequence(key)))
        none = (0, 0, 0, 0)
        if rng.random() >= self.prob:
            return self.NONE, 1.0, none
        if self.mixup_alpha > 0.0 and self.cutmix_alpha > 0.0:
            cutmix = rng.random() < self.switch_prob
        else:
            cutmix = self.cutmix_alpha > 0.0
        if not cutmix:
            return self.MIXUP, float(rng.beta(self.mixup_alpha, self.mixup_alpha)), none
        lam = float(rng.beta(self.cutmix_alpha, self.cutmix_alpha))
        r = math.sqrt(1.0 - lam)
        cut_h, cut_w = int(out_h * r), int(out_w * r)
        cy, cx = int(rng.integers(out_h)), int(rng.integers(out_w))
        y0, y1 = min(max(cy - cut_h // 2, 0), out_h), min(max(cy + cut_h // 2, 0), out_h)
        x0, x1 = min(max(cx - cut_w // 2, 0), out_w), min(max(cx + cut_w // 2, 0), out_w)
        lam = 1.0 - (y1 - y0) * (x1 - x0) / float(out_h * out_w)
        return self.CUTMIX, lam, (y0, y1, x0, x1)


#: torchvision's ``_AUGMENTATION_SPACE`` order; K5p's op ids are the positions in it
POLICY_OPS = ("Identity", "ShearX", "ShearY", "TranslateX", "TranslateY", "Rotate", "Brightness", "Color",
              "Contrast", "Sharpness", "Posterize", "Solarize", "AutoContrast", "Equalize")


def _int_arg(name: str, value, lo: int, hi: Optional[int] = None) -> int:
    if isinstance(value, bool) or not isinstance(value, (int, np.integer)) or value < lo or (hi is not None
                                                                                          and value > hi):
        rng = f"[{lo}, {hi}]" if hi is not None else f">= {lo}"
        raise ValueError(f"{name} must be an integer {rng}, got {value!r}")
    return int(value)


class TrivialAugmentWide:
    """TrivialAugmentWide (Müller & Hutter 2021) for ``DeviceImageAugment(..., policy=...)``: one op
    per training sample, a random magnitude bin and sign, as torchvision's
    ``TrivialAugmentWide(num_magnitude_bins)`` with NEAREST interpolation and fill 0."""

    native = 1
    num_ops = 1
    magnitude = 0

    def __init__(self, num_magnitude_bins: int = 31) -> None:
        self.num_magnitude_bins = _int_arg("num_magnitude_bins", num_magnitude_bins, 2)

    def magnitudes(self, height: int, width: int) -> Tensor:
        """fp32 [14, num_magnitude_bins]: torchvision's unsigned magnitude table (0 for the ops
        without a magnitude)."""
        nb = self.num_magnitude_bins
        lin = lambda hi: torch.linspace(0.0, hi, nb)  # noqa: E731
        rows = [None, lin(0.99), lin(0.99), lin(32.0), lin(32.0), lin(135.0), lin(0.99), lin(0.99), lin(0.99),
                lin(0.99), (8 - (torch.arange(nb) / ((nb - 1) / 6))).round().int(), torch.linspace(1.0, 0.0, nb),
                None, None]
        return torch.stack([torch.zeros(nb) if r is None else r.float() for r in rows])

    def __repr__(self) -> str:
        return f"TrivialAugmentWide(num_magnitude_bins={self.num_magnitude_bins})"


class RandAugment:
    """RandAugment (Cubuk et al. 2020) for ``DeviceImageAugment(..., policy=...)``: ``num_ops``
    (1 to 4) random ops per training sample at the fixed ``magnitude`` bin with a random sign, as
    torchvision's ``RandAugment`` with NEAREST interpolation and fill 0."""

    native = 2

    def __init__(self, num_ops: int = 2, magnitude: int = 9, num_magnitude_bins: int = 31) -> None:
        self.num_ops = _int_arg("num_ops", num_ops, 1, 4)
        self.num_magnitude_bins = _int_arg("num_magnitude_bins", num_magnitude_bins, 2)
        self.magnitude = _int_arg("magnitude", magnitude, 0, self.num_magnitude_bins - 1)

    def magnitudes(self, height: int, width: int) -> Tensor:
        """fp32 [14, num_magnitude_bins]; TranslateX / TranslateY scale with ``width`` / ``height``."""
        nb = self.num_magnitude_bins
        lin = lambda hi: torch.linspace(0.0, hi, nb)  # noqa: E731
        rows = [None, lin(0.3), lin(0.3), lin(150.0 / 331.0 * width), lin(150.0 / 331.0 * height), lin(30.0),
                lin(0.9), lin(0.9), lin(0.9), lin(0.9), (8 - (torch.arange(nb) / ((nb - 1) / 4))).round().int(),
                torch.linspace(1.0, 0.0, nb), None, None]
        return torch.stack([torch.zeros(nb) if r is None else r.float() for r in rows])

    def __repr__(self) -> str:
        return (f"RandAugment(num_ops={self.num_ops}, magnitude={self.magnitude}, "
                f"num_magnitude_bins={self.num_magnitude_bins})")


class RandomErasing:
    """Random erasing (Zhong et al. 2020) of the normalised training images, as torchvision's
    ``RandomErasing(p, scale, ratio, value)``: ``value`` a number, one number per channel, or
    ``"random"`` (standard normal values from the device's counter-based generator, not torch's
    stream)."""

    def __init__(self, p: float = 0.5, scale=(0.02, 0.33), ratio=(0.3, 3.3), value=0.0) -> None:
        if not (isinstance(p, (int, float)) and not isinstance(p, bool) and 0.0 <= p <= 1.0):
            raise ValueError(f"p must be in [0, 1], got {p!r}")
        try:
            lo, hi = (float(v) for v in scale)
        except (TypeError, ValueError):
            raise ValueError(f"scale must be a pair of numbers, got {scale!r}") from None
        if not 0.0 <= lo <= hi <= 1.0:
            raise ValueError(f"scale must satisfy 0 <= scale[0] <= scale[1] <= 1, got {scale!r}")
        self.p = float(p)
        self.scale = (lo, hi)
        self.ratio = _pair("ratio", ratio)
        if isinstance(value, str):
            if value != "random":
                raise ValueError(f"value must be a number, a sequence of numbers or 'random', got {value!r}")
            self.value: Optional[List[float]] = None
        else:
            vals = [value] if isinstance(value, (int, float)) else list(value)
            if not 1 <= len(vals) <= 4 or not all(isinstance(v, (int, float)) and math.isfinite(v) for v in vals):
                raise ValueError(f"value must be a finite number or 1 to 4 of them, got {value!r}")
            self.value = [float(v) for v in vals]

    @property
    def random(self) -> bool:
        return self.value is None

    def values(self, channels: int) -> List[float]:
        """The erasing value of every channel (``value`` is not "random")."""
        if len(self.value) not in (1, channels):
            raise ValueError(f"RandomErasing value has {len(self.value)} entries for {channels}-channel images")
        return self.value * channels if len(self.value) == 1 else list(self.value)

    def __repr__(self) -> str:
        v = "random" if self.value is None else self.value
        return f"RandomErasing(p={self.p}, scale={self.scale}, ratio={self.ratio}, value={v!r})"


def _dist_rank() -> int:
    import torch.distributed as dist
    return dist.get_rank() if dist.is_available() and dist.is_initialized() else 0


class DeviceImageAugment(DeviceBatchTransform):
    """Training-time image augmentation on the device, K5a (``frl_augment_images``): one pass from
    the raw uint8 images [B, C, H, W] of a batch to the normalised model input.

    ``mode="rrc"``: random resized crop (area share ``crop_scale``, aspect ``crop_ratio``, the
    torchvision defaults) resized bilinearly to ``out_size``; evaluation splits take the centred
    ``round(H * eval_crop) x round(W * eval_crop)`` box, resized.
    ``mode="pad_crop"``: random ``out_size`` crop of the image zero-padded by ``pad`` on every side;
    evaluation splits take the centred ``out_size`` box.
    Random modes mirror each sample with p = 1/2 when ``flip``.  The draws are keyed by
    (``seed``, epoch, dataset index) — not by the batch, its order or the rank — and come from a
    counter-based generator on the device: torch's global RNG is not touched.
    Normalisation: ``mean`` / ``std`` in the [0, 1] domain of x / 255 (torchvision's ``Normalize``
    after ``ToDtype(scale=True)``), or the raw ``scale`` / ``bias`` of ``x * scale[c] + bias[c]``.
    ``mix``: a ``BatchMix``; training batches are then mixed in the same pass
    (``frl_augment_mix_images``) and their targets by ``frl_mix_targets``.  Its draws are keyed by
    (``seed``, epoch, rank, the batch's ordinal since ``set_epoch``).  Evaluation splits are not
    mixed and keep their targets as they are.
    ``policy``: a ``TrivialAugmentWide`` or ``RandAugment``; ``erasing``: a ``RandomErasing``.
    With either, training images go through K5p (``frl_augment_policy_images``): the same crop and
    flip, then the policy on the uint8 crop, the normalisation and the erasing, as torchvision v2
    does them; a mixed batch is then mixed over the finished images (``frl_mix_images``).  Their
    draws are keyed as the crop's.  Images need 1 or 3 channels with a policy, and a
    C x out_h x out_w crop of at most ``_native.POLICY_SMEM_BYTES`` bytes.
    With ``memory_format = torch.channels_last`` the images come out [B, C, out_h, out_w] with
    channels_last strides (``frl_augment_images_nhwc`` / ``frl_augment_mix_images_nhwc``), the same
    values as the NCHW output.
    """

    needs_index = True
    honours_memory_format = True
    MODES = ("rrc", "pad_crop")

    def __init__(self, image_field: str, target_fields: Sequence[str], *, mode: str = "rrc",
                 out_size=224, crop_scale=(0.08, 1.0), crop_ratio=(3.0 / 4.0, 4.0 / 3.0), pad: int = 4,
                 mean: Optional[Sequence[float]] = None, std: Optional[Sequence[float]] = None,
                 scale: Optional[Sequence[float]] = None, bias: Optional[Sequence[float]] = None,
                 seed: int = 0, eval_crop: float = 0.875, flip: bool = True,
                 mix: Optional[BatchMix] = None,
                 policy: Optional[Union[TrivialAugmentWide, RandAugment]] = None,
                 erasing: Optional[RandomErasing] = None) -> None:
        if mode not in self.MODES:
            raise ValueError(f"mode must be one of {self.MODES}, got {mode!r}")
        oh, ow = (out_size, out_size) if isinstance(out_size, int) else tuple(out_size)
        if not (int(oh) == oh >= 1 and int(ow) == ow >= 1):
            raise ValueError(f"out_size must be >= 1, got {out_size!r}")
        self.image_field = image_field
        self.target_fields = list(target_fields)
        self.mode = mode
        self.out_size = (int(oh), int(ow))
        self.crop_scale = _pair("crop_scale", crop_scale)
        self.crop_ratio = _pair("crop_ratio", crop_ratio)
        if int(pad) != pad or pad < 0:
            raise ValueError(f"pad must be an integer >= 0, got {pad!r}")
        self.pad = int(pad)
        if not (0.0 < float(eval_crop) <= 1.0):
            raise ValueError(f"eval_crop must be in (0, 1], got {eval_crop!r}")
        self.eval_crop = float(eval_crop)
        if int(seed) != seed or not 0 <= seed < 2 ** 64:
            raise ValueError(f"seed must be an integer in [0, 2**64), got {seed!r}")
        self.seed = int(seed)
        self.flip = bool(flip)
        if (mean is None) != (std is None):
            raise ValueError("mean and std go together")
        if mean is not None and (scale is not None or bias is not None):
            raise ValueError("give mean/std or scale/bias, not both")
        if mean is not None:
            if len(mean) != len(std) or not 1 <= len(mean) <= 4:
                raise ValueError(f"mean and std need one value per channel (1 to 4), got {mean!r}, {std!r}")
            if any(float(s) <= 0.0 for s in std):
                raise ValueError(f"std must be > 0, got {std!r}")
            scale = [1.0 / (255.0 * float(s)) for s in std]
            bias = [-float(m) / float(s) for m, s in zip(mean, std)]
        for name, v in (("scale", scale), ("bias", bias)):
            if v is not None and not 1 <= len(v) <= 4:
                raise ValueError(f"{name} needs one value per channel (1 to 4), got {v!r}")
        if scale is not None and bias is not None and len(scale) != len(bias):
            raise ValueError("scale and bias need the same number of channels")
        self.scale = None if scale is None else [float(v) for v in scale]
        self.bias = None if bias is None else [float(v) for v in bias]
        if mix is not None and not isinstance(mix, BatchMix):
            raise ValueError(f"mix must be a BatchMix or None, got {mix!r}")
        self.mix = mix
        if policy is not None and not isinstance(policy, (TrivialAugmentWide, RandAugment)):
            raise ValueError(f"policy must be a TrivialAugmentWide, a RandAugment or None, got {policy!r}")
        if erasing is not None and not isinstance(erasing, RandomErasing):
            raise ValueError(f"erasing must be a RandomErasing or None, got {erasing!r}")
        self.policy = policy
        self.erasing = erasing
        self._policy_tabs: Dict[Any, Tuple[Optional[Tensor], Optional[Tensor]]] = {}
        self.epoch = 0
        self.ordinal = 0          # training batches served since set_epoch (keys the mix draws)
        self._targets_checked = False
        self._coef: Dict[Any, Tuple[Optional[Tensor], Optional[Tensor]]] = {}

    def set_epoch(self, epoch: int) -> None:
        self.epoch = int(epoch)
        self.ordinal = 0

    def check_image(self, channels: int, height: int, width: int) -> None:
        """ValueError unless images of this shape can be served."""
        if not 1 <= channels <= 4:
            raise ValueError(f"{self.image_field!r}: images need 1 to 4 channels, got {channels}")
        for name, v in (("scale", self.scale), ("bias", self.bias)):
            if v is not None and len(v) != channels:
                raise ValueError(f"{name} has {len(v)} values for {channels}-channel images")
        oh, ow = self.out_size
        if self.mode == "pad_crop" and (oh > height + 2 * self.pad or ow > width + 2 * self.pad):
            raise ValueError(f"out_size {self.out_size} does not fit {height}x{width} images padded by {self.pad}")
        if self.mode == "rrc" and (round(height * self.eval_crop) < 1 or round(width * self.eval_crop) < 1):
            raise ValueError(f"eval_crop {self.eval_crop} leaves no pixel of {height}x{width} images")
        if self.policy is not None or self.erasing is not None:
            from . import _native
            if self.policy is not None and channels not in (1, 3):
                raise ValueError(f"{self.policy!r} needs 1- or 3-channel images (torchvision's colour ops), "
                                 f"got {channels}")
            if channels > 3:
                raise ValueError(f"RandomErasing on the device serves 1 to 3 channels, got {channels}")
            if channels * oh * ow > _native.POLICY_SMEM_BYTES:
                raise ValueError(f"a {channels}x{oh}x{ow} crop ({channels * oh * ow} bytes) does not fit one CTA's "
                                 f"shared memory ({_native.POLICY_SMEM_BYTES} bytes): out_size too large for "
                                 f"policy / erasing")
            if self.erasing is not None and not self.erasing.random:
                self.erasing.values(channels)

    def native_mode(self, split: Split) -> int:
        from . import _native
        if split == Split.TRAIN:
            return _native.AUG_RRC if self.mode == "rrc" else _native.AUG_PAD_CROP
        return _native.AUG_CENTER_RESIZE if self.mode == "rrc" else _native.AUG_CENTER_CROP

    def _coefs(self, x: Tensor):
        import torch
        if x.dtype != torch.uint8 or x.dim() != 4:
            raise ValueError(f"{self.image_field!r} must be uint8 [B, C, H, W], got {x.dtype} {tuple(x.shape)}")
        self.check_image(*x.shape[1:])
        if x.device not in self._coef:
            self._coef[x.device] = tuple(None if v is None else torch.tensor(v, dtype=torch.float32, device=x.device)
                                         for v in (self.scale, self.bias))
        return self._coef[x.device]

    def _native_args(self, split: Split, sc, bi, params_out):
        return dict(seed=self.seed, epoch=self.epoch, mode=self.native_mode(split), scale_range=self.crop_scale,
                    ratio_range=self.crop_ratio, eval_crop=self.eval_crop, pad=self.pad, flip=self.flip, scale=sc,
                    bias=bi, params_out=params_out)

    def _out(self, x: Tensor, out_dtype) -> Tensor:
        return torch.empty((x.shape[0], x.shape[1]) + self.out_size, dtype=out_dtype, device=x.device,
                           memory_format=self.memory_format)

    def augment(self, x: Tensor, index: Tensor, split: Split, out_dtype, params_out=None) -> Tensor:
        """The normalised, augmented images [B, C, out_h, out_w] of ``out_dtype``, in
        ``memory_format``."""
        from . import _native
        sc, bi = self._coefs(x)
        out = self._out(x, out_dtype)
        _native.augment_images(x.contiguous(), index, out, **self._native_args(split, sc, bi, params_out))
        return out

    def _policy_tables(self, x: Tensor):
        """(magnitude table, erasing values) on ``x``'s device, built once per device."""
        if x.device not in self._policy_tabs:
            oh, ow = self.out_size
            mags = None if self.policy is None else self.policy.magnitudes(oh, ow).to(x.device).contiguous()
            ev = None
            if self.erasing is not None and not self.erasing.random:
                ev = torch.tensor(self.erasing.values(x.shape[1]), dtype=torch.float32, device=x.device)
            self._policy_tabs[x.device] = (mags, ev)
        return self._policy_tabs[x.device]

    def augment_policy(self, x: Tensor, index: Tensor, out_dtype, params_out=None, policy_out=None) -> Tensor:
        """Training images [B, C, out_h, out_w] of ``out_dtype`` in ``memory_format``: K5a's crop and
        flip, then ``policy``, the affine and ``erasing`` (K5p, ``frl_augment_policy_images``)."""
        from . import _native
        sc, bi = self._coefs(x)
        mags, ev = self._policy_tables(x)
        out = self._out(x, out_dtype)
        pol, er = self.policy, self.erasing
        _native.augment_policy_images(
            x.contiguous(), index, out, seed=self.seed, epoch=self.epoch, mode=self.native_mode(Split.TRAIN),
            scale_range=self.crop_scale, ratio_range=self.crop_ratio, pad=self.pad, flip=self.flip,
            policy=_native.POLICY_NONE if pol is None else pol.native, num_ops=1 if pol is None else pol.num_ops,
            magnitude=0 if pol is None else pol.magnitude, mags=mags, erase_p=0.0 if er is None else er.p,
            erase_scale=(0.02, 0.33) if er is None else er.scale, erase_ratio=(0.3, 3.3) if er is None else er.ratio,
            erase_random=er is not None and er.random, erase_value=ev, scale=sc, bias=bi, params_out=params_out,
            policy_out=policy_out)
        return out

    def augment_mixed(self, x: Tensor, index: Tensor, out_dtype, mode: int, lam: float, box,
                      params_out=None) -> Tensor:
        """Training images [B, C, out_h, out_w] with sample i mixed with sample B-1-i (``mode``
        ``BatchMix.MIXUP`` or ``CUTMIX``) in the augmentation pass, in ``memory_format``."""
        from . import _native
        sc, bi = self._coefs(x)
        out = self._out(x, out_dtype)
        _native.augment_mix_images(x.contiguous(), index, out, mix_mode=mode, lam=lam, box=box,
                                   **self._native_args(Split.TRAIN, sc, bi, params_out))
        return out

    def mix_targets(self, raw: Dict[str, Tensor], lam: float) -> List[Tuple[Tensor, ...]]:
        """The target fields of a training batch mixed with ``lam`` (1.0: one-hot class targets and
        the floating fields as they are)."""
        import torch
        from . import _native
        if not self._targets_checked:
            for f in self.target_fields:
                t = raw[f]
                if f in self.mix.classes:
                    if t.dtype != torch.int64 or t.dim() != 1:
                        raise ValueError(f"target field {f!r} is listed in BatchMix.classes, so it must hold "
                                         f"int64 class indices [B], got {t.dtype} {tuple(t.shape)}")
                elif not t.is_floating_point() or t.dtype not in (torch.float32, torch.bfloat16):
                    raise ValueError(f"target field {f!r} can not be mixed: it is neither listed in "
                                     f"BatchMix.classes nor fp32/bf16, got {t.dtype}")
            self._targets_checked = True
        out = []
        for f in self.target_fields:
            t = raw[f].contiguous()
            if f in self.mix.classes:
                dst = torch.empty((t.shape[0], self.mix.classes[f]), dtype=torch.float32, device=t.device)
                _native.mix_targets(t, dst, lam, self.mix.classes[f])
            elif lam == 1.0:
                dst = raw[f]
            else:
                dst = torch.empty_like(t)
                _native.mix_targets(t, dst, lam)
            out.append((dst,))
        return out

    def apply(self, raw, split, out_dtype, index=None):
        if index is None:
            raise ValueError("DeviceImageAugment.apply needs index= (the dataset row of every sample)")
        per_sample = (self.policy is not None or self.erasing is not None) and split == Split.TRAIN
        if self.mix is None or split != Split.TRAIN:
            if per_sample:
                out = self.augment_policy(raw[self.image_field], index, out_dtype)
            else:
                out = self.augment(raw[self.image_field], index, split, out_dtype)
            return [out], [(raw[f],) for f in self.target_fields]
        mode, lam, box = self.mix.draw(self.seed, self.epoch, _dist_rank(), self.ordinal, *self.out_size)
        self.ordinal += 1
        x = raw[self.image_field]
        if per_sample:
            # Mixup / CutMix over the finished images (frl_mix_images): a bf16 Mixup rounds twice
            from . import _native
            out = self.augment_policy(x, index, out_dtype)
            if mode != BatchMix.NONE:
                _native.mix_images(out, mix_mode=mode, lam=lam, box=box)
            return [out], self.mix_targets(raw, lam)
        if mode == BatchMix.NONE:
            out = self.augment(x, index, split, out_dtype)
        else:
            out = self.augment_mixed(x, index, out_dtype, mode, lam, box)
        return [out], self.mix_targets(raw, lam)
