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
    """

    needs_index = True
    MODES = ("rrc", "pad_crop")

    def __init__(self, image_field: str, target_fields: Sequence[str], *, mode: str = "rrc",
                 out_size=224, crop_scale=(0.08, 1.0), crop_ratio=(3.0 / 4.0, 4.0 / 3.0), pad: int = 4,
                 mean: Optional[Sequence[float]] = None, std: Optional[Sequence[float]] = None,
                 scale: Optional[Sequence[float]] = None, bias: Optional[Sequence[float]] = None,
                 seed: int = 0, eval_crop: float = 0.875, flip: bool = True,
                 mix: Optional[BatchMix] = None) -> None:
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

    def augment(self, x: Tensor, index: Tensor, split: Split, out_dtype, params_out=None) -> Tensor:
        """The normalised, augmented images [B, C, out_h, out_w] of ``out_dtype``."""
        import torch
        from . import _native
        sc, bi = self._coefs(x)
        out = torch.empty((x.shape[0], x.shape[1]) + self.out_size, dtype=out_dtype, device=x.device)
        _native.augment_images(x.contiguous(), index, out, **self._native_args(split, sc, bi, params_out))
        return out

    def augment_mixed(self, x: Tensor, index: Tensor, out_dtype, mode: int, lam: float, box,
                      params_out=None) -> Tensor:
        """Training images [B, C, out_h, out_w] with sample i mixed with sample B-1-i (``mode``
        ``BatchMix.MIXUP`` or ``CUTMIX``) in the augmentation pass."""
        import torch
        from . import _native
        sc, bi = self._coefs(x)
        out = torch.empty((x.shape[0], x.shape[1]) + self.out_size, dtype=out_dtype, device=x.device)
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
        if self.mix is None or split != Split.TRAIN:
            out = self.augment(raw[self.image_field], index, split, out_dtype)
            return [out], [(raw[f],) for f in self.target_fields]
        mode, lam, box = self.mix.draw(self.seed, self.epoch, _dist_rank(), self.ordinal, *self.out_size)
        self.ordinal += 1
        x = raw[self.image_field]
        if mode == BatchMix.NONE:
            out = self.augment(x, index, split, out_dtype)
        else:
            out = self.augment_mixed(x, index, out_dtype, mode, lam, box)
        return [out], self.mix_targets(raw, lam)
