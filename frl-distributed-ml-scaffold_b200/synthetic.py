"""Synthetic multitask Problems used by the parity tests and the benchmark.

The reference ships no concrete ``Problem``, so the configurations BASELINE.json
names are defined here, written purely against the plugin API.  Every builder takes the API
namespace as an argument: pass ``frl_b200`` to run on this package, or the reference imported
as ``frldistml.scaffold`` (oracle only) to run the very same Problem on the reference Solver.

* ``make_toy_problem``  — config 1: 64-d input, 2x128 trunk, MSE head (w=0.5) + CE head (w=2).
* ``make_mlp_problem``  — configs 2/3: 4096-d input, 3x4096 trunk, CE head (1000) + MSE head (64).
* ``make_resnet_problem`` — config 4 (torchvision resnet18 trunk + one CE head, 11 689 512
  parameters) and config 5 (resnet50 trunk + heads 2048->{1000 CE, 100 CE, 10 MSE, 4 MSE},
  25 790 618 parameters) on synthetic 3xHxW images.
* ``make_text_problem`` — next-byte prediction over the lines of two ``TextDataset`` corpora
  (``write_text_corpus`` / ``write_mixed_text_corpus`` write seeded ones).
"""
import importlib
from types import SimpleNamespace
from typing import Any, Dict, List, NamedTuple, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.nn as nn


def api_namespace(pkg_name: str) -> SimpleNamespace:
    """Collect the plugin-API names from a package laid out like the reference."""
    mod = lambda n: importlib.import_module(f"{pkg_name}.{n}")     # noqa: E731
    types, problem, mt = mod("types"), mod("problem"), mod("multitask_problem")
    return SimpleNamespace(
        name=pkg_name, types=types, Split=types.Split, RunOpts=types.RunOpts,
        OptimOpts=types.OptimOpts, OptAlgorithm=types.OptAlgorithm, Mode=types.Mode,
        SampleSummary=types.SampleSummary,
        Ordering=problem.Ordering, Problem=problem.Problem,
        MultiTaskProblem=mt.MultiTaskProblem, MultiTaskTransform=mt.MultiTaskTransform,
        Task=mod("task").Task, criteria=mod("criteria"), model=mod("model"),
        MultifieldDataset=mod("storage_layers.dataset").MultifieldDataset)


class NoTransformState(NamedTuple):
    pass


class IndexMeta(NamedTuple):
    index: Any = None


class NoMeta(NamedTuple):
    pass


class BatchMeta(NamedTuple):
    index: Any = None


def _array_dataset_class(ns):
    class ArrayDataset(ns.MultifieldDataset):
        """In-memory dataset: one ndarray per field, first axis = sample."""

        def __init__(self, split, fields: Dict[str, np.ndarray], transform) -> None:
            self.data_type = split
            self._fields = fields
            self._transform = transform
            self._n = len(next(iter(fields.values())))
            self.served: List[int] = []          # access order, for the index-parity tests

        def __len__(self) -> int:
            return self._n

        def set_accessor(self, accessor) -> None:
            pass

        def get_raw_item(self, idx: int) -> Dict[str, np.ndarray]:
            item = {k: np.asarray(v[idx]) for k, v in self._fields.items()}
            item["index"] = np.asarray(idx, dtype=np.int64)
            return item

        def __getitem__(self, idx: int):
            self.served.append(int(idx))
            return self._transform(self.get_raw_item(idx), self.data_type)

    return ArrayDataset


def _affine_device_transform(shift: float, scale: float, target_fields):
    """Batched twin of ``CenteringTransform``: x -> (x - shift) * scale on the device (K5)."""
    import torch
    from . import _native
    from .transform import DeviceBatchTransform

    class AffineDeviceTransform(DeviceBatchTransform):
        bf16_wire_fields = ("x",)

        def __init__(self) -> None:
            self.shift, self.scale = float(shift), float(scale)
            self.target_fields = list(target_fields)
            self._coef = {}

        def apply(self, raw, split, out_dtype):
            x = raw["x"]
            out = torch.empty(x.shape, dtype=out_dtype, device=x.device)
            key = x.device
            if key not in self._coef:          # y = x*scale + (-shift*scale)
                self._coef[key] = (torch.tensor([self.scale], device=x.device),
                                   torch.tensor([-self.shift * self.scale], device=x.device))
            sc, bi = self._coef[key]
            _native.preproc_affine(x, out, inner=max(x.numel(), 1), channels=1, scale=sc, bias=bi)
            # task order is the Problem's: targets are looked up by the tasks' field names
            return [out], [(raw[f],) for f in self.target_fields]

    return AffineDeviceTransform()


def _channel_affine_device_transform(scale, bias, target_fields):
    """Batched twin of ``ChannelAffineTransform``: raw images [B, C, H, W] (uint8 or float) ->
    x * scale[c] + bias[c] in ``out_dtype``, one ``frl_preproc_affine`` pass (K5); channels_last
    images (``memory_format``, 1 to 4 channels) from one ``frl_preproc_affine_nhwc`` pass."""
    import torch
    from . import _native
    from .transform import DeviceBatchTransform

    class ChannelAffineDeviceTransform(DeviceBatchTransform):
        honours_memory_format = True

        def __init__(self) -> None:
            self.scale, self.bias = [float(v) for v in scale], [float(v) for v in bias]
            self.target_fields = list(target_fields)
            self._coef = {}

        def apply(self, raw, split, out_dtype):
            x = raw["x"]
            nhwc = self.memory_format is torch.channels_last and x.dim() == 4 and x.shape[1] <= 4
            out = torch.empty(x.shape, dtype=out_dtype, device=x.device,
                              memory_format=torch.channels_last if nhwc else torch.contiguous_format)
            if x.device not in self._coef:
                self._coef[x.device] = (torch.tensor(self.scale, device=x.device),
                                        torch.tensor(self.bias, device=x.device))
            sc, bi = self._coef[x.device]
            if _native.is_nhwc(out):
                _native.preproc_affine_nhwc(x, out, scale=sc, bias=bi)
            else:
                inner = max(x[0, 0].numel(), 1)
                _native.preproc_affine(x, out, inner=inner, channels=x.shape[1], scale=sc, bias=bi)
            return [out], [(raw[f],) for f in self.target_fields]

    return ChannelAffineDeviceTransform()


def _pinned_dataset_class(ns):
    """ArrayDataset whose fields also exist as pinned host tensors + a batched device transform
    (the H100 input path); the per-sample path stays available and equivalent."""
    import torch
    Base = _array_dataset_class(ns)

    class PinnedArrayDataset(Base):
        def __init__(self, split, fields, transform, shift, scale, target_fields,
                     channel_affine=None, device_transform=None) -> None:
            super().__init__(split, fields, transform)
            pin = torch.cuda.is_available()
            self.pinned_fields = {k: (torch.from_numpy(v).pin_memory() if pin else torch.from_numpy(v))
                                  for k, v in fields.items()}
            if device_transform is not None:
                self.device_transform = device_transform
            elif channel_affine is not None:
                self.device_transform = _channel_affine_device_transform(*channel_affine, target_fields)
            else:
                self.device_transform = _affine_device_transform(shift, scale, target_fields)

    return PinnedArrayDataset


def _indexed_datasets(ns, folder: str, datasets_fields, transform, shift, scale, target_fields):
    """The same fields written as ``.idx``/``.bin`` files (one sub-folder per split, as the
    reference lays datasets out) and served from the mapped files."""
    import os
    from . import indexed_dataset as idm
    out = []
    for split, fields in datasets_fields:
        sub = os.path.join(folder, split.value)
        idm.write_fields(sub, fields)
        names = list(fields)
        raw = idm.MultifieldIndexedDataset(sub, fields=names, filenames=names)
        out.append(idm.TransformedIndexedDataset(
            raw, split, transform, device_transform=_affine_device_transform(shift, scale, target_fields)))
    return out


def _task_classes(ns):
    class RegressionTask(ns.Task):
        def __init__(self, in_dim: int, out_dim: int, weight: float, field: str = "y_reg",
                     name: str = "reg") -> None:
            self._in, self._out, self._w, self._field, self.name = in_dim, out_dim, weight, field, name

        @property
        def network_head(self) -> nn.Module:
            return nn.Linear(self._in, self._out)

        @property
        def criterion(self):
            return nn.MSELoss()

        @property
        def criterion_weight(self) -> float:
            return self._w

        def get_target(self, tensors, transform):
            return (tensors[self._field],), IndexMeta(index=tensors["index"])

        def compute_batch_metrics(self, meta, target, output):
            err = ((output.float() - target[0].float()) ** 2).reshape(len(output), -1).mean(1)
            # device outputs -> device metrics: the loop keeps them in HBM and reads the whole
            # split back once (SamplerState's device-side fold); host outputs -> the reference's
            # numpy arrays
            return {self.name + "_MSE": err if err.is_cuda else err.numpy()}

        @property
        def rankable_metrics(self):
            return {(self.name + "_MSE", ns.Ordering.DESC)}

        def summarize_epoch_metrics(self, batch_metrics):
            return {self.name + "_MSE": float(np.mean(batch_metrics[self.name + "_MSE"]))}

        def summarize_epoch_samples(self, data, target, meta, output, metric):
            return [ns.SampleSummary(text="%s: %d samples" % (self.name, len(output)))]

    class ClassificationTask(ns.Task):
        def __init__(self, in_dim: int, n_classes: int, weight: float, field: str = "y_cls",
                     name: str = "cls", label_smoothing: float = 0.0) -> None:
            self._in, self._out, self._w, self._field, self.name = in_dim, n_classes, weight, field, name
            self.label_smoothing = float(label_smoothing)

        @property
        def network_head(self) -> nn.Module:
            return nn.Linear(self._in, self._out)

        @property
        def criterion(self):
            return nn.CrossEntropyLoss(label_smoothing=self.label_smoothing)

        @property
        def criterion_weight(self) -> float:
            return self._w

        def get_target(self, tensors, transform):
            return (tensors[self._field],), NoMeta()

        def compute_batch_metrics(self, meta, target, output):
            y = target[0]
            if y.is_floating_point() and y.dim() == 2:
                y = y.argmax(1)           # mixed (probability) targets: the dominant class
            wrong = (output.argmax(1) != y).float()
            return {self.name + "_err": wrong if wrong.is_cuda else wrong.numpy()}

        @property
        def rankable_metrics(self):
            return {(self.name + "_err", ns.Ordering.DESC)}

        def summarize_epoch_metrics(self, batch_metrics):
            return {self.name + "_err": float(np.mean(batch_metrics[self.name + "_err"]))}

        def summarize_epoch_samples(self, data, target, meta, output, metric):
            return []

    return RegressionTask, ClassificationTask


def _problem_class(ns):
    class CenteringTransform(ns.MultiTaskTransform):
        """x -> (x - shift) * scale, the whole 'online preprocessing' of the synthetic configs."""

        def __init__(self, tasks, shift: float, scale: float) -> None:
            super().__init__(tasks, IndexMeta)
            self.shift, self.scale = shift, scale

        def transform_source_data(self, tensors, split):
            return [(tensors["x"] - self.shift) * self.scale], NoTransformState()

    class ChannelAffineTransform(ns.MultiTaskTransform):
        """Raw image [C, H, W] (uint8 or float) -> x * scale[c] + bias[c] in fp32: the usual
        /255, -mean, /std normalisation folded into one multiply-add per pixel."""

        def __init__(self, tasks, scale, bias) -> None:
            super().__init__(tasks, IndexMeta)
            self.scale = torch.tensor([float(v) for v in scale]).view(-1, 1, 1)
            self.bias = torch.tensor([float(v) for v in bias]).view(-1, 1, 1)

        def transform_source_data(self, tensors, split):
            return [tensors["x"].float() * self.scale + self.bias], NoTransformState()

    class CenterCropTransform(ns.MultiTaskTransform):
        """Per-sample path of an augmenting Problem (``DeviceImageAugment``): the deterministic
        centre crop of evaluation splits, resized bilinearly, then x * scale[c] + bias[c].  The
        random crops of the training split exist on the device only."""

        def __init__(self, tasks, augment) -> None:
            super().__init__(tasks, IndexMeta)
            self.augment = augment
            self.scale = torch.tensor(augment.scale or [1.0]).view(-1, 1, 1)
            self.bias = torch.tensor(augment.bias or [0.0]).view(-1, 1, 1)

        def transform_source_data(self, tensors, split):
            if split == ns.Split.TRAIN:
                raise RuntimeError("the training split of an augmenting Problem is served by the device "
                                   "path only (DeviceBatchLoader + DeviceImageAugment); its per-sample "
                                   "transform covers the evaluation splits")
            x = tensors["x"]
            c, H, W = x.shape
            aug = self.augment
            oh, ow = aug.out_size
            ch, cw = (round(H * aug.eval_crop), round(W * aug.eval_crop)) if aug.mode == "rrc" else (oh, ow)
            top, left = round((H - ch) / 2), round((W - cw) / 2)
            crop = torch.zeros(c, ch, cw)           # zero fill where the box leaves the image
            y0, y1, x0, x1 = max(top, 0), min(top + ch, H), max(left, 0), min(left + cw, W)
            crop[:, y0 - top:y1 - top, x0 - left:x1 - left] = x[:, y0:y1, x0:x1].float()
            if (ch, cw) != (oh, ow):
                crop = nn.functional.interpolate(crop[None], size=(oh, ow), mode="bilinear",
                                                 align_corners=False, antialias=False)[0]
            return [crop * self.scale + self.bias], NoTransformState()

    class SyntheticMultiTaskProblem(ns.MultiTaskProblem):
        BatchMetaType = BatchMeta

        def __init__(self, tasks, trunk_dims: Sequence[int], datasets_fields, save_dir: str,
                     shift: float, scale: float, criterion_kind: str = "parallel",
                     pinned: bool = False, base_factory=None, indexed_dir: Optional[str] = None,
                     channel_affine=None, augment=None) -> None:
            self._tasks = tasks
            self._trunk_dims = list(trunk_dims)
            self._base_factory = base_factory
            self._save_dir = save_dir
            self._criterion_kind = criterion_kind
            if augment is not None:
                self.transform = CenterCropTransform(tasks, augment)
                ds_cls = _pinned_dataset_class(ns)
                self._datasets = [ds_cls(split, fields, self.transform, shift, scale,
                                         [t._field for t in tasks], device_transform=augment)
                                  for split, fields in datasets_fields]
                return
            if channel_affine is not None:
                self.transform = ChannelAffineTransform(tasks, *channel_affine)
            else:
                self.transform = CenteringTransform(tasks, shift, scale)
            if indexed_dir is not None:
                self._datasets = _indexed_datasets(ns, indexed_dir, datasets_fields, self.transform,
                                                   shift, scale, [t._field for t in tasks])
            elif pinned:
                ds_cls = _pinned_dataset_class(ns)
                self._datasets = [ds_cls(split, fields, self.transform, shift, scale,
                                         [t._field for t in tasks], channel_affine=channel_affine)
                                  for split, fields in datasets_fields]
            else:
                ds_cls = _array_dataset_class(ns)
                self._datasets = [ds_cls(split, fields, self.transform)
                                  for split, fields in datasets_fields]

        @property
        def datasets(self):
            return self._datasets

        @property
        def save_dir(self) -> str:
            return self._save_dir

        @property
        def anno_param(self):
            return None

        def get_model_base(self) -> nn.Module:
            if self._base_factory is not None:
                return self._base_factory()
            layers: List[nn.Module] = [ns.model.ListSelect(sel_index=0, num_elements=1)]
            for d_in, d_out in zip(self._trunk_dims[:-1], self._trunk_dims[1:]):
                layers += [nn.Linear(d_in, d_out), nn.ReLU()]
            return nn.Sequential(*layers)

        def get_criterion(self):
            mods = [t.criterion for t in self._tasks]
            names = [t.name for t in self._tasks]
            weights = [t.criterion_weight for t in self._tasks]
            c = ns.criteria
            if self._criterion_kind == "parallel":
                return c.ParallelCriterion(mods, weights, names)
            if self._criterion_kind == "uncertainty":
                LT = ns.types.LossType
                kinds = [LT.MSE if isinstance(m, nn.MSELoss) else LT.CrossEntropy for m in mods]
                return c.UncertaintyWeightedCriterion(mods, kinds, names, weights)
            if self._criterion_kind == "gradnorm":
                return c.GradNormWeightedCriterion(mods, names, alpha=1.5, base_weights=weights)
            raise ValueError(self._criterion_kind)

    return SyntheticMultiTaskProblem


def synthetic_fields(n: int, in_dim: int, reg_dim: int, n_classes: int, seed: int,
                     uniform_x: bool) -> Dict[str, np.ndarray]:
    rs = np.random.RandomState(seed)
    x = rs.rand(n, in_dim) if uniform_x else rs.randn(n, in_dim)
    return {"x": x.astype(np.float32),
            "y_reg": rs.randn(n, reg_dim).astype(np.float32),
            "y_cls": rs.randint(0, n_classes, size=n).astype(np.int64)}


def make_toy_problem(ns, save_dir: str, n_train: int = 512, n_test: int = 128,
                     criterion_kind: str = "parallel", pinned: bool = False,
                     indexed_dir: Optional[str] = None):
    """Config 1: trunk 64->128->128, reg head 128->4 (w 0.5), cls head 128->10 (w 2)."""
    Reg, Cls = _task_classes(ns)
    tasks = [Reg(128, 4, 0.5), Cls(128, 10, 2.0)]
    fields = [(ns.Split.TRAIN, synthetic_fields(n_train, 64, 4, 10, 0, True)),
              (ns.Split.TEST, synthetic_fields(n_test, 64, 4, 10, 1, True))]
    return _problem_class(ns)(tasks, [64, 128, 128], fields, save_dir, shift=0.5, scale=2.0,
                              criterion_kind=criterion_kind, pinned=pinned, indexed_dir=indexed_dir)


def synthetic_fields_fast(n: int, in_dim: int, reg_dim: int, n_classes: int, seed: int
                          ) -> Dict[str, np.ndarray]:
    """Same shapes/distributions as ``synthetic_fields`` from torch's (multi-threaded) generator:
    for the multi-GB host datasets of the benchmark, where numpy's scalar generator takes minutes."""
    g = torch.Generator().manual_seed(seed)
    return {"x": torch.randn(n, in_dim, generator=g).numpy(),
            "y_reg": torch.randn(n, reg_dim, generator=g).numpy(),
            "y_cls": torch.randint(0, n_classes, (n,), generator=g).numpy()}


def make_mlp_problem(ns, save_dir: str, n_train: int = 8192, n_test: int = 0, width: int = 4096,
                     n_classes: int = 1000, reg_dim: int = 64, depth: int = 3, pinned: bool = False,
                     fast_fields: bool = False):
    """Configs 2/3: trunk depth x [Linear(width,width)+ReLU], CE head width->1000 (w 1), MSE
    head width->64 (w 1); x ~ N(0,1)."""
    Reg, Cls = _task_classes(ns)
    tasks = [Cls(width, n_classes, 1.0), Reg(width, reg_dim, 1.0)]
    train = (synthetic_fields_fast(n_train, width, reg_dim, n_classes, 0) if fast_fields
             else synthetic_fields(n_train, width, reg_dim, n_classes, 0, False))
    fields = [(ns.Split.TRAIN, train)]
    if n_test:
        fields.append((ns.Split.TEST, synthetic_fields(n_test, width, reg_dim, n_classes, 1, False)))
    return _problem_class(ns)(tasks, [width] * (depth + 1), fields, save_dir, shift=0.0, scale=1.0,
                              pinned=pinned)


RESNET_CONFIGS = {
    # name: (torchvision arch, [(kind, out_dim, field, task name)])
    "resnet18": ("resnet18", [("cls", 1000, "y_cls", "cls")]),
    "resnet50x4": ("resnet50", [("cls", 1000, "y_cls", "cls1000"), ("cls", 100, "y_cls2", "cls100"),
                                ("reg", 10, "y_reg", "reg10"), ("reg", 4, "y_reg2", "reg4")]),
}


#: the usual ImageNet normalisation as x_u8 * scale[c] + bias[c]
IMAGE_MEAN, IMAGE_STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
U8_CHANNEL_AFFINE = (tuple(1.0 / (255.0 * s) for s in IMAGE_STD),
                     tuple(-m / s for m, s in zip(IMAGE_MEAN, IMAGE_STD)))


def resnet_fields(n: int, image: int, heads, seed: int, uint8: bool = False) -> Dict[str, np.ndarray]:
    g = torch.Generator().manual_seed(seed)
    if uint8:
        fields = {"x": torch.randint(0, 256, (n, 3, image, image), generator=g, dtype=torch.uint8).numpy()}
    else:
        fields = {"x": torch.randn(n, 3, image, image, generator=g).numpy()}
    for kind, dim, field, _ in heads:
        if kind == "cls":
            fields[field] = torch.randint(0, dim, (n,), generator=g).numpy()
        else:
            fields[field] = torch.randn(n, dim, generator=g).numpy()
    return fields


def make_resnet_problem(ns, save_dir: str, config: str = "resnet18", image: int = 224,
                        n_train: int = 64, n_test: int = 0, pinned: bool = False,
                        uint8: bool = False, augment: Optional[str] = None,
                        stored_image: Optional[int] = None, mixup_alpha: float = 0.0,
                        cutmix_alpha: float = 0.0, label_smoothing: float = 0.0,
                        policy: Optional[str] = None, random_erasing: float = 0.0):
    """Configs 4/5: a torchvision ResNet trunk (its ``fc`` removed) behind
    ``ListSelect`` and one ``nn.Linear`` head per task; x ~ N(0,1) of shape [3, image, image], or
    (``uint8``) raw 8-bit images normalised per channel by the transform (150 kB/sample over
    PCIe instead of 602 kB).

    ``augment`` (``uint8`` only): ``"rrc"`` (random resized crop + flip, ImageNet-style) or
    ``"pad_crop"`` (crop of the image zero-padded by 4 + flip, CIFAR-style) on the device
    (``transform.DeviceImageAugment``, K5a) from stored ``stored_image`` x ``stored_image`` images
    to the model's ``image`` x ``image``; evaluation splits take the centre crop.  The datasets are
    then pinned; their per-sample transform serves the evaluation splits only.
    ``mixup_alpha`` / ``cutmix_alpha`` (need ``augment``): Mixup / CutMix of the training batches
    (``transform.BatchMix`` over every head's target field) in the augmentation pass.
    ``label_smoothing``: the classification heads' ``CrossEntropyLoss(label_smoothing=...)``.
    ``policy`` (needs ``augment``): ``"ta_wide"`` (``TrivialAugmentWide()``) or ``"ra"``
    (``RandAugment()``) on the training crops; ``random_erasing``: ``RandomErasing(p=...)`` of the
    training images when > 0 (K5p)."""
    import torchvision
    stored = image if stored_image is None else int(stored_image)
    if augment is None and stored != image:
        raise ValueError("stored_image differs from image only for an augmenting Problem (augment=...)")
    arch, heads = RESNET_CONFIGS[config]
    aug = None
    mix = None
    if (policy is not None or random_erasing) and augment is None:
        raise ValueError("policy / random_erasing run on the device augmentation path: pass augment=...")
    if mixup_alpha or cutmix_alpha:
        from .transform import BatchMix
        if augment is None:
            raise ValueError("mixup_alpha / cutmix_alpha mix on the device augmentation path: pass augment=...")
        mix = BatchMix({field: dim for kind, dim, field, _ in heads if kind == "cls"},
                       mixup_alpha=mixup_alpha, cutmix_alpha=cutmix_alpha)
    if augment is not None:
        from .transform import DeviceImageAugment
        if not uint8:
            raise ValueError("augment works on raw uint8 images: pass uint8=True")
        if augment not in DeviceImageAugment.MODES:
            raise ValueError(f"augment must be None or one of {DeviceImageAugment.MODES}, got {augment!r}")
        from .transform import RandAugment, RandomErasing, TrivialAugmentWide
        policies = {None: None, "ta_wide": TrivialAugmentWide, "ra": RandAugment}
        if policy not in policies:
            raise ValueError(f"policy must be None, 'ta_wide' or 'ra', got {policy!r}")
        pol = None if policy is None else policies[policy]()
        erasing = RandomErasing(p=random_erasing) if random_erasing else None
        aug = DeviceImageAugment("x", [field for _, _, field, _ in heads], mode=augment, out_size=image, pad=4,
                                 scale=U8_CHANNEL_AFFINE[0], bias=U8_CHANNEL_AFFINE[1], mix=mix, policy=pol,
                                 erasing=erasing)
        aug.check_image(3, stored, stored)
    feat = {"resnet18": 512, "resnet50": 2048}[arch]
    Reg, Cls = _task_classes(ns)
    tasks = [Cls(feat, dim, 1.0, field=field, name=name, label_smoothing=label_smoothing) if kind == "cls"
             else Reg(feat, dim, 1.0, field=field, name=name)
             for kind, dim, field, name in heads]

    def base_factory() -> nn.Module:
        net = getattr(torchvision.models, arch)(weights=None)
        net.fc = nn.Identity()
        return nn.Sequential(ns.model.ListSelect(sel_index=0, num_elements=1), net)

    fields = [(ns.Split.TRAIN, resnet_fields(n_train, stored, heads, 0, uint8))]
    if n_test:
        fields.append((ns.Split.TEST, resnet_fields(n_test, stored, heads, 1, uint8)))
    return _problem_class(ns)(tasks, [], fields, save_dir, shift=0.0, scale=1.0, pinned=pinned,
                              base_factory=base_factory,
                              channel_affine=U8_CHANNEL_AFFINE if uint8 else None, augment=aug)


# ---- text: next-byte prediction over TextDataset lines ---------------------------------------

def write_text_corpus(path: str, n_lines: int, seed: int, seq_len: int = 32,
                      max_len: Optional[int] = None) -> None:
    """A deterministic newline-separated corpus: empty lines and lines shorter than, exactly
    ``seq_len + 1`` and longer than that, bytes drawn from 0x00-0xFF except ``\\n``, and no
    trailing newline (so the last line loses two bytes, as in the reference's TextDataset)."""
    rs = np.random.RandomState(seed)
    row = seq_len + 1
    max_len = max_len or 3 * row
    forced = [0, 1, row - 1, row, row + 1, max_len]
    lengths = np.concatenate([np.asarray(forced[:n_lines], dtype=np.int64),
                              rs.randint(0, max_len + 1, size=max(n_lines - len(forced), 0))])
    values = np.delete(np.arange(256, dtype=np.uint8), 0x0A)
    body = values[rs.randint(0, 255, size=int(lengths.sum()))]
    out = np.empty(int(lengths.sum()) + max(n_lines - 1, 0), dtype=np.uint8)
    pos = src = 0
    for i, n in enumerate(lengths):
        out[pos:pos + n] = body[src:src + n]
        pos += int(n)
        src += int(n)
        if i + 1 < n_lines:
            out[pos] = 0x0A
            pos += 1
    with open(path, "wb") as f:
        f.write(out.tobytes())


class PositionsToClasses(nn.Module):
    """[B, L, C] per-position logits -> [B, C, L], the layout ``nn.CrossEntropyLoss`` takes for
    per-position classes."""

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return x.transpose(1, 2)


def _text_device_transform():
    """Batched twin of the text transform: x = line[:, :-1], y = line[:, 1:] as int64."""
    from .transform import DeviceBatchTransform

    class NextByteDeviceTransform(DeviceBatchTransform):
        def apply(self, raw, split, out_dtype):
            line = raw["line"]
            return [line[:, :-1].long()], [(line[:, 1:].long(),)]

        def meta(self, raw, index):
            return {}                      # the per-sample transform's meta has no fields

    return NextByteDeviceTransform()


def make_text_problem(ns, save_dir: str, train_path, test_path, seq_len: int = 32,
                      device_batches: bool = False, hidden: int = 128):
    """Next-byte prediction on the lines of two text files: Embedding(256, 64), then per position
    Linear(64, hidden) + ReLU + Linear(hidden, 256), one CrossEntropyLoss(ignore_index=0) task
    (padding bytes are not predicted).  ``device_batches``: hand the datasets the batched twin
    of the transform, so the loop serves them through ``DeviceBatchLoader`` (K8t)."""
    text = importlib.import_module(f"{ns.name}.text_dataset")
    as_path = getattr(text, "StoragePath", str)          # the reference's TextDataset takes StoragePaths

    class NextByteTask(ns.Task):
        name = "next_byte"

        @property
        def network_head(self) -> nn.Module:
            return nn.Sequential(nn.Linear(hidden, 256), PositionsToClasses())

        @property
        def criterion(self):
            return nn.CrossEntropyLoss(ignore_index=0)

        @property
        def criterion_weight(self) -> float:
            return 1.0

        def get_target(self, tensors, transform):
            return (tensors["line"][1:].long(),), NoMeta()

        def compute_batch_metrics(self, meta, target, output):
            y = target[0]
            wrong = ((output.argmax(1) != y) & (y != 0)).float().mean(1)
            return {"byte_err": wrong if wrong.is_cuda else wrong.numpy()}

        @property
        def rankable_metrics(self):
            return {("byte_err", ns.Ordering.DESC)}

        def summarize_epoch_metrics(self, batch_metrics):
            return {"byte_err": float(np.mean(batch_metrics["byte_err"]))}

        def summarize_epoch_samples(self, data, target, meta, output, metric):
            return []

    class NextByteTransform(ns.MultiTaskTransform):
        def transform_source_data(self, tensors, split):
            return [tensors["line"][:-1].long()], NoTransformState()

    class TextProblem(ns.MultiTaskProblem):
        BatchMetaType = BatchMeta

        def __init__(self) -> None:
            self._tasks = [NextByteTask()]
            self.transform = NextByteTransform(self._tasks, NoMeta)
            kw = {"device_transform": _text_device_transform()} if device_batches else {}
            self._datasets = [text.TextDataset(split, as_path(str(path)), self.transform, seq_len, **kw)
                              for split, path in ((ns.Split.TRAIN, train_path), (ns.Split.TEST, test_path))]

        @property
        def datasets(self):
            return self._datasets

        @property
        def save_dir(self) -> str:
            return save_dir

        @property
        def anno_param(self):
            return None

        def get_model_base(self) -> nn.Module:
            return nn.Sequential(ns.model.ListSelect(sel_index=0, num_elements=1), nn.Embedding(256, 64),
                                 nn.Linear(64, hidden), nn.ReLU())

        def get_criterion(self):
            return ns.criteria.ParallelCriterion([t.criterion for t in self._tasks], [1.0],
                                                 [t.name for t in self._tasks])

    return TextProblem()


def write_mixed_text_corpus(path: str, n_bytes: int, seed: int, short_mean: int = 120,
                            long_mean: int = 2048, long_share: float = 0.1) -> None:
    """About ``n_bytes`` of seeded text for measurements: line lengths drawn from a mixture of
    two exponentials (means ``short_mean`` and ``long_mean`` bytes), bytes 0x00-0xFF except
    ``\\n``."""
    rs = np.random.RandomState(seed)
    mean = (1 - long_share) * short_mean + long_share * long_mean
    n_lines = max(1, int(n_bytes / (mean + 1)))
    long = rs.rand(n_lines) < long_share
    lengths = np.where(long, rs.exponential(long_mean, n_lines), rs.exponential(short_mean, n_lines)).astype(np.int64)
    ends = np.cumsum(lengths + 1) - 1                   # position of each line's newline
    values = np.delete(np.arange(256, dtype=np.uint8), 0x0A)
    out = values[rs.randint(0, 255, size=int(ends[-1]))]
    out[ends[:-1]] = 0x0A
    with open(path, "wb") as f:
        f.write(out.tobytes())
