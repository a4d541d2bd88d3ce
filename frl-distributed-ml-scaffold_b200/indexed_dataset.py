"""``.idx`` / ``.bin`` indexed datasets — the on-disk format that feeds the training loop
(reference storage_layers/dataset.py:555-655, storage_layers/posix_storage.py:47-80,
indexed_dataset.py:40-133).

Format (all int64, little endian), exactly what the reference reads and writes::

    idx = [magic, version, type_code, itemsize, N, S,
           dimoffsets[0..N], dataoffsets[0..N], sizes[0..S-1]]        # 6 + 2(N+1) + S words
    bin = frame 0 | frame 1 | ...                                       # raw items, no padding

``type_code - 1`` indexes ``np_types``; frame ``i`` has ``dimoffsets[i+1] - dimoffsets[i]``
dimensions ``sizes[dimoffsets[i] : dimoffsets[i+1]]`` and starts at item ``dataoffsets[i]``.  The
reference's writer stores ``magic = version = 0`` (dataset.py:618-619) and its reader checks
neither (dataset.py:567-568): both are preserved.  Like the reference's reader, this one assumes
every frame has the shape of frame 0 (dataset.py:586-594).

What is added for the H100 path: a fixed-shape indexed file IS a row-major ``[N, framesize]``
array, so ``MultifieldIndexedDataset.host_fields`` exposes the memory-mapped ``.bin`` files as
zero-copy CPU tensors and the batched input path (``DeviceBatchLoader``, ``host`` mode) lets the
native gather pool copy a minibatch's frames from the page cache straight into pinned staging —
no per-sample ``__getitem__``, ``.copy()``, ``from_numpy`` or ``default_collate``.
"""
import os
import warnings
from contextlib import contextmanager
from itertools import chain
from typing import Any, Dict, Iterator, List, Optional, Sequence, Sized, Tuple, Union

import numpy as np
import torch

from .storage_layers.dataset import DatasetField, MultifieldDataset
from .types import Split

np_types = ["uint8", "int8", "int16", "int32", "int64", "float32", "float64", None]

PathLike = Union[str, "os.PathLike[str]", Any]      # also objects with a ``.path`` (StoragePath)


def _fs_path(p: PathLike) -> str:
    inner = getattr(p, "path", None)
    return str(inner if inner is not None else p)


class IndexedDatasetReader(Sized):
    """Header parsing shared by every reader (reference dataset.py:555-604)."""

    scheme = ""

    dtype: np.dtype
    N: int
    S: int
    ndim: int
    size: np.ndarray
    framesize: int

    def _init_from_index_data(self, idx: np.ndarray) -> None:
        if idx.ndim != 1 or len(idx) < 6:
            raise ValueError("index file too short: %d int64 words" % idx.size)
        code = int(idx[2])
        if not 1 <= code <= len(np_types) or np_types[code - 1] is None:
            raise AssertionError("unrecognized type")
        self.dtype = np.dtype(np_types[code - 1])
        assert self.dtype.itemsize == idx[3]
        self.N = int(idx[4])
        self.S = int(idx[5])
        need = 6 + 2 * (self.N + 1) + self.S
        if self.N < 1 or self.S < 0 or len(idx) < need:
            raise ValueError("index file truncated: %d words, header announces %d" % (len(idx), need))
        ofs = 6
        dimoffsets = idx[ofs: ofs + self.N + 1]
        ofs += self.N + 1
        datoffsets = idx[ofs: ofs + self.N + 1]
        ofs += self.N + 1
        sizes = idx[ofs: ofs + self.S]
        # every frame is assumed to have the shape of frame 0, as in the reference
        self.ndim = int(dimoffsets[1] - dimoffsets[0])
        so = int(dimoffsets[0])
        self.size = sizes[so: so + self.ndim]
        assert datoffsets[0] == 0, "first data frame must be at the start of the .bin file"
        self.framesize = int(datoffsets[1] - datoffsets[0])
        self._uniform = bool(
            np.array_equal(np.diff(datoffsets), np.full(self.N, self.framesize))
            and np.array_equal(np.diff(dimoffsets), np.full(self.N, self.ndim)))

    def __len__(self) -> int:
        return self.N

    def set_accessor(self, accessor) -> None:
        return

    def __getitem__(self, index: int):
        raise NotImplementedError


class PosixIndexedDatasetReader(IndexedDatasetReader):
    """Memory-mapped reader (reference posix_storage.py:47-80)."""

    scheme = "file"

    def __init__(self, *, idxfile: PathLike, binfile: PathLike) -> None:
        self.datafilename = _fs_path(binfile)
        idx = np.fromfile(_fs_path(idxfile), dtype="int64")
        self._init_from_index_data(idx)
        self.data = np.memmap(self.datafilename, dtype=self.dtype, mode="r")

    def __getitem__(self, index: int):
        assert index >= 0 and index < self.N, "index out of range"
        data = self.data[self.framesize * index: self.framesize * (index + 1)]
        return data.reshape(self.size).copy()            # a private copy, as the reference returns

    def __setstate__(self, state):
        state["data"] = np.memmap(state["datafilename"], dtype=state["dtype"], mode="r")
        self.__dict__.update(state)

    def __getstate__(self):
        state = self.__dict__.copy()
        del state["data"]
        return state

    # ---- batched access (H100 path) -------------------------------------------------------------
    def frames_tensor(self) -> torch.Tensor:
        """The whole ``.bin`` file as a zero-copy CPU tensor ``[N, *frame shape]`` over the page
        cache.  Requires every frame to have frame 0's shape and the file to hold N frames."""
        if not self._uniform:
            raise ValueError("%s: frames differ in shape; batched access needs fixed-size frames"
                             % self.datafilename)
        n_items = self.N * self.framesize
        if len(self.data) < n_items:
            raise ValueError("%s holds %d items, the index announces %d" % (
                self.datafilename, len(self.data), n_items))
        flat = np.asarray(self.data[:n_items])
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", UserWarning)      # read-only mapping: never written
            t = torch.from_numpy(flat)
        return t.view((self.N,) + tuple(int(d) for d in self.size))


class IndexedDatasetWriter:
    """Streams frames to ``.bin`` and writes the ``.idx`` header on ``flush``
    (reference dataset.py:607-655)."""

    def __init__(self, *, idxfile, binfile) -> None:
        self._idxfile = idxfile
        self._binfile = binfile
        self._sizes: List[Tuple[int, ...]] = []
        self._dtype: Optional[np.dtype] = None

    def _generate_idx(self) -> np.ndarray:
        if not self._sizes:
            raise AssertionError("Cannot write empty dataset")
        dtype = self._dtype
        ranks = np.fromiter((len(shape) for shape in self._sizes), dtype=np.int64, count=len(self._sizes))
        items = np.fromiter((int(np.prod(shape, dtype=np.int64)) for shape in self._sizes),
                            dtype=np.int64, count=len(self._sizes))
        header = np.array([0, 0,                                   # magic, version: the reference writes 0, 0
                           np_types.index(dtype.name) + 1, dtype.itemsize,
                           len(self._sizes), int(ranks.sum())], dtype=np.int64)
        zero = np.zeros(1, dtype=np.int64)
        dims = np.fromiter(chain.from_iterable(self._sizes), dtype=np.int64, count=int(ranks.sum()))
        return np.concatenate([header, zero, np.cumsum(ranks), zero, np.cumsum(items), dims])

    def flush(self) -> None:
        self._idxfile.write(self._generate_idx().tobytes())

    def push_back(self, frame: np.ndarray) -> None:
        self._sizes.append(frame.shape)
        if self._dtype is not None:
            assert self._dtype == frame.dtype, "Frames must all have same dtype"
        else:
            self._dtype = frame.dtype
        self._binfile.write(frame.tobytes())


class IndexedDatasetReaderFactory:
    @staticmethod
    def get(idxfile: PathLike, binfile: PathLike) -> IndexedDatasetReader:
        return PosixIndexedDatasetReader(idxfile=idxfile, binfile=binfile)


class IndexedDatasetWriterFactory:
    @staticmethod
    @contextmanager
    def get(idxfile: PathLike, binfile: PathLike) -> Iterator[IndexedDatasetWriter]:
        with open(_fs_path(idxfile), "wb") as idx_f, open(_fs_path(binfile), "wb") as bin_f:
            writer = IndexedDatasetWriter(idxfile=idx_f, binfile=bin_f)
            yield writer
            writer.flush()


RawDatasets = Dict[DatasetField, IndexedDatasetReader]


class MultifieldIndexedDataset(MultifieldDataset):
    """Several indexed files describing different fields of the same samples
    (reference indexed_dataset.py:65-133): item ``i`` is ``{field: frame i of that file}``."""

    def __init__(self, folder_path: PathLike, *, fields: List[DatasetField],
                 filenames: List[str]) -> None:
        assert len(fields) == len(filenames), "Number of properties should equal number of filenames"
        self.datasets: RawDatasets = {}
        for field, name in zip(fields, filenames):
            self.datasets[field] = self.get_dataset(folder_path, name)
        self.length = len(self.datasets[fields[0]])
        for field, dataset in self.datasets.items():
            assert len(dataset) == self.length, (
                "dataset %s should have same number of samples as %s (%d vs %d)"
                % (field, fields[0], len(dataset), self.length))

    def __len__(self) -> int:
        return self.length

    def get_raw_item(self, idx: int) -> Dict[DatasetField, np.ndarray]:
        return self[idx]

    def __getitem__(self, index: int) -> Dict[str, np.ndarray]:
        return {field: dataset[index] for field, dataset in self.datasets.items()}

    def get_dataset(self, folder_path: PathLike, filename: str) -> IndexedDatasetReader:
        folder = _fs_path(folder_path)
        return IndexedDatasetReaderFactory.get(idxfile=os.path.join(folder, filename + ".idx"),
                                               binfile=os.path.join(folder, filename + ".bin"))

    def set_accessor(self, accessor) -> None:
        for key, dataset in self.datasets.items():
            dataset.set_accessor(accessor.with_multifield_dataset_field(key))

    @property
    def host_fields(self) -> Dict[DatasetField, torch.Tensor]:
        """``{field: zero-copy [N, ...] CPU tensor over the mapped .bin}`` for the batched path."""
        return {field: ds.frames_tensor() for field, ds in self.datasets.items()}


class TransformedIndexedDataset(MultifieldDataset):
    """A split served from indexed files: the per-sample protocol of the reference's
    ``MultiFolderDataset`` (indexed_dataset.py:166-225: ``transform(raw, split=...)``) plus the
    two attributes the batched input path looks for (``pinned_fields``, ``device_transform``).
    Adds the ``index`` field the synthetic datasets carry, so metas line up."""

    def __init__(self, dataset: MultifieldIndexedDataset, data_type: Split, transform,
                 device_transform=None) -> None:
        self._dataset = dataset
        self.data_type = data_type
        self.transform = transform
        if device_transform is not None:
            self.pinned_fields = dataset.host_fields          # CPU tensors: served by the host pool
            self.device_transform = device_transform

    def set_accessor(self, accessor) -> None:
        self._dataset.set_accessor(accessor)

    def __len__(self) -> int:
        return len(self._dataset)

    def get_raw_item(self, idx: int) -> Dict[DatasetField, np.ndarray]:
        item = self._dataset[idx]
        item["index"] = np.asarray(idx, dtype=np.int64)
        return item

    def __getitem__(self, idx: int):
        data = self.get_raw_item(idx)
        if self.transform is None:
            return data, None, None
        return self.transform(data, self.data_type)


def write_fields(folder: PathLike, fields: Dict[str, np.ndarray]) -> None:
    """Write ``{filename: array [N, ...]}`` as one indexed file per field (frame = array[i])."""
    folder = _fs_path(folder)
    os.makedirs(folder, exist_ok=True)
    for name, arr in fields.items():
        with IndexedDatasetWriterFactory.get(os.path.join(folder, name + ".idx"),
                                             os.path.join(folder, name + ".bin")) as w:
            for frame in arr:
                w.push_back(np.asarray(frame))      # tobytes() is C-order; 0-d frames stay 0-d
