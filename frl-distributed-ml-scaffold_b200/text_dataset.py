"""Newline-separated text corpus held in memory, one sample per line (reference
``text_dataset.TextDataset``: same class name, constructor, attributes and samples).

Sample ``i`` is the bytes of line ``i``, cut or padded with ``PAD`` to ``seq_len + 1``.  The
line-start table is the reference's, quirks included: ``starts = [0] + [p + 1 for each '\\n' at
p]``, and ``n_bytes - 1`` is appended when the last entry differs from it, so a last line without
a newline loses its last two bytes, a trailing newline adds one empty sample, and the slice
``data[starts[i] : starts[i+1] - 1]`` follows numpy's rules for negative and reversed bounds.

The corpus is read once into one anonymous shared mapping (forked ranks and ``DataLoader``
workers share its pages) whose allocation is rounded up to 16 bytes with a zero tail, and the
start table is built with vectorised numpy in bounded chunks.  For the batched input path the
dataset exposes the corpus as a ``device_loader.PaddedLines`` field: ``DeviceBatchLoader``
page-locks the mapping in place on first use, in the rank process, and the ``frl_gather_lines``
kernel (K8t) pulls each minibatch's padded lines over PCIe.  Pinning at construction would
initialise CUDA in the parent process, and ``Solver.solve`` would then spawn its ranks instead of
forking them, each receiving a pickled copy of the corpus.
"""
import logging
import mmap
import os
import weakref
from typing import Any, Dict, Optional

import numpy as np

from .device_loader import PaddedLines
from .indexed_dataset import PathLike, _fs_path
from .storage_layers.dataset import DatasetField, MultifieldDataset
from .types import Split

logger = logging.getLogger(__name__)

#: bytes scanned per step while building the line-start table (bounds the temporaries)
N_CHUNK_BYTES = 64 * 1024 * 1024

_CUDA_HOST_REGISTER_MAPPED = 2
_CUDA_HOST_REGISTER_READ_ONLY = 8


def line_starts(data: np.ndarray, chunk_bytes: int = N_CHUNK_BYTES) -> np.ndarray:
    """The reference's line-start table of ``data`` (uint8 [n_bytes]) as int64."""
    n = int(data.shape[0])
    parts = [np.zeros(1, dtype=np.int64)]
    for off in range(0, n, chunk_bytes):
        hits = np.flatnonzero(data[off:off + chunk_bytes] == 0x0A)
        parts.append(hits.astype(np.int64) + (off + 1))
    starts = np.concatenate(parts)
    if starts[-1] != n - 1:
        starts = np.append(starts, np.int64(n - 1))
    return starts


def _unpin(pid: int, addr: int, _keep_alive) -> None:
    if os.getpid() == pid:            # a forked child never registered the pages itself
        import torch
        torch.cuda.cudart().cudaHostUnregister(addr)


class HostCorpus:
    """The bytes of a corpus in one anonymous shared mapping of ``alloc_bytes`` (``n_bytes``
    rounded up to 16, zero tail), pinned on demand."""

    def __init__(self, n_bytes: int) -> None:
        self.n_bytes = int(n_bytes)
        self.alloc_bytes = max(16, (self.n_bytes + 15) // 16 * 16)
        self._mm = mmap.mmap(-1, self.alloc_bytes)              # MAP_SHARED | MAP_ANONYMOUS, zeroed
        self._init_views()

    def _init_views(self) -> None:
        self.array = np.frombuffer(self._mm, dtype=np.uint8, count=self.n_bytes)
        self._pinned_in: Optional[int] = None

    @classmethod
    def from_file(cls, path: str, chunk_bytes: int = N_CHUNK_BYTES) -> "HostCorpus":
        corpus = cls(os.path.getsize(path))
        view = memoryview(corpus._mm)
        with open(path, "rb") as f:
            off = 0
            while off < corpus.n_bytes:
                got = f.readinto(view[off:min(off + chunk_bytes, corpus.n_bytes)])
                if not got:
                    raise IOError("%s: short read at byte %d of %d" % (path, off, corpus.n_bytes))
                off += got
        view.release()
        return corpus

    def pin(self) -> int:
        """Page-lock the mapping in place (mapped, read-only for the device) once per process and
        return its device-usable address (unified addressing: the host address)."""
        if self._pinned_in != os.getpid():
            import torch
            cudart = torch.cuda.cudart()
            addr = np.frombuffer(self._mm, dtype=np.uint8).ctypes.data
            rc = cudart.cudaHostRegister(addr, self.alloc_bytes,
                                         _CUDA_HOST_REGISTER_MAPPED | _CUDA_HOST_REGISTER_READ_ONLY)
            if int(rc) != 0:
                # devices without cudaDevAttrHostRegisterReadOnlySupported reject the read-only
                # flag; the kernel never writes the corpus, so a plain mapped registration serves.
                # The failed call left its error in the runtime torch checks after its launches.
                import ctypes
                ctypes.CDLL("libcudart.so.12").cudaGetLastError()
                logger.info("read-only host registration refused (%s); registering mapped",
                            cudart.cudaGetErrorString(rc))
                rc = cudart.cudaHostRegister(addr, self.alloc_bytes, _CUDA_HOST_REGISTER_MAPPED)
            if int(rc) != 0:
                raise RuntimeError("cudaHostRegister of a %d-byte text corpus failed: %s"
                                   % (self.alloc_bytes, cudart.cudaGetErrorString(rc)))
            self._pinned_in = os.getpid()
            self._addr = addr
            weakref.finalize(self, _unpin, self._pinned_in, addr, self._mm)
        return self._addr

    def __getstate__(self) -> Dict[str, Any]:
        # an anonymous mapping cannot be pickled: the receiver gets its own copy of the bytes
        return {"n_bytes": self.n_bytes, "data": bytes(self._mm[:self.n_bytes])}

    def __setstate__(self, state: Dict[str, Any]) -> None:
        self.__init__(state["n_bytes"])
        self._mm[:self.n_bytes] = state["data"]


class TextDataset(MultifieldDataset):
    FIELD_KEY = "line"
    PAD = 0

    def __init__(self, data_type: Split, txt_file_path: PathLike, transform, seq_len: int, *,
                 device_transform=None) -> None:
        """``device_transform``: the batched twin of ``transform``
        (``transform.DeviceBatchTransform``); with it the loop serves this split through
        ``DeviceBatchLoader`` instead of per-sample ``__getitem__``."""
        path = _fs_path(txt_file_path)
        self._corpus = HostCorpus.from_file(path)
        self._sample_indices = line_starts(self._corpus.array)
        logger.info("Loaded %s: %d bytes, %d samples", path, self._corpus.n_bytes, len(self))
        self._seq_len = seq_len + 1
        self.data_type = data_type
        self._transform = transform
        self.pinned_fields = {self.FIELD_KEY: PaddedLines(self._corpus, self._sample_indices,
                                                          self._seq_len, self.PAD)}
        if device_transform is not None:
            self.device_transform = device_transform

    def __len__(self) -> int:
        return len(self._sample_indices) - 1

    def get_raw_item(self, idx: int) -> Dict[DatasetField, np.ndarray]:
        full = self._corpus.array[self._sample_indices[idx]:self._sample_indices[idx + 1] - 1]
        n = min(self._seq_len, full.shape[0])
        packed = np.full((self._seq_len,), self.PAD, dtype=np.uint8)
        packed[:n] = full[:n]
        return {self.FIELD_KEY: packed}

    def __getitem__(self, idx: int):
        return self._transform(self.get_raw_item(idx), split=self.data_type)

    def set_accessor(self, accessor) -> None:
        pass
