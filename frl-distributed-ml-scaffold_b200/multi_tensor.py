"""Segment tables for the multi-tensor kernels (``frl_flatten_grads``, ``frl_*_mt``).

A ``GradSegTable`` describes a run of arena slots: per slot the arena offset and length (fixed)
and where this step's gradient lies (changes every eager step — autograd allocates gradient
tensors afresh — and is fixed inside a captured CUDA graph).  The working copy is plain host
memory; an upload snapshots it into the next row of a small ring of pinned buffers and issues one
asynchronous copy from there (an async copy reads its pinned source when it EXECUTES, and the host
runs a few steps ahead of the device: the ring keeps step k's pointers intact until step k's copy
has run — the loop's lagged loss check bounds the host's lead to NAN_CHECK_LAG + 1 steps).
"""
import ctypes as C
from typing import Dict, List, Optional, Sequence

import torch

from . import _native

_SEG_BYTES = C.sizeof(_native.GradSeg)


def grad_usable_in_place(g: torch.Tensor, slot) -> bool:
    """Can the kernels read ``g`` where it is?  Dense, in the parameter's own (contiguous)
    layout, fp32 or bf16, 16-byte aligned — what cuDNN / cuBLAS / the normalisation kernels hand
    to autograd.  Anything else (channels_last weight gradients, sparse, fp16, odd views) is
    copied into the arena slice by the caller instead."""
    return (g.is_cuda and g.layout == torch.strided and g.is_contiguous()
            and g.dtype in (torch.float32, torch.bfloat16) and g.numel() == slot.numel
            and g.data_ptr() % 16 == 0)


class GradSegTable:
    RING = 8

    def __init__(self, slots: Sequence, device: torch.device) -> None:
        self.slots = list(slots)
        self.n_segs = len(self.slots)
        self.device = device
        tile = _native.mt_tile_elems()
        prefix = [0]
        for s in self.slots:
            prefix.append(prefix[-1] + (((s.numel + 3) // 4 * 4) + tile - 1) // tile)
        self.n_tiles = prefix[-1]
        nbytes = max(self.n_segs, 1) * _SEG_BYTES
        self._host = torch.zeros(nbytes, dtype=torch.uint8)
        self._segs = (_native.GradSeg * max(self.n_segs, 1)).from_address(self._host.data_ptr())
        self._ring = torch.zeros(self.RING, nbytes, dtype=torch.uint8, pin_memory=device.type == "cuda")
        self._ring_i = 0
        for i, s in enumerate(self.slots):
            self._segs[i].arena_off = s.offset
            self._segs[i].numel = s.numel
        self._dev = torch.zeros(nbytes, dtype=torch.uint8, device=device)
        self._prefix_dev = torch.tensor(prefix, dtype=torch.int64, device=device)
        counts = torch.tensor([b - a for a, b in zip(prefix[:-1], prefix[1:])], dtype=torch.int64)
        self._tile_seg_dev = torch.repeat_interleave(torch.arange(self.n_segs, dtype=torch.int32),
                                                     counts).to(device) if self.n_segs else \
            torch.zeros(1, dtype=torch.int32, device=device)
        self._row_of: Dict[int, int] = {s.index: i for i, s in enumerate(self.slots)}
        self._dirty = True
        self.external = 0            # slots whose gradient currently lies outside the arena

    @property
    def segs_dev_ptr(self) -> int:
        return self._dev.data_ptr()

    @property
    def prefix_dev_ptr(self) -> int:
        return self._prefix_dev.data_ptr()

    @property
    def tile_seg_dev_ptr(self) -> int:
        return self._tile_seg_dev.data_ptr()

    def point(self, slot, ptr: int, dtype: torch.dtype) -> None:
        row = self._segs[self._row_of[slot.index]]
        code = _native.dtype_code(dtype)
        if (row.g or 0) != ptr or row.g_dtype != code:       # ctypes reads a NULL pointer as None
            row.g = ptr
            row.g_dtype = code
            self._dirty = True

    def upload(self) -> None:
        """Make the device copy current on the current stream (no-op when no pointer changed since
        the last upload)."""
        if self._dirty and self.n_segs:
            row = self._ring[self._ring_i % self.RING]
            self._ring_i += 1
            row.copy_(self._host)
            self._dev.copy_(row, non_blocking=True)
            self._dirty = False
