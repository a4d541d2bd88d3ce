"""Symmetric (peer- and multicast-mapped) arena memory for the fused NVLS step.

The gradient arena and the weight vector every rank's module reads (bf16 shadow, or the fp32
master in FP32 mode) are allocated through ``torch.distributed._symmetric_memory`` so each has
the same offset on every GPU of the box, a multicast address on the NVSwitch and a signal pad.
PyTorch is used for the plumbing only (cuMem/multicast object setup and handle exchange); the
kernel that uses the mappings is ``frl_nvls_*`` (csrc/nvls.cu).
"""
import logging
import os
from typing import Optional

import torch
import torch.distributed as dist

logger = logging.getLogger(__name__)


class NvlsLink:
    """What the K7 launches need besides the bucket pointers."""
    __slots__ = ("rank", "world", "pads_dev", "pad_base", "max_blocks", "tail_blocks", "mc_grad", "mc_out",
                 "grad_esz", "out_esz", "handles", "scratch", "flags")

    def __init__(self):
        self.handles = []


class SymmetricAllocator:
    def __init__(self, device: torch.device, group=None) -> None:
        import torch.distributed._symmetric_memory as symm_mem
        self._sm = symm_mem
        self.device = device
        self.group = group if group is not None else dist.group.WORLD
        self.handles = {}
        try:        # needed by older torch releases, a deprecated no-op on newer ones
            import warnings
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                symm_mem.enable_symm_mem_for_group(self.group.group_name)
        except Exception:                            # noqa: BLE001
            pass

    def __call__(self, numel: int, dtype: torch.dtype) -> torch.Tensor:
        t = self._sm.empty(numel, dtype=dtype, device=self.device)
        hdl = self._sm.rendezvous(t, self.group)
        t.zero_()
        self.handles[t.data_ptr()] = hdl
        return t

    def handle_of(self, t: torch.Tensor):
        return self.handles[t.data_ptr()]


def try_make_allocator(device: torch.device, world_size: int) -> Optional[SymmetricAllocator]:
    """Allocator if this process group can use NVSwitch multicast, else None (NCCL path)."""
    if world_size < 2 or device.type != "cuda" or os.environ.get("FRL_B200_NVLS", "1") == "0":
        return None
    try:
        alloc = SymmetricAllocator(device)
        probe = alloc(1024, torch.float32)
        ok = alloc.handle_of(probe).multicast_ptr != 0
    except Exception as e:                           # noqa: BLE001
        logger.info("symmetric memory unavailable (%s): using NCCL all-reduce", e)
        alloc, ok = None, False
    flag = torch.tensor([1 if ok else 0], device=device)
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    if int(flag.item()) != 1:
        logger.info("NVSwitch multicast not available on every rank: using NCCL all-reduce")
        return None
    return alloc


def make_link(alloc: SymmetricAllocator, grad: torch.Tensor, out: torch.Tensor,
              max_blocks: int = 32, tail_blocks: int = 0) -> NvlsLink:
    hg, ho = alloc.handle_of(grad), alloc.handle_of(out)
    link = NvlsLink()
    link.rank, link.world = hg.rank, hg.world_size
    link.pads_dev = hg.signal_pad_ptrs_dev
    link.pad_base = 0
    if hg.signal_pad_size // 4 < 64 or link.world > 32:
        raise RuntimeError("signal pad too small")
    link.max_blocks = max(1, min(max_blocks, 1024))
    # grid of the launch for the bucket that becomes ready LAST: nothing of backward runs beside it
    # any more, so it may take the SMs the other launches leave to the GEMMs (0 = same grid)
    link.tail_blocks = max(1, min(tail_blocks, 1024)) if tail_blocks > 0 else link.max_blocks
    link.scratch = torch.zeros(8 + max(link.max_blocks, link.tail_blocks), dtype=torch.int32, device=grad.device)
    link.mc_grad, link.mc_out = hg.multicast_ptr, ho.multicast_ptr
    link.grad_esz, link.out_esz = grad.element_size(), out.element_size()
    link.handles = [hg, ho]
    # barriers inside the update kernel (default; not tuned on H100) or as
    # separate 1-CTA launches (wins when the grid is large and ranks arrive skewed)
    link.flags = 1 if os.environ.get("FRL_B200_NVLS_SPLIT_SYNC", "0") != "0" else 0
    if link.mc_grad == 0 or link.mc_out == 0:
        raise RuntimeError("no multicast mapping")
    return link
