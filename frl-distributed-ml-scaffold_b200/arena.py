"""Flat parameter / gradient / optimizer-state arenas in HBM.

Everything the update kernel streams lives in a handful of contiguous fp32 (and bf16) vectors
with one shared element layout:

    master  fp32 [N]   authoritative weights (what checkpoints store)
    lp      bf16 [N]   shadow weights the bf16 forward/backward reads (BF16 mode only)
    grad    [N]        gradient bucket memory, fp32 or bf16 — what NCCL all-reduces in place
    state_k fp32 [N]   optimizer state (momentum / exp_avg / exp_avg_sq / ...), owned by the
                       optimizer, same layout

``param.data`` of every trainable parameter is re-pointed at its slice of ``master`` (FP32
mode) or ``lp`` (BF16 mode, model parameters only), so the user's ``nn.Module`` reads arena
memory directly and one kernel launch over ``[lo, hi)`` updates any contiguous run of tensors.
Slices start at multiples of 8 elements (32 B fp32 / 16 B bf16) so every slice is 128-bit
aligned in both precisions; the padding elements stay zero and are inert under every rule.

This replaces the per-tensor ``torch.optim`` state and the DDP reducer's bucket copies
(reference solver.py:162-188, 287-289).
"""
from contextlib import contextmanager
from typing import Dict, Iterable, List, Optional, Sequence, Tuple

import torch
import torch.nn as nn

from .types import Precision

ALIGN_ELEMS = 8


def _round_up(x: int, a: int) -> int:
    return (x + a - 1) // a * a


class ArenaSlot:
    __slots__ = ("param", "offset", "numel", "shape", "is_model", "uses_lp", "index")

    def __init__(self, param, offset, numel, shape, is_model, uses_lp, index):
        self.param = param
        self.offset = offset
        self.numel = numel
        self.shape = shape
        self.is_model = is_model
        self.uses_lp = uses_lp
        self.index = index          # position in the optimizer's flat parameter list

    @property
    def end(self) -> int:
        return self.offset + self.numel


class ParamArena:
    def __init__(self, model_params: Iterable[nn.Parameter],
                 criterion_params: Iterable[nn.Parameter] = (),
                 *, device: torch.device, precision: Precision = Precision.FP32,
                 shared_allocator=None, adjacent: Sequence[Sequence[nn.Parameter]] = ()) -> None:
        """``shared_allocator(numel, dtype) -> zeroed tensor``: where the vectors other ranks must
        reach (``grad`` and the weights the modules read) come from — symmetric/multicast memory
        for the fused NVLS step; default ``torch.zeros``.

        ``adjacent``: groups of model parameters to lay out back to back, in the given order,
        where the first member would have gone (e.g. the weights of all task heads, so that one
        GEMM can treat them as a single [sum(C_i), K] matrix).  A group is honoured only if every
        member but the last has a multiple of 8 elements (no padding in between); the slot list
        stays sorted by offset, ``ArenaSlot.index`` keeps the optimizer's parameter position."""
        self.device = torch.device(device)
        self.precision = precision
        self.all_params: List[nn.Parameter] = []
        self.slots: List[ArenaSlot] = []
        seen = set()
        off = 0
        model_params = list(model_params)
        criterion_params = list(criterion_params)
        # optimizer positions follow the reference's parameter order, whatever the layout
        position, uniq = {}, []
        for p in model_params + criterion_params:
            if id(p) not in position:
                position[id(p)] = len(uniq)
                uniq.append(p)
        self.all_params = uniq
        model_ids = {id(p) for p in model_params}
        lead = {}                                     # id(first member) -> whole group
        grouped = set()
        self.adjacent_groups: List[List[nn.Parameter]] = []
        for group in adjacent:
            group = list(group)
            ok = (len(group) >= 2 and all(id(p) in model_ids and p.requires_grad for p in group)
                  and len({id(p) for p in group}) == len(group)
                  and not any(id(p) in grouped for p in group)
                  and all(p.numel() % ALIGN_ELEMS == 0 for p in group[:-1]))
            if ok:
                lead[id(group[0])] = group
                grouped.update(id(p) for p in group)
                self.adjacent_groups.append(group)

        def laid_out(params):
            for p in params:
                if id(p) in lead:
                    yield from lead[id(p)]
                elif id(p) not in grouped:
                    yield p

        for is_model, group in ((True, list(laid_out(model_params))), (False, criterion_params)):
            for p in group:
                if id(p) in seen:
                    continue
                seen.add(id(p))
                idx = position[id(p)]
                if not p.requires_grad:
                    continue
                if p.dtype != torch.float32:
                    raise TypeError(f"arena expects fp32 parameters at wrap time, got {p.dtype}")
                uses_lp = is_model and precision.bf16_storage
                self.slots.append(ArenaSlot(p, off, p.numel(), tuple(p.shape), is_model, uses_lp, idx))
                off = _round_up(off + p.numel(), ALIGN_ELEMS)
            if is_model:
                self.model_end = off        # padded end of the model-parameter range
        self.numel = off
        self.grad_dtype = torch.bfloat16 if precision.bf16_storage else torch.float32

        def shared(dtype):
            if shared_allocator is not None and self.numel > 0:
                return shared_allocator(self.numel, dtype)
            return torch.zeros(self.numel, dtype=dtype, device=self.device)

        bf16_mode = precision.bf16_storage
        self.master = (torch.zeros(self.numel, dtype=torch.float32, device=self.device)
                       if bf16_mode else shared(torch.float32))
        with torch.no_grad():
            for s in self.slots:
                self.master[s.offset:s.end].copy_(s.param.detach().reshape(-1))
        self.lp: Optional[torch.Tensor] = None
        if bf16_mode:
            self.lp = shared(torch.bfloat16)
            self.lp.copy_(self.master)
        self.grad = shared(self.grad_dtype)
        self._by_id: Dict[int, ArenaSlot] = {id(s.param): s for s in self.slots}
        self._repoint()

    # -- views ---------------------------------------------------------------------------------
    def _storage_for(self, s: ArenaSlot) -> torch.Tensor:
        return self.lp if s.uses_lp else self.master

    def _repoint(self) -> None:
        for s in self.slots:
            s.param.data = self._storage_for(s)[s.offset:s.end].view(s.shape)
            s.param.grad = None

    def slot_of(self, p: nn.Parameter) -> ArenaSlot:
        return self._by_id[id(p)]

    def grad_view(self, s: ArenaSlot) -> torch.Tensor:
        return self.grad[s.offset:s.end].view(s.shape)

    def master_view(self, s: ArenaSlot) -> torch.Tensor:
        return self.master[s.offset:s.end].view(s.shape)

    def new_state(self) -> torch.Tensor:
        return torch.zeros(self.numel, dtype=torch.float32, device=self.device)

    @property
    def n_trainable(self) -> int:
        return sum(s.numel for s in self.slots)

    # -- bf16 shadow maintenance ---------------------------------------------------------------
    def refresh_shadow(self) -> None:
        """master -> lp after the master was written from outside the update kernel."""
        if self.lp is not None:
            self.lp.copy_(self.master)

    def load_master_from_params(self, tensors: Sequence[Tuple[nn.Parameter, torch.Tensor]]) -> None:
        with torch.no_grad():
            for p, value in tensors:
                s = self._by_id.get(id(p))
                if s is None:
                    p.data.copy_(value)
                else:
                    self.master_view(s).copy_(value)
        self.refresh_shadow()

    # -- export --------------------------------------------------------------------------------
    @contextmanager
    def exported(self, cpu: bool = True, module: Optional[nn.Module] = None):
        """Temporarily give every parameter a private fp32 copy of its master weights.

        Inside the block the module pickles / ``state_dict``s exactly like an un-wrapped fp32
        module (what the reference's checkpoint files hold, reference solver.py:632-651).
        ``module``: also present its reduced-precision floating buffers (BatchNorm statistics,
        where a BF16-mode run had to keep them in bf16) as fp32 for the duration.
        """
        saved = []
        saved_bufs = []
        try:
            if module is not None:
                for buf in module.buffers():
                    if buf.is_floating_point() and buf.dtype != torch.float32:
                        saved_bufs.append((buf, buf.data))
                        buf.data = buf.data.float()
            for s in self.slots:
                saved.append((s.param, s.param.data, s.param.grad))
                clone = self.master_view(s).detach().clone()
                s.param.data = clone.cpu() if cpu else clone
                s.param.grad = None
            yield self
        finally:
            for p, data, grad in saved:
                p.data = data
                p.grad = grad
            for buf, data in saved_bufs:
                buf.data = data

    def buckets(self, cap_bytes: int, first_cap_bytes: Optional[int] = None
                ) -> List[Tuple[int, int]]:
        """Contiguous element ranges ``[lo, hi)`` covering the arena, listed in the order their
        gradients become ready (last parameters first), each at most ``cap_bytes`` of gradient
        (a single larger tensor gets its own bucket).  A bucket that is still tiny (< 1 % of the
        cap: a lone bias) when the next tensor would overflow it absorbs that tensor instead of
        closing: a layer's bias and weight gradients are produced by the same backward call, and
        every bucket costs a launch and, with the fused NVLS step, two cross-GPU barriers."""
        esz = 2 if self.grad_dtype == torch.bfloat16 else 4
        out: List[Tuple[int, int]] = []
        hi = self.numel
        cur_lo = hi
        cap = first_cap_bytes or cap_bytes
        for s in reversed(self.slots):
            if (hi - s.offset) * esz > cap and cur_lo < hi:
                if (hi - cur_lo) * esz * 100 < cap_bytes:      # tiny open bucket: take the tensor in
                    out.append((s.offset, hi))
                    hi = cur_lo = s.offset
                    cap = cap_bytes
                    continue
                out.append((cur_lo, hi))
                hi = cur_lo
                cap = cap_bytes
            cur_lo = s.offset
        if hi > 0:
            out.append((0, hi))
        return out
