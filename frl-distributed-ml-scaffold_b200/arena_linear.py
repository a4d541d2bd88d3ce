"""``nn.Linear`` whose parameter gradients are born in the gradient arena.

The reference lets autograd allocate ``weight.grad`` wherever the caching allocator pleases and
DDP then copies it into a bucket, pre-divides, all-reduces and copies it back (reference
solver.py:287-289 -> torch Reducer).  For exact ``nn.Linear`` modules — the layers where a
Problem's forward really is a dense contraction — the solver swaps the module's ``forward`` for
one autograd Function, ``_ArenaLinearFn``, while the model is wrapped:

  forward   y = x W^T + b                      (cuBLAS, unchanged)
  backward  dX = dY W                          (cuBLAS)
            dW = dY^T X   written by cuBLAS straight into the weight's slice of the grad arena
            db = colsum(dY) by ``frl_colsum`` straight into the bias's slice

so the bucket NCCL reduces is complete the moment the layer's backward returns: no flatten
copy, no separate bias-reduction pass through a generic reduce kernel.  Outside a pipeline
step (``autograd.grad`` calls of GradNorm / debugGrad) the Function returns ordinary gradients.

Unless ``FRL_B200_FUSE_RELU=0``, a ``nn.Linear`` directly followed by a ``nn.ReLU`` inside a
``nn.Sequential`` (each module used exactly once, no hooks) runs as one unit:

  forward   y = relu(x W^T + b)                one cuBLASLt GEMM with the bias+ReLU epilogue
                                               (``torch._addmm_activation``); the ReLU module
                                               becomes a pass-through
  backward  dZ = threshold_backward(dY, y, 0), ONE pass (``frl_drelu_colsum``, K6b) instead of
            db = colsum(dZ)                    threshold_backward + a reduction
            dX = dZ W, dW = dZ^T X             as above

In a ``Precision.FP8`` run a site whose weight lives in the bf16 shadow and whose widths are
multiples of 16 (``fp8_site_qualifies``) runs its three GEMMs on the FP8 tensor cores
(``torch._scaled_mm``, tensor-wise scales, bf16 output, fp32 accumulation) for every call whose
flattened row count is a multiple of 16; other calls take the bf16 GEMMs above.  Each operand
is quantised by K9 at a power-of-two scale from its own amax (``frl_fp8_amax`` +
``frl_fp8_quantize``), one pass giving the row-major copy and, for backward, the transposed one:

  forward   Y  = Xq Wq^T (+ b)        Xq, Wq e4m3; saved for backward: Xq^T, Wq^T (not bf16 X)
  backward  dX = dZq (Wq^T)^T         dZq e5m2
            dW = dZq^T (Xq^T)^T       into the arena as above; db as above

Whatever the variant, backward runs one protocol: form dZ (on a ReLU site inside a step,
``frl_drelu_colsum`` writes the bias gradient with it), compute dX, and only then write dW
(``LinearSite.weight_grad``), the bias gradient if not yet written, and mark the slots ready
(``LinearSite.backward_done``): marking a slot ready can launch the bucket's update, which
overwrites W.  So can the dW GEMM itself: on one GPU with SGD (``GradBucketPipeline.fused_dw_update``)
a bf16 weight applied once per forward whose shape fits the tile gets its gradient and its update
from one kernel (``frl_dw_gemm_sgd``, K12).
"""
import os
import types
from collections import Counter
from typing import List, Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _native
from .types import Precision

KERNELS = _native

#: FP8 GEMM operands need K, N (and, for the weight gradient, M) to be multiples of 16
FP8_MULTIPLE = 16


def fp8_site_qualifies(uses_lp: bool, in_features: int, out_features: int) -> bool:
    """Whether an FP8 run runs a Linear site's GEMMs in FP8 (the row count is checked per call):
    the weight lives in the bf16 shadow and both widths are multiples of 16."""
    return bool(uses_lp) and in_features % FP8_MULTIPLE == 0 and out_features % FP8_MULTIPLE == 0


def fp8_call_qualifies(x: torch.Tensor) -> bool:
    """Per call: a bf16/fp32 input whose flattened row count is a positive multiple of 16 and
    whose rows start on a 16-byte boundary (a contiguous input is quantised in place; any other
    is copied first)."""
    if x.dim() == 0 or x.shape[-1] == 0 or x.dtype not in (torch.bfloat16, torch.float32):
        return False
    m = x.numel() // x.shape[-1]
    return m > 0 and m % FP8_MULTIPLE == 0 and (not x.is_contiguous() or x.data_ptr() % 16 == 0)


def _fp8_quantize(t2: torch.Tensor, fmt: int, rowmajor: bool, transposed: bool):
    """(row-major codes or None, transposed codes or None, 1/scale as a device scalar) of the
    contiguous 2-D ``t2`` at the scale its own amax implies (K9: two launches, no host sync)."""
    sc = torch.empty(2, dtype=torch.float32, device=t2.device)          # [amax, 1/scale]
    dt = _native.FP8_DTYPE[fmt]
    q = torch.empty(t2.shape, dtype=dt, device=t2.device) if rowmajor else None
    qt = torch.empty((t2.shape[1], t2.shape[0]), dtype=dt, device=t2.device) if transposed else None
    KERNELS.fp8_amax(t2, sc[:1])
    KERNELS.fp8_quantize(t2, sc[:1], fmt, q, qt, sc[1:])
    return q, qt, sc[1]


def _fp8_mm(a, b_t, scale_a, scale_b, bias=None, out=None):
    """a @ b_t^T in bf16 for row-major fp8 ``a`` [M, K] and ``b_t`` [N, K] (b_t.t() is the
    column-major [K, N] operand ``torch._scaled_mm`` wants)."""
    return torch._scaled_mm(a, b_t.t(), scale_a, scale_b, bias=bias, out_dtype=torch.bfloat16,
                            use_fast_accum=False, out=out)


def _fp8_operands(x, weight, transposed: bool):
    x2 = x.reshape(-1, x.shape[-1])
    if not x2.is_contiguous():
        x2 = x2.contiguous()
    xq, xtq, sx = _fp8_quantize(x2, _native.FP8_E4M3, True, transposed)
    wq, wtq, sw = _fp8_quantize(weight, _native.FP8_E4M3, True, transposed)
    return xq, xtq, sx, wq, wtq, sw


class _DenseGemms:
    """dX and dW of a dense (bf16/fp32) site from its saved (X, W) and dZ [M, N]."""
    row_multiple = 1

    def __init__(self, saved, dz, need_dx):
        x, self.weight = saved[0], saved[1]
        self.x2 = x.reshape(-1, x.shape[-1])
        self.dz, self.dzt = dz, dz.t()

    def dx(self):
        return self.dz.matmul(self.weight)

    def dw(self, dzt, out=None):
        """Rows of dW = dZ^T X for the rows ``dzt`` of dZ^T."""
        return torch.mm(dzt, self.x2, out=out)

    def dw_add(self, gw):
        gw.addmm_(self.dzt, self.x2)


class _Fp8Gemms:
    """The same on the FP8 tensor cores from the saved Xq^T, Wq^T and their scales: dZ is quantised
    to e5m2, the row-major copy only if dX is needed.  A row block of dW must be a multiple of 16
    rows."""
    row_multiple = FP8_MULTIPLE

    def __init__(self, saved, dz, need_dx):
        self.xtq, self.wtq, self.sx, self.sw = saved[:4]
        self.dzq, self.dzt, self.sdz = _fp8_quantize(dz, _native.FP8_E5M2, need_dx, True)

    def dx(self):
        return _fp8_mm(self.dzq, self.wtq, self.sdz, self.sw)

    def dw(self, dzt, out=None):
        return _fp8_mm(dzt, self.xtq, self.sdz, self.sx, out=out)

    def dw_add(self, gw):
        gw.add_(self.dw(self.dzt))


class _ArenaLinearFn(torch.autograd.Function):
    """One Linear site, with the ReLU it absorbed if it has one (``site.relu``), with dense or FP8
    (``fp8``) GEMMs; see the module docstring.  ``for_backward`` (FP8 only): whether the call
    records a graph (grad mode on and an input requires grad); otherwise nothing is saved and only
    the row-major copies the forward GEMM reads are made."""

    @staticmethod
    def forward(ctx, x, weight, bias, site, fp8, for_backward):
        ctx.site, ctx.fp8, ctx.has_bias, ctx.x_shape = site, fp8, bias is not None, x.shape
        relu = site.relu is not None
        if not (fp8 or relu) and x.dim() <= 2:
            ctx.save_for_backward(x, weight)
            return F.linear(x, weight, bias)
        # N-D input: F.linear would return a VIEW of its 2-D result, and autograd forbids in-place
        # ops (nn.ReLU(inplace=True)) on a view created inside a custom Function: write the GEMM
        # into a 2-D view of a fresh N-D tensor instead and return that tensor
        y = torch.empty(*x.shape[:-1], weight.shape[0], dtype=torch.bfloat16 if fp8 else x.dtype,
                        device=x.device)
        y2 = y.view(-1, weight.shape[0])
        if fp8:
            xq, xtq, sx, wq, wtq, sw = _fp8_operands(x, weight, for_backward)
            _fp8_mm(xq, wq, sx, sw, bias=bias, out=y2)
            if relu:
                y.relu_()
            saved = (xtq, wtq, sx, sw) if for_backward else ()
        else:
            x2 = x.reshape(-1, x.shape[-1])
            if relu:
                torch._addmm_activation(bias, x2, weight.t(), use_gelu=False, out=y2)
            elif bias is not None:
                torch.addmm(bias, x2, weight.t(), out=y2)
            else:
                torch.mm(x2, weight.t(), out=y2)
            saved = (x, weight)
        if relu and saved:
            saved += (y,)
        ctx.save_for_backward(*saved)
        return y

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, dy):
        site, saved = ctx.site, ctx.saved_tensors
        relu = site.relu is not None
        pipe = site.pipeline
        in_step = pipe is not None and pipe.step_open
        dz = dy.reshape(-1, dy.shape[-1])
        if relu or ctx.fp8:
            dz = dz.contiguous()
        db_written = False
        if relu:
            y2 = saved[-1].reshape(-1, dz.shape[1])
            if in_step:                              # dZ and the bias gradient in one pass
                dz_relu = torch.empty_like(dz)
                KERNELS.drelu_colsum(dz, y2, dz_relu, pipe.arena.grad_view(site.bslot),
                                     accumulate=not site.bstate.first_touch(pipe.step_id))
                dz, db_written = dz_relu, True
            else:
                dz = torch.ops.aten.threshold_backward(dz, y2, 0)     # stock ReLU backward, NaN/inf included
        need_dx = ctx.needs_input_grad[0]
        gemms = (_Fp8Gemms if ctx.fp8 else _DenseGemms)(saved, dz, need_dx)
        # dX first: marking the weight's slot ready may launch the bucket's update on the side
        # stream, and that update overwrites the very weight dX = dZ W reads
        dx = gemms.dx().view(ctx.x_shape) if need_dx else None
        if in_step:
            site.weight_grad(pipe, gemms)
            if ctx.has_bias and not db_written and site.bslot is not None:
                KERNELS.colsum(dz.contiguous(), pipe.arena.grad_view(site.bslot),
                               accumulate=not site.bstate.first_touch(pipe.step_id))
            site.backward_done(pipe)
            return dx, None, None, None, None, None
        dw = gemms.dw(gemms.dzt) if ctx.needs_input_grad[1] else None
        db = dz.sum(0) if (ctx.has_bias and ctx.needs_input_grad[2]) else None
        return dx, dw, db, None, None, None


class _ArenaMultiHeadFn(torch.autograd.Function):
    """All task heads of a ``MultiTaskModel`` (exact ``nn.Linear`` layers on the same trunk
    output) as one autograd unit.  Forward: one GEMM per head, as before (their outputs are
    separate tensors for the criterion).  Backward: the heads' weights lie back to back in the
    arena (``ParamArena(adjacent=...)``), so with dY = [dY_1 | ... | dY_T]

        dX   = dY W_cat            ONE GEMM instead of T GEMMs and T-1 accumulate passes
        dW   = dY^T X              ONE GEMM writing every head's weight gradient in place
        db   = colsum(dY)          ONE launch when the biases are adjacent too, else one per head
    """

    @staticmethod
    def forward(ctx, x, site, *params):
        ctx.site = site
        ctx.save_for_backward(x)
        ctx.n_heads = len(params) // 2
        return tuple(F.linear(x, params[2 * i], params[2 * i + 1]) for i in range(ctx.n_heads))

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, *dys):
        (x,) = ctx.saved_tensors
        site = ctx.site
        pipe = site.pipeline
        dy = torch.cat(dys, dim=1)
        dx = dy.matmul(site.weight_cat()) if ctx.needs_input_grad[0] else None
        none = (None,) * (2 * ctx.n_heads)
        if pipe is not None and pipe.step_open:
            gw = site.grad_weight_cat()
            if site.heads[0].wstate.first_touch(pipe.step_id):
                torch.mm(dy.t(), x, out=gw)
            else:
                gw.addmm_(dy.t(), x)
            for h in site.heads[1:]:
                h.wstate.first_touch(pipe.step_id)
            gb = site.grad_bias_cat()
            if gb is not None:
                first = site.heads[0].bstate.first_touch(pipe.step_id)
                for h in site.heads[1:]:
                    h.bstate.first_touch(pipe.step_id)
                KERNELS.colsum(dy, gb, accumulate=not first)
            else:
                for h, dyi in zip(site.heads, dys):
                    KERNELS.colsum(dyi.contiguous(), pipe.arena.grad_view(h.bslot),
                                   accumulate=not h.bstate.first_touch(pipe.step_id))
            for h in site.heads:
                h.backward_done(pipe)
            return (dx, None) + none
        grads = []
        for i, dyi in enumerate(dys):
            grads += [dyi.t().mm(x) if ctx.needs_input_grad[2 + 2 * i] else None,
                      dyi.sum(0) if ctx.needs_input_grad[3 + 2 * i] else None]
        return (dx, None) + tuple(grads)


class MultiHeadSite:
    """The task heads of one ``MultiTaskModel`` whose weights (and, if their sizes allow, biases)
    are adjacent in the arena."""

    def __init__(self, model, heads: List["LinearSite"], pipeline) -> None:
        self.model = model
        self.heads = heads
        self.pipeline = pipeline
        arena = pipeline.arena
        self.rows = sum(h.module.out_features for h in heads)
        self.cols = heads[0].module.in_features
        self._w_lo = heads[0].wslot.offset
        ends = [h.wslot.end for h in heads]
        starts = [h.wslot.offset for h in heads]
        assert all(e == s for e, s in zip(ends[:-1], starts[1:])), "head weights are not adjacent"
        self._w_hi = ends[-1]
        b_adjacent = all(h.bslot.end == n.bslot.offset for h, n in zip(heads[:-1], heads[1:]))
        self._b = (heads[0].bslot.offset, heads[-1].bslot.end) if b_adjacent else None
        self._arena = arena

    def weight_cat(self) -> torch.Tensor:
        a = self._arena
        store = a.lp if self.heads[0].wslot.uses_lp else a.master
        return store[self._w_lo:self._w_hi].view(self.rows, self.cols)

    def grad_weight_cat(self) -> torch.Tensor:
        return self._arena.grad[self._w_lo:self._w_hi].view(self.rows, self.cols)

    def grad_bias_cat(self) -> Optional[torch.Tensor]:
        return None if self._b is None else self._arena.grad[self._b[0]:self._b[1]]


def head_layout_groups(model: nn.Module) -> List[List[nn.Parameter]]:
    """Parameter groups ``ParamArena(adjacent=...)`` should lay out back to back so the heads of a
    ``MultiTaskModel`` can run as one backward unit: [all head weights], [all head biases]."""
    from .model import MultiTaskModel
    if type(model) is not MultiTaskModel or os.environ.get("FRL_B200_FUSE_HEADS", "1") == "0":
        return []
    heads = list(model.additional_layers)
    if len(heads) < 2 or any(type(h) is not nn.Linear or h.bias is None for h in heads):
        return []
    if len({h.in_features for h in heads}) != 1 or len({id(h.weight) for h in heads}) != len(heads):
        return []
    return [[h.weight for h in heads], [h.bias for h in heads]]


def _multihead_forward(self, x):
    site = self._frl_heads
    shared = self.model_base(x)
    if shared.dim() == 2 and torch.is_grad_enabled() and shared.is_contiguous():
        params = []
        for h in site.heads:
            h.count_forward()
            params += [h.module.weight, h.module.bias]
        return list(_ArenaMultiHeadFn.apply(shared, site, *params))
    return [head(shared) for head in self.additional_layers]


class SlotState:
    """Per-PARAMETER bookkeeping shared by every site that uses the parameter (a module applied
    several times per forward, or weights tied across modules): which step first wrote the
    gradient slice (store vs. accumulate) and how many backward passes are still to come."""
    __slots__ = ("touched_step", "fwd_gen", "fwd_count", "bwd_step", "bwd_count")

    def __init__(self) -> None:
        self.touched_step = -1
        self.fwd_gen = -1
        self.fwd_count = 0
        self.bwd_step = -1
        self.bwd_count = 0

    def first_touch(self, step_id: int) -> bool:
        first = self.touched_step != step_id
        self.touched_step = step_id
        return first

    def count_forward(self, gen: int) -> None:
        if self.fwd_gen != gen:
            self.fwd_gen, self.fwd_count = gen, 0
        self.fwd_count += 1

    def backward_complete(self, step_id: int, gen: int) -> bool:
        """One more backward pass through a user of this parameter; True when every forward
        application counted for this step has been matched (unknown count = complete)."""
        if self.bwd_step != step_id:
            self.bwd_step, self.bwd_count = step_id, 0
        self.bwd_count += 1
        return self.fwd_gen != gen or self.bwd_count >= self.fwd_count


class LinearSite:
    """Per-module bookkeeping: arena slots of weight/bias and the owning pipeline.

    A bucket must not be reduced/updated before the LAST contribution to each of its gradients
    has been accumulated (stock DDP waits for autograd's AccumulateGrad, which runs once per
    parameter per backward).  Here gradients are written from inside the layer's backward, so the
    site counts its applications in the forward pass (training mode, autograd on) and marks its
    slots ready only when as many backward passes have run; anything left over is marked by
    ``GradBucketPipeline.finish_step`` (after ``backward()`` returned nothing can be missing)."""
    __slots__ = ("module", "wslot", "bslot", "pipeline", "relu", "wstate", "bstate", "multihead", "fp8")

    def __init__(self, module, wslot, bslot, pipeline):
        self.module = module
        self.wslot = wslot
        self.bslot = bslot
        self.pipeline = pipeline
        self.relu = None              # the nn.ReLU this layer absorbed (FRL_B200_FUSE_RELU)
        self.multihead = None         # on the first head: the MultiHeadSite of its model
        self.fp8 = False              # Precision.FP8 and fp8_site_qualifies: FP8 GEMMs per call
        states = pipeline.slot_states
        self.wstate = states.setdefault(wslot.index, SlotState())
        self.bstate = states.setdefault(bslot.index, SlotState()) if bslot is not None else None

    def weight_grad(self, pipe, gemms) -> None:
        """dW = dZ^T X by ``gemms`` (``_DenseGemms`` / ``_Fp8Gemms``) into the weight's arena slice
        (store on the step's first touch, accumulate after).  A weight the pipeline exchanges in two
        row blocks (``row_split``: the layer whose dW ends backward) is computed as two GEMMs and
        the first block handed over in between, provided this is the parameter's only application
        in the step and the block is a multiple of ``gemms.row_multiple`` rows."""
        gw = pipe.arena.grad_view(self.wslot)
        st = self.wstate
        if not st.first_touch(pipe.step_id):
            gemms.dw_add(gw)
            return
        rows = pipe.row_split(self.wslot)
        only_use = st.fwd_gen == pipe.forward_gen and st.fwd_count == 1
        if rows and rows % gemms.row_multiple == 0 and only_use:
            gemms.dw(gemms.dzt[:rows], out=gw[:rows])
            pipe.rows_ready(self.wslot, rows)
            gemms.dw(gemms.dzt[rows:], out=gw[rows:])
        elif (pipe.fused_dw_update and only_use and not rows and type(gemms) is _DenseGemms
              and self.wslot.uses_lp and _native.dw_gemm_fits(gemms.dz, gemms.x2, gw)):
            pipe.update_in_dw_gemm(self.wslot, gemms.dz, gemms.x2, gw)
        else:
            gemms.dw(gemms.dzt, out=gw)

    def count_forward(self) -> None:
        pipe = self.pipeline
        if pipe is not None and self.module.training and torch.is_grad_enabled():
            gen = pipe.forward_gen
            self.wstate.count_forward(gen)
            if self.bstate is not None:
                self.bstate.count_forward(gen)

    def backward_done(self, pipe) -> None:
        step, gen = pipe.step_id, pipe.forward_gen
        if self.wstate.backward_complete(step, gen):
            pipe.mark_ready(self.wslot)
        else:
            pipe.defer_ready(self.wslot)
        if self.bstate is not None:
            if self.bstate.backward_complete(step, gen):
                pipe.mark_ready(self.bslot)
            else:
                pipe.defer_ready(self.bslot)


def _for_backward(*tensors) -> bool:
    return torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in tensors)


def _forward(self, x):
    site = self._frl_site
    site.count_forward()                  # here, not inside the Function: grad mode is off in there
    fp8 = site.fp8 and fp8_call_qualifies(x)
    return _ArenaLinearFn.apply(x, self.weight, self.bias, site, fp8,
                                fp8 and _for_backward(x, self.weight, self.bias))


def _identity(self, x):
    return x


def _has_hooks(mod: nn.Module) -> bool:
    return bool(mod._forward_hooks or mod._forward_pre_hooks or mod._backward_hooks
                or getattr(mod, "_backward_pre_hooks", None))


def _fuse_relu_pairs(model: nn.Module, sites: List[LinearSite]) -> int:
    """Mark Linear -> ReLU neighbours of nn.Sequential containers as fused units."""
    uses = Counter(id(child) for mod in model.modules() for child in mod._modules.values()
                   if child is not None)
    by_module = {id(s.module): s for s in sites}
    fused = 0
    for seq in model.modules():
        if type(seq) is not nn.Sequential:
            continue
        kids = list(seq._modules.values())
        for lin, act in zip(kids, kids[1:]):
            site = by_module.get(id(lin))
            if site is None or site.bslot is None or type(act) is not nn.ReLU or site.relu is not None:
                continue
            if uses[id(lin)] != 1 or uses[id(act)] != 1 or _has_hooks(lin) or _has_hooks(act):
                continue
            if "forward" in act.__dict__:
                continue
            site.relu = act
            fused += 1
    return fused


def patch_linears(model: nn.Module, pipeline) -> List[LinearSite]:
    """Route every exact ``nn.Linear`` whose weight lives in the arena through the Function."""
    sites: List[LinearSite] = []
    arena = pipeline.arena
    for mod in model.modules():
        if type(mod) is not nn.Linear or "forward" in mod.__dict__:
            continue
        if id(mod.weight) not in arena._by_id:
            continue
        if not mod.weight.is_cuda and KERNELS is _native:
            continue                     # the kernels are CUDA-only (CPU tensors: host-logic tests)
        wslot = arena.slot_of(mod.weight)
        bslot = arena.slot_of(mod.bias) if (mod.bias is not None and id(mod.bias) in arena._by_id) else None
        if mod.bias is not None and bslot is None:
            continue                     # frozen bias: leave the module alone
        site = LinearSite(mod, wslot, bslot, pipeline)
        site.fp8 = (arena.precision is Precision.FP8
                    and fp8_site_qualifies(wslot.uses_lp, mod.in_features, mod.out_features))
        sites.append(site)
    if os.environ.get("FRL_B200_FUSE_RELU", "1") != "0":
        _fuse_relu_pairs(model, sites)
    _attach_multihead(model, sites, pipeline)
    for site in sites:
        if site.multihead is not None:              # the fused task heads stay bf16
            for h in site.multihead.heads:
                h.fp8 = False
    repatch_linears(sites)
    return sites


def _attach_multihead(model: nn.Module, sites: List[LinearSite], pipeline) -> None:
    """Run the heads as one backward unit if the arena laid their weights out adjacently."""
    groups = head_layout_groups(model)
    if not groups or "forward" in model.__dict__ or _has_hooks(model):
        return
    by_module = {id(s.module): s for s in sites}
    heads = [by_module.get(id(h)) for h in model.additional_layers]
    if any(h is None or h.relu is not None or h.bslot is None for h in heads):
        return
    if any(a.wslot.end != b.wslot.offset for a, b in zip(heads[:-1], heads[1:])):
        return                                   # the arena did not honour the weight group
    uses = Counter(id(child) for mod in model.modules() for child in mod._modules.values()
                   if child is not None)
    if any(uses[id(h.module)] != 1 or _has_hooks(h.module) for h in heads):
        return
    msite = MultiHeadSite(model, heads, pipeline)
    for s in sites:
        if s is heads[0]:
            s.multihead = msite


def unpatch_linears(sites: List[LinearSite]) -> None:
    for site in sites:
        site.module.__dict__.pop("forward", None)
        site.module.__dict__.pop("_frl_site", None)
        if site.relu is not None:
            site.relu.__dict__.pop("forward", None)
        if site.multihead is not None:
            site.multihead.model.__dict__.pop("forward", None)
            site.multihead.model.__dict__.pop("_frl_heads", None)


def repatch_linears(sites: List[LinearSite]) -> None:
    for site in sites:
        site.module._frl_site = site
        site.module.forward = types.MethodType(_forward, site.module)
        if site.relu is not None:
            site.relu.forward = types.MethodType(_identity, site.relu)
        if site.multihead is not None:
            site.multihead.model._frl_heads = site.multihead
            site.multihead.model.forward = types.MethodType(_multihead_forward, site.multihead.model)
