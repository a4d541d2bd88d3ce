"""Per-bucket gradient pipeline: flatten -> all-reduce -> fused update.

Stands where the reference wraps the model in ``DistributedDataParallel`` (reference
solver.py:265-294) and later calls ``clip_grad_norm_`` / ``optimizer.step()`` (reference
solver_worker.py:585-592).  Differences that matter on H100:

* ``nn.Linear`` gradients are written straight into the flat ``grad`` arena by ``arena_linear``;
  every other gradient (convolutions, normalisation layers: cuDNN allocates its own output) is
  left where autograd put it and handed to the kernels through a segment table
  (``multi_tensor.GradSegTable``): on one GPU the fused update reads it in place
  (``frl_*_mt``: no flatten pass at all), with several GPUs ONE ``frl_flatten_grads`` launch per
  bucket gathers the bucket's stragglers into the slice NCCL / the NVLS kernel reduce **in place**
  — no per-tensor copy kernels, no copy-out;
* the 1/world mean and the clip coefficient are folded into the update kernel's gradient read;
* each bucket's all-reduce is issued on a side stream the moment its last gradient is ready and
  its fused update is chained right behind it, overlapping the rest of backward;
* with clipping enabled the updates wait for the global norm (two-phase tail), computed by one
  reduction kernel over the model range with no host sync;
* an optimizer whose update needs whole tensors (``needs_whole_tensors``: LARS, LAMB) takes the
  clipping path's shape: per-bucket all-reduce only, then one update over the whole segment table;
* with gradient accumulation (k > 1) no bucket is launched during backward: one K10 launch per
  microbatch folds every gradient into an fp32 accumulator, and the microbatch that closes a group
  all-reduces the accumulator per bucket, clips and updates from it;
* with a weight EMA (``ema.WeightEMA``) every optimizer update is followed by one K11 launch on the
  compute stream, behind the update and, with eager per-bucket updates, behind the join with the
  side stream; never inside a captured graph (the tail runs after the replay);
* on one GPU with SGD and bf16 shadow weights (``fused_dw_update``), a Linear layer whose dW GEMM
  qualifies (``arena_linear.LinearSite.weight_grad``) updates its weight in that GEMM's epilogue
  (K12), under the tensor-core work of the following tiles; the tail then updates only the slots
  K12 did not (heads, biases, anything else).
"""
import os
from typing import Callable, Dict, List, NamedTuple, Optional, Tuple

import torch
import torch.distributed as dist
import torch.nn as nn

from . import _native
from .arena import ParamArena
from .fused_optim import FusedArenaOptimizer, FusedSGD
from .types import Precision

KERNELS = _native     # swapped by CPU tests of the host logic


class MicroBatch(NamedTuple):
    """Position of one microbatch of a training split under gradient accumulation."""
    first: bool        # opens a group: K10 overwrites the accumulator
    closes: bool       # closes a group: the update runs after its backward
    rows: int          # n_i
    weight: float      # w_i = n_i / B
    group_rows: int    # N: rows of the group it belongs to


def accumulation_plan(n_batches: int, k: int, batch_size: int = 1,
                      n_samples: Optional[int] = None) -> List[MicroBatch]:
    """Groups of ``k`` consecutive microbatches of one split.  Microbatch ``j`` closes a group if
    ``(j + 1) % k == 0`` or it is the split's last, so the last group may be short; no group
    crosses a split.  Every microbatch has ``batch_size`` rows except the last, which has what
    is left of ``n_samples`` (default: a full one)."""
    if n_batches <= 0:
        return []
    last = batch_size if n_samples is None else n_samples - (n_batches - 1) * batch_size
    if not 0 < last <= batch_size:
        raise ValueError("%r samples do not make %d batches of %d" % (n_samples, n_batches, batch_size))
    rows = [batch_size] * (n_batches - 1) + [last]
    plan: List[MicroBatch] = []
    for lo in range(0, n_batches, k):
        group = rows[lo:lo + k]
        n_group = sum(group)
        for i, n in enumerate(group):
            plan.append(MicroBatch(first=i == 0, closes=i == len(group) - 1, rows=n,
                                   weight=n / batch_size, group_rows=n_group))
    return plan


class _TableSet:
    """Segment tables of one pipeline, built on first use, one per (use, set of slots): the step's
    gradients of every slot (K10, the 1-GPU update that reads them in place), per bucket the
    stragglers to flatten, the end-of-step update of the slots that got a gradient, the
    accumulator.  A CUDA-graph capture gets a set of its own: captured uploads read the set's
    pinned rows at every replay, so nothing else may ever rewrite them."""

    def __init__(self, arena) -> None:
        self.arena = arena
        self._tables: Dict[Tuple, object] = {}

    def get(self, use, slots):
        key = (use, tuple(s.index for s in slots))
        t = self._tables.get(key)
        if t is None:
            from .multi_tensor import GradSegTable
            t = self._tables[key] = GradSegTable(slots, self.arena.device)
        return t

    def whole(self):
        return self.get("grads", self.arena.slots)


class _Bucket:
    __slots__ = ("lo", "hi", "slots", "pending", "work", "launched", "replicated")

    def __init__(self, lo: int, hi: int):
        self.lo, self.hi = lo, hi
        self.slots = []
        self.pending = 0
        self.work = None
        self.launched = False
        self.replicated = False      # fused-NVLS runs: this bucket keeps the NCCL + K2 path


class GradBucketPipeline:
    def __init__(self, arena: ParamArena, optimizer: FusedArenaOptimizer, *,
                 process_group=None, world_size: int = 1, clip_norm: float = 0.0,
                 bucket_cap_mb: float = 25.0, first_bucket_mb: Optional[float] = 1.0,
                 eager_update: bool = True, nvls_link=None, accumulation: int = 1, ema=None) -> None:
        self.arena = arena
        self.optimizer = optimizer
        self.pg = process_group
        self.world = world_size
        self.clip_norm = float(clip_norm or 0.0)
        self.grad_scale = 1.0 / world_size
        self.distributed = world_size > 1
        self.on_cuda = arena.device.type == "cuda"
        if isinstance(accumulation, bool) or int(accumulation) != accumulation or accumulation < 1:
            raise ValueError("gradient accumulation must be an integer >= 1, got %r" % (accumulation,))
        self.accumulation = int(accumulation)
        # eager: update a bucket on the side stream as soon as it is complete (and reduced) while
        # backward is still running.  Needs no global norm, so clipping turns it off.  On one GPU
        # the caller decides (the persistent cuBLAS GEMMs leave the update few SMs to overlap on,
        # so a single tail launch is cheaper to issue).  An optimizer that needs whole tensors
        # (per-tensor norms) turns it off as well: its update is one tail over every slot.  So does
        # gradient accumulation: a microbatch's gradients go into the accumulator, not to an update.
        self.whole_tensors = optimizer.needs_whole_tensors
        self.eager = (eager_update and self.clip_norm == 0.0 and not self.whole_tensors
                      and self.accumulation == 1 and (self.distributed or self.on_cuda))

        cap = int(bucket_cap_mb * 1024 * 1024)
        first = int(first_bucket_mb * 1024 * 1024) if (first_bucket_mb and self.distributed) else None
        ranges = arena.buckets(cap, first) if (self.distributed or self.eager) else [(0, arena.numel)]
        use_nvls = nvls_link is not None and self.distributed and self.eager
        if use_nvls and arena.lp is not None and arena.model_end < arena.numel:
            # BF16 mode: criterion parameters read the fp32 master, which the fused NVLS step keeps
            # current only on the owning rank -> give them their own, replicated (NCCL) bucket
            cut = arena.model_end
            split = []
            for lo, hi in ranges:
                split += [(cut, hi), (lo, cut)] if lo < cut < hi else [(lo, hi)]
            ranges = split
        # Tail split.  The bucket that becomes ready LAST (the first layer's weight: its dW GEMM is
        # the final kernel of backward) is the only one whose exchange cannot hide behind backward
        # work.  When that bucket starts with a large 2-D weight, the weight's rows are cut in two
        # buckets: the layer computes dW as two row-block GEMMs and hands over the first half
        # (``rows_ready``) while the second is still running, so only half of the exchange is
        # exposed.  The cut is STATIC (decided here, not per step): with the fused NVLS step the
        # launch ranges define which rank owns which shard of the master weights and state.
        self._row_split: Dict[int, int] = {}            # slot.index -> rows in the first half
        min_bytes = int(os.environ.get("FRL_B200_TAIL_SPLIT_MIN_BYTES", str(4 << 20)))
        # at larger worlds a half-bucket exchange is mostly its two cross-GPU barriers, and one
        # more launch can cost more than the exposed half saves -> on by default at world 2 only
        # (not tuned on H100)
        want_split = os.environ.get("FRL_B200_TAIL_SPLIT", "1" if world_size == 2 else "0") != "0"
        if self.distributed and self.eager and ranges and want_split:
            lo, hi = ranges[-1]
            esz = 2 if arena.grad_dtype == torch.bfloat16 else 4
            head = next((s for s in arena.slots if s.offset == lo), None)
            if (head is not None and len(head.shape) == 2 and head.end <= hi
                    and head.shape[0] >= 2 and (head.end - lo) * esz >= min_bytes
                    and 2 * (head.end - lo) >= hi - lo):
                rows = head.shape[0] // 2
                if (rows * head.shape[1]) % 8 == 0:       # launch ranges stay 8-element aligned
                    mid = lo + rows * head.shape[1]
                    ranges = ranges[:-1] + [(lo, mid), (mid, hi)]
                    self._row_split[head.index] = rows
        self.buckets: List[_Bucket] = [_Bucket(lo, hi) for lo, hi in ranges]
        if use_nvls and arena.lp is not None:
            for b in self.buckets:
                b.replicated = b.lo >= arena.model_end
        self._last_bucket = self.buckets[-1] if self.buckets else None      # last in launch order
        self._buckets_of: Dict[int, List[_Bucket]] = {}
        for s in arena.slots:
            for b in self.buckets:                   # launch order; a row-split slot is in two
                inside = (s.offset < b.hi and s.end > b.lo) if s.end > s.offset else (b.lo <= s.offset < b.hi)
                if inside:
                    b.slots.append(s)
                    self._buckets_of.setdefault(id(s.param), []).append(b)
        self._n_slots = len(arena.slots)
        self._ready = 0
        self._ready_ids = set()
        self._handles = []
        for s in arena.slots:
            self._handles.append(s.param.register_post_accumulate_grad_hook(self._make_hook(s)))

        # high priority: the (short) reduce/update kernels should not queue behind GEMM CTAs
        self.side_stream = torch.cuda.Stream(device=arena.device, priority=-1) if self.on_cuda else None
        self.clip_out = None
        self.clip_scratch = None
        if self.clip_norm > 0.0:
            self.clip_out = torch.zeros(3, dtype=torch.float32, device=arena.device)
            nbytes = KERNELS.reduce_scratch_bytes()
            self.clip_scratch = torch.zeros((nbytes + 3) // 4, dtype=torch.int32, device=arena.device)
        # fused NVLS step: all-reduce + update + weight broadcast are ONE kernel per bucket
        # (csrc/nvls.cu); needs per-bucket updates, so clipping keeps the NCCL + K2/K3 path
        self.nvls = nvls_link if use_nvls else None
        if self.nvls is not None:
            optimizer.nvls = self.nvls
        # weight EMA: needs the whole master on every rank, which the fused NVLS step does not keep
        if ema is not None and self.nvls is not None:
            raise ValueError("a weight EMA cannot be combined with the fused NVLS step (K7)")
        self.ema = ema
        self._step_open = False
        self.step_id = 0
        self.linear_sites = []
        # arena_linear bookkeeping: per-parameter touch/application counters, the generation the
        # forward-application counts belong to (advanced when a step ends) and slots whose layer
        # ran a backward pass but expects more (module applied several times per forward)
        self.slot_states = {}
        self.forward_gen = 0
        self._deferred = {}
        # gradients autograd allocated itself, by slot index, kept alive until the kernels that
        # read them in place have been enqueued (multi-tensor path; CUDA only)
        self.mt_enabled = (self.on_cuda and hasattr(KERNELS, "flatten_grads")
                           and os.environ.get("FRL_B200_MT_GRADS", "1") != "0")
        self._ext: Dict[int, torch.Tensor] = {}
        self.tables = _TableSet(arena)
        self._keep_ext = False       # replay of a captured step: the capture owns the references
        # timing taps (bench): list of (start_event, end_event, lo, hi) for update launches
        self.record_update_events = False
        self.update_events: List[Tuple[torch.cuda.Event, torch.cuda.Event, int, int]] = []
        self.accumulate_events: List[Tuple[torch.cuda.Event, torch.cuda.Event]] = []     # K10 launches

        # gradient accumulation (k > 1): after each microbatch's backward ONE K10 launch folds every
        # gradient, weighted, into an fp32 arena-shaped accumulator; the microbatch that closes a
        # group runs the exchange and the update from it.  k == 1 allocates and launches nothing.
        self.acc: Optional[torch.Tensor] = None
        if self.accumulation > 1:
            self.acc = torch.zeros(arena.numel, dtype=torch.float32, device=arena.device)
            # (w, first) of the next K10 launch, device-resident so one captured graph serves
            # every position inside a group; uploaded from a pinned ring like the optimizer's scalars
            # (1, 1) until set_microbatch() says otherwise, as the by-value defaults below: a caller
            # that never sets a position gets one microbatch per group (weight 1), never a zero update
            self._acc_dyn = torch.ones(2, dtype=torch.float32, device=arena.device)
            self._acc_dyn_host = torch.zeros(self._ACC_RING, 2, dtype=torch.float32, pin_memory=self.on_cuda)
            self._acc_dyn_slot = 0
            self._acc_dyn_last: Optional[Tuple[float, float]] = (1.0, 1.0)
        self._acc_first = True
        self._acc_closes = True
        self._acc_weight = 1.0
        self._acc_scale = self.grad_scale
        self._acc_seen = set()         # slots that got a gradient in some microbatch of the open group
        self.last_ready: frozenset = frozenset()
        # K12: one GPU, one tail update (eager per-bucket updates would race the GEMM for the same
        # weights' state), no global norm, no accumulator, plain SGD on bf16 shadow weights
        self.fused_dw_update = (
            not self.distributed and not self.eager and self.clip_norm == 0.0 and self.accumulation == 1
            and type(optimizer) is FusedSGD and arena.precision is Precision.BF16
            and hasattr(KERNELS, "dw_gemm_sgd") and (self.on_cuda or KERNELS is not _native)
            and os.environ.get("FRL_B200_FUSED_DW_UPDATE", "1") != "0")
        self.dw_updated: set = set()      # slot indices K12 updated in this step

    _ACC_RING = 16

    @property
    def accumulator_bytes(self) -> int:
        return 0 if self.acc is None else self.acc.numel() * 4

    def set_microbatch(self, *, first: bool, closes: bool, weight: float = 1.0,
                       group_scale: float = 1.0) -> None:
        """Position of the next microbatch in its accumulation group (k > 1; call before its
        forward, never inside a CUDA-graph capture).  ``first``: it opens the group (K10 overwrites
        the accumulator); ``closes``: the update runs after its backward; ``weight``: n_i / B, its
        rows over the batch size; ``group_scale``: B / N, the batch size over the group's rows."""
        if self.acc is None:
            return
        self._acc_first, self._acc_closes = bool(first), bool(closes)
        self._acc_weight = float(weight)
        self._acc_scale = float(group_scale) / self.world
        if first:
            self._acc_seen.clear()
        vals = (self._acc_weight, 1.0 if first else 0.0)
        if vals != self._acc_dyn_last:
            if self.on_cuda:
                row = self._acc_dyn_host[self._acc_dyn_slot % self._ACC_RING]
                self._acc_dyn_slot += 1
                row[0], row[1] = vals
                self._acc_dyn.copy_(row, non_blocking=True)
            else:
                self._acc_dyn.copy_(torch.tensor(vals, dtype=torch.float32))
            self._acc_dyn_last = vals

    # -- step protocol ---------------------------------------------------------------------------
    def begin_step(self) -> None:
        """Call before ``backward()``."""
        self._ready = 0
        self._ready_ids.clear()
        self._deferred.clear()
        for b in self.buckets:
            b.pending = len(b.slots)
            b.work = None
            b.launched = False
        self.optimizer.begin_step()
        self.dw_updated = set()        # a new set: a captured step keeps the one it filled
        self.step_id += 1
        self._step_open = True

    @property
    def step_open(self) -> bool:
        return self._step_open

    def _make_hook(self, slot) -> Callable[[nn.Parameter], None]:
        from .multi_tensor import grad_usable_in_place

        def hook(param: nn.Parameter) -> None:
            g = param.grad
            if g is not None:
                dst = self.arena.grad_view(slot)
                if g.data_ptr() != dst.data_ptr():
                    if self.mt_enabled and self._step_open and grad_usable_in_place(g, slot):
                        self._ext[slot.index] = g     # read in place / gathered per bucket later
                    else:
                        dst.copy_(g)          # odd layouts, CPU tensors: flatten this one now
                param.grad = None             # next backward steals again instead of accumulating
            self.mark_ready(slot)
        return hook

    # -- multi-tensor plumbing ---------------------------------------------------------------------
    def _table(self, use, slots, acc: bool = False, ready=None):
        """The table of ``slots`` for ``use``, pointed at this step's gradients and uploaded: each
        slot's slice of the accumulator (``acc``), else the gradient autograd left outside the
        arena (a straggler) or the arena slice; NULL for a slot whose index is not in ``ready``."""
        table = self.tables.get(use, slots)
        g = self.acc if acc else self.arena.grad
        base, esz = g.data_ptr(), g.element_size()
        for s in slots:
            ext = None if acc else self._ext.get(s.index)
            if ready is not None and s.index not in ready:
                table.point(s, 0, g.dtype)
            elif ext is not None:
                table.point(s, ext.data_ptr(), ext.dtype)
            else:
                table.point(s, base + s.offset * esz, g.dtype)
        table.upload()
        return table

    def _flatten_stragglers(self, slots, key, side: bool) -> None:
        """ONE launch: gather the listed slots' out-of-arena gradients into their arena slices
        (cast to the arena's gradient dtype) on the current stream."""
        ext = [s for s in slots if s.index in self._ext]
        if not ext:
            return
        KERNELS.flatten_grads(self._table(key, ext), self.arena.grad, scale=1.0)
        for s in ext:
            g = self._ext.pop(s.index) if not self._keep_ext else self._ext[s.index]
            if side:
                g.record_stream(torch.cuda.current_stream())

    def materialize_grads(self) -> None:
        """Debug/inspection aid: make ``arena.grad`` hold every gradient of the open step."""
        self._flatten_stragglers(self.arena.slots, "all", side=False)

    def detach_grad_refs(self):
        """Hand the straggler references and the table set to a captured graph (which replays
        kernels that read exactly these addresses); the pipeline continues with fresh ones."""
        refs, tables = self._ext, self.tables
        self._ext, self.tables = {}, _TableSet(self.arena)
        return refs, tables

    def mark_ready(self, slot) -> None:
        if not self._step_open or id(slot.param) in self._ready_ids:
            return
        self._ready_ids.add(id(slot.param))
        self._ready += 1
        for b in self._buckets_of[id(slot.param)]:
            if b.launched:                    # the first half of a row-split weight went ahead
                continue
            b.pending -= 1
            if b.pending == 0 and (self.distributed or self.eager) and self.acc is None:
                self._launch_bucket(b)

    def row_split(self, slot) -> int:
        """Rows of the slot's first half if its weight gradient is exchanged in two row blocks
        (tail split, see ``__init__``), else 0."""
        return self._row_split.get(slot.index, 0)

    def rows_ready(self, slot, rows: int) -> None:
        """Rows ``[0, rows)`` of the slot's gradient are final and the rest is still being
        computed: launch every bucket that lies inside them and waits for nothing else."""
        if not self._step_open:
            return
        done = slot.offset + rows * slot.shape[1]
        for b in self._buckets_of[id(slot.param)]:
            if not b.launched and b.hi <= done and b.pending == 1:
                b.pending = 0
                self._launch_bucket(b)

    def update_in_dw_gemm(self, slot, dz, x, gw) -> None:
        """K12: gw = dz^T x into the slot's gradient and the slot's update from it, in one kernel
        (``fused_dw_update``; the caller checked the shapes).  The tail leaves the slot alone."""
        self.optimizer.update_in_dw_gemm(slot, dz, x, gw, grad_scale=self.grad_scale)
        self.dw_updated.add(slot.index)

    def defer_ready(self, slot) -> None:
        """The slot's gradient was written but more contributions are expected in this backward;
        ``mark_ready`` follows from the last one, or from ``finish_step`` at the latest."""
        self._deferred[slot.index] = slot

    def _launch_bucket(self, b: _Bucket) -> None:
        """Bucket complete: (all-reduce it and) update it on the side stream, behind everything
        the compute stream has issued so far.  Runs in the autograd thread, so it is kept lean:
        no context managers, one event."""
        if self.on_cuda:
            cur = torch.cuda.current_stream()
            self.side_stream.wait_stream(cur)
            torch.cuda.set_stream(self.side_stream)
        try:
            if self._ext:
                self._flatten_stragglers(b.slots, id(b), side=self.on_cuda)
            fused = self.nvls is not None and not b.replicated      # K7: reduce + update + broadcast
            if self.distributed and not fused:
                b.work = dist.all_reduce(self.arena.grad[b.lo:b.hi], op=dist.ReduceOp.SUM,
                                         group=self.pg, async_op=True)
                if self.eager:
                    b.work.wait()             # stream-level wait, the host does not block
            if self.eager:
                tap = self._tap()
                if fused:
                    nv = self.nvls
                    grid = nv.max_blocks
                    if b is self._last_bucket:        # runs alone: backward has nothing left to issue
                        nv.max_blocks = nv.tail_blocks
                    try:
                        self.optimizer.apply_range_nvls(b.lo, b.hi, grad_scale=self.grad_scale)
                    finally:
                        nv.max_blocks = grid
                else:
                    self.optimizer.apply_range(b.lo, b.hi, grad_scale=self.grad_scale)
                self._tap_end(tap, self.update_events, b.lo, b.hi)
        finally:
            if self.on_cuda:
                torch.cuda.set_stream(cur)
        b.launched = True

    def _tap(self):
        """Timing tap (bench): a pair of events, the first recorded now, or None while it is off."""
        if not (self.record_update_events and self.on_cuda):
            return None
        tap = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
        tap[0].record()
        return tap

    @staticmethod
    def _tap_end(tap, events, *span) -> None:
        """Close a ``_tap()`` window: record its end event and append ``(start, end, *span)``."""
        if tap is not None:
            tap[1].record()
            events.append(tap + span)

    def finish_step(self, defer_tail: bool = False) -> None:
        """Call after ``backward()`` returned: reduces/updates whatever is still outstanding and
        re-joins the side stream.  ``defer_tail=True`` (CUDA-graph capture) leaves the tail
        launches (norm + update of whatever was not updated eagerly) to ``run_tail()``."""
        if not self._step_open:
            raise RuntimeError("finish_step() without begin_step()")
        for slot in list(self._deferred.values()):    # backward() has returned: nothing is missing
            self.mark_ready(slot)
        self._deferred.clear()
        self.forward_gen += 1
        self._step_open = False
        partial = self._ready != self._n_slots
        if partial and self.distributed:
            missing = [s.index for s in self.arena.slots if id(s.param) not in self._ready_ids]
            # same contract as DDP with find_unused_parameters=False (the reference's setting)
            raise RuntimeError(
                "Expected to have finished reduction for every parameter, but parameters at "
                f"indices {missing} did not receive a gradient in this step")
        if self.acc is not None:
            # k > 1: fold this microbatch into the accumulator; the group's last one updates.
            # Inside a capture the K10 launch is recorded and the update is left to run_tail().
            self._accumulate_microbatch(keep_refs=defer_tail)
        else:
            if self.distributed and not self.eager:
                cur = torch.cuda.current_stream() if self.on_cuda else None
                if cur is not None:
                    torch.cuda.set_stream(self.side_stream)
                for b in self.buckets:
                    b.work.wait()
                if cur is not None:
                    torch.cuda.set_stream(cur)
            if self.on_cuda and (self.distributed or self.eager):
                torch.cuda.current_stream().wait_stream(self.side_stream)
            if partial:
                # one GPU, some parameters got no gradient: updated at once, capture or not (inside
                # a capture without the EMA step: run_tail() updates again and steps the EMA)
                self._end_update([s for s in self.arena.slots if id(s.param) in self._ready_ids],
                                 ema=not defer_tail)
                return
        if not defer_tail:
            self.run_tail()

    @property
    def has_tail(self) -> bool:
        """True if a step ends with tail launches (not everything is updated eagerly)."""
        return not self.eager

    def run_tail(self, grad_refs=None, tables=None, ready=None, dw_updated=None) -> None:
        """The deferred part of ``finish_step(defer_tail=True)``; also what a CUDA-graph replay
        of the captured step is followed by (then with the capture's gradient references and
        segment tables: the replayed backward wrote to exactly those addresses).  With gradient
        accumulation: the update from the accumulator if this microbatch closes its group;
        ``ready`` names the slots the replayed K10 launch accumulated; ``dw_updated`` the slots
        the replayed K12 launches updated."""
        if self.acc is not None:
            if ready is not None:
                self._acc_seen |= ready
            if self._acc_closes:
                self._end_update(acc=True)
            return
        if grad_refs is not None:
            mine = (self._ext, self.tables, self.dw_updated)
            self._ext, self.tables, self._keep_ext = grad_refs, tables, True
            if dw_updated is not None:
                self.dw_updated = dw_updated
        try:
            if self.has_tail:
                self._end_update()
            else:
                self.optimizer.end_step()
                if self.ema is not None:
                    self.ema.update()
        finally:
            if grad_refs is not None:
                (self._ext, self.tables, self.dw_updated), self._keep_ext = mine, False

    def _end_update(self, present=None, acc: bool = False, ema: bool = True) -> None:
        """Every update that is not a bucket's eager one, then the optimizer's step count and
        (``ema``) the weight EMA's step.
        ``present``: the slots that got a gradient (default: all) -- torch.optim skips the others
        (no weight decay, no momentum decay), so they keep their weights and state.  ``acc``: the
        group is closed, update from the accumulator (fp32; exchanged per bucket on several GPUs)
        at ``_acc_scale`` = B / (world * N), which turns the weighted sum into the group's mean."""
        slots, n = self.arena.slots, self.arena.numel
        if acc:
            grads, scale = self.acc, self._acc_scale
            if self.distributed:
                for b in self.buckets:
                    dist.all_reduce(grads[b.lo:b.hi], op=dist.ReduceOp.SUM, group=self.pg)
            else:
                present = [s for s in slots if s.index in self._acc_seen]
        else:
            grads, scale = self.arena.grad, self.grad_scale
        have = {s.index for s in (slots if present is None else present)}
        every = len(have) == len(slots)
        window = self._tap() if acc else None     # accumulation: ONE timed window, K3 included
        coef = None
        if not acc and (self.clip_norm > 0.0 or not every):
            # the norm and the runs' flat updates read the arena: gather the stragglers into it
            self._flatten_stragglers(slots, "all", side=False)
        if self.clip_norm > 0.0:
            # the global norm over the model range only (criterion parameters are not clipped);
            # a missing gradient counts as zero
            if not acc:
                for s in slots:
                    if s.index not in have and s.is_model:
                        grads[s.offset:s.end].zero_()
            n_model = self.arena.model_end
            KERNELS.grad_sumsq_clip(grads[:n_model], n_model, pre_scale=scale, max_norm=self.clip_norm,
                                    out3=self.clip_out, scratch=self.clip_scratch)
            coef = self.clip_out[2:3]
        if not acc:
            have -= self.dw_updated               # K12 updated these inside their dW GEMMs
        if self.whole_tensors or (not acc and self._ext and coef is None and not self.distributed):
            # one update over a table of the present slots: whole tensors (per-tensor norms), or on
            # one GPU every gradient read where it lies -- no flatten pass
            table = self._table("acc" if acc else "grads", [s for s in slots if s.index in have], acc=acc)
            tap = None if acc else self._tap()
            self.optimizer.apply_table(table, grad_scale=scale, clip_coef_dev=coef)
            self._tap_end(tap, self.update_events, 0, n)
        else:
            done = [(b.lo, b.hi) for b in self.buckets if b.launched and self.eager]
            runs = [(0, n)] if len(have) == len(slots) else self._runs(
                lambda s: s.index in have and not any(a <= s.offset < z for a, z in done))
            for lo, hi in runs:
                tap = None if acc else self._tap()
                self.optimizer.apply_range(lo, hi, grad_scale=scale, clip_coef_dev=coef,
                                           grad_src=grads if acc else None)
                self._tap_end(tap, self.update_events, lo, hi)
        self._tap_end(window, self.update_events, 0, n)
        if not self._keep_ext:
            self._ext.clear()
        self.optimizer.end_step()
        if ema and self.ema is not None:
            self.ema.update()

    def _runs(self, keep) -> List[Tuple[int, int]]:
        """Arena ranges ``[lo, hi)`` of the maximal runs of consecutive slots with ``keep(slot)``."""
        runs: List[Tuple[int, int]] = []
        run_lo = prev_end = None
        for s in self.arena.slots:
            if not keep(s):
                if run_lo is not None:
                    runs.append((run_lo, prev_end))
                    run_lo = None
                continue
            if run_lo is None:
                run_lo = s.offset
            prev_end = s.end
        if run_lo is not None:
            runs.append((run_lo, prev_end))
        return runs

    # -- gradient accumulation (k > 1) -------------------------------------------------------------
    def _accumulate_microbatch(self, keep_refs: bool = False) -> None:
        """ONE K10 launch over the whole table: every gradient of this microbatch, where it lies,
        times n_i / B into the accumulator; slots without a gradient point at NULL (nothing added,
        zeroed when the microbatch opens its group)."""
        slots = self.arena.slots
        self.last_ready = frozenset(s.index for s in slots if id(s.param) in self._ready_ids)
        self._acc_seen |= self.last_ready
        table = self._table("grads", slots, ready=self.last_ready)
        tap = self._tap()
        KERNELS.grad_accumulate_mt(self.acc, table, w=self._acc_weight, first=self._acc_first,
                                   dyn=self._acc_dyn)
        self._tap_end(tap, self.accumulate_events)
        if not keep_refs:
            self._ext.clear()            # the launch is enqueued: stream order protects the reads

    # -- one-time synchronisation ----------------------------------------------------------------
    def broadcast_parameters(self, src: int = 0) -> None:
        """Replicas start identical to rank ``src`` (DDP does this in its constructor)."""
        if not self.distributed:
            return
        dist.broadcast(self.arena.master, src=src, group=self.pg)
        self.arena.refresh_shadow()

    def sync_sharded_state(self) -> None:
        """Fused NVLS step only: every rank holds the current fp32 master / optimizer state of its
        own shards; before a checkpoint export make them whole everywhere (collective call)."""
        if self.nvls is None:
            return
        opt = self.optimizer
        vecs = list(opt._vec.values())
        if self.arena.lp is not None:
            vecs.append(self.arena.master)         # FP32 mode multicasts the master itself
        for vec in vecs:
            whole = torch.zeros_like(vec)
            for b in self.buckets:
                if b.replicated:
                    if self.nvls.rank == 0:
                        whole[b.lo:b.hi] = vec[b.lo:b.hi]
                    continue
                a, z = opt.shard_of(b.lo, b.hi)
                whole[a:z] = vec[a:z]
            dist.all_reduce(whole, op=dist.ReduceOp.SUM, group=self.pg)
            vec.copy_(whole)

    def remove_hooks(self) -> None:
        for h in self._handles:
            h.remove()
        self._handles = []
        self.unpatch_linears()

    # -- nn.Linear gradients written directly into the arena ---------------------------------------
    def patch_linears(self, model: nn.Module) -> int:
        from .arena_linear import patch_linears
        self.linear_sites = patch_linears(model, self)
        return len(self.linear_sites)

    def unpatch_linears(self) -> None:
        from .arena_linear import unpatch_linears
        unpatch_linears(self.linear_sites)

    def repatch_linears(self) -> None:
        from .arena_linear import repatch_linears
        repatch_linears(self.linear_sites)


class BufferBroadcaster:
    """Module buffers (BatchNorm statistics) follow rank 0 before every forward, as DDP's
    ``broadcast_buffers=True`` default does for the reference — but as ONE broadcast per dtype
    over a flat buffer arena the buffers are re-pointed into."""

    def __init__(self, module: nn.Module, *, process_group=None, world_size: int = 1) -> None:
        self.pg = process_group
        self.enabled = world_size > 1
        self.flat: List[torch.Tensor] = []
        if not self.enabled:
            return
        by_dtype = {}
        for buf in module.buffers():
            by_dtype.setdefault(buf.dtype, []).append(buf)
        for dtype, bufs in by_dtype.items():
            total = sum(b.numel() for b in bufs)
            if total == 0:
                continue
            flat = torch.empty(total, dtype=dtype, device=bufs[0].device)
            off = 0
            for b in bufs:
                n = b.numel()
                flat[off:off + n].copy_(b.reshape(-1))
                b.data = flat[off:off + n].view(b.shape)
                off += n
            self.flat.append(flat)

    def sync(self, src: int = 0) -> None:
        if self.enabled:
            for flat in self.flat:
                dist.broadcast(flat, src=src, group=self.pg)
