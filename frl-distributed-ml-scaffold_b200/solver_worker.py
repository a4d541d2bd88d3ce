"""Per-rank epoch / minibatch loop — the hot path (reference solver_worker.py:377-832).

Same observable behaviour as the reference's ``SolverWorker`` (split order, train/eval modes,
per-minibatch loss bookkeeping, amortised metric hooks, per-epoch summaries and the yielded
``FractionalPerformanceSummary``), restructured so that a training step never synchronises the
host with the device:

* fused criterion writes ``[total, sub-losses]`` of step *k* into row *k* of a pinned,
  device-mapped loss log; the host reads rows two steps late (NaN guard) and the whole log once
  per split (epoch means) instead of ``2 + T`` ``.item()`` calls per step;
* ``backward()`` deposits gradients in the flat arena, ``GradBucketPipeline`` all-reduces and
  applies the fused optimizer update per bucket;
* inputs arrive through pinned memory with asynchronous copies (the reference's
  ``pin_memory=self.device == Device.GPU`` compares a ``torch.device`` with an Enum and is
  always False, reference solver_worker.py:829);
* one watchdog thread per split is kicked per step instead of spawning a Timer per step.
"""
from contextlib import contextmanager, nullcontext
import io
import os
import queue
import threading
import itertools
import json
import logging
import random
import time
from math import ceil
from typing import Any, Dict, Iterator, List, NamedTuple, Optional, Sequence, Tuple, Union

import numpy as np
import torch
import torch.utils.data

from . import _native
from .arena import ParamArena
from .criteria import BaseParallelCriterion, GradNormWeightedCriterion
from .ema import EMA_STATE_KEY
from .fused_optim import FusedArenaOptimizer
from .grad_sync import BufferBroadcaster, GradBucketPipeline, accumulation_plan
from .model import MultiTaskModel
from .problem import BatchMetrics, Ordering, Problem
from .sampler import ScaffoldSampler
from .storage_layers.dataset import MultifieldDataset, NullAccessor, SubsetMultifieldDataset
from .types import Mode, Precision, RunOpts, SampleSummary, Split
from .watchdog import StepWatchdog

logger = logging.getLogger(__name__)

# samples kept per split so an exported network's input/output mapping can be validated
MODEL_CONVERSION_TEST_SAMPLE_CT: int = 2
NAN_CHECK_LAG = 2          # steps the host may run ahead of the loss log it inspects

JSON = str
RawMetas = Dict[str, Union[torch.Tensor, List[Union[str, float]]]]


class SingleSample(NamedTuple):
    data: List[torch.Tensor]
    target: List[Tuple[torch.Tensor, ...]]
    meta: Dict[str, Any]
    output: List[torch.Tensor]
    metric: Dict[str, float]


class SerializableSampleSummary(NamedTuple):
    """``SampleSummary`` with the figure pre-serialised to JSON so it can cross the pipe."""
    image: Optional[np.ndarray]
    text: Optional[str]
    plot: Optional[JSON] = None
    source: Optional[str] = None


class FractionalEpochSplitPerformanceSummary(NamedTuple):
    nSamples: int
    losses: Dict[str, float]
    metrics: Dict[str, float]
    samples: List[SerializableSampleSummary]
    worstSamples: List[SerializableSampleSummary]
    testIO: List[SingleSample]


class FractionalPerformanceSummary(NamedTuple):
    epoch: int
    modelBuffer: bytes
    optimizerStateBuffer: bytes
    performance: Dict[Split, FractionalEpochSplitPerformanceSummary]


def stack_recursive(items):
    assert len(items) > 0
    first = items[0]
    if isinstance(first, Sequence) and not torch.is_tensor(first):
        return [torch.stack([it[i] for it in items]) for i in range(len(first))]
    return torch.stack(list(items))


def stat_to_str(stats: Dict[str, Tuple[np.ndarray, np.ndarray]]) -> str:
    """``{metric: (bin counts, bin values)}`` -> cumulative-fraction table."""
    out = ""
    for name, (counts, values) in stats.items():
        cum = np.cumsum(counts)
        total = cum[-1]
        out += "\n" + name + "\n"
        out += "".join("{:.3f}: {:.3f}\t".format(values[i], (cum[i] / total) if total != 0 else 0.0)
                       for i in range(len(cum)))
    return out + "\n"


class AverageMeter:
    def __init__(self) -> None:
        self.val = 0.0
        self.avg = 0.0
        self.sum = 0.0
        self.count = 0

    def update(self, val: float, n: int = 1) -> None:
        self.val = val
        self.sum += val * n
        self.count += n
        self.avg = self.sum / self.count


class EpochTimer:
    def __init__(self) -> None:
        self.batch = AverageMeter()
        self.epoch = AverageMeter()


class LossLog:
    """Pinned, device-mapped ``[capacity, 1+T]`` fp32 ring the criterion kernel writes into."""

    def __init__(self, n_tasks: int, capacity: int, device: torch.device) -> None:
        self.width = 1 + n_tasks
        self.capacity = max(capacity, 1)
        self.on_cuda = device.type == "cuda"
        self.rows = torch.full((self.capacity, self.width), float("inf"), dtype=torch.float32,
                               pin_memory=self.on_cuda)
        self.nan_flag = torch.zeros(1, dtype=torch.int32, pin_memory=self.on_cuda)
        self.events: List[Optional[torch.cuda.Event]] = [None] * self.capacity

    def row(self, step: int) -> torch.Tensor:
        return self.rows[step % self.capacity]

    def mark(self, step: int) -> None:
        if self.on_cuda:
            ev = torch.cuda.Event()
            ev.record()
            self.events[step % self.capacity] = ev

    def wait(self, step: int) -> None:
        ev = self.events[step % self.capacity]
        if ev is not None:
            ev.synchronize()


class _MetricWorker:
    """One background thread + one CUDA stream that fold retained minibatches into per-sample
    metrics.  The Problem's ``compute_batch_metrics`` hook returns host arrays, i.e. it ends in a
    device-to-host read; called from the training thread (as the reference does every
    ``metricAmortizationSchedule`` steps, solver_worker.py:286-312) that read drains the whole
    launch pipeline — about one step of idle GPU per window at H100 step times.  Here the read
    blocks only this thread; jobs run FIFO, so per-sample metrics keep their order."""

    def __init__(self, device: torch.device) -> None:
        self.device = device
        self.stream = torch.cuda.Stream(device=device)
        self._jobs: "queue.Queue" = queue.Queue()
        self._error: Optional[BaseException] = None
        self._thread = threading.Thread(target=self._run, name="frl-metrics", daemon=True)
        self._thread.start()

    def _run(self) -> None:
        torch.cuda.set_device(self.device)
        while True:
            job = self._jobs.get()
            try:
                if job is None:
                    return
                fn, ready = job
                if self._error is None:
                    with torch.no_grad(), torch.cuda.stream(self.stream):
                        self.stream.wait_event(ready)
                        fn()
                    self.stream.synchronize()       # before the window's tensors are released
            except BaseException as e:              # noqa: BLE001  (re-raised in the loop's thread)
                self._error = e
            finally:
                self._jobs.task_done()

    def submit(self, fn, ready: "torch.cuda.Event") -> None:
        self.raise_pending()
        self._jobs.put((fn, ready))

    def drain(self) -> None:
        self._jobs.join()
        self.raise_pending()

    def raise_pending(self) -> None:
        if self._error is not None:
            err, self._error = self._error, None
            raise err

    def close(self) -> None:
        self._jobs.put(None)


class SamplerState:
    """Keeps the last few minibatches on the device and folds them into per-sample metrics,
    a random sample set and the worst-k samples (reference solver_worker.py:189-374).

    Each window is folded by tensor ops on the device of its outputs, whatever the Problem's hook
    returns: the metrics go into per-split columns, the random picks are row-gathered by
    host-known positions, the worst-k set is a running buffer merged per window with ``topk``.
    Nothing is read back until ``finish()`` reads everything at once."""

    def __init__(self, problem: Problem, n_samples: int, dataset_len: int,
                 device: torch.device, n_vis: int) -> None:
        self._problem = problem
        self._device = device
        self._n_samples = n_samples
        self._n_vis = min(n_samples, ceil(n_vis * (n_samples / dataset_len)))
        n_random = min(max(self._n_vis, MODEL_CONVERSION_TEST_SAMPLE_CT), n_samples)
        self._random_indices = frozenset(random.sample(range(n_samples), n_random))
        self._cur_samples = 0
        self._rankable_metric, self._ordering = problem.get_rankable_metric()
        self._allow_non_positive_definite = ("MSE" not in self._rankable_metric
                                             and "EucDist" not in self._rankable_metric)
        self._metas: List[RawMetas] = []
        self._data: List[List[torch.Tensor]] = []
        self._targets: List[List[Tuple[torch.Tensor, ...]]] = []
        self._outputs: List[List[torch.Tensor]] = []
        # Where the fold runs.  The reference calls the Problem's hooks synchronously on the
        # training thread (solver_worker.py:286-312) and so does this loop by default; a hook that
        # returns host arrays then costs one pipeline drain per window.  Two ways around it:
        #   * the hook returns DEVICE tensors (``metrics_on_device``): the fold is pure device
        #     work, it stays on the training thread/stream and never blocks it;
        #   * the Problem declares ``metric_hooks_thread_safe = True`` (or FRL_B200_ASYNC_METRICS=1):
        #     host-returning hooks run on a worker thread + side stream.  Opt-in, because hooks
        #     that touch the model, global RNGs or backend flags would race with the next steps.
        self._runner: Optional[_MetricWorker] = None
        want_async = os.environ.get("FRL_B200_ASYNC_METRICS")
        if want_async is None:
            want_async = "1" if getattr(problem, "metric_hooks_thread_safe", False) else "0"
        if device.type == "cuda" and want_async != "0":
            self._runner = _MetricWorker(device)
        self._dev_mode = False               # the hook returned device tensors (``metrics_on_device``)
        # per-sample metric columns and meta (tensor columns, or host lists), over the split
        self._cols: Dict[str, torch.Tensor] = {}
        self._meta: Dict[str, Union[torch.Tensor, list]] = {}
        self._dev_random: List[Dict[str, Any]] = []
        self._dev_worst: Optional[Dict[str, Any]] = None
        # filled by finish()
        self._data_metric: Dict[str, np.ndarray] = {}
        self._random_samples: List[SingleSample] = []
        self._worst_samples: List[SingleSample] = []

    @staticmethod
    def _cat_metas(metas: List[RawMetas]) -> RawMetas:
        merged: RawMetas = {}
        for key, first in metas[0].items():
            vals = [m[key] for m in metas]
            if torch.is_tensor(first):
                merged[key] = torch.cat(vals)
            elif isinstance(first, list):
                merged[key] = list(itertools.chain.from_iterable(vals))
            else:
                raise ValueError("Unsure how to concatenate meta field with type %s" % type(first))
        return merged

    def append_sample(self, raw_metas: RawMetas, data, *, outputs, targets) -> None:
        self._metas.append(raw_metas)
        self._data.append([t.detach() for t in data])
        self._outputs.append([t.detach() for t in outputs])
        self._targets.append([tuple(t.detach() for t in head) for head in targets])

    @property
    def metrics_on_device(self) -> bool:
        """The Problem's hook returned device tensors: folding a window is pure device work
        (no host read), so it needs no worker thread and can be queued behind the last steps."""
        return self._dev_mode

    def compute_metrics(self) -> None:
        """Fold the retained minibatches (a 'window') into the split's metrics.  With a metric
        worker the fold of a host-returning hook runs on its thread/stream and this returns at
        once; ``finish()`` joins."""
        if not self._data:
            return
        window = (self._metas, self._data, self._outputs, self._targets)
        self._metas, self._data, self._outputs, self._targets = [], [], [], []
        if self._runner is None or self._dev_mode:
            self._fold(*window)
            return
        ready = torch.cuda.Event()
        ready.record()                       # everything the window holds has been enqueued
        self._runner.submit(lambda: self._fold(*window), ready)

    def __enter__(self) -> "SamplerState":
        return self

    def __exit__(self, *exc) -> None:
        if self._runner is not None:         # the loop raised before finish(): stop the thread
            self._runner.close()
            self._runner = None

    @staticmethod
    def _gather_rows(batches: List[torch.Tensor], idx: torch.Tensor) -> torch.Tensor:
        """Rows ``idx`` (device int64, window-relative) of the retained minibatch list.  The host
        does not know ``idx`` (it comes out of a device ``topk``) and the minibatches are separate
        tensors: K8w (``frl_gather_window_rows``) walks a table of their base pointers — one launch,
        only the picked rows move (concatenating the window first was a 0.3 GB device copy per
        amortisation window at batch 4096 x 4096 bf16, twice: random picks and worst-k).
        channels_last [B, C, H, W] batches are gathered as the [B, H, W, C] rows they store (each
        sample is contiguous in NHWC too); the rows come back channels_last [k, C, H, W]."""
        if batches[0].is_cuda and all(_native.is_nhwc(b) for b in batches):
            rows = _native.gather_window_rows([b.permute(0, 2, 3, 1) for b in batches], idx)
            return rows.permute(0, 3, 1, 2)
        if batches[0].is_cuda:
            return _native.gather_window_rows([b if b.is_contiguous() else b.contiguous() for b in batches], idx)
        return (batches[0] if len(batches) == 1 else torch.cat(batches)).index_select(0, idx)

    def _pick(self, idx: torch.Tensor, base: int, data_batches, target, output) -> Dict[str, Any]:
        """Rows ``idx`` (window-relative, device) of everything a ``SingleSample`` shows; metrics
        and meta are looked up by global position from the per-split columns at the end."""
        n_fields = len(data_batches[0])
        return {"pos": idx + base,
                "data": [self._gather_rows([d[f] for d in data_batches], idx) for f in range(n_fields)],
                "target": [tuple(t.index_select(0, idx) for t in head) for head in target],
                "output": [o.index_select(0, idx) for o in output]}

    def _fold(self, metas, data_batches, outputs, targets) -> None:
        meta = self._problem.refine_batch_meta(self._cat_metas(metas))
        n_heads = len(outputs[0])
        target = [tuple(torch.cat([t[h][j] for t in targets])
                        for j in range(len(targets[0][h]))) for h in range(n_heads)]
        output = [torch.cat([o[h] for o in outputs]) for h in range(n_heads)]
        output = [o.float() if o.dtype == torch.bfloat16 else o for o in output]
        base, n_group, dev = self._cur_samples, sum(len(d[0]) for d in data_batches), output[0].device
        self._cur_samples += n_group

        sample_metric = self._problem.compute_batch_metrics(
            meta=meta, target=target, output=output, device=self._device)
        for k, v in meta._asdict().items():
            if torch.is_tensor(v):
                col = self._meta.get(k)
                if col is None:
                    col = self._meta[k] = torch.zeros((self._n_samples,) + tuple(v.shape[1:]),
                                                      dtype=v.dtype, device=v.device)
                col[base:base + n_group] = v
            else:            # names, ids as lists; a None field stays None per sample
                self._meta.setdefault(k, []).extend([None] * n_group if v is None else v)
        if not sample_metric:
            return
        self._dev_mode = all(torch.is_tensor(v) and v.is_cuda for v in sample_metric.values())
        for k, v in sample_metric.items():
            # host arrays are uploaded (a few KB: the hook has just synchronised to produce them)
            v = torch.as_tensor(v, device=dev).reshape(n_group)
            if v.dtype in (torch.bfloat16, torch.float16):
                v = v.float()
            col = self._cols.get(k)
            if col is None:
                col = self._cols[k] = torch.zeros(self._n_samples, dtype=v.dtype, device=dev)
            col[base:base + n_group] = v
        if self._n_vis <= 0:
            return
        picks = sorted(j - base for j in self._random_indices if base <= j < base + n_group)
        if picks:
            # a few int64s from pageable memory: the driver stages them, the host does not wait
            # for the device (a pinned allocation here would cost a system call)
            idx = torch.tensor(picks, dtype=torch.int64, device=dev)
            self._dev_random.append(self._pick(idx, base, data_batches, target, output))
        # worst-k of this window, merged into the running set, ranked in float64
        metric = self._cols[self._rankable_metric][base:base + n_group].double()
        valid = (torch.ones_like(metric, dtype=torch.bool) if self._allow_non_positive_definite
                 else metric >= 0)
        score = -metric if self._ordering == Ordering.DESC else metric
        # every valid sample outranks every invalid one, also a valid one that ranks as -inf
        score = torch.where(valid, score.clamp(min=torch.finfo(torch.float64).min), float("-inf"))
        top_score, top_idx = torch.topk(score, min(self._n_vis, n_group))
        cand = self._pick(top_idx, base, data_batches, target, output)
        cand["score"], cand["valid"] = top_score, valid.index_select(0, top_idx)
        if self._dev_worst is not None:
            merged = _tree_map(lambda a, b: torch.cat([a, b]), self._dev_worst, cand)
            sel = torch.topk(merged["score"], min(self._n_vis, merged["score"].numel()))[1]
            cand = _tree_map(lambda t: t.index_select(0, sel), merged)
        self._dev_worst = cand

    def finish(self) -> None:
        """All windows folded (re-raises what a fold raised); call before reading results.

        The split's single device-to-host read: metric columns, meta, the picks, the worst-k
        set — every copy issued asynchronously into pinned memory, ONE stream synchronisation."""
        if self._runner is not None:
            self._runner.drain()
            self._runner.close()
            self._runner = None
        pending: List[Tuple[torch.Tensor, torch.Tensor]] = []
        requests: List[torch.Tensor] = []

        def host(t: torch.Tensor) -> int:
            """Queue ``t`` for the read-back; returns its ticket."""
            requests.append(t.contiguous())
            return len(requests) - 1

        def flush() -> List[torch.Tensor]:
            # everything is packed into ONE device buffer (a single concatenation launch) and moved
            # by ONE copy into ONE pinned staging block, then carved into aligned views: a pinned
            # allocation per tensor is a system call, and even the 22 separate
            # device-to-host copies of an MLP split cost the host time to issue
            parts, offs, total = [], [], 0
            pad = None
            for t in requests:
                flat = t.reshape(-1).view(torch.uint8)
                offs.append(total)
                parts.append(flat)
                total += flat.numel()
                gap = -total % 16
                if gap:
                    if pad is None:
                        pad = torch.zeros(16, dtype=torch.uint8, device=t.device)
                    parts.append(pad[:gap])
                    total += gap
            if total == 0:
                return [torch.empty(t.shape, dtype=t.dtype) for t in requests]
            packed = torch.cat(parts)
            # (host tensors only when the fold ran without a device)
            stage = _pinned_block(total) if packed.is_cuda else torch.empty(total, dtype=torch.uint8)
            stage[:total].copy_(packed, non_blocking=True)
            pending.append((stage, packed))               # keep the source alive until the sync
            return [stage[o:o + t.numel() * t.element_size()].view(t.dtype).view(t.shape)
                    for t, o in zip(requests, offs)]

        t_begin = time.perf_counter()
        n = self._cur_samples
        cols_h = {k: host(v[:n]) for k, v in self._cols.items()}
        # device meta joins the read-back; host meta (CPU columns, lists) is already here
        meta_h = {k: host(v[:n]) for k, v in self._meta.items() if torch.is_tensor(v) and v.is_cuda}
        random_h = [_tree_map(host, p) for p in self._dev_random]
        worst_h = [_tree_map(host, self._dev_worst)] if self._dev_worst is not None else []
        t_q = time.perf_counter()
        landed = flush()
        t_f = time.perf_counter()
        if self._device.type == "cuda":
            torch.cuda.current_stream(self._device).synchronize()
        t_s = time.perf_counter()
        pending.clear()
        tracing = bool(os.environ.get("FRL_B200_EPOCH_TRACE"))
        prof = None
        if tracing:
            logger.info("finish trace: %d tensors queued (built in %.2f ms), flush issued in %.2f ms, sync waited %.2f ms",
                        len(requests), 1e3 * (t_q - t_begin), 1e3 * (t_f - t_q), 1e3 * (t_s - t_f))
            if os.environ.get("FRL_B200_EPOCH_TRACE") == "profile":
                import cProfile
                prof = cProfile.Profile()
                prof.enable()

        cols_h, meta_h, random_h, worst_h = _tree_map(landed.__getitem__, (cols_h, meta_h, random_h, worst_h))

        def own(t: torch.Tensor) -> torch.Tensor:
            # a pageable copy out of the staging block by plain memcpy.  ``clone()``/``copy_`` of a
            # CPU tensor above ATen's grain size (32 768 elements) is an OpenMP parallel region:
            # waking a 128-thread pool that sleeps between epochs costs milliseconds PER CALL;
            # numpy's copy is single-threaded (numpy has no bfloat16: those go as their int16 bits)
            if t.dtype == torch.bfloat16:
                return own(t.view(torch.int16)).view(torch.bfloat16)
            return torch.from_numpy(t.numpy().copy())

        self._data_metric = {k: v.numpy().copy() for k, v in cols_h.items()}
        meta = {k: own(meta_h[k]) if k in meta_h else v for k, v in self._meta.items()}

        def samples_of(p, rows) -> List[SingleSample]:
            pos = p["pos"].tolist()
            return [SingleSample(data=[own(x[r]) for x in p["data"]],
                                 target=[tuple(own(x[r]) for x in h) for h in p["target"]],
                                 meta={k: v[pos[r]] for k, v in meta.items()},
                                 output=[own(x[r]) for x in p["output"]],
                                 metric={k: v[pos[r]] for k, v in self._data_metric.items()})
                    for r in rows]

        for p in random_h:
            self._random_samples.extend(samples_of(p, range(p["pos"].numel())))
        for p in worst_h:
            # the valid ones, ascending by score (the order a drained min-heap would give)
            ranked = sorted((s, r) for r, (s, ok) in enumerate(zip(p["score"].tolist(), p["valid"].tolist()))
                            if ok)
            self._worst_samples = samples_of(p, [r for _, r in ranked])
        self._dev_random, self._dev_worst = [], None
        if tracing:
            logger.info("finish trace: host-side assembly after the sync %.2f ms", 1e3 * (time.perf_counter() - t_s))
        if prof is not None:
            import io as _io
            import pstats
            prof.disable()
            out = _io.StringIO()
            pstats.Stats(prof, stream=out).sort_stats("cumulative").print_stats(14)
            logger.info("finish profile:\n%s", out.getvalue())

    @property
    def n_samples(self) -> int:
        return self._n_samples

    @property
    def random_samples(self) -> List[SingleSample]:
        return self._random_samples

    @property
    def worst_samples(self) -> List[SingleSample]:
        """Ascending by rank score: the most extreme sample last."""
        return self._worst_samples

    @property
    def data_metric(self) -> Dict[str, np.ndarray]:
        """Per-sample metrics of the whole split, one array per metric (the reference grows
        Python lists of scalars per sample, solver_worker.py:318-319; same length and order)."""
        return self._data_metric


def _tree_map(fn, *trees):
    """``fn`` over the matching leaves of nested dicts / lists / tuples of the same shape."""
    first = trees[0]
    if isinstance(first, dict):
        return {k: _tree_map(fn, *(t[k] for t in trees)) for k in first}
    if isinstance(first, (list, tuple)):
        return type(first)(_tree_map(fn, *xs) for xs in zip(*trees))
    return fn(*trees)


def _planned_order(sampler, accessor) -> List[int]:
    """``list(iter(sampler))`` as the reference hands it to its dataset cache — or, when the
    accessor is the null one that ignores the order, just that call's side effect on the global
    RNG: a stock ``RandomSampler`` draws one int64 seed and shuffles with a private generator, a
    ``ScaffoldSampler`` seeds a private generator with the epoch.  Materialising the order is
    O(len(dataset)) Python objects per split per epoch, comparable to the epoch's whole step
    time on an H100."""
    if isinstance(accessor, NullAccessor):
        if (type(sampler) is torch.utils.data.RandomSampler and not sampler.replacement
                and sampler.generator is None and sampler._num_samples is None):
            torch.empty((), dtype=torch.int64).random_()
            return []
        if isinstance(sampler, ScaffoldSampler):
            return []
    return list(iter(sampler))


_PINNED_BLOCKS: Dict[int, torch.Tensor] = {}


def _pinned_block(nbytes: int) -> torch.Tensor:
    """A process-wide, grow-only pinned staging block (uint8), reused by every split's read-back."""
    have = _PINNED_BLOCKS.get(0)
    if have is None or have.numel() < nbytes:
        # twice what is asked for: the payload varies from split to split with the number of random
        # picks, and every regrowth is a cudaHostAlloc, slow with several ranks page-locking at once
        have = _PINNED_BLOCKS[0] = torch.empty(max(2 * nbytes, 4 << 20), dtype=torch.uint8, pin_memory=True)
    return have


@contextmanager
def _gc_paused():
    """Cyclic GC off for the duration (unless FRL_B200_GC_IN_LOOP=1), restored on any exit."""
    import gc
    pause = gc.isenabled() and os.environ.get("FRL_B200_GC_IN_LOOP", "0") == "0"
    if pause:
        gc.disable()
    try:
        yield
    finally:
        if pause:
            gc.enable()
            if os.environ.get("FRL_B200_EPOCH_TRACE"):
                t0 = time.perf_counter()
                n = gc.collect()
                logger.info("gc trace: explicit collection after the loop: %.2f ms, %d unreachable, %d tracked objects",
                            1e3 * (time.perf_counter() - t0), n, len(gc.get_objects()))


class SolverWorker:
    def __init__(self, model: torch.nn.Module, criterion: BaseParallelCriterion,
                 optimizer: FusedArenaOptimizer, device: torch.device, run_opts: RunOpts,
                 cache=None, *, local_rank: int, node_idx: int, node_count: int,
                 pipeline: Optional[GradBucketPipeline] = None,
                 buffers: Optional[BufferBroadcaster] = None,
                 precision: Precision = Precision.FP32,
                 serialize_state: bool = True, graph_step: bool = False, ema=None,
                 channels_last: bool = False) -> None:
        self.model = model
        self.criterion = criterion
        self.optimizer = optimizer
        self.device = device
        self.run_opts = run_opts
        self.precision = precision
        self.accessor = NullAccessor(process_idx=local_rank)
        self.arena: ParamArena = optimizer.arena
        self.pipeline = pipeline or GradBucketPipeline(
            self.arena, optimizer, clip_norm=run_opts.optim.gradientClip)
        self.buffers = buffers
        self.ema = ema                 # ema.WeightEMA: held-out splits of a TRAIN run evaluate with it
        self.channels_last = channels_last       # True: device transforms are asked for NHWC batches
        self.cur_epoch = 0
        self._node_idx = node_idx
        self._node_count = node_count
        self._local_rank = local_rank
        self._serialize_state = serialize_state
        self._state_wanted = True      # False for epochs whose state the parent will not save
        self.loss_history: List[Tuple[int, Split, np.ndarray]] = []
        # CUDA-graph replay of the training step (opt-in: the Problem's forward must be
        # capturable — static shapes, no host syncs)
        self.graphed = None
        if graph_step and device.type == "cuda" and not run_opts.debugGrad \
                and not isinstance(criterion, GradNormWeightedCriterion):
            from .graph_step import GraphedTrainStep
            self.graphed = GraphedTrainStep(self)
        self.save_every = 1
        self.optimizer.zero_grad()
        if device.type == "cuda":
            import torch.backends.cudnn as cudnn
            cudnn.benchmark = os.environ.get("FRL_B200_CUDNN_BENCHMARK", "1") != "0"
            if not precision.bf16_storage:
                # parity mode: plain fp32 contractions (TF32 is on by default for convolutions)
                torch.backends.cuda.matmul.allow_tf32 = False
                cudnn.allow_tf32 = False

    # ------------------------------------------------------------------------------------------
    # one epoch over every split
    # ------------------------------------------------------------------------------------------
    def _pass_one_epoch(self, problem: Problem, loaders: Dict[Split, Any], mode: Mode
                        ) -> Dict[Split, FractionalEpochSplitPerformanceSummary]:
        epoch_stats: Dict[Split, FractionalEpochSplitPerformanceSummary] = {}
        names = list(self.criterion.loss_names)
        n_tasks = len(names)
        avg_grad_contributions = [0.0] * n_tasks
        contribution_count = 0
        amort = self.run_opts.metricAmortizationSchedule
        log_freq = self.run_opts.lossLoggingFreq
        dist_on = torch.distributed.is_available() and torch.distributed.is_initialized()

        trace = [] if os.environ.get("FRL_B200_EPOCH_TRACE") else None
        if not getattr(self, "_gc_frozen", False) and os.environ.get("FRL_B200_GC_IN_LOOP", "0") == "0":
            # everything alive now (model, optimizer, arena, datasets, loaders) lives as long as the
            # run: move it to the permanent generation so the collections that follow every
            # minibatch loop traverse only what an epoch created (the collection at the loop's end
            # is milliseconds, more for the ResNet Problems)
            import gc
            gc.collect()
            gc.freeze()
            self._gc_frozen = True

        def mark(what: str) -> None:
            if trace is not None:
                trace.append((what, time.perf_counter()))

        for data_type, loader in loaders.items():
            mark("split start")
            if dist_on:
                loader.sampler.set_epoch(self.cur_epoch)
            if hasattr(loader, "set_epoch"):
                # per-epoch device-side draws (DeviceImageAugment); cur_epoch resumes from the
                # checkpoint's epoch, so a resumed run continues the same stream
                loader.set_epoch(self.cur_epoch)
            # the planned order goes to the (null) cache accessor; drawing it also keeps the
            # global RNG stream identical to the reference's (solver_worker.py:431)
            self.accessor.set_sequence_indices(_planned_order(loader.sampler, self.accessor))
            loader.dataset.set_accessor(self.accessor)
            logger.info("Starting split %s" % data_type.name)

            training = (mode == Mode.TRAIN) and (data_type == Split.TRAIN)
            self.model.train(training)
            self.criterion.train(training)

            timer = EpochTimer()
            epoch_start = time.time()
            dataset = [d for d in problem.datasets if d.data_type == data_type][0]
            sampler_state = SamplerState(
                problem, len(loader.sampler), len(dataset), self.device,
                max(self.run_opts.numVisualizedSamples, MODEL_CONVERSION_TEST_SAMPLE_CT))
            n_batches = len(loader)
            # gradient accumulation: which microbatches open / close a group, and their weights
            plan = None
            if training and self.pipeline.accumulation > 1:
                plan = accumulation_plan(n_batches, self.pipeline.accumulation, loader.batch_size,
                                         len(loader.sampler))
            log = LossLog(n_tasks, n_batches, self.device)
            # with a weight EMA, the splits a TRAIN run only evaluates run on the averaged weights
            weights = (self.ema.swapped() if self.ema is not None and mode == Mode.TRAIN
                       and data_type != Split.TRAIN else nullcontext())
            checked = 0
            batch_start = time.time()
            mark("setup done")

            # The cyclic garbage collector stays out of the minibatch loop: a generation-2 pass over
            # a process holding a model, an optimizer and a loader takes milliseconds — several
            # steps — and fires wherever the allocation counter happens to trip (the first batch of
            # an epoch is then served late).  A step leaves no reference cycles behind
            # (its autograd graph is dropped explicitly below); FRL_B200_GC_IN_LOOP=1 keeps the
            # collector on for Problems whose hooks do.
            with weights, StepWatchdog(self.run_opts.minibatchTimeoutMs) as dog, sampler_state, _gc_paused():
                for minibatch_idx, (data, target, raw_meta) in enumerate(loader):
                    dog.kick()
                    if minibatch_idx < 3:
                        mark("batch %d served" % minibatch_idx)
                    data = [t if t.is_cuda else t.to(self.device, non_blocking=True) for t in data]
                    target = [tuple(t if t.is_cuda else t.to(self.device, non_blocking=True)
                                    for t in head) for head in target]
                    self.criterion.set_step_sink(log.row(minibatch_idx), log.nan_flag)
                    self.criterion._sink_written = False
                    if plan is not None:
                        mb = plan[minibatch_idx]
                        if data[0].shape[0] != mb.rows:
                            raise RuntimeError("gradient accumulation: minibatch %d has %d rows, the loader "
                                               "promised %d" % (minibatch_idx, data[0].shape[0], mb.rows))
                        self.pipeline.set_microbatch(first=mb.first, closes=mb.closes, weight=mb.weight,
                                                     group_scale=loader.batch_size / mb.group_rows)
                    output, total_loss, sub_loss, grad_norms = self._pass_one_minibatch(
                        minibatch_idx, data_type, data, target)
                    self._finish_loss_row(log, minibatch_idx, total_loss, sub_loss)

                    if grad_norms is not None:
                        contribution_count += 1
                        for i in range(n_tasks):
                            avg_grad_contributions[i] += (
                                grad_norms[i] - avg_grad_contributions[i]) / contribution_count

                    # lagged NaN guard: inspect rows the device has certainly finished
                    while checked <= minibatch_idx - NAN_CHECK_LAG:
                        log.wait(checked)
                        self._raise_if_nan(log, checked, data_type)
                        checked += 1

                    with torch.no_grad():
                        if minibatch_idx % amort == 0:
                            sampler_state.compute_metrics()
                        if self.graphed is not None and training:
                            output = [o.clone() for o in output]   # static graph buffers
                        sampler_state.append_sample(raw_meta, data, outputs=output, targets=target)
                        if log_freq > 0 and minibatch_idx % log_freq == 0:
                            self._summarize_times(dataset.data_type, timer)
                            log.wait(minibatch_idx)
                            row = log.row(minibatch_idx).tolist()
                            losses = dict(zip(names, row[1:]))
                            losses["total_loss"] = row[0]
                            logger.info("{}: {}".format(minibatch_idx, json.dumps(losses)))
                    # drop the autograd graph of this step now: its AccumulateGrad nodes would
                    # otherwise still be alive (and bound to this stream) when the next step is
                    # captured into a CUDA graph
                    output = total_loss = sub_loss = None
                    timer.batch.update(time.time() - batch_start)
                    batch_start = time.time()

                mark("last step issued")
                # the last window's fold is queued BEHIND the last steps (device-returning hooks:
                # pure device work, no host read) so the stream drains once, not twice; a NaN in
                # the last steps is still raised first — the fold's results are simply dropped
                # with the exception
                fold_early = sampler_state.metrics_on_device
                if fold_early:
                    sampler_state.compute_metrics()
                    mark("last window folded")
                if self.device.type == "cuda":
                    torch.cuda.current_stream().synchronize()
                mark("stream drained")
                while checked < n_batches:
                    self._raise_if_nan(log, checked, data_type)
                    checked += 1
                mark("nan guard done")
                if not fold_early:           # host-returning hooks: after the NaN guard, as before
                    sampler_state.compute_metrics()
                    mark("last window folded (late)")
                sampler_state.finish()
                mark("finish done")
            mark("loop context exited")
            timer.epoch.update(time.time() - epoch_start)

            per_step = log.rows[:n_batches].numpy()
            split_loss = {name: per_step[:, 1 + i].astype(np.float64).tolist()
                          for i, name in enumerate(names)}
            # per-step [total, sub-losses...] of every split, in the order they were run
            self.loss_history.append((self.cur_epoch, data_type, per_step.copy()))
            mark("metrics joined")
            epoch_stats[data_type] = self._epoch_summary(
                problem, sampler_state, dataset, split_loss, timer, mode)
            mark("summary done")
            if trace:
                t0 = trace[0][1]
                logger.info("epoch trace (ms since split start): " + ", ".join(
                    "%s %.2f" % (w, 1e3 * (ts - t0)) for w, ts in trace))
                trace.clear()

        if self.run_opts.debugGrad:
            logger.info("Task grad contributions: " + ", ".join(
                "%s: %f" % (n, c) for n, c in zip(names, avg_grad_contributions)))
        return epoch_stats

    def _finish_loss_row(self, log: LossLog, step: int, total_loss, sub_loss) -> None:
        """Make sure row ``step`` of the log gets written, then fence it with an event.

        The criteria of this package write the row themselves (the fused kernel does it from
        inside the forward launch).  A user subclass of ``BaseParallelCriterion`` that does not
        gets the same row from one small async device-to-host copy."""
        if not getattr(self.criterion, "_sink_written", False):
            with torch.no_grad():
                row = torch.stack([total_loss.detach().float()]
                                  + [v.detach().float() for v in sub_loss.values()])
                log.row(step).copy_(row, non_blocking=True)
        log.mark(step)

    def _raise_if_nan(self, log: LossLog, step: int, data_type: Split) -> None:
        if np.isnan(log.rows[step % log.capacity, 0].item()):
            raise FloatingPointError(
                "Losses become NaN for dataset {} at iteration {} minibatch {}!".format(
                    data_type.value, self.cur_epoch, step))

    # ------------------------------------------------------------------------------------------
    # one minibatch
    # ------------------------------------------------------------------------------------------
    def _cast_inputs(self, data: Sequence[torch.Tensor]) -> List[torch.Tensor]:
        if not self.precision.bf16_storage:
            return list(data)
        out = []
        for t in data:
            if t.is_cuda and t.dtype == torch.float32:
                lp = torch.empty_like(t, dtype=torch.bfloat16)
                # in the tensor's own storage order: a channels_last batch stays channels_last
                _native.cast_scale(t if _native.is_nhwc(t) else t.contiguous(), lp, 1.0)
                out.append(lp)
            else:
                out.append(t)
        return out

    def _pass_one_minibatch(self, minibatch_idx: int, data_type: Split,
                            data: Sequence[torch.Tensor],
                            target: Sequence[Tuple[torch.Tensor, ...]]):
        training = self.model.training
        debug_grad = (self.run_opts.debugGrad and isinstance(self.model, MultiTaskModel)
                      and minibatch_idx % 10 == 0)
        needs_graph = training or debug_grad or isinstance(self.criterion, GradNormWeightedCriterion)

        if training and self.graphed is not None and not debug_grad:
            sink = self.criterion._sink
            captured = self.graphed.ready_for(data, target)
            if captured is not None:
                output, total_loss, sub_loss = captured.run(data, target, sink)
                return output, total_loss, sub_loss, None
            self.criterion.set_step_sink(sink, self.criterion._nan_flag)

        if self.buffers is not None:
            self.buffers.sync()
        with torch.set_grad_enabled(needs_graph):
            output = self.model(self._cast_inputs(data))
            final_shared_params = None
            if debug_grad or isinstance(self.criterion, GradNormWeightedCriterion):
                final_shared_params = self.model.final_shared_params(output)
                if isinstance(self.criterion, GradNormWeightedCriterion):
                    self.criterion.set_shared_params(final_shared_params)
            total_loss, sub_loss = self.criterion(output, target)

        grad_norms: Optional[List[float]] = None
        if training:
            if debug_grad:
                grad_norms = [torch.autograd.grad(loss, final_shared_params, retain_graph=True)[0]
                              .norm().item() for loss in sub_loss.values()]
            self.pipeline.begin_step()
            total_loss.backward()
            self.pipeline.finish_step()
        return output, total_loss, sub_loss, grad_norms

    # ------------------------------------------------------------------------------------------
    # summaries
    # ------------------------------------------------------------------------------------------
    def _refine_sample_set(self, problem: Problem, samples: List[SingleSample]):
        assert len(samples) > 0, "Can't refine an empty sample set"
        first = samples[0]
        target = [stack_recursive([tuple(t.detach().cpu() for t in s.target[i]) for s in samples])
                  for i in range(len(first.target))]
        raw_meta = {}
        for key in first.meta:
            vals = [s.meta[key] for s in samples]
            raw_meta[key] = torch.stack(vals) if torch.is_tensor(vals[0]) else vals
        meta = problem.refine_batch_meta(raw_meta)
        output = [torch.stack([s.output[i] for s in samples]).cpu() for i in range(len(first.output))]
        data = [torch.stack([s.data[i] for s in samples]).cpu() for i in range(len(first.data))]
        metric = {key: np.array([s.metric[key] for s in samples]) for key in first.metric}
        return data, target, meta, output, metric

    @staticmethod
    def _serialize_sample_summaries(summaries: Sequence[SampleSummary]
                                    ) -> List[SerializableSampleSummary]:
        return [SerializableSampleSummary(image=s.image, text=s.text,
                                          plot=json.dumps(s.plot) if s.plot else None,
                                          source=s.source) for s in summaries]

    def _summarize_times(self, split: Split, timer: EpochTimer) -> None:
        logger.info("<{}>\tEpoch: {}\tAvg Batch Time: {:.3f}\tEpoch Time: {: .3f}".format(
            split.value.upper(), self.cur_epoch, timer.batch.avg, timer.epoch.sum))

    def _epoch_summary(self, problem: Problem, sampler: SamplerState, dataset: MultifieldDataset,
                       split_loss: Dict[str, List[float]], timer: EpochTimer, mode: Mode
                       ) -> FractionalEpochSplitPerformanceSummary:
        tag = dataset.data_type.value.upper()
        self._summarize_times(dataset.data_type, timer)
        logger.info("<{}>\tEpoch: {}\tLearning rate: {}\t".format(
            tag, self.cur_epoch, self.optimizer.param_groups[0]["lr"]))
        # unweighted mean over minibatches, as the reference (solver_worker.py:681)
        epoch_split_loss = {k: float(np.mean(v)) if len(v) else float("nan")
                            for k, v in split_loss.items()}
        logger.info("<{}>\tEpoch: {}\t{}".format(
            tag, self.cur_epoch, "".join("{}: {:.3f}\t".format(k, v) for k, v in epoch_split_loss.items())))
        epoch_data_metric = problem.summarize_epoch_metrics(sampler.data_metric)
        logger.info("<{}>\tEpoch: {}\t{}".format(
            tag, self.cur_epoch, "".join("{}: {:.3f}\t".format(k, v) for k, v in epoch_data_metric.items())))

        summary = FractionalEpochSplitPerformanceSummary(
            nSamples=sampler.n_samples, losses=epoch_split_loss, metrics=epoch_data_metric,
            samples=[], worstSamples=[],
            testIO=sampler.random_samples[:MODEL_CONVERSION_TEST_SAMPLE_CT])
        if self.run_opts.numVisualizedSamples == 0:
            return summary
        picked, worst = [], []
        if sampler.random_samples:
            picked = problem.summarize_epoch_samples(
                *self._refine_sample_set(problem, sampler.random_samples))
        if sampler.worst_samples:
            worst = problem.summarize_epoch_samples(
                *self._refine_sample_set(problem, sampler.worst_samples))
        return summary._replace(samples=self._serialize_sample_summaries(picked),
                                worstSamples=self._serialize_sample_summaries(worst))

    def _get_worker_performance_summary(
            self, epoch_stats: Dict[Split, FractionalEpochSplitPerformanceSummary]
    ) -> FractionalPerformanceSummary:
        """Model + optimizer state as device-agnostic bytes (reference solver_worker.py:733-761).

        Only the rank whose state the parent will use serialises (``serialize_state``); the
        exported module is a plain fp32 module: arena views are swapped for private copies of
        the master weights for the duration of the pickle."""
        model_bytes = b""
        optim_bytes = b""
        if self._state_wanted:
            self.pipeline.sync_sharded_state()        # collective; no-op unless fused NVLS step
        if self._serialize_state and self._state_wanted:
            was_training = self.model.training
            self.model.eval()
            self.pipeline.unpatch_linears()          # pickle plain nn.Linear modules
            try:
                with self.arena.exported(cpu=True, module=self.model):
                    with io.BytesIO() as buf:
                        torch.save(self.model, buf)
                        model_bytes = buf.getvalue()
            finally:
                self.pipeline.repatch_linears()
            with io.BytesIO() as buf:
                state = self.optimizer.state_dict()
                for entry in state["state"].values():
                    for k, v in entry.items():
                        if torch.is_tensor(v):
                            entry[k] = v.cpu()
                if self.ema is not None:
                    # travels to the parent with the optimizer state, which writes it to <stem>.ema
                    state[EMA_STATE_KEY] = self.ema.state_dict()
                torch.save(state, buf)
                optim_bytes = buf.getvalue()
            self.model.train(was_training)
        return FractionalPerformanceSummary(epoch=self.cur_epoch, modelBuffer=model_bytes,
                                            optimizerStateBuffer=optim_bytes,
                                            performance=epoch_stats)

    # ------------------------------------------------------------------------------------------
    # entry points
    # ------------------------------------------------------------------------------------------
    def train(self, problem: Problem, startEpoch: int, nEpochs: int, batchSize: int,
              scheduler) -> Iterator[FractionalPerformanceSummary]:
        self.cur_epoch = startEpoch
        assert Split.TRAIN in [d.data_type for d in problem.datasets], \
            "training dataset should be included"
        logger.info("Model layers")
        logger.info(str(self.model.modules))
        loaders = self._get_loaders(problem, batchSize=batchSize)
        while self.cur_epoch < nEpochs:
            self.cur_epoch += 1
            logger.info("Starting epoch %d" % self.cur_epoch)
            epoch_stats = self._pass_one_epoch(problem, loaders, Mode.TRAIN)
            logger.info("Finished epoch %d" % self.cur_epoch)
            scheduler.step()                      # once per epoch
            self._state_wanted = (self.cur_epoch % self.save_every == 0
                                  or self.cur_epoch == nEpochs)
            yield self._get_worker_performance_summary(epoch_stats)

    def eval(self, problem: Problem, batchSize: int) -> Iterator[FractionalPerformanceSummary]:
        logger.info("Model layers:")
        logger.info(str(self.model.modules))
        loaders = self._get_loaders(problem, batchSize=batchSize)
        epoch_stats = self._pass_one_epoch(problem, loaders, Mode.EVAL)
        self._state_wanted = False                # the parent writes no files in EVAL mode
        yield self._get_worker_performance_summary(epoch_stats)

    def _get_loaders(self, problem: Problem, batchSize: int
                     ) -> Dict[Split, torch.utils.data.DataLoader]:
        loaders = {}
        dist_on = torch.distributed.is_available() and torch.distributed.is_initialized()
        for dataset in problem.datasets:
            sampler = None
            if dist_on:
                sampler = ScaffoldSampler(dataset, shuffle_type=self.run_opts.shuffleType,
                                          node_idx=self._node_idx, node_count=self._node_count)
            split = dataset.data_type
            if self.run_opts.maxEpochImages > 0:
                logger.info("Using %d images per epoch." % self.run_opts.maxEpochImages)
                dataset = SubsetMultifieldDataset(dataset, range(self.run_opts.maxEpochImages))
            from .device_loader import DeviceBatchLoader, supports_device_batches
            if self.device.type == "cuda" and supports_device_batches(dataset):
                # raw dataset in pinned host memory: rows pulled by the GPU, transform on device
                out_dtype = torch.bfloat16 if self.precision.bf16_storage else torch.float32
                if self.channels_last:
                    dataset.device_transform.memory_format = torch.channels_last
                loaders[split] = DeviceBatchLoader(dataset, batch_size=batchSize, sampler=sampler,
                                                   device=self.device, out_dtype=out_dtype)
                ld = loaders[split]
                logger.info("input path for split %s: batched device loader (%s%s), wire dtypes %s",
                            split.value, ld.path,
                            ", %d gather threads" % ld.threads if ld.path == "host" else ", %d CTAs" % ld.blocks,
                            {k: str(v).replace("torch.", "") for k, v in ld._wire_dtype.items()})
                continue
            if self.device.type == "cuda":
                logger.warning(
                    "input path for split %s: per-sample DataLoader (__getitem__ + Python transform + "
                    "collate, as the reference) — the dataset does not expose `pinned_fields` + a "
                    "`device_transform` (transform.DeviceBatchTransform), so the host, not the GPU, "
                    "sets the step rate at large batches", split.value)
            loaders[split] = torch.utils.data.DataLoader(
                dataset, batch_size=batchSize, shuffle=sampler is None,
                num_workers=self.run_opts.numThreads,
                pin_memory=self.device.type == "cuda", sampler=sampler)
        return loaders
