"""Batched, device-side input pipeline for datasets that live in pinned host memory.

The reference feeds the loop through ``DataLoader`` -> per-sample ``__getitem__`` -> Python
``MultifieldTransform`` -> ``default_collate`` -> pageable H2D copy (reference
solver_worker.py:462-469, 805-832; transform.py:25-38): host Python per sample, which starves an
H100 at batch 4096.  A dataset that exposes

    pinned_fields     Dict[str, Tensor]   whole raw dataset, one pinned host tensor per field
                                          (or a ``PaddedLines`` text corpus: ragged rows)
    device_transform  DeviceBatchTransform

is consumed here instead: the index stream comes from the very same sampler/``DataLoader``
machinery (so sample order and global-RNG consumption stay bit-identical to the reference), the
raw rows of the next batches travel to HBM while the current batch trains, and the per-sample
arithmetic runs once per batch on the device (``frl_preproc_affine``).

Three ways to move the rows (``FRL_B200_INPUT_PATH``):

``kernel`` (default) ``frl_gather_rows``: 16 small CTAs (256 threads, no shared memory) pull the rows
                    over PCIe with 16-byte LSU loads on a high-priority copy stream — no host CPU
                    work, no staging copy in host DRAM;
``tma``             ``frl_gather_rows_tma``: the same with ``cp.async.bulk`` through 2 CTAs;
``host``            native worker threads (``frl_gather_pool_*``) copy the rows of batch *k+2* into
                    a pinned staging buffer, the copy engine moves batch *k+1* to HBM as one
                    contiguous DMA per field, the SMs see nothing of it.  The only path for
                    sources that are not pinned (memory-mapped ``.bin`` files), and the only one
                    that can ship bf16 over PCIe (``FRL_B200_INPUT_WIRE=bf16``).

A ``PaddedLines`` field (lines of a text corpus, each cut or padded to a fixed row) is only
served by ``kernel``: ``frl_gather_lines`` pulls the lines from the page-locked corpus into uint8
slots; ``auto`` selects it and ``tma`` / ``host`` are refused.

Alone, every path is bound by PCIe.  Under the training step, CTAs that occupy SMs for the
length of a batch transfer slow the GEMMs: the TMA kernel's 128 KB of staging takes an SM from
the GEMMs per CTA, the LSU kernel's CTAs fit beside them.  The host path costs 3x the payload
in host DRAM traffic and 16-24 busy threads, so its speed depends on how many ranks share a
socket and on the neighbours' load.  Which path is fastest on H100 has not been measured; the
default (``kernel``) is not tuned on H100.
"""
from collections import deque
from typing import Dict, Iterator, List, Optional, Tuple

import math
import os

import torch
import torch.utils.data

from . import _native
from .transform import DeviceBatchTransform
from .types import Split


class _IndexOnly(torch.utils.data.Dataset):
    def __init__(self, n: int) -> None:
        self._n = n

    def __len__(self) -> int:
        return self._n

    def __getitem__(self, i: int) -> int:
        return i

    def __getitems__(self, items: List[int]) -> List[int]:      # batched fetch: no per-sample call
        return items


def _collate_indices(items: List[int]) -> torch.Tensor:
    return torch.tensor(items, dtype=torch.int64)


def randperm_quiet(n: int, generator: torch.Generator) -> torch.Tensor:
    """``torch.randperm(n, generator=generator)`` — the same values, the same generator state
    afterwards — with intra-op parallelism off for the call.  The draw itself is serial
    (Fisher-Yates on the generator); only the initial ``arange`` fill is parallel, and waking a
    64-128-thread OpenMP team that went to sleep during the previous epoch costs milliseconds
    per epoch."""
    threads = torch.get_num_threads()
    if threads == 1:
        return torch.randperm(n, generator=generator)
    torch.set_num_threads(1)
    try:
        return torch.randperm(n, generator=generator)
    finally:
        torch.set_num_threads(threads)


class PaddedLines:
    """A ragged byte field in ``pinned_fields``: row ``i`` is line ``i`` of a text corpus,
    ``corpus[starts[i] : starts[i+1] - 1]``, cut or padded with ``pad`` to ``row_len`` bytes
    (``text_dataset.TextDataset``).  ``corpus`` provides ``pin() -> device-usable address``,
    ``n_bytes`` and ``alloc_bytes`` (16-byte aligned, a multiple of 16); ``starts`` is the int64
    line-start table, uploaded to each device once.  Served by ``frl_gather_lines`` (K8t)."""

    def __init__(self, corpus, starts, row_len: int, pad: int = 0) -> None:
        self.corpus = corpus
        self.starts = starts
        self.row_len = int(row_len)
        self.pad = int(pad)
        self._starts_dev: Dict[torch.device, torch.Tensor] = {}

    def starts_on(self, device: torch.device) -> torch.Tensor:
        if device not in self._starts_dev:
            self._starts_dev[device] = torch.from_numpy(self.starts).to(device)
        return self._starts_dev[device]

    def __getstate__(self):
        state = self.__dict__.copy()
        state["_starts_dev"] = {}
        return state


def supports_device_batches(dataset) -> bool:
    return (isinstance(getattr(dataset, "pinned_fields", None), dict)
            and isinstance(getattr(dataset, "device_transform", None), DeviceBatchTransform))


def _local_world() -> int:
    local_world = int(os.environ.get("LOCAL_WORLD_SIZE", "0") or 0)
    if local_world < 1:
        local_world = 1
        if torch.distributed.is_available() and torch.distributed.is_initialized():
            local_world = max(1, min(torch.distributed.get_world_size(), torch.cuda.device_count() or 1))
    return local_world


def default_input_path() -> str:
    """``kernel`` everywhere (not tuned on H100): it needs nothing from the host but PCIe reads.
    ``host`` can be faster when ONE rank has the node's CPUs and DRAM to itself, but it costs
    host DRAM 3x the PCIe payload (gather read + staging write + DMA read) and 16-24 busy threads:
    several ranks on one socket compete for it, and on a shared host its speed follows the
    neighbours' load.
    The LSU kernel's CTAs (256 threads, no shared memory) fit beside the GEMM CTAs on an SM; the
    TMA kernel's 128 KB of staging does not, so each of its CTAs takes an SM from the GEMMs."""
    return "kernel"


def default_gather_threads() -> int:
    """Worker threads for the host gather: this rank's share of the cores it may run on."""
    env = os.environ.get("FRL_B200_INPUT_THREADS")
    if env:
        return max(1, int(env))
    try:
        avail = len(os.sched_getaffinity(0))
    except AttributeError:
        avail = os.cpu_count() or 4
    local_world = _local_world()
    share = min(avail, (os.cpu_count() or avail) // local_world)
    return max(1, min(share - 2, 24))


class DeviceBatchLoader:
    """Iterates ``(data, target, raw_meta)`` like the reference's DataLoader, already on device."""

    def __init__(self, dataset, *, batch_size: int, sampler, device: torch.device,
                 out_dtype: torch.dtype = torch.float32, depth: int = 3,
                 path: Optional[str] = None) -> None:
        self.dataset = dataset
        self.device = device
        self.batch_size = batch_size
        self.out_dtype = out_dtype
        self.depth = max(depth, 2)
        # same construction as the reference's loader -> same sampler classes, same RNG draws
        self._index_loader = torch.utils.data.DataLoader(
            _IndexOnly(len(dataset)), batch_size=batch_size, shuffle=sampler is None,
            sampler=sampler, num_workers=0, collate_fn=_collate_indices)
        self.sampler = self._index_loader.sampler
        self._fields: Dict[str, torch.Tensor] = dataset.pinned_fields
        # ragged text fields: only the GPU-pulled LSU kernel (K8t) serves them
        self._lines: Dict[str, PaddedLines] = {k: v for k, v in self._fields.items() if isinstance(v, PaddedLines)}
        for name, t in self._fields.items():
            if name not in self._lines and (t.is_cuda or not t.is_contiguous()):
                raise ValueError(f"field {name!r} must be a contiguous host tensor")
        # sources the GPU can read directly (pinned, device-mapped) or only the CPU can (e.g. a
        # memory-mapped .bin file: served by the host gather pool)
        all_pinned = all(t.is_pinned() for name, t in self._fields.items() if name not in self._lines)
        # high priority: the next batch's transfer should start as soon as it is submitted
        self._copy_stream = torch.cuda.Stream(device=device, priority=-1)
        self.path = path or os.environ.get("FRL_B200_INPUT_PATH", "auto")
        if self._lines:
            if self.path not in ("auto", "kernel"):
                raise ValueError("input path %r cannot serve the padded text field(s) %s: only the "
                                 "GPU-pulled kernel path gathers ragged lines"
                                 % (self.path, ", ".join(repr(k) for k in self._lines)))
            self.path = "kernel"
        if self.path == "auto":
            self.path = default_input_path() if all_pinned else "host"
        if self.path != "host" and not all_pinned:
            raise ValueError("input path %r needs pinned host tensors; these fields are plain "
                             "CPU memory (use the host path)" % self.path)
        if self.path not in ("host", "tma", "kernel"):
            raise ValueError(f"unknown input path {self.path!r}")
        # CTAs of the GPU-pulled paths: each LSU CTA keeps 32 KB of PCIe reads in flight, 8 of them
        # cover the ~110 KB the link needs; more only take SMs from the step's GEMMs
        self.blocks = int(os.environ.get("FRL_B200_INPUT_BLOCKS", "2" if self.path == "tma" else "8"))
        # wire dtype per field: fp32 fields the dataset's transform declares bf16-tolerant
        # (``bf16_wire_fields``) travel over PCIe as bf16 when the run computes in bf16 — half the
        # bytes of the step's dominant transfer.  FRL_B200_INPUT_WIRE: "auto" (default: do it),
        # "native" (never), "bf16" (same as auto).  GPU-pulled paths read a bf16 copy of the field
        # made ONCE here (the declared tolerance is the dataset author's statement that rounding
        # the raw field is as good as rounding the transformed one); the host path converts while
        # it gathers (the source may be a memory-mapped file that must stay as it is).
        self.wire = os.environ.get("FRL_B200_INPUT_WIRE", "auto")
        tolerant = set(getattr(dataset.device_transform, "bf16_wire_fields", ()) or ())
        self._wire_dtype: Dict[str, torch.dtype] = {}
        for name, t in self._fields.items():
            if name in self._lines:
                self._wire_dtype[name] = torch.uint8
                continue
            cvt = (self.wire in ("auto", "bf16") and out_dtype == torch.bfloat16
                   and t.dtype == torch.float32 and name in tolerant)
            self._wire_dtype[name] = torch.bfloat16 if cvt else t.dtype
        if self.path != "host":
            converted = {}
            cache = getattr(dataset, "_frl_wire_cache", None)
            if cache is None:
                cache = {}
                try:
                    dataset._frl_wire_cache = cache       # epochs / loaders of one run share it
                except AttributeError:
                    pass
            for name, t in self._fields.items():
                if name not in self._lines and self._wire_dtype[name] != t.dtype:
                    key = (name, t.data_ptr(), self._wire_dtype[name])
                    if key not in cache:
                        cache[key] = t.to(self._wire_dtype[name]).pin_memory()
                    converted[name] = cache[key]
            if converted:
                self._fields = {k: converted.get(k, v) for k, v in self._fields.items()}
        # the corpus is page-locked in this (rank) process, its start table uploaded, on first use
        self._line_src = {name: (f.corpus.pin(), f.starts_on(device)) for name, f in self._lines.items()}
        row_shape = {name: ((f.row_len,) if name in self._lines else tuple(f.shape[1:]))
                     for name, f in self._fields.items()}
        self._slots = []
        for _ in range(self.depth):
            slot = {name: torch.empty((batch_size,) + row_shape[name], dtype=self._wire_dtype[name],
                                      device=device) for name in self._fields}
            slot["__idx_host"] = torch.empty(batch_size, dtype=torch.int64, pin_memory=True)
            slot["__idx_dev"] = torch.empty(batch_size, dtype=torch.int64, device=device)
            self._slots.append(slot)
        self._ready = [torch.cuda.Event() for _ in range(self.depth)]
        self._freed = [torch.cuda.Event() for _ in range(self.depth)]
        self._pool = None
        self.threads = 0
        if self.path == "host":
            self._pool = _native.HostGatherPool(default_gather_threads())
            self.threads = self._pool.n_threads
            self._n_stage = self.depth + 1
            self._stage = [{name: torch.empty((batch_size,) + tuple(t.shape[1:]),
                                              dtype=self._wire_dtype[name], pin_memory=True)
                            for name, t in self._fields.items()}
                           for _ in range(self._n_stage)]
            self._stage_idx = [torch.empty(batch_size, dtype=torch.int64, pin_memory=True)
                               for _ in range(self._n_stage)]
            self._dma_done = [torch.cuda.Event() for _ in range(self._n_stage)]
        self.h2d_bytes_per_batch = sum(
            math.prod(row_shape[name]) * torch.empty(0, dtype=self._wire_dtype[name]).element_size()
            for name in self._fields) * batch_size + 8 * batch_size

    def __len__(self) -> int:
        return len(self._index_loader)

    def set_epoch(self, epoch: int) -> None:
        """Tell the dataset's transform which epoch the next pass belongs to (its per-sample
        random draws may be keyed by it)."""
        self.dataset.device_transform.set_epoch(epoch)

    def _index_batches(self) -> Iterator[torch.Tensor]:
        """int64 index tensors, one per minibatch, in the order the reference's
        ``enumerate(DataLoader)`` would serve them — and with the same draws from the global
        RNG: iterating a DataLoader takes ``_base_seed`` when the iterator is built, then a
        ``RandomSampler`` takes its permutation seed on the first ``next``.  For the stock
        samplers the permutation stays a tensor: ``randperm(n).tolist()`` plus the per-batch list
        handling is O(n) Python work per epoch, ~60 ns per sample against ~360 ns per sample of
        H100 step time."""
        sampler = self.sampler
        perm = None
        if (type(sampler) is torch.utils.data.RandomSampler and not sampler.replacement
                and sampler.generator is None and sampler._num_samples is None):
            torch.empty((), dtype=torch.int64).random_()                  # DataLoader iterator: _base_seed
            seed = int(torch.empty((), dtype=torch.int64).random_().item())   # RandomSampler.__iter__
            gen = torch.Generator()
            gen.manual_seed(seed)
            import time as _time
            t0 = _time.perf_counter()
            perm = randperm_quiet(len(sampler.data_source), gen)
            if os.environ.get("FRL_B200_EPOCH_TRACE"):
                print("loader trace: randperm(%d) %.2f ms" % (perm.numel(), 1e3 * (_time.perf_counter() - t0)),
                      flush=True, file=__import__("sys").stderr)
        elif hasattr(sampler, "rank_index_tensor"):                       # ScaffoldSampler
            torch.empty((), dtype=torch.int64).random_()                  # DataLoader iterator: _base_seed
            perm = sampler.rank_index_tensor()
        if perm is None:
            yield from self._index_loader
            return
        for lo in range(0, perm.numel(), self.batch_size):
            yield perm[lo:lo + self.batch_size]

    # -- SM paths: the GPU pulls the rows of batch k into device slot k % depth -------------------
    def _upload(self, k: int, idx: torch.Tensor) -> int:
        s = k % self.depth
        slot = self._slots[s]
        n = idx.numel()
        self._ready[s].synchronize()      # the slot's previous index upload has left the pinned row
        slot["__idx_host"][:n].copy_(idx)
        with torch.cuda.stream(self._copy_stream):
            self._copy_stream.wait_event(self._freed[s])          # previous user of the slot is done
            slot["__idx_dev"][:n].copy_(slot["__idx_host"][:n], non_blocking=True)
            for name, src in self._fields.items():
                if name in self._lines:
                    corpus = src.corpus
                    addr, starts_dev = self._line_src[name]
                    _native.gather_lines(addr, corpus.n_bytes, corpus.alloc_bytes, starts_dev,
                                         slot["__idx_dev"][:n], slot[name][:n], pad=src.pad,
                                         max_blocks=self.blocks)
                    continue
                row_bytes = src[0].numel() * src.element_size()
                wide = row_bytes >= 4096 and row_bytes % 16 == 0
                if wide and self.path == "tma":
                    _native.gather_rows_tma(src, slot["__idx_dev"][:n], slot[name][:n],
                                            max_blocks=self.blocks)
                else:
                    _native.gather_rows(src, slot["__idx_dev"][:n], slot[name][:n],
                                        max_blocks=self.blocks if wide else 8)
            self._ready[s].record()
        return n

    # -- host path: gather into staging slot g % n_stage, later one DMA per field ------------------
    def _submit_gather(self, g: int, idx: torch.Tensor):
        st = g % self._n_stage
        self._dma_done[st].synchronize()          # the DMA that last read this staging slot is over
        n = idx.numel()
        self._stage_idx[st][:n].copy_(idx)
        ticket = 0
        for name, src in self._fields.items():
            if self._wire_dtype[name] != src.dtype:
                ticket = self._pool.submit_f32_to_bf16(src, idx, self._stage[st][name])
            else:
                ticket = self._pool.submit(src, idx, self._stage[st][name])
        return st, n, ticket

    def _issue_dma(self, k: int, st: int, n: int, ticket: int) -> int:
        self._pool.wait(ticket)
        s = k % self.depth
        slot = self._slots[s]
        with torch.cuda.stream(self._copy_stream):
            self._copy_stream.wait_event(self._freed[s])
            slot["__idx_dev"][:n].copy_(self._stage_idx[st][:n], non_blocking=True)
            for name in self._fields:
                slot[name][:n].copy_(self._stage[st][name][:n], non_blocking=True)
            self._ready[s].record()
            self._dma_done[st].record()
        return n

    def __iter__(self) -> Iterator[Tuple[List[torch.Tensor], List[Tuple[torch.Tensor, ...]], dict]]:
        split: Split = self.dataset.data_type
        transform: DeviceBatchTransform = self.dataset.device_transform
        import time as _time
        t_iter = _time.perf_counter()
        trace = os.environ.get("FRL_B200_EPOCH_TRACE")
        for ev in self._freed:
            ev.record()
        batches = self._index_batches()
        uploaded = deque()        # sizes of the batches whose transfer has been issued
        k_up = 0
        if self.path == "host":
            for ev in self._dma_done:
                ev.record()
            gathered = deque()
            g = 0

            def gather_next() -> None:
                nonlocal g
                try:
                    idx = next(batches)
                except StopIteration:
                    return
                gathered.append(self._submit_gather(g, idx))
                g += 1

            def upload_next() -> None:
                nonlocal k_up
                if gathered:
                    uploaded.append(self._issue_dma(k_up, *gathered.popleft()))
                    k_up += 1

            gather_next()
            gather_next()
            upload_next()
            advance = lambda: (upload_next(), gather_next())           # noqa: E731
        else:
            def advance() -> None:
                nonlocal k_up
                try:
                    idx = next(batches)
                except StopIteration:
                    return
                uploaded.append(self._upload(k_up, idx))
                k_up += 1

            advance()
        if trace:
            print("loader trace: first upload issued %.2f ms after iter()" % (1e3 * (_time.perf_counter() - t_iter)),
                  flush=True, file=__import__("sys").stderr)
        k = 0
        while uploaded:
            advance()                             # keep the next transfers in flight
            if trace and k == 0:
                print("loader trace: second upload issued %.2f ms" % (1e3 * (_time.perf_counter() - t_iter)), flush=True, file=__import__("sys").stderr)
            n = uploaded.popleft()
            s = k % self.depth
            slot = self._slots[s]
            torch.cuda.current_stream().wait_event(self._ready[s])
            raw = {name: slot[name][:n] for name in self._fields}
            if getattr(transform, "needs_index", False):
                data, target = transform.apply(raw, split, self.out_dtype, index=slot["__idx_dev"][:n])
            else:
                data, target = transform.apply(raw, split, self.out_dtype)
            meta = transform.meta(raw, slot["__idx_dev"][:n])
            # the loop retains targets/meta of the last minibatches for its amortised metrics,
            # the slot is recycled `depth` batches from now: hand out no views of it
            owned = {t.untyped_storage().data_ptr() for t in slot.values() if t.is_cuda}
            keep = lambda t: (t.clone() if torch.is_tensor(t) and t.is_cuda     # noqa: E731
                              and t.untyped_storage().data_ptr() in owned else t)
            data = [keep(t) for t in data]
            target = [tuple(keep(t) for t in head) for head in target]
            meta = {k: keep(v) for k, v in meta.items()}
            if trace and k == 0:
                print("loader trace: first batch ready to yield %.2f ms" % (1e3 * (_time.perf_counter() - t_iter)), flush=True, file=__import__("sys").stderr)
            yield data, target, meta
            # the consumer has issued everything that reads this slot: let the copy stream reuse it
            self._freed[s].record()
            k += 1
