"""The launches that end a step of ``grad_sync.GradBucketPipeline``, pinned for every configuration:
optimizer (SGD with momentum, Adam, LARS, LAMB) x clip x (every gradient present, one layer unused)
x accumulation (k = 1, k = 3 with a short last group) x gradients (read in place where autograd
left them, or copied into the arena) x (``finish_step()``, or ``finish_step(defer_tail=True)`` and
the CUDA-graph hand-over to ``run_tail``), on one rank and on two ranks over gloo.

The kernels are the CPU doubles of ``oracle.optim_np`` / ``layerwise_oracle``, each launch also
logged as one line ``kernel where source xscale [first] [clip]``:

* ``where``: the arena range ``lo:hi`` of a flat launch, or the slot indices of a segment table;
* ``source``: where the gradients were read: ``arena``, ``accumulator``, ``in-place`` (where autograd
  left them) or ``NULL``; for a table, the slots grouped by source;
* ``xscale``: the gradient scale (K3: its pre-scale; K10: the microbatch weight);
* ``clip``: a device clip coefficient was passed.

The same runs are checked against ``torch.optim`` (one rank) and for replica agreement (two ranks).

Some sequences are pinned as they are, not as they should be:

* a step in which a parameter got no gradient updates inside ``finish_step(defer_tail=True)``
  already, and the hand-over's ``run_tail`` then updates every slot once more;
* with clipping, the hand-over's whole-tensor update reads the gradients in place, not the arena
  copies the norm was computed from (the same values in fp32);
* such a step gathers its gradients into the arena even when a whole-tensor update could read them
  in place.
"""
import itertools
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn as nn

import frl_b200  # noqa: F401
from frl_b200 import fused_optim, grad_sync, multi_tensor
from frl_b200.arena import ParamArena
from frl_b200.grad_sync import accumulation_plan
from frl_b200.types import LayerAdaptation, OptAlgorithm, OptimOpts
from layerwise_oracle import LayerwiseTorch, _read
from test_accumulation_host import AccumKernelDouble

f32 = np.float32
_SGD = OptimOpts(algo=OptAlgorithm.SGD, lr=0.05, momentum=0.9, weightDecay=1e-2)
_ADAM = OptimOpts(algo=OptAlgorithm.ADAM, lr=0.01, weightDecay=1e-2)
OPTS = {"sgd": (_SGD, LayerAdaptation.NONE), "adam": (_ADAM, LayerAdaptation.NONE),
        "lars": (_SGD, LayerAdaptation.LARS), "lamb": (_ADAM, LayerAdaptation.LAMB)}
CLIP = 0.05
B, N_ROWS, N_MB = 4, 14, 4         # per rank: microbatches of 4, 4, 4 and 2 rows


class RecordingDouble(AccumKernelDouble):
    """The CPU kernel doubles plus ``flatten_grads`` and the K2-mt entry points, every launch logged."""

    def __init__(self):
        super().__init__()
        self.log = []
        self.pipe = None

    def _source(self, ptr):
        if not ptr:
            return "NULL"
        for name, t in (("arena", self.pipe.arena.grad), ("accumulator", self.pipe.acc)):
            if t is not None and t.data_ptr() <= ptr < t.data_ptr() + t.numel() * t.element_size():
                return name
        return "in-place"

    def _range(self, g, n):
        src = self._source(g.data_ptr())
        base = self.pipe.acc if src == "accumulator" else self.pipe.arena.grad
        lo = (g.data_ptr() - base.data_ptr()) // base.element_size()
        return "%d:%d %s" % (lo, lo + n, src)

    def _slots(self, table):
        by_src = {}
        for i, s in enumerate(table.slots):
            by_src.setdefault(self._source(table._segs[i].g or 0), []).append(str(s.index))
        return " ".join("[%s] %s" % (" ".join(idx), src) for src, idx in by_src.items())

    def _log(self, name, where, scale, clip=None, first=False):
        self.log.append("%s %s x%g%s%s" % (name, where, scale, " first" if first else "",
                                            " clip" if clip is not None else ""))

    def _rows(self, table):
        for i, s in enumerate(table.slots):
            row = table._segs[i]
            yield s, torch.from_numpy(_read(row.g, s.numel, row.g_dtype))

    @staticmethod
    def _cut(vec, s):
        return None if vec is None else vec[s.offset:s.end]

    def sgd_momentum(self, p, g, buf, p_lp, n, **kw):
        self._log("sgd", self._range(g, n), kw["grad_scale"], kw.get("grad_scale_dev"))
        super().sgd_momentum(p, g, buf, p_lp, n, **kw)

    def adam(self, p, g, m, v, vmax, p_lp, n, **kw):
        self._log("adam", self._range(g, n), kw["grad_scale"], kw.get("grad_scale_dev"))
        super().adam(p, g, m, v, vmax, p_lp, n, **kw)

    def grad_sumsq_clip(self, g, n, **kw):
        self._log("sumsq", self._range(g, n), kw["pre_scale"])
        super().grad_sumsq_clip(g, n, **kw)

    def grad_accumulate_mt(self, acc, table, *, w=1.0, first=False, dyn=None):
        self._log("accumulate", self._slots(table), w, first=first)
        super().grad_accumulate_mt(acc, table, w=w, first=first, dyn=dyn)

    def lars_mt(self, p, buf, p_lp, table, *args, **kw):
        self._log("lars_mt", self._slots(table), kw["grad_scale"], kw.get("grad_scale_dev"))
        super().lars_mt(p, buf, p_lp, table, *args, **kw)

    def lamb_mt(self, p, m, v, p_lp, table, *args, **kw):
        self._log("lamb_mt", self._slots(table), kw["grad_scale"], kw.get("grad_scale_dev"))
        super().lamb_mt(p, m, v, p_lp, table, *args, **kw)

    def flatten_grads(self, table, arena_grad, *, scale=1.0):
        self._log("flatten", self._slots(table), scale)
        for s, g in self._rows(table):
            arena_grad[s.offset:s.end] = (g * scale).to(arena_grad.dtype)

    def sgd_momentum_mt(self, p, buf, p_lp, table, **kw):
        self._log("sgd_mt", self._slots(table), kw["grad_scale"])
        for s, g in self._rows(table):
            super().sgd_momentum(self._cut(p, s), g, self._cut(buf, s), self._cut(p_lp, s), s.numel, **kw)

    def adam_mt(self, p, m, v, vmax, p_lp, table, **kw):
        self._log("adam_mt", self._slots(table), kw["grad_scale"])
        for s, g in self._rows(table):
            super().adam(self._cut(p, s), g, self._cut(m, s), self._cut(v, s), self._cut(vmax, s),
                         self._cut(p_lp, s), s.numel, **kw)


class _Net(nn.Module):
    def __init__(self):
        super().__init__()
        torch.manual_seed(3)
        self.l0, self.l1, self.l2 = nn.Linear(7, 5), nn.Linear(5, 5), nn.Linear(5, 2)
        self.extra = nn.Parameter(torch.tensor([1.0]))          # criterion-side: never clipped

    def model_params(self):
        return [p for m in (self.l0, self.l1, self.l2) for p in m.parameters()]

    def loss(self, x, skip):
        """``skip``: leave the middle layer (slots 2 and 3) out, so it gets no gradient."""
        h = self.l0(x).relu()
        if not skip:
            h = self.l1(h).relu()
        return self.l2(h).square().mean() * self.extra.sum() * 3


def _in_place(g, slot):
    return g.layout == torch.strided and g.is_contiguous() and g.numel() == slot.numel


def _run(double, opt, clip, k, in_place, defer, skip, xs, rank=0, world=1):
    """Train over ``xs`` (N_MB microbatches per rank, ``k`` per update); returns (log, parameters)."""
    net = _Net()
    arena = ParamArena(net.model_params(), [net.extra], device="cpu")
    optim_opts, la = OPTS[opt]
    optimizer = fused_optim.create_fused_optimizer(arena, optim_opts, la)
    kw = dict(bucket_cap_mb=0.0001, first_bucket_mb=0.00005) if world > 1 else {}
    pipe = grad_sync.GradBucketPipeline(arena, optimizer, world_size=world, clip_norm=clip, accumulation=k, **kw)
    pipe.mt_enabled = in_place
    double.pipe, double.log = pipe, []
    for j, mb in enumerate(accumulation_plan(N_MB, k, B, N_ROWS)):
        pipe.set_microbatch(first=mb.first, closes=mb.closes, weight=mb.weight, group_scale=B / mb.group_rows)
        pipe.begin_step()
        net.loss(xs[j * B * world:(j + 1) * B * world][rank::world], skip).backward()
        if defer:                       # what a CUDA-graph capture and its replay do, minus the graph
            pipe.finish_step(defer_tail=True)
            refs, tables = pipe.detach_grad_refs()
            pipe.run_tail(refs, tables, pipe.last_ready)
        else:
            pipe.finish_step()
    pipe.remove_hooks()
    return double.log, [p.detach().clone() for p in net.parameters()]


def _torch_reference(opt, clip, k, skip, xs):
    net = _Net()
    params = net.model_params() + [net.extra]
    o, la = OPTS[opt]
    if la is LayerAdaptation.LARS:
        ref = LayerwiseTorch(params, "lars", lr=o.lr, momentum=o.momentum, weight_decay=o.weightDecay)
    elif la is LayerAdaptation.LAMB:
        ref = LayerwiseTorch(params, "lamb", lr=o.lr, weight_decay=o.weightDecay, eps=o.epsilon)
    elif o.algo == OptAlgorithm.SGD:
        ref = torch.optim.SGD(params, lr=o.lr, momentum=o.momentum, weight_decay=o.weightDecay)
    else:
        ref = torch.optim.Adam(params, lr=o.lr, weight_decay=o.weightDecay, eps=o.epsilon)
    lo = 0
    for j, mb in enumerate(accumulation_plan(N_MB, k, B, N_ROWS)):
        if mb.closes:
            hi = j * B + mb.rows
            ref.zero_grad()
            net.loss(xs[lo:hi], skip).backward()
            if clip:
                torch.nn.utils.clip_grad_norm_([p for p in net.model_params() if p.grad is not None], clip)
            ref.step()
            lo = hi
    return [p.detach().clone() for p in net.parameters()]


def _key(opt, clip, skip, k, in_place):
    return "%s %s %s k%d %s" % (opt, "clip" if clip else "noclip", "partial" if skip else "all", k,
                                "in-place" if in_place else "arena")


# ---- the pinned sequences ------------------------------------------------------------------------
# k = 1: the sequence of ONE step (the run makes four); k = 3: the whole run (a group of three
# microbatches, then a short group of one).  finish_step() and the hand-over to run_tail() launch
# the same, except where DEFERRED lists what the hand-over launches instead.

EXPECTED = {
    "sgd noclip all k1 in-place": [
        "sgd_mt [0 1 2 3 4 5 6] in-place x1",
    ],
    "sgd noclip all k1 arena": [
        "sgd 0:120 arena x1",
    ],
    "sgd noclip all k3 in-place": [
        "accumulate [0 1 2 3 4 5 6] in-place x1 first", "accumulate [0 1 2 3 4 5 6] in-place x1",
        "accumulate [0 1 2 3 4 5 6] in-place x1", "sgd 0:120 accumulator x0.333333",
        "accumulate [0 1 2 3 4 5 6] in-place x0.5 first", "sgd 0:120 accumulator x2",
    ],
    "sgd noclip all k3 arena": [
        "accumulate [0 1 2 3 4 5 6] arena x1 first", "accumulate [0 1 2 3 4 5 6] arena x1",
        "accumulate [0 1 2 3 4 5 6] arena x1", "sgd 0:120 accumulator x0.333333",
        "accumulate [0 1 2 3 4 5 6] arena x0.5 first", "sgd 0:120 accumulator x2",
    ],
    "sgd noclip partial k1 in-place": [
        "flatten [0 1 4 5 6] in-place x1", "sgd 0:45 arena x1", "sgd 88:113 arena x1",
    ],
    "sgd noclip partial k1 arena": [
        "sgd 0:45 arena x1", "sgd 88:113 arena x1",
    ],
    "sgd noclip partial k3 in-place": [
        "accumulate [0 1 4 5 6] in-place [2 3] NULL x1 first",
        "accumulate [0 1 4 5 6] in-place [2 3] NULL x1", "accumulate [0 1 4 5 6] in-place [2 3] NULL x1",
        "sgd 0:45 accumulator x0.333333", "sgd 88:113 accumulator x0.333333",
        "accumulate [0 1 4 5 6] in-place [2 3] NULL x0.5 first", "sgd 0:45 accumulator x2",
        "sgd 88:113 accumulator x2",
    ],
    "sgd noclip partial k3 arena": [
        "accumulate [0 1 4 5 6] arena [2 3] NULL x1 first", "accumulate [0 1 4 5 6] arena [2 3] NULL x1",
        "accumulate [0 1 4 5 6] arena [2 3] NULL x1", "sgd 0:45 accumulator x0.333333",
        "sgd 88:113 accumulator x0.333333", "accumulate [0 1 4 5 6] arena [2 3] NULL x0.5 first",
        "sgd 0:45 accumulator x2", "sgd 88:113 accumulator x2",
    ],
    "sgd clip all k1 in-place": [
        "flatten [0 1 2 3 4 5 6] in-place x1", "sumsq 0:112 arena x1", "sgd 0:112 arena x1 clip",
        "sgd 112:120 arena x1",
    ],
    "sgd clip all k1 arena": [
        "sumsq 0:112 arena x1", "sgd 0:112 arena x1 clip", "sgd 112:120 arena x1",
    ],
    "sgd clip all k3 in-place": [
        "accumulate [0 1 2 3 4 5 6] in-place x1 first", "accumulate [0 1 2 3 4 5 6] in-place x1",
        "accumulate [0 1 2 3 4 5 6] in-place x1", "sumsq 0:112 accumulator x0.333333",
        "sgd 0:112 accumulator x0.333333 clip", "sgd 112:120 accumulator x0.333333",
        "accumulate [0 1 2 3 4 5 6] in-place x0.5 first", "sumsq 0:112 accumulator x2",
        "sgd 0:112 accumulator x2 clip", "sgd 112:120 accumulator x2",
    ],
    "sgd clip all k3 arena": [
        "accumulate [0 1 2 3 4 5 6] arena x1 first", "accumulate [0 1 2 3 4 5 6] arena x1",
        "accumulate [0 1 2 3 4 5 6] arena x1", "sumsq 0:112 accumulator x0.333333",
        "sgd 0:112 accumulator x0.333333 clip", "sgd 112:120 accumulator x0.333333",
        "accumulate [0 1 2 3 4 5 6] arena x0.5 first", "sumsq 0:112 accumulator x2",
        "sgd 0:112 accumulator x2 clip", "sgd 112:120 accumulator x2",
    ],
    "sgd clip partial k1 in-place": [
        "flatten [0 1 4 5 6] in-place x1", "sumsq 0:112 arena x1", "sgd 0:45 arena x1 clip",
        "sgd 88:112 arena x1 clip", "sgd 112:113 arena x1",
    ],
    "sgd clip partial k1 arena": [
        "sumsq 0:112 arena x1", "sgd 0:45 arena x1 clip", "sgd 88:112 arena x1 clip", "sgd 112:113 arena x1",
    ],
    "sgd clip partial k3 in-place": [
        "accumulate [0 1 4 5 6] in-place [2 3] NULL x1 first",
        "accumulate [0 1 4 5 6] in-place [2 3] NULL x1", "accumulate [0 1 4 5 6] in-place [2 3] NULL x1",
        "sumsq 0:112 accumulator x0.333333", "sgd 0:45 accumulator x0.333333 clip",
        "sgd 88:112 accumulator x0.333333 clip", "sgd 112:113 accumulator x0.333333",
        "accumulate [0 1 4 5 6] in-place [2 3] NULL x0.5 first", "sumsq 0:112 accumulator x2",
        "sgd 0:45 accumulator x2 clip", "sgd 88:112 accumulator x2 clip", "sgd 112:113 accumulator x2",
    ],
    "sgd clip partial k3 arena": [
        "accumulate [0 1 4 5 6] arena [2 3] NULL x1 first", "accumulate [0 1 4 5 6] arena [2 3] NULL x1",
        "accumulate [0 1 4 5 6] arena [2 3] NULL x1", "sumsq 0:112 accumulator x0.333333",
        "sgd 0:45 accumulator x0.333333 clip", "sgd 88:112 accumulator x0.333333 clip",
        "sgd 112:113 accumulator x0.333333", "accumulate [0 1 4 5 6] arena [2 3] NULL x0.5 first",
        "sumsq 0:112 accumulator x2", "sgd 0:45 accumulator x2 clip", "sgd 88:112 accumulator x2 clip",
        "sgd 112:113 accumulator x2",
    ],
    "adam noclip all k1 in-place": [
        "adam_mt [0 1 2 3 4 5 6] in-place x1",
    ],
    "adam noclip all k1 arena": [
        "adam 0:120 arena x1",
    ],
    "adam noclip all k3 in-place": [
        "accumulate [0 1 2 3 4 5 6] in-place x1 first", "accumulate [0 1 2 3 4 5 6] in-place x1",
        "accumulate [0 1 2 3 4 5 6] in-place x1", "adam 0:120 accumulator x0.333333",
        "accumulate [0 1 2 3 4 5 6] in-place x0.5 first", "adam 0:120 accumulator x2",
    ],
    "adam noclip all k3 arena": [
        "accumulate [0 1 2 3 4 5 6] arena x1 first", "accumulate [0 1 2 3 4 5 6] arena x1",
        "accumulate [0 1 2 3 4 5 6] arena x1", "adam 0:120 accumulator x0.333333",
        "accumulate [0 1 2 3 4 5 6] arena x0.5 first", "adam 0:120 accumulator x2",
    ],
    "adam noclip partial k1 in-place": [
        "flatten [0 1 4 5 6] in-place x1", "adam 0:45 arena x1", "adam 88:113 arena x1",
    ],
    "adam noclip partial k1 arena": [
        "adam 0:45 arena x1", "adam 88:113 arena x1",
    ],
    "adam noclip partial k3 in-place": [
        "accumulate [0 1 4 5 6] in-place [2 3] NULL x1 first",
        "accumulate [0 1 4 5 6] in-place [2 3] NULL x1", "accumulate [0 1 4 5 6] in-place [2 3] NULL x1",
        "adam 0:45 accumulator x0.333333", "adam 88:113 accumulator x0.333333",
        "accumulate [0 1 4 5 6] in-place [2 3] NULL x0.5 first", "adam 0:45 accumulator x2",
        "adam 88:113 accumulator x2",
    ],
    "adam noclip partial k3 arena": [
        "accumulate [0 1 4 5 6] arena [2 3] NULL x1 first", "accumulate [0 1 4 5 6] arena [2 3] NULL x1",
        "accumulate [0 1 4 5 6] arena [2 3] NULL x1", "adam 0:45 accumulator x0.333333",
        "adam 88:113 accumulator x0.333333", "accumulate [0 1 4 5 6] arena [2 3] NULL x0.5 first",
        "adam 0:45 accumulator x2", "adam 88:113 accumulator x2",
    ],
    "adam clip all k1 in-place": [
        "flatten [0 1 2 3 4 5 6] in-place x1", "sumsq 0:112 arena x1", "adam 0:112 arena x1 clip",
        "adam 112:120 arena x1",
    ],
    "adam clip all k1 arena": [
        "sumsq 0:112 arena x1", "adam 0:112 arena x1 clip", "adam 112:120 arena x1",
    ],
    "adam clip all k3 in-place": [
        "accumulate [0 1 2 3 4 5 6] in-place x1 first", "accumulate [0 1 2 3 4 5 6] in-place x1",
        "accumulate [0 1 2 3 4 5 6] in-place x1", "sumsq 0:112 accumulator x0.333333",
        "adam 0:112 accumulator x0.333333 clip", "adam 112:120 accumulator x0.333333",
        "accumulate [0 1 2 3 4 5 6] in-place x0.5 first", "sumsq 0:112 accumulator x2",
        "adam 0:112 accumulator x2 clip", "adam 112:120 accumulator x2",
    ],
    "adam clip all k3 arena": [
        "accumulate [0 1 2 3 4 5 6] arena x1 first", "accumulate [0 1 2 3 4 5 6] arena x1",
        "accumulate [0 1 2 3 4 5 6] arena x1", "sumsq 0:112 accumulator x0.333333",
        "adam 0:112 accumulator x0.333333 clip", "adam 112:120 accumulator x0.333333",
        "accumulate [0 1 2 3 4 5 6] arena x0.5 first", "sumsq 0:112 accumulator x2",
        "adam 0:112 accumulator x2 clip", "adam 112:120 accumulator x2",
    ],
    "adam clip partial k1 in-place": [
        "flatten [0 1 4 5 6] in-place x1", "sumsq 0:112 arena x1", "adam 0:45 arena x1 clip",
        "adam 88:112 arena x1 clip", "adam 112:113 arena x1",
    ],
    "adam clip partial k1 arena": [
        "sumsq 0:112 arena x1", "adam 0:45 arena x1 clip", "adam 88:112 arena x1 clip",
        "adam 112:113 arena x1",
    ],
    "adam clip partial k3 in-place": [
        "accumulate [0 1 4 5 6] in-place [2 3] NULL x1 first",
        "accumulate [0 1 4 5 6] in-place [2 3] NULL x1", "accumulate [0 1 4 5 6] in-place [2 3] NULL x1",
        "sumsq 0:112 accumulator x0.333333", "adam 0:45 accumulator x0.333333 clip",
        "adam 88:112 accumulator x0.333333 clip", "adam 112:113 accumulator x0.333333",
        "accumulate [0 1 4 5 6] in-place [2 3] NULL x0.5 first", "sumsq 0:112 accumulator x2",
        "adam 0:45 accumulator x2 clip", "adam 88:112 accumulator x2 clip", "adam 112:113 accumulator x2",
    ],
    "adam clip partial k3 arena": [
        "accumulate [0 1 4 5 6] arena [2 3] NULL x1 first", "accumulate [0 1 4 5 6] arena [2 3] NULL x1",
        "accumulate [0 1 4 5 6] arena [2 3] NULL x1", "sumsq 0:112 accumulator x0.333333",
        "adam 0:45 accumulator x0.333333 clip", "adam 88:112 accumulator x0.333333 clip",
        "adam 112:113 accumulator x0.333333", "accumulate [0 1 4 5 6] arena [2 3] NULL x0.5 first",
        "sumsq 0:112 accumulator x2", "adam 0:45 accumulator x2 clip", "adam 88:112 accumulator x2 clip",
        "adam 112:113 accumulator x2",
    ],
    "lars noclip all k1 in-place": [
        "lars_mt [0 1 2 3 4 5 6] in-place x1",
    ],
    "lars noclip all k1 arena": [
        "lars_mt [0 1 2 3 4 5 6] arena x1",
    ],
    "lars noclip all k3 in-place": [
        "accumulate [0 1 2 3 4 5 6] in-place x1 first", "accumulate [0 1 2 3 4 5 6] in-place x1",
        "accumulate [0 1 2 3 4 5 6] in-place x1", "lars_mt [0 1 2 3 4 5 6] accumulator x0.333333",
        "accumulate [0 1 2 3 4 5 6] in-place x0.5 first", "lars_mt [0 1 2 3 4 5 6] accumulator x2",
    ],
    "lars noclip all k3 arena": [
        "accumulate [0 1 2 3 4 5 6] arena x1 first", "accumulate [0 1 2 3 4 5 6] arena x1",
        "accumulate [0 1 2 3 4 5 6] arena x1", "lars_mt [0 1 2 3 4 5 6] accumulator x0.333333",
        "accumulate [0 1 2 3 4 5 6] arena x0.5 first", "lars_mt [0 1 2 3 4 5 6] accumulator x2",
    ],
    "lars noclip partial k1 in-place": [
        "flatten [0 1 4 5 6] in-place x1", "lars_mt [0 1 4 5 6] arena x1",
    ],
    "lars noclip partial k1 arena": [
        "lars_mt [0 1 4 5 6] arena x1",
    ],
    "lars noclip partial k3 in-place": [
        "accumulate [0 1 4 5 6] in-place [2 3] NULL x1 first",
        "accumulate [0 1 4 5 6] in-place [2 3] NULL x1", "accumulate [0 1 4 5 6] in-place [2 3] NULL x1",
        "lars_mt [0 1 4 5 6] accumulator x0.333333", "accumulate [0 1 4 5 6] in-place [2 3] NULL x0.5 first",
        "lars_mt [0 1 4 5 6] accumulator x2",
    ],
    "lars noclip partial k3 arena": [
        "accumulate [0 1 4 5 6] arena [2 3] NULL x1 first", "accumulate [0 1 4 5 6] arena [2 3] NULL x1",
        "accumulate [0 1 4 5 6] arena [2 3] NULL x1", "lars_mt [0 1 4 5 6] accumulator x0.333333",
        "accumulate [0 1 4 5 6] arena [2 3] NULL x0.5 first", "lars_mt [0 1 4 5 6] accumulator x2",
    ],
    "lars clip all k1 in-place": [
        "flatten [0 1 2 3 4 5 6] in-place x1", "sumsq 0:112 arena x1",
        "lars_mt [0 1 2 3 4 5 6] arena x1 clip",
    ],
    "lars clip all k1 arena": [
        "sumsq 0:112 arena x1", "lars_mt [0 1 2 3 4 5 6] arena x1 clip",
    ],
    "lars clip all k3 in-place": [
        "accumulate [0 1 2 3 4 5 6] in-place x1 first", "accumulate [0 1 2 3 4 5 6] in-place x1",
        "accumulate [0 1 2 3 4 5 6] in-place x1", "sumsq 0:112 accumulator x0.333333",
        "lars_mt [0 1 2 3 4 5 6] accumulator x0.333333 clip",
        "accumulate [0 1 2 3 4 5 6] in-place x0.5 first", "sumsq 0:112 accumulator x2",
        "lars_mt [0 1 2 3 4 5 6] accumulator x2 clip",
    ],
    "lars clip all k3 arena": [
        "accumulate [0 1 2 3 4 5 6] arena x1 first", "accumulate [0 1 2 3 4 5 6] arena x1",
        "accumulate [0 1 2 3 4 5 6] arena x1", "sumsq 0:112 accumulator x0.333333",
        "lars_mt [0 1 2 3 4 5 6] accumulator x0.333333 clip", "accumulate [0 1 2 3 4 5 6] arena x0.5 first",
        "sumsq 0:112 accumulator x2", "lars_mt [0 1 2 3 4 5 6] accumulator x2 clip",
    ],
    "lars clip partial k1 in-place": [
        "flatten [0 1 4 5 6] in-place x1", "sumsq 0:112 arena x1", "lars_mt [0 1 4 5 6] arena x1 clip",
    ],
    "lars clip partial k1 arena": [
        "sumsq 0:112 arena x1", "lars_mt [0 1 4 5 6] arena x1 clip",
    ],
    "lars clip partial k3 in-place": [
        "accumulate [0 1 4 5 6] in-place [2 3] NULL x1 first",
        "accumulate [0 1 4 5 6] in-place [2 3] NULL x1", "accumulate [0 1 4 5 6] in-place [2 3] NULL x1",
        "sumsq 0:112 accumulator x0.333333", "lars_mt [0 1 4 5 6] accumulator x0.333333 clip",
        "accumulate [0 1 4 5 6] in-place [2 3] NULL x0.5 first", "sumsq 0:112 accumulator x2",
        "lars_mt [0 1 4 5 6] accumulator x2 clip",
    ],
    "lars clip partial k3 arena": [
        "accumulate [0 1 4 5 6] arena [2 3] NULL x1 first", "accumulate [0 1 4 5 6] arena [2 3] NULL x1",
        "accumulate [0 1 4 5 6] arena [2 3] NULL x1", "sumsq 0:112 accumulator x0.333333",
        "lars_mt [0 1 4 5 6] accumulator x0.333333 clip",
        "accumulate [0 1 4 5 6] arena [2 3] NULL x0.5 first", "sumsq 0:112 accumulator x2",
        "lars_mt [0 1 4 5 6] accumulator x2 clip",
    ],
    "lamb noclip all k1 in-place": [
        "lamb_mt [0 1 2 3 4 5 6] in-place x1",
    ],
    "lamb noclip all k1 arena": [
        "lamb_mt [0 1 2 3 4 5 6] arena x1",
    ],
    "lamb noclip all k3 in-place": [
        "accumulate [0 1 2 3 4 5 6] in-place x1 first", "accumulate [0 1 2 3 4 5 6] in-place x1",
        "accumulate [0 1 2 3 4 5 6] in-place x1", "lamb_mt [0 1 2 3 4 5 6] accumulator x0.333333",
        "accumulate [0 1 2 3 4 5 6] in-place x0.5 first", "lamb_mt [0 1 2 3 4 5 6] accumulator x2",
    ],
    "lamb noclip all k3 arena": [
        "accumulate [0 1 2 3 4 5 6] arena x1 first", "accumulate [0 1 2 3 4 5 6] arena x1",
        "accumulate [0 1 2 3 4 5 6] arena x1", "lamb_mt [0 1 2 3 4 5 6] accumulator x0.333333",
        "accumulate [0 1 2 3 4 5 6] arena x0.5 first", "lamb_mt [0 1 2 3 4 5 6] accumulator x2",
    ],
    "lamb noclip partial k1 in-place": [
        "flatten [0 1 4 5 6] in-place x1", "lamb_mt [0 1 4 5 6] arena x1",
    ],
    "lamb noclip partial k1 arena": [
        "lamb_mt [0 1 4 5 6] arena x1",
    ],
    "lamb noclip partial k3 in-place": [
        "accumulate [0 1 4 5 6] in-place [2 3] NULL x1 first",
        "accumulate [0 1 4 5 6] in-place [2 3] NULL x1", "accumulate [0 1 4 5 6] in-place [2 3] NULL x1",
        "lamb_mt [0 1 4 5 6] accumulator x0.333333", "accumulate [0 1 4 5 6] in-place [2 3] NULL x0.5 first",
        "lamb_mt [0 1 4 5 6] accumulator x2",
    ],
    "lamb noclip partial k3 arena": [
        "accumulate [0 1 4 5 6] arena [2 3] NULL x1 first", "accumulate [0 1 4 5 6] arena [2 3] NULL x1",
        "accumulate [0 1 4 5 6] arena [2 3] NULL x1", "lamb_mt [0 1 4 5 6] accumulator x0.333333",
        "accumulate [0 1 4 5 6] arena [2 3] NULL x0.5 first", "lamb_mt [0 1 4 5 6] accumulator x2",
    ],
    "lamb clip all k1 in-place": [
        "flatten [0 1 2 3 4 5 6] in-place x1", "sumsq 0:112 arena x1",
        "lamb_mt [0 1 2 3 4 5 6] arena x1 clip",
    ],
    "lamb clip all k1 arena": [
        "sumsq 0:112 arena x1", "lamb_mt [0 1 2 3 4 5 6] arena x1 clip",
    ],
    "lamb clip all k3 in-place": [
        "accumulate [0 1 2 3 4 5 6] in-place x1 first", "accumulate [0 1 2 3 4 5 6] in-place x1",
        "accumulate [0 1 2 3 4 5 6] in-place x1", "sumsq 0:112 accumulator x0.333333",
        "lamb_mt [0 1 2 3 4 5 6] accumulator x0.333333 clip",
        "accumulate [0 1 2 3 4 5 6] in-place x0.5 first", "sumsq 0:112 accumulator x2",
        "lamb_mt [0 1 2 3 4 5 6] accumulator x2 clip",
    ],
    "lamb clip all k3 arena": [
        "accumulate [0 1 2 3 4 5 6] arena x1 first", "accumulate [0 1 2 3 4 5 6] arena x1",
        "accumulate [0 1 2 3 4 5 6] arena x1", "sumsq 0:112 accumulator x0.333333",
        "lamb_mt [0 1 2 3 4 5 6] accumulator x0.333333 clip", "accumulate [0 1 2 3 4 5 6] arena x0.5 first",
        "sumsq 0:112 accumulator x2", "lamb_mt [0 1 2 3 4 5 6] accumulator x2 clip",
    ],
    "lamb clip partial k1 in-place": [
        "flatten [0 1 4 5 6] in-place x1", "sumsq 0:112 arena x1", "lamb_mt [0 1 4 5 6] arena x1 clip",
    ],
    "lamb clip partial k1 arena": [
        "sumsq 0:112 arena x1", "lamb_mt [0 1 4 5 6] arena x1 clip",
    ],
    "lamb clip partial k3 in-place": [
        "accumulate [0 1 4 5 6] in-place [2 3] NULL x1 first",
        "accumulate [0 1 4 5 6] in-place [2 3] NULL x1", "accumulate [0 1 4 5 6] in-place [2 3] NULL x1",
        "sumsq 0:112 accumulator x0.333333", "lamb_mt [0 1 4 5 6] accumulator x0.333333 clip",
        "accumulate [0 1 4 5 6] in-place [2 3] NULL x0.5 first", "sumsq 0:112 accumulator x2",
        "lamb_mt [0 1 4 5 6] accumulator x2 clip",
    ],
    "lamb clip partial k3 arena": [
        "accumulate [0 1 4 5 6] arena [2 3] NULL x1 first", "accumulate [0 1 4 5 6] arena [2 3] NULL x1",
        "accumulate [0 1 4 5 6] arena [2 3] NULL x1", "sumsq 0:112 accumulator x0.333333",
        "lamb_mt [0 1 4 5 6] accumulator x0.333333 clip",
        "accumulate [0 1 4 5 6] arena [2 3] NULL x0.5 first", "sumsq 0:112 accumulator x2",
        "lamb_mt [0 1 4 5 6] accumulator x2 clip",
    ],
}
DEFERRED = {
    "sgd noclip partial k1 in-place": [
        "flatten [0 1 4 5 6] in-place x1", "sgd 0:45 arena x1", "sgd 88:113 arena x1", "sgd 0:120 arena x1",
    ],
    "sgd noclip partial k1 arena": [
        "sgd 0:45 arena x1", "sgd 88:113 arena x1", "sgd 0:120 arena x1",
    ],
    "sgd clip partial k1 in-place": [
        "flatten [0 1 4 5 6] in-place x1", "sumsq 0:112 arena x1", "sgd 0:45 arena x1 clip",
        "sgd 88:112 arena x1 clip", "sgd 112:113 arena x1", "sumsq 0:112 arena x1", "sgd 0:112 arena x1 clip",
        "sgd 112:120 arena x1",
    ],
    "sgd clip partial k1 arena": [
        "sumsq 0:112 arena x1", "sgd 0:45 arena x1 clip", "sgd 88:112 arena x1 clip", "sgd 112:113 arena x1",
        "sumsq 0:112 arena x1", "sgd 0:112 arena x1 clip", "sgd 112:120 arena x1",
    ],
    "adam noclip partial k1 in-place": [
        "flatten [0 1 4 5 6] in-place x1", "adam 0:45 arena x1", "adam 88:113 arena x1",
        "adam 0:120 arena x1",
    ],
    "adam noclip partial k1 arena": [
        "adam 0:45 arena x1", "adam 88:113 arena x1", "adam 0:120 arena x1",
    ],
    "adam clip partial k1 in-place": [
        "flatten [0 1 4 5 6] in-place x1", "sumsq 0:112 arena x1", "adam 0:45 arena x1 clip",
        "adam 88:112 arena x1 clip", "adam 112:113 arena x1", "sumsq 0:112 arena x1",
        "adam 0:112 arena x1 clip", "adam 112:120 arena x1",
    ],
    "adam clip partial k1 arena": [
        "sumsq 0:112 arena x1", "adam 0:45 arena x1 clip", "adam 88:112 arena x1 clip",
        "adam 112:113 arena x1", "sumsq 0:112 arena x1", "adam 0:112 arena x1 clip", "adam 112:120 arena x1",
    ],
    "lars noclip partial k1 in-place": [
        "flatten [0 1 4 5 6] in-place x1", "lars_mt [0 1 4 5 6] arena x1", "lars_mt [0 1 2 3 4 5 6] arena x1",
    ],
    "lars noclip partial k1 arena": [
        "lars_mt [0 1 4 5 6] arena x1", "lars_mt [0 1 2 3 4 5 6] arena x1",
    ],
    "lars clip all k1 in-place": [
        "flatten [0 1 2 3 4 5 6] in-place x1", "sumsq 0:112 arena x1",
        "lars_mt [0 1 2 3 4 5 6] in-place x1 clip",
    ],
    "lars clip partial k1 in-place": [
        "flatten [0 1 4 5 6] in-place x1", "sumsq 0:112 arena x1", "lars_mt [0 1 4 5 6] arena x1 clip",
        "sumsq 0:112 arena x1", "lars_mt [0 1 2 3 4 5 6] arena x1 clip",
    ],
    "lars clip partial k1 arena": [
        "sumsq 0:112 arena x1", "lars_mt [0 1 4 5 6] arena x1 clip", "sumsq 0:112 arena x1",
        "lars_mt [0 1 2 3 4 5 6] arena x1 clip",
    ],
    "lamb noclip partial k1 in-place": [
        "flatten [0 1 4 5 6] in-place x1", "lamb_mt [0 1 4 5 6] arena x1", "lamb_mt [0 1 2 3 4 5 6] arena x1",
    ],
    "lamb noclip partial k1 arena": [
        "lamb_mt [0 1 4 5 6] arena x1", "lamb_mt [0 1 2 3 4 5 6] arena x1",
    ],
    "lamb clip all k1 in-place": [
        "flatten [0 1 2 3 4 5 6] in-place x1", "sumsq 0:112 arena x1",
        "lamb_mt [0 1 2 3 4 5 6] in-place x1 clip",
    ],
    "lamb clip partial k1 in-place": [
        "flatten [0 1 4 5 6] in-place x1", "sumsq 0:112 arena x1", "lamb_mt [0 1 4 5 6] arena x1 clip",
        "sumsq 0:112 arena x1", "lamb_mt [0 1 2 3 4 5 6] arena x1 clip",
    ],
    "lamb clip partial k1 arena": [
        "sumsq 0:112 arena x1", "lamb_mt [0 1 4 5 6] arena x1 clip", "sumsq 0:112 arena x1",
        "lamb_mt [0 1 2 3 4 5 6] arena x1 clip",
    ],
}
EXPECTED_2RANKS = {
    "sgd noclip all k1 in-place": [
        "flatten [6] in-place x1", "all_reduce 112:120 arena", "sgd 112:120 arena x0.5",
        "flatten [4 5] in-place x1", "all_reduce 88:112 arena", "sgd 88:112 arena x0.5",
        "flatten [3] in-place x1", "all_reduce 80:88 arena", "sgd 80:88 arena x0.5",
        "flatten [2] in-place x1", "all_reduce 48:80 arena", "sgd 48:80 arena x0.5",
        "flatten [1] in-place x1", "all_reduce 40:48 arena", "sgd 40:48 arena x0.5",
        "flatten [0] in-place x1", "all_reduce 0:40 arena", "sgd 0:40 arena x0.5",
    ],
    "sgd noclip all k1 arena": [
        "all_reduce 112:120 arena", "sgd 112:120 arena x0.5", "all_reduce 88:112 arena",
        "sgd 88:112 arena x0.5", "all_reduce 80:88 arena", "sgd 80:88 arena x0.5", "all_reduce 48:80 arena",
        "sgd 48:80 arena x0.5", "all_reduce 40:48 arena", "sgd 40:48 arena x0.5", "all_reduce 0:40 arena",
        "sgd 0:40 arena x0.5",
    ],
    "sgd noclip all k3 in-place": [
        "accumulate [0 1 2 3 4 5 6] in-place x1 first", "accumulate [0 1 2 3 4 5 6] in-place x1",
        "accumulate [0 1 2 3 4 5 6] in-place x1", "all_reduce 112:120 accumulator",
        "all_reduce 88:112 accumulator", "all_reduce 80:88 accumulator", "all_reduce 48:80 accumulator",
        "all_reduce 40:48 accumulator", "all_reduce 0:40 accumulator", "sgd 0:120 accumulator x0.166667",
        "accumulate [0 1 2 3 4 5 6] in-place x0.5 first", "all_reduce 112:120 accumulator",
        "all_reduce 88:112 accumulator", "all_reduce 80:88 accumulator", "all_reduce 48:80 accumulator",
        "all_reduce 40:48 accumulator", "all_reduce 0:40 accumulator", "sgd 0:120 accumulator x1",
    ],
    "sgd noclip all k3 arena": [
        "accumulate [0 1 2 3 4 5 6] arena x1 first", "accumulate [0 1 2 3 4 5 6] arena x1",
        "accumulate [0 1 2 3 4 5 6] arena x1", "all_reduce 112:120 accumulator",
        "all_reduce 88:112 accumulator", "all_reduce 80:88 accumulator", "all_reduce 48:80 accumulator",
        "all_reduce 40:48 accumulator", "all_reduce 0:40 accumulator", "sgd 0:120 accumulator x0.166667",
        "accumulate [0 1 2 3 4 5 6] arena x0.5 first", "all_reduce 112:120 accumulator",
        "all_reduce 88:112 accumulator", "all_reduce 80:88 accumulator", "all_reduce 48:80 accumulator",
        "all_reduce 40:48 accumulator", "all_reduce 0:40 accumulator", "sgd 0:120 accumulator x1",
    ],
    "sgd clip all k1 in-place": [
        "flatten [6] in-place x1", "all_reduce 112:120 arena", "flatten [4 5] in-place x1",
        "all_reduce 88:112 arena", "flatten [3] in-place x1", "all_reduce 80:88 arena",
        "flatten [2] in-place x1", "all_reduce 48:80 arena", "flatten [1] in-place x1",
        "all_reduce 40:48 arena", "flatten [0] in-place x1", "all_reduce 0:40 arena",
        "sumsq 0:112 arena x0.5", "sgd 0:112 arena x0.5 clip", "sgd 112:120 arena x0.5",
    ],
    "sgd clip all k1 arena": [
        "all_reduce 112:120 arena", "all_reduce 88:112 arena", "all_reduce 80:88 arena",
        "all_reduce 48:80 arena", "all_reduce 40:48 arena", "all_reduce 0:40 arena", "sumsq 0:112 arena x0.5",
        "sgd 0:112 arena x0.5 clip", "sgd 112:120 arena x0.5",
    ],
    "sgd clip all k3 in-place": [
        "accumulate [0 1 2 3 4 5 6] in-place x1 first", "accumulate [0 1 2 3 4 5 6] in-place x1",
        "accumulate [0 1 2 3 4 5 6] in-place x1", "all_reduce 112:120 accumulator",
        "all_reduce 88:112 accumulator", "all_reduce 80:88 accumulator", "all_reduce 48:80 accumulator",
        "all_reduce 40:48 accumulator", "all_reduce 0:40 accumulator", "sumsq 0:112 accumulator x0.166667",
        "sgd 0:112 accumulator x0.166667 clip", "sgd 112:120 accumulator x0.166667",
        "accumulate [0 1 2 3 4 5 6] in-place x0.5 first", "all_reduce 112:120 accumulator",
        "all_reduce 88:112 accumulator", "all_reduce 80:88 accumulator", "all_reduce 48:80 accumulator",
        "all_reduce 40:48 accumulator", "all_reduce 0:40 accumulator", "sumsq 0:112 accumulator x1",
        "sgd 0:112 accumulator x1 clip", "sgd 112:120 accumulator x1",
    ],
    "sgd clip all k3 arena": [
        "accumulate [0 1 2 3 4 5 6] arena x1 first", "accumulate [0 1 2 3 4 5 6] arena x1",
        "accumulate [0 1 2 3 4 5 6] arena x1", "all_reduce 112:120 accumulator",
        "all_reduce 88:112 accumulator", "all_reduce 80:88 accumulator", "all_reduce 48:80 accumulator",
        "all_reduce 40:48 accumulator", "all_reduce 0:40 accumulator", "sumsq 0:112 accumulator x0.166667",
        "sgd 0:112 accumulator x0.166667 clip", "sgd 112:120 accumulator x0.166667",
        "accumulate [0 1 2 3 4 5 6] arena x0.5 first", "all_reduce 112:120 accumulator",
        "all_reduce 88:112 accumulator", "all_reduce 80:88 accumulator", "all_reduce 48:80 accumulator",
        "all_reduce 40:48 accumulator", "all_reduce 0:40 accumulator", "sumsq 0:112 accumulator x1",
        "sgd 0:112 accumulator x1 clip", "sgd 112:120 accumulator x1",
    ],
    "adam noclip all k1 in-place": [
        "flatten [6] in-place x1", "all_reduce 112:120 arena", "adam 112:120 arena x0.5",
        "flatten [4 5] in-place x1", "all_reduce 88:112 arena", "adam 88:112 arena x0.5",
        "flatten [3] in-place x1", "all_reduce 80:88 arena", "adam 80:88 arena x0.5",
        "flatten [2] in-place x1", "all_reduce 48:80 arena", "adam 48:80 arena x0.5",
        "flatten [1] in-place x1", "all_reduce 40:48 arena", "adam 40:48 arena x0.5",
        "flatten [0] in-place x1", "all_reduce 0:40 arena", "adam 0:40 arena x0.5",
    ],
    "adam noclip all k1 arena": [
        "all_reduce 112:120 arena", "adam 112:120 arena x0.5", "all_reduce 88:112 arena",
        "adam 88:112 arena x0.5", "all_reduce 80:88 arena", "adam 80:88 arena x0.5", "all_reduce 48:80 arena",
        "adam 48:80 arena x0.5", "all_reduce 40:48 arena", "adam 40:48 arena x0.5", "all_reduce 0:40 arena",
        "adam 0:40 arena x0.5",
    ],
    "adam noclip all k3 in-place": [
        "accumulate [0 1 2 3 4 5 6] in-place x1 first", "accumulate [0 1 2 3 4 5 6] in-place x1",
        "accumulate [0 1 2 3 4 5 6] in-place x1", "all_reduce 112:120 accumulator",
        "all_reduce 88:112 accumulator", "all_reduce 80:88 accumulator", "all_reduce 48:80 accumulator",
        "all_reduce 40:48 accumulator", "all_reduce 0:40 accumulator", "adam 0:120 accumulator x0.166667",
        "accumulate [0 1 2 3 4 5 6] in-place x0.5 first", "all_reduce 112:120 accumulator",
        "all_reduce 88:112 accumulator", "all_reduce 80:88 accumulator", "all_reduce 48:80 accumulator",
        "all_reduce 40:48 accumulator", "all_reduce 0:40 accumulator", "adam 0:120 accumulator x1",
    ],
    "adam noclip all k3 arena": [
        "accumulate [0 1 2 3 4 5 6] arena x1 first", "accumulate [0 1 2 3 4 5 6] arena x1",
        "accumulate [0 1 2 3 4 5 6] arena x1", "all_reduce 112:120 accumulator",
        "all_reduce 88:112 accumulator", "all_reduce 80:88 accumulator", "all_reduce 48:80 accumulator",
        "all_reduce 40:48 accumulator", "all_reduce 0:40 accumulator", "adam 0:120 accumulator x0.166667",
        "accumulate [0 1 2 3 4 5 6] arena x0.5 first", "all_reduce 112:120 accumulator",
        "all_reduce 88:112 accumulator", "all_reduce 80:88 accumulator", "all_reduce 48:80 accumulator",
        "all_reduce 40:48 accumulator", "all_reduce 0:40 accumulator", "adam 0:120 accumulator x1",
    ],
    "adam clip all k1 in-place": [
        "flatten [6] in-place x1", "all_reduce 112:120 arena", "flatten [4 5] in-place x1",
        "all_reduce 88:112 arena", "flatten [3] in-place x1", "all_reduce 80:88 arena",
        "flatten [2] in-place x1", "all_reduce 48:80 arena", "flatten [1] in-place x1",
        "all_reduce 40:48 arena", "flatten [0] in-place x1", "all_reduce 0:40 arena",
        "sumsq 0:112 arena x0.5", "adam 0:112 arena x0.5 clip", "adam 112:120 arena x0.5",
    ],
    "adam clip all k1 arena": [
        "all_reduce 112:120 arena", "all_reduce 88:112 arena", "all_reduce 80:88 arena",
        "all_reduce 48:80 arena", "all_reduce 40:48 arena", "all_reduce 0:40 arena", "sumsq 0:112 arena x0.5",
        "adam 0:112 arena x0.5 clip", "adam 112:120 arena x0.5",
    ],
    "adam clip all k3 in-place": [
        "accumulate [0 1 2 3 4 5 6] in-place x1 first", "accumulate [0 1 2 3 4 5 6] in-place x1",
        "accumulate [0 1 2 3 4 5 6] in-place x1", "all_reduce 112:120 accumulator",
        "all_reduce 88:112 accumulator", "all_reduce 80:88 accumulator", "all_reduce 48:80 accumulator",
        "all_reduce 40:48 accumulator", "all_reduce 0:40 accumulator", "sumsq 0:112 accumulator x0.166667",
        "adam 0:112 accumulator x0.166667 clip", "adam 112:120 accumulator x0.166667",
        "accumulate [0 1 2 3 4 5 6] in-place x0.5 first", "all_reduce 112:120 accumulator",
        "all_reduce 88:112 accumulator", "all_reduce 80:88 accumulator", "all_reduce 48:80 accumulator",
        "all_reduce 40:48 accumulator", "all_reduce 0:40 accumulator", "sumsq 0:112 accumulator x1",
        "adam 0:112 accumulator x1 clip", "adam 112:120 accumulator x1",
    ],
    "adam clip all k3 arena": [
        "accumulate [0 1 2 3 4 5 6] arena x1 first", "accumulate [0 1 2 3 4 5 6] arena x1",
        "accumulate [0 1 2 3 4 5 6] arena x1", "all_reduce 112:120 accumulator",
        "all_reduce 88:112 accumulator", "all_reduce 80:88 accumulator", "all_reduce 48:80 accumulator",
        "all_reduce 40:48 accumulator", "all_reduce 0:40 accumulator", "sumsq 0:112 accumulator x0.166667",
        "adam 0:112 accumulator x0.166667 clip", "adam 112:120 accumulator x0.166667",
        "accumulate [0 1 2 3 4 5 6] arena x0.5 first", "all_reduce 112:120 accumulator",
        "all_reduce 88:112 accumulator", "all_reduce 80:88 accumulator", "all_reduce 48:80 accumulator",
        "all_reduce 40:48 accumulator", "all_reduce 0:40 accumulator", "sumsq 0:112 accumulator x1",
        "adam 0:112 accumulator x1 clip", "adam 112:120 accumulator x1",
    ],
    "lars noclip all k1 in-place": [
        "flatten [6] in-place x1", "all_reduce 112:120 arena", "flatten [4 5] in-place x1",
        "all_reduce 88:112 arena", "flatten [3] in-place x1", "all_reduce 80:88 arena",
        "flatten [2] in-place x1", "all_reduce 48:80 arena", "flatten [1] in-place x1",
        "all_reduce 40:48 arena", "flatten [0] in-place x1", "all_reduce 0:40 arena",
        "lars_mt [0 1 2 3 4 5 6] arena x0.5",
    ],
    "lars noclip all k1 arena": [
        "all_reduce 112:120 arena", "all_reduce 88:112 arena", "all_reduce 80:88 arena",
        "all_reduce 48:80 arena", "all_reduce 40:48 arena", "all_reduce 0:40 arena",
        "lars_mt [0 1 2 3 4 5 6] arena x0.5",
    ],
    "lars noclip all k3 in-place": [
        "accumulate [0 1 2 3 4 5 6] in-place x1 first", "accumulate [0 1 2 3 4 5 6] in-place x1",
        "accumulate [0 1 2 3 4 5 6] in-place x1", "all_reduce 112:120 accumulator",
        "all_reduce 88:112 accumulator", "all_reduce 80:88 accumulator", "all_reduce 48:80 accumulator",
        "all_reduce 40:48 accumulator", "all_reduce 0:40 accumulator",
        "lars_mt [0 1 2 3 4 5 6] accumulator x0.166667", "accumulate [0 1 2 3 4 5 6] in-place x0.5 first",
        "all_reduce 112:120 accumulator", "all_reduce 88:112 accumulator", "all_reduce 80:88 accumulator",
        "all_reduce 48:80 accumulator", "all_reduce 40:48 accumulator", "all_reduce 0:40 accumulator",
        "lars_mt [0 1 2 3 4 5 6] accumulator x1",
    ],
    "lars noclip all k3 arena": [
        "accumulate [0 1 2 3 4 5 6] arena x1 first", "accumulate [0 1 2 3 4 5 6] arena x1",
        "accumulate [0 1 2 3 4 5 6] arena x1", "all_reduce 112:120 accumulator",
        "all_reduce 88:112 accumulator", "all_reduce 80:88 accumulator", "all_reduce 48:80 accumulator",
        "all_reduce 40:48 accumulator", "all_reduce 0:40 accumulator",
        "lars_mt [0 1 2 3 4 5 6] accumulator x0.166667", "accumulate [0 1 2 3 4 5 6] arena x0.5 first",
        "all_reduce 112:120 accumulator", "all_reduce 88:112 accumulator", "all_reduce 80:88 accumulator",
        "all_reduce 48:80 accumulator", "all_reduce 40:48 accumulator", "all_reduce 0:40 accumulator",
        "lars_mt [0 1 2 3 4 5 6] accumulator x1",
    ],
    "lars clip all k1 in-place": [
        "flatten [6] in-place x1", "all_reduce 112:120 arena", "flatten [4 5] in-place x1",
        "all_reduce 88:112 arena", "flatten [3] in-place x1", "all_reduce 80:88 arena",
        "flatten [2] in-place x1", "all_reduce 48:80 arena", "flatten [1] in-place x1",
        "all_reduce 40:48 arena", "flatten [0] in-place x1", "all_reduce 0:40 arena",
        "sumsq 0:112 arena x0.5", "lars_mt [0 1 2 3 4 5 6] arena x0.5 clip",
    ],
    "lars clip all k1 arena": [
        "all_reduce 112:120 arena", "all_reduce 88:112 arena", "all_reduce 80:88 arena",
        "all_reduce 48:80 arena", "all_reduce 40:48 arena", "all_reduce 0:40 arena", "sumsq 0:112 arena x0.5",
        "lars_mt [0 1 2 3 4 5 6] arena x0.5 clip",
    ],
    "lars clip all k3 in-place": [
        "accumulate [0 1 2 3 4 5 6] in-place x1 first", "accumulate [0 1 2 3 4 5 6] in-place x1",
        "accumulate [0 1 2 3 4 5 6] in-place x1", "all_reduce 112:120 accumulator",
        "all_reduce 88:112 accumulator", "all_reduce 80:88 accumulator", "all_reduce 48:80 accumulator",
        "all_reduce 40:48 accumulator", "all_reduce 0:40 accumulator", "sumsq 0:112 accumulator x0.166667",
        "lars_mt [0 1 2 3 4 5 6] accumulator x0.166667 clip",
        "accumulate [0 1 2 3 4 5 6] in-place x0.5 first", "all_reduce 112:120 accumulator",
        "all_reduce 88:112 accumulator", "all_reduce 80:88 accumulator", "all_reduce 48:80 accumulator",
        "all_reduce 40:48 accumulator", "all_reduce 0:40 accumulator", "sumsq 0:112 accumulator x1",
        "lars_mt [0 1 2 3 4 5 6] accumulator x1 clip",
    ],
    "lars clip all k3 arena": [
        "accumulate [0 1 2 3 4 5 6] arena x1 first", "accumulate [0 1 2 3 4 5 6] arena x1",
        "accumulate [0 1 2 3 4 5 6] arena x1", "all_reduce 112:120 accumulator",
        "all_reduce 88:112 accumulator", "all_reduce 80:88 accumulator", "all_reduce 48:80 accumulator",
        "all_reduce 40:48 accumulator", "all_reduce 0:40 accumulator", "sumsq 0:112 accumulator x0.166667",
        "lars_mt [0 1 2 3 4 5 6] accumulator x0.166667 clip", "accumulate [0 1 2 3 4 5 6] arena x0.5 first",
        "all_reduce 112:120 accumulator", "all_reduce 88:112 accumulator", "all_reduce 80:88 accumulator",
        "all_reduce 48:80 accumulator", "all_reduce 40:48 accumulator", "all_reduce 0:40 accumulator",
        "sumsq 0:112 accumulator x1", "lars_mt [0 1 2 3 4 5 6] accumulator x1 clip",
    ],
    "lamb noclip all k1 in-place": [
        "flatten [6] in-place x1", "all_reduce 112:120 arena", "flatten [4 5] in-place x1",
        "all_reduce 88:112 arena", "flatten [3] in-place x1", "all_reduce 80:88 arena",
        "flatten [2] in-place x1", "all_reduce 48:80 arena", "flatten [1] in-place x1",
        "all_reduce 40:48 arena", "flatten [0] in-place x1", "all_reduce 0:40 arena",
        "lamb_mt [0 1 2 3 4 5 6] arena x0.5",
    ],
    "lamb noclip all k1 arena": [
        "all_reduce 112:120 arena", "all_reduce 88:112 arena", "all_reduce 80:88 arena",
        "all_reduce 48:80 arena", "all_reduce 40:48 arena", "all_reduce 0:40 arena",
        "lamb_mt [0 1 2 3 4 5 6] arena x0.5",
    ],
    "lamb noclip all k3 in-place": [
        "accumulate [0 1 2 3 4 5 6] in-place x1 first", "accumulate [0 1 2 3 4 5 6] in-place x1",
        "accumulate [0 1 2 3 4 5 6] in-place x1", "all_reduce 112:120 accumulator",
        "all_reduce 88:112 accumulator", "all_reduce 80:88 accumulator", "all_reduce 48:80 accumulator",
        "all_reduce 40:48 accumulator", "all_reduce 0:40 accumulator",
        "lamb_mt [0 1 2 3 4 5 6] accumulator x0.166667", "accumulate [0 1 2 3 4 5 6] in-place x0.5 first",
        "all_reduce 112:120 accumulator", "all_reduce 88:112 accumulator", "all_reduce 80:88 accumulator",
        "all_reduce 48:80 accumulator", "all_reduce 40:48 accumulator", "all_reduce 0:40 accumulator",
        "lamb_mt [0 1 2 3 4 5 6] accumulator x1",
    ],
    "lamb noclip all k3 arena": [
        "accumulate [0 1 2 3 4 5 6] arena x1 first", "accumulate [0 1 2 3 4 5 6] arena x1",
        "accumulate [0 1 2 3 4 5 6] arena x1", "all_reduce 112:120 accumulator",
        "all_reduce 88:112 accumulator", "all_reduce 80:88 accumulator", "all_reduce 48:80 accumulator",
        "all_reduce 40:48 accumulator", "all_reduce 0:40 accumulator",
        "lamb_mt [0 1 2 3 4 5 6] accumulator x0.166667", "accumulate [0 1 2 3 4 5 6] arena x0.5 first",
        "all_reduce 112:120 accumulator", "all_reduce 88:112 accumulator", "all_reduce 80:88 accumulator",
        "all_reduce 48:80 accumulator", "all_reduce 40:48 accumulator", "all_reduce 0:40 accumulator",
        "lamb_mt [0 1 2 3 4 5 6] accumulator x1",
    ],
    "lamb clip all k1 in-place": [
        "flatten [6] in-place x1", "all_reduce 112:120 arena", "flatten [4 5] in-place x1",
        "all_reduce 88:112 arena", "flatten [3] in-place x1", "all_reduce 80:88 arena",
        "flatten [2] in-place x1", "all_reduce 48:80 arena", "flatten [1] in-place x1",
        "all_reduce 40:48 arena", "flatten [0] in-place x1", "all_reduce 0:40 arena",
        "sumsq 0:112 arena x0.5", "lamb_mt [0 1 2 3 4 5 6] arena x0.5 clip",
    ],
    "lamb clip all k1 arena": [
        "all_reduce 112:120 arena", "all_reduce 88:112 arena", "all_reduce 80:88 arena",
        "all_reduce 48:80 arena", "all_reduce 40:48 arena", "all_reduce 0:40 arena", "sumsq 0:112 arena x0.5",
        "lamb_mt [0 1 2 3 4 5 6] arena x0.5 clip",
    ],
    "lamb clip all k3 in-place": [
        "accumulate [0 1 2 3 4 5 6] in-place x1 first", "accumulate [0 1 2 3 4 5 6] in-place x1",
        "accumulate [0 1 2 3 4 5 6] in-place x1", "all_reduce 112:120 accumulator",
        "all_reduce 88:112 accumulator", "all_reduce 80:88 accumulator", "all_reduce 48:80 accumulator",
        "all_reduce 40:48 accumulator", "all_reduce 0:40 accumulator", "sumsq 0:112 accumulator x0.166667",
        "lamb_mt [0 1 2 3 4 5 6] accumulator x0.166667 clip",
        "accumulate [0 1 2 3 4 5 6] in-place x0.5 first", "all_reduce 112:120 accumulator",
        "all_reduce 88:112 accumulator", "all_reduce 80:88 accumulator", "all_reduce 48:80 accumulator",
        "all_reduce 40:48 accumulator", "all_reduce 0:40 accumulator", "sumsq 0:112 accumulator x1",
        "lamb_mt [0 1 2 3 4 5 6] accumulator x1 clip",
    ],
    "lamb clip all k3 arena": [
        "accumulate [0 1 2 3 4 5 6] arena x1 first", "accumulate [0 1 2 3 4 5 6] arena x1",
        "accumulate [0 1 2 3 4 5 6] arena x1", "all_reduce 112:120 accumulator",
        "all_reduce 88:112 accumulator", "all_reduce 80:88 accumulator", "all_reduce 48:80 accumulator",
        "all_reduce 40:48 accumulator", "all_reduce 0:40 accumulator", "sumsq 0:112 accumulator x0.166667",
        "lamb_mt [0 1 2 3 4 5 6] accumulator x0.166667 clip", "accumulate [0 1 2 3 4 5 6] arena x0.5 first",
        "all_reduce 112:120 accumulator", "all_reduce 88:112 accumulator", "all_reduce 80:88 accumulator",
        "all_reduce 48:80 accumulator", "all_reduce 40:48 accumulator", "all_reduce 0:40 accumulator",
        "sumsq 0:112 accumulator x1", "lamb_mt [0 1 2 3 4 5 6] accumulator x1 clip",
    ],
}


@pytest.fixture()
def double(monkeypatch):
    d = RecordingDouble()
    monkeypatch.setattr(fused_optim, "KERNELS", d)
    monkeypatch.setattr(grad_sync, "KERNELS", d)
    monkeypatch.setattr(multi_tensor, "grad_usable_in_place", _in_place)
    return d


@pytest.mark.parametrize("in_place", [True, False], ids=["in-place", "arena"])
@pytest.mark.parametrize("k", [1, 3])
@pytest.mark.parametrize("skip", [False, True], ids=["all", "partial"])
@pytest.mark.parametrize("clip", [0.0, CLIP], ids=["noclip", "clip"])
@pytest.mark.parametrize("opt", list(OPTS))
def test_one_rank_launch_sequence(double, opt, clip, skip, k, in_place):
    key = _key(opt, clip, skip, k, in_place)
    xs = torch.randn(N_ROWS, 7, generator=torch.Generator().manual_seed(11))
    want = EXPECTED[key] * (N_MB if k == 1 else 1)
    log, params = _run(double, opt, clip, k, in_place, False, skip, xs)
    assert log == want
    ref = _torch_reference(opt, clip, k, skip, xs)
    for a, b in zip(params, ref):
        np.testing.assert_allclose(a.numpy(), b.numpy(), rtol=1e-4, atol=1e-6)
    log, deferred = _run(double, opt, clip, k, in_place, True, skip, xs)
    if key in DEFERRED:
        assert log == DEFERRED[key] * N_MB
    else:
        assert log == want
        for a, b in zip(deferred, params):
            assert torch.equal(a, b)


# ---- two ranks over gloo -------------------------------------------------------------------------

_CONFIGS_2RANKS = list(itertools.product(OPTS, (0.0, CLIP), (1, 3), (True, False)))


def _rank_main(rank, world, port, out_dir):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    d = RecordingDouble()
    fused_optim.KERNELS = grad_sync.KERNELS = d
    multi_tensor.grad_usable_in_place = _in_place
    all_reduce = dist.all_reduce

    def logged_all_reduce(t, *args, **kw):
        d.log.append("all_reduce %s" % d._range(t, t.numel()))
        return all_reduce(t, *args, **kw)

    dist.all_reduce = logged_all_reduce
    xs = torch.randn(N_ROWS * world, 7, generator=torch.Generator().manual_seed(12))
    out = {}
    for opt, clip, k, in_place in _CONFIGS_2RANKS:
        out[_key(opt, clip, False, k, in_place)] = [_run(d, opt, clip, k, in_place, defer, False, xs, rank, world)
                                                    for defer in (False, True)]
    torch.save(out, os.path.join(out_dir, f"r{rank}.pt"))
    dist.destroy_process_group()


def test_two_rank_launch_sequences(tmp_path):
    world = 2
    port = 35500 + (os.getpid() % 2000)
    mp.spawn(_rank_main, args=(world, port, str(tmp_path)), nprocs=world, join=True)
    r0, r1 = torch.load(tmp_path / "r0.pt"), torch.load(tmp_path / "r1.pt")
    assert sorted(r0) == sorted(EXPECTED_2RANKS)
    for key, want in EXPECTED_2RANKS.items():
        want = want * (N_MB if " k1 " in key else 1)
        for (log0, p0), (log1, p1) in zip(r0[key], r1[key]):
            assert log0 == log1 == want, key
            for a, b in zip(p0, p1):
                assert torch.equal(a, b), key                  # replicas stay identical
        for a, b in zip(r0[key][0][1], r0[key][1][1]):
            assert torch.equal(a, b), key                      # finish_step == the hand-over
