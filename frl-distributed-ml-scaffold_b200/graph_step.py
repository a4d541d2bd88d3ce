"""CUDA-graph replay of the training step.

The reference's minibatch is ~60 kernel launches issued from Python (forward, T loss modules,
autograd, DDP hooks, optimizer); on an H100 the GPU finishes them in about the time one CPU
core needs to issue them, and with per-bucket collectives the host becomes the
bottleneck.  Shapes are static from step to step, so after a few eager steps the whole
sequence — input cast, model forward, fused criterion, backward with gradients landing in the
arena, per-bucket NCCL all-reduce and fused update on the side stream — is captured once into a
CUDA graph and replayed with a single launch.

What stays outside the graph (cheap, and needs per-step values):
  * filling the static input buffers (the cast kernel writes them directly in BF16 mode);
  * per-step scalars (lr, Adam bias corrections): uploaded to the optimizer's ``dyn`` block,
    which the captured update kernels read from device memory; with gradient accumulation the
    K10 launch's (weight, first) likewise, and the group-closing update runs after the replay;
  * on one GPU the tail update (and the clip-norm kernel) so it can be timed and tuned alone;
  * the 4*(1+T)-byte copy of the loss vector into the pinned loss log.
"""
from typing import Dict, List, Optional, Sequence, Tuple

import gc
import logging

import torch

from . import _native

logger = logging.getLogger(__name__)

#: kernels of this library executed through graph replays (the C-side launch counter only sees
#: direct launches): each replay adds the number of frl_* launches recorded at capture time
REPLAYED_LAUNCHES = 0


def _signature(data: Sequence[torch.Tensor], target) -> Tuple:
    sig = [(tuple(t.shape), t.dtype) for t in data]
    for head in target:
        sig.append(tuple((tuple(t.shape), t.dtype) for t in head))
    return tuple(sig)


class GraphedTrainStep:
    WARMUP_STEPS = 2      # eager steps of a given signature before it is captured (cuDNN/cuBLAS
                          # pick their algorithms on the first call of every shape)

    def __init__(self, worker) -> None:
        self.worker = worker
        self._seen: Dict[Tuple, int] = {}
        self._graphs: Dict[Tuple, "_Captured"] = {}
        self.enabled = True

    def ready_for(self, data, target) -> Optional["_Captured"]:
        """Captured graph for this batch signature, capturing it when it has warmed up."""
        sig = _signature(data, target)
        cap = self._graphs.get(sig)
        if cap is not None:
            return cap
        n = self._seen.get(sig, 0)
        self._seen[sig] = n + 1
        if n < self.WARMUP_STEPS or self.worker.optimizer._steps < 1:
            return None
        if not self.enabled:
            return None
        try:
            cap = _Captured(self.worker, data, target)
        except Exception as e:                     # noqa: BLE001
            # not capturable (host sync in the Problem's forward, a stale autograd graph bound
            # to another stream, ...): stay on the eager path for the rest of the run
            logger.warning("CUDA-graph capture of the training step failed (%s); "
                           "continuing with eager launches", str(e).splitlines()[0],
                           exc_info=bool(__import__("os").environ.get("FRL_B200_DEBUG")))
            self.enabled = False
            w = self.worker
            w.pipeline._step_open = False
            w.optimizer._in_step = False
            w.optimizer.disable_dynamic_scalars()
            torch.cuda.synchronize()
            return None
        self._graphs[sig] = cap
        return cap


class _Captured:
    def __init__(self, worker, data, target) -> None:
        self.worker = worker
        w = worker
        bf16 = w.precision.bf16_storage
        self.static_in: List[torch.Tensor] = []
        self.cast_in: List[bool] = []
        for t in data:
            cast = bf16 and t.dtype == torch.float32
            self.static_in.append(torch.empty_like(t, dtype=torch.bfloat16 if cast else t.dtype))
            self.cast_in.append(cast)
        self.static_tgt = [tuple(torch.empty_like(t) for t in head) for head in target]
        self._fill(data, target)

        w.optimizer.enable_dynamic_scalars()
        w.criterion.set_step_sink(None, None)
        gc.collect()                  # free autograd graphs of earlier (eager) steps
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        launches_before = _native.launch_count()
        with torch.cuda.graph(self.graph, capture_error_mode="thread_local"):
            if w.buffers is not None:
                w.buffers.sync()
            output = w.model(self.static_in)
            total, sub = w.criterion(output, self.static_tgt)
            w.pipeline.begin_step()
            total.backward()
            w.pipeline.finish_step(defer_tail=True)
        # gradients autograd allocated inside the capture (conv / norm layers) and the segment
        # tables that name them now belong to this graph: the replayed backward writes to exactly
        # those addresses, the tail update / the captured flatten launches read them there
        self.grad_refs, self.tables = w.pipeline.detach_grad_refs()
        self.ready = w.pipeline.last_ready     # slots the captured K10 launch accumulates (k > 1)
        self.dw_updated = w.pipeline.dw_updated    # slots the captured K12 launches update
        # capture executed nothing on the device, but begin_step() counted a step: undo it, the
        # replay performs the step for real (finish_step(defer_tail=True) left the optimizer's
        # step counter to run_tail())
        w.pipeline.step_id -= 1
        self.frl_kernels = _native.launch_count() - launches_before
        self.output = [o.detach() for o in output]
        self.names = list(sub.keys())
        self._total, self._sub = total.detach(), {k: v.detach() for k, v in sub.items()}
        # the fused criterion returns views of one [1+T] vector: copy that in one go
        base = getattr(total, "_base", None)
        self._loss_vec = base.detach() if (base is not None and base.dim() == 1
                                           and base.numel() == 1 + len(self.names)
                                           and base.dtype == torch.float32) else None

    def _fill(self, data, target) -> None:
        for dst, src, cast in zip(self.static_in, data, self.cast_in):
            if cast:
                _native.cast_scale(src if _native.is_nhwc(src) else src.contiguous(), dst, 1.0)
            else:
                dst.copy_(src, non_blocking=True)
        for dhead, shead in zip(self.static_tgt, target):
            for d, s in zip(dhead, shead):
                d.copy_(s, non_blocking=True)

    def run(self, data, target, sink_row: Optional[torch.Tensor]):
        w = self.worker
        self._fill(data, target)
        w.optimizer.refresh_dynamic_scalars()
        self.graph.replay()
        global REPLAYED_LAUNCHES
        REPLAYED_LAUNCHES += self.frl_kernels
        w.pipeline.step_id += 1
        # tail update (1 GPU / clipping) + step counter; with accumulation the group's update
        w.pipeline.run_tail(self.grad_refs, self.tables, self.ready, self.dw_updated)
        if sink_row is not None:
            row = self._loss_vec
            if row is None:
                row = torch.stack([self._total.float()] + [self._sub[k].float() for k in self.names])
            sink_row.copy_(row, non_blocking=True)
            w.criterion._sink_written = True
        return self.output, self._total, self._sub
