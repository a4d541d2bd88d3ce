"""Weight EMA: an exponential moving average of the model's weights, kept on the device.

Stands where a user of the reference would wrap the model in
``torch.optim.swa_utils.AveragedModel(model, multi_avg_fn=get_ema_multi_avg_fn(decay),
use_buffers=True)`` and call ``update_parameters(model)`` after every ``optimizer.step()``
(reference solver_worker.py:592).  Same arithmetic, different shape:

* the averaged parameters are ONE fp32 vector over the model range ``[0, arena.model_end)`` of the
  flat arena, updated from the fp32 master weights by one K11 launch (``frl_weight_ema``) per
  optimizer update; criterion parameters are not averaged;
* floating buffers (BatchNorm running statistics) get the same lerp through
  ``torch._foreach_lerp_``, non-floating ones (``num_batches_tracked``) are copied;
* evaluation and export swap the averaged values into the arena (and the bf16 shadow) in place
  instead of keeping a second module.
"""
from contextlib import contextmanager
from typing import Any, Dict, List, Tuple

import torch
import torch.nn as nn

from . import _native
from .arena import ParamArena

KERNELS = _native     # swapped by CPU tests of the host logic

# the top-level key under which the EMA travels from a rank to the parent inside the optimizer-state
# bytes; the parent takes it out before it writes the checkpoint's "optimizer"
EMA_STATE_KEY = "weight_ema"
# elements exchanged per step of a swap: the transient buffer is at most 16 MiB
SWAP_CHUNK = 4 << 20


class WeightEMA:
    """EMA of the model range of ``arena``'s master weights and of ``module``'s buffers.

    ``update()`` after every optimizer update: the first copies (``ema = w``), every later one is
    ``ema = lerp(ema, w, 1 - decay)`` in fp32, torch's lerp formula, with ``1 - decay`` formed in
    double and rounded to fp32 once.  ``swapped()`` puts the averaged values where the module reads
    its weights for the duration of a block."""

    def __init__(self, arena: ParamArena, module: nn.Module, decay: float) -> None:
        if not 0.0 <= decay < 1.0:
            raise ValueError("EMA decay %r outside [0, 1)" % (decay,))
        self.arena = arena
        self.module = module
        self.decay = float(decay)
        self.weight = 1.0 - self.decay             # double; the kernel rounds it to fp32
        self.n = arena.model_end
        self.ema = arena.master[:self.n].clone()   # what a run with 0 updates evaluates with
        self.buffers: List[Tuple[str, torch.Tensor, torch.Tensor]] = [
            (name, b, b.detach().clone()) for name, b in module.named_buffers()]
        self.updates = 0
        self._swapped = False

    @property
    def nbytes(self) -> int:
        return self.ema.numel() * 4 + sum(e.numel() * e.element_size() for _, _, e in self.buffers)

    @torch.no_grad()
    def update(self) -> None:
        """One EMA step on the current stream, behind the optimizer update that precedes it."""
        if self._swapped:
            raise RuntimeError("WeightEMA.update() inside swapped()")
        first = self.updates == 0
        # the first update is K11 at weight 1, which returns the master weights (torch's lerp at
        # weight 1 is its end point): the same one launch per update, whatever its position
        KERNELS.weight_ema(self.ema, self.arena.master[:self.n], 1.0 if first else self.weight)
        floats = [(e, b) for _, b, e in self.buffers if b.is_floating_point() and not first]
        if floats:
            torch._foreach_lerp_([e for e, _ in floats], [b.detach() for _, b in floats], self.weight)
        for _, b, e in self.buffers:
            if first or not b.is_floating_point():
                e.copy_(b.detach())
        self.updates += 1

    @torch.no_grad()
    def _exchange(self) -> None:
        """Swap the averaged and the live values: model range of the master in chunks through one
        transient buffer of at most ``SWAP_CHUNK`` elements, then the bf16 shadow from the master,
        then the buffers.  Pure copies: swapping twice restores every bit."""
        master = self.arena.master
        tmp = torch.empty(min(self.n, SWAP_CHUNK), dtype=torch.float32, device=master.device)
        for lo in range(0, self.n, SWAP_CHUNK):
            hi = min(lo + SWAP_CHUNK, self.n)
            t = tmp[:hi - lo]
            t.copy_(master[lo:hi])
            master[lo:hi].copy_(self.ema[lo:hi])
            self.ema[lo:hi].copy_(t)
        if self.arena.lp is not None:
            # the shadow is the round-to-nearest-even cast of the master, as every update writes it
            self.arena.lp[:self.n].copy_(master[:self.n])
        for _, b, e in self.buffers:
            t = b.detach().clone()
            b.detach().copy_(e)
            e.copy_(t)

    @contextmanager
    def swapped(self):
        """The module computes with the averaged weights and buffers inside the block; the live
        ones are back, bit for bit, when it is left (also when it raises)."""
        if self._swapped:
            raise RuntimeError("WeightEMA.swapped() is not reentrant")
        self._exchange()
        self._swapped = True
        try:
            yield self
        finally:
            self._exchange()
            self._swapped = False

    # -- checkpoints ---------------------------------------------------------------------------
    def state_dict(self) -> Dict[str, Any]:
        """``{"decay", "updates", "state_dict"}``: ``state_dict`` is the module's fp32 CPU
        ``state_dict()`` with the averaged values in it, keyed like the main checkpoint's."""
        buffers = {name for name, _, _ in self.buffers}
        with self.swapped(), self.arena.exported(cpu=True, module=self.module):
            # parameters are private CPU copies inside exported(); buffers are the live tensors
            sd = {k: v.detach().to("cpu", copy=k in buffers) for k, v in self.module.state_dict().items()}
        return {"decay": self.decay, "updates": self.updates, "state_dict": sd}

    @torch.no_grad()
    def load_state_dict(self, blob: Dict[str, Any]) -> None:
        """Averaged values and update count from what ``state_dict()`` wrote."""
        sd = blob["state_dict"]
        names = {id(p): name for name, p in self.module.named_parameters()}
        for s in self.arena.slots:
            if s.is_model:
                self.ema[s.offset:s.end].copy_(sd[names[id(s.param)]].reshape(-1))
        for name, _, e in self.buffers:
            e.copy_(sd[name])
        self.updates = int(blob["updates"])
