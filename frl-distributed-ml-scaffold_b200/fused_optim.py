"""Arena optimizers: ``torch.optim``-compatible front, one fused kernel launch per bucket behind.

``create_fused_optimizer`` is the H100 counterpart of the reference's ``_create_optimizer``
(reference solver.py:162-188): same three algorithms, same hyper-parameter mapping
(``OptimOpts.momentum`` feeds SGD *and* RMSprop, ``epsilon``/``amsgrad`` feed Adam, weight decay
is L2-coupled and applies to every parameter).  ``state_dict()`` / ``load_state_dict()`` speak
torch's per-parameter format so the reference's ``.checkpoint.pth`` files stay interchangeable.
``FusedLars`` / ``FusedLamb`` (an extension, ``types.LayerAdaptation``) keep SGD's / Adam's state
format and update whole tensors through the K2-lw kernels.  ``FusedAdam8bit`` (an extension,
``types.OptimizerState``) keeps Adam's moments as 8-bit block-wise codes (K2-q8) and speaks
``torch.optim.Adam``'s format in its state dict.  ``FusedAdafactor`` (an extension, chosen with
``Solver.solve(..., adafactor=True)``) is ``torch.optim.Adafactor``'s rule and state format (K2-af).
``FusedMuon`` (an extension, ``Solver.solve(..., muon=True)``) is ``torch.optim.Muon`` (K14) for the
model's 2-D weights and this module's Adam (K2-mt) for every other parameter.  ``adamw=True`` (an
extension, ``Solver.solve(..., adamw=True)``) turns the Adam rule of ``FusedAdam``, ``FusedAdam8bit``
and ``FusedMuon``'s Adam group into ``torch.optim.AdamW``'s decoupled weight decay (``frl_adamw*``).
On an arena with bf16 master weights (an extension, ``types.MasterWeights.BF16``) ``FusedSGD``,
``FusedAdam``, ``FusedRMSprop`` and ``FusedLion`` update the model range through the stochastic-rounding kernels
(``frl_*_sr``, ``frl_*_mt_sr``) and keep ``sr_seed`` / ``sr_updates`` in their param group.
``FusedLion`` (an extension, ``Solver.solve(..., lion=True)``) is Lion's sign-momentum rule with
decoupled weight decay on SGD's state shape (``frl_lion*``); it too has SR forms.

Known limitation: the step count (Adam's bias corrections) is ONE number for the whole arena.
``torch.optim`` keeps one per parameter and does not advance it for a parameter whose gradient
is ``None`` in a step; here a parameter that misses gradients for some steps (world size 1 only:
with several ranks a missing gradient is DDP's error, as in the reference) keeps being corrected
with the global count, ``state_dict()`` writes that count for every parameter and
``load_state_dict()`` takes the maximum over the loaded entries.  Models whose parameters all
receive a gradient every step — every configuration of BASELINE.json — are unaffected.
"""
from typing import Any, Dict, List, Optional, Tuple

import numpy as np
import torch

from . import _native
from .arena import ParamArena
from .types import LayerAdaptation, MasterWeights, OptAlgorithm, OptimizerState, OptimOpts, Precision

# Kernel entry points; tests exercising host logic on CPU swap this for an oracle-backed double.
KERNELS = _native

# default key of the stochastic-rounding draws (param group ``sr_seed``, a uint64)
SR_SEED = 0x5EED_B16F_0000_0001


class _ShiftedBase:
    """``data_ptr()`` of an fp32 vector whose element 0 has arena index ``base``, minus ``base``
    elements: the arena-base pointer the segment-table kernels add arena offsets to.  Only listed
    segments are touched, and with bf16 master weights those (criterion parameters) lie at or
    above ``base``."""

    def __init__(self, vec: torch.Tensor, base: int) -> None:
        self._ptr = vec.data_ptr() - base * vec.element_size()

    def data_ptr(self) -> int:
        return self._ptr


class FusedArenaOptimizer(torch.optim.Optimizer):
    """Base: owns the fp32 state vectors (same layout as the arena) and the step counter."""

    STATE_NAMES: Tuple[str, ...] = ()

    @property
    def needs_whole_tensors(self) -> bool:
        """True if an update needs every gradient of a tensor at once (per-tensor norms), or if the
        optimizer has several param groups (one grouped segment-table update, K2-mt grouped): the
        pipeline then updates once after backward, never per bucket or per shard."""
        return self.grouped

    def __init__(self, arena: ParamArena, defaults: Dict[str, Any],
                 param_groups: Optional[List[Dict[str, Any]]] = None) -> None:
        self.arena = arena
        params = arena.all_params
        if not params:
            raise ValueError("optimizer got an empty parameter list")
        super().__init__(params if param_groups is None else param_groups, defaults)
        # state-dict position of each parameter: consecutive group by group (torch's numbering)
        self._pos: Dict[int, int] = {}
        self._group_of: Dict[int, int] = {}
        for gi, g in enumerate(self.param_groups):
            for p in g["params"]:
                self._group_of[id(p)] = gi
                self._pos[id(p)] = len(self._pos)
        if param_groups is not None and set(self._pos) != {id(p) for p in params}:
            raise ValueError("the param groups must hold exactly the arena's parameters")
        self.grouped = len(self.param_groups) > 1
        self._vec: Dict[str, torch.Tensor] = {}
        self._steps = 0                # completed optimizer steps
        self._in_step = False
        # device-resident per-step scalars (lr, Adam bias corrections): set when the step is
        # replayed from a CUDA graph, where by-value kernel arguments are frozen at capture
        self._dyn: Optional[torch.Tensor] = None
        self._dyn_last: Optional[Tuple[float, ...]] = None
        self._grad_src: Optional[torch.Tensor] = None      # apply_range(grad_src=...)
        # fused NVLS step (world > 1): set by the pipeline; each rank then updates only its
        # 1/world shard of every bucket (master + state), the weights arrive by multicast
        self.nvls = None
        # bf16 master weights: the model range is updated with stochastic rounding
        self.sr = bool(getattr(arena, "bf16_master", False))
        if self.sr:
            self.param_groups[0].setdefault("sr_seed", SR_SEED)
            self.param_groups[0]["sr_updates"] = 0
        if self.grouped:
            # one dyn row per group, read by every grouped launch (eager or replayed), so there are no
            # by-value lr / wd arguments a captured graph would freeze
            self._dyn = torch.zeros(len(self.param_groups), KERNELS.GROUP_DYN_COLS, dtype=torch.float32,
                                    device=arena.device)

    @property
    def sr_seed(self) -> int:
        return int(self.hyper["sr_seed"])

    # -- device-resident scalars -----------------------------------------------------------------
    def _dyn_values(self) -> Tuple[float, ...]:
        """Scalars of the NEXT step (``_steps + 1``) in the layout the kernel's ``dyn`` expects."""
        return self._dyn_row(self.hyper)

    def _dyn_row(self, h: Dict[str, Any]) -> Tuple[float, ...]:
        """``_dyn_values`` for the lr / weight decay of param group ``h``."""
        return (float(h["lr"]),)

    def _group_rows(self) -> np.ndarray:
        """The grouped ``dyn`` table of the next step: per group, columns 0-2 its ``_dyn_row``, column
        3 the update count (uint32 bits), column 4 its weight decay (the L2-coupled rules' wd)."""
        rows = np.zeros((len(self.param_groups), KERNELS.GROUP_DYN_COLS), dtype=np.float32)
        for gi, h in enumerate(self.param_groups):
            vals = self._dyn_row(h)
            rows[gi, :len(vals)] = vals
            rows[gi, 4] = float(h["weight_decay"])
        rows.view(np.uint32)[:, 3] = self._steps + 1
        return rows

    def enable_dynamic_scalars(self) -> None:
        if self._dyn is None:
            self._dyn = torch.zeros(4, dtype=torch.float32, device=self.arena.device)
            self._dyn_last = None
        self.refresh_dynamic_scalars()

    def disable_dynamic_scalars(self) -> None:
        """Back to by-value scalars (a failed CUDA-graph capture continues with eager launches).  With
        several param groups the rows stay: every grouped launch and K12 read them, eager or not, and
        the segment tables point at them; the next step uploads them afresh."""
        if self.grouped:
            self._dyn_last = None
        else:
            self._dyn = None

    _DYN_RING = 16        # pinned staging rows; the host never runs this many steps ahead

    def refresh_dynamic_scalars(self) -> None:
        """Upload the scalars if they changed: 16 bytes from a ring of pinned rows, so the copy is
        truly asynchronous (a pageable source makes the driver synchronise the stream first,
        which serialises the host's work for step k+1 with the device's work for step k; Adam's
        bias corrections change every step)."""
        if self._dyn is None:
            return
        if self.grouped:
            self._refresh_group_rows()
            return
        vals = self._dyn_values()
        if self.sr:        # dyn[3]: the update count of the stochastic rounding, as uint32 bits
            if len(vals) > 3:
                raise RuntimeError("%s: no dyn slot left for the update count" % type(self).__name__)
            vals = vals + (0.0,) * (3 - len(vals)) + (self._steps + 1,)
        if vals != self._dyn_last:
            if self._dyn.is_cuda:
                if getattr(self, "_dyn_host", None) is None:
                    self._dyn_host = torch.zeros(self._DYN_RING, 4, dtype=torch.float32, pin_memory=True)
                    self._dyn_slot = 0
                row = self._dyn_host[self._dyn_slot % self._DYN_RING]
                self._dyn_slot += 1
                for i, v in enumerate(vals):
                    row[i] = v
                if self.sr:
                    row.view(torch.int32)[3] = vals[3]
                self._dyn.copy_(row, non_blocking=True)
            else:
                host = torch.tensor(list(vals) + [0.0] * (4 - len(vals)), dtype=torch.float32)
                if self.sr:
                    host.view(torch.int32)[3] = vals[3]
                self._dyn.copy_(host)
            self._dyn_last = vals

    def _refresh_group_rows(self) -> None:
        rows = self._group_rows()
        if self._dyn_last is not None and np.array_equal(rows.view(np.uint32), self._dyn_last):
            return
        if self._dyn.is_cuda:
            if getattr(self, "_dyn_host", None) is None:
                self._dyn_host = torch.zeros((self._DYN_RING,) + rows.shape, dtype=torch.float32, pin_memory=True)
                self._dyn_slot = 0
            row = self._dyn_host[self._dyn_slot % self._DYN_RING]
            self._dyn_slot += 1
            row.copy_(torch.from_numpy(rows))
            self._dyn.copy_(row, non_blocking=True)
        else:
            self._dyn.copy_(torch.from_numpy(rows))
        self._dyn_last = rows.view(np.uint32).copy()

    def _slot_hyper(self, slot) -> Tuple[Dict[str, Any], Optional[torch.Tensor]]:
        """The param group of ``slot`` and the ``dyn`` its single-slot launches read (K12): its
        group's row with several groups, which columns 0-3 make a valid ``dyn`` of the rule."""
        if not self.grouped:
            return self.hyper, self._dyn
        gi = self._group_of[id(slot.param)]
        return self.param_groups[gi], self._dyn[gi]

    def _seg_groups(self, table):
        """The group arrays of ``table`` (``_native.SegGroups``), built on first use and kept on the
        table: each slot's group, FRL_LW_CLIPPED on model slots, and the shared ``dyn`` rows."""
        groups = getattr(table, "param_groups", None)
        if groups is None:
            groups = table.param_groups = KERNELS.SegGroups(
                [self._group_of[id(s.param)] for s in table.slots],
                [KERNELS.LW_CLIPPED if s.is_model else 0 for s in table.slots], self._dyn)
        return groups

    # -- state vectors ---------------------------------------------------------------------------
    def _state(self, name: str) -> torch.Tensor:
        v = self._vec.get(name)
        if v is None:
            v = self._vec[name] = self.arena.new_state()
        return v

    @property
    def hyper(self) -> Dict[str, Any]:
        return self.param_groups[0]

    # -- stepping --------------------------------------------------------------------------------
    def begin_step(self) -> None:
        """Open step ``_steps + 1``; per-bucket ``apply_range`` calls share its number."""
        self._in_step = True
        # an EAGER step after a graph was captured (ragged last batch, a second batch signature):
        # the kernels still read the device-resident scalars, so they must be this step's.  Never
        # inside a capture: the copy would be frozen into the graph and undo the per-replay upload.
        if self._dyn is not None and not (self._dyn.is_cuda and torch.cuda.is_current_stream_capturing()):
            self.refresh_dynamic_scalars()

    def end_step(self) -> None:
        self._steps += 1
        self._in_step = False

    def apply_range(self, lo: int, hi: int, *, grad_scale: float = 1.0,
                    clip_coef_dev: Optional[torch.Tensor] = None,
                    grad_src: Optional[torch.Tensor] = None) -> None:
        """Update arena elements ``[lo, hi)``.  ``clip_coef_dev`` (a device scalar written by
        the norm kernel) multiplies model-parameter gradients only — the reference clips
        ``model.parameters()`` and leaves criterion parameters alone
        (reference solver_worker.py:588-591).  ``grad_src``: an arena-shaped gradient vector read
        instead of ``arena.grad`` (the fp32 gradient accumulator).  With several param groups: the
        whole slots inside ``[lo, hi)`` through the grouped segment-table update."""
        if hi <= lo:
            return
        if self.grouped:
            if grad_src is not None:
                raise ValueError("a grouped update reads its gradients through a segment table, not grad_src")
            _WholeTensorMixin.apply_range(self, lo, hi, grad_scale=grad_scale, clip_coef_dev=clip_coef_dev)
            return
        self._grad_src = grad_src
        try:
            split = self.arena.model_end
            if (clip_coef_dev is not None or self.sr) and lo < split < hi:
                self._launch(lo, split, grad_scale, clip_coef_dev)
                self._launch(split, hi, grad_scale, None)
            else:
                self._launch(lo, hi, grad_scale, clip_coef_dev if lo < split else None)
        finally:
            self._grad_src = None

    def _launch(self, lo: int, hi: int, grad_scale: float, coef) -> None:
        raise NotImplementedError

    def apply_table(self, table, *, grad_scale: float = 1.0,
                    clip_coef_dev: Optional[torch.Tensor] = None) -> None:
        """Update every arena slot listed in ``table`` (a ``multi_tensor.GradSegTable`` whose device
        copy is current), reading each gradient where the table says it lies (K2-mt).  With several
        param groups: the grouped forms (K2-mt grouped, K2-mt-sr grouped), each slot with its group's
        lr / weight decay; ``clip_coef_dev`` then multiplies the gradients of model parameters only."""
        if self.grouped:
            self._apply_grouped(table, grad_scale, clip_coef_dev)
            return
        if clip_coef_dev is not None:
            raise ValueError("K2-mt takes no clip coefficient: clipped updates go through apply_range")
        if not table.n_segs:
            return
        if not self.sr:
            self._launch_mt(table, grad_scale)
            return
        model, crit = self._sr_split(table)
        for (sub, idx), launch in ((model, self._launch_mt_sr), (crit, self._launch_mt)):
            if sub is not None:
                _gather_segs(table, sub, idx)
                launch(sub, grad_scale)

    def _launch_mt(self, table, grad_scale: float) -> None:
        raise NotImplementedError

    def _launch_mt_sr(self, table, grad_scale: float) -> None:
        raise NotImplementedError

    def _apply_grouped(self, table, grad_scale: float, coef) -> None:
        if not table.n_segs:
            return
        if not self.sr:
            self._launch_mt_grouped(table, self._seg_groups(table), grad_scale, coef)
            return
        model, crit = self._sr_split(table)
        for (sub, idx), launch in ((model, self._launch_mt_grouped_sr), (crit, self._launch_mt_grouped)):
            if sub is not None:
                _gather_segs(table, sub, idx)
                launch(sub, self._seg_groups(sub), grad_scale, coef)

    def _launch_mt_grouped(self, table, groups, grad_scale: float, coef) -> None:
        raise NotImplementedError

    def _launch_mt_grouped_sr(self, table, groups, grad_scale: float, coef) -> None:
        raise NotImplementedError

    def _sr_split(self, table):
        """Bf16 master weights: the sub-tables of ``table``'s model slots (K2-mt-sr) and criterion
        slots (K2-mt on their fp32 master), with the rows of ``table`` they take; kept on the table."""
        split = getattr(table, "sr_split", None)
        if split is None:
            from .multi_tensor import GradSegTable
            dev = self.arena.device
            split = []
            for keep in (lambda s: s.is_model, lambda s: not s.is_model):
                part = [(i, s) for i, s in enumerate(table.slots) if keep(s)]
                rows = torch.tensor([i for i, _ in part], dtype=torch.int64)
                split.append((GradSegTable([s for _, s in part], dev), (rows, rows.to(dev))) if part else (None, None))
            split = table.sr_split = tuple(split)
        return split

    def _master_base(self):
        """What the segment-table kernels take as the fp32 master's arena base pointer."""
        a = self.arena
        return a.master if a.master_base == 0 else _ShiftedBase(a.master, a.master_base)

    def _lp_mt(self):
        """The bf16 shadow the fp32 segment-table kernels write: none with bf16 master weights (their
        segments are then criterion parameters, which read the fp32 master)."""
        return None if self.sr else self.arena.lp

    # -- fused all-reduce + update + broadcast (K7) ------------------------------------------------
    def apply_range_nvls(self, lo: int, hi: int, *, grad_scale: float) -> None:
        if hi > lo:
            split = bool(self.nvls.flags & KERNELS.NVLS_EXTERNAL_SYNC)
            if split:
                KERNELS.nvls_barrier(self.nvls, 0)     # every rank's bucket gradients are written
            self._launch_nvls(lo, hi, grad_scale)
            if split:
                KERNELS.nvls_barrier(self.nvls, 1)     # every replica has every shard

    def _launch_nvls(self, lo: int, hi: int, grad_scale: float) -> None:
        raise NotImplementedError

    def _nvls_ptrs(self, lo: int):
        k = self.nvls
        return k.mc_grad + lo * k.grad_esz, k.mc_out + lo * k.out_esz

    def shard_of(self, lo: int, hi: int) -> Tuple[int, int]:
        """Element range of bucket ``[lo, hi)`` this rank owns under the fused NVLS step (same
        formula as csrc/nvls.cu)."""
        k = self.nvls
        n = hi - lo
        per = ((n + k.world - 1) // k.world + 7) // 8 * 8
        a = min(lo + k.rank * per, hi)
        return a, min(a + per, hi)

    @torch.no_grad()
    def step(self, closure=None, *, grad_scale: float = 1.0,
             clip_coef_dev: Optional[torch.Tensor] = None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        self.begin_step()
        self.apply_range(0, self.arena.numel, grad_scale=grad_scale, clip_coef_dev=clip_coef_dev)
        self.end_step()
        return loss

    def zero_grad(self, set_to_none: bool = True) -> None:
        # Gradients are overwritten (first touch is a store, not an accumulate), so there is
        # nothing to clear in the arena; dropping stray .grad tensors keeps autograd stealing.
        for p in self.arena.all_params:
            p.grad = None

    # -- views used by the launchers -------------------------------------------------------------
    def _slices(self, lo: int, hi: int):
        """(weights, gradient, bf16 shadow) of ``[lo, hi)``; with bf16 master weights and ``lo`` in the
        model range (``_use_sr``) the weights are the bf16 vector and there is no shadow."""
        a = self.arena
        g = a.grad if self._grad_src is None else self._grad_src
        if self._use_sr(lo):
            return a.lp[lo:hi], g[lo:hi], None
        lp = a.lp[lo:hi] if (a.lp is not None and lo < a.model_end) else None
        return a.master[lo - a.master_base:hi - a.master_base], g[lo:hi], lp

    def _use_sr(self, lo: int) -> bool:
        """Does a launch starting at ``lo`` (never straddling ``model_end``) take the SR kernels?"""
        return self.sr and lo < self.arena.model_end

    # -- torch-format (de)serialisation ----------------------------------------------------------
    def _per_param_extra(self) -> Dict[str, Any]:
        return {}

    def state_dict(self) -> Dict[str, Any]:
        state: Dict[int, Dict[str, Any]] = {}
        if self._steps > 0:
            for s in sorted(self.arena.slots, key=lambda s: self._pos[id(s.param)]):     # torch's key order
                entry = dict(self._per_param_extra())
                for torch_name, vec_name in self.STATE_NAMES:
                    if vec_name in self._vec:
                        entry[torch_name] = ParamArena.slot_view(self._vec[vec_name], s).clone(
                            memory_format=torch.contiguous_format)
                state[self._pos[id(s.param)]] = entry
        if self.sr:
            self.hyper["sr_updates"] = self._steps
        groups, first = [], 0
        for g in self.param_groups:
            packed = {k: v for k, v in g.items() if k != "params"}
            packed["params"] = list(range(first, first + len(g["params"])))
            first += len(g["params"])
            groups.append(packed)
        return {"state": state, "param_groups": groups}

    def load_state_dict(self, state_dict: Dict[str, Any]) -> None:
        groups = state_dict["param_groups"]
        mine = [len(g["params"]) for g in self.param_groups]
        theirs = [len(g["params"]) for g in groups]
        if mine != theirs:
            raise ValueError("loaded state dict has a different number of parameters/groups: %d param groups of %s "
                             "params; this optimizer has %d of %s" % (len(theirs), theirs, len(mine), mine))
        for mine_g, theirs_g in zip(self.param_groups, groups):
            for k, v in theirs_g.items():
                if k != "params":
                    mine_g[k] = v
        by_index = {self._pos[id(s.param)]: s for s in self.arena.slots}
        steps = 0
        for idx, entry in state_dict["state"].items():
            s = by_index.get(int(idx))
            if s is None:
                continue
            for torch_name, vec_name in self.STATE_NAMES:
                if torch_name in entry and entry[torch_name] is not None:
                    ParamArena.slot_view(self._state(vec_name), s).copy_(entry[torch_name])
            if "step" in entry:
                steps = max(steps, int(float(entry["step"])))
            elif entry:
                steps = max(steps, 1)
        self._steps = steps
        self._load_sr_keys(groups[0])

    def _load_sr_keys(self, group: Dict[str, Any]) -> None:
        """Bf16 master weights: the update count comes from ``sr_updates`` where the dict has it (a
        bf16-master checkpoint), so the stochastic rounding continues with the draws it left off at.
        An fp32-master optimizer drops the two keys again (its state dict stays torch's)."""
        h = self.hyper
        if self.sr:
            if "sr_updates" in group:
                self._steps = int(group["sr_updates"])
            h["sr_seed"] = int(group.get("sr_seed", h.get("sr_seed", SR_SEED)))
        else:
            h.pop("sr_seed", None)
            h.pop("sr_updates", None)


class FusedSGD(FusedArenaOptimizer):
    STATE_NAMES = (("momentum_buffer", "momentum_buffer"),)

    def __init__(self, arena, lr, momentum=0.0, dampening=0.0, weight_decay=0.0, param_groups=None):
        super().__init__(arena, dict(lr=lr, momentum=momentum, dampening=dampening,
                                     weight_decay=weight_decay, nesterov=False, maximize=False,
                                     foreach=None, differentiable=False, fused=None), param_groups)

    def _launch(self, lo, hi, grad_scale, coef):
        h = self.hyper
        p, g, lp = self._slices(lo, hi)
        mu = float(h["momentum"])
        buf = self._state("momentum_buffer")[lo:hi] if mu != 0.0 else None
        if self._use_sr(lo):
            KERNELS.sgd_momentum_sr(p, g, buf, hi - lo, arena_off=lo, seed=self.sr_seed, t=self._steps + 1,
                                    lr=float(h["lr"]), mu=mu, dampening=float(h["dampening"]),
                                    wd=float(h["weight_decay"]), grad_scale=grad_scale, grad_scale_dev=coef,
                                    first_step=(self._steps == 0), dyn=self._dyn)
            return
        KERNELS.sgd_momentum(p, g, buf, lp, hi - lo, lr=float(h["lr"]), mu=mu,
                             dampening=float(h["dampening"]), wd=float(h["weight_decay"]),
                             grad_scale=grad_scale, grad_scale_dev=coef,
                             first_step=(self._steps == 0), dyn=self._dyn)

    def update_in_dw_gemm(self, slot, dz, x, gw, *, grad_scale: float = 1.0) -> None:
        """K12: the weight gradient gw = dz^T x of ``slot`` and, in the same kernel, this step's
        update of the slot from exactly that bf16 gradient (what ``_launch`` over the slot does); with
        several param groups, the slot's group's lr / weight decay and ``dyn`` row."""
        h, dyn = self._slot_hyper(slot)
        a = self.arena
        mu = float(h["momentum"])
        buf = self._state("momentum_buffer")[slot.offset:slot.end] if mu != 0.0 else None
        if self._use_sr(slot.offset):
            KERNELS.dw_gemm_sgd_sr(dz, x, gw, a.lp[slot.offset:slot.end], buf, arena_off=slot.offset,
                                   seed=self.sr_seed, t=self._steps + 1, lr=float(h["lr"]), mu=mu,
                                   dampening=float(h["dampening"]), wd=float(h["weight_decay"]),
                                   grad_scale=grad_scale, first_step=(self._steps == 0), dyn=dyn)
            return
        KERNELS.dw_gemm_sgd(dz, x, gw, a.master[slot.offset:slot.end], buf, a.lp[slot.offset:slot.end],
                            lr=float(h["lr"]), mu=mu, dampening=float(h["dampening"]),
                            wd=float(h["weight_decay"]), grad_scale=grad_scale,
                            first_step=(self._steps == 0), dyn=dyn)

    def _launch_mt(self, table, grad_scale):
        h = self.hyper
        mu = float(h["momentum"])
        KERNELS.sgd_momentum_mt(self._master_base(), self._state("momentum_buffer") if mu != 0.0 else None,
                                self._lp_mt(), table, lr=float(h["lr"]), mu=mu,
                                dampening=float(h["dampening"]), wd=float(h["weight_decay"]),
                                grad_scale=grad_scale, first_step=(self._steps == 0), dyn=self._dyn)

    def _launch_mt_sr(self, table, grad_scale):
        h = self.hyper
        mu = float(h["momentum"])
        KERNELS.sgd_momentum_mt_sr(self.arena.lp, self._state("momentum_buffer") if mu != 0.0 else None, table,
                                   seed=self.sr_seed, t=self._steps + 1, lr=float(h["lr"]), mu=mu,
                                   dampening=float(h["dampening"]), wd=float(h["weight_decay"]),
                                   grad_scale=grad_scale, first_step=(self._steps == 0), dyn=self._dyn)

    def _launch_mt_grouped(self, table, groups, grad_scale, coef):
        h = self.hyper
        mu = float(h["momentum"])
        KERNELS.sgd_momentum_mt_grouped(self._master_base(), self._state("momentum_buffer") if mu != 0.0 else None,
                                        self._lp_mt(), table, groups, mu=mu, dampening=float(h["dampening"]),
                                        grad_scale=grad_scale, grad_scale_dev=coef, first_step=(self._steps == 0))

    def _launch_mt_grouped_sr(self, table, groups, grad_scale, coef):
        h = self.hyper
        mu = float(h["momentum"])
        KERNELS.sgd_momentum_mt_grouped_sr(self.arena.lp, self._state("momentum_buffer") if mu != 0.0 else None,
                                           table, groups, seed=self.sr_seed, mu=mu, dampening=float(h["dampening"]),
                                           grad_scale=grad_scale, grad_scale_dev=coef,
                                           first_step=(self._steps == 0))

    def _launch_nvls(self, lo, hi, grad_scale):
        h = self.hyper
        mu = float(h["momentum"])
        mc_g, mc_out = self._nvls_ptrs(lo)
        buf = self._state("momentum_buffer")[lo:hi] if mu != 0.0 else None
        KERNELS.nvls_sgd(self.arena.master[lo:hi], buf, mc_g, mc_out, hi - lo, self.nvls,
                         lr=float(h["lr"]), mu=mu, dampening=float(h["dampening"]),
                         wd=float(h["weight_decay"]), grad_scale=grad_scale,
                         first_step=(self._steps == 0),
                         g_dtype=KERNELS.dtype_code(self.arena.grad.dtype), dyn=self._dyn)


class FusedAdam(FusedArenaOptimizer):
    """Adam with torch's L2-coupled weight decay, or with ``adamw=True`` torch 2.11's
    ``Adam(decoupled_weight_decay=True)``, which ``torch.optim.AdamW`` is: each step first scales
    the parameter by fp32(1 - lr * weight_decay), then takes Adam's step with no decay in the
    gradient (the ``frl_adamw*`` kernels).  The param group's ``decoupled_weight_decay`` says which,
    so ``state_dict()`` is ``torch.optim.Adam``'s or ``torch.optim.AdamW``'s format."""

    STATE_NAMES = (("exp_avg", "exp_avg"), ("exp_avg_sq", "exp_avg_sq"),
                   ("max_exp_avg_sq", "max_exp_avg_sq"))

    def __init__(self, arena, lr, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, amsgrad=False,
                 adamw=False, param_groups=None):
        self.adamw = bool(adamw)
        super().__init__(arena, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay,
                                     amsgrad=amsgrad, maximize=False, foreach=None,
                                     capturable=False, differentiable=False, fused=None,
                                     decoupled_weight_decay=self.adamw), param_groups)

    def _kernel(self, name: str):
        """The Adam entry point ``name`` of ``KERNELS``, or its AdamW form (adam -> adamw)."""
        return getattr(KERNELS, name.replace("adam", "adamw", 1) if self.adamw else name)

    def _per_param_extra(self):
        return {"step": torch.tensor(float(self._steps))}

    def _dyn_row(self, h):
        step = self._steps + 1
        bc1 = 1.0 - float(h["betas"][0]) ** step
        bc2 = 1.0 - float(h["betas"][1]) ** step
        vals = (-(float(h["lr"]) / bc1), bc2 ** 0.5)
        if self.adamw:          # dyn[2]: the decay factor, formed in double and rounded once to fp32
            vals += (float(np.float32(1.0 - float(h["lr"]) * float(h["weight_decay"]))),)
        return vals

    def load_state_dict(self, state_dict: Dict[str, Any]) -> None:
        """Moments, step and hyper-parameters as the base class loads them; an AdamW optimizer takes
        ``torch.optim.Adam`` and ``torch.optim.AdamW`` state dicts alike and keeps reporting the rule
        it runs (``decoupled_weight_decay=True``)."""
        super().load_state_dict(state_dict)
        if self.adamw:
            for g in self.param_groups:
                g["decoupled_weight_decay"] = True

    def _launch(self, lo, hi, grad_scale, coef):
        h = self.hyper
        p, g, lp = self._slices(lo, hi)
        vmax = self._state("max_exp_avg_sq")[lo:hi] if h["amsgrad"] else None
        if self._use_sr(lo):
            self._kernel("adam_sr")(p, g, self._state("exp_avg")[lo:hi], self._state("exp_avg_sq")[lo:hi], vmax,
                                    hi - lo, arena_off=lo, seed=self.sr_seed, lr=float(h["lr"]),
                                    beta1=float(h["betas"][0]), beta2=float(h["betas"][1]), eps=float(h["eps"]),
                                    wd=float(h["weight_decay"]), step=self._steps + 1, grad_scale=grad_scale,
                                    grad_scale_dev=coef, dyn=self._dyn)
            return
        self._kernel("adam")(p, g, self._state("exp_avg")[lo:hi], self._state("exp_avg_sq")[lo:hi], vmax,
                             lp, hi - lo, lr=float(h["lr"]), beta1=float(h["betas"][0]),
                             beta2=float(h["betas"][1]), eps=float(h["eps"]),
                             wd=float(h["weight_decay"]), step=self._steps + 1,
                             grad_scale=grad_scale, grad_scale_dev=coef, dyn=self._dyn)

    def _launch_mt(self, table, grad_scale):
        h = self.hyper
        self._kernel("adam_mt")(self._master_base(), self._state("exp_avg"), self._state("exp_avg_sq"),
                                self._state("max_exp_avg_sq") if h["amsgrad"] else None, self._lp_mt(), table,
                                lr=float(h["lr"]), beta1=float(h["betas"][0]), beta2=float(h["betas"][1]),
                                eps=float(h["eps"]), wd=float(h["weight_decay"]), step=self._steps + 1,
                                grad_scale=grad_scale, dyn=self._dyn)

    def _launch_mt_sr(self, table, grad_scale):
        h = self.hyper
        self._kernel("adam_mt_sr")(self.arena.lp, self._state("exp_avg"), self._state("exp_avg_sq"),
                                   self._state("max_exp_avg_sq") if h["amsgrad"] else None, table,
                                   seed=self.sr_seed, lr=float(h["lr"]), beta1=float(h["betas"][0]),
                                   beta2=float(h["betas"][1]), eps=float(h["eps"]), wd=float(h["weight_decay"]),
                                   step=self._steps + 1, grad_scale=grad_scale, dyn=self._dyn)

    def _launch_mt_grouped(self, table, groups, grad_scale, coef):
        h = self.hyper
        self._kernel("adam_mt_grouped")(self._master_base(), self._state("exp_avg"), self._state("exp_avg_sq"),
                                        self._state("max_exp_avg_sq") if h["amsgrad"] else None, self._lp_mt(),
                                        table, groups, beta1=float(h["betas"][0]), beta2=float(h["betas"][1]),
                                        eps=float(h["eps"]), grad_scale=grad_scale, grad_scale_dev=coef)

    def _launch_mt_grouped_sr(self, table, groups, grad_scale, coef):
        h = self.hyper
        self._kernel("adam_mt_grouped_sr")(self.arena.lp, self._state("exp_avg"), self._state("exp_avg_sq"),
                                           self._state("max_exp_avg_sq") if h["amsgrad"] else None, table, groups,
                                           seed=self.sr_seed, beta1=float(h["betas"][0]),
                                           beta2=float(h["betas"][1]), eps=float(h["eps"]), grad_scale=grad_scale,
                                           grad_scale_dev=coef)

    def _launch_nvls(self, lo, hi, grad_scale):
        h = self.hyper
        mc_g, mc_out = self._nvls_ptrs(lo)
        vmax = self._state("max_exp_avg_sq")[lo:hi] if h["amsgrad"] else None
        self._kernel("nvls_adam")(self.arena.master[lo:hi], self._state("exp_avg")[lo:hi],
                                  self._state("exp_avg_sq")[lo:hi], vmax, mc_g, mc_out, hi - lo, self.nvls,
                                  lr=float(h["lr"]), beta1=float(h["betas"][0]), beta2=float(h["betas"][1]),
                                  eps=float(h["eps"]), wd=float(h["weight_decay"]), step=self._steps + 1,
                                  grad_scale=grad_scale, g_dtype=KERNELS.dtype_code(self.arena.grad.dtype),
                                  dyn=self._dyn)


class FusedRMSprop(FusedArenaOptimizer):
    STATE_NAMES = (("square_avg", "square_avg"), ("momentum_buffer", "momentum_buffer"))

    def __init__(self, arena, lr, alpha=0.99, eps=1e-8, weight_decay=0.0, momentum=0.0, param_groups=None):
        super().__init__(arena, dict(lr=lr, momentum=momentum, alpha=alpha, eps=eps,
                                     centered=False, weight_decay=weight_decay, capturable=False,
                                     foreach=None, maximize=False, differentiable=False), param_groups)

    def _per_param_extra(self):
        return {"step": torch.tensor(float(self._steps))}

    def _launch(self, lo, hi, grad_scale, coef):
        h = self.hyper
        p, g, lp = self._slices(lo, hi)
        mu = float(h["momentum"])
        buf = self._state("momentum_buffer")[lo:hi] if mu != 0.0 else None
        if self._use_sr(lo):
            KERNELS.rmsprop_sr(p, g, self._state("square_avg")[lo:hi], buf, hi - lo, arena_off=lo, seed=self.sr_seed,
                               t=self._steps + 1, lr=float(h["lr"]), alpha=float(h["alpha"]), eps=float(h["eps"]),
                               wd=float(h["weight_decay"]), mu=mu, grad_scale=grad_scale, grad_scale_dev=coef,
                               dyn=self._dyn)
            return
        KERNELS.rmsprop(p, g, self._state("square_avg")[lo:hi], buf, lp, hi - lo,
                        lr=float(h["lr"]), alpha=float(h["alpha"]), eps=float(h["eps"]),
                        wd=float(h["weight_decay"]), mu=mu, grad_scale=grad_scale,
                        grad_scale_dev=coef, dyn=self._dyn)

    def _launch_mt(self, table, grad_scale):
        h = self.hyper
        mu = float(h["momentum"])
        KERNELS.rmsprop_mt(self._master_base(), self._state("square_avg"),
                           self._state("momentum_buffer") if mu != 0.0 else None, self._lp_mt(), table,
                           lr=float(h["lr"]), alpha=float(h["alpha"]), eps=float(h["eps"]),
                           wd=float(h["weight_decay"]), mu=mu, grad_scale=grad_scale, dyn=self._dyn)

    def _launch_mt_sr(self, table, grad_scale):
        h = self.hyper
        mu = float(h["momentum"])
        KERNELS.rmsprop_mt_sr(self.arena.lp, self._state("square_avg"),
                              self._state("momentum_buffer") if mu != 0.0 else None, table, seed=self.sr_seed,
                              t=self._steps + 1, lr=float(h["lr"]), alpha=float(h["alpha"]), eps=float(h["eps"]),
                              wd=float(h["weight_decay"]), mu=mu, grad_scale=grad_scale, dyn=self._dyn)

    def _launch_mt_grouped(self, table, groups, grad_scale, coef):
        h = self.hyper
        mu = float(h["momentum"])
        KERNELS.rmsprop_mt_grouped(self._master_base(), self._state("square_avg"),
                                   self._state("momentum_buffer") if mu != 0.0 else None, self._lp_mt(), table, groups,
                                   alpha=float(h["alpha"]), eps=float(h["eps"]), mu=mu, grad_scale=grad_scale,
                                   grad_scale_dev=coef)

    def _launch_mt_grouped_sr(self, table, groups, grad_scale, coef):
        h = self.hyper
        mu = float(h["momentum"])
        KERNELS.rmsprop_mt_grouped_sr(self.arena.lp, self._state("square_avg"),
                                      self._state("momentum_buffer") if mu != 0.0 else None, table, groups,
                                      seed=self.sr_seed, alpha=float(h["alpha"]), eps=float(h["eps"]), mu=mu,
                                      grad_scale=grad_scale, grad_scale_dev=coef)

    def _launch_nvls(self, lo, hi, grad_scale):
        h = self.hyper
        mu = float(h["momentum"])
        mc_g, mc_out = self._nvls_ptrs(lo)
        buf = self._state("momentum_buffer")[lo:hi] if mu != 0.0 else None
        KERNELS.nvls_rmsprop(self.arena.master[lo:hi], self._state("square_avg")[lo:hi], buf, mc_g,
                             mc_out, hi - lo, self.nvls, lr=float(h["lr"]), alpha=float(h["alpha"]),
                             eps=float(h["eps"]), wd=float(h["weight_decay"]), mu=mu,
                             grad_scale=grad_scale,
                             g_dtype=KERNELS.dtype_code(self.arena.grad.dtype), dyn=self._dyn)


class FusedLion(FusedArenaOptimizer):
    """Lion (Chen et al. 2023, *Symbolic Discovery of Optimization Algorithms*, Algorithm 2) with
    decoupled weight decay on every parameter the optimizer owns: per element,
    ``p *= fp32(1 - lr*wd)``, ``p -= lr * sign(lerp(exp_avg, g, 1 - beta1))``, then
    ``exp_avg = lerp(exp_avg, g, 1 - beta2)``.  One state vector, so SGD-with-momentum's state size
    and bytes per update; the ``frl_lion*`` kernels on every path SGD has, K12 included.
    ``state_dict()`` is the layout of the published Lion implementations (lion-pytorch, timm): group
    ``lr``, ``betas``, ``weight_decay`` and per-parameter ``exp_avg``.  Lion wants a 3-10x smaller lr
    than AdamW; nothing here rescales it."""

    STATE_NAMES = (("exp_avg", "exp_avg"),)

    def __init__(self, arena, lr, betas=(0.9, 0.99), weight_decay=0.0, param_groups=None):
        super().__init__(arena, dict(lr=lr, betas=tuple(betas), weight_decay=weight_decay), param_groups)

    def _dyn_row(self, h):
        lr = float(h["lr"])       # dyn[1]: the decay factor, formed in double and rounded once to fp32
        return (lr, float(np.float32(1.0 - lr * float(h["weight_decay"]))))

    def _hyper(self, h: Optional[Dict[str, Any]] = None) -> Dict[str, float]:
        h = self.hyper if h is None else h
        return dict(lr=float(h["lr"]), beta1=float(h["betas"][0]), beta2=float(h["betas"][1]),
                    wd=float(h["weight_decay"]))

    def load_state_dict(self, state_dict: Dict[str, Any]) -> None:
        """A Lion state dict only: one holding another optimizer's state (SGD's ``momentum_buffer``,
        Adam's ``exp_avg_sq``, ...) or another optimizer's param group (no ``betas``, or SGD's
        ``momentum``; also before its first step, when the state is empty) is refused with a
        ValueError naming the keys."""
        for entry in state_dict["state"].values():
            foreign = sorted(k for k in entry if k not in ("exp_avg", "step"))
            if foreign:
                raise ValueError("a Lion optimizer cannot load another optimizer's state dict (found %s; Lion "
                                 "keeps exp_avg only)" % foreign)
        for g in state_dict["param_groups"]:
            if "betas" not in g or "momentum" in g:
                raise ValueError("a Lion optimizer cannot load another optimizer's state dict (param group keys %s; "
                                 "Lion's group has betas and no momentum)" % sorted(k for k in g if k != "params"))
        super().load_state_dict(state_dict)
        for g in self.param_groups:
            g["betas"] = tuple(g["betas"])

    def _launch(self, lo, hi, grad_scale, coef):
        p, g, lp = self._slices(lo, hi)
        m = self._state("exp_avg")[lo:hi]
        if self._use_sr(lo):
            KERNELS.lion_sr(p, g, m, hi - lo, arena_off=lo, seed=self.sr_seed, t=self._steps + 1, **self._hyper(),
                            grad_scale=grad_scale, grad_scale_dev=coef, dyn=self._dyn)
            return
        KERNELS.lion(p, g, m, lp, hi - lo, **self._hyper(), grad_scale=grad_scale, grad_scale_dev=coef,
                     dyn=self._dyn)

    def update_in_dw_gemm(self, slot, dz, x, gw, *, grad_scale: float = 1.0) -> None:
        """K12: the weight gradient gw = dz^T x of ``slot`` and, in the same kernel, this step's Lion
        update of the slot from exactly that bf16 gradient (what ``_launch`` over the slot does); with
        several param groups, the slot's group's lr / weight decay and ``dyn`` row."""
        a = self.arena
        h, dyn = self._slot_hyper(slot)
        m = self._state("exp_avg")[slot.offset:slot.end]
        if self._use_sr(slot.offset):
            KERNELS.dw_gemm_lion_sr(dz, x, gw, a.lp[slot.offset:slot.end], m, arena_off=slot.offset,
                                    seed=self.sr_seed, t=self._steps + 1, **self._hyper(h), grad_scale=grad_scale,
                                    dyn=dyn)
            return
        KERNELS.dw_gemm_lion(dz, x, gw, a.master[slot.offset:slot.end], m, a.lp[slot.offset:slot.end],
                             **self._hyper(h), grad_scale=grad_scale, dyn=dyn)

    def _launch_mt(self, table, grad_scale):
        KERNELS.lion_mt(self._master_base(), self._state("exp_avg"), self._lp_mt(), table, **self._hyper(),
                        grad_scale=grad_scale, dyn=self._dyn)

    def _launch_mt_sr(self, table, grad_scale):
        KERNELS.lion_mt_sr(self.arena.lp, self._state("exp_avg"), table, seed=self.sr_seed, t=self._steps + 1,
                           **self._hyper(), grad_scale=grad_scale, dyn=self._dyn)

    def _launch_mt_grouped(self, table, groups, grad_scale, coef):
        h = self.hyper
        KERNELS.lion_mt_grouped(self._master_base(), self._state("exp_avg"), self._lp_mt(), table, groups,
                                beta1=float(h["betas"][0]), beta2=float(h["betas"][1]), grad_scale=grad_scale,
                                grad_scale_dev=coef)

    def _launch_mt_grouped_sr(self, table, groups, grad_scale, coef):
        h = self.hyper
        KERNELS.lion_mt_grouped_sr(self.arena.lp, self._state("exp_avg"), table, groups, seed=self.sr_seed,
                                   beta1=float(h["betas"][0]), beta2=float(h["betas"][1]), grad_scale=grad_scale,
                                   grad_scale_dev=coef)

    def _launch_nvls(self, lo, hi, grad_scale):
        mc_g, mc_out = self._nvls_ptrs(lo)
        KERNELS.nvls_lion(self.arena.master[lo:hi], self._state("exp_avg")[lo:hi], mc_g, mc_out, hi - lo, self.nvls,
                          **self._hyper(), grad_scale=grad_scale, g_dtype=KERNELS.dtype_code(self.arena.grad.dtype),
                          dyn=self._dyn)


def is_adapted(slot) -> bool:
    """Layer-wise adaptation applies to tensors of 2 or more dimensions (``types.LayerAdaptation``)."""
    return len(slot.shape) >= 2


class _WholeTensorMixin:
    """An update over whole tensors through a segment table (``apply_table``): the pipeline runs it
    once after backward.  The flat-bucket and fused NVLS launchers of the base rule see parts of
    tensors: never reached, and refused rather than silently wrong."""

    @property
    def needs_whole_tensors(self) -> bool:
        return True

    def _launch(self, lo, hi, grad_scale, coef):
        raise RuntimeError("%s updates whole tensors: use apply_table / apply_range" % type(self).__name__)

    def _launch_mt(self, table, grad_scale):
        raise RuntimeError("%s updates through its own segment-table kernel: use apply_table" % type(self).__name__)

    def _launch_nvls(self, lo, hi, grad_scale):
        raise RuntimeError("%s has no fused NVLS step (its update needs whole tensors)" % type(self).__name__)

    def apply_range(self, lo: int, hi: int, *, grad_scale: float = 1.0,
                    clip_coef_dev: Optional[torch.Tensor] = None) -> None:
        """Whole slots inside ``[lo, hi)``, gradients read from the arena."""
        from .multi_tensor import GradSegTable
        tables = self.__dict__.setdefault("_range_tables", {})
        table = tables.get((lo, hi))
        if table is None:
            slots = [s for s in self.arena.slots if lo <= s.offset and s.end <= hi]
            cut = [s.index for s in self.arena.slots if s.offset < hi and s.end > lo and s not in slots]
            if cut:
                raise ValueError("%s takes whole tensors: [%d, %d) cuts the slots of parameters %s"
                                 % (type(self).__name__, lo, hi, cut))
            table = tables[(lo, hi)] = GradSegTable(slots, self.arena.device)
            g = self.arena.grad
            for s in slots:
                table.point(s, g.data_ptr() + s.offset * g.element_size(), g.dtype)
        table.upload()
        self.apply_table(table, grad_scale=grad_scale, clip_coef_dev=clip_coef_dev)


class _LayerwiseMixin(_WholeTensorMixin):
    """K2-lw: trust-ratio updates over a segment table (``frl_lars_mt`` / ``frl_lamb_mt``).  The
    per-table device buffers (adaptation flags, ratios, scratch) are built on first use and kept on
    the table, so a CUDA-graph capture's table set owns its own."""

    def _lw_buffers(self, table):
        bufs = getattr(table, "layerwise", None)
        if bufs is None:
            dev = self.arena.device
            flags = torch.tensor([(KERNELS.LW_ADAPTED if is_adapted(s) else 0)
                                  | (KERNELS.LW_CLIPPED if s.is_model else 0) for s in table.slots],
                                 dtype=torch.int32).to(dev)
            ratio = torch.ones(max(table.n_segs, 1), dtype=torch.float32, device=dev)
            nbytes = KERNELS.layerwise_scratch_bytes(table.n_tiles, table.n_segs)
            scratch = torch.zeros((nbytes + 15) // 16 * 4, dtype=torch.int32, device=dev)
            bufs = table.layerwise = (flags, ratio, scratch)
        return bufs

    def apply_table(self, table, *, grad_scale: float = 1.0,
                    clip_coef_dev: Optional[torch.Tensor] = None) -> None:
        """Update every slot of ``table``; ``clip_coef_dev`` multiplies the gradients of model
        parameters only, as in ``apply_range``."""
        if table.n_segs:
            self._launch_lw(table, grad_scale, clip_coef_dev, *self._lw_buffers(table))

    def last_ratios(self, table) -> torch.Tensor:
        """Trust ratio of each slot of ``table`` from its last update (device tensor)."""
        return self._lw_buffers(table)[1][:table.n_segs]


class FusedLars(_LayerwiseMixin, FusedSGD):
    """LARS: layer-wise trust ratio on the SGD rule (``types.LayerAdaptation.LARS``).  State and
    ``state_dict()`` are ``torch.optim.SGD``'s (``momentum_buffer`` in SGD's units)."""

    def __init__(self, arena, lr, momentum=0.0, weight_decay=0.0):
        super().__init__(arena, lr=lr, momentum=momentum, dampening=0.0, weight_decay=weight_decay)

    def _launch_lw(self, table, grad_scale, coef, flags, ratio, scratch):
        h = self.hyper
        mu = float(h["momentum"])
        KERNELS.lars_mt(self.arena.master, self._state("momentum_buffer") if mu != 0.0 else None,
                        self.arena.lp, table, flags, ratio, scratch, lr=float(h["lr"]), mu=mu,
                        wd=float(h["weight_decay"]), grad_scale=grad_scale, grad_scale_dev=coef,
                        first_step=(self._steps == 0), dyn=self._dyn)


class FusedLamb(_LayerwiseMixin, FusedAdam):
    """LAMB: layer-wise trust ratio on the Adam rule (``types.LayerAdaptation.LAMB``) with
    DECOUPLED weight decay on adapted tensors (part of the update direction, scaled by the ratio),
    unlike ``FusedAdam``'s L2-coupled decay.  State and ``state_dict()`` are
    ``torch.optim.Adam``'s, so checkpoints move between LAMB and Adam in both directions."""

    def __init__(self, arena, lr, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0):
        super().__init__(arena, lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, amsgrad=False)

    def _dyn_values(self):
        h = self.hyper
        step = self._steps + 1
        bc1 = 1.0 - float(h["betas"][0]) ** step
        bc2 = 1.0 - float(h["betas"][1]) ** step
        return (float(h["lr"]), 1.0 / bc1, bc2 ** 0.5)

    def _launch_lw(self, table, grad_scale, coef, flags, ratio, scratch):
        h = self.hyper
        KERNELS.lamb_mt(self.arena.master, self._state("exp_avg"), self._state("exp_avg_sq"), self.arena.lp,
                        table, flags, ratio, scratch, lr=float(h["lr"]), beta1=float(h["betas"][0]),
                        beta2=float(h["betas"][1]), eps=float(h["eps"]), wd=float(h["weight_decay"]),
                        step=self._steps + 1, grad_scale=grad_scale, grad_scale_dev=coef, dyn=self._dyn)


# ---- 8-bit block-wise Adam state (K2-q8) ----------------------------------------------------------

Q8_BLOCK = 256           # elements per quantisation block; blocks start at each tensor's first element
_DECADES = (1e-6, 1e-5, 1e-4, 1e-3, 1e-2, 1e-1, 1.0)


def q8_tables() -> Tuple[np.ndarray, np.ndarray]:
    """The storage format's two code tables (the dynamic tree map), fp32, increasing:
    ``MAG7`` (128 entries, ``exp_avg`` magnitudes: code = sign bit << 7 | index) and ``MAG8``
    (256 entries, ``exp_avg_sq``).  Each entry is formed in float64 and rounded once to fp32; both
    hold 0 and 1.  csrc/adam8.cu builds the same tables from the same expression."""
    mag7, mag8 = [0.0], [0.0]
    for i, dec in enumerate(_DECADES):
        n7, n8 = 1 << i, 2 << i
        mag7 += [dec * (0.1 + 0.9 * (j + 0.5) / n7) for j in range(n7)]
        mag8 += [dec * (0.1 + 0.9 * (j + 0.5) / n8) for j in range(n8)]
    mag7[-1] = 1.0                      # replaces the largest, 0.99296875
    mag8.append(1.0)
    return np.asarray(mag7, dtype=np.float32), np.asarray(mag8, dtype=np.float32)


def q8_block_bases(slots) -> Tuple[Dict[int, int], int]:
    """Global index of each slot's first block (by slot index): a prefix sum of ceil(numel / 256)
    over ``slots`` in arena order, and the total number of blocks."""
    bases, n = {}, 0
    for s in sorted(slots, key=lambda s: s.offset):
        bases[s.index] = n
        n += (s.numel + Q8_BLOCK - 1) // Q8_BLOCK
    return bases, n


class FusedAdam8bit(_WholeTensorMixin, FusedAdam):
    """Adam (``FusedAdam``'s rule and hyper-parameters, no amsgrad) with ``exp_avg`` /
    ``exp_avg_sq`` kept as 8-bit block-wise codes (``types.OptimizerState.Q8``): one byte per
    arena element per state plus one fp32 absmax per 256-element block, updated by one K2-q8 launch
    over a segment table after backward.  ``state_dict()`` writes ``torch.optim.Adam``'s format with
    the decoded fp32 moments; ``load_state_dict()`` encodes them, so checkpoints move between
    ``torch.optim.Adam``, ``FusedAdam`` and this optimizer in both directions, and a run resumed
    from its own checkpoint continues bit for bit (decode-then-encode returns the same codes).
    ``adamw=True``: ``FusedAdam``'s AdamW rule (K2-q8 AdamW) and ``torch.optim.AdamW``'s format."""

    STATE_NAMES = (("exp_avg", "exp_avg"), ("exp_avg_sq", "exp_avg_sq"))

    def __init__(self, arena, lr, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, adamw=False):
        super().__init__(arena, lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, amsgrad=False,
                         adamw=adamw)
        self._qbase, self.q8_blocks = q8_block_bases(arena.slots)
        dev = arena.device
        self.codes = {n: torch.zeros(arena.numel, dtype=torch.uint8, device=dev) for n, _ in self.STATE_NAMES}
        self.absmax = {n: torch.zeros(max(self.q8_blocks, 1), dtype=torch.float32, device=dev)
                       for n, _ in self.STATE_NAMES}
        self._all_table = None

    @property
    def state_bytes(self) -> int:
        """Device bytes of the optimizer state (codes and absmax of both moments)."""
        return sum(t.numel() * t.element_size() for d in (self.codes, self.absmax) for t in d.values())

    @property
    def fp32_state_bytes(self) -> int:
        """What ``FusedAdam`` keeps for the same arena: two fp32 arena-shaped vectors."""
        return 2 * 4 * self.arena.numel

    def _q8_buffers(self, table):
        """Per-table device arrays, kept on the table: each slot's first block, and its flags
        (``LW_CLIPPED``: model parameters take the clip coefficient)."""
        bufs = getattr(table, "adam8", None)
        if bufs is None:
            dev = self.arena.device
            qbase = torch.tensor([self._qbase[s.index] for s in table.slots] or [0], dtype=torch.int64).to(dev)
            flags = torch.tensor([KERNELS.LW_CLIPPED if s.is_model else 0 for s in table.slots] or [0],
                                 dtype=torch.int32).to(dev)
            bufs = table.adam8 = (qbase, flags)
        return bufs

    def apply_table(self, table, *, grad_scale: float = 1.0,
                    clip_coef_dev: Optional[torch.Tensor] = None) -> None:
        """Update every slot of ``table`` (K2-q8); ``clip_coef_dev`` multiplies the gradients of
        model parameters only, as in ``apply_range``."""
        if not table.n_segs:
            return
        h = self.hyper
        qbase, flags = self._q8_buffers(table)
        self._kernel("adam8_mt")(self.arena.master, self.codes["exp_avg"], self.codes["exp_avg_sq"],
                                 self.absmax["exp_avg"], self.absmax["exp_avg_sq"], self.arena.lp, table, qbase, flags,
                                 lr=float(h["lr"]), beta1=float(h["betas"][0]), beta2=float(h["betas"][1]),
                                 eps=float(h["eps"]), wd=float(h["weight_decay"]), step=self._steps + 1,
                                 grad_scale=grad_scale, grad_scale_dev=clip_coef_dev, dyn=self._dyn)

    def _every_slot(self):
        if self._all_table is None:
            from .multi_tensor import GradSegTable
            self._all_table = GradSegTable(self.arena.slots, self.arena.device)     # gradients not read
            self._all_table.upload()
        return self._all_table, self._q8_buffers(self._all_table)[0]

    def decoded(self, name: str) -> torch.Tensor:
        """``exp_avg`` or ``exp_avg_sq`` decoded into a fresh fp32 arena-shaped vector."""
        table, qbase = self._every_slot()
        out = self.arena.new_state()
        KERNELS.q8_decode_mt(self.codes[name], self.absmax[name], out, self._state_code(name), table, qbase)
        return out

    def _encode(self, name: str, x: torch.Tensor) -> None:
        table, qbase = self._every_slot()
        KERNELS.q8_encode_mt(x, self.codes[name], self.absmax[name], self._state_code(name), table, qbase)

    @staticmethod
    def _state_code(name: str) -> int:
        return KERNELS.Q8_EXP_AVG if name == "exp_avg" else KERNELS.Q8_EXP_AVG_SQ

    def state_dict(self) -> Dict[str, Any]:
        self._vec = {n: self.decoded(n) for n, _ in self.STATE_NAMES} if self._steps > 0 else {}
        try:
            return super().state_dict()
        finally:
            self._vec = {}

    def load_state_dict(self, state_dict: Dict[str, Any]) -> None:
        for g in state_dict["param_groups"]:
            if g.get("amsgrad", False):
                raise ValueError("8-bit Adam state holds no max_exp_avg_sq: an amsgrad state dict cannot be loaded")
        self._vec = {}
        try:
            super().load_state_dict(state_dict)       # fills fp32 vectors through _state()
            for name, _ in self.STATE_NAMES:
                self._encode(name, self._vec[name] if name in self._vec else self.arena.new_state())
        finally:
            self._vec = {}


# ---- Adafactor (K2-af) -----------------------------------------------------------------------------

def adafactor_shape(shape) -> Tuple[int, int, int]:
    """(B, R, C) of a parameter under Adafactor: a tensor of 2 or more dimensions is B = prod of
    the leading dimensions matrices of [R, C] = its last two (factored); any other is
    (1, 0, numel), kept unfactored.  The kernel's shape array takes (1, 0, 0) for a tensor with no
    elements (``kernel_shape``): nothing to update."""
    shape = tuple(int(x) for x in shape)
    if len(shape) >= 2:
        return int(np.prod(shape[:-2], dtype=np.int64)), shape[-2], shape[-1]
    return 1, 0, int(np.prod(shape, dtype=np.int64))


def adafactor_kernel_shape(shape) -> Tuple[int, int, int]:
    return (1, 0, 0) if int(np.prod(tuple(shape), dtype=np.int64)) == 0 else adafactor_shape(shape)


def adafactor_state_elems(shape) -> int:
    b, r, c = adafactor_shape(shape)
    return b * (r + c) if len(tuple(shape)) >= 2 else c


class FusedAdafactor(_WholeTensorMixin, FusedArenaOptimizer):
    """Adafactor (Shazeer & Stern, ICML 2018) with ``torch.optim.Adafactor``'s rule, defaults and
    state-dict format: no first moment, the second moment of a 2-D or higher tensor factored into
    ``row_var`` / ``col_var``, a relative step size and update clipping, decoupled weight decay on
    every parameter.  The state lives in one compact fp32 buffer (row_var then col_var, or the
    variance, per slot in arena order), updated by the three K2-af launches over a segment table
    after backward."""

    def __init__(self, arena, lr=1e-2, beta2_decay=-0.8, eps=(None, 1e-3), d=1.0, weight_decay=0.0):
        super().__init__(arena, dict(lr=lr, beta2_decay=beta2_decay, eps=tuple(eps), d=d, weight_decay=weight_decay,
                                     foreach=None, maximize=False))
        self._off: Dict[int, int] = {}
        n = 0
        for s in sorted(arena.slots, key=lambda s: s.offset):
            self._off[s.index] = n
            n += adafactor_state_elems(s.shape)
        self.state_buf = torch.zeros(max(n, 1), dtype=torch.float32, device=arena.device)
        self._state_elems = n

    @property
    def state_bytes(self) -> int:
        """Device bytes of the optimizer state (row / column factors and unfactored variances)."""
        return 4 * self._state_elems

    @property
    def fp32_state_bytes(self) -> int:
        """What ``FusedAdam`` keeps for the same arena: two fp32 arena-shaped vectors."""
        return 2 * 4 * self.arena.numel

    def _eps1(self) -> float:
        e = self.hyper["eps"][0]
        return float(torch.finfo(torch.float32).eps) if e is None else float(e)

    def _dyn_values(self):
        h = self.hyper
        t = float(self._steps + 1)
        lr = float(h["lr"])
        return (lr, t ** float(h["beta2_decay"]), min(lr, 1.0 / t ** 0.5))

    def _af_plan(self, table):
        """Per-table device arrays, kept on the table: (B, R, C), state offset, flags
        (``LW_CLIPPED``: model parameters take the clip coefficient), the band table and the
        zero-initialised scratch."""
        plan = getattr(table, "adafactor", None)
        if plan is None:
            dev = self.arena.device
            shape = torch.tensor([adafactor_kernel_shape(s.shape) for s in table.slots] or [(1, 0, 1)],
                                 dtype=torch.int64)
            work, seg_info = KERNELS.adafactor_plan(shape)
            off = torch.tensor([self._off[s.index] for s in table.slots] or [0], dtype=torch.int64)
            flags = torch.tensor([KERNELS.LW_CLIPPED if s.is_model else 0 for s in table.slots] or [0],
                                 dtype=torch.int32)
            nbytes = KERNELS.adafactor_scratch_bytes(shape)
            scratch = torch.zeros((nbytes + 15) // 16 * 4, dtype=torch.int32, device=dev)
            plan = table.adafactor = (shape.to(dev), off.to(dev), flags.to(dev), work.to(dev), seg_info.to(dev),
                                      scratch, shape)
        return plan

    def apply_table(self, table, *, grad_scale: float = 1.0,
                    clip_coef_dev: Optional[torch.Tensor] = None) -> None:
        """Update every slot of ``table`` (K2-af); ``clip_coef_dev`` multiplies the gradients of
        model parameters only, as in ``apply_range``."""
        if not table.n_segs:
            return
        h = self.hyper
        KERNELS.adafactor_mt(self.arena.master, self.state_buf, self.arena.lp, table, self._af_plan(table),
                             lr=float(h["lr"]), beta2_decay=float(h["beta2_decay"]), eps1=self._eps1(),
                             eps2=float(h["eps"][1]), d=float(h["d"]), wd=float(h["weight_decay"]),
                             step=self._steps + 1, grad_scale=grad_scale, grad_scale_dev=clip_coef_dev,
                             dyn=self._dyn)

    def _slot_state(self, s) -> Dict[str, torch.Tensor]:
        """Views of slot ``s``'s state in torch's shapes."""
        b, r, c = adafactor_shape(s.shape)
        o = self._off[s.index]
        if len(s.shape) < 2:
            return {"variance": self.state_buf[o:o + c].view(s.shape)}
        lead = tuple(s.shape[:-2])
        return {"row_var": self.state_buf[o:o + b * r].view(lead + (r, 1)),
                "col_var": self.state_buf[o + b * r:o + b * (r + c)].view(lead + (1, c))}

    def state_dict(self) -> Dict[str, Any]:
        state: Dict[int, Dict[str, Any]] = {}
        if self._steps > 0:
            for s in sorted(self.arena.slots, key=lambda s: s.index):
                entry = {"step": torch.tensor(float(self._steps), dtype=torch.float32)}
                entry.update({k: v.clone() for k, v in self._slot_state(s).items()})
                state[s.index] = entry
        groups = []
        for g in self.param_groups:
            packed = {k: v for k, v in g.items() if k != "params"}
            packed["params"] = list(range(len(g["params"])))
            groups.append(packed)
        return {"state": state, "param_groups": groups}

    def load_state_dict(self, state_dict: Dict[str, Any]) -> None:
        groups = state_dict["param_groups"]
        if len(groups) != 1 or len(groups[0]["params"]) != len(self.arena.all_params):
            raise ValueError("loaded state dict has a different number of parameters/groups")
        for entry in state_dict["state"].values():
            if "exp_avg" in entry or "exp_avg_sq" in entry or "momentum_buffer" in entry or "square_avg" in entry:
                raise ValueError("an Adafactor optimizer cannot load another optimizer's state dict "
                                 "(found %s)" % sorted(k for k in entry if k != "step"))
        for k, v in groups[0].items():
            if k != "params":
                self.param_groups[0][k] = tuple(v) if k == "eps" else v
        by_index = {s.index: s for s in self.arena.slots}
        steps = 0
        for idx, entry in state_dict["state"].items():
            s = by_index.get(int(idx))
            if s is None:
                continue
            for name, view in self._slot_state(s).items():
                if name in entry:
                    view.copy_(entry[name].reshape(view.shape))
            if "step" in entry:
                steps = max(steps, int(float(entry["step"])))
        self._steps = steps


def check_adafactor(optim_opts: OptimOpts, layer_adaptation: LayerAdaptation,
                    optimizer_state: OptimizerState, adafactor: bool) -> None:
    """Adafactor needs Adam without amsgrad, no layer adaptation and fp32 optimizer state; anything
    else is a ValueError naming the values."""
    if not adafactor:
        return
    st = OptimizerState(optimizer_state)
    la = LayerAdaptation(layer_adaptation)
    if not (optim_opts.algo == OptAlgorithm.ADAM and not optim_opts.amsgrad and la is LayerAdaptation.NONE
            and st is OptimizerState.FP32):
        raise ValueError("adafactor cannot be combined with optimizer %r%s, layer adaptation %r and optimizer "
                         "state %r (adafactor needs adam without amsgrad, layer adaptation none and optimizer "
                         "state fp32)" % (getattr(optim_opts.algo, "value", optim_opts.algo),
                                          " with amsgrad" if optim_opts.amsgrad else "", la.value, st.value))


# ---- Muon (K14) for the model's matrices, Adam (K2-mt) for the rest ------------------------------------

MUON_NS_COEFFICIENTS = (3.4445, -4.7750, 2.0315)


def is_muon_slot(slot) -> bool:
    """Muon updates the model parameters with exactly two dimensions (Linear weights, embeddings,
    task heads); biases, normalisation affine parameters, conv kernels and criterion parameters
    stay with Adam."""
    return slot.is_model and len(slot.shape) == 2


def _gather_segs(parent, sub, idx: Tuple[torch.Tensor, torch.Tensor]) -> None:
    """Copy rows ``idx`` (host, device) of ``parent``'s segment table into ``sub``: the host copy, and
    the device copy on the stream, so a captured CUDA graph re-reads the parent's rows on every
    replay."""
    from .multi_tensor import _SEG_BYTES
    n = sub.n_segs
    sub._host.view(-1, _SEG_BYTES)[:n] = parent._host.view(-1, _SEG_BYTES)[idx[0]]
    torch.index_select(parent._dev.view(-1, _SEG_BYTES), 0, idx[1], out=sub._dev.view(-1, _SEG_BYTES)[:n])


class FusedMuon(_WholeTensorMixin, FusedAdam):
    """``torch.optim.Muon`` (group 0: the model's 2-D parameters, ``is_muon_slot``) plus
    ``FusedAdam``'s rule (group 1: every other parameter), updated once after backward: K14 over
    the Muon matrices, K2-mt over the rest.  Inside a Muon slot's range ``exp_avg`` holds the
    momentum buffer and ``exp_avg_sq`` the two bf16 Newton-Schulz iterates, so the state costs
    what Adam's does; K14's Gram workspace (``workspace_bytes``) comes on top.  ``state_dict()``
    has the two groups in torch's format; ``split_muon_state_dict`` / ``join_muon_state_dict``
    convert it to and from a ``torch.optim.Muon`` plus a ``torch.optim.Adam`` (with ``adamw=True``,
    a ``torch.optim.AdamW``: group 1 then runs ``FusedAdam``'s AdamW rule)."""

    STATE_NAMES = (("exp_avg", "exp_avg"), ("exp_avg_sq", "exp_avg_sq"))

    def __init__(self, arena, lr, weight_decay=0.0, momentum=0.95, eps=1e-8, betas=(0.9, 0.999), nesterov=True,
                 ns_coefficients=MUON_NS_COEFFICIENTS, muon_eps=1e-7, ns_steps=5,
                 adjust_lr_fn="match_rms_adamw", adamw=False):
        super().__init__(arena, lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, amsgrad=False,
                         adamw=adamw)
        muon_ids = {id(s.param) for s in arena.slots if is_muon_slot(s)}
        self.muon_params = [p for p in arena.all_params if id(p) in muon_ids]
        self.adam_params = [p for p in arena.all_params if id(p) not in muon_ids]
        adam = dict(self.param_groups[0])
        adam["params"] = self.adam_params
        muon = dict(lr=lr, weight_decay=weight_decay, momentum=momentum, nesterov=nesterov,
                    ns_coefficients=tuple(ns_coefficients), eps=muon_eps, ns_steps=ns_steps,
                    adjust_lr_fn=adjust_lr_fn, params=self.muon_params)
        self.param_groups = [muon, adam]
        self._muon_rows = [(s.offset, s.shape[0], s.shape[1]) for s in arena.slots if is_muon_slot(s)]
        # one Gram workspace for every table's plan (their launches are stream-ordered): sized for
        # all the Muon matrices, any subset fits
        self.workspace_bytes = KERNELS.muon_plan_bytes(torch.tensor(
            [(0,) + r for r in self._muon_rows], dtype=torch.int64).reshape(-1, 4))[2] if self._muon_rows else 0
        self._workspace: Optional[torch.Tensor] = None

    @property
    def hyper(self) -> Dict[str, Any]:
        return self.param_groups[1]

    @property
    def muon_group(self) -> Dict[str, Any]:
        return self.param_groups[0]

    def _dyn_values(self):
        # dyn[0], dyn[1]: K2-mt's Adam scalars; then AdamW's decay factor, if any; last: K14's lr,
        # which K14 reads as its dyn[2] (``_muon_dyn``)
        return super()._dyn_values() + (float(self.muon_group["lr"]),)

    def _muon_dyn(self) -> Optional[torch.Tensor]:
        """The ``dyn`` K14 is given: the block itself, or with AdamW (whose decay factor takes
        dyn[2]) the block from its second float, so that K14's dyn[2] is the Muon lr."""
        if self._dyn is None or not self.adamw:
            return self._dyn
        return self._dyn[1:]

    def _split(self, table):
        """Per-table pieces, kept on the table: K14's plan over its Muon slots and the K2-mt
        tables of the other slots (all of them; model parameters; criterion parameters) with the
        rows of ``table`` they take."""
        split = getattr(table, "muon", None)
        if split is None:
            from .multi_tensor import GradSegTable
            dev = self.arena.device
            rows = list(enumerate(table.slots))
            mu = [(i, s) for i, s in rows if is_muon_slot(s)]
            rest = [(i, s) for i, s in rows if not is_muon_slot(s)]
            plan = None
            if mu:
                shape = torch.tensor([(i, s.offset, s.shape[0], s.shape[1]) for i, s in mu], dtype=torch.int64)
                if self._workspace is None:
                    self._workspace = torch.zeros((self.workspace_bytes + 127) // 128 * 32, dtype=torch.int32,
                                                  device=dev)
                plan = KERNELS.muon_plan(shape, self._state("exp_avg_sq"), self._workspace)
            subs = []
            for keep in (lambda s: True, lambda s: s.is_model, lambda s: not s.is_model):
                part = [(i, s) for i, s in rest if keep(s)]
                sub = GradSegTable([s for _, s in part], dev) if part else None
                rows_of = torch.tensor([i for i, _ in part], dtype=torch.int64)
                idx = (rows_of, rows_of.to(dev)) if part else None
                subs.append((sub, idx))
            split = table.muon = (plan, subs)
        return split

    def apply_table(self, table, *, grad_scale: float = 1.0,
                    clip_coef_dev: Optional[torch.Tensor] = None) -> None:
        """Update every slot of ``table``: one K2-mt launch over the non-Muon slots (two under
        clipping when the table also holds criterion parameters, which are not clipped), then K14
        over the Muon slots."""
        if not table.n_segs:
            return
        plan, (every, model, crit) = self._split(table)
        h, g = self.hyper, self.muon_group
        if plan is not None:          # refuse before any launch, not after Adam's half of the step
            KERNELS.check_muon_hyper(lr=g["lr"], wd=g["weight_decay"], momentum=g["momentum"],
                                     ns_steps=g["ns_steps"], eps=g["eps"], adjust_lr_fn=g["adjust_lr_fn"])
        launches = [(every, clip_coef_dev)] if clip_coef_dev is None or crit[0] is None else \
            [(model, clip_coef_dev), (crit, None)]
        for (sub, idx), coef in launches:
            if sub is None:
                continue
            _gather_segs(table, sub, idx)
            self._kernel("adam_mt")(self.arena.master, self._state("exp_avg"), self._state("exp_avg_sq"), None,
                                    self.arena.lp, sub, lr=float(h["lr"]), beta1=float(h["betas"][0]),
                                    beta2=float(h["betas"][1]), eps=float(h["eps"]), wd=float(h["weight_decay"]),
                                    step=self._steps + 1, grad_scale=grad_scale, grad_scale_dev=coef, dyn=self._dyn)
        if plan is not None:
            KERNELS.muon_mt(self.arena.master, self._state("exp_avg"), self.arena.lp, table, plan,
                            lr=float(g["lr"]), wd=float(g["weight_decay"]), momentum=float(g["momentum"]),
                            nesterov=bool(g["nesterov"]), ns_coefficients=tuple(g["ns_coefficients"]),
                            ns_steps=g["ns_steps"], eps=float(g["eps"]), adjust_lr_fn=g["adjust_lr_fn"],
                            grad_scale=grad_scale, grad_scale_dev=clip_coef_dev, dyn=self._muon_dyn())

    def _positions(self) -> Dict[int, int]:
        """torch's state-dict index of each parameter: group 0's, then group 1's."""
        return {id(p): i for i, p in enumerate(self.muon_params + self.adam_params)}

    def state_dict(self) -> Dict[str, Any]:
        state: Dict[int, Dict[str, Any]] = {}
        pos = self._positions()
        if self._steps > 0:
            for s in sorted(self.arena.slots, key=lambda s: pos[id(s.param)]):
                view = lambda name: ParamArena.slot_view(self._state(name), s).clone(
                    memory_format=torch.contiguous_format)
                if is_muon_slot(s):
                    state[pos[id(s.param)]] = {"momentum_buffer": view("exp_avg")}
                else:
                    state[pos[id(s.param)]] = {"step": torch.tensor(float(self._steps)),
                                               "exp_avg": view("exp_avg"), "exp_avg_sq": view("exp_avg_sq")}
        groups, base = [], 0
        for g in self.param_groups:
            packed = {k: v for k, v in g.items() if k != "params"}
            packed["params"] = list(range(base, base + len(g["params"])))
            base += len(g["params"])
            groups.append(packed)
        return {"state": state, "param_groups": groups}

    def load_state_dict(self, state_dict: Dict[str, Any]) -> None:
        groups = state_dict["param_groups"]
        if len(groups) != 2:
            raise ValueError("a Muon optimizer takes a state dict with two param groups (Muon, Adam), got %d; "
                             "join a torch.optim.Muon and a torch.optim.Adam state dict with join_muon_state_dict"
                             % len(groups))
        if len(groups[0]["params"]) != len(self.muon_params) or len(groups[1]["params"]) != len(self.adam_params):
            raise ValueError("loaded state dict has %d Muon and %d Adam parameters, this optimizer %d and %d"
                             % (len(groups[0]["params"]), len(groups[1]["params"]), len(self.muon_params),
                                len(self.adam_params)))
        for mine, theirs in zip(self.param_groups, groups):
            for k, v in theirs.items():
                if k != "params":
                    mine[k] = tuple(v) if k == "ns_coefficients" else v
        position = {q: j for j, q in enumerate(list(groups[0]["params"]) + list(groups[1]["params"]))}
        params = self.muon_params + self.adam_params
        slots = {id(s.param): s for s in self.arena.slots}
        steps = 0
        for key, entry in state_dict["state"].items():
            if key not in position:
                continue
            s = slots.get(id(params[position[key]]))
            if s is None:
                continue
            names = ((("momentum_buffer", "exp_avg"),) if is_muon_slot(s) else
                     (("exp_avg", "exp_avg"), ("exp_avg_sq", "exp_avg_sq")))
            for torch_name, vec in names:
                if entry.get(torch_name) is not None:
                    ParamArena.slot_view(self._state(vec), s).copy_(entry[torch_name])
            if "step" in entry:
                steps = max(steps, int(float(entry["step"])))
            elif entry:
                steps = max(steps, 1)
        self._steps = steps
        if self.adamw:
            self.hyper["decoupled_weight_decay"] = True


def split_muon_state_dict(sd: Dict[str, Any]) -> Tuple[Dict[str, Any], Dict[str, Any]]:
    """A ``FusedMuon`` state dict -> (``torch.optim.Muon`` state dict over group 0's parameters,
    ``torch.optim.Adam`` state dict over group 1's; ``torch.optim.AdamW``'s under AdamW)."""
    groups = sd["param_groups"]
    if len(groups) != 2:
        raise ValueError("a Muon state dict has two param groups (Muon, Adam), got %d" % len(groups))
    out = []
    for g in groups:
        ids = list(g["params"])
        state = {j: sd["state"][i] for j, i in enumerate(ids) if i in sd["state"]}
        packed = dict(g)
        packed["params"] = list(range(len(ids)))
        out.append({"state": state, "param_groups": [packed]})
    return out[0], out[1]


def join_muon_state_dict(muon_sd: Dict[str, Any], adam_sd: Dict[str, Any]) -> Dict[str, Any]:
    """The inverse of ``split_muon_state_dict``: one ``torch.optim.Muon`` and one ``torch.optim.Adam``
    or ``torch.optim.AdamW`` state dict (one group each) -> a ``FusedMuon`` state dict."""
    state, groups, base = {}, [], 0
    for sd in (muon_sd, adam_sd):
        if len(sd["param_groups"]) != 1:
            raise ValueError("join_muon_state_dict takes one-group Muon and Adam state dicts")
        g = sd["param_groups"][0]
        ids = list(g["params"])
        for j, i in enumerate(ids):
            if i in sd["state"]:
                state[base + j] = sd["state"][i]
        packed = dict(g)
        packed["params"] = list(range(base, base + len(ids)))
        groups.append(packed)
        base += len(ids)
    return {"state": state, "param_groups": groups}


def check_muon(optim_opts: OptimOpts, layer_adaptation: LayerAdaptation, optimizer_state: OptimizerState,
               adafactor: bool, muon: bool) -> None:
    """Muon needs Adam without amsgrad (for the other parameters), no layer adaptation, fp32
    optimizer state and no Adafactor; anything else is a ValueError naming the values."""
    if not muon:
        return
    st = OptimizerState(optimizer_state)
    la = LayerAdaptation(layer_adaptation)
    if not (optim_opts.algo == OptAlgorithm.ADAM and not optim_opts.amsgrad and la is LayerAdaptation.NONE
            and st is OptimizerState.FP32 and not adafactor):
        raise ValueError("muon cannot be combined with optimizer %r%s, layer adaptation %r, optimizer state %r%s "
                         "(muon needs adam without amsgrad, layer adaptation none, optimizer state fp32 and no "
                         "adafactor)" % (getattr(optim_opts.algo, "value", optim_opts.algo),
                                         " with amsgrad" if optim_opts.amsgrad else "", la.value, st.value,
                                         " and adafactor" if adafactor else ""))


def check_adamw(optim_opts: OptimOpts, layer_adaptation: LayerAdaptation, optimizer_state: OptimizerState,
                adafactor: bool, adamw: bool) -> None:
    """AdamW is a form of the Adam rule: it needs ``OptAlgorithm.ADAM`` (amsgrad, 8-bit state and
    Muon as Adam allows them), no layer adaptation (LAMB's decay is already decoupled) and no
    Adafactor; anything else is a ValueError naming the values."""
    if not adamw:
        return
    st = OptimizerState(optimizer_state)
    la = LayerAdaptation(layer_adaptation)
    if not (optim_opts.algo == OptAlgorithm.ADAM and la is LayerAdaptation.NONE and not adafactor):
        raise ValueError("adamw cannot be combined with optimizer %r%s, layer adaptation %r, optimizer state %r%s "
                         "(adamw needs adam, layer adaptation none and no adafactor)"
                         % (getattr(optim_opts.algo, "value", optim_opts.algo),
                            " with amsgrad" if optim_opts.amsgrad else "", la.value, st.value,
                            " and adafactor" if adafactor else ""))


def check_lion(optim_opts: OptimOpts, layer_adaptation: LayerAdaptation, lion: bool) -> None:
    """Lion replaces SGD-with-momentum's rule and keeps its state shape: it needs ``OptAlgorithm.SGD``
    and no layer adaptation; anything else is a ValueError naming the values.  (Adafactor, Muon,
    AdamW and 8-bit state need Adam, so their own checks refuse them next to Lion.)"""
    if not lion:
        return
    la = LayerAdaptation(layer_adaptation)
    if not (optim_opts.algo == OptAlgorithm.SGD and la is LayerAdaptation.NONE):
        raise ValueError("lion cannot be combined with optimizer %r and layer adaptation %r (lion needs sgd, "
                         "whose momentum is its beta1, and layer adaptation none)"
                         % (getattr(optim_opts.algo, "value", optim_opts.algo), la.value))


def check_master_weights(master_weights: MasterWeights, precision: Precision, layer_adaptation: LayerAdaptation,
                         optimizer_state: OptimizerState, adafactor: bool, muon: bool) -> None:
    """Bf16 master weights need a bf16-storage precision and an update with a stochastic-rounding
    kernel (SGD, Adam / AdamW, RMSprop); every other combination is a ValueError naming it."""
    if MasterWeights(master_weights) is not MasterWeights.BF16:
        return
    why = None
    if not Precision(precision).bf16_storage:
        why = "precision %s (there is no bf16 weight storage to keep)" % Precision(precision).value
    elif LayerAdaptation(layer_adaptation) is not LayerAdaptation.NONE:
        why = "layer adaptation %s" % LayerAdaptation(layer_adaptation).value
    elif adafactor:
        why = "adafactor"
    elif muon:
        why = "muon"
    elif OptimizerState(optimizer_state) is OptimizerState.Q8:
        why = "optimizer state %s" % OptimizerState.Q8.value
    if why is not None:
        raise ValueError("master_weights=bf16 cannot be combined with %s: stochastic rounding is implemented for "
                         "the sgd, adam / adamw and rmsprop updates in bf16 and fp8 precision" % why)


def check_optimizer_state(optim_opts: OptimOpts, layer_adaptation: LayerAdaptation,
                          optimizer_state: OptimizerState) -> None:
    """8-bit state needs Adam without amsgrad and without layer adaptation; anything else is a
    ValueError naming the values."""
    st = OptimizerState(optimizer_state)
    la = LayerAdaptation(layer_adaptation)
    if st is OptimizerState.Q8 and not (optim_opts.algo == OptAlgorithm.ADAM and not optim_opts.amsgrad
                                        and la is LayerAdaptation.NONE):
        raise ValueError("optimizer state %r cannot be combined with optimizer %r%s and layer adaptation %r "
                         "(8-bit state needs adam without amsgrad and layer adaptation none)"
                         % (st.value, getattr(optim_opts.algo, "value", optim_opts.algo),
                            " with amsgrad" if optim_opts.amsgrad else "", la.value))


GROUP_KEYS = ("params", "lr", "weight_decay")


def no_decay_1d_groups(model) -> List[Dict[str, Any]]:
    """The param groups of the ``no_decay_1d`` switch: every model parameter with ``ndim <= 1``
    (biases, normalisation parameters) in one group with ``weight_decay = 0``; none if there is no
    such parameter."""
    flat = [p for p in model.parameters() if p.ndim <= 1]
    return [{"params": flat, "weight_decay": 0.0}] if flat else []


def resolve_param_groups(model, criterion_params, hook_groups) -> Optional[List[Dict[str, Any]]]:
    """The canonical param groups of an optimizer from the groups a Problem's ``get_param_groups``
    hook (or the ``no_decay_1d`` switch) returned; None if there are none (``hook_groups`` None).

    Canonical order, which numbers the params of the state dict: the hook's groups in the order
    returned, then one default group (``OptimOpts``' lr / weightDecay, no keys of its own) with every
    remaining model parameter in ``model.parameters()`` order followed by the criterion parameters;
    the default group is omitted if empty.  A group is a dict with ``params`` (model parameters) and
    optionally ``lr`` / ``weight_decay`` (absolute values, torch's meaning).  Any other key, an empty
    group, a parameter listed twice, one that is not in ``model.parameters()`` and a criterion
    parameter are each a ValueError."""
    if hook_groups is None:
        return None
    model_params = list(model.parameters())
    model_ids = {id(p) for p in model_params}
    crit = list(criterion_params)
    crit_ids = {id(p) for p in crit}
    seen = set()
    out: List[Dict[str, Any]] = []
    for gi, g in enumerate(hook_groups):
        if not isinstance(g, dict) or "params" not in g:
            raise ValueError("param group %d must be a dict with a 'params' key, got %r" % (gi, type(g).__name__))
        extra = sorted(str(k) for k in g if k not in GROUP_KEYS)
        if extra:
            raise ValueError("param group %d has key %s: a group may set only 'lr' and 'weight_decay' (momentum, "
                             "betas, eps and the rest are per optimizer)" % (gi, ", ".join(repr(k) for k in extra)))
        params = [g["params"]] if isinstance(g["params"], torch.Tensor) else list(g["params"])
        if not params:
            raise ValueError("param group %d is empty" % gi)
        for p in params:
            if id(p) in crit_ids:
                raise ValueError("param group %d lists a criterion parameter: groups hold model parameters only" % gi)
            if id(p) not in model_ids:
                raise ValueError("param group %d lists a parameter that is not in model.parameters()" % gi)
            if id(p) in seen:
                raise ValueError("param group %d lists a parameter that an earlier group already holds" % gi)
            seen.add(id(p))
        group: Dict[str, Any] = {"params": params}
        for k in ("lr", "weight_decay"):
            if k in g:
                group[k] = float(g[k])
        out.append(group)
    rest = [p for p in model_params if id(p) not in seen] + [p for p in crit if id(p) not in model_ids]
    if rest:
        out.append({"params": rest})
    return out


def check_param_groups(layer_adaptation: LayerAdaptation, optimizer_state: OptimizerState, adafactor: bool,
                       muon: bool, grouped: bool) -> None:
    """Param groups (a Problem's ``get_param_groups`` hook or ``no_decay_1d``) need SGD, Adam / AdamW,
    RMSprop or Lion; LARS / LAMB (their decay exclusion is built in), 8-bit state, Adafactor and Muon
    are a ValueError naming the combination."""
    if not grouped:
        return
    why = None
    if LayerAdaptation(layer_adaptation) is not LayerAdaptation.NONE:
        why = "layer adaptation %s" % LayerAdaptation(layer_adaptation).value
    elif OptimizerState(optimizer_state) is OptimizerState.Q8:
        why = "optimizer state %s" % OptimizerState.Q8.value
    elif adafactor:
        why = "adafactor"
    elif muon:
        why = "muon"
    if why is not None:
        raise ValueError("param groups (get_param_groups / no_decay_1d) cannot be combined with %s: per-group lr and "
                         "weight decay are implemented for sgd, adam / adamw, rmsprop and lion" % why)


def check_layer_adaptation(optim_opts: OptimOpts, layer_adaptation: LayerAdaptation) -> None:
    """LARS needs the SGD rule, LAMB the Adam rule without amsgrad; anything else is a ValueError."""
    la = LayerAdaptation(layer_adaptation)
    ok = (la is LayerAdaptation.NONE
          or (la is LayerAdaptation.LARS and optim_opts.algo == OptAlgorithm.SGD)
          or (la is LayerAdaptation.LAMB and optim_opts.algo == OptAlgorithm.ADAM and not optim_opts.amsgrad))
    if not ok:
        raise ValueError("layer adaptation %r cannot be combined with optimizer %r%s (LARS needs sgd, "
                         "LAMB needs adam without amsgrad)"
                         % (la.value, getattr(optim_opts.algo, "value", optim_opts.algo),
                            " with amsgrad" if optim_opts.amsgrad else ""))


def create_fused_optimizer(arena: ParamArena, optim_opts: OptimOpts,
                           layer_adaptation: LayerAdaptation = LayerAdaptation.NONE,
                           optimizer_state: OptimizerState = OptimizerState.FP32,
                           adafactor: bool = False, muon: bool = False, adamw: bool = False,
                           lion: bool = False, param_groups: Optional[List[Dict[str, Any]]] = None
                           ) -> FusedArenaOptimizer:
    """Same dispatch and argument mapping as the reference's ``_create_optimizer``; with a layer
    adaptation, its LARS / LAMB counterpart; with 8-bit optimizer state, ``FusedAdam8bit``; with
    ``adafactor``, ``FusedAdafactor`` (``lr`` caps the relative step, ``weightDecay`` is its
    decoupled decay; ``epsilon`` and ``momentum`` are unused); with ``muon``, ``FusedMuon`` (one
    ``lr`` and ``weightDecay`` for both groups, ``momentum`` is Muon's, ``epsilon`` Adam's); with
    ``adamw``, the Adam rule of whichever of ``FusedAdam``, ``FusedAdam8bit`` or ``FusedMuon`` is
    chosen takes decoupled weight decay (``torch.optim.AdamW``); with ``lion``, ``FusedLion`` (``momentum``
    is beta1, beta2 is 0.99, ``weightDecay`` its decoupled decay).  ``param_groups``: the canonical groups
    of ``resolve_param_groups`` (SGD, Adam / AdamW, RMSprop and Lion only)."""
    check_layer_adaptation(optim_opts, layer_adaptation)
    check_optimizer_state(optim_opts, layer_adaptation, optimizer_state)
    check_adafactor(optim_opts, layer_adaptation, optimizer_state, adafactor)
    check_muon(optim_opts, layer_adaptation, optimizer_state, adafactor, muon)
    check_adamw(optim_opts, layer_adaptation, optimizer_state, adafactor, adamw)
    check_lion(optim_opts, layer_adaptation, lion)
    check_param_groups(layer_adaptation, optimizer_state, adafactor, muon, param_groups is not None)
    check_master_weights(getattr(arena, "master_weights", MasterWeights.FP32), arena.precision, layer_adaptation,
                         optimizer_state, adafactor, muon)
    if muon:
        return FusedMuon(arena, lr=optim_opts.lr, weight_decay=optim_opts.weightDecay,
                         momentum=optim_opts.momentum, eps=optim_opts.epsilon, adamw=adamw)
    if adafactor:
        return FusedAdafactor(arena, lr=optim_opts.lr, weight_decay=optim_opts.weightDecay)
    if OptimizerState(optimizer_state) is OptimizerState.Q8:
        return FusedAdam8bit(arena, lr=optim_opts.lr, weight_decay=optim_opts.weightDecay, eps=optim_opts.epsilon,
                             adamw=adamw)
    if layer_adaptation == LayerAdaptation.LARS:
        return FusedLars(arena, lr=optim_opts.lr, momentum=optim_opts.momentum,
                         weight_decay=optim_opts.weightDecay)
    if layer_adaptation == LayerAdaptation.LAMB:
        return FusedLamb(arena, lr=optim_opts.lr, weight_decay=optim_opts.weightDecay, eps=optim_opts.epsilon)
    algo = optim_opts.algo
    if algo == OptAlgorithm.RMSPROP:
        return FusedRMSprop(arena, lr=optim_opts.lr, momentum=optim_opts.momentum,
                            weight_decay=optim_opts.weightDecay, param_groups=param_groups)
    if algo == OptAlgorithm.SGD and lion:
        return FusedLion(arena, lr=optim_opts.lr, betas=(optim_opts.momentum, 0.99),
                         weight_decay=optim_opts.weightDecay, param_groups=param_groups)
    if algo == OptAlgorithm.SGD:
        return FusedSGD(arena, lr=optim_opts.lr, momentum=optim_opts.momentum,
                        weight_decay=optim_opts.weightDecay, param_groups=param_groups)
    if algo == OptAlgorithm.ADAM:
        return FusedAdam(arena, lr=optim_opts.lr, weight_decay=optim_opts.weightDecay,
                         eps=optim_opts.epsilon, amsgrad=optim_opts.amsgrad, adamw=adamw,
                         param_groups=param_groups)
    raise ValueError("Unknown optimization algorithm type")
