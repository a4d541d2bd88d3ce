"""TEST INFRASTRUCTURE — CPU restatement of the reference's per-rank training loop.

Plain PyTorch on the CPU, no import from the product package.  It restates, citing the
reference line by line, exactly the part of the reference the H100 path replaces:

    _create_optimizer            solver.py:162-188      -> make_optimizer
    create_lr_scheduler + get_lr solver.py:191-218, lr_scheduler.py:29-33, 65-78 -> lr_at_epoch
    ParallelCriterion.forward    criteria.py:42-61      -> parallel_criterion
    UncertaintyWeightedCriterion criteria.py:108-148    -> uncertainty_criterion
    GradNormWeightedCriterion    criteria.py:151-260    -> GradNormOracle
    MultiTaskModel.final_shared_params  model.py:32-50  -> final_shared_param
    MaskedLoss.forward           criteria.py:272-287    -> masked_loss
    SolverWorker._pass_one_epoch / _pass_one_minibatch   solver_worker.py:412-594 -> train
    ScaffoldSampler.__iter__ / per_node_randperm         sampler.py:17-87 -> rank_indices

The arithmetic underneath (autograd, nn losses, torch.optim, randperm, DataLoader) is the
third-party PyTorch the reference itself calls (un-pinned there; torch 2.11.0 here).

Pinned against the live reference by ``oracle/make_golden.py`` (fixtures in ``tests/golden``)
and ``tests/test_oracle_pinning.py``.
"""
import math
from bisect import bisect_right
from itertools import chain
from typing import Any, Dict, List, NamedTuple, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.nn as nn


# ----------------------------------------------------------------------------------------------
# options (plain records so the oracle does not depend on anybody's types module)
# ----------------------------------------------------------------------------------------------

class OptimSpec(NamedTuple):
    algo: str                      # "sgd" | "adam" | "rmsprop"   (types.py:57-60)
    lr: float = 0.001
    scheduler: str = "drop"        # "drop" | "multistep"          (types.py:73-75)
    weight_decay: float = 0.00001
    momentum: float = 0.9
    epsilon: float = 1e-8
    amsgrad: bool = False
    gradient_clip: float = 0.0


class RunSpec(NamedTuple):
    optim: OptimSpec
    batch_size: int
    n_epochs: int = 75


def spec_from_run_opts(run_opts) -> RunSpec:
    """Translate a scaffold ``RunOpts`` (reference's or this repo's: same field names)."""
    o = run_opts.optim
    return RunSpec(optim=OptimSpec(algo=o.algo.value, lr=o.lr, scheduler=o.lr_scheduler.algo.value,
                                   weight_decay=o.weightDecay, momentum=o.momentum,
                                   epsilon=o.epsilon, amsgrad=o.amsgrad,
                                   gradient_clip=o.gradientClip),
                   batch_size=run_opts.batchSize, n_epochs=run_opts.nEpochs)


# ----------------------------------------------------------------------------------------------
# optimizer / schedule
# ----------------------------------------------------------------------------------------------

def make_optimizer(params, o: OptimSpec) -> torch.optim.Optimizer:
    """reference solver.py:162-188 — note momentum feeds RMSprop too and eps only Adam."""
    if o.algo == "rmsprop":
        return torch.optim.RMSprop(params, lr=o.lr, momentum=o.momentum, weight_decay=o.weight_decay)
    if o.algo == "sgd":
        return torch.optim.SGD(params, lr=o.lr, momentum=o.momentum, weight_decay=o.weight_decay)
    if o.algo == "adam":
        return torch.optim.Adam(params, lr=o.lr, weight_decay=o.weight_decay, eps=o.epsilon,
                                amsgrad=o.amsgrad)
    raise ValueError("Unknown optimization algorithm type")


def lr_at_epoch(base_lr: float, epoch: int, n_epochs: int, scheduler: str) -> float:
    """Learning rate in force DURING 1-based ``epoch``.

    The scheduler is constructed with last_epoch=-1 (its constructor performs one step, so
    last_epoch = 0 during epoch 1) and stepped once after every epoch
    (solver_worker.py:790) => last_epoch = epoch - 1 during ``epoch``.
    drop:      base * 0.1 ** #{d in drops : last_epoch + 1 >= d}, drops = floor(n*.66667),
               floor(n*.9) iff n > 10                       (solver.py:195-198, lr_scheduler.py:29-33)
    multistep: milestones floor(n*{.33333,.66667,.9}), gamma .1, linear warm-up from 1e-3 over
               5 epochs                                     (solver.py:203-213, lr_scheduler.py:65-78)
    """
    last = epoch - 1
    if scheduler == "drop":
        drops = [np.floor(n_epochs * 0.66667), np.floor(n_epochs * 0.9)] if n_epochs > 10 else []
        return base_lr * 0.1 ** int(np.sum([last + 1 >= d for d in drops]))
    if scheduler == "multistep":
        miles = [np.floor(n_epochs * r) for r in (0.33333, 0.66667, 0.9)]
        wf = 1
        if last < 5:
            alpha = last / 5
            wf = (1.0 / 1000) * (1 - alpha) + alpha
        return base_lr * wf * 0.1 ** bisect_right(miles, last)
    raise ValueError("Unknown optimization algorithm type")


# ----------------------------------------------------------------------------------------------
# sampler
# ----------------------------------------------------------------------------------------------

def per_node_randperm(n: int, node_idx: int, node_count: int, generator) -> List[int]:
    """reference sampler.py:17-34."""
    target = math.ceil(n / node_count)
    start = node_idx * target
    actual = min(n - start, target)
    idx = (torch.randperm(actual, generator=generator) + target * node_idx).tolist()
    idx += idx[: target - actual]
    return idx


def rank_indices(n: int, epoch: int, rank: int, world: int, shuffle_type: str = "randperm",
                 node_idx: int = 0, node_count: int = 1) -> List[int]:
    """reference sampler.py:55-87: seed = epoch, pad with the head, stride by rank."""
    g = torch.Generator()
    g.manual_seed(epoch)
    if shuffle_type == "per_node_randperm":
        node_size = world // node_count
        return per_node_randperm(n, node_idx, node_count, g)[rank % node_size:: node_size]
    idx = torch.randperm(n, generator=g).tolist()
    num_samples = math.ceil(n / world)
    total = num_samples * world
    idx += idx[: total - len(idx)]
    return idx[rank:total:world]


# ----------------------------------------------------------------------------------------------
# criteria
# ----------------------------------------------------------------------------------------------

def masked_loss(inner, output, target, mask):
    """reference criteria.py:272-287."""
    if mask.sum() == 0:
        return inner(output - output, target - target)
    mask = mask.bool()
    return inner(output[mask], target[mask])


def _apply_loss(module, out, tgt_tuple):
    inner = getattr(module, "loss_layer", None)
    if inner is not None and len(tgt_tuple) == 2:
        return masked_loss(inner, out, tgt_tuple[0], tgt_tuple[1])
    return module(out, *tgt_tuple)


def parallel_criterion(loss_modules, weights, names, outputs, targets):
    """reference criteria.py:42-61: split[name] = w * loss(out_i, *tgt_i); total = sum()."""
    split = {}
    for i, (loss, w, name) in enumerate(zip(loss_modules, weights, names)):
        split[name] = w * _apply_loss(loss, outputs[i], targets[i])
    return sum(split.values()), split


def uncertainty_criterion(loss_modules, kinds, names, log_variance, outputs, targets):
    """reference criteria.py:108-148 (kinds: "mse" | "crossentropy")."""
    split, costs = {}, []
    for i, (loss, kind, name) in enumerate(zip(loss_modules, kinds, names)):
        raw = _apply_loss(loss, outputs[i], targets[i])
        if kind == "mse":
            split[name] = 1.0 / (2.0 * torch.exp(log_variance[i])) * raw
        else:
            split[name] = 1.0 / torch.exp(log_variance[i]) * raw
        costs.append(0.5 * log_variance[i])
    return sum(split.values()) + sum(costs), split


def final_shared_param(trunk_params: Sequence[nn.Parameter], outputs: Sequence[torch.Tensor]):
    """reference model.py:32-50: breadth-first walk from the FIRST head's grad_fn; the first
    AccumulateGrad node whose variable is a trunk parameter."""
    from queue import Queue
    todo = Queue()
    todo.put(outputs[0].grad_fn)
    while not todo.empty():
        fn = todo.get()
        for nxt, _ in fn.next_functions:
            if hasattr(nxt, "variable") and any(nxt.variable is p for p in trunk_params):
                return nxt.variable
            if nxt is not None:
                todo.put(nxt)
    raise RuntimeError("Unable to find any shared parameters in the model")


class GradNormOracle:
    """reference criteria.py:151-260, stated as a plain object: ``weight_factors`` is the
    trainable T-vector (zeros), the baseline losses are captured by the first call."""

    def __init__(self, loss_modules, names, alpha: float, base_weights=None) -> None:
        self.loss_modules, self.names, self.alpha = list(loss_modules), list(names), alpha
        self.T = len(self.loss_modules)
        self.weight_factors = nn.Parameter(torch.zeros(self.T))
        self.base_weights = base_weights or [1] * self.T
        self.baseline: Optional[List[float]] = None

    def __call__(self, outputs, targets, shared_param):
        T = self.T
        task = [self.base_weights[i] * self.loss_modules[i](outputs[i], *targets[i])      # :183-186
                for i in range(T)]
        if self.baseline is None:                                                         # :188-189
            self.baseline = [l.item() for l in task]
        inv = [task[i] / self.baseline[i] for i in range(T)]                              # :193-196
        mean_inv = sum(inv) / len(inv)
        rel = [r / mean_inv for r in inv]                                                 # :198-201
        dl = [g.detach() for g in torch.autograd.grad(task, outputs, retain_graph=True)]  # :207-212
        weights = self.weight_factors.softmax(0) * T                                      # :219
        norms = [torch.autograd.grad(outputs[i], shared_param, weights[i] * dl[i],        # :224-234
                                     retain_graph=True, create_graph=True)[0].norm()
                 for i in range(T)]
        mean_norm = sum(norms) / len(norms)                                               # :239
        wanted = [mean_norm * (r ** self.alpha) for r in rel]                             # :240-243
        grad_loss = sum(torch.nn.functional.l1_loss(n, w.detach())                        # :244-248
                        for n, w in zip(norms, wanted))
        weighted = [weights[i].detach() * task[i] for i in range(T)]                      # :253-256
        return sum(weighted) + grad_loss, dict(zip(self.names, task))                     # :258-260


# ----------------------------------------------------------------------------------------------
# the loop
# ----------------------------------------------------------------------------------------------

def reference_minibatch(model, criterion_fn, opt, model_params, gradient_clip, data, target,
                        training=True):
    """One pass of SolverWorker._pass_one_minibatch (solver_worker.py:533-594) on the CPU:
    forward, criterion, NaN guard, zero_grad, backward, optional clip, optimizer step."""
    output = model(data)
    total, sub = criterion_fn(output, target)
    if torch.isnan(total).any():
        raise FloatingPointError("Losses become NaN")
    if training:
        opt.zero_grad()
        total.backward()
        if gradient_clip:
            torch.nn.utils.clip_grad_norm_(model_params, gradient_clip)
        opt.step()
    return output, total, sub


class Trace(NamedTuple):
    losses: Dict[Tuple[int, str], np.ndarray]     # (epoch, split) -> [n_minibatch, 1+T] fp32
    indices: Dict[Tuple[int, str], List[int]]     # (epoch, split) -> sample ids in trained order
    lrs: List[float]                              # lr in force during each epoch
    first_grads: Optional[List[np.ndarray]]       # model grads at the very first training step
    params: List[np.ndarray]                      # model parameters after the last epoch
    loss_names: List[str]


def train(model: nn.Module, loss_modules: Sequence[nn.Module], loss_weights: Sequence[float],
          loss_names: Sequence[str], datasets: Sequence[Tuple[str, Any]], spec: RunSpec,
          extra_params: Sequence[nn.Parameter] = (), criterion_fn=None,
          max_steps: Optional[int] = None, device: Optional[torch.device] = None) -> Trace:
    """Restatement of SolverWorker.train on one CPU rank (world_size 1).

    ``datasets``: ``[(split_name, torch Dataset)]`` in Problem order; the split named
    "training" is trained on, every other split is evaluated (forward + loss only) —
    solver_worker.py:427-442.  Every split is shuffled with a RandomSampler and the planned
    order is drawn once before iterating (solver_worker.py:431, 824-831), which consumes the
    global RNG exactly as the reference does.

    ``device``: run the very same stock-PyTorch loop on that device instead of the CPU (the
    reference's own GPU path minus DDP: ``model.to(device)`` before the optimizer is built,
    batches moved per step, solver.py:304-310, solver_worker.py:465-469) — used where CPU-vs-GPU
    convolution rounding would drown what a test wants to see.
    """
    if device is not None:
        model.to(device)
        for m in loss_modules or ():
            m.to(device)
    params = list(chain(model.parameters(), extra_params))
    opt = make_optimizer(params, spec.optim)
    model_params = list(model.parameters())
    loaders = {name: torch.utils.data.DataLoader(ds, batch_size=spec.batch_size, shuffle=True,
                                                 num_workers=0, pin_memory=False)
               for name, ds in datasets}
    if criterion_fn is None:
        def criterion_fn(outputs, targets):
            return parallel_criterion(loss_modules, loss_weights, loss_names, outputs, targets)

    losses, indices, lrs = {}, {}, []
    first_grads = None
    steps = 0
    for epoch in range(1, spec.n_epochs + 1):
        lr = lr_at_epoch(spec.optim.lr, epoch, spec.n_epochs, spec.optim.scheduler)
        for group in opt.param_groups:
            group["lr"] = lr
        lrs.append(lr)
        for split, loader in loaders.items():
            list(iter(loader.sampler))                     # planned order for the cache (:431)
            training = split == "training"
            model.train(training)
            rows, order = [], []
            for data, target, meta in loader:
                if "index" in meta:
                    order += [int(i) for i in meta["index"]]
                if device is not None:                     # (:465-469)
                    data = [t.to(device) for t in data]
                    target = [tuple(t.to(device) for t in head) for head in target]
                output = model(data)                       # (:551) data is a List[Tensor]
                total, sub = criterion_fn(output, target)  # (:567)
                if torch.isnan(total).any():               # (:569-573)
                    raise FloatingPointError(
                        "Losses become NaN for dataset {} at iteration {} minibatch {}!".format(
                            split, epoch, len(rows)))
                if training:
                    opt.zero_grad()                        # (:585)
                    total.backward()                       # (:586)
                    if first_grads is None:
                        first_grads = [p.grad.detach().cpu().clone().numpy() for p in model_params]
                    if spec.optim.gradient_clip:           # (:588-591) model params only
                        torch.nn.utils.clip_grad_norm_(model_params, spec.optim.gradient_clip)
                    opt.step()                             # (:592)
                    steps += 1
                rows.append([total.item()] + [sub[n].item() for n in loss_names])
                if max_steps is not None and steps >= max_steps:
                    break
            losses[(epoch, split)] = np.asarray(rows, dtype=np.float32)
            indices[(epoch, split)] = order
            if max_steps is not None and steps >= max_steps:
                break
        if max_steps is not None and steps >= max_steps:
            break
    return Trace(losses=losses, indices=indices, lrs=lrs, first_grads=first_grads,
                 params=[p.detach().cpu().clone().numpy() for p in model_params],
                 loss_names=list(loss_names))
