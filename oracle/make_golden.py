"""TEST INFRASTRUCTURE — generate ``tests/golden/*`` from the LIVE, unmodified reference.

Runs only in the build container (needs ``/root/reference``):

    python -m oracle.make_golden

For every configuration below the reference's own ``LocalSolver.solve`` is run on the CPU
(``cpuonly, singleThreaded, numThreads=0``) on the synthetic toy Problem (the very class
definitions of ``frl_b200.synthetic`` instantiated against the reference's API namespace), with
``SolverWorker._pass_one_minibatch`` wrapped to record per-step losses, the learning rate, the
first gradients; final parameters come from the ``final_model.pth`` the reference writes.
The same run is then repeated with ``oracle/ref_loop.train`` and must agree bit-for-bit on the
losses/parameters (same machine, same torch) — that is what pins the restatement.
Also dumps sampler index lists and learning-rate tables computed by the reference's classes.
"""
import json
import os
import shutil
import sys
import tempfile

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
GOLDEN_DIR = os.path.join(REPO, "tests", "golden")

from oracle import ref_loop                      # noqa: E402
from oracle.ref_shim import import_reference     # noqa: E402

CONFIGS = {
    # name: (algo, lr, scheduler, nEpochs, clip, amsgrad, criterion_kind)
    # lr 0.008, not 0.01: at 0.01 a trunk pre-activation of the second epoch is 7e-9 against terms
    # summing to 0.79 in magnitude (1e-8 relative, below fp32 resolution), so its ReLU decision,
    # and with it 32 first-layer weights, depends on the summation order of the GEMM.  The
    # smallest one left (shared by every toy configuration: the first forward, trunk layer 2,
    # sample 55, unit 8) is 8.9e-8 against 0.79, about one fp32 ulp of the sum: a future
    # divergence confined to one trunk unit should be looked for there first
    "toy_sgd": ("sgd", 0.008, "drop", 2, 0.0, False, "parallel"),
    "toy_adam_clip": ("adam", 0.003, "multistep", 3, 1.0, False, "parallel"),
    "toy_adam_amsgrad": ("adam", 0.003, "drop", 2, 0.0, True, "parallel"),
    "toy_rmsprop": ("rmsprop", 0.0005, "drop", 2, 0.0, False, "parallel"),
    "toy_uncertainty": ("sgd", 0.01, "drop", 2, 0.0, False, "uncertainty"),
    "toy_gradnorm": ("sgd", 0.01, "drop", 2, 0.0, False, "gradnorm"),
}
SEED = 0
BATCH = 64


def _run_opts(ns, algo, lr, sched, n_epochs, clip, amsgrad):
    t = ns.types
    optim = t.OptimOpts(algo=t.OptAlgorithm(algo), lr=lr,
                        lr_scheduler=t.LRSchedulerOpts(algo=t.LRSchedulerAlgorithm(sched)),
                        gradientClip=clip, amsgrad=amsgrad)
    return t.RunOpts(optim=optim, batchSize=BATCH, cpuonly=True, nEpochs=n_epochs, numThreads=0,
                     singleThreaded=True, minibatchTimeoutMs=600000, numVisualizedSamples=4)


def run_live_reference(name, cfg):
    """-> dict of arrays recorded from the reference Solver itself."""
    import frl_b200  # noqa: F401  (only for the synthetic Problem definitions)
    from frl_b200 import synthetic
    import_reference()
    ns = synthetic.api_namespace("frldistml.scaffold")
    from frldistml.scaffold import solver_worker as ref_sw
    from frldistml.scaffold.local_solver import LocalSolver

    algo, lr, sched, n_epochs, clip, amsgrad, kind = cfg
    save_dir = tempfile.mkdtemp(prefix="frl_golden_")
    problem = synthetic.make_toy_problem(ns, save_dir, criterion_kind=kind)
    run_opts = _run_opts(ns, algo, lr, sched, n_epochs, clip, amsgrad)

    rec = {"rows": [], "lr": [], "split": [], "epoch": [], "first_grads": None}
    orig = ref_sw.SolverWorker._pass_one_minibatch

    def wrapped(self, minibatch_idx, data_type, data, target):
        out = orig(self, minibatch_idx, data_type, data, target)
        _, total, sub, _ = out
        rec["rows"].append([total.item()] + [sub[n].item() for n in self.criterion.loss_names])
        rec["lr"].append(self.optimizer.param_groups[0]["lr"])
        rec["split"].append(data_type.value)
        rec["epoch"].append(self.cur_epoch)
        if rec["first_grads"] is None and self.model.training and clip == 0.0:
            rec["first_grads"] = [p.grad.detach().clone().numpy() for p in self.model.parameters()]
        return out

    ref_sw.SolverWorker._pass_one_minibatch = wrapped
    try:
        torch.manual_seed(SEED)
        LocalSolver.solve(run_opts, problem)
    finally:
        ref_sw.SolverWorker._pass_one_minibatch = orig

    final = torch.load(os.path.join(save_dir, "final_model.pth"), weights_only=False)
    out = {"rows": np.asarray(rec["rows"], dtype=np.float32),
           "lr": np.asarray(rec["lr"], dtype=np.float64),
           "epoch": np.asarray(rec["epoch"], dtype=np.int64),
           "is_train": np.asarray([s == "training" for s in rec["split"]]),
           "served_train": np.asarray(problem.datasets[0].served, dtype=np.int64),
           "served_test": np.asarray(problem.datasets[1].served, dtype=np.int64)}
    for i, (k, v) in enumerate(final["state_dict"].items()):
        out["param_%02d" % i] = v.numpy()
    if rec["first_grads"] is not None:
        for i, g in enumerate(rec["first_grads"]):
            out["grad_%02d" % i] = g
    out["param_names"] = np.asarray(list(final["state_dict"].keys()))
    shutil.rmtree(save_dir, ignore_errors=True)
    return out


def run_oracle(name, cfg):
    """Same configuration through oracle/ref_loop.py (no scaffold package on the path of the
    arithmetic; the synthetic Problem only supplies model, loss modules and datasets)."""
    import frl_b200  # noqa: F401
    from frl_b200 import synthetic
    ns = synthetic.api_namespace("frl_b200")
    algo, lr, sched, n_epochs, clip, amsgrad, kind = cfg
    problem = synthetic.make_toy_problem(ns, "/tmp/unused", criterion_kind=kind)
    spec = ref_loop.RunSpec(optim=ref_loop.OptimSpec(algo=algo, lr=lr, scheduler=sched,
                                                     gradient_clip=clip, amsgrad=amsgrad),
                            batch_size=BATCH, n_epochs=n_epochs)
    torch.manual_seed(SEED)
    model = problem.get_model()
    crit = problem.get_criterion()
    datasets = [(d.data_type.value, d) for d in problem.datasets]
    if kind == "uncertainty":
        kinds = [k.value for k in crit.loss_types]

        def criterion_fn(outputs, targets):
            return ref_loop.uncertainty_criterion(list(crit.loss_modules), kinds, crit.loss_names,
                                                  crit.log_variance, outputs, targets)
        return ref_loop.train(model, None, None, crit.loss_names, datasets, spec,
                              extra_params=[crit.log_variance], criterion_fn=criterion_fn), problem
    if kind == "gradnorm":
        # reference solver_worker.py:551-567: the loop looks up the last shared trunk parameter
        # on every minibatch and hands it to the criterion before calling it
        gn = ref_loop.GradNormOracle(list(crit._loss_modules), crit.loss_names, crit._alpha,
                                     list(crit._base_weights))
        trunk = list(model.model_base.parameters())

        def criterion_fn(outputs, targets):
            return gn(outputs, targets, ref_loop.final_shared_param(trunk, outputs))
        return ref_loop.train(model, None, None, crit.loss_names, datasets, spec,
                              extra_params=[gn.weight_factors], criterion_fn=criterion_fn), problem
    return ref_loop.train(model, list(crit.loss_modules), list(crit.loss_weights),
                          list(crit.loss_names), datasets, spec), problem


def sampler_goldens():
    import_reference()
    from frldistml.scaffold.sampler import ScaffoldSampler
    from frldistml.scaffold.types import ShuffleType
    import torch.distributed as dist
    out = {}
    cases = [("randperm", 10, 4, 1), ("randperm", 1000, 8, 1), ("randperm", 17, 2, 1),
             ("per_node_randperm", 11, 4, 2), ("per_node_randperm", 100, 8, 2)]
    real = (dist.get_world_size, dist.get_rank)
    try:
        for kind, n, world, nodes in cases:
            for epoch in (1, 2):
                per_rank = []
                for rank in range(world):
                    dist.get_world_size = lambda *a, **k: world
                    dist.get_rank = lambda *a, **k: rank
                    node_size = world // nodes
                    s = ScaffoldSampler(list(range(n)), shuffle_type=ShuffleType(kind),
                                        node_idx=rank // node_size, node_count=nodes)
                    s.set_epoch(epoch)
                    per_rank.append(list(iter(s)))
                out["%s_n%d_w%d_nodes%d_e%d" % (kind, n, world, nodes, epoch)] = per_rank
    finally:
        dist.get_world_size, dist.get_rank = real
    return out


def lr_goldens():
    import_reference()
    from frldistml.scaffold.solver import create_lr_scheduler
    from frldistml.scaffold import types as t
    out = {}
    for sched in ("drop", "multistep"):
        for n_epochs in (2, 10, 12, 75):
            opt = torch.optim.SGD([torch.nn.Parameter(torch.zeros(1))], lr=0.1)
            ro = t.RunOpts(optim=t.OptimOpts(algo=t.OptAlgorithm.SGD, lr=0.1,
                                             lr_scheduler=t.LRSchedulerOpts(
                                                 algo=t.LRSchedulerAlgorithm(sched))),
                           batchSize=1, nEpochs=n_epochs)
            sch = create_lr_scheduler(ro, opt)
            lrs = []
            for _ in range(n_epochs):
                lrs.append(opt.param_groups[0]["lr"])
                opt.step()
                sch.step()
            out["%s_n%d" % (sched, n_epochs)] = lrs
    # the reference's own known-answer test (tests/test_solver.py:17-34): resume at epoch 60
    opt = torch.optim.Adam({torch.Tensor()}, lr=0.01, weight_decay=0.0001, eps=1e-8)
    opt.param_groups[0]["initial_lr"] = 0.01
    ro = t.RunOpts(nEpochs=75, mode=t.Mode.TRAIN, batchSize=16,
                   optim=t.OptimOpts(lr=0.01, algo=t.OptAlgorithm.ADAM))
    create_lr_scheduler(ro, opt, 60)
    out["kat_resume60_adam_lr0.01_n75"] = [opt.param_groups[0]["lr"]]
    return out


def main(only=()):
    """``python -m oracle.make_golden [config ...]``: regenerate everything, or only the named
    configurations (their entries are merged into the existing pinning report)."""
    os.makedirs(GOLDEN_DIR, exist_ok=True)
    report = {}
    report_path = os.path.join(GOLDEN_DIR, "pinning_report.json")
    if only and os.path.exists(report_path):
        report = json.load(open(report_path))["configs"]
    for name, cfg in CONFIGS.items():
        if only and name not in only:
            continue
        live = run_live_reference(name, cfg)
        trace, problem = run_oracle(name, cfg)
        rows = np.concatenate([trace.losses[k] for k in sorted(
            trace.losses, key=lambda ek: (ek[0], 0 if ek[1] == "training" else 1))])
        same_rows = bool(np.array_equal(rows, live["rows"]))
        n_param = len([k for k in live if k.startswith("param_") and k != "param_names"])
        same_params = all(np.array_equal(trace.params[i], live["param_%02d" % i])
                          for i in range(n_param))
        same_idx = (list(live["served_train"]) == sum(
            (trace.indices[k] for k in sorted(trace.indices) if k[1] == "training"), []))
        report[name] = {"config": list(cfg), "oracle_rows_bit_equal": same_rows,
                        "oracle_params_bit_equal": bool(same_params),
                        "oracle_indices_equal": bool(same_idx),
                        "n_steps": int(len(live["rows"])),
                        "max_abs_row_diff": float(np.max(np.abs(rows - live["rows"])))}
        print(name, report[name])
        np.savez_compressed(os.path.join(GOLDEN_DIR, name + ".npz"), **live)
    if not only:
        with open(os.path.join(GOLDEN_DIR, "samplers.json"), "w") as f:
            json.dump(sampler_goldens(), f)
        with open(os.path.join(GOLDEN_DIR, "lr_schedules.json"), "w") as f:
            json.dump(lr_goldens(), f)
    with open(report_path, "w") as f:
        json.dump({"torch": torch.__version__, "seed": SEED, "batch": BATCH, "configs": report},
                  f, indent=1)


if __name__ == "__main__":
    main(tuple(sys.argv[1:]))
