"""Step time with the ``no_decay_1d`` switch off and on, through ``Solver.build_worker`` on one GPU, in one
process, the two arms of each workload alternating: 5 rounds of 50 steps each (after 10 warm-up steps
per arm), median (min-max) over the rounds.

* ``mlp sgd``: the headline MLP (3 x Linear(4096, 4096) trunk, heads 1000 + 64), batch 4096, bf16,
  inputs resident in HBM, the step replayed from a CUDA graph; SGD, momentum 0.9, lr 1e-2, weight
  decay 1e-5.  Off: K12 for the trunk's weights and one tail ``frl_sgd_momentum``; on: K12 with each
  weight's group row and one tail ``frl_sgd_momentum_mt_grouped``.
* ``mlp adamw``: the same MLP with AdamW, lr 1e-3, weight decay 1e-5 (off: ``frl_adamw``; on:
  ``frl_adamw_mt_grouped``).
* ``resnet18`` (SGD) and ``resnet50x4`` (Adam, as ``tools/bench_channels_last.py`` runs it): batch 256, 224 x 224 uint8 images through the device
  transform, bf16, channels_last, eager launches (``tools/bench_channels_last.py``'s workers).

Step time from CUDA events around each round.  The card's name, power limit and max SM clock are
read in the same run and printed with the table.  The target is switch on <= 1.02 x off.

    python tools/bench_param_groups.py [--rounds 5] [--steps 50] [--only mlp,resnet] [--json out.json]
"""
import argparse
import json
import os
import statistics
import sys
import tempfile

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tools"))

import torch  # noqa: E402

import frl_b200  # noqa: E402,F401
from frl_b200 import synthetic  # noqa: E402
from frl_b200.solver import Solver, SolverWorkerArgs  # noqa: E402
from frl_b200.types import Device, Precision, Split  # noqa: E402

DEV = torch.device("cuda", 0)
BATCH = 4096


def card():
    from bench_lion import card as read_card
    return read_card()


def mlp_worker(rule, no_decay):
    ns = synthetic.api_namespace("frl_b200")
    t = ns.types
    save_dir = tempfile.mkdtemp(prefix="frl_b200_bench_groups_")
    torch.manual_seed(0)
    problem = synthetic.make_mlp_problem(ns, save_dir, n_train=64, width=4096, n_classes=1000, reg_dim=64, depth=3)
    algo = t.OptAlgorithm.ADAM if rule == "adamw" else t.OptAlgorithm.SGD
    run_opts = t.RunOpts(optim=t.OptimOpts(algo=algo, lr=1e-3 if rule == "adamw" else 1e-2, momentum=0.9,
                                           weightDecay=1e-5),
                         batchSize=BATCH, nEpochs=1, numThreads=0, singleThreaded=True, numVisualizedSamples=0)
    args = SolverWorkerArgs(run_opts=run_opts, problem=problem, save_dir=save_dir, run_device=Device.GPU,
                            node_idx=0, node_count=1, rank=0, local_rank=0, world_size=1, group_name=None,
                            init_method="", precision=Precision.BF16, graph_step=True, adamw=rule == "adamw",
                            no_decay_1d=no_decay)
    worker, _, _ = Solver.build_worker(args)
    worker.model.train()
    worker.criterion.train()
    assert worker.optimizer.grouped == no_decay
    gen = torch.Generator(device=DEV).manual_seed(1234)
    pool = []
    for _ in range(4):
        x = torch.randn(BATCH, 4096, device=DEV, generator=gen)
        pool.append(([x], [(torch.randint(0, 1000, (BATCH,), device=DEV, generator=gen),),
                           (torch.randn(BATCH, 64, device=DEV, generator=gen),)]))
    state = {"i": 0}

    def step():
        data, target = pool[state["i"] % len(pool)]
        worker._pass_one_minibatch(state["i"], Split.TRAIN, data, target)
        state["i"] += 1
    return worker, step


def resnet_worker(model, no_decay):
    import bench_channels_last as bcl
    # bench_channels_last builds its args without the switch, which the worker then reads from
    # FRL_B200_NO_DECAY_1D
    os.environ["FRL_B200_NO_DECAY_1D"] = "1" if no_decay else "0"
    try:
        worker, step = bcl.make_worker(model, channels_last=True, graph=False)
    finally:
        os.environ.pop("FRL_B200_NO_DECAY_1D", None)
    assert worker.optimizer.grouped == no_decay
    return worker, step


def fmt(xs):
    return "%.3f (%.3f-%.3f)" % (statistics.median(xs), min(xs), max(xs))


def bench(name, make, rounds, steps, warmup):
    arms = {}
    for no_decay in (False, True):
        worker, step = make(no_decay)
        for _ in range(warmup):
            step()
        arms[no_decay] = (worker, step)
    torch.cuda.synchronize()
    ms = {False: [], True: []}
    for _ in range(rounds):
        for no_decay in (False, True):
            step = arms[no_decay][1]
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(steps):
                step()
            e1.record()
            torch.cuda.synchronize()
            ms[no_decay].append(e0.elapsed_time(e1) / steps)
    off, on = statistics.median(ms[False]), statistics.median(ms[True])
    groups = len(arms[True][0].optimizer.param_groups)
    print("%-18s switch off %s ms  on (%d groups) %s ms  on / off %.4f" % (name, fmt(ms[False]), groups, fmt(ms[True]),
                                                                         on / off), flush=True)
    del arms
    torch.cuda.empty_cache()
    return {"off_ms": ms[False], "on_ms": ms[True], "on_over_off": on / off, "within_1.02": on <= 1.02 * off,
            "groups_on": groups}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--only", default="mlp,resnet")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_param_groups.py measures on a GPU; none is visible")
    torch.cuda.set_device(0)
    result = {"card": card(), "torch": torch.__version__}
    print("card: %s" % result["card"], flush=True)
    only = args.only.split(",")
    if "mlp" in only:
        for rule in ("sgd", "adamw"):
            result["mlp_" + rule] = bench("mlp " + rule, lambda nd, r=rule: mlp_worker(r, nd), args.rounds,
                                          args.steps, args.warmup)
    if "resnet" in only:
        for model in ("resnet18", "resnet50x4"):
            result[model] = bench(model, lambda nd, m=model: resnet_worker(m, nd), args.rounds, args.steps,
                                  args.warmup)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
