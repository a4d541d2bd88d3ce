"""Lion against SGD with momentum and AdamW through ``Solver.build_worker`` on one GPU, in one process,
the three arms alternating: 5 rounds of 50 steps each (after 10 warm-up steps per arm), median
(min-max) over the rounds.

* ``sgd``: SGD, momentum 0.9, lr 1e-2, weight decay 1e-5; the trunk's weights take their update in
  the dW GEMM (K12, ``frl_dw_gemm_sgd``), the rest one tail ``frl_sgd_momentum``.
* ``lion``: the same options with ``lion=True`` (beta1 0.9, beta2 0.99), lr 1e-4: K12 runs
  ``frl_dw_gemm_lion``, the tail ``frl_lion``.
* ``adamw``: Adam, lr 1e-3, decoupled weight decay 1e-5 (``frl_adamw``; K12 does not apply).

The workload is the headline MLP (3 x Linear(4096, 4096) trunk, heads 1000 + 64), batch 4096, bf16,
inputs resident in HBM, the step replayed from a CUDA graph.  Step time from CUDA events around each
round.  Resident memory of an arm: ``torch.cuda.memory_allocated()`` after its warm-up steps (state
vectors and graph pool included) less before its build, with the shared input pool already allocated.

The card's name, power limit and max SM clock are read in the same run and printed with the table.

    python tools/bench_lion.py [--rounds 5] [--steps 50] [--json out.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import torch  # noqa: E402

import frl_b200  # noqa: E402,F401
from frl_b200 import synthetic  # noqa: E402
from frl_b200.solver import Solver, SolverWorkerArgs  # noqa: E402
from frl_b200.types import Device, Precision  # noqa: E402

DEV = torch.device("cuda", 0)
ARMS = ("sgd", "lion", "adamw")
BATCH = 4096


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                              "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = "nvidia-smi unavailable (%s)" % e
    return out or torch.cuda.get_device_name(0)


def build(arm):
    ns = synthetic.api_namespace("frl_b200")
    t = ns.types
    save_dir = tempfile.mkdtemp(prefix="frl_b200_bench_lion_")
    torch.manual_seed(0)
    problem = synthetic.make_mlp_problem(ns, save_dir, n_train=64, width=4096, n_classes=1000, reg_dim=64, depth=3)
    algo = t.OptAlgorithm.ADAM if arm == "adamw" else t.OptAlgorithm.SGD
    lr = {"sgd": 1e-2, "lion": 1e-4, "adamw": 1e-3}[arm]
    run_opts = t.RunOpts(optim=t.OptimOpts(algo=algo, lr=lr, momentum=0.9, weightDecay=1e-5),
                         batchSize=BATCH, nEpochs=1, numThreads=0, singleThreaded=True, numVisualizedSamples=0)
    args = SolverWorkerArgs(run_opts=run_opts, problem=problem, save_dir=save_dir, run_device=Device.GPU,
                            node_idx=0, node_count=1, rank=0, local_rank=0, world_size=1, group_name=None,
                            init_method="", precision=Precision.BF16, graph_step=True, adamw=arm == "adamw",
                            lion=arm == "lion")
    worker, _, _ = Solver.build_worker(args)
    worker.model.train()
    worker.criterion.train()
    assert worker.pipeline.fused_dw_update == (arm != "adamw")
    return worker


def batches(gen, n=4):
    out = []
    for _ in range(n):
        x = torch.randn(BATCH, 4096, device=DEV, generator=gen)
        out.append(([x], [(torch.randint(0, 1000, (BATCH,), device=DEV, generator=gen),),
                          (torch.randn(BATCH, 64, device=DEV, generator=gen),)]))
    return out


def run(worker, pool, i0, k):
    from frl_b200.types import Split
    for i in range(i0, i0 + k):
        data, target = pool[i % len(pool)]
        worker._pass_one_minibatch(i, Split.TRAIN, data, target)


def fmt(xs):
    return "%.3f (%.3f-%.3f)" % (statistics.median(xs), min(xs), max(xs))


def bench(rounds, steps, warmup):
    gen = torch.Generator(device=DEV).manual_seed(1234)
    pool = batches(gen)
    workers, resident = {}, {}
    for arm in ARMS:
        torch.cuda.synchronize()
        m0 = torch.cuda.memory_allocated()
        workers[arm] = build(arm)
        run(workers[arm], pool, 0, warmup)
        torch.cuda.synchronize()
        resident[arm] = (torch.cuda.memory_allocated() - m0) / 2 ** 20
    step_ms = {arm: [] for arm in ARMS}
    pos = {arm: warmup for arm in ARMS}
    for _ in range(rounds):
        for arm in ARMS:
            w = workers[arm]
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            run(w, pool, pos[arm], steps)
            e1.record()
            torch.cuda.synchronize()
            step_ms[arm].append(e0.elapsed_time(e1) / steps)
            pos[arm] += steps
    out = {}
    for arm in ARMS:
        out[arm] = {"step_ms": step_ms[arm], "step_median_ms": statistics.median(step_ms[arm]),
                    "resident_mib": resident[arm]}
        print("mlp %-6s step %s ms  resident %.1f MiB" % (arm, fmt(step_ms[arm]), resident[arm]), flush=True)
    med = {arm: out[arm]["step_median_ms"] for arm in ARMS}
    out["goals"] = {"lion_over_sgd_step": med["lion"] / med["sgd"],
                    "lion_step_within_1.03x_sgd": med["lion"] <= 1.03 * med["sgd"],
                    "lion_step_below_adamw": med["lion"] < med["adamw"],
                    "adamw_minus_lion_resident_mib": resident["adamw"] - resident["lion"]}
    print(json.dumps(out["goals"]), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_lion.py measures on a GPU; none is visible")
    torch.cuda.set_device(0)
    result = {"card": card(), "torch": torch.__version__}
    print("card:", result["card"], flush=True)
    result["mlp"] = bench(args.rounds, args.steps, args.warmup)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
