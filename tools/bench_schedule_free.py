"""Schedule-Free AdamW / SGD against AdamW and SGD with momentum through ``Solver.build_worker`` on one GPU:
the headline MLP step, the four arms alternating in one process, 5 rounds of 50 steps each (after 10
warm-up steps per arm), median (min-max) over the rounds.

* ``adamw``: Adam, lr 1e-3, decoupled weight decay 1e-5 (``frl_adamw``).
* ``sf_adamw``: the same options with ``schedule_free=True`` (``frl_sf_adamw``).
* ``sgd``: SGD, momentum 0.9, lr 1e-2, weight decay 1e-5; the trunk's weights take their update in the
  dW GEMM (K12), the rest one tail ``frl_sgd_momentum``.
* ``sf_sgd``: the same options with ``schedule_free=True`` (``frl_sf_sgd``; K12 does not apply, so this
  arm shows what Schedule-Free SGD gives up against K12).

The workload is the headline MLP (3 x Linear(4096, 4096) trunk, heads 1000 + 64), batch 4096, bf16,
inputs resident in HBM, the step replayed from a CUDA graph.  Step time from CUDA events around each
round.  Resident and peak memory of each arm are read in a fresh process of their own (``--memory ARM``):
``torch.cuda.memory_allocated()`` after 10 steps, and ``torch.cuda.max_memory_allocated()``.  One
held-out swap (x into the bf16 shadow and back, ``FusedScheduleFree.swapped()``) of the ``sf_adamw``
worker is timed with CUDA events, median of 20.

The card's name, power limit and max SM clock are read in the same run and printed with the table.

    python tools/bench_schedule_free.py [--rounds 5] [--steps 50] [--json out.json]
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
from frl_b200.types import Device, Precision, ScheduleFree, Split  # noqa: E402

DEV = torch.device("cuda", 0)
ARMS = ("adamw", "sf_adamw", "sgd", "sf_sgd")
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
    save_dir = tempfile.mkdtemp(prefix="frl_b200_bench_sf_")
    torch.manual_seed(0)
    problem = synthetic.make_mlp_problem(ns, save_dir, n_train=64, width=4096, n_classes=1000, reg_dim=64, depth=3)
    adam = arm in ("adamw", "sf_adamw")
    run_opts = t.RunOpts(optim=t.OptimOpts(algo=t.OptAlgorithm.ADAM if adam else t.OptAlgorithm.SGD,
                                           lr=1e-3 if adam else 1e-2, momentum=0.9, weightDecay=1e-5),
                         batchSize=BATCH, nEpochs=1, numThreads=0, singleThreaded=True, numVisualizedSamples=0)
    args = SolverWorkerArgs(run_opts=run_opts, problem=problem, save_dir=save_dir, run_device=Device.GPU,
                            node_idx=0, node_count=1, rank=0, local_rank=0, world_size=1, group_name=None,
                            init_method="", precision=Precision.BF16, graph_step=True, adamw=arm == "adamw",
                            schedule_free=ScheduleFree() if arm.startswith("sf_") else None)
    worker, _, _ = Solver.build_worker(args)
    worker.model.train()
    worker.criterion.train()
    assert worker.pipeline.fused_dw_update == (arm == "sgd")
    return worker


def batches(gen, n=4):
    out = []
    for _ in range(n):
        x = torch.randn(BATCH, 4096, device=DEV, generator=gen)
        out.append(([x], [(torch.randint(0, 1000, (BATCH,), device=DEV, generator=gen),),
                          (torch.randn(BATCH, 64, device=DEV, generator=gen),)]))
    return out


def run(worker, pool, i0, k):
    for i in range(i0, i0 + k):
        data, target = pool[i % len(pool)]
        worker._pass_one_minibatch(i, Split.TRAIN, data, target)


def fmt(xs):
    return "%.3f (%.3f-%.3f)" % (statistics.median(xs), min(xs), max(xs))


def memory(arm, warmup):
    """Resident and peak MiB of one arm, alone in this process."""
    pool = batches(torch.Generator(device=DEV).manual_seed(1234))
    torch.cuda.synchronize()
    m0 = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    w = build(arm)
    run(w, pool, 0, warmup)
    torch.cuda.synchronize()
    return {"arm": arm, "resident_mib": (torch.cuda.memory_allocated() - m0) / 2 ** 20,
            "peak_mib": (torch.cuda.max_memory_allocated() - m0) / 2 ** 20}


def memory_in_fresh_process(arm, warmup):
    res = subprocess.run([sys.executable, os.path.abspath(__file__), "--memory", arm, "--warmup", str(warmup)],
                         capture_output=True, text=True, timeout=900)
    lines = [ln for ln in res.stdout.splitlines() if ln.startswith("{")]
    if res.returncode != 0 or not lines:
        raise RuntimeError("memory run of %s failed:\n%s" % (arm, res.stderr[-3000:]))
    return json.loads(lines[-1])


def swap_ms(worker, n=20):
    times = []
    for _ in range(n + 2):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        with worker.optimizer.swapped():
            pass
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
    return times[2:]


def bench(rounds, steps, warmup):
    gen = torch.Generator(device=DEV).manual_seed(1234)
    pool = batches(gen)
    workers = {}
    for arm in ARMS:
        workers[arm] = build(arm)
        run(workers[arm], pool, 0, warmup)
    torch.cuda.synchronize()
    step_ms = {arm: [] for arm in ARMS}
    pos = {arm: warmup for arm in ARMS}
    for _ in range(rounds):
        for arm in ARMS:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            run(workers[arm], pool, pos[arm], steps)
            e1.record()
            torch.cuda.synchronize()
            step_ms[arm].append(e0.elapsed_time(e1) / steps)
            pos[arm] += steps
    swap = swap_ms(workers["sf_adamw"])
    del workers
    torch.cuda.empty_cache()
    out = {}
    for arm in ARMS:
        mem = memory_in_fresh_process(arm, warmup)
        out[arm] = {"step_ms": step_ms[arm], "step_median_ms": statistics.median(step_ms[arm]), **mem}
        print("mlp %-8s step %s ms  resident %.1f MiB  peak %.1f MiB"
              % (arm, fmt(step_ms[arm]), mem["resident_mib"], mem["peak_mib"]), flush=True)
    print("held-out swap in and out (sf_adamw, bf16 shadow): %s ms" % fmt(swap), flush=True)
    med = {arm: out[arm]["step_median_ms"] for arm in ARMS}
    out["swap_ms"] = swap
    out["goals"] = {"sf_adamw_over_adamw_step": med["sf_adamw"] / med["adamw"],
                    "sf_adamw_step_within_1.03x": med["sf_adamw"] <= 1.03 * med["adamw"],
                    "sf_adamw_minus_adamw_resident_mib": out["sf_adamw"]["resident_mib"] - out["adamw"]["resident_mib"],
                    "sf_sgd_minus_sgd_resident_mib": out["sf_sgd"]["resident_mib"] - out["sgd"]["resident_mib"],
                    "sf_sgd_over_sgd_with_k12_step": med["sf_sgd"] / med["sgd"]}
    print(json.dumps(out["goals"]), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--memory", choices=ARMS, default=None, help=argparse.SUPPRESS)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_schedule_free.py measures on a GPU; none is visible")
    torch.cuda.set_device(0)
    if args.memory:
        print(json.dumps(memory(args.memory, args.warmup)), flush=True)
        return
    result = {"card": card(), "torch": torch.__version__}
    print("card:", result["card"], flush=True)
    result["mlp"] = bench(args.rounds, args.steps, args.warmup)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
