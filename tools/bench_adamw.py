"""AdamW against Adam through ``Solver.build_worker`` on one GPU, in one process, the two arms
alternating: 5 rounds of 50 steps each (after 10 warm-up steps per arm), median (min-max) over the
rounds.  Both arms use the same lr (1e-3) and weight decay (1e-2); Adam's is L2-coupled, AdamW's
decoupled.

* ``mlp``: the headline MLP (3 x Linear(4096, 4096) trunk, heads 1000 + 64), batch 4096, bf16,
  inputs resident in HBM, the step replayed from a CUDA graph.  Step time from CUDA events around
  each round; update time from the pipeline's events around every update launch, in 6 eager steps
  after each round (the first 2 dropped).
* ``resnet50x4``: the 4-task heads over a ResNet-50 trunk, batch 256 at 224 x 224, bf16, eager
  launches; step time from CUDA events around each round.

The card's name, power limit and max SM clock are read in the same run and printed with the table.

    python tools/bench_adamw.py [--workloads mlp,resnet50x4] [--rounds 5] [--steps 50] [--json out.json]
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
ARMS = ("adam", "adamw")
BATCH = {"mlp": 4096, "resnet50x4": 256}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                              "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = "nvidia-smi unavailable (%s)" % e
    return out or torch.cuda.get_device_name(0)


def build(workload, adamw):
    ns = synthetic.api_namespace("frl_b200")
    t = ns.types
    save_dir = tempfile.mkdtemp(prefix="frl_b200_bench_adamw_")
    torch.manual_seed(0)
    if workload == "mlp":
        problem = synthetic.make_mlp_problem(ns, save_dir, n_train=64, width=4096, n_classes=1000, reg_dim=64,
                                             depth=3)
    else:
        problem = synthetic.make_resnet_problem(ns, save_dir, workload, image=224, n_train=64)
    run_opts = t.RunOpts(optim=t.OptimOpts(algo=t.OptAlgorithm.ADAM, lr=1e-3, weightDecay=1e-2),
                         batchSize=BATCH[workload], nEpochs=1, numThreads=0, singleThreaded=True,
                         numVisualizedSamples=0)
    args = SolverWorkerArgs(run_opts=run_opts, problem=problem, save_dir=save_dir, run_device=Device.GPU,
                            node_idx=0, node_count=1, rank=0, local_rank=0, world_size=1, group_name=None,
                            init_method="", precision=Precision.BF16, graph_step=workload == "mlp", adamw=adamw)
    worker, _, _ = Solver.build_worker(args)
    worker.model.train()
    worker.criterion.train()
    assert worker.optimizer.adamw is adamw
    return worker


def batches(workload, gen, n=4):
    B = BATCH[workload]
    out = []
    for _ in range(n):
        if workload == "mlp":
            x = torch.randn(B, 4096, device=DEV, generator=gen)
            out.append(([x], [(torch.randint(0, 1000, (B,), device=DEV, generator=gen),),
                              (torch.randn(B, 64, device=DEV, generator=gen),)]))
        else:
            x = torch.randn(B, 3, 224, 224, device=DEV, generator=gen)
            target = []
            for kind, dim, _, _ in synthetic.RESNET_CONFIGS[workload][1]:
                target.append((torch.randint(0, dim, (B,), device=DEV, generator=gen),) if kind == "cls"
                              else (torch.randn(B, dim, device=DEV, generator=gen),))
            out.append(([x], target))
    return out


def run(worker, pool, i0, k):
    from frl_b200.types import Split
    for i in range(i0, i0 + k):
        data, target = pool[i % len(pool)]
        worker._pass_one_minibatch(i, Split.TRAIN, data, target)


def update_ms(worker, pool, i0):
    """Per-step update time from the pipeline's events, over eager steps (a replayed graph's launches
    carry no events)."""
    graphed, worker.graphed = worker.graphed, None
    pipe = worker.pipeline
    pipe.update_events.clear()
    pipe.record_update_events = True
    run(worker, pool, i0, 6)
    torch.cuda.synchronize()
    pipe.record_update_events = False
    worker.graphed = graphed
    ev = pipe.update_events
    per_step = max(len(ev) // 6, 1)
    ms = sum(e0.elapsed_time(e1) for e0, e1, _, _ in ev[2 * per_step:]) / 4
    pipe.update_events.clear()
    return ms


def bench(workload, rounds, steps, warmup):
    gen = torch.Generator(device=DEV).manual_seed(1234)
    pool = batches(workload, gen)
    workers = {arm: build(workload, arm == "adamw") for arm in ARMS}
    step_ms = {arm: [] for arm in ARMS}
    upd_ms = {arm: [] for arm in ARMS}
    pos = {arm: 0 for arm in ARMS}
    for arm in ARMS:
        run(workers[arm], pool, 0, warmup)
        pos[arm] = warmup
    torch.cuda.synchronize()
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
            if workload == "mlp":
                upd_ms[arm].append(update_ms(w, pool, pos[arm]))
                pos[arm] += 6
    out = {}
    for arm in ARMS:
        rec = {"step_ms": step_ms[arm], "step_median_ms": statistics.median(step_ms[arm])}
        if upd_ms[arm]:
            rec.update(update_ms=upd_ms[arm], update_median_ms=statistics.median(upd_ms[arm]))
        out[arm] = rec
        line = "%-10s %-6s step %.3f ms (%.3f-%.3f)" % (workload, arm, rec["step_median_ms"], min(step_ms[arm]),
                                                          max(step_ms[arm]))
        if upd_ms[arm]:
            line += "  update %.3f ms (%.3f-%.3f)" % (rec["update_median_ms"], min(upd_ms[arm]), max(upd_ms[arm]))
        print(line, flush=True)
    out["adamw_over_adam_step"] = out["adamw"]["step_median_ms"] / out["adam"]["step_median_ms"]
    if workload == "mlp":
        out["adamw_over_adam_update"] = out["adamw"]["update_median_ms"] / out["adam"]["update_median_ms"]
    print(json.dumps({workload: {k: v for k, v in out.items() if k.startswith("adamw_over")}}), flush=True)
    del workers
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="mlp,resnet50x4")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_adamw.py measures on a GPU; none is visible")
    torch.cuda.set_device(0)
    torch.backends.cudnn.benchmark = True
    result = {"card": card(), "torch": torch.__version__}
    print("card:", result["card"], flush=True)
    for wl in args.workloads.split(","):
        result[wl] = bench(wl, args.rounds, args.steps, args.warmup)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
