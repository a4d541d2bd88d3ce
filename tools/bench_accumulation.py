#!/usr/bin/env python
"""Throughput of the headline workload with gradient accumulation (1 GPU, BF16, CUDA-graph replay by
default), in one process: one batch of 4096 rows per update against 4 x 1024 and 8 x 512.

    python tools/bench_accumulation.py [--configs 4096x1,1024x4,512x8] [--groups 20] [--warmup 3]
                                       [--repeats 5] [--graph 1]

Each configuration (microbatch rows B x microbatches k per update) gets its own worker, built from
the same seed through ``Solver.build_worker`` as ``bench.py`` builds it, and trains on a pool of
device-resident synthetic batches of its B.  After a GEMM spin-up and the warm-up groups (which
include the CUDA-graph capture), the configurations take turns: each repeat times ``--groups``
groups (k microbatches, one update) of every configuration between two CUDA events, so slow drift of
the shared machine falls on all alike.  A last window per configuration times the update per group
with CUDA events around it, and K10 per microbatch from ``torch.profiler`` kernel time (K10 runs
inside the replayed graph).  The workers are built one after the other: a configuration's peak is
``torch.cuda.max_memory_allocated()`` after its warm-up groups, with the peak statistics reset before
its worker was built, less what was allocated then.  Prints one JSON
line per configuration (ms per 4096 samples and samples/s: median, min and max over the repeats; K10
and update times; peak memory) and one with the card's name and power limit, read by the same
command.
"""
import argparse
import json
import os
import sys
import tempfile
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tools"))

import torch  # noqa: E402

import bench  # noqa: E402
import frl_b200  # noqa: E402,F401
from bench_layerwise import card  # noqa: E402
from frl_b200 import synthetic  # noqa: E402
from frl_b200.solver import Solver, SolverWorkerArgs  # noqa: E402
from frl_b200.solver_worker import LossLog  # noqa: E402
from frl_b200.types import Device, Precision  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="4096x1,1024x4,512x8")
    ap.add_argument("--algo", default="sgd")
    ap.add_argument("--groups", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--graph", type=int, default=1)
    args = ap.parse_args()
    args.workload, args.image = "mlp", 0
    assert torch.cuda.is_available(), "bench_accumulation needs a GPU"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    os.environ["FRL_B200_CUDA_GRAPH"] = "1" if args.graph else "0"
    ns = synthetic.api_namespace("frl_b200")
    t = ns.types
    configs = [tuple(int(v) for v in c.split("x")) for c in args.configs.split(",")]
    W, G, R = args.warmup, args.groups, args.repeats
    gen = torch.Generator(device=dev).manual_seed(1234)

    def group(run, k):
        w = run["worker"]
        for j in range(k):
            i = run["step"]
            data, target = run["pool"][i % len(run["pool"])]
            w.pipeline.set_microbatch(first=j == 0, closes=j == k - 1, weight=1.0, group_scale=1.0 / k)
            w.criterion.set_step_sink(run["log"].row(i), run["log"].nan_flag)
            w._pass_one_minibatch(i, t.Split.TRAIN, data, target)
            run["step"] += 1

    # built one after the other: the peak memory of a configuration is measured from the memory
    # allocated before its worker was built to the end of its warm-up groups (graph capture included)
    runs = {}
    for B, k in configs:
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(dev)
        base = torch.cuda.memory_allocated(dev)
        save_dir = tempfile.mkdtemp(prefix="frl_b200_accum_")
        torch.manual_seed(0)
        args.batch = B
        problem = bench.build_problem(ns, save_dir, args)
        wargs = SolverWorkerArgs(run_opts=bench.run_opts_for(ns, args.algo, B), problem=problem,
                                 save_dir=save_dir, run_device=Device.GPU, node_idx=0, node_count=1, rank=0,
                                 local_rank=0, world_size=1, group_name=None, init_method="",
                                 precision=Precision.BF16, grad_accumulation=k)
        worker, _, _ = Solver.build_worker(wargs)
        worker.model.train()
        worker.criterion.train()
        n_steps = k * (2 * W + G * (R + 1)) + 8
        runs[(B, k)] = {"worker": worker, "log": LossLog(len(worker.criterion.loss_names), n_steps, dev),
                        "step": 0, "ms": [], "pool": [bench.synthetic_batch(args, B, gen, dev) for _ in range(4)]}
        for _ in range(W):           # warm-up groups (graph capture included) while only this one is measured
            group(runs[(B, k)], k)
        torch.cuda.synchronize()
        runs[(B, k)]["peak"] = torch.cuda.max_memory_allocated(dev) - base

    spin = torch.randn(4096, 4096, device=dev, dtype=torch.bfloat16)
    t_spin = time.perf_counter()
    while time.perf_counter() - t_spin < 0.5:
        for _ in range(20):
            spin = (spin @ spin).clamp_(-1, 1)
        torch.cuda.synchronize()
    del spin
    for c in configs:
        for _ in range(W):
            group(runs[c], c[1])
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(R):
        for c in configs:
            run = runs[c]
            e0.record()
            for _ in range(G):
                group(run, c[1])
            e1.record()
            torch.cuda.synchronize()
            run["ms"].append(e0.elapsed_time(e1) / G)

    from torch.profiler import ProfilerActivity, profile
    for c in configs:
        # the update alone: CUDA events around it (it runs after the graph replay, outside it); K10
        # runs inside the replayed graph, so its time is torch.profiler's kernel time
        run = runs[c]
        pipe = run["worker"].pipeline
        pipe.update_events.clear()
        torch.cuda.synchronize()
        pipe.record_update_events = True
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(G):
                group(run, c[1])
            torch.cuda.synchronize()
        pipe.record_update_events = False
        run["k10_ms"] = sum(e.device_time_total for e in prof.key_averages()
                            if "grad_accumulate_kernel" in e.key) / 1e3 / (G * c[1])
        run["update_ms"] = sum(a.elapsed_time(b) for a, b, _, _ in pipe.update_events) / G

    info = card()
    for B, k in configs:
        run = runs[(B, k)]
        ms = sorted(run["ms"])
        med = ms[len(ms) // 2]
        rows = B * k
        w = run["worker"]
        print(json.dumps({
            "microbatch_rows": B, "microbatches_per_update": k, "algo": args.algo, "precision": "bf16",
            "step_issue": "CUDA graph replay" if args.graph else "eager",
            "graphs_captured": len(w.graphed._graphs) if w.graphed is not None else 0,
            "ms_per_%d_samples" % rows: {"median": round(med, 4), "min": round(ms[0], 4), "max": round(ms[-1], 4)},
            "samples_per_s": {"median": round(rows * 1e3 / med, 1), "min": round(rows * 1e3 / ms[-1], 1),
                              "max": round(rows * 1e3 / ms[0], 1)},
            "k10_ms_per_microbatch": round(run["k10_ms"], 4), "update_ms_per_group": round(run["update_ms"], 4),
            "accumulator_MiB": round(w.pipeline.accumulator_bytes / 2 ** 20, 1),
            "max_memory_allocated_MiB": round(run["peak"] / 2 ** 20, 1),
            "repeats": R, "groups_per_repeat": G, "warmup_groups": W,
            "last_losses": [round(v, 6) for v in run["log"].rows[max(run["step"] - 4, 0):run["step"], 0].tolist()]}),
            flush=True)
    print(json.dumps({"card": info}), flush=True)


if __name__ == "__main__":
    main()
