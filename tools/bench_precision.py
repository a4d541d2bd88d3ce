#!/usr/bin/env python
"""Step time of the headline workload in BF16 against FP8 (1 GPU), in one process.

    python tools/bench_precision.py [--batch 4096] [--algo sgd] [--steps 50] [--warmup 5]
                                    [--repeats 5] [--graph 1] [--precisions bf16,fp8]

Each precision gets its own worker, built from the same seed through ``Solver.build_worker`` as
``bench.py`` builds it (``build_problem`` / ``run_opts_for`` / ``synthetic_batch`` are bench.py's),
and trains on the same pool of device-resident synthetic batches.  After a GEMM spin-up and the
warm-up steps (which include the CUDA-graph capture), the precisions take turns: each repeat times
``--steps`` steps of every precision between two CUDA events, so slow drift of the shared machine
falls on both alike.  Prints one JSON line per precision (ms/step and samples/s: median, min and
max over the repeats; the losses of every step) and one with the card's name and power limit,
read by the same command.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import torch  # noqa: E402

import bench  # noqa: E402
import frl_b200  # noqa: E402,F401
from frl_b200 import synthetic  # noqa: E402
from frl_b200.solver import Solver, SolverWorkerArgs  # noqa: E402
from frl_b200.solver_worker import LossLog  # noqa: E402
from frl_b200.types import Device, Precision  # noqa: E402


def card():
    """Name, power limit and max SM clock of GPU 0 as nvidia-smi reports them (read only)."""
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = "nvidia-smi unavailable: %s" % e
    return {"torch_device": torch.cuda.get_device_name(0), "nvidia_smi": out}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--algo", default="sgd", choices=["sgd", "adam"])
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--graph", type=int, default=1)
    ap.add_argument("--precisions", default="bf16,fp8")
    args = ap.parse_args()
    args.workload, args.image = "mlp", 0
    assert torch.cuda.is_available(), "bench_precision needs a GPU"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    os.environ["FRL_B200_CUDA_GRAPH"] = "1" if args.graph else "0"
    ns = synthetic.api_namespace("frl_b200")
    t = ns.types
    precs = [Precision(p) for p in args.precisions.split(",")]
    W, K, R = args.warmup, args.steps, args.repeats

    runs = {}
    for p in precs:
        save_dir = tempfile.mkdtemp(prefix="frl_b200_prec_")
        torch.manual_seed(0)
        problem = bench.build_problem(ns, save_dir, args)
        wargs = SolverWorkerArgs(run_opts=bench.run_opts_for(ns, args.algo, args.batch), problem=problem,
                                 save_dir=save_dir, run_device=Device.GPU, node_idx=0, node_count=1, rank=0,
                                 local_rank=0, world_size=1, group_name=None, init_method="", precision=p)
        worker, _, _ = Solver.build_worker(wargs)
        worker.model.train()
        worker.criterion.train()
        log = LossLog(len(worker.criterion.loss_names), W + K * R + 8, dev)
        runs[p] = {"worker": worker, "log": log, "step": 0, "ms": [],
                   "fp8_sites": sum(s.fp8 for s in worker.pipeline.linear_sites)}
    gen = torch.Generator(device=dev).manual_seed(1234)
    pool = [bench.synthetic_batch(args, args.batch, gen, dev) for _ in range(4)]

    def step(run):
        i = run["step"]
        data, target = pool[i % len(pool)]
        run["worker"].criterion.set_step_sink(run["log"].row(i), run["log"].nan_flag)
        out = run["worker"]._pass_one_minibatch(i, t.Split.TRAIN, data, target)
        run["step"] += 1
        return out

    spin = torch.randn(4096, 4096, device=dev, dtype=torch.bfloat16)
    t_spin = time.perf_counter()
    while time.perf_counter() - t_spin < 0.5:
        for _ in range(20):
            spin = (spin @ spin).clamp_(-1, 1)
        torch.cuda.synchronize()
    del spin
    for p in precs:
        for _ in range(W):
            step(runs[p])
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(R):
        for p in precs:
            run = runs[p]
            e0.record()
            for _ in range(K):
                step(run)
            e1.record()
            torch.cuda.synchronize()
            run["ms"].append(e0.elapsed_time(e1) / K)

    info = card()
    for p in precs:
        run = runs[p]
        ms = sorted(run["ms"])
        med = ms[len(ms) // 2]
        losses = run["log"].rows[:run["step"], 0].tolist()
        print(json.dumps({
            "precision": p.value, "workload": bench.workload_name(args), "fp8_linear_sites": run["fp8_sites"],
            "step_issue": "CUDA graph replay" if args.graph else "eager",
            "ms_per_step": {"median": round(med, 4), "min": round(ms[0], 4), "max": round(ms[-1], 4)},
            "samples_per_s": {"median": round(args.batch * 1e3 / med, 1), "min": round(args.batch * 1e3 / ms[-1], 1),
                              "max": round(args.batch * 1e3 / ms[0], 1)},
            "repeats": R, "steps_per_repeat": K, "warmup": W,
            "losses": [round(v, 6) for v in losses]}), flush=True)
    print(json.dumps({"card": info}), flush=True)


if __name__ == "__main__":
    main()
