#!/usr/bin/env python
"""Cost of the weight EMA on the headline workload (1 GPU, 2-task MLP, batch 4096, BF16, SGD, inputs
resident on the device, CUDA-graph replay by default), in one process: EMA off against EMA on.

    python tools/bench_ema.py [--decay 0.9999] [--steps 50] [--warmup 5] [--repeats 5] [--graph 1]

Both configurations get their own worker, built from the same seed through ``Solver.build_worker``
as ``bench.py`` builds it, and train on a pool of device-resident synthetic batches.  After a GEMM
spin-up and the warm-up steps (which include the CUDA-graph capture) they take turns: each repeat
times ``--steps`` steps of each between two CUDA events, so slow drift of the shared machine falls
on both alike.  A last window of the EMA run records K11 with ``torch.profiler`` (kernel time; K11
runs after the graph replay, once per update).

Memory is measured in a fresh process per configuration (``--memory-of``), so that both carry the
process's one-time allocations (cuBLAS workspaces, the capture stream's pool, native scratch)
alike: ``torch.cuda.max_memory_allocated()`` and ``torch.cuda.memory_allocated()`` after the build,
the warm-up steps (graph capture included), ``--steps`` more steps and, with the EMA, one swap in and
out as a held-out split does.  Prints one JSON line per configuration (ms per step and samples/s:
median, min and max over the repeats; peak and resident memory) and one with the card's name, power
limit and max SM clock, read by the same command.
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
sys.path.insert(0, os.path.join(REPO, "tools"))

import torch  # noqa: E402

import bench  # noqa: E402
import frl_b200  # noqa: E402,F401
from bench_layerwise import card  # noqa: E402
from frl_b200 import ema as ema_mod, synthetic  # noqa: E402
from frl_b200.solver import Solver, SolverWorkerArgs  # noqa: E402
from frl_b200.solver_worker import LossLog  # noqa: E402
from frl_b200.types import Device, Precision  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--decay", type=float, default=0.9999)
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--graph", type=int, default=1)
    ap.add_argument("--memory-of", default=None, help="internal: measure the memory of one configuration")
    args = ap.parse_args()
    args.workload, args.image, args.algo = "mlp", 0, "sgd"
    assert torch.cuda.is_available(), "bench_ema needs a GPU"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    os.environ["FRL_B200_CUDA_GRAPH"] = "1" if args.graph else "0"
    ns = synthetic.api_namespace("frl_b200")
    t = ns.types
    W, S, R, B = args.warmup, args.steps, args.repeats, args.batch
    gen = torch.Generator(device=dev).manual_seed(1234)
    configs = [("ema off", 0.0), ("ema on", args.decay)]

    def step(run):
        w = run["worker"]
        i = run["step"]
        data, target = run["pool"][i % len(run["pool"])]
        w.criterion.set_step_sink(run["log"].row(i), run["log"].nan_flag)
        w._pass_one_minibatch(i, t.Split.TRAIN, data, target)
        run["step"] += 1

    def build(decay):
        save_dir = tempfile.mkdtemp(prefix="frl_b200_ema_bench_")
        torch.manual_seed(0)
        problem = bench.build_problem(ns, save_dir, args)
        wargs = SolverWorkerArgs(run_opts=bench.run_opts_for(ns, args.algo, B), problem=problem,
                                 save_dir=save_dir, run_device=Device.GPU, node_idx=0, node_count=1, rank=0,
                                 local_rank=0, world_size=1, group_name=None, init_method="",
                                 precision=Precision.BF16, ema_decay=decay)
        worker, _, _ = Solver.build_worker(wargs)
        worker.model.train()
        worker.criterion.train()
        n_steps = 2 * W + S * (R + 1) + 8
        return {"worker": worker, "log": LossLog(len(worker.criterion.loss_names), n_steps, dev),
                "step": 0, "ms": [], "pool": [bench.synthetic_batch(args, B, gen, dev) for _ in range(4)]}

    if args.memory_of is not None:
        run = build(dict(configs)[args.memory_of])
        for _ in range(W + S):
            step(run)
        if run["worker"].ema is not None:
            with run["worker"].ema.swapped():
                pass
        torch.cuda.synchronize()
        print(json.dumps({"config": args.memory_of,
                          "max_memory_allocated_MiB": round(torch.cuda.max_memory_allocated(dev) / 2 ** 20, 1),
                          "memory_allocated_MiB": round(torch.cuda.memory_allocated(dev) / 2 ** 20, 1)}), flush=True)
        return

    memory = {}
    for name, _ in configs:
        cmd = [sys.executable, os.path.abspath(__file__), "--memory-of", name, "--decay", str(args.decay),
               "--batch", str(B), "--steps", str(S), "--warmup", str(W), "--graph", str(args.graph)]
        out = subprocess.run(cmd, capture_output=True, text=True, check=True).stdout
        memory[name] = json.loads(out.strip().splitlines()[-1])

    runs = {}
    for name, decay in configs:
        runs[name] = build(decay)
        for _ in range(W):             # warm-up steps (graph capture included)
            step(runs[name])
        torch.cuda.synchronize()

    spin = torch.randn(4096, 4096, device=dev, dtype=torch.bfloat16)
    t_spin = time.perf_counter()
    while time.perf_counter() - t_spin < 0.5:
        for _ in range(20):
            spin = (spin @ spin).clamp_(-1, 1)
        torch.cuda.synchronize()
    del spin
    for name, _ in configs:
        for _ in range(W):
            step(runs[name])
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(R):
        for name, _ in configs:
            run = runs[name]
            e0.record()
            for _ in range(S):
                step(run)
            e1.record()
            torch.cuda.synchronize()
            run["ms"].append(e0.elapsed_time(e1) / S)

    from torch.profiler import ProfilerActivity, profile
    run = runs["ema on"]
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(S):
            step(run)
        torch.cuda.synchronize()
    k11 = [e for e in prof.key_averages() if "weight_ema_kernel" in e.key]
    k11_ms = sum(e.device_time_total for e in k11) / 1e3 / S
    ema = run["worker"].ema
    n = ema.ema.numel()

    info = card()
    for name, decay in configs:
        run = runs[name]
        ms = sorted(run["ms"])
        med = ms[len(ms) // 2]
        w = run["worker"]
        rec = {
            "config": name, "decay": decay, "batch": B, "algo": args.algo, "precision": "bf16",
            "step_issue": "CUDA graph replay" if args.graph else "eager",
            "graphs_captured": len(w.graphed._graphs) if w.graphed is not None else 0,
            "ms_per_step": {"median": round(med, 4), "min": round(ms[0], 4), "max": round(ms[-1], 4)},
            "samples_per_s": {"median": round(B * 1e3 / med, 1), "min": round(B * 1e3 / ms[-1], 1),
                              "max": round(B * 1e3 / ms[0], 1)},
            "max_memory_allocated_MiB": memory[name]["max_memory_allocated_MiB"],
            "memory_allocated_MiB": memory[name]["memory_allocated_MiB"],
            "memory": "own process per configuration",
            "repeats": R, "steps_per_repeat": S, "warmup_steps": W,
            "last_losses": [round(v, 6) for v in run["log"].rows[max(run["step"] - 4, 0):run["step"], 0].tolist()]}
        if w.ema is not None:
            rec.update({"ema_updates": w.ema.updates, "ema_MiB": round(w.ema.nbytes / 2 ** 20, 1),
                        "k11_ms_per_update": round(k11_ms, 4), "k11_launches_profiled": sum(e.count for e in k11),
                        "k11_GBps": round(12 * n / (k11_ms * 1e-3) / 1e9, 1) if k11_ms > 0 else None,
                        "swap_transient_MiB": round(min(n, ema_mod.SWAP_CHUNK) * 4 / 2 ** 20, 1)})
        print(json.dumps(rec), flush=True)
    print(json.dumps({"card": info}), flush=True)


if __name__ == "__main__":
    main()
