#!/usr/bin/env python
"""Step time of the headline workload with and without layer-wise adaptation (1 GPU, BF16), in one
process: SGD against LARS and Adam against LAMB.

    python tools/bench_layerwise.py [--batch 4096] [--steps 50] [--warmup 5] [--repeats 5] [--graph 1]

Each configuration gets its own worker, built from the same seed through ``Solver.build_worker`` as
``bench.py`` builds it (``build_problem`` / ``run_opts_for`` / ``synthetic_batch`` are bench.py's),
and trains on the same pool of device-resident synthetic batches.  After a GEMM spin-up and the
warm-up steps (which include the CUDA-graph capture), the configurations take turns: each repeat
times ``--steps`` steps of every configuration between two CUDA events, so slow drift of the shared
machine falls on all alike.  A last window of ``--steps`` steps per configuration times the update
alone (CUDA events around the tail update, which runs outside the captured graph) and reports the
bytes the update must move per parameter over that time against the data-sheet 3.35 TB/s.  Prints
one JSON line per configuration (ms/step and samples/s: median, min and max over the repeats; update
time and bandwidth; the losses of every step) and one with the card's name and power limit, read by
the same command.
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
from frl_b200.types import Device, LayerAdaptation, Precision  # noqa: E402

HBM_BYTES_PER_S = 3.35e12      # H100 SXM data sheet, not measured
# bytes the update moves per parameter with bf16 gradients and a bf16 shadow (momentum 0.9 for SGD
# and LARS): K2 SGD reads g, w, buf and writes w, buf, shadow; LARS adds a stats pass reading g, w;
# Adam reads g, w, m, v and writes w, m, v, shadow; LAMB's stats pass reads g, w, m, v and writes
# m, v, its apply pass reads w, m, v and writes w and the shadow
UPDATE_BYTES = {("sgd", "none"): 20, ("sgd", "lars"): 26, ("adam", "none"): 28, ("adam", "lamb"): 40}
CONFIGS = [("sgd", "none"), ("sgd", "lars"), ("adam", "none"), ("adam", "lamb")]


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
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--graph", type=int, default=1)
    args = ap.parse_args()
    args.workload, args.image = "mlp", 0
    assert torch.cuda.is_available(), "bench_layerwise needs a GPU"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    os.environ["FRL_B200_CUDA_GRAPH"] = "1" if args.graph else "0"
    ns = synthetic.api_namespace("frl_b200")
    t = ns.types
    configs = CONFIGS
    W, K, R = args.warmup, args.steps, args.repeats

    runs = {}
    for p in configs:
        save_dir = tempfile.mkdtemp(prefix="frl_b200_lw_")
        torch.manual_seed(0)
        problem = bench.build_problem(ns, save_dir, args)
        wargs = SolverWorkerArgs(run_opts=bench.run_opts_for(ns, p[0], args.batch), problem=problem,
                                 save_dir=save_dir, run_device=Device.GPU, node_idx=0, node_count=1, rank=0,
                                 local_rank=0, world_size=1, group_name=None, init_method="",
                                 precision=Precision.BF16, layer_adaptation=LayerAdaptation(p[1]))
        worker, _, _ = Solver.build_worker(wargs)
        worker.model.train()
        worker.criterion.train()
        log = LossLog(len(worker.criterion.loss_names), W + K * (R + 1) + 8, dev)
        runs[p] = {"worker": worker, "log": log, "step": 0, "ms": []}
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
    for p in configs:
        for _ in range(W):
            step(runs[p])
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(R):
        for p in configs:
            run = runs[p]
            e0.record()
            for _ in range(K):
                step(run)
            e1.record()
            torch.cuda.synchronize()
            run["ms"].append(e0.elapsed_time(e1) / K)

    for p in configs:                 # update alone: events around the tail update of every step
        pipe = runs[p]["worker"].pipeline
        pipe.update_events.clear()
        pipe.record_update_events = True
        for _ in range(K):
            step(runs[p])
        torch.cuda.synchronize()
        pipe.record_update_events = False
        runs[p]["update_ms"] = sum(a.elapsed_time(b) for a, b, _, _ in pipe.update_events) / K

    info = card()
    for p in configs:
        run = runs[p]
        ms = sorted(run["ms"])
        med = ms[len(ms) // 2]
        losses = run["log"].rows[:run["step"], 0].tolist()
        n = run["worker"].arena.n_trainable
        upd_s = run["update_ms"] * 1e-3
        args.algo = p[0]
        print(json.dumps({
            "algo": p[0], "layer_adaptation": p[1], "precision": "bf16", "workload": bench.workload_name(args),
            "step_issue": "CUDA graph replay" if args.graph else "eager",
            "update_ms": round(run["update_ms"], 4), "update_bytes_per_param": UPDATE_BYTES[p],
            "update_GB_per_s": round(UPDATE_BYTES[p] * n / upd_s / 1e9, 1),
            "update_share_of_3.35TB_per_s": round(UPDATE_BYTES[p] * n / upd_s / HBM_BYTES_PER_S, 3),
            "ms_per_step": {"median": round(med, 4), "min": round(ms[0], 4), "max": round(ms[-1], 4)},
            "samples_per_s": {"median": round(args.batch * 1e3 / med, 1), "min": round(args.batch * 1e3 / ms[-1], 1),
                              "max": round(args.batch * 1e3 / ms[0], 1)},
            "repeats": R, "steps_per_repeat": K, "warmup": W,
            "losses": [round(v, 6) for v in losses]}), flush=True)
    print(json.dumps({"card": info}), flush=True)


if __name__ == "__main__":
    main()
