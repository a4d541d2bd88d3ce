#!/usr/bin/env python
"""Adam with fp32 optimizer state against Adam with 8-bit block-wise state (K2-q8) and against
Adafactor (K2-af, ``adafactor=True``) on the headline workload (1 GPU, BF16, batch 4096, inputs resident, CUDA-graph replay).

    python tools/bench_optimizer_state.py [--batch 4096] [--steps 50] [--warmup 5] [--repeats 5] [--graph 1]

Both arms get their own worker, built from the same seed through ``Solver.build_worker`` as
``bench.py`` builds it, and train on the same pool of device-resident synthetic batches.  After a
GEMM spin-up and the warm-up steps (which include the CUDA-graph capture) the arms take turns: each
repeat times ``--steps`` steps of every arm between two CUDA events.  A last window of ``--steps``
steps per arm times the update alone (CUDA events around the tail update).  Memory comes from a
fresh process per arm (``--memory-arm``), so one arm's allocations never inflate the other's:
peak (``max_memory_allocated``) over warm-up and ``--steps`` steps, and what stays allocated after
them.  Prints one JSON line per arm and one with the card's name and power limit, read by the same
command.
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
from frl_b200.types import Device, OptimizerState, Precision  # noqa: E402

HBM_BYTES_PER_S = 3.35e12      # H100 SXM data sheet, not measured
# bytes the update moves per parameter with bf16 gradients and a bf16 shadow: K2-mt Adam reads g, w,
# m, v and writes w, m, v, shadow (28); K2-q8 reads g, w and both codes and writes w, both codes and
# the shadow (16), plus 2 x 8 bytes of absmax per 256-element block (counted from the layout below);
# K2-af reads g three times and w twice and writes w and the shadow (20; its factored state is not
# counted)
ARMS = ["fp32", "8bit", "adafactor"]


def card():
    """Name, power limit and max SM clock of GPU 0 as nvidia-smi reports them (read only)."""
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = "nvidia-smi unavailable: %s" % e
    return {"torch_device": torch.cuda.get_device_name(0), "nvidia_smi": out}


def build(ns, args, arm):
    save_dir = tempfile.mkdtemp(prefix="frl_b200_optstate_")
    torch.manual_seed(0)
    problem = bench.build_problem(ns, save_dir, args)
    wargs = SolverWorkerArgs(run_opts=bench.run_opts_for(ns, "adam", args.batch), problem=problem,
                             save_dir=save_dir, run_device=Device.GPU, node_idx=0, node_count=1, rank=0,
                             local_rank=0, world_size=1, group_name=None, init_method="",
                             precision=Precision.BF16,
                             optimizer_state=OptimizerState.FP32 if arm == "adafactor" else OptimizerState(arm),
                             adafactor=arm == "adafactor")
    worker, _, _ = Solver.build_worker(wargs)
    worker.model.train()
    worker.criterion.train()
    return worker


def update_bytes(worker):
    opt = worker.optimizer
    n = worker.arena.n_trainable
    if getattr(opt, "q8_blocks", None) is not None:
        return 16 * n + 16 * opt.q8_blocks
    if getattr(opt, "state_buf", None) is not None:
        return 20 * n
    return 28 * n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--graph", type=int, default=1)
    ap.add_argument("--memory-arm", choices=ARMS, default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    args.workload, args.image, args.algo = "mlp", 0, "adam"
    assert torch.cuda.is_available(), "bench_optimizer_state needs a GPU"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    os.environ["FRL_B200_CUDA_GRAPH"] = "1" if args.graph else "0"
    ns = synthetic.api_namespace("frl_b200")
    t = ns.types
    W, K, R = args.warmup, args.steps, args.repeats
    arms = [args.memory_arm] if args.memory_arm else ARMS

    runs = {}
    for a in arms:
        worker = build(ns, args, a)
        log = LossLog(len(worker.criterion.loss_names), W + K * (R + 1) + 8, dev)
        runs[a] = {"worker": worker, "log": log, "step": 0, "ms": []}
    gen = torch.Generator(device=dev).manual_seed(1234)
    pool = [bench.synthetic_batch(args, args.batch, gen, dev) for _ in range(4)]

    def step(run):
        i = run["step"]
        data, target = pool[i % len(pool)]
        run["worker"].criterion.set_step_sink(run["log"].row(i), run["log"].nan_flag)
        out = run["worker"]._pass_one_minibatch(i, t.Split.TRAIN, data, target)
        run["step"] += 1
        return out

    if args.memory_arm:
        run = runs[args.memory_arm]
        for _ in range(W + K):
            step(run)
        torch.cuda.synchronize()
        opt = run["worker"].optimizer
        state = opt.state_bytes if hasattr(opt, "state_bytes") else sum(
            v.numel() * v.element_size() for v in opt._vec.values())
        print(json.dumps({"arm": args.memory_arm, "peak_MiB": round(torch.cuda.max_memory_allocated() / 2 ** 20, 1),
                          "resident_MiB": round(torch.cuda.memory_allocated() / 2 ** 20, 1),
                          "optimizer_state_MiB": round(state / 2 ** 20, 1)}), flush=True)
        return

    spin = torch.randn(4096, 4096, device=dev, dtype=torch.bfloat16)
    t_spin = time.perf_counter()
    while time.perf_counter() - t_spin < 0.5:
        for _ in range(20):
            spin = (spin @ spin).clamp_(-1, 1)
        torch.cuda.synchronize()
    del spin
    for a in arms:
        for _ in range(W):
            step(runs[a])
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(R):
        for a in arms:
            run = runs[a]
            e0.record()
            for _ in range(K):
                step(run)
            e1.record()
            torch.cuda.synchronize()
            run["ms"].append(e0.elapsed_time(e1) / K)

    for a in arms:                    # update alone: events around the tail update of every step
        pipe = runs[a]["worker"].pipeline
        pipe.update_events.clear()
        pipe.record_update_events = True
        for _ in range(K):
            step(runs[a])
        torch.cuda.synchronize()
        pipe.record_update_events = False
        runs[a]["update_ms"] = sum(x.elapsed_time(y) for x, y, _, _ in pipe.update_events) / K

    memory = {}
    for a in arms:                    # a fresh process per arm
        res = subprocess.run([sys.executable, os.path.abspath(__file__), "--memory-arm", a, "--batch", str(args.batch),
                              "--steps", str(K), "--warmup", str(W), "--graph", str(args.graph)],
                             capture_output=True, text=True, timeout=900)
        lines = [ln for ln in res.stdout.splitlines() if ln.startswith("{")]
        memory[a] = json.loads(lines[-1]) if lines else {"error": res.stderr[-2000:]}

    info = card()
    for a in arms:
        run = runs[a]
        ms = sorted(run["ms"])
        med = ms[len(ms) // 2]
        losses = run["log"].rows[:run["step"], 0].tolist()
        nbytes = update_bytes(run["worker"])
        n = run["worker"].arena.n_trainable
        upd_s = run["update_ms"] * 1e-3
        print(json.dumps({
            "optimizer_state": a, "algo": "adam", "precision": "bf16", "workload": bench.workload_name(args),
            "step_issue": "CUDA graph replay" if args.graph else "eager",
            "update_ms": round(run["update_ms"], 4), "update_bytes_per_param": round(nbytes / n, 3),
            "update_GB_per_s": round(nbytes / upd_s / 1e9, 1),
            "update_share_of_3.35TB_per_s": round(nbytes / upd_s / HBM_BYTES_PER_S, 3),
            "ms_per_step": {"median": round(med, 4), "min": round(ms[0], 4), "max": round(ms[-1], 4)},
            "memory": memory[a],
            "repeats": R, "steps_per_repeat": K, "warmup": W,
            "losses": [round(v, 6) for v in losses[::10]]}), flush=True)
    print(json.dumps({"card": info}), flush=True)


if __name__ == "__main__":
    main()
