#!/usr/bin/env python
"""K12 (the weight-gradient GEMM with the SGD update in its epilogue) on the headline workload's
shapes, and the whole step with and without it, in one process.

    python tools/bench_dw_update.py [--steps 50] [--warmup 5] [--repeats 5] [--iters 40]

Kernel level, at the trunk's dW GEMM (dZ [4096, 4096] and X [4096, 4096] row-major bf16,
gw = dZ^T X [4096, 4096]), each arm captured in its own CUDA graph and replayed between two CUDA
events after a 256 MiB write that evicts L2, the arms taking turns ``--iters`` times:

* ``torch.mm``       torch.mm(dZ.t(), X, out=gw) (cuBLAS)
* ``k12_plain``      frl_dw_gemm: the same product
* ``mm_plus_k2``     torch.mm, then K2 (frl_sgd_momentum) over the 16.8 M weights of that slice
* ``k12_update``     frl_dw_gemm_sgd: both in one kernel

Whole step: the 2-task MLP (batch 4096, BF16, SGD with momentum, inputs resident on the device,
CUDA-graph replay), one worker built with ``FRL_B200_FUSED_DW_UPDATE=1`` and one with ``=0`` from
the same seed and trained on the same batches; after the warm-up steps (graph capture included)
they take turns, ``--repeats`` windows of ``--steps`` steps each, and the losses of their last
steps are printed side by side.  Prints one JSON line per measurement (median, min, max) and
one with the card's name, power limit and max SM clock, read by the same command.
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
from frl_b200 import _native, synthetic  # noqa: E402
from frl_b200.solver import Solver, SolverWorkerArgs  # noqa: E402
from frl_b200.solver_worker import LossLog  # noqa: E402
from frl_b200.types import Device, Precision  # noqa: E402


def _stats(ms):
    ms = sorted(ms)
    return {"median": round(ms[len(ms) // 2], 4), "min": round(ms[0], 4), "max": round(ms[-1], 4)}


def kernels(dev, iters):
    n = 4096
    g = torch.Generator(device=dev).manual_seed(0)
    dz = torch.randn(n, n, device=dev, generator=g).to(torch.bfloat16)
    x = torch.randn(n, n, device=dev, generator=g).to(torch.bfloat16)
    gw = torch.empty(n, n, device=dev, dtype=torch.bfloat16)
    p = torch.randn(n * n, device=dev, generator=g)
    buf = torch.randn(n * n, device=dev, generator=g)
    lp = p.to(torch.bfloat16)
    sgd = dict(lr=1e-3, mu=0.9, dampening=0.0, wd=0.0)
    arms = {
        "torch.mm": lambda: torch.mm(dz.t(), x, out=gw),
        "k12_plain": lambda: _native.dw_gemm(dz, x, gw),
        "mm_plus_k2": lambda: (torch.mm(dz.t(), x, out=gw),
                               _native.sgd_momentum(p, gw.view(-1), buf, lp, n * n, **sgd)),
        "k12_update": lambda: _native.dw_gemm_sgd(dz, x, gw, p, buf, lp, **sgd),
    }
    graphs = {}
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for f in arms.values():
            for _ in range(3):
                f()
    torch.cuda.current_stream().wait_stream(side)
    for name, f in arms.items():
        graphs[name] = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graphs[name]):
            f()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    ms = {k: [] for k in arms}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(iters):
        for name, gr in graphs.items():
            flush.zero_()
            e0.record()
            gr.replay()
            e1.record()
            e1.synchronize()
            ms[name].append(e0.elapsed_time(e1))
    flop = 2.0 * n ** 3
    for name in arms:
        s = _stats(ms[name])
        print(json.dumps({"kernel": name, "shape": "dZ^T X, dZ [4096, 4096], X [4096, 4096] bf16",
                          "ms": s, "tflops_at_median": round(flop / (s["median"] * 1e-3) / 1e12, 1),
                          "l2": "cold (256 MiB write before every replay)", "iters": iters}), flush=True)


def whole_step(dev, args):
    ns = synthetic.api_namespace("frl_b200")
    t = ns.types
    W, S, R, B = args.warmup, args.steps, args.repeats, 4096
    args.workload, args.image, args.algo, args.batch = "mlp", 0, "sgd", B
    os.environ["FRL_B200_CUDA_GRAPH"] = "1"

    def build(fused):
        os.environ["FRL_B200_FUSED_DW_UPDATE"] = fused
        save_dir = tempfile.mkdtemp(prefix="frl_b200_dw_bench_")
        torch.manual_seed(0)
        problem = bench.build_problem(ns, save_dir, args)
        wargs = SolverWorkerArgs(run_opts=bench.run_opts_for(ns, args.algo, B), problem=problem,
                                 save_dir=save_dir, run_device=Device.GPU, node_idx=0, node_count=1, rank=0,
                                 local_rank=0, world_size=1, group_name=None, init_method="",
                                 precision=Precision.BF16)
        worker, _, _ = Solver.build_worker(wargs)
        worker.model.train()
        worker.criterion.train()
        gen = torch.Generator(device=dev).manual_seed(1234)      # both arms train on the same batches
        return {"worker": worker, "step": 0, "ms": [],
                "log": LossLog(len(worker.criterion.loss_names), 2 * W + S * R + 8, dev),
                "pool": [bench.synthetic_batch(args, B, gen, dev) for _ in range(4)]}

    def step(run):
        w, i = run["worker"], run["step"]
        data, target = run["pool"][i % len(run["pool"])]
        w.criterion.set_step_sink(run["log"].row(i), run["log"].nan_flag)
        w._pass_one_minibatch(i, t.Split.TRAIN, data, target)
        run["step"] += 1

    runs = {"fused (FRL_B200_FUSED_DW_UPDATE=1)": build("1"), "tail update (FRL_B200_FUSED_DW_UPDATE=0)": build("0")}
    os.environ.pop("FRL_B200_FUSED_DW_UPDATE")
    spin = torch.randn(4096, 4096, device=dev, dtype=torch.bfloat16)
    t_spin = time.perf_counter()
    while time.perf_counter() - t_spin < 0.5:
        for _ in range(20):
            spin = (spin @ spin).clamp_(-1, 1)
        torch.cuda.synchronize()
    del spin
    for run in runs.values():
        for _ in range(W):
            step(run)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(R):
        for run in runs.values():
            e0.record()
            for _ in range(S):
                step(run)
            e1.record()
            torch.cuda.synchronize()
            run["ms"].append(e0.elapsed_time(e1) / S)
    for name, run in runs.items():
        p = run["worker"].pipeline
        print(json.dumps({"step": name, "ms_per_step": _stats(run["ms"]),
                          "k12_slots": sorted(p.dw_updated), "repeats": R, "steps_per_repeat": S,
                          "warmup_steps": W, "last_losses": [round(v, 6) for v in
                                                             run["log"].rows[run["step"] - 3:run["step"], 0].tolist()]}),
              flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--iters", type=int, default=40)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_dw_update needs a GPU"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    kernels(dev, args.iters)
    whole_step(dev, args)
    print(json.dumps({"card": card()}), flush=True)


if __name__ == "__main__":
    main()
