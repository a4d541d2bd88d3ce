"""Update-kernel time of bf16 master weights with stochastic rounding against the fp32 master.

One segment table over an arena of the headline MLP's size (54.7 M parameters in 8 slots, bf16
gradients), alternating the fp32-master K2-mt launch (fp32 weights + bf16 shadow) and its SR form
(bf16 weights only) in one process: ``--reps`` rounds of ``--iters`` launches each, CUDA events
around every round, median (min-max) per launch, and the achieved HBM rate from the bytes each
form must move.  Prints one JSON line; reads the card, its power limit and SM clock in the same
process (nvidia-smi).

``--steps``: also the training step of the headline MLP (width 4096, depth 3, 54.7 M parameters,
batch 4096, BF16, CUDA-graph replay) with SGD (the dW-GEMM update, K12) and Adam (K2-mt), fp32 and bf16
master weights built side by side and stepped alternately: ``--reps`` windows of ``--iters`` steps, CUDA
events around each window, median (min-max) ms per step, and device memory after each build.

    python tools/bench_master_weights.py [--n 54700000] [--iters 50] [--reps 5] [--steps]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import frl_b200  # noqa: E402,F401
from frl_b200 import _native  # noqa: E402
from frl_b200.multi_tensor import GradSegTable  # noqa: E402

HBM_PEAK = 3.35e12     # H100 SXM data sheet, bytes/s


class _Slot:
    def __init__(self, i, off, n):
        self.index, self.offset, self.numel, self.shape, self.is_model = i, off, n, (n,), True
        self.end = off + n


def _card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm",
                               "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except OSError as e:
        return "nvidia-smi unavailable: %s" % e


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=54_700_000)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    dev = torch.device("cuda")
    per = (a.n // 8 + 7) // 8 * 8
    slots = [_Slot(i, i * per, per) for i in range(8)]
    total = 8 * per
    table = GradSegTable(slots, dev)
    g = torch.randn(total, device=dev).to(torch.bfloat16) * 1e-3
    for s in slots:
        table.point(s, g.data_ptr() + 2 * s.offset, torch.bfloat16)
    table.upload()
    w32 = torch.randn(total, device=dev)
    lp = w32.to(torch.bfloat16)
    w16 = lp.clone()
    m, v = torch.zeros(total, device=dev), torch.zeros(total, device=dev)
    buf = torch.zeros(total, device=dev)
    hyper = dict(lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, wd=0.0, step=1)
    sgd = dict(lr=1e-3, mu=0.9, dampening=0.0, wd=0.0)
    arms = {
        "adam_fp32": (lambda: _native.adam_mt(w32, m, v, None, lp, table, **hyper), 4 + 4 + 2 + 16 + 2),
        "adam_sr": (lambda: _native.adam_mt_sr(w16, m, v, None, table, seed=1, **hyper), 2 + 2 + 2 + 16),
        "sgd_fp32": (lambda: _native.sgd_momentum_mt(w32, buf, lp, table, **sgd), 4 + 4 + 2 + 8 + 2),
        "sgd_sr": (lambda: _native.sgd_momentum_mt_sr(w16, buf, table, seed=1, t=1, **sgd), 2 + 2 + 2 + 8),
    }
    for f, _ in arms.values():          # warm up every instantiation
        f()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for _ in range(a.reps):
        for k, (f, _) in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.iters):
                f()
            e1.record()
            e1.synchronize()
            times[k].append(e0.elapsed_time(e1) / a.iters * 1e-3)
    out = {"card": _card(), "elements": total, "iters": a.iters, "reps": a.reps}
    for k, (_, bpp) in arms.items():
        med = statistics.median(times[k])
        out[k] = {"median_us": round(med * 1e6, 1), "min_us": round(min(times[k]) * 1e6, 1),
                  "max_us": round(max(times[k]) * 1e6, 1), "bytes_per_param": bpp,
                  "TBps": round(bpp * total / med / 1e12, 3), "share_of_3.35TBps": round(bpp * total / med / HBM_PEAK, 3)}
    out["adam_sr_over_fp32"] = round(out["adam_sr"]["median_us"] / out["adam_fp32"]["median_us"], 3)
    out["sgd_sr_over_fp32"] = round(out["sgd_sr"]["median_us"] / out["sgd_fp32"]["median_us"], 3)
    if a.steps:
        del g, w32, lp, w16, m, v, buf, table
        torch.cuda.empty_cache()
        out["steps"] = step_arms(a.iters, a.reps)
    print(json.dumps(out))


def step_arms(iters, reps):
    import tempfile
    from frl_b200 import synthetic
    from frl_b200.solver import Solver, SolverWorkerArgs
    from frl_b200.types import Device, MasterWeights, OptAlgorithm, Precision, Split
    ns = synthetic.api_namespace("frl_b200")
    t = ns.types
    gen = torch.Generator().manual_seed(0)
    batches = [(torch.randn(4096, 4096, generator=gen).cuda(), torch.randint(0, 1000, (4096,), generator=gen).cuda(),
                torch.randn(4096, 64, generator=gen).cuda()) for _ in range(4)]
    res = {}
    for algo in (OptAlgorithm.SGD, OptAlgorithm.ADAM):
        workers = {}
        for master in (MasterWeights.FP32, MasterWeights.BF16):
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.manual_seed(0)
            problem = synthetic.make_mlp_problem(ns, tempfile.mkdtemp(prefix="frl_b200_mwb_"), n_train=8)
            run_opts = t.RunOpts(optim=t.OptimOpts(algo=algo, lr=0.01 if algo == OptAlgorithm.SGD else 1e-3,
                                                   momentum=0.9, weightDecay=1e-5),
                                 batchSize=4096, nEpochs=1, numThreads=0, singleThreaded=True, numVisualizedSamples=0)
            args = SolverWorkerArgs(run_opts=run_opts, problem=problem, save_dir=problem.save_dir,
                                    run_device=Device.GPU, node_idx=0, node_count=1, rank=0, local_rank=0,
                                    world_size=1, group_name=None, init_method="", precision=Precision.BF16,
                                    graph_step=True, master_weights=master)
            w = Solver.build_worker(args)[0]
            w.model.train()
            w.criterion.train()
            torch.cuda.synchronize()
            workers[master] = (w, torch.cuda.memory_allocated() - base)
        times = {m: [] for m in workers}
        step = 0
        for r in range(reps + 1):                # window 0 warms up (the graph is captured after 2 steps)
            for m, (w, _) in workers.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for i in range(iters):
                    x, y, rg = batches[(step + i) % 4]
                    w._pass_one_minibatch(step + i, Split.TRAIN, [x], [(y,), (rg,)])
                e1.record()
                e1.synchronize()
                if r:
                    times[m].append(e0.elapsed_time(e1) / iters)
            step += iters
        arm = {}
        for m, (w, mem) in workers.items():
            ts = times[m]
            arm[m.value] = {"ms_per_step_median": round(statistics.median(ts), 4), "min": round(min(ts), 4),
                            "max": round(max(ts), 4), "MiB_after_build": round(mem / 2 ** 20, 1),
                            "k12": bool(w.pipeline.fused_dw_update)}
        arm["bf16_over_fp32"] = round(arm["bf16"]["ms_per_step_median"] / arm["fp32"]["ms_per_step_median"], 3)
        arm["MiB_saved"] = round(arm["fp32"]["MiB_after_build"] - arm["bf16"]["MiB_after_build"], 1)
        res[algo.value] = arm
        del workers
        torch.cuda.empty_cache()
    return res


if __name__ == "__main__":
    main()
