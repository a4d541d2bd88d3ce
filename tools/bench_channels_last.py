#!/usr/bin/env python
"""Step time of the ResNet workloads with NCHW and channels_last (NHWC) training, one GPU.

    python tools/bench_channels_last.py [--models resnet18,resnet50x4] [--rounds 5] [--steps 30]
                                        [--json out.json]

resnet18 with SGD and resnet50x4 (a ResNet-50 trunk with 4 heads) with Adam, batch 256, 224 x 224,
bf16, uint8 images normalised on the device by the channel-affine transform (K5, or K5 NHWC with
channels_last).  For each model and each step issue (eager launches, CUDA-graph replay) one process
builds an NCHW and an NHWC worker and times them alternately: ``--rounds`` x ``--steps`` steps each,
CUDA events around every round; reported is the median step time of the rounds with their min and
max.  Then, per (model, layout):

* peak device memory of ``--mem-steps`` eager steps, in a fresh process per arm;
* a torch.profiler pass over 5 eager steps that sums the device time per step of layout-conversion
  kernels: cuDNN's ``nchwToNhwc`` / ``nhwcToNchw`` and ATen copies (``copy_`` / elementwise copy
  kernels).
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

CONFIGS = {"resnet18": "sgd", "resnet50x4": "adam"}
BATCH, IMAGE = 256, 224


def make_worker(model, channels_last, graph):
    import torch
    from frl_b200 import synthetic
    from frl_b200.solver import Solver, SolverWorkerArgs
    from frl_b200.types import Device, Precision
    ns = synthetic.api_namespace("frl_b200")
    t = ns.types
    save_dir = tempfile.mkdtemp(prefix="frl_b200_cl_bench_")
    torch.manual_seed(0)
    problem = synthetic.make_resnet_problem(ns, save_dir, model, image=IMAGE, n_train=BATCH, pinned=True, uint8=True)
    algo = t.OptAlgorithm(CONFIGS[model])
    run_opts = t.RunOpts(optim=t.OptimOpts(algo=algo, lr=1e-3 if algo == t.OptAlgorithm.ADAM else 0.01),
                         batchSize=BATCH, nEpochs=1, numThreads=0, singleThreaded=True, numVisualizedSamples=0)
    args = SolverWorkerArgs(run_opts=run_opts, problem=problem, save_dir=save_dir, run_device=Device.GPU,
                            node_idx=0, node_count=1, rank=0, local_rank=0, world_size=1, group_name=None,
                            init_method="", precision=Precision.BF16, graph_step=graph, channels_last=channels_last)
    worker, _, _ = Solver.build_worker(args)
    worker.model.train()
    worker.criterion.train()
    transform = problem.datasets[0].device_transform
    if channels_last:
        transform.memory_format = torch.channels_last
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(1)
    raw = {"x": torch.randint(0, 256, (BATCH, 3, IMAGE, IMAGE), generator=g, device=dev, dtype=torch.uint8)}
    for kind, dim, field, _ in synthetic.RESNET_CONFIGS[model][1]:
        raw[field] = (torch.randint(0, dim, (BATCH,), generator=g, device=dev) if kind == "cls"
                      else torch.randn(BATCH, dim, generator=g, device=dev))
    from frl_b200.solver_worker import LossLog
    log = LossLog(len(worker.criterion.loss_names), 1 << 12, dev)
    from frl_b200.types import Split
    state = {"i": 0}

    def step():
        data, target = transform.apply(raw, Split.TRAIN, torch.bfloat16)
        worker.criterion.set_step_sink(log.row(state["i"]), log.nan_flag)
        worker._pass_one_minibatch(state["i"], Split.TRAIN, data, target)
        state["i"] += 1
    return worker, step


def time_pair(model, graph, rounds, steps, warmup):
    import torch
    arms = {layout: make_worker(model, layout == "NHWC", graph)[1] for layout in ("NCHW", "NHWC")}
    for step in arms.values():
        for _ in range(warmup):
            step()
    torch.cuda.synchronize()
    per = {k: [] for k in arms}
    for _ in range(rounds):
        for layout, step in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(steps):
                step()
            e1.record()
            torch.cuda.synchronize()
            per[layout].append(e0.elapsed_time(e1) / steps)
    return {k: {"median_ms": round(statistics.median(v), 2), "min_ms": round(min(v), 2), "max_ms": round(max(v), 2),
                "rounds_ms": [round(x, 2) for x in v]} for k, v in per.items()}


CONVERSION_KEYS = ("nchwtonhwc", "nhwctonchw")


def profile_arm(model, layout, steps=5):
    import torch
    from torch.profiler import ProfilerActivity, profile
    _, step = make_worker(model, layout == "NHWC", False)
    for _ in range(3):
        step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            step()
        torch.cuda.synchronize()
    conv_us, copy_us, total_us, names = 0.0, 0.0, 0.0, {}
    for ev in prof.key_averages():
        us = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
        if us <= 0 or ev.key.startswith("aten::") or ev.key.startswith("cuda"):
            continue
        total_us += us
        k = ev.key.lower()
        if any(c in k for c in CONVERSION_KEYS):
            conv_us += us
            names[ev.key[:90]] = round(us / steps, 1)
        elif "copy" in k and ("elementwise" in k or "direct_copy" in k or "copy_kernel" in k):
            copy_us += us
            names[ev.key[:90]] = round(us / steps, 1)
    return {"cudnn_layout_conversion_us_per_step": round(conv_us / steps, 1),
            "aten_copy_us_per_step": round(copy_us / steps, 1),
            "device_us_per_step": round(total_us / steps, 1), "kernels": names}


def peak_memory(model, layout, steps):
    import torch
    _, step = make_worker(model, layout == "NHWC", False)
    torch.cuda.reset_peak_memory_stats()
    for _ in range(steps):
        step()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() / 2 ** 30


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="resnet18,resnet50x4")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--mem-steps", type=int, default=3)
    ap.add_argument("--json", default=None)
    ap.add_argument("--mem-arm", default=None, help=argparse.SUPPRESS)       # model:layout, in a child process
    args = ap.parse_args()
    import torch
    import frl_b200  # noqa: F401
    os.environ.setdefault("FRL_B200_CUDNN_BENCHMARK", "1")
    if args.mem_arm:
        model, layout = args.mem_arm.split(":")
        print(json.dumps({"peak_gib": round(peak_memory(model, layout, args.mem_steps), 2)}))
        return
    torch.cuda.set_device(0)
    import pynvml
    pynvml.nvmlInit()
    h = pynvml.nvmlDeviceGetHandleByIndex(0)
    card = {"name": pynvml.nvmlDeviceGetName(h), "power_limit_w": pynvml.nvmlDeviceGetPowerManagementLimit(h) / 1e3}
    card["name"] = card["name"].decode() if isinstance(card["name"], bytes) else card["name"]
    out = {"card": card, "batch": BATCH, "image": IMAGE, "precision": "bf16", "inputs": "uint8, K5 on the device",
           "rounds": args.rounds, "steps_per_round": args.steps, "models": {}}
    print(json.dumps(card), flush=True)
    for model in args.models.split(","):
        res = out["models"][model] = {"optimizer": CONFIGS[model]}
        for graph in (False, True):
            key = "graph" if graph else "eager"
            res[key] = time_pair(model, graph, args.rounds, args.steps, args.warmup)
            print(json.dumps({model: {key: res[key]}}), flush=True)
            torch.cuda.empty_cache()
        for layout in ("NCHW", "NHWC"):
            res.setdefault("profile", {})[layout] = profile_arm(model, layout)
            print(json.dumps({model: {"profile": {layout: res["profile"][layout]}}}), flush=True)
            torch.cuda.empty_cache()
            child = subprocess.run([sys.executable, os.path.abspath(__file__), "--mem-arm", "%s:%s" % (model, layout),
                                    "--mem-steps", str(args.mem_steps)], capture_output=True, text=True)
            if child.returncode != 0:
                raise RuntimeError(child.stderr[-3000:])
            res.setdefault("peak_gib", {})[layout] = json.loads(child.stdout.strip().splitlines()[-1])["peak_gib"]
            print(json.dumps({model: {"peak_gib": {layout: res["peak_gib"][layout]}}}), flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
