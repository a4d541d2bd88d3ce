"""Muon's update on the headline MLP's shapes (1 GPU): K14 + K2-mt (``FusedMuon.apply_table``)
against stock ``torch.optim.Muon`` + ``torch.optim.Adam(foreach=True)`` on the same parameters
and bf16 gradients, and Adam alone (K2-mt over every tensor) for scale.  The arms alternate over
5 rounds of 50 updates; each round's time comes from CUDA events around the 50 updates and the
table reports the median with min and max.  Memory: peak and resident allocated bytes per arm,
each in a fresh process.

    python tools/bench_muon.py [--rounds 5] [--steps 50] [--json out.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import torch  # noqa: E402
import torch.nn as nn  # noqa: E402

import frl_b200  # noqa: E402,F401
from frl_b200 import fused_optim  # noqa: E402
from frl_b200.arena import ParamArena  # noqa: E402
from frl_b200.multi_tensor import GradSegTable  # noqa: E402
from frl_b200.types import Precision  # noqa: E402

DEV = torch.device("cuda", 0)
# the headline MLP: 3 trunk Linear(4096, 4096), heads 4096->1000 and 4096->64, with their biases
SHAPES = [(4096, 4096), (4096,)] * 3 + [(1000, 4096), (1000,), (64, 4096), (64,)]
ARMS = ["k14", "torch", "adam"]


def build(arm):
    torch.manual_seed(0)
    params = [nn.Parameter(torch.randn(sh) * 0.02) for sh in SHAPES]
    grads = [torch.randn(sh, device=DEV).bfloat16() for sh in SHAPES]
    if arm == "torch":
        ps = [nn.Parameter(p.detach().to(DEV)) for p in params]
        for p, g in zip(ps, grads):
            p.grad = g.float()
        mats = [p for p in ps if p.ndim == 2]
        om = torch.optim.Muon(mats, lr=1e-3, weight_decay=1e-5, adjust_lr_fn="match_rms_adamw")
        oa = torch.optim.Adam([p for p in ps if p.ndim != 2], lr=1e-3, weight_decay=1e-5, foreach=True)

        def step():
            om.step()
            oa.step()
        return step
    arena = ParamArena(params, device=DEV, precision=Precision.BF16)
    opt = (fused_optim.FusedMuon(arena, lr=1e-3, weight_decay=1e-5) if arm == "k14"
           else fused_optim.FusedAdam(arena, lr=1e-3, weight_decay=1e-5))
    table = GradSegTable(arena.slots, DEV)
    for s, g in zip(arena.slots, grads):
        table.point(s, g.data_ptr(), g.dtype)
    table.upload()

    def step():
        opt.begin_step()
        opt.apply_table(table)
        opt.end_step()
    return step


def memory(arm):
    step = build(arm)
    step()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    step()
    torch.cuda.synchronize()
    print(json.dumps({"arm": arm, "peak_MiB": torch.cuda.max_memory_allocated() / 2 ** 20,
                      "resident_MiB": torch.cuda.memory_allocated() / 2 ** 20}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--json", default=None)
    ap.add_argument("--memory-arm", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.memory_arm:
        memory(args.memory_arm)
        return
    steps = {arm: build(arm) for arm in ARMS}
    for arm in ARMS:
        for _ in range(3):
            steps[arm]()
    torch.cuda.synchronize()
    times = {arm: [] for arm in ARMS}
    for _ in range(args.rounds):
        for arm in ARMS:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.steps):
                steps[arm]()
            e1.record()
            torch.cuda.synchronize()
            times[arm].append(e0.elapsed_time(e1) / args.steps)
    rows = []
    for arm in ARMS:
        res = subprocess.run([sys.executable, os.path.abspath(__file__), "--memory-arm", arm], capture_output=True,
                             text=True, check=True)
        mem = json.loads(res.stdout.strip().splitlines()[-1])
        t = times[arm]
        rows.append({"arm": arm, "update_ms_median": round(statistics.median(t), 3), "min": round(min(t), 3),
                     "max": round(max(t), 3), "peak_MiB": round(mem["peak_MiB"], 1),
                     "resident_MiB": round(mem["resident_MiB"], 1)})
        print(json.dumps(rows[-1]), flush=True)
    k14, ref = rows[0]["update_ms_median"], rows[1]["update_ms_median"]
    print(json.dumps({"k14_over_torch_muon": round(k14 / ref, 3)}), flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
