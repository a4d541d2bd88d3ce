#!/usr/bin/env python
"""In-process sweep of the fused NVLS step's launch knobs (grid size, barrier placement) on the
bench workload, one torchrun launch:

    torchrun --nproc-per-node N tools/sweep_nvls.py [--bucket-mb 48] [--blocks 32,66,132] [--steps 40]

Prints one line per configuration (rank 0): ms/step as max over ranks of the CUDA-event time.
"""
import argparse
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import bench  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bucket-mb", type=float, default=48.0)
    ap.add_argument("--blocks", default="32,66,132")
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=8)
    ap.add_argument("--algo", default="sgd")
    ap.add_argument("--sync", default="0,1", help="0 = barriers in-kernel, 1 = separate launches")
    args = ap.parse_args()
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    import frl_b200  # noqa: F401
    from frl_b200 import synthetic
    from frl_b200.graph_step import GraphedTrainStep
    from frl_b200.solver import Solver, SolverWorkerArgs, bind_to_gpu_numa_node
    from frl_b200.solver_worker import LossLog
    from frl_b200.types import Device, Precision

    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    bind_to_gpu_numa_node(local_rank)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    ns = synthetic.api_namespace("frl_b200")
    t = ns.types
    B = 4096
    torch.manual_seed(0)
    save_dir = "/tmp/frl_b200_sweep_%d" % rank
    os.makedirs(save_dir, exist_ok=True)
    problem = bench.build_problem(ns, save_dir)
    os.environ["FRL_B200_BUCKET_MB"] = str(args.bucket_mb)
    os.environ["FRL_B200_CUDA_GRAPH"] = "1"
    os.environ["FRL_B200_NVLS_BLOCKS"] = "1024"          # scratch sized for the largest grid
    wargs = SolverWorkerArgs(run_opts=bench.run_opts_for(ns, args.algo, B), problem=problem,
                             save_dir=save_dir, run_device=Device.GPU, node_idx=0, node_count=1,
                             rank=rank, local_rank=local_rank, world_size=world, group_name=None,
                             init_method="env://", precision=Precision.BF16)
    worker, _, _ = Solver.build_worker(wargs)
    worker.model.train()
    worker.criterion.train()
    link = worker.pipeline.nvls
    gen = torch.Generator(device=dev).manual_seed(1234 + rank)
    pool = []
    for _ in range(4):
        x = torch.randn(B, bench.WIDTH, device=dev, generator=gen)
        y = torch.randint(0, bench.N_CLASSES, (B,), device=dev, generator=gen)
        r = torch.randn(B, bench.REG_DIM, device=dev, generator=gen)
        pool.append(([x], [(y,), (r,)]))
    n_tasks = len(worker.criterion.loss_names)
    log_ring = LossLog(n_tasks, 4096, dev)
    step_no = [0]

    def step():
        i = step_no[0]
        step_no[0] += 1
        data, target = pool[i % 4]
        worker.criterion.set_step_sink(log_ring.row(i), log_ring.nan_flag)
        worker._pass_one_minibatch(i, t.Split.TRAIN, data, target)

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def measure(tag):
        worker.graphed = GraphedTrainStep(worker)          # re-capture with the current knobs
        for _ in range(args.warmup):
            step()
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.steps):
            step()
        e1.record()
        barrier()
        ms = e0.elapsed_time(e1) / args.steps
        if world > 1:
            tv = torch.tensor([ms], device=dev, dtype=torch.float64)
            dist.all_reduce(tv, op=dist.ReduceOp.MAX)
            ms = tv.item()
        if rank == 0:
            print("SWEEP world %d buckets %d (%g MiB) %-26s %.4f ms/step  %.0f samples/s" % (
                world, len(worker.pipeline.buckets), args.bucket_mb, tag, ms, world * B / ms * 1e3), flush=True)

    if link is None:
        measure("no-nvls")
    else:
        for sync in [int(v) for v in args.sync.split(",")]:
            for blocks in [int(b) for b in args.blocks.split(",")]:
                link.max_blocks = blocks
                link.flags = sync
                measure("sync=%s blocks=%d" % ("split" if sync else "inkernel", blocks))
    if world > 1:
        import gc
        worker.graphed = None
        gc.collect()
        barrier()
        os._exit(0)


if __name__ == "__main__":
    main()
