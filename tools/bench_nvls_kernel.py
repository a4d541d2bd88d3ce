"""Stand-alone timing of the fused NVLS kernel (K7) and of NCCL all-reduce + K2 on the same
bucket, no concurrent GEMMs:  torchrun --nproc-per-node N tools/bench_nvls_kernel.py"""
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402
import torch.nn as nn  # noqa: E402

import frl_b200  # noqa: E402,F401
from frl_b200 import fused_optim  # noqa: E402
from frl_b200.arena import ParamArena  # noqa: E402
from frl_b200.symm import make_link, try_make_allocator  # noqa: E402
from frl_b200.types import OptAlgorithm, OptimOpts, Precision  # noqa: E402


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    alloc = try_make_allocator(dev, world)
    assert alloc is not None
    n_elems = 4096 * 4096 + 4096          # one MLP layer: the bucket size of the benchmark config
    p = nn.Parameter(torch.randn(n_elems, device=dev) * 0.01)
    arena = ParamArena([p], device=dev, precision=Precision.BF16, shared_allocator=alloc)
    opt = fused_optim.create_fused_optimizer(arena, OptimOpts(algo=OptAlgorithm.SGD, lr=0.01))
    arena.grad.copy_(torch.randn(arena.numel, device=dev) * 1e-3)
    opt._steps = 1
    gbytes = arena.numel * 2
    res = {}
    for blocks in (16, 32, 64, 96, 132):
        link = make_link(alloc, arena.grad, arena.lp, max_blocks=blocks)
        opt.nvls = link
        for _ in range(5):
            opt.apply_range_nvls(0, arena.numel, grad_scale=1.0 / world)
        dist.barrier(); torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(20):
            opt.apply_range_nvls(0, arena.numel, grad_scale=1.0 / world)
        e1.record(); torch.cuda.synchronize()
        res["nvls_%d" % blocks] = e0.elapsed_time(e1) / 20
    opt.nvls = None
    for _ in range(5):
        dist.all_reduce(arena.grad); opt.apply_range(0, arena.numel, grad_scale=1.0 / world)
    dist.barrier(); torch.cuda.synchronize()
    e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
    t_ar = t_k2 = 0.0
    for _ in range(20):
        e0.record(); dist.all_reduce(arena.grad); e1.record()
        opt.apply_range(0, arena.numel, grad_scale=1.0 / world); e2.record()
        torch.cuda.synchronize()
        t_ar += e0.elapsed_time(e1) / 20; t_k2 += e1.elapsed_time(e2) / 20
    if rank == 0:
        link_bytes = gbytes * (1 + 1.0 / world)
        print("K7_STANDALONE world", world, "bucket MB", gbytes / 1e6,
              {k: round(v, 4) for k, v in res.items()},
              "best GB/s per direction", round(link_bytes / (min(res.values()) * 1e-3) / 1e9, 1),
              "| nccl allreduce ms", round(t_ar, 4), "k2 ms", round(t_k2, 4), flush=True)
    dist.barrier()
    os._exit(0)


if __name__ == "__main__":
    main()
