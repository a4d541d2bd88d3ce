"""Two or more ranks under torch.distributed.run: bf16 master weights with stochastic rounding through the
bucket pipeline with the real kernels (per-bucket all-reduce, then frl_*_sr launches per bucket; buckets
that straddle the model / criterion boundary split in two).  Prints MASTER_WEIGHTS_MP_OK per rank.

* The replicas agree bit for bit (bf16 weights, the criterion's fp32 master, optimizer state).
* Against one GPU at the global batch: the rounding draws depend on arena index and update count only,
  so the runs differ only where the all-reduced gradient's reassociation moves a value across a
  rounding threshold.
* The fused NVLS step (K7) is not used with bf16 master weights, so there is no NCCL-only arm: with
  ``--backend gloo`` (both ranks on GPU 0) the script says ``MASTER_WEIGHTS_NCCL not run``.

    python -m torch.distributed.run --nproc-per-node 2 tests/run_master_weights_mp.py [--backend nccl]
"""
import argparse
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402
import torch.nn as nn  # noqa: E402

import frl_b200  # noqa: E402,F401
from frl_b200 import fused_optim, grad_sync  # noqa: E402
from frl_b200.arena import ParamArena  # noqa: E402
from frl_b200.types import MasterWeights, OptAlgorithm, OptimOpts, Precision  # noqa: E402

STEPS, BATCH = 4, 64


def _net():
    return nn.Sequential(nn.Linear(256, 512), nn.ReLU(), nn.Linear(512, 384), nn.ReLU(), nn.Linear(384, 10))


def train(dev, rank, world, algo):
    torch.manual_seed(5 + rank)                      # replicas differ until the broadcast
    net = _net().to(dev)
    scale = nn.Parameter(torch.ones(10, device=dev) + rank)       # a criterion parameter (fp32 master)
    arena = ParamArena(net.parameters(), [scale], device=dev, precision=Precision.BF16,
                       master_weights=MasterWeights.BF16)
    opts = OptimOpts(algo=algo, lr=1e-2 if algo == OptAlgorithm.ADAM else 0.05, momentum=0.9, weightDecay=1e-3)
    opt = fused_optim.create_fused_optimizer(arena, opts)
    assert opt.sr
    pipe = grad_sync.GradBucketPipeline(arena, opt, world_size=world, bucket_cap_mb=0.25, first_bucket_mb=0.25,
                                        eager_update=True)
    if world > 1:
        assert pipe.eager and len(pipe.buckets) > 1 and pipe.nvls is None
        # the bucket holding the last Linear and the criterion parameter is launched in two parts
        assert any(b.lo < arena.model_end < b.hi for b in pipe.buckets)
        pipe.broadcast_parameters(src=0)
    g = torch.Generator(device=dev).manual_seed(11)
    for _ in range(STEPS):
        x = torch.randn(BATCH, 256, generator=g, device=dev)
        pipe.begin_step()
        out = net(x[rank::world].to(torch.bfloat16)).float()
        (out.square() * scale).mean().backward()
        pipe.finish_step()
    torch.cuda.synchronize()
    pipe.remove_hooks()
    state = torch.cat([v.flatten() for v in opt._vec.values()])
    return arena.lp.float().clone(), arena.master.clone(), state


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--backend", default="nccl")
    args = ap.parse_args()
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    dev = torch.device("cuda", int(os.environ["LOCAL_RANK"]) if args.backend == "nccl" else 0)
    torch.cuda.set_device(dev)
    dist.init_process_group(args.backend, rank=rank, world_size=world)
    for algo in (OptAlgorithm.SGD, OptAlgorithm.ADAM):
        w, m, st = train(dev, rank, world, algo)
        for name, v in (("weights", w), ("criterion master", m), ("state", st)):
            first = v.clone()
            dist.broadcast(first, src=0)
            assert torch.equal(first, v), "replicas differ: %s (%s)" % (name, algo.value)
        w1, m1, _ = train(dev, 0, 1, algo)
        err = float((w - w1).norm() / (w1 - _initial_arena(dev)).norm())
        # the all-reduced bf16 gradient differs from the one-GPU gradient in rounding; Adam's division by
        # sqrt(v) carries that into the weights where v is small.  Measured on an H100 (2 ranks, gloo):
        # 0.024 (SGD), 0.051 (Adam)
        assert err < 0.1, (algo.value, err)
        torch.testing.assert_close(m, m1, rtol=1e-3, atol=1e-5)
        print("rank %d %s: update gap to 1 GPU at the global batch %.2e" % (rank, algo.value, err), flush=True)
    if rank == 0:
        print("MASTER_WEIGHTS_NCCL %s" % ("ran (the per-bucket NCCL path above)" if args.backend == "nccl"
                                          else "not run: needs --backend nccl with one GPU per rank"), flush=True)
    dist.barrier()
    print("MASTER_WEIGHTS_MP_OK rank %d" % rank, flush=True)
    dist.destroy_process_group()


def _initial_arena(dev):
    """The bf16 weights rank 0 starts from (the broadcast source), in arena layout."""
    torch.manual_seed(5)
    net = _net().to(dev)
    arena = ParamArena(net.parameters(), [nn.Parameter(torch.ones(10, device=dev))], device=dev,
                       precision=Precision.BF16, master_weights=MasterWeights.BF16)
    return arena.lp.float().clone()


if __name__ == "__main__":
    main()
