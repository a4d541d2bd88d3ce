"""Two ranks under torch.distributed.run (one GPU each over NCCL, or both on GPU 0 over gloo):
gradient accumulation through the bucket pipeline with the real kernels.  Each rank runs microbatches of 16 rows, 2 per update (K10 per
microbatch reading the gradients autograd allocated in place, fp32 all-reduce of the accumulator per
bucket, one update from it), against the same 2 ranks at 32 rows per step without accumulation
(all-reduce + K2 per bucket).  Prints ACCUM_MP_OK per rank.

    python -m torch.distributed.run --nproc-per-node 2 tests/run_accum_mp.py [--backend nccl]

``--backend gloo`` puts both ranks on GPU 0 (NCCL needs one GPU per rank).
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
from frl_b200.types import LayerAdaptation, OptAlgorithm, OptimOpts  # noqa: E402

GROUPS, MICRO = 4, 16          # rows per rank and microbatch


def opts(algo, clip):
    if algo in ("sgd", "lars"):
        return OptimOpts(algo=OptAlgorithm.SGD, lr=0.1, momentum=0.9, weightDecay=1e-4, gradientClip=clip)
    return OptimOpts(algo=OptAlgorithm.ADAM, lr=1e-3, weightDecay=1e-4, gradientClip=clip)


def train(algo, clip, k, dev, rank, world):
    torch.manual_seed(5 + rank)                      # replicas differ until the broadcast
    net = nn.Sequential(nn.Linear(256, 512), nn.ReLU(), nn.Linear(512, 384), nn.ReLU(), nn.Linear(384, 10)).to(dev)
    o = opts(algo, clip)
    arena = ParamArena(net.parameters(), device=dev)
    la = LayerAdaptation.LARS if algo == "lars" else LayerAdaptation.NONE
    opt = fused_optim.create_fused_optimizer(arena, o, la)
    pipe = grad_sync.GradBucketPipeline(arena, opt, world_size=world, clip_norm=o.gradientClip,
                                        bucket_cap_mb=0.25, eager_update=True, accumulation=k)
    assert (pipe.acc is not None) == (k > 1) and len(pipe.buckets) > 1
    pipe.broadcast_parameters(src=0)
    g = torch.Generator(device=dev).manual_seed(11)
    for _ in range(GROUPS):
        # the group's rows on this rank: MICRO of each of the 2 global microbatches
        xs = [torch.randn(MICRO * world, 256, generator=g, device=dev)[rank::world] for _ in range(2)]
        parts = xs if k == 2 else [torch.cat(xs)]
        for j, x in enumerate(parts):
            pipe.set_microbatch(first=j == 0, closes=j == len(parts) - 1, weight=1.0, group_scale=0.5)
            pipe.begin_step()
            net(x).square().mean().backward()
            pipe.finish_step()
    torch.cuda.synchronize()
    assert opt._steps == GROUPS
    pipe.remove_hooks()
    return arena.master.clone()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--backend", default="nccl")
    args = ap.parse_args()
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    dev = torch.device("cuda", int(os.environ["LOCAL_RANK"]) if args.backend == "nccl" else 0)
    torch.cuda.set_device(dev)
    dist.init_process_group(args.backend, rank=rank, world_size=world)
    for algo, clip in (("sgd", 0.0), ("adam", 0.0), ("sgd", 0.05), ("lars", 0.0)):
        got = train(algo, clip, 2, dev, rank, world)
        first = got.clone()
        dist.broadcast(first, src=0)
        assert torch.equal(first, got), (algo, clip, "replicas differ")
        want = train(algo, clip, 1, dev, rank, world)
        err = float(((got - want).abs() / (want.abs() + 1e-6)).max())
        # Adam divides by sqrt(v) + eps: where a gradient element is near zero, the fp32 rounding of
        # two 16-row sums against one 32-row GEMM moves its step by a visible fraction of lr (1e-3)
        atol = 1e-5 if algo == "adam" else 1e-6
        torch.testing.assert_close(got, want, rtol=1e-5, atol=atol, msg=lambda m: "%s clip %s: %s" % (algo, clip, m))
        print("rank %d %s clip %s: max rel diff to batch 32 without accumulation %.2e" % (rank, algo, clip, err),
              flush=True)
    dist.barrier()
    print("ACCUM_MP_OK rank %d" % rank, flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
