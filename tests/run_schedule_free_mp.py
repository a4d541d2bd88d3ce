"""Two or more ranks under torch.distributed.run: Schedule-Free AdamW and SGD through the bucket pipeline
with the real kernels.  Prints SF_MP_OK per rank.

Gradients are all-reduced per bucket in place, then one ``frl_sf_*`` launch per bucket (the eager
per-bucket K2 path; Schedule-Free has no fused NVLS step).  The replicas agree bit for bit (y, z and
exp_avg_sq), and match one GPU at the global batch to fp32 reassociation of the summed gradient.

    python -m torch.distributed.run --nproc-per-node 2 tests/run_schedule_free_mp.py [--backend nccl]

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
from frl_b200.types import OptAlgorithm, OptimOpts, ScheduleFree  # noqa: E402

STEPS, BATCH = 4, 64
OPTS = {"adamw": OptimOpts(algo=OptAlgorithm.ADAM, lr=1e-3, weightDecay=0.1),
        "sgd": OptimOpts(algo=OptAlgorithm.SGD, lr=1e-2, momentum=0.9, weightDecay=0.1)}


def _net():
    return nn.Sequential(nn.Linear(256, 512), nn.ReLU(), nn.Linear(512, 384), nn.ReLU(), nn.Linear(384, 10))


def train(dev, rank, world, rule):
    torch.manual_seed(5 + rank)                      # replicas differ until the broadcast
    net = _net().to(dev)
    arena = ParamArena(net.parameters(), device=dev)
    opt = fused_optim.create_fused_optimizer(arena, OPTS[rule], schedule_free=ScheduleFree(warmup_steps=2))
    assert isinstance(opt, fused_optim.FusedScheduleFree)
    pipe = grad_sync.GradBucketPipeline(arena, opt, world_size=world, bucket_cap_mb=0.25, eager_update=True)
    if world > 1:
        assert pipe.eager and len(pipe.buckets) > 1 and pipe.nvls is None
        pipe.broadcast_parameters(src=0)
    g = torch.Generator(device=dev).manual_seed(11)
    for _ in range(STEPS):
        x = torch.randn(BATCH, 256, generator=g, device=dev)
        pipe.begin_step()
        net(x[rank::world]).square().mean().backward()
        pipe.finish_step()
    torch.cuda.synchronize()
    pipe.remove_hooks()
    assert opt.hyper["k"] == STEPS
    return torch.cat([arena.master] + [opt._state(n) for n in sorted(opt._vec)])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--backend", default="nccl")
    args = ap.parse_args()
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    dev = torch.device("cuda", int(os.environ["LOCAL_RANK"]) if args.backend == "nccl" else 0)
    torch.cuda.set_device(dev)
    dist.init_process_group(args.backend, rank=rank, world_size=world)
    for rule in ("adamw", "sgd"):
        got = train(dev, rank, world, rule)
        first = got.clone()
        dist.broadcast(first, src=0)
        assert torch.equal(first, got), "%s: replicas differ" % rule
        want = train(dev, 0, 1, rule)
        # the summed gradient differs from the single-GPU one by fp32 reassociation only
        torch.testing.assert_close(got, want, rtol=1e-4, atol=1e-6)
        print("rank %d %s: replicas bit-identical, within fp32 reassociation of 1 GPU at the global batch"
              % (rank, rule), flush=True)
    dist.barrier()
    print("SF_MP_OK rank %d" % rank, flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
