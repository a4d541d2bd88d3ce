"""Two ranks under torch.distributed.run (one GPU each, NCCL): LARS and LAMB through the bucket
pipeline with the real kernels (gradients gathered per bucket, all-reduced in place, then one K2-lw
update over the whole table) against one GPU at the global batch.  Prints LAYERWISE_MP_OK per rank.

    python -m torch.distributed.run --nproc-per-node 2 tests/run_layerwise_mp.py [--backend nccl]

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

STEPS, BATCH = 4, 64


def opts(mode, clip):
    if mode == "lars":
        return OptimOpts(algo=OptAlgorithm.SGD, lr=0.5, weightDecay=1e-4, gradientClip=clip)
    return OptimOpts(algo=OptAlgorithm.ADAM, lr=1e-3, weightDecay=1e-2, gradientClip=clip)


def train(mode, clip, dev, rank, world):
    torch.manual_seed(5 + rank)                      # replicas differ until the broadcast
    net = nn.Sequential(nn.Linear(256, 512), nn.ReLU(), nn.Linear(512, 384), nn.ReLU(), nn.Linear(384, 10)).to(dev)
    o = opts(mode, clip)
    arena = ParamArena(net.parameters(), device=dev)
    opt = fused_optim.create_fused_optimizer(arena, o, LayerAdaptation(mode))
    pipe = grad_sync.GradBucketPipeline(arena, opt, world_size=world, clip_norm=o.gradientClip,
                                        bucket_cap_mb=0.25, eager_update=True)
    if world > 1:
        # whole-tensor updates: no eager per-bucket update, no fused NVLS step, no tail split
        assert not pipe.eager and pipe.nvls is None and not pipe._row_split and len(pipe.buckets) > 1
        pipe.broadcast_parameters(src=0)
    g = torch.Generator(device=dev).manual_seed(11)
    for _ in range(STEPS):
        x = torch.randn(BATCH, 256, generator=g, device=dev)
        pipe.begin_step()
        net(x[rank::world]).square().mean().backward()
        pipe.finish_step()
    torch.cuda.synchronize()
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
    for mode, clip in (("lars", 0.0), ("lamb", 0.0), ("lars", 0.01), ("lamb", 0.01)):
        got = train(mode, clip, dev, rank, world)
        first = got.clone()
        dist.broadcast(first, src=0)
        assert torch.equal(first, got), (mode, clip, "replicas differ")
        want = train(mode, clip, dev, 0, 1)
        err = float(((got - want).abs() / (want.abs() + 1e-6)).max())
        torch.testing.assert_close(got, want, rtol=2e-5, atol=1e-6, msg=lambda m: "%s clip %s: %s" % (mode, clip, m))
        print("rank %d %s clip %s: max rel diff to 1 GPU at the global batch %.2e" % (rank, mode, clip, err), flush=True)
    dist.barrier()
    print("LAYERWISE_MP_OK rank %d" % rank, flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
