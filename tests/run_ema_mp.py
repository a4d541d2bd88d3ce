"""Two ranks under torch.distributed.run, both on GPU 0 over gloo: the weight EMA through the bucket
pipeline with the real kernels and eager per-bucket updates.  Every rank keeps its own EMA of the
whole master (no fused NVLS step); the EMAs are bit-identical across ranks and equal to a torch lerp
chain over the live weights taken after every update.  Prints EMA_MP_OK per rank.

    python -m torch.distributed.run --nproc-per-node 2 tests/run_ema_mp.py
"""
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
from frl_b200.ema import WeightEMA  # noqa: E402
from frl_b200.types import OptAlgorithm, OptimOpts  # noqa: E402

STEPS, ROWS, DECAY = 6, 16, 0.9


def train(algo, dev, rank, world):
    torch.manual_seed(5 + rank)                      # replicas differ until the broadcast
    net = nn.Sequential(nn.Linear(256, 512), nn.ReLU(), nn.Linear(512, 384), nn.ReLU(), nn.Linear(384, 10)).to(dev)
    if algo == "sgd":
        o = OptimOpts(algo=OptAlgorithm.SGD, lr=0.1, momentum=0.9, weightDecay=1e-4)
    else:
        o = OptimOpts(algo=OptAlgorithm.ADAM, lr=1e-3, weightDecay=1e-4)
    arena = ParamArena(net.parameters(), device=dev)
    opt = fused_optim.create_fused_optimizer(arena, o)
    ema = WeightEMA(arena, net, DECAY)               # the first update copies the broadcast weights
    pipe = grad_sync.GradBucketPipeline(arena, opt, world_size=world, bucket_cap_mb=0.25, eager_update=True,
                                        ema=ema)
    pipe.broadcast_parameters(src=0)
    assert pipe.eager and pipe.nvls is None and len(pipe.buckets) > 1
    chain = None
    g = torch.Generator(device=dev).manual_seed(11)
    for _ in range(STEPS):
        x = torch.randn(ROWS * world, 256, generator=g, device=dev)[rank::world]
        pipe.begin_step()
        net(x).square().mean().backward()
        pipe.finish_step()
        live = arena.master[:arena.model_end]
        chain = live.clone() if chain is None else torch.lerp(chain, live, 1.0 - DECAY)
    torch.cuda.synchronize()
    assert opt._steps == STEPS and ema.updates == STEPS
    pipe.remove_hooks()
    return ema.ema.clone(), chain


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    for algo in ("sgd", "adam"):
        got, chain = train(algo, dev, rank, world)
        assert torch.equal(got, chain), (algo, "EMA differs from the lerp chain over the live weights")
        first = got.clone()
        dist.broadcast(first, src=0)
        assert torch.equal(first, got), (algo, "replicas' EMAs differ")
        print("rank %d %s: EMA of %d elements identical across ranks and to the lerp chain" % (rank, algo, got.numel()),
              flush=True)
    dist.barrier()
    print("EMA_MP_OK rank %d" % rank, flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
