"""Two ranks under torch.distributed.run over gloo, both on GPU 0: a small conv net trained with a
channels_last arena through the bucket pipeline (per-bucket all-reduce, then the fused update) with
the real kernels.  The conv weights keep channels_last strides, the replicas agree bit for bit, and
the run matches one GPU at the global batch to fp32 reassociation.  Prints CHANNELS_LAST_MP_OK per rank.

    python -m torch.distributed.run --nproc-per-node 2 tests/run_channels_last_mp.py
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
from frl_b200.types import LayerAdaptation, OptAlgorithm, OptimizerState, OptimOpts  # noqa: E402

STEPS, BATCH = 4, 16
OPTS = OptimOpts(algo=OptAlgorithm.SGD, lr=0.05, momentum=0.9)


def _net():
    return nn.Sequential(nn.Conv2d(3, 16, 3, padding=1), nn.ReLU(), nn.Conv2d(16, 32, 3, stride=2, padding=1),
                         nn.ReLU(), nn.AdaptiveAvgPool2d(1), nn.Flatten(), nn.Linear(32, 10))


def train(dev, rank, world):
    torch.manual_seed(5 + rank)                      # replicas differ until the broadcast
    net = _net().to(dev)
    arena = ParamArena(net.parameters(), device=dev, channels_last=True)
    opt = fused_optim.create_fused_optimizer(arena, OPTS, LayerAdaptation.NONE, OptimizerState.FP32, False, False,
                                             False)
    pipe = grad_sync.GradBucketPipeline(arena, opt, world_size=world, bucket_cap_mb=0.01, eager_update=True)
    if world > 1:
        pipe.broadcast_parameters(src=0)
    g = torch.Generator(device=dev).manual_seed(11)
    for _ in range(STEPS):
        x = torch.randn(BATCH, 3, 16, 16, generator=g, device=dev)
        pipe.begin_step()
        net(x[rank::world]).square().mean().backward()
        pipe.finish_step()
    torch.cuda.synchronize()
    for m in (net[0], net[2]):
        assert m.weight.is_contiguous(memory_format=torch.channels_last) and not m.weight.is_contiguous()
    pipe.remove_hooks()
    return arena.master.clone()


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    got = train(dev, rank, world)
    first = got.cpu()
    dist.broadcast(first, src=0)
    assert torch.equal(first, got.cpu()), "replicas differ"
    want = train(dev, 0, 1)
    torch.testing.assert_close(got, want, rtol=1e-4, atol=1e-6)
    dist.barrier()
    print("CHANNELS_LAST_MP_OK rank %d" % rank, flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
