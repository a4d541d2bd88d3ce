"""Two ranks under torch.distributed.run (one GPU each, NCCL): Adafactor through the bucket pipeline
with the real kernels (gradients all-reduced per bucket in place, then the K2-af launches over the
whole table) against one GPU at the global batch, with and without clipping.  Prints
ADAFACTOR_MP_OK per rank.

    python -m torch.distributed.run --nproc-per-node 2 tests/run_adafactor_mp.py [--backend nccl]

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
from frl_b200.types import LayerAdaptation, OptAlgorithm, OptimizerState, OptimOpts  # noqa: E402

STEPS, BATCH = 4, 64


def train(clip, dev, rank, world):
    torch.manual_seed(5 + rank)                      # replicas differ until the broadcast
    net = nn.Sequential(nn.Linear(256, 512), nn.ReLU(), nn.Linear(512, 384), nn.ReLU(), nn.Linear(384, 10)).to(dev)
    o = OptimOpts(algo=OptAlgorithm.ADAM, lr=1e-2, weightDecay=1e-2, gradientClip=clip)
    arena = ParamArena(net.parameters(), device=dev)
    opt = fused_optim.create_fused_optimizer(arena, o, LayerAdaptation.NONE, OptimizerState.FP32, adafactor=True)
    assert type(opt) is fused_optim.FusedAdafactor
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
    for clip in (0.0, 0.01):
        got = train(clip, dev, rank, world)
        first = got.clone()
        dist.broadcast(first, src=0)
        assert torch.equal(first, got), (clip, "replicas differ")
        want = train(clip, dev, 0, 1)
        err = float(((got - want).abs() / (want.abs() + 1e-6)).max())
        # the summed gradient differs from the single-GPU one by fp32 reassociation (1 ulp)
        torch.testing.assert_close(got, want, rtol=1e-5, atol=1e-6, msg=lambda m: "clip %s: %s" % (clip, m))
        print("rank %d clip %s: max rel diff to 1 GPU at the global batch %.2e" % (rank, clip, err), flush=True)
    dist.barrier()
    print("ADAFACTOR_MP_OK rank %d" % rank, flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
