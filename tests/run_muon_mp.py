"""Two ranks under torch.distributed.run (one GPU each, NCCL): Muon through the bucket pipeline with
the real kernels (gradients all-reduced per bucket in place, then one K2-mt launch and K14 over the
whole table) against one GPU at the global batch, with and without clipping.  Every rank runs the
same Newton-Schulz, so the replicas agree bit for bit.  Prints MUON_MP_OK per rank.

    python -m torch.distributed.run --nproc-per-node 2 tests/run_muon_mp.py [--backend nccl]

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
    o = o._replace(momentum=0.9)
    opt = fused_optim.create_fused_optimizer(arena, o, LayerAdaptation.NONE, OptimizerState.FP32, muon=True)
    assert type(opt) is fused_optim.FusedMuon
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
    return arena.master.clone(), [(s.offset, s.end, fused_optim.is_muon_slot(s)) for s in arena.slots]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--backend", default="nccl")
    args = ap.parse_args()
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    dev = torch.device("cuda", int(os.environ["LOCAL_RANK"]) if args.backend == "nccl" else 0)
    torch.cuda.set_device(dev)
    dist.init_process_group(args.backend, rank=rank, world_size=world)
    for clip in (0.0, 0.01):
        torch.manual_seed(5)
        p0 = [p.detach().reshape(-1) for p in nn.Sequential(
            nn.Linear(256, 512), nn.ReLU(), nn.Linear(512, 384), nn.ReLU(), nn.Linear(384, 10)).parameters()]
        got, slots = train(clip, dev, rank, world)
        first = got.clone()
        dist.broadcast(first, src=0)
        assert torch.equal(first, got), (clip, "replicas differ")
        want, _ = train(clip, dev, 0, 1)
        worst = 0.0
        for (lo, hi, is_muon), q in zip(slots, p0):
            a, b, q = got[lo:hi], want[lo:hi], q.to(dev)
            # the summed gradient differs from the single-GPU one by fp32 reassociation (1 ulp),
            # which flips bf16 roundings of the Muon iterate; Newton-Schulz amplifies them, the
            # momentum carries them over the steps, and the changed weights change every later
            # gradient, the Adam parameters' too: measured on an H100, up to 7.8e-2 of a parameter's
            # update after 4 steps.  Every parameter is held to 0.15 of its update.
            err = float((a - b).norm() / (b - q).norm())
            assert err < 0.15, (clip, lo, is_muon, err)
            worst = max(worst, err)
        print("rank %d clip %s: worst update gap to 1 GPU at the global batch %.2e" % (rank, clip, worst),
              flush=True)
    dist.barrier()
    print("MUON_MP_OK rank %d" % rank, flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
