"""Two or more ranks under torch.distributed.run: Lion through the bucket pipeline with the real
kernels.  Prints LION_MP_OK per rank.

* The per-bucket K2 arm: gradients all-reduced per bucket in place, then one ``frl_lion`` launch per
  bucket, against one GPU at the global batch.  The replicas agree bit for bit (weights and
  ``exp_avg``).
* The K7 arm (``frl_nvls_lion``, fused all-reduce + Lion + multicast of the weights), only with
  ``--backend nccl`` on two or more GPUs whose driver gives multicast memory: against the NCCL + K2
  arm.  Elsewhere it prints ``LION_K7 not run`` and why.

    python -m torch.distributed.run --nproc-per-node 2 tests/run_lion_mp.py [--backend nccl]

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
LR = 1e-3
OPTS = OptimOpts(algo=OptAlgorithm.SGD, lr=LR, momentum=0.9, weightDecay=0.1)


def _net():
    return nn.Sequential(nn.Linear(256, 512), nn.ReLU(), nn.Linear(512, 384), nn.ReLU(), nn.Linear(384, 10))


def train(dev, rank, world, alloc=None):
    from frl_b200.symm import make_link
    torch.manual_seed(5 + rank)                      # replicas differ until the broadcast
    net = _net().to(dev)
    arena = ParamArena(net.parameters(), device=dev, shared_allocator=alloc)
    opt = fused_optim.create_fused_optimizer(arena, OPTS, LayerAdaptation.NONE, OptimizerState.FP32, False, False,
                                             False, True)
    assert type(opt) is fused_optim.FusedLion
    link = make_link(alloc, arena.grad, arena.master, max_blocks=8) if alloc is not None else None
    pipe = grad_sync.GradBucketPipeline(arena, opt, world_size=world, bucket_cap_mb=0.25, eager_update=True,
                                        nvls_link=link)
    if world > 1:
        assert pipe.eager and len(pipe.buckets) > 1 and (pipe.nvls is not None) == (alloc is not None)
        pipe.broadcast_parameters(src=0)
    g = torch.Generator(device=dev).manual_seed(11)
    for _ in range(STEPS):
        x = torch.randn(BATCH, 256, generator=g, device=dev)
        pipe.begin_step()
        net(x[rank::world]).square().mean().backward()
        pipe.finish_step()
    torch.cuda.synchronize()
    pipe.sync_sharded_state()
    pipe.remove_hooks()
    return torch.cat([p.detach().reshape(-1).float() for p in net.parameters()]), opt._state("exp_avg").clone()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--backend", default="nccl")
    args = ap.parse_args()
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    dev = torch.device("cuda", int(os.environ["LOCAL_RANK"]) if args.backend == "nccl" else 0)
    torch.cuda.set_device(dev)
    dist.init_process_group(args.backend, rank=rank, world_size=world)
    torch.manual_seed(5)
    p0 = torch.cat([p.detach().reshape(-1) for p in _net().parameters()]).to(dev)
    got, state = train(dev, rank, world)
    first = got.clone()
    dist.broadcast(first, src=0)
    assert torch.equal(first, got), "replicas differ"
    want, _ = train(dev, 0, 1)
    m_first = state.clone()
    dist.broadcast(m_first, src=0)
    assert torch.equal(m_first, state), "exp_avg differs across replicas"
    # the summed gradient differs from the single-GPU one by fp32 reassociation: exp_avg within a few
    # roundings; a weight within a few roundings except where such a change flips sign(c) near c = 0,
    # which moves it by 2 lr per flip
    want, want_m = train(dev, 0, 1)
    torch.testing.assert_close(state, want_m, rtol=1e-5, atol=1e-7)
    eps = float(torch.finfo(torch.float32).eps)
    close = (got - want).abs() <= 8 * eps * (want.abs() + LR) * STEPS
    flips = int((~close).sum())
    assert flips <= 8 and float((got - want).abs().max()) <= 2 * LR * STEPS + 1e-6, flips
    print("rank %d K2 arm: %d of %d weights off by a sign flip, the rest within a few roundings of 1 GPU at "
          "the global batch" % (rank, flips, got.numel()), flush=True)

    alloc = None
    if args.backend == "nccl" and world >= 2:
        from frl_b200.symm import try_make_allocator
        alloc = try_make_allocator(dev, world)
    if alloc is None:
        if rank == 0:
            print("LION_K7 not run: %s" % ("needs --backend nccl (one GPU per rank)" if args.backend != "nccl"
                                            else "no multicast memory on these GPUs"), flush=True)
    else:
        w7, s7 = train(dev, rank, world, alloc)
        # in-switch vs ring reduction order only: exp_avg within fp32 rounding, weights up to sign flips
        torch.testing.assert_close(s7, state, rtol=1e-5, atol=1e-7)
        assert int(((w7 - got).abs() > 1e-6).sum()) <= 8
        if rank == 0:
            print("LION_K7 ok world %d" % world, flush=True)
    dist.barrier()
    print("LION_MP_OK rank %d" % rank, flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
