"""Two or more ranks under torch.distributed.run: AdamW through the bucket pipeline with the real
kernels.  Prints ADAMW_MP_OK per rank.

* The per-bucket K2 arm: gradients all-reduced per bucket in place, then one ``frl_adamw`` launch
  per bucket, against one GPU at the global batch.  The replicas agree bit for bit.
* The K7 arm (``frl_nvls_adamw``, fused all-reduce + AdamW + multicast of the weights), only with
  ``--backend nccl`` on two or more GPUs whose driver gives multicast memory: against the NCCL + K2
  arm, as tests/run_ddp_vs_oracle.py compares K7 with NCCL + K2 for the other rules.  Elsewhere it
  prints ``ADAMW_K7 not run`` and why.

    python -m torch.distributed.run --nproc-per-node 2 tests/run_adamw_mp.py [--backend nccl]

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
OPTS = OptimOpts(algo=OptAlgorithm.ADAM, lr=1e-2, weightDecay=0.1)


def _net():
    return nn.Sequential(nn.Linear(256, 512), nn.ReLU(), nn.Linear(512, 384), nn.ReLU(), nn.Linear(384, 10))


def train(dev, rank, world, alloc=None):
    from frl_b200.symm import make_link
    torch.manual_seed(5 + rank)                      # replicas differ until the broadcast
    net = _net().to(dev)
    arena = ParamArena(net.parameters(), device=dev, shared_allocator=alloc)
    opt = fused_optim.create_fused_optimizer(arena, OPTS, LayerAdaptation.NONE, OptimizerState.FP32, False, False,
                                             True)
    assert type(opt) is fused_optim.FusedAdam and opt.adamw
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
    return torch.cat([p.detach().reshape(-1).float() for p in net.parameters()]), opt._state("exp_avg_sq").clone()


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
    # the summed gradient differs from the single-GPU one by fp32 reassociation; Adam's division by
    # sqrt(v) carries such a last-bit change into the weights where v is small
    err = float((got - want).norm() / (want - p0).norm())
    assert err < 1e-3, err
    print("rank %d K2 arm: update gap to 1 GPU at the global batch %.2e" % (rank, err), flush=True)

    alloc = None
    if args.backend == "nccl" and world >= 2:
        from frl_b200.symm import try_make_allocator
        alloc = try_make_allocator(dev, world)
    if alloc is None:
        if rank == 0:
            print("ADAMW_K7 not run: %s" % ("needs --backend nccl (one GPU per rank)" if args.backend != "nccl"
                                            else "no multicast memory on these GPUs"), flush=True)
    else:
        w7, s7 = train(dev, rank, world, alloc)
        # in-switch vs ring reduction order only: fp32 rounding, Adam's bound as in run_ddp_vs_oracle
        torch.testing.assert_close(w7, got, rtol=1e-4, atol=5e-6)
        eps = float(torch.finfo(torch.float32).eps)
        torch.testing.assert_close(s7, state, rtol=1e-4, atol=max(1e-9, 4 * world * eps * float(state.abs().max())))
        if rank == 0:
            print("ADAMW_K7 ok world %d" % world, flush=True)
    dist.barrier()
    print("ADAMW_MP_OK rank %d" % rank, flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
