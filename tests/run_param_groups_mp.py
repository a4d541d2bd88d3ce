"""Two or more ranks under torch.distributed.run: param groups through the bucket pipeline with the real
kernels.  Prints PARAM_GROUPS_MP_OK per rank.

Three groups (the first weight at half the lr, every 1-D parameter without weight decay, the rest at
OptimOpts' values).  With groups the pipeline all-reduces the gradients per bucket, with no eager
update and no fused NVLS step, then runs one grouped table launch (K2-mt grouped) over the reduced
arena gradients.  Arms: SGD-momentum, AdamW, and SGD-momentum with gradient accumulation (k = 2, the
accumulator all-reduced per bucket).  In each arm the replicas agree bit for bit (weights and state),
and they match one GPU at the global batch within fp32 reassociation of the summed gradient.

The run uses the backend it is given: ``--backend gloo`` puts both ranks on GPU 0, ``--backend nccl``
needs one GPU per rank.  Under gloo the NCCL run prints ``PARAM_GROUPS_NCCL not run`` and why.

    python -m torch.distributed.run --nproc-per-node 2 tests/run_param_groups_mp.py [--backend nccl]
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
from frl_b200.types import OptAlgorithm, OptimOpts  # noqa: E402

STEPS, BATCH = 4, 64
ARMS = {
    "sgd": (OptimOpts(algo=OptAlgorithm.SGD, lr=1e-2, momentum=0.9, weightDecay=0.1), {}, 1, "momentum_buffer"),
    "adamw": (OptimOpts(algo=OptAlgorithm.ADAM, lr=1e-3, weightDecay=0.1), {"adamw": True}, 1, "exp_avg"),
    "sgd_accum": (OptimOpts(algo=OptAlgorithm.SGD, lr=1e-2, momentum=0.9, weightDecay=0.1), {}, 2,
                  "momentum_buffer"),
}


def _net():
    return nn.Sequential(nn.Linear(256, 512), nn.LayerNorm(512), nn.ReLU(), nn.Linear(512, 384), nn.ReLU(),
                         nn.Linear(384, 10))


def _groups(net, lr):
    return fused_optim.resolve_param_groups(net, [], [
        {"params": [net[0].weight], "lr": 0.5 * lr},
        {"params": [p for p in net.parameters() if p.ndim <= 1], "weight_decay": 0.0}])


def train(arm, dev, rank, world):
    opts, kw, accum, state_name = ARMS[arm]
    torch.manual_seed(5 + rank)                      # replicas differ until the broadcast
    net = _net().to(dev)
    arena = ParamArena(net.parameters(), device=dev)
    opt = fused_optim.create_fused_optimizer(arena, opts, param_groups=_groups(net, opts.lr), **kw)
    assert opt.grouped and len(opt.param_groups) == 3
    pipe = grad_sync.GradBucketPipeline(arena, opt, world_size=world, bucket_cap_mb=0.25, eager_update=True,
                                        accumulation=accum)
    assert pipe.whole_tensors and not pipe.eager and pipe.nvls is None
    if world > 1:
        assert len(pipe.buckets) > 1
        pipe.broadcast_parameters(src=0)
    g = torch.Generator(device=dev).manual_seed(11)
    for step in range(STEPS * accum):
        x = torch.randn(BATCH, 256, generator=g, device=dev)
        if accum > 1:
            pipe.set_microbatch(first=step % accum == 0, closes=step % accum == accum - 1, weight=1.0,
                                group_scale=1.0 / accum)
        pipe.begin_step()
        net(x[rank::world]).square().mean().backward()
        pipe.finish_step()
    torch.cuda.synchronize()
    assert opt._steps == STEPS
    pipe.remove_hooks()
    return torch.cat([p.detach().reshape(-1).float() for p in net.parameters()]), opt._state(state_name).clone()


def _same_on_every_rank(t):
    first = t.clone()
    dist.broadcast(first, src=0)
    return torch.equal(first, t)


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
    for arm in ARMS:
        got, state = train(arm, dev, rank, world)
        assert _same_on_every_rank(got), "%s: replicas differ" % arm
        assert _same_on_every_rank(state), "%s: optimizer state differs across replicas" % arm
        want, want_state = train(arm, dev, 0, 1)
        # one GPU at the global batch: the per-rank gradient means summed in another order, so fp32
        # reassociation only; measured against the update size to stay meaningful for every weight
        moved = (want - p0).abs().max()
        err = (got - want).abs().max()
        assert err <= 1e-3 * moved, (arm, float(err), float(moved))
        torch.testing.assert_close(state, want_state, rtol=1e-3, atol=1e-6)
        print("rank %d %s: replicas bit-equal, max |w - w_1gpu| %.3e of a max update %.3e"
              % (rank, arm, float(err), float(moved)), flush=True)
    if rank == 0:
        if args.backend == "nccl":
            print("PARAM_GROUPS_NCCL ok world %d" % world, flush=True)
        else:
            print("PARAM_GROUPS_NCCL not run: %s" % (
                "needs --backend nccl and one GPU per rank; %d GPU(s) visible" % torch.cuda.device_count()),
                flush=True)
    dist.barrier()
    print("PARAM_GROUPS_MP_OK rank %d" % rank, flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
