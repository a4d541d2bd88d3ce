"""Multi-GPU parity helper (launched under torchrun by test_multi_gpu_pipeline_matches_oracle,
or by hand:  torchrun --nproc-per-node 2 tests/run_ddp_vs_oracle.py).

N ranks train the toy 2-task model with the real kernels + NCCL bucket all-reduce on their
share of every batch; rank 0 then checks the weights against the single-process CPU oracle fed
the concatenated batch (mean of per-rank mean losses == global mean for MSE/CE with
equal per-rank batch)."""
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import frl_b200  # noqa: E402,F401
from frl_b200 import fused_optim, grad_sync, synthetic  # noqa: E402
from frl_b200.arena import ParamArena  # noqa: E402
from frl_b200.types import OptAlgorithm, OptimOpts  # noqa: E402
from oracle import ref_loop  # noqa: E402


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    torch.backends.cuda.matmul.allow_tf32 = False
    ns = synthetic.api_namespace("frl_b200")
    from frl_b200.symm import make_link, try_make_allocator
    alloc = try_make_allocator(dev, world)
    if rank == 0:
        print("NVLS_AVAILABLE", alloc is not None, flush=True)
    # (algo, clip, nvls): nvls True = barriers as separate launches (default), "inkernel" = inside K7
    combos = [("sgd", 0.0, False), ("adam", 0.0, False), ("rmsprop", 0.0, False), ("sgd", 0.05, False)]
    if alloc is not None:
        combos += [("sgd", 0.0, True), ("adam", 0.0, True), ("rmsprop", 0.0, True), ("sgd", 0.0, "inkernel")]
    nccl_result = {}            # algo -> (weights, optimizer state) of the NCCL + K2 run
    for algo, clip, nvls in combos:
        torch.manual_seed(123 + rank)                 # different init per rank: broadcast must fix
        problem = synthetic.make_toy_problem(ns, "/tmp/unused")
        model = problem.get_model().to(dev)
        crit = problem.get_criterion().to(dev)
        arena = ParamArena(model.parameters(), crit.parameters(), device=dev,
                           shared_allocator=alloc if nvls else None)
        lr = 0.002 if algo == "rmsprop" else 0.02
        opt = fused_optim.create_fused_optimizer(arena, OptimOpts(algo=OptAlgorithm(algo), lr=lr))
        link = make_link(alloc, arena.grad, arena.master, max_blocks=8) if nvls else None
        if link is not None:
            link.flags = 0 if nvls == "inkernel" else 1
        pipe = grad_sync.GradBucketPipeline(arena, opt, world_size=world, clip_norm=clip,
                                            bucket_cap_mb=0.02, first_bucket_mb=0.005, nvls_link=link)
        assert (pipe.nvls is not None) == bool(nvls)
        if pipe._row_split:          # FRL_B200_TAIL_SPLIT_MIN_BYTES=0: the split + early hand-over path
            pipe.patch_linears(model)
            if rank == 0:
                print("TAIL_SPLIT rows", dict(pipe._row_split), "buckets",
                      [(b.lo, b.hi) for b in pipe.buckets[-2:]], flush=True)
        pipe.broadcast_parameters(0)
        assert len(pipe.buckets) >= 3
        g = torch.Generator().manual_seed(7)
        B = 32 * world
        batches = [(torch.rand(B, 64, generator=g), torch.randn(B, 4, generator=g),
                    torch.randint(0, 10, (B,), generator=g)) for _ in range(4)]
        model.train()
        for x, yr, yc in batches:
            sl = slice(rank, None, world)
            out = model([x[sl].to(dev)])
            total, _ = crit(out, [(yr[sl].to(dev),), (yc[sl].to(dev),)])
            pipe.begin_step()
            total.backward()
            pipe.finish_step()
        torch.cuda.synchronize()
        mine = torch.cat([p.detach().reshape(-1).float() for p in model.parameters()])
        gathered = [torch.empty_like(mine) for _ in range(world)]
        dist.all_gather(gathered, mine)
        if rank == 0:
            for other in gathered[1:]:
                assert torch.equal(other, gathered[0]), "replicas diverged"
            torch.manual_seed(123)
            ref_problem = synthetic.make_toy_problem(ns, "/tmp/unused")
            ref = ref_problem.get_model()
            rc = ref_problem.get_criterion()
            ropt = ref_loop.make_optimizer(ref.parameters(), ref_loop.OptimSpec(algo=algo, lr=lr))
            ref.train()
            for x, yr, yc in batches:
                out = ref([x])
                total, _ = ref_loop.parallel_criterion(list(rc.loss_modules), list(rc.loss_weights),
                                                       list(rc.loss_names), out, [(yr,), (yc,)])
                ropt.zero_grad()
                total.backward()
                if clip:
                    torch.nn.utils.clip_grad_norm_(ref.parameters(), clip)
                ropt.step()
            want = torch.cat([p.detach().reshape(-1) for p in ref.parameters()])
            # Adam's m/(sqrt(v)+eps) amplifies fp32 rounding where v is tiny; a step moves a weight by ~lr
            # Adam / RMSprop divide by sqrt(v)+eps: where v is tiny fp32 rounding is amplified; one
            # step moves a weight by ~lr (Adam) or ~10*lr (RMSprop with momentum)
            tol = {"sgd": dict(rtol=2e-4, atol=2e-6), "adam": dict(rtol=1e-3, atol=5e-5),
                   "rmsprop": dict(rtol=2e-3, atol=3e-4)}[algo]
            np.testing.assert_allclose(mine.cpu().numpy(), want.numpy(), **tol)
        # the fused NVLS step against the NCCL + K2 step: identical per-rank forward/backward, only
        # the reduction order differs (in-switch vs ring) -> agreement to fp32 rounding, including
        # the sharded optimizer state once it has been made whole again (collective call)
        pipe.sync_sharded_state()
        state_name = {"sgd": "momentum_buffer", "adam": "exp_avg_sq", "rmsprop": "square_avg"}[algo]
        state = torch.cat([v[state_name].reshape(-1) for v in opt.state_dict()["state"].values()])
        if clip == 0.0 and not nvls:
            nccl_result[algo] = (mine.clone(), state.clone())
        if nvls and rank == 0:
            w_ref, s_ref = nccl_result[algo]
            # a sum of `world` terms in another order differs by <= (world-1) eps sum|g_i|: the
            # bound scales with the magnitude of the terms, not of a (possibly cancelling) result
            # (at world 2 both orders give the same bits).  Adam / RMSprop then divide by sqrt(v):
            # a last-bit change of a gradient moves a weight by a visible fraction of lr where v
            # is tiny, so their bound is the oracle bound above, 10x tighter.
            eps = float(torch.finfo(torch.float32).eps)
            wtol = {"sgd": dict(rtol=2e-5, atol=2e-7 * max(1, world // 2)),
                    "adam": dict(rtol=1e-4, atol=5e-6), "rmsprop": dict(rtol=2e-4, atol=3e-5)}[algo]
            torch.testing.assert_close(mine, w_ref, **wtol)
            torch.testing.assert_close(state, s_ref, rtol=2e-5 if algo == "sgd" else 1e-4,
                                       atol=max(1e-9, 4 * world * eps * float(s_ref.abs().max())))
        if rank == 0:
            print("DDP_PARITY_OK", algo, clip, ("nvls-" + str(nvls)) if nvls else "nccl", "world", world, flush=True)
        pipe.remove_hooks()
        dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
