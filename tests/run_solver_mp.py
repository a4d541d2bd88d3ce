"""Helper for test_multiprocess_entry_point_with_pipes: runs LocalSolver.solve in its default
(multi-process) mode from a fresh interpreter, so the parent holds no CUDA context and the
ranks can be forked exactly as in the reference."""
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import frl_b200  # noqa: E402,F401
from frl_b200 import synthetic  # noqa: E402
from frl_b200.local_solver import LocalSolver  # noqa: E402
from oracle.make_golden import CONFIGS  # noqa: E402


def main(save_dir: str) -> None:
    ns = synthetic.api_namespace("frl_b200")
    t = ns.types
    n_gpu = torch.cuda.device_count()
    run_opts = t.RunOpts(optim=t.OptimOpts(algo=t.OptAlgorithm.SGD, lr=CONFIGS["toy_sgd"][1]), batchSize=64,
                         nEpochs=2, numThreads=0, numVisualizedSamples=4)
    torch.manual_seed(0)
    problem = synthetic.make_toy_problem(ns, save_dir)
    assert not torch.cuda.is_initialized()
    summary = LocalSolver.solve(run_opts, problem)
    assert summary.epoch == 2
    losses = summary.performance[t.Split.TRAIN].losses
    assert all(np.isfinite(v) for v in losses.values()), losses
    assert os.path.exists(os.path.join(save_dir, "final_model.pth"))
    if n_gpu == 1:
        g = np.load(os.path.join(REPO, "tests", "golden", "toy_sgd.npz"))
        rows = g["rows"][(g["epoch"] == 2) & g["is_train"]]
        assert abs(losses["reg"] - rows[:, 1].mean()) < 1e-4 * abs(rows[:, 1].mean())
    print("MP_SOLVE_OK world", n_gpu, losses)


if __name__ == "__main__":
    main(sys.argv[1])
