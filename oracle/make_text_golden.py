"""TEST INFRASTRUCTURE — generate ``tests/golden/text_lm.npz`` from the LIVE, unmodified reference.

    python -m oracle.make_text_golden

The reference's own ``LocalSolver.solve`` runs on the CPU the next-byte text Problem of
``frl_b200.synthetic.make_text_problem`` instantiated against the reference's API namespace, so
its datasets are the reference's ``TextDataset`` over two seeded corpora
(``synthetic.write_text_corpus``).  Recorded as in ``oracle/make_golden.py``: per-step loss rows,
learning rates, epochs, train/test flags, the order both splits served their samples in, and the
final parameters the reference writes.
"""
import os
import shutil
import sys
import tempfile

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
GOLDEN_DIR = os.path.join(REPO, "tests", "golden")

from oracle.make_golden import BATCH, SEED, _run_opts     # noqa: E402
from oracle.ref_shim import import_reference              # noqa: E402

NAME = "text_lm"
# (algo, lr, scheduler, nEpochs, clip, amsgrad, criterion kind), as make_golden.CONFIGS
CONFIG = ("sgd", 0.02, "drop", 2, 0.0, False, "parallel")
SEQ_LEN = 32
# (file name, lines, seed) of the two corpora; 600 lines at batch 64 leave a ragged last batch
CORPORA = (("train.txt", 600, 1), ("test.txt", 150, 2))


def write_corpora(folder: str):
    """-> (train path, test path) of the corpora the golden run used."""
    import frl_b200  # noqa: F401
    from frl_b200 import synthetic
    paths = []
    for name, n_lines, seed in CORPORA:
        path = os.path.join(folder, name)
        synthetic.write_text_corpus(path, n_lines, seed, seq_len=SEQ_LEN)
        paths.append(path)
    return tuple(paths)


def run_live_reference():
    import frl_b200  # noqa: F401  (only for the synthetic Problem definitions)
    from frl_b200 import synthetic
    import_reference()
    ns = synthetic.api_namespace("frldistml.scaffold")
    from frldistml.scaffold import solver_worker as ref_sw
    from frldistml.scaffold.local_solver import LocalSolver
    from frldistml.scaffold.text_dataset import TextDataset

    save_dir = tempfile.mkdtemp(prefix="frl_text_golden_")
    train_path, test_path = write_corpora(save_dir)
    problem = synthetic.make_text_problem(ns, save_dir, train_path, test_path, seq_len=SEQ_LEN)
    algo, lr, sched, n_epochs, clip, amsgrad, _ = CONFIG
    run_opts = _run_opts(ns, algo, lr, sched, n_epochs, clip, amsgrad)

    rec = {"rows": [], "lr": [], "split": [], "epoch": []}
    served = {id(d): [] for d in problem.datasets}
    orig_step = ref_sw.SolverWorker._pass_one_minibatch
    orig_get = TextDataset.__getitem__

    def step(self, minibatch_idx, data_type, data, target):
        out = orig_step(self, minibatch_idx, data_type, data, target)
        _, total, sub, _ = out
        rec["rows"].append([total.item()] + [sub[n].item() for n in self.criterion.loss_names])
        rec["lr"].append(self.optimizer.param_groups[0]["lr"])
        rec["split"].append(data_type.value)
        rec["epoch"].append(self.cur_epoch)
        return out

    def get(self, idx):
        served[id(self)].append(int(idx))
        return orig_get(self, idx)

    ref_sw.SolverWorker._pass_one_minibatch = step
    TextDataset.__getitem__ = get
    try:
        torch.manual_seed(SEED)
        LocalSolver.solve(run_opts, problem)
    finally:
        ref_sw.SolverWorker._pass_one_minibatch = orig_step
        TextDataset.__getitem__ = orig_get

    final = torch.load(os.path.join(save_dir, "final_model.pth"), weights_only=False)
    out = {"rows": np.asarray(rec["rows"], dtype=np.float32),
           "lr": np.asarray(rec["lr"], dtype=np.float64),
           "epoch": np.asarray(rec["epoch"], dtype=np.int64),
           "is_train": np.asarray([s == "training" for s in rec["split"]]),
           "served_train": np.asarray(served[id(problem.datasets[0])], dtype=np.int64),
           "served_test": np.asarray(served[id(problem.datasets[1])], dtype=np.int64)}
    for i, (k, v) in enumerate(final["state_dict"].items()):
        out["param_%02d" % i] = v.numpy()
    out["param_names"] = np.asarray(list(final["state_dict"].keys()))
    shutil.rmtree(save_dir, ignore_errors=True)
    return out


def main():
    out = run_live_reference()
    os.makedirs(GOLDEN_DIR, exist_ok=True)
    np.savez_compressed(os.path.join(GOLDEN_DIR, NAME + ".npz"), **out)
    print(NAME, "steps", len(out["rows"]), "first/last loss", out["rows"][0, 0], out["rows"][-1, 0])


if __name__ == "__main__":
    main()
