"""Helper for test_two_ranks_share_one_pinned_corpus: LocalSolver.solve on every GPU (forked
ranks) with the next-byte text Problem, once through the batched device path and once through
the per-sample DataLoader.  Both must report the same losses, and while the device run trains,
the ranks' proportional share (Pss) of the corpus mapping must sum to about one corpus: the
forked ranks page-lock the parent's pages in place instead of copying them."""
import os
import sys
import threading

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import frl_b200  # noqa: E402,F401
from frl_b200 import synthetic  # noqa: E402
from frl_b200.local_solver import LocalSolver  # noqa: E402


def _children(pid: int):
    out = []
    for tid in os.listdir("/proc/%d/task" % pid):
        with open("/proc/%d/task/%s/children" % (pid, tid)) as f:
            out += [int(c) for c in f.read().split()]
    return out


def _mapping_pss(pid: int, addr: int) -> int:
    """Pss in bytes of the mapping of ``pid`` that starts at ``addr`` (0 if none)."""
    want = "%x-" % addr
    found = False
    with open("/proc/%d/smaps" % pid) as f:
        for line in f:
            if "-" in line.split(" ")[0] and not line.startswith(("Pss", "Rss")):
                found = line.startswith(want)
            elif found and line.startswith("Pss:"):
                return int(line.split()[1]) * 1024
    return 0


def run(ns, folder, device_batches, watch=None):
    t = ns.types
    run_opts = t.RunOpts(optim=t.OptimOpts(algo=t.OptAlgorithm.SGD, lr=0.02), batchSize=512, nEpochs=1,
                         numThreads=0, numVisualizedSamples=4)
    problem = synthetic.make_text_problem(ns, folder, os.path.join(folder, "train.txt"),
                                          os.path.join(folder, "test.txt"), device_batches=device_batches)
    corpus = problem.datasets[0]._corpus
    addr = np.frombuffer(corpus._mm, dtype=np.uint8).ctypes.data
    peak = [0]
    stop = threading.Event()

    def sample():
        while not stop.wait(0.05):
            try:
                peak[0] = max(peak[0], sum(_mapping_pss(c, addr) for c in _children(os.getpid())))
            except (FileNotFoundError, ProcessLookupError):
                pass

    th = threading.Thread(target=sample, daemon=True)
    th.start()
    torch.manual_seed(0)
    try:
        summary = LocalSolver.solve(run_opts, problem)
    finally:
        stop.set()
        th.join()
    return summary.performance[t.Split.TRAIN].losses, peak[0], corpus.n_bytes


def main(folder: str) -> None:
    ns = synthetic.api_namespace("frl_b200")
    synthetic.write_text_corpus(os.path.join(folder, "train.txt"), 200000, 1, seq_len=32)
    synthetic.write_text_corpus(os.path.join(folder, "test.txt"), 5000, 2, seq_len=32)
    assert not torch.cuda.is_initialized()
    fast, pss, corpus_bytes = run(ns, folder, True)
    plain, _, _ = run(ns, folder, False)
    for k in plain:
        assert abs(fast[k] - plain[k]) <= 1e-5 * abs(plain[k]), (k, fast[k], plain[k])
    assert 0 < pss <= 1.1 * corpus_bytes, (pss, corpus_bytes)
    print("TEXT_MP_OK world", torch.cuda.device_count(), fast, "corpus Pss over ranks", pss, "of", corpus_bytes)


if __name__ == "__main__":
    main(sys.argv[1])
