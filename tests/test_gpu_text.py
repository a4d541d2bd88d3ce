"""The text input path on the GPU: the K8t line gather against TextDataset.get_raw_item, the
batched loader against the per-sample DataLoader, and Solver.solve on the next-byte Problem
against the reference's own run (tests/golden/text_lm.npz, oracle/make_text_golden.py)."""
import os
import tempfile

import numpy as np
import pytest
import torch

import frl_b200  # noqa: F401
from frl_b200 import _native, synthetic, text_dataset
from frl_b200.device_loader import DeviceBatchLoader
from frl_b200.solver import Solver
from frl_b200.types import Precision, Split
from oracle import make_text_golden as mtg
from oracle.make_golden import BATCH, SEED
from test_text_dataset import EDGE_FILES

pytestmark = pytest.mark.gpu


def _identity(raw, split):
    return raw


def _corpora(folder):
    paths = []
    for k, (data, _) in enumerate(EDGE_FILES):
        paths.append(os.path.join(folder, "edge%d.txt" % k))
        with open(paths[-1], "wb") as f:
            f.write(data)
    for seed, (n_lines, max_len) in enumerate(((2000, 90), (300, 9000))):
        paths.append(os.path.join(folder, "random%d.txt" % seed))
        synthetic.write_text_corpus(paths[-1], n_lines, seed, seq_len=16, max_len=max_len)
    return paths


def _gather(ds, idx, row_len, pad=0, offset=0):
    """K8t into a [len(idx), row_len] view that starts ``offset`` bytes into its allocation."""
    dev = torch.device("cuda", 0)
    field = ds.pinned_fields["line"]
    addr = field.corpus.pin()
    idx_dev = torch.as_tensor(idx, dtype=torch.int64).to(dev)
    buf = torch.full((len(idx) * row_len + offset + 32,), 0xEE, dtype=torch.uint8, device=dev)
    dst = buf[offset:offset + len(idx) * row_len].view(len(idx), row_len)
    _native.gather_lines(addr, field.corpus.n_bytes, field.corpus.alloc_bytes, field.starts_on(dev), idx_dev, dst,
                         pad=pad)
    torch.cuda.synchronize()
    host = buf.cpu()
    assert (host[:offset] == 0xEE).all() and (host[offset + len(idx) * row_len:] == 0xEE).all()
    return dst.cpu().numpy()


def _want(ds, idx, row_len, pad):
    rows = []
    for i in idx:
        i = int(i) if 0 <= int(i) < len(ds) else 0         # out of range reads line 0
        full = ds._corpus.array[ds._sample_indices[i]:ds._sample_indices[i + 1] - 1]
        n = min(row_len, full.shape[0])
        row = np.full(row_len, pad, dtype=np.uint8)
        row[:n] = full[:n]
        rows.append(row)
    return np.stack(rows)


@pytest.mark.parametrize("row_len", [1, 15, 16, 17, 257, 4097])
def test_gather_lines_equals_get_raw_item(tmp_path, row_len):
    rs = np.random.RandomState(row_len)
    for path in _corpora(str(tmp_path)):
        ds = text_dataset.TextDataset(Split.TRAIN, path, _identity, row_len - 1)
        if len(ds) == 0:
            continue
        for batch in (1, 3, 4096):
            idx = rs.randint(0, len(ds), size=batch)
            got = _gather(ds, idx, row_len)
            want = np.stack([ds.get_raw_item(int(i))["line"] for i in idx])
            assert np.array_equal(got, want), (path, batch)


def test_gather_lines_pad_out_of_range_and_odd_dst_offset(tmp_path):
    path = _corpora(str(tmp_path))[-1]
    for row_len in (17, 257):
        ds = text_dataset.TextDataset(Split.TRAIN, path, _identity, row_len - 1)
        idx = np.concatenate([np.arange(len(ds)), [-1, len(ds), len(ds) + 5, -(1 << 40)]])
        for offset in (0, 1, 7):
            got = _gather(ds, idx, row_len, pad=0xA5, offset=offset)
            assert np.array_equal(got, _want(ds, idx, row_len, 0xA5)), (row_len, offset)


def _loader_batches(ds, batch, seed, depth=2):
    torch.manual_seed(seed)
    ld = DeviceBatchLoader(ds, batch_size=batch, sampler=None, device=torch.device("cuda", 0), depth=depth)
    out = [(d[0].cpu(), t[0][0].cpu()) for d, t, _ in ld]
    return ld, out


def test_device_loader_serves_the_per_sample_batches(tmp_path, ns, monkeypatch):
    path = _corpora(str(tmp_path))[-2]
    fast = synthetic.make_text_problem(ns, str(tmp_path), path, path, seq_len=16, device_batches=True)
    plain = synthetic.make_text_problem(ns, str(tmp_path), path, path, seq_len=16)
    ld, got = _loader_batches(fast.datasets[0], 48, SEED)
    assert ld.path == "kernel" and ld._wire_dtype == {"line": torch.uint8}
    assert ld.h2d_bytes_per_batch == 48 * 17 + 8 * 48
    torch.manual_seed(SEED)
    want = [(d[0], t[0][0]) for d, t, _ in torch.utils.data.DataLoader(plain.datasets[0], batch_size=48, shuffle=True)]
    assert len(got) == len(want) and got[-1][0].shape[0] == len(plain.datasets[0]) % 48
    for (gx, gy), (wx, wy) in zip(got, want):
        assert gx.dtype == wx.dtype == torch.int64 and torch.equal(gx, wx) and torch.equal(gy, wy)
    for bad in ("host", "tma"):
        monkeypatch.setenv("FRL_B200_INPUT_PATH", bad)
        with pytest.raises(ValueError, match="'line'"):
            DeviceBatchLoader(fast.datasets[0], batch_size=48, sampler=None, device=torch.device("cuda", 0))


def _solve(ns, device_batches, precision=Precision.FP32, **over):
    folder = tempfile.mkdtemp(prefix="frl_b200_text_")
    train, test = mtg.write_corpora(folder)
    problem = synthetic.make_text_problem(ns, folder, train, test, seq_len=mtg.SEQ_LEN,
                                          device_batches=device_batches)
    algo, lr, sched, n_epochs, clip, amsgrad, _ = mtg.CONFIG
    t = ns.types
    optim = t.OptimOpts(algo=t.OptAlgorithm(algo), lr=lr,
                        lr_scheduler=t.LRSchedulerOpts(algo=t.LRSchedulerAlgorithm(sched)),
                        gradientClip=clip, amsgrad=amsgrad)
    kw = dict(optim=optim, batchSize=BATCH, nEpochs=n_epochs, numThreads=0, singleThreaded=True,
              numVisualizedSamples=4)
    kw.update(over)
    captured = {}
    orig = Solver.build_worker.__func__

    def spy(cls, args):
        worker, sch, ckpt = orig(cls, args)
        captured["worker"] = worker
        return worker, sch, ckpt

    served = {id(d): [] for d in problem.datasets}
    real_get = text_dataset.TextDataset.__getitem__

    def get(self, idx):
        served[id(self)].append(int(idx))
        return real_get(self, idx)

    Solver.build_worker = classmethod(spy)
    text_dataset.TextDataset.__getitem__ = get
    try:
        torch.manual_seed(SEED)
        list(Solver.solve(t.RunOpts(**kw), problem, group_name=None, init_method="file:///tmp/unused",
                          precision=precision))
    finally:
        Solver.build_worker = classmethod(orig)
        text_dataset.TextDataset.__getitem__ = real_get
    rows = np.concatenate([r for _, _, r in captured["worker"].loss_history])
    return rows, [served[id(d)] for d in problem.datasets], folder, captured["worker"]


def _check_params(g, folder, tol=2e-4):
    final = torch.load(os.path.join(folder, "final_model.pth"), weights_only=False)
    names = list(g["param_names"])
    assert list(final["state_dict"].keys()) == names
    for i, k in enumerate(names):
        np.testing.assert_allclose(final["state_dict"][k].numpy(), g["param_%02d" % i], rtol=tol, atol=tol * 1e-2)


@pytest.mark.parametrize("graph", ["0", "1"])
def test_text_problem_on_the_device_path_matches_reference(ns, golden_dir, monkeypatch, graph):
    monkeypatch.setenv("FRL_B200_CUDA_GRAPH", graph)
    g = np.load(os.path.join(golden_dir, "text_lm.npz"))
    # metricAmortizationSchedule 5 > the loader's 3 slots: retained targets outlive slot reuse
    rows, served, folder, worker = _solve(ns, device_batches=True, metricAmortizationSchedule=5)
    assert served == [[], []]                      # the per-sample __getitem__ never ran
    if graph == "1":
        assert worker.graphed is not None
    assert rows.shape == g["rows"].shape
    np.testing.assert_allclose(rows, g["rows"], rtol=1e-5, atol=1e-6)
    _check_params(g, folder)


def test_text_problem_per_sample_path_serves_the_golden_order(ns, golden_dir):
    g = np.load(os.path.join(golden_dir, "text_lm.npz"))
    rows, served, folder, _ = _solve(ns, device_batches=False)
    assert served[0] == list(g["served_train"]) and served[1] == list(g["served_test"])
    np.testing.assert_allclose(rows, g["rows"], rtol=1e-5, atol=1e-6)
    _check_params(g, folder)


def test_text_problem_bf16_tracks_the_reference(ns, golden_dir):
    g = np.load(os.path.join(golden_dir, "text_lm.npz"))
    rows, _, _, worker = _solve(ns, device_batches=True, precision=Precision.BF16)
    assert worker.arena.lp is not None
    np.testing.assert_allclose(rows, g["rows"], rtol=1e-2, atol=1e-3)


def test_two_ranks_share_one_pinned_corpus(tmp_path):
    """>= 2 GPUs only: both paths give the same loss rows at world size 2, and the ranks share
    the corpus pages (summed proportional set size about one corpus)."""
    import subprocess
    import sys
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    script = os.path.join(os.path.dirname(__file__), "run_text_mp.py")
    out = subprocess.run([sys.executable, script, str(tmp_path)], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
    assert "TEXT_MP_OK" in out.stdout
