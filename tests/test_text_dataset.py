"""TextDataset against the reference's, bit for bit, and the host side of its batched path.

The reference side is computed live where the reference can be imported and read from
tests/golden/live/text_dataset_samples.pt elsewhere (oracle/live_golden.py)."""
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest
import torch

import frl_b200  # noqa: F401
from frl_b200 import _native, synthetic, text_dataset
from frl_b200.types import Split
from oracle.live_golden import reference_side

# the edge cases of the reference's line-start table: (file bytes, starts)
EDGE_FILES = [
    (b"hello\n\nworld abc\nlast line no nl", [0, 6, 7, 17, 31]),
    (b"a\nbb\n", [0, 2, 5, 4]),
    (b"\n", [0, 1, 0]),
    (b"", [0, -1]),
    (b"\n\nab\r\n\xc3\xa9\x00z", [0, 1, 2, 6, 9]),
]
SEQ_LENS = (1, 6, 64)


def _identity(raw, split):
    return raw


def _files(folder):
    paths = []
    for k, (data, _) in enumerate(EDGE_FILES):
        path = os.path.join(folder, "edge%d.txt" % k)
        with open(path, "wb") as f:
            f.write(data)
        paths.append(path)
    path = os.path.join(folder, "seeded.txt")
    synthetic.write_text_corpus(path, 300, 7, seq_len=6)
    paths.append(path)
    return paths


def _samples(cls, path, seq_len, wrap=str):
    ds = cls(Split.TRAIN, wrap(path), _identity, seq_len)
    items = [ds.get_raw_item(i)["line"] for i in range(len(ds))]
    stacked = np.stack(items) if items else np.zeros((0, seq_len + 1), np.uint8)
    return {"len": len(ds), "dtype": str(items[0].dtype) if items else "uint8",
            "items": torch.from_numpy(stacked.copy())}


def test_samples_match_the_reference_bit_for_bit(tmp_path):
    paths = _files(str(tmp_path))

    def reference():
        from oracle.ref_shim import import_reference
        import_reference()
        import importlib
        ref = importlib.import_module("frldistml.scaffold.text_dataset")
        return {"%s_%d" % (os.path.basename(p), s): _samples(ref.TextDataset, p, s, ref.StoragePath)
                for p in paths for s in SEQ_LENS}

    want, _ = reference_side("text_dataset_samples", reference)
    for p in paths:
        for s in SEQ_LENS:
            key = "%s_%d" % (os.path.basename(p), s)
            got = _samples(text_dataset.TextDataset, p, s)
            assert got["len"] == want[key]["len"], key
            assert got["dtype"] == want[key]["dtype"] == "uint8"
            assert torch.equal(got["items"], want[key]["items"]), key


def test_edge_case_tables_and_samples(tmp_path):
    paths = _files(str(tmp_path))
    for (data, starts), path in zip(EDGE_FILES, paths):
        ds = text_dataset.TextDataset(Split.TRAIN, path, _identity, 6)
        assert ds._sample_indices.dtype == np.int64
        assert ds._sample_indices.tolist() == starts
    ds = text_dataset.TextDataset(Split.TRAIN, paths[0], _identity, 6)
    assert [bytes(ds.get_raw_item(i)["line"]).rstrip(b"\0") for i in range(len(ds))] == \
        [b"hello", b"", b"world a", b"last li"]


def test_paths_may_be_pathlike_or_carry_a_path_attribute(tmp_path):
    import pathlib

    class StorageLike:
        def __init__(self, p):
            self.path = pathlib.PurePosixPath(p)
    path = _files(str(tmp_path))[-1]
    a = text_dataset.TextDataset(Split.TEST, path, _identity, 6)
    for wrapped in (pathlib.Path(path), StorageLike(path)):
        b = text_dataset.TextDataset(Split.TEST, wrapped, _identity, 6)
        assert np.array_equal(a._sample_indices, b._sample_indices)


def test_chunked_line_starts_equal_one_chunk(tmp_path):
    path = _files(str(tmp_path))[-1]
    data = np.fromfile(path, dtype=np.uint8)
    whole = text_dataset.line_starts(data, chunk_bytes=1 << 30)
    for chunk in (1, 7, 16, 333):
        assert np.array_equal(text_dataset.line_starts(data, chunk_bytes=chunk), whole)


def test_corpus_allocation_is_16_byte_aligned_with_a_zero_tail(tmp_path):
    for path in _files(str(tmp_path)):
        corpus = text_dataset.TextDataset(Split.TRAIN, path, _identity, 6)._corpus
        assert corpus.alloc_bytes % 16 == 0 and corpus.alloc_bytes >= max(corpus.n_bytes, 16)
        whole = np.frombuffer(corpus._mm, dtype=np.uint8)
        assert whole.ctypes.data % 16 == 0 and whole.size == corpus.alloc_bytes
        assert not whole[corpus.n_bytes:].any()
        assert bytes(whole[:corpus.n_bytes]) == open(path, "rb").read()


def test_pickle_round_trip_and_dataloader_workers(tmp_path, ns):
    path = _files(str(tmp_path))[-1]
    problem = synthetic.make_text_problem(ns, str(tmp_path), path, path, seq_len=6)
    ds = problem.datasets[0]
    # the problem's transform is a local class; pickle a dataset with a module-level one
    plain = text_dataset.TextDataset(Split.TRAIN, path, _identity, 6)
    clone = pickle.loads(pickle.dumps(plain))
    assert len(clone) == len(plain) == len(ds)
    for i in range(len(ds)):
        assert np.array_equal(clone.get_raw_item(i)["line"], plain.get_raw_item(i)["line"])
        assert np.array_equal(clone[i]["line"], ds.get_raw_item(i)["line"])
    serial = torch.utils.data.default_collate([ds[i] for i in range(len(ds))])
    loader = torch.utils.data.DataLoader(ds, batch_size=len(ds), shuffle=False, num_workers=2)
    (batch,) = list(loader)
    assert torch.equal(batch[0][0], serial[0][0]) and torch.equal(batch[1][0][0], serial[1][0][0])
    assert serial[0][0].dtype == torch.int64 and serial[0][0].shape == (len(ds), 6)


def test_construction_does_not_initialise_cuda(tmp_path):
    path = _files(str(tmp_path))[-1]
    code = ("import sys; sys.path.insert(0, %r)\n"
            "import torch, frl_b200\n"
            "from frl_b200 import synthetic\n"
            "ns = synthetic.api_namespace('frl_b200')\n"
            "p = synthetic.make_text_problem(ns, %r, %r, %r, seq_len=6, device_batches=True)\n"
            "assert len(p.datasets[0]) > 0 and p.datasets[0].pinned_fields['line'].row_len == 7\n"
            "print('CUDA_INIT', torch.cuda.is_initialized())\n"
            % (os.path.dirname(os.path.dirname(os.path.abspath(__file__))), str(tmp_path), path, path))
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr[-3000:]
    assert "CUDA_INIT False" in out.stdout


def test_device_transform_is_opt_in(tmp_path, ns):
    from frl_b200.device_loader import PaddedLines, supports_device_batches
    path = _files(str(tmp_path))[-1]
    plain = synthetic.make_text_problem(ns, str(tmp_path), path, path, seq_len=6)
    fast = synthetic.make_text_problem(ns, str(tmp_path), path, path, seq_len=6, device_batches=True)
    assert not supports_device_batches(plain.datasets[0])
    assert supports_device_batches(fast.datasets[0])
    field = fast.datasets[0].pinned_fields["line"]
    assert isinstance(field, PaddedLines) and field.row_len == 7 and field.pad == 0


def test_gather_lines_argument_errors_without_a_gpu():
    lib = _native.lib()
    fake = 1 << 20                      # never dereferenced: every call below fails validation
    args = dict(corpus=fake, n=100, alloc=112, starts=fake, n_lines=3, idx=fake, dst=fake, rows=4,
                row_len=7, pad=0)

    def call(**over):
        a = dict(args, **over)
        return lib.frl_gather_lines(a["corpus"], a["n"], a["alloc"], a["starts"], a["n_lines"], a["idx"],
                                    a["dst"], a["rows"], a["row_len"], a["pad"], 0, None)

    for name in ("corpus", "starts", "idx", "dst"):
        assert call(**{name: None}) < 0
        assert b"null pointer" in lib.frl_last_error()
    assert call(alloc=100) < 0                     # 100 bytes need 112 allocated
    assert b"rounded up to 16" in lib.frl_last_error()
    assert call(corpus=fake + 8) == -2             # FRL_E_ALIGN
    assert b"aligned" in lib.frl_last_error()
    assert call(pad=256) < 0 and call(n_lines=0) < 0 and call(rows=-1) < 0
