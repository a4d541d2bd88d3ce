"""``.idx`` / ``.bin`` indexed datasets: the on-disk format that feeds the loop.

* golden files written by the UNMODIFIED reference's writer (oracle/make_indexed_golden.py) are
  read back frame by frame and compared with what the reference's own reader returned for them
  (``manifest.json``); this repo's writer must reproduce the golden bytes exactly;
* the reference's own tests for this path (tests/test_indexed_dataset.py: header synthesised by
  hand with magic 0 / version 1, write->read round trip, reader survives pickling into another
  process) are restated against this repo's classes;
* writer and reader are compared with the reference's on random frames (live where the reference
  is present, else its recorded side under tests/golden/live);
* the batched path: ``host_fields`` (zero-copy [N, ...] tensors over the mapped .bin) gathered by
  the native host pool equals per-sample ``__getitem__`` + stacking.
"""
import io
import itertools
import json
import multiprocessing
import os
import pickle
from functools import reduce
from operator import mul

import numpy as np
import pytest
import torch

import frl_b200  # noqa: F401
from frl_b200 import _native
from frl_b200 import indexed_dataset as idm
from oracle.live_golden import plain, reference_side
from oracle.make_indexed_golden import FILES, frames_of

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "indexed")


def _reader(name, folder=GOLD):
    return idm.PosixIndexedDatasetReader(idxfile=os.path.join(folder, name + ".idx"),
                                         binfile=os.path.join(folder, name + ".bin"))


@pytest.mark.parametrize("name", sorted(FILES))
def test_reader_returns_what_the_reference_reader_returned(name):
    want = json.load(open(os.path.join(GOLD, "manifest.json")))[name]
    r = _reader(name)
    assert len(r) == want["len"] and str(r.dtype) == want["dtype"]
    assert r.framesize == want["framesize"] and [int(d) for d in r.size] == want["size"]
    frames = frames_of(name)                       # what was pushed into the reference's writer
    for i in range(len(r)):
        got = r[i]
        assert got.dtype == frames[i].dtype and got.shape == frames[i].shape
        assert np.array_equal(got, frames[i])
        assert float(np.asarray(got, dtype=np.float64).sum()) == want["frame_sums"][i]
        assert got.flags.writeable and got.base is None       # a private copy, not a view of the map
    assert np.asarray(r[0]).ravel().tolist() == want["first_frame"]
    with pytest.raises(AssertionError):
        r[len(r)]
    with pytest.raises(AssertionError):
        r[-1]


@pytest.mark.parametrize("name", sorted(FILES))
def test_writer_reproduces_the_reference_writers_bytes(name, tmp_path):
    with idm.IndexedDatasetWriterFactory.get(str(tmp_path / "f.idx"), str(tmp_path / "f.bin")) as w:
        for f in frames_of(name):
            w.push_back(f)
    for ext in (".idx", ".bin"):
        assert (tmp_path / ("f" + ext)).read_bytes() == open(os.path.join(GOLD, name + ext), "rb").read()


def test_writer_rejects_mixed_dtypes_and_empty_datasets():
    w = idm.IndexedDatasetWriter(idxfile=io.BytesIO(), binfile=io.BytesIO())
    with pytest.raises(AssertionError):
        w.flush()                                   # "Cannot write empty dataset"
    w.push_back(np.zeros(3, dtype=np.float32))
    with pytest.raises(AssertionError):
        w.push_back(np.zeros(3, dtype=np.float64))  # "Frames must all have same dtype"


# ---- the reference's own tests, restated (reference tests/test_indexed_dataset.py) -----------------

def _reference_test_content(type_name, num_frames, single_frame_dims, start_value=0):
    """Header synthesised as the reference's test does (:39-87): magic 0, version 1."""
    dtype = np.dtype(type_name)
    frame_dims = [single_frame_dims] * num_frames
    frame_ndims = [0] + [len(d) for d in frame_dims]
    frame_sizes = [0] + [reduce(mul, d, 1) for d in frame_dims]
    index = np.array([0, 1, idm.np_types.index(type_name) + 1, dtype.itemsize, num_frames,
                      sum(frame_ndims), *np.cumsum(frame_ndims), *np.cumsum(frame_sizes),
                      *itertools.chain.from_iterable(frame_dims)], dtype="int64")
    data = np.arange(0, np.cumsum(frame_sizes)[-1], dtype=dtype) + start_value
    return index, data


def _write_pair(folder, base, index, data):
    index.tofile(os.path.join(folder, base + ".idx"))
    data.tofile(os.path.join(folder, base + ".bin"))


def test_reading_element(tmp_path):                          # reference :110-139
    num_frames, dims = 10, (128, 128)
    _write_pair(str(tmp_path), "TEST_FILE", *_reference_test_content("float64", num_frames, dims))
    ds = idm.MultifieldIndexedDataset(str(tmp_path), fields=["TEST"], filenames=["TEST_FILE"])
    assert len(ds) == num_frames
    assert ds[0]["TEST"].shape == dims and ds[num_frames - 1]["TEST"].shape == dims
    n = dims[0] * dims[1]
    for i in (0, 3, num_frames - 1):
        assert np.array_equal(ds[i]["TEST"], i * n + np.arange(n, dtype=np.float64).reshape(dims))
    assert ds.get_raw_item(2)["TEST"].dtype == np.float64


def _mp_worker(blob, orig_len, frames):
    ds = pickle.loads(blob)
    assert orig_len == len(ds), "Dataset size must match original"
    for idx, frame in frames.items():
        assert np.array_equal(ds[idx], frame)


def test_multiprocessing(tmp_path):                          # reference :141-169
    _write_pair(str(tmp_path), "TEST_FILE", *_reference_test_content("float64", 10, (128, 128)))
    ds = _reader("TEST_FILE", str(tmp_path))
    frames = {i: ds[i] for i in (0, len(ds) - 2)}
    blob = pickle.dumps(ds)                                   # the map itself is not pickled
    assert len(blob) < 4096
    p = multiprocessing.get_context("spawn").Process(target=_mp_worker, args=(blob, len(ds), frames))
    p.start()
    p.join()
    assert p.exitcode == 0


def test_write_read(tmp_path):                               # reference :172-187
    data1 = np.arange(100).reshape(10, 5, 2)
    data2 = data1 + 1000
    idx, binf = str(tmp_path / "dataset.idx"), str(tmp_path / "dataset.bin")
    with idm.IndexedDatasetWriterFactory.get(idxfile=idx, binfile=binf) as w:
        w.push_back(data1)
        w.push_back(data2)
    r = idm.PosixIndexedDatasetReader(idxfile=idx, binfile=binf)
    assert np.array_equal(data1, r[0]) and np.array_equal(data2, r[1])


def test_multifield_dataset_checks_lengths(tmp_path):
    idm.write_fields(str(tmp_path), {"a": np.zeros((4, 3), np.float32), "b": np.zeros((5, 2), np.float32)})
    with pytest.raises(AssertionError, match="should have same number of samples"):
        idm.MultifieldIndexedDataset(str(tmp_path), fields=["a", "b"], filenames=["a", "b"])
    with pytest.raises(AssertionError):
        idm.MultifieldIndexedDataset(str(tmp_path), fields=["a"], filenames=["a", "b"])


def test_malformed_index_files_are_rejected(tmp_path):
    good = np.fromfile(os.path.join(GOLD, "pose.idx"), dtype="int64")
    r = idm.IndexedDatasetReader()
    with pytest.raises(ValueError, match="too short"):
        r._init_from_index_data(good[:4])
    with pytest.raises(ValueError, match="truncated"):
        r._init_from_index_data(good[:-3])
    bad = good.copy()
    bad[2] = 8                                               # np_types[7] is None
    with pytest.raises(AssertionError, match="unrecognized type"):
        r._init_from_index_data(bad)
    bad = good.copy()
    bad[3] = 2                                               # itemsize does not match the dtype
    with pytest.raises(AssertionError):
        r._init_from_index_data(bad)


# ---- comparison with the reference ----------------------------------------------------------------

def test_writer_and_reader_match_the_live_reference(tmp_path):
    rs = np.random.RandomState(7)
    cases = []
    for dt, shape, n in [("float32", (3, 4), 5), ("uint8", (2, 3, 5), 7), ("int64", (), 4),
                         ("float64", (128,), 3), ("int16", (1,), 1), ("int8", (4, 1, 2), 9),
                         ("int32", (17,), 33)]:
        cases.append((dt, shape, [np.asarray(rs.randn(*shape) * 50).astype(dt) for _ in range(n)]))
    idx, binf = str(tmp_path / "x.idx"), str(tmp_path / "x.bin")

    def as_bytes(t):
        return t.numpy().tobytes()

    def reference():
        from oracle.ref_shim import import_reference
        import_reference()
        from frldistml.scaffold.storage import StoragePath
        from frldistml.scaffold.storage_layers.dataset import IndexedDatasetWriter as RefWriter
        from frldistml.scaffold.storage_layers.posix_storage import PosixIndexedDatasetReader as RefReader
        out = []
        for _, _, frames in cases:
            ref_i, ref_b = io.BytesIO(), io.BytesIO()
            rw = RefWriter(idxfile=ref_i, binfile=ref_b)
            for f in frames:
                rw.push_back(f)
            rw.flush()
            open(idx, "wb").write(ref_i.getvalue())
            open(binf, "wb").write(ref_b.getvalue())
            ref = RefReader(idxfile=StoragePath(idx), binfile=StoragePath(binf))
            out.append({"idx": torch.frombuffer(bytearray(ref_i.getvalue()), dtype=torch.uint8),
                        "bin": torch.frombuffer(bytearray(ref_b.getvalue()), dtype=torch.uint8),
                        "len": len(ref), "framesize": int(ref.framesize), "dtype": str(np.dtype(ref.dtype)),
                        "frames": [plain(np.asarray(ref[i])) for i in range(len(ref))],
                        "frame_dtypes": [str(np.asarray(ref[i]).dtype) for i in range(len(ref))]})
        return out

    recorded, _ = reference_side("indexed_writer_reader", reference)
    for (dt, shape, frames), ref in zip(cases, recorded):
        mine_i, mine_b = io.BytesIO(), io.BytesIO()
        w = idm.IndexedDatasetWriter(idxfile=mine_i, binfile=mine_b)
        for f in frames:
            w.push_back(f)
        w.flush()
        assert mine_i.getvalue() == as_bytes(ref["idx"]) and mine_b.getvalue() == as_bytes(ref["bin"]), (dt, shape)
        open(idx, "wb").write(as_bytes(ref["idx"]))
        open(binf, "wb").write(as_bytes(ref["bin"]))
        mine = idm.PosixIndexedDatasetReader(idxfile=idx, binfile=binf)
        assert len(mine) == ref["len"] and mine.framesize == ref["framesize"]
        assert str(np.dtype(mine.dtype)) == ref["dtype"]
        for i in range(len(frames)):
            a, b = mine[i], ref["frames"][i]
            assert str(a.dtype) == ref["frame_dtypes"][i] and tuple(a.shape) == tuple(b.shape)
            assert torch.equal(plain(np.asarray(a)), b)


# ---- batched access: mapped .bin -> native host pool ---------------------------------------------

def test_host_fields_gathered_by_the_pool_equal_per_sample_reads(tmp_path):
    rs = np.random.RandomState(3)
    n = 257
    fields = {"img": (rs.rand(n, 3, 16, 16) * 255).astype(np.uint8),
              "pose": rs.randn(n, 6).astype(np.float32),
              "label": rs.randint(0, 10, size=(n, 1)).astype(np.int64)}
    idm.write_fields(str(tmp_path), fields)
    ds = idm.MultifieldIndexedDataset(str(tmp_path), fields=list(fields), filenames=list(fields))
    host = ds.host_fields
    assert set(host) == set(fields)
    pool = _native.HostGatherPool(3)
    idx = torch.randperm(n)[:100].contiguous()
    for name, t in host.items():
        assert t.shape == fields[name].shape and not t.is_pinned()
        assert np.array_equal(t.numpy(), fields[name])                       # zero-copy view of the file
        out = torch.zeros((100,) + tuple(t.shape[1:]), dtype=t.dtype)
        pool.wait(pool.submit(t, idx, out))
        want = np.stack([ds[int(i)][name] for i in idx])                     # the per-sample path
        assert np.array_equal(out.numpy(), want)
    pool.close()


def test_batched_access_refuses_ragged_files(tmp_path):
    idx, binf = str(tmp_path / "r.idx"), str(tmp_path / "r.bin")
    with idm.IndexedDatasetWriterFactory.get(idx, binf) as w:
        w.push_back(np.zeros((2, 3), np.float32))
        w.push_back(np.zeros((4, 3), np.float32))
    r = idm.PosixIndexedDatasetReader(idxfile=idx, binfile=binf)
    assert len(r) == 2 and r[0].shape == (2, 3)               # per-sample reads keep working (frame-0 shape)
    with pytest.raises(ValueError, match="fixed-size frames"):
        r.frames_tensor()


# ---- Concat / Subset containers over indexed datasets (reference dataset.py:518-552) ---------------

def test_concat_and_subset_containers_match_the_live_reference(tmp_path):
    import frl_b200.storage_layers.dataset as my_ds
    rs = np.random.RandomState(9)
    sizes = [5, 1, 7]
    for k, n in enumerate(sizes):
        idm.write_fields(str(tmp_path / ("part%d" % k)),
                         {"a": rs.randn(n, 3).astype(np.float32), "b": rs.randint(0, 9, (n, 2)).astype(np.int64)})

    class Recorder:
        def __init__(self, log, offset=0, field=None):
            self.log, self.offset, self.field = log, offset, field

        def with_dataset_global_offset(self, offset):
            return Recorder(self.log, offset, self.field)

        def with_multifield_dataset_field(self, field):
            self.log.append((self.offset, field))
            return Recorder(self.log, self.offset, field)

    picks = [12, 0, 5, 5, 3]

    def observe(concat, subset):
        log = []
        seen = {"len": len(concat),
                "raw": [{k: (plain(np.asarray(v)), str(np.asarray(v).dtype)) for k, v in concat.get_raw_item(i).items()}
                        for i in range(len(concat))],
                "items": [{k: plain(np.asarray(v)) for k, v in concat[i].items()} for i in range(len(concat))]}
        concat.set_accessor(Recorder(log))
        sub = subset(concat, picks)
        seen.update(log=log, sub_len=len(sub),
                    sub=[{k: plain(np.asarray(sub[j][k])) for k in ("a", "b")} for j in range(len(sub))])
        return seen

    def reference():
        from oracle.ref_shim import import_reference
        import_reference()
        import frldistml.scaffold.storage_layers.dataset as ref_ds
        from frldistml.scaffold.indexed_dataset import MultifieldIndexedDataset as RefMulti
        from frldistml.scaffold.storage import StoragePath
        ref_parts = [RefMulti(StoragePath(str(tmp_path / ("part%d" % k))), fields=["a", "b"], filenames=["a", "b"])
                     for k in range(3)]
        return observe(ref_ds.ConcatMultifieldDataset(ref_parts), ref_ds.SubsetMultifieldDataset)

    ref, _ = reference_side("indexed_concat_subset", reference)
    mine_parts = [idm.MultifieldIndexedDataset(str(tmp_path / ("part%d" % k)), fields=["a", "b"], filenames=["a", "b"])
                  for k in range(3)]
    mine = observe(my_ds.ConcatMultifieldDataset(mine_parts), my_ds.SubsetMultifieldDataset)
    assert mine["len"] == ref["len"] == sum(sizes)
    for a, b in zip(mine["raw"], ref["raw"]):
        assert list(a) == list(b) and all(torch.equal(a[k][0], b[k][0]) and a[k][1] == b[k][1] for k in a)
    for c, d in zip(mine["items"], ref["items"]):
        assert list(c) == list(d) and all(torch.equal(c[k], d[k]) for k in c)
    assert [tuple(e) for e in mine["log"]] == [tuple(e) for e in ref["log"]] == \
        [(0, "a"), (0, "b"), (5, "a"), (5, "b"), (6, "a"), (6, "b")]
    assert mine["sub_len"] == ref["sub_len"] == 5
    for j in range(5):
        assert all(torch.equal(mine["sub"][j][k], ref["sub"][j][k]) for k in ("a", "b"))
