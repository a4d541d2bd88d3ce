#!/usr/bin/env python
"""Stand-alone timing of the candidate host->HBM row-gather paths (one GPU).

    python tools/probe_input_path.py [rows_per_batch] [row_elems]
    python tools/probe_input_path.py --text [batch] [seq_len]
    python tools/probe_input_path.py --augment [batch]

Prints GB/s of: contiguous cudaMemcpyAsync (PCIe reference), frl_gather_rows at several grid
sizes, frl_gather_rows_tma, the native host gather pool per thread count (plain and with the
fp32 -> bf16 wire conversion), and the host cost of drawing one index batch from the DataLoader
machinery.

``--text``: batches/s served by ``DeviceBatchLoader`` (K8t + the batched transform) against the
per-sample ``DataLoader`` (``TextDataset.__getitem__`` + transform + ``default_collate``) at 4 and
16 workers, over the same 256 MB seeded corpus, no model; host clock around a device synchronise.

``--augment``: the same comparison for augmented 256 x 256 -> 224 x 224 training images:
``DeviceBatchLoader`` + K5a against torchvision v2 transforms in a per-sample ``DataLoader``.
"""
import os
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import torch  # noqa: E402
import frl_b200  # noqa: E402,F401
from frl_b200 import _native  # noqa: E402



def probe_text(batch: int, seq_len: int, n_batches: int = 40) -> None:
    import tempfile
    from frl_b200 import synthetic
    from frl_b200.device_loader import DeviceBatchLoader
    ns = synthetic.api_namespace("frl_b200")
    dev = torch.device("cuda", 0)
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "corpus.txt")
        synthetic.write_mixed_text_corpus(path, 256 << 20, 0)
        fast = synthetic.make_text_problem(ns, tmp, path, path, seq_len=seq_len, device_batches=True)
        plain = synthetic.make_text_problem(ns, tmp, path, path, seq_len=seq_len)
        print("text corpus %d lines, batch %d x %d B" % (len(fast.datasets[0]), batch, seq_len + 1))

        def rate(loader, to_device):
            it = iter(loader)
            next(it)                                        # warm-up: workers started, first batch
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(n_batches):
                data, target, _ = next(it)
                if to_device:
                    data[0].to(dev, non_blocking=True)
                    target[0][0].to(dev, non_blocking=True)
            torch.cuda.synchronize()
            return n_batches / (time.perf_counter() - t0)

        ld = DeviceBatchLoader(fast.datasets[0], batch_size=batch, sampler=None, device=dev)
        print("DeviceBatchLoader (K8t, %d CTAs): %8.1f batches/s" % (ld.blocks, rate(ld, False)), flush=True)
        for workers in (4, 16):
            dl = torch.utils.data.DataLoader(plain.datasets[0], batch_size=batch, shuffle=True,
                                             num_workers=workers, pin_memory=True)
            print("per-sample DataLoader, %2d workers: %8.1f batches/s" % (workers, rate(dl, True)), flush=True)


class _PerSampleImages(torch.utils.data.Dataset):
    """uint8 [N, C, H, W] images + labels through a per-sample torchvision transform."""

    def __init__(self, x, y, transform) -> None:
        self.x, self.y, self.transform = x, y, transform

    def __len__(self) -> int:
        return len(self.x)

    def __getitem__(self, i):
        return self.transform(torch.from_numpy(self.x[i])), int(self.y[i])


def probe_augment(batch: int = 256, stored: int = 256, out: int = 224, n_batches: int = 20) -> None:
    """Batches/s of augmented ImageNet-shaped training input, no model: ``DeviceBatchLoader`` with
    K5a (random resized crop + flip + normalise on the device, bf16 out) against a per-sample
    ``DataLoader`` running torchvision v2 RandomResizedCrop(antialias=False) + RandomHorizontalFlip +
    ToDtype + Normalize on the host at 4 and 16 workers (fp32, pinned, copied to the GPU).  Host
    clock around a device synchronise, after one warm-up batch."""
    import subprocess
    import tempfile
    import torchvision.transforms.v2 as T
    from frl_b200 import synthetic
    from frl_b200.device_loader import DeviceBatchLoader
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip(), flush=True)
    ns = synthetic.api_namespace("frl_b200")
    dev = torch.device("cuda", 0)
    n = batch * (n_batches + 2)
    with tempfile.TemporaryDirectory() as tmp:
        prob = synthetic.make_resnet_problem(ns, tmp, "resnet18", image=out, n_train=n, uint8=True,
                                             augment="rrc", stored_image=stored)
        train = prob.datasets[0]
        print("%d images 3x%dx%d uint8 -> 3x%dx%d, batch %d" % (n, stored, stored, out, out, batch), flush=True)

        def rate(loader, to_device):
            it = iter(loader)
            next(it)                                        # warm-up: workers started, first batch
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(n_batches):
                data, target, *_ = next(it)
                if to_device:
                    data = data.to(dev, non_blocking=True)
                    target.to(dev, non_blocking=True)
            torch.cuda.synchronize()
            return n_batches / (time.perf_counter() - t0)

        ld = DeviceBatchLoader(train, batch_size=batch, sampler=None, device=dev, out_dtype=torch.bfloat16)
        ld.set_epoch(1)
        print("DeviceBatchLoader + K5a (%s path): %8.1f batches/s" % (ld.path, rate(ld, False)), flush=True)
        tf = T.Compose([T.RandomResizedCrop(out, antialias=False), T.RandomHorizontalFlip(),
                        T.ToDtype(torch.float32, scale=True),
                        T.Normalize(list(synthetic.IMAGE_MEAN), list(synthetic.IMAGE_STD))])
        per_sample = _PerSampleImages(train._fields["x"], train._fields["y_cls"], tf)
        for workers in (4, 16):
            dl = torch.utils.data.DataLoader(per_sample, batch_size=batch, shuffle=True, num_workers=workers,
                                             pin_memory=True)
            print("per-sample DataLoader (torchvision v2), %2d workers: %8.1f batches/s"
                  % (workers, rate(dl, True)), flush=True)


if len(sys.argv) > 1 and sys.argv[1] == "--augment":
    torch.cuda.set_device(0)
    probe_augment(int(sys.argv[2]) if len(sys.argv) > 2 else 256)
    sys.exit(0)

if len(sys.argv) > 1 and sys.argv[1] == "--text":
    torch.cuda.set_device(0)
    probe_text(int(sys.argv[2]) if len(sys.argv) > 2 else 4096, int(sys.argv[3]) if len(sys.argv) > 3 else 256)
    sys.exit(0)

B = int(sys.argv[1]) if len(sys.argv) > 1 else 4096
W = int(sys.argv[2]) if len(sys.argv) > 2 else 4096
NB = 16
dev = torch.device("cuda", 0)
torch.cuda.set_device(0)
try:
    from frl_b200.solver import bind_to_gpu_numa_node
    bind_to_gpu_numa_node(0)
except Exception as e:  # noqa: BLE001
    print("numa bind failed:", e)
src = torch.randn(NB * B, W).pin_memory()
dst = torch.empty(B, W, device=dev)
nbytes = B * W * 4
print("rows %d x %d B = %.1f MB per batch" % (B, W * 4, nbytes / 1e6))


def timed(fn, reps=6, sync_host=False):
    best = 1e9
    for r in range(reps):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        e0.record()
        fn(r)
        e1.record()
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        ms = e0.elapsed_time(e1)
        if sync_host:
            ms = (t1 - t0) * 1e3
        if r > 0:
            best = min(best, ms)
    return best


def report(name, ms):
    print("%-42s %8.3f ms  %7.1f GB/s" % (name, ms, nbytes / ms / 1e6), flush=True)


perms = [torch.randperm(NB * B)[:B].contiguous() for _ in range(8)]
perms_dev = [p.to(dev) for p in perms]
perms_pin = [p.pin_memory() for p in perms]

report("cudaMemcpyAsync contiguous", timed(lambda r: dst.copy_(src[r * B:(r + 1) * B], non_blocking=True)))
for blocks in (32, 66, 132, 264, 528, 1056):
    report("frl_gather_rows blocks=%d" % blocks,
           timed(lambda r: _native.gather_rows(src, perms_dev[r], dst, max_blocks=blocks)))
ok = torch.equal(dst.cpu(), src[perms[5]])
print("gather_rows correct:", ok)
for blocks in (16, 33, 66, 132, 264):
    try:
        dst.zero_()
        report("frl_gather_rows_tma blocks=%d" % blocks,
               timed(lambda r: _native.gather_rows_tma(src, perms_dev[r], dst, max_blocks=blocks)))
        print("   correct:", torch.equal(dst.cpu(), src[perms[5]]))
    except Exception as e:  # noqa: BLE001
        print("tma variant failed:", e)
        break
side = torch.cuda.Stream()
torch.cuda.set_stream(side)          # batched copies are not allowed on the legacy default stream
for blocks in (1, 2, 3, 4, 8):
    report("frl_gather_rows_tma blocks=%d" % blocks,
           timed(lambda r: _native.gather_rows_tma(src, perms_dev[r], dst, max_blocks=blocks)))
for blocks in (2, 4, 8, 16):
    report("frl_gather_rows blocks=%d" % blocks,
           timed(lambda r: _native.gather_rows(src, perms_dev[r], dst, max_blocks=blocks)))
# (cudaMemcpyBatchAsync with one descriptor per row is left out: its host cost grows with the rows)
stage = torch.empty(B, W).pin_memory()
for th in (1, 4, 8, 16, 32):
    pool = _native.HostGatherPool(th)
    t = []
    for r in range(5):
        t0 = time.perf_counter()
        pool.wait(pool.submit(src, perms[r], stage))
        t.append(time.perf_counter() - t0)
    pool.close()
    report("frl_gather_pool threads=%d (host)" % th, min(t[1:]) * 1e3)
print("   correct:", torch.equal(stage, src[perms[4]]))
stage16 = torch.empty(B, W, dtype=torch.bfloat16).pin_memory()
pool = _native.HostGatherPool(16)
t = []
for r in range(5):
    t0 = time.perf_counter()
    pool.wait(pool.submit_f32_to_bf16(src, perms[r], stage16))
    t.append(time.perf_counter() - t0)
pool.close()
report("frl_gather_pool f32->bf16 wire, 16 threads", min(t[1:]) * 1e3)
print("   correct:", torch.equal(stage16, src[perms[4]].to(torch.bfloat16)))

# host cost of the index stream (DataLoader + sampler machinery, as DeviceBatchLoader uses it)
from frl_b200.device_loader import _IndexOnly, _collate_indices  # noqa: E402
import torch.utils.data as tud  # noqa: E402
ld = tud.DataLoader(_IndexOnly(NB * B), batch_size=B, shuffle=True, num_workers=0, collate_fn=_collate_indices)
t0 = time.perf_counter()
n = 0
for idx in ld:
    n += 1
t1 = time.perf_counter()
print("index DataLoader: %.3f ms per batch of %d (host)" % ((t1 - t0) * 1e3 / n, B))
samp = tud.RandomSampler(_IndexOnly(NB * B))
t0 = time.perf_counter()
allidx = torch.tensor(list(iter(samp)), dtype=torch.int64)
t1 = time.perf_counter()
print("list(sampler) -> tensor once per epoch: %.3f ms per batch-equivalent" % ((t1 - t0) * 1e3 / NB))
