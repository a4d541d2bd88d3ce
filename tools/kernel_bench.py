#!/usr/bin/env python
"""Micro-benchmark of every hand-written kernel at the BASELINE shapes (1 GPU).

    python tools/kernel_bench.py [--only k2,k2lw,k2q8,k2af,k2w,k2lion,k2g,k3,k5a,k5nhwc,k13,k14,...] [--iters 20] [--json out.json]

Each kernel is timed with CUDA events on the launching stream over ROTATING operand sets whose
total size exceeds the 50 MB L2 (so every launch streams from HBM), after 3 warm-up launches.
Reported: average launch time, algorithmic bytes, achieved GB/s and the fraction of the measured
copy bandwidth in MEASURED_PEAKS.json (else the H100 SXM data-sheet 3.35 TB/s).
"""
import argparse
import json
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import torch  # noqa: E402

import frl_b200  # noqa: E402,F401
from frl_b200 import _native, criteria  # noqa: E402

DEV = torch.device("cuda", 0)
L2_BYTES = 50 << 20


def peak_gbs():
    p = os.path.join(REPO, "MEASURED_PEAKS.json")
    return json.load(open(p))["hbm_gbs"] if os.path.exists(p) else 3350.0


WARMUP = 3
MAX_SETS = 0          # > 0: cap the number of rotating operand sets (ncu runs)


def timed(name, fn_of_set, n_sets, bytes_per_launch, iters, note="", graph=False):
    """``graph``: capture the ``iters`` launches in a CUDA graph and time one replay, so that a
    kernel shorter than its Python + ctypes issue time is still timed on the device."""
    for i in range(WARMUP):
        fn_of_set(i % n_sets)
    torch.cuda.synchronize()
    if graph:
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for i in range(iters):
                fn_of_set(i % n_sets)
        g.replay()
        torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    if graph:
        g.replay()
    else:
        for i in range(iters):
            fn_of_set(i % n_sets)
    e1.record()
    torch.cuda.synchronize()
    us = 1e3 * e0.elapsed_time(e1) / iters
    gbs = bytes_per_launch / us / 1e3
    rec = {"kernel": name, "us": round(us, 2), "bytes": int(bytes_per_launch), "GBps": round(gbs, 1),
           "frac_of_measured_hbm": round(gbs / peak_gbs(), 3), "sets": n_sets, "note": note}
    print(json.dumps(rec), flush=True)
    return rec


def sets_for(bytes_per_set):
    n = max(2, -(-2 * L2_BYTES // max(bytes_per_set, 1)))
    return min(n, MAX_SETS) if MAX_SETS > 0 else n


def bench_k2(iters):
    out = []
    for label, n, algo in (("mlp", 54_703_144, "sgd"), ("mlp", 54_703_144, "adam"),
                           ("r18", 11_689_512, "sgd"), ("r50x4", 25_790_618, "adam")):
        n = (n + 7) // 8 * 8
        p = torch.randn(n, device=DEV)
        lp = torch.empty(n, device=DEV, dtype=torch.bfloat16)
        g = torch.randn(n, device=DEV).bfloat16()
        s0, s1 = torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
        if algo == "sgd":
            def fn(i, p=p, g=g, s0=s0, lp=lp, n=n):
                _native.sgd_momentum(p, g, s0, lp, n, lr=0.01, mu=0.9, dampening=0.0, wd=1e-5,
                                     first_step=False)
            bpp = 20
        else:
            def fn(i, p=p, g=g, s0=s0, s1=s1, lp=lp, n=n):
                _native.adam(p, g, s0, s1, None, lp, n, lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8,
                             wd=1e-5, step=3)
            bpp = 28
        out.append(timed("K2 %s %s bf16-grad (%d elems)" % (algo, label, n), fn, 1, bpp * n, iters,
                         "one set: the arena itself is %d MB" % (bpp * n >> 20)))
    return out


def bench_k2mt(iters):
    """K2-mt / K1 on the parameter lists of BASELINE configs 4/5: 62 / 167 tensors, gradients in
    separately allocated bf16 tensors (what cuDNN hands to autograd), segment table in HBM."""
    import torchvision
    from frl_b200.multi_tensor import GradSegTable

    class Slot:
        def __init__(self, index, offset, numel):
            self.index, self.offset, self.numel = index, offset, numel

    out = []
    for label, arch, heads, algo in (("r18", "resnet18", [(512, 1000)], "sgd"),
                                     ("r50x4", "resnet50", [(2048, 1000), (2048, 100), (2048, 10), (2048, 4)], "adam")):
        net = getattr(torchvision.models, arch)(weights=None)
        sizes = [p.numel() for n, p in net.named_parameters() if not n.startswith("fc.")]
        for i, o in heads:
            sizes += [i * o, o]
        slots, off = [], 0
        for i, n in enumerate(sizes):
            slots.append(Slot(i, off, n))
            off = (off + n + 7) // 8 * 8
        n = off
        grads = [torch.randn(s.numel, device=DEV).bfloat16() for s in slots]
        table = GradSegTable(slots, DEV)
        for s_, g in zip(slots, grads):
            table.point(s_, g.data_ptr(), g.dtype)
        table.upload()
        p = torch.randn(n, device=DEV)
        lp = torch.empty(n, device=DEV, dtype=torch.bfloat16)
        s0, s1 = torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
        flat = torch.empty(n, device=DEV, dtype=torch.bfloat16)
        n_real = sum(sizes)
        if algo == "sgd":
            def fn(i, p=p, s0=s0, lp=lp, table=table):
                _native.sgd_momentum_mt(p, s0, lp, table, lr=0.01, mu=0.9, dampening=0.0, wd=1e-5, first_step=False)
            bpp = 20
        else:
            def fn(i, p=p, s0=s0, s1=s1, lp=lp, table=table):
                _native.adam_mt(p, s0, s1, None, lp, table, lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, wd=1e-5, step=3)
            bpp = 28
        out.append(timed("K2-mt %s %s: %d tensors, %d params, gradients read in place" % (algo, label, len(sizes), n_real),
                         fn, 1, bpp * n_real, iters))
        out.append(timed("K1 flatten_grads %s: %d tensors -> bf16 arena, one launch" % (label, len(sizes)),
                         lambda i, table=table, flat=flat: _native.flatten_grads(table, flat, scale=1.0), 1,
                         4 * n_real, iters))
    return out


def bench_k2lw(iters):
    """K2-lw (LARS, LAMB) over the headline MLP's 10 tensors (54.7 M parameters), bf16 gradients in
    the arena, bf16 shadow, timed from a CUDA graph.  The arena is far larger than L2, so every
    launch streams from HBM.  The pair of launches is timed with CUDA events; each phase is then
    timed on its own from the kernel durations ``torch.profiler`` records over one replay.
    Bytes per parameter: LARS stats reads g, w (6), apply reads g, w, buf and writes w, buf,
    shadow (20); LAMB stats reads g, w, m, v and writes m, v (22), apply reads w, m, v and writes
    w, shadow (18)."""
    from torch.profiler import ProfilerActivity, profile
    from frl_b200.multi_tensor import GradSegTable

    class Slot:
        def __init__(self, index, offset, shape):
            self.index, self.offset, self.shape = index, offset, shape
            self.numel = 1
            for d in shape:
                self.numel *= d
            self.is_model = True

    shapes = [(4096, 4096), (4096,)] * 3 + [(1000, 4096), (1000,), (64, 4096), (64,)]
    slots, off = [], 0
    for i, sh in enumerate(shapes):
        slots.append(Slot(i, off, sh))
        off = (off + slots[-1].numel + 7) // 8 * 8
    n, n_real = off, sum(s.numel for s in slots)
    grad = torch.randn(n, device=DEV).bfloat16()
    table = GradSegTable(slots, DEV)
    for s in slots:
        table.point(s, grad.data_ptr() + 2 * s.offset, grad.dtype)
    table.upload()
    flags = torch.tensor([_native.LW_CLIPPED | (_native.LW_ADAPTED if len(s.shape) >= 2 else 0) for s in slots],
                         dtype=torch.int32, device=DEV)
    ratio = torch.ones(len(slots), device=DEV)
    scratch = torch.zeros((_native.layerwise_scratch_bytes(table.n_tiles, table.n_segs) + 3) // 4,
                          dtype=torch.int32, device=DEV)
    p = torch.randn(n, device=DEV) * 0.02
    lp = torch.empty(n, device=DEV, dtype=torch.bfloat16)
    s0, s1 = torch.zeros(n, device=DEV), torch.rand(n, device=DEV) * 1e-4
    out = []
    for algo, stats_bpp, apply_bpp in (("lars", 6, 20), ("lamb", 22, 18)):
        if algo == "lars":
            def fn(i):
                _native.lars_mt(p, s0, lp, table, flags, ratio, scratch, lr=0.01, mu=0.9, wd=1e-5,
                                first_step=False)
        else:
            def fn(i):
                _native.lamb_mt(p, s0, s1, lp, table, flags, ratio, scratch, lr=1e-3, beta1=0.9, beta2=0.999,
                                eps=1e-8, wd=1e-5, step=3)
        out.append(timed("K2-lw %s mlp bf16-grad, both phases (%d tensors, %d params)" % (algo, len(slots), n_real),
                         fn, 1, (stats_bpp + apply_bpp) * n_real, iters, graph=True))
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for i in range(iters):
                fn(i)
        g.replay()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            g.replay()
            torch.cuda.synchronize()
        for phase, bpp in (("lw_stats_kernel", stats_bpp), ("lw_apply_kernel", apply_bpp)):
            us = sum(e.device_time_total for e in prof.key_averages() if phase in e.key) / iters
            if us <= 0:
                raise RuntimeError("torch.profiler recorded no %s kernels in the graph replay" % phase)
            gbs = bpp * n_real / us / 1e3
            rec = {"kernel": "K2-lw %s %s" % (algo, phase), "us": round(us, 2), "bytes": bpp * n_real,
                   "GBps": round(gbs, 1), "frac_of_measured_hbm": round(gbs / peak_gbs(), 3),
                   "note": "torch.profiler kernel time over one replay of %d launches" % iters}
            print(json.dumps(rec), flush=True)
            out.append(rec)
    return out


def bench_k2q8(iters):
    """K2-q8 (Adam with 8-bit block-wise state) over the headline MLP's 10 tensors (54.7 M
    parameters), bf16 gradients in the arena, bf16 shadow, timed from a CUDA graph next to K2-mt
    Adam (``frl_adam_mt``, fp32 state) on the same arena.  The arena is far larger than L2, so every
    launch streams from HBM.  Bytes from the layout: K2-q8 reads g (2) and reads and writes the
    master (8), both codes (4) and the shadow (2), plus 2 x 8 bytes of absmax per 256-element block;
    K2-mt Adam moves 28 bytes per parameter."""
    from frl_b200.fused_optim import q8_block_bases
    from frl_b200.multi_tensor import GradSegTable

    class Slot:
        def __init__(self, index, offset, shape):
            self.index, self.offset, self.shape = index, offset, shape
            self.numel = 1
            for d in shape:
                self.numel *= d
            self.is_model = True

    shapes = [(4096, 4096), (4096,)] * 3 + [(1000, 4096), (1000,), (64, 4096), (64,)]
    slots, off = [], 0
    for i, sh in enumerate(shapes):
        slots.append(Slot(i, off, sh))
        off = (off + slots[-1].numel + 7) // 8 * 8
    n, n_real = off, sum(s.numel for s in slots)
    grad = torch.randn(n, device=DEV).bfloat16()
    table = GradSegTable(slots, DEV)
    for s in slots:
        table.point(s, grad.data_ptr() + 2 * s.offset, grad.dtype)
    table.upload()
    bases, n_blocks = q8_block_bases(slots)
    qbase = torch.tensor([bases[s.index] for s in slots], dtype=torch.int64, device=DEV)
    flags = torch.full((len(slots),), _native.LW_CLIPPED, dtype=torch.int32, device=DEV)
    p = torch.randn(n, device=DEV) * 0.02
    lp = torch.empty(n, device=DEV, dtype=torch.bfloat16)
    m, v = torch.randn(n, device=DEV) * 1e-3, torch.rand(n, device=DEV) * 1e-6
    mq, vq = torch.zeros(n, dtype=torch.uint8, device=DEV), torch.zeros(n, dtype=torch.uint8, device=DEV)
    ma, va = torch.zeros(n_blocks, device=DEV), torch.zeros(n_blocks, device=DEV)
    _native.q8_encode_mt(m, mq, ma, _native.Q8_EXP_AVG, table, qbase)
    _native.q8_encode_mt(v, vq, va, _native.Q8_EXP_AVG_SQ, table, qbase)

    def q8(i):
        _native.adam8_mt(p, mq, vq, ma, va, lp, table, qbase, flags, lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8,
                         wd=1e-5, step=3)

    def fp32(i):
        _native.adam_mt(p, m, v, None, lp, table, lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, wd=1e-5, step=3)

    q8_bytes = 16 * n_real + 2 * 8 * n_blocks
    return [timed("K2-q8 adam 8-bit state mlp bf16-grad (%d tensors, %d params, %d blocks)"
                  % (len(slots), n_real, n_blocks), q8, 1, q8_bytes, iters,
                  "%.2f B/param" % (q8_bytes / n_real), graph=True),
            timed("K2-mt adam fp32 state mlp bf16-grad (%d tensors, %d params)" % (len(slots), n_real), fp32, 1,
                  28 * n_real, iters, "28 B/param", graph=True)]


def bench_k2w(iters):
    """K2-mt AdamW (``frl_adamw_mt``) beside K2-mt Adam (``frl_adam_mt``) on the headline MLP's arena
    (10 tensors, 54.7 M parameters), bf16 gradients in the arena, bf16 shadow, fp32 state, each timed
    from a CUDA graph.  Both rules move 28 bytes per parameter, so the arena (1.5 GB of traffic per
    launch) is far larger than L2 and every launch streams from HBM.  Five rounds, Adam and AdamW
    alternating; the last two records are the medians (min-max) and AdamW / Adam."""
    from frl_b200.multi_tensor import GradSegTable

    class Slot:
        def __init__(self, index, offset, shape):
            self.index, self.offset, self.shape = index, offset, shape
            self.numel = 1
            for d in shape:
                self.numel *= d
            self.is_model = True

    shapes = [(4096, 4096), (4096,)] * 3 + [(1000, 4096), (1000,), (64, 4096), (64,)]
    slots, off = [], 0
    for i, sh in enumerate(shapes):
        slots.append(Slot(i, off, sh))
        off = (off + slots[-1].numel + 7) // 8 * 8
    n, n_real = off, sum(s.numel for s in slots)
    grad = torch.randn(n, device=DEV).bfloat16()
    table = GradSegTable(slots, DEV)
    for s in slots:
        table.point(s, grad.data_ptr() + 2 * s.offset, grad.dtype)
    table.upload()
    p = torch.randn(n, device=DEV) * 0.02
    lp = torch.empty(n, device=DEV, dtype=torch.bfloat16)
    m, v = torch.randn(n, device=DEV) * 1e-3, torch.rand(n, device=DEV) * 1e-6
    kw = dict(lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, wd=1e-2, step=3)
    fns = {"adam": lambda i: _native.adam_mt(p, m, v, None, lp, table, **kw),
           "adamw": lambda i: _native.adamw_mt(p, m, v, None, lp, table, **kw)}
    out, times = [], {"adam": [], "adamw": []}
    for r in range(5):
        for rule in ("adam", "adamw"):
            rec = timed("K2-mt %s fp32 state mlp bf16-grad (%d tensors, %d params) round %d"
                        % (rule, len(slots), n_real, r), fns[rule], 1, 28 * n_real, iters, "28 B/param", graph=True)
            times[rule].append(rec["us"])
            out.append(rec)
    med = {k: sorted(t)[len(t) // 2] for k, t in times.items()}
    summary = {"kernel": "K2-mt adamw vs adam, median of 5 (min-max)",
               "adam_us": "%.1f (%.1f-%.1f)" % (med["adam"], min(times["adam"]), max(times["adam"])),
               "adamw_us": "%.1f (%.1f-%.1f)" % (med["adamw"], min(times["adamw"]), max(times["adamw"])),
               "adamw_over_adam": round(med["adamw"] / med["adam"], 4),
               "within_5pct": med["adamw"] <= 1.05 * med["adam"]}
    print(json.dumps(summary), flush=True)
    out.append(summary)
    return out


def bench_k2lion(iters):
    """K2-mt Lion (``frl_lion_mt``) beside K2-mt SGD with momentum (``frl_sgd_momentum_mt``) on the
    headline MLP's arena (10 tensors, 54.7 M parameters), bf16 gradients in the arena, bf16 shadow, one
    fp32 state vector, each timed from a CUDA graph.  Both rules move 20 bytes per parameter (1.1 GB
    per launch, far larger than L2).  Five rounds, SGD and Lion alternating; the last record holds the
    medians (min-max), Lion / SGD and Lion's share of the data-sheet 3.35 TB/s."""
    from frl_b200.multi_tensor import GradSegTable

    class Slot:
        def __init__(self, index, offset, shape):
            self.index, self.offset, self.shape = index, offset, shape
            self.numel = 1
            for d in shape:
                self.numel *= d
            self.is_model = True

    shapes = [(4096, 4096), (4096,)] * 3 + [(1000, 4096), (1000,), (64, 4096), (64,)]
    slots, off = [], 0
    for i, sh in enumerate(shapes):
        slots.append(Slot(i, off, sh))
        off = (off + slots[-1].numel + 7) // 8 * 8
    n, n_real = off, sum(s.numel for s in slots)
    grad = torch.randn(n, device=DEV).bfloat16()
    table = GradSegTable(slots, DEV)
    for s in slots:
        table.point(s, grad.data_ptr() + 2 * s.offset, grad.dtype)
    table.upload()
    p = torch.randn(n, device=DEV) * 0.02
    lp = torch.empty(n, device=DEV, dtype=torch.bfloat16)
    m = torch.randn(n, device=DEV) * 1e-3
    fns = {"sgd": lambda i: _native.sgd_momentum_mt(p, m, lp, table, lr=1e-2, mu=0.9, dampening=0.0, wd=1e-5),
           "lion": lambda i: _native.lion_mt(p, m, lp, table, lr=1e-4, beta1=0.9, beta2=0.99, wd=1e-5)}
    out, times = [], {"sgd": [], "lion": []}
    for r in range(5):
        for rule in ("sgd", "lion"):
            rec = timed("K2-mt %s mlp bf16-grad (%d tensors, %d params) round %d" % (rule, len(slots), n_real, r),
                        fns[rule], 1, 20 * n_real, iters, "20 B/param", graph=True)
            times[rule].append(rec["us"])
            out.append(rec)
    med = {k: sorted(t)[len(t) // 2] for k, t in times.items()}
    lion_tbs = 20 * n_real / med["lion"] / 1e6
    summary = {"kernel": "K2-mt lion vs sgd momentum, median of 5 (min-max)",
               "sgd_us": "%.1f (%.1f-%.1f)" % (med["sgd"], min(times["sgd"]), max(times["sgd"])),
               "lion_us": "%.1f (%.1f-%.1f)" % (med["lion"], min(times["lion"]), max(times["lion"])),
               "lion_over_sgd": round(med["lion"] / med["sgd"], 4),
               "within_3pct": med["lion"] <= 1.03 * med["sgd"],
               "lion_TBps": round(lion_tbs, 3), "lion_frac_of_3.35TBps": round(lion_tbs / 3.35, 3),
               "at_least_0.83": lion_tbs / 3.35 >= 0.83}
    print(json.dumps(summary), flush=True)
    out.append(summary)
    return out


def bench_k2af(iters):
    """K2-af (Adafactor: stats, norm and apply launches) over the headline MLP's 10 tensors, bf16
    gradients in the arena, bf16 shadow, timed from a CUDA graph next to K2-mt SGD
    (``frl_sgd_momentum_mt`` without momentum) on the same arena.  Bytes: g read three times (6),
    the master read twice and written once (12), the shadow written (2): 20 B/param, SGD's count;
    the factored state (about 47 K floats) is not counted."""
    from frl_b200.fused_optim import FusedAdafactor
    from frl_b200.multi_tensor import GradSegTable

    class Slot:
        def __init__(self, index, offset, shape):
            self.index, self.offset, self.shape = index, offset, shape
            self.numel = 1
            for d in shape:
                self.numel *= d
            self.is_model = True

    class Arena:
        pass

    shapes = [(4096, 4096), (4096,)] * 3 + [(1000, 4096), (1000,), (64, 4096), (64,)]
    slots, off = [], 0
    for i, sh in enumerate(shapes):
        slots.append(Slot(i, off, sh))
        off = (off + slots[-1].numel + 7) // 8 * 8
    n, n_real = off, sum(s.numel for s in slots)
    grad = torch.randn(n, device=DEV).bfloat16()
    table = GradSegTable(slots, DEV)
    for s in slots:
        table.point(s, grad.data_ptr() + 2 * s.offset, grad.dtype)
    table.upload()
    a = Arena()
    a.slots, a.numel, a.device = slots, n, torch.device(DEV)
    a.all_params = [torch.nn.Parameter(torch.zeros(1)) for _ in slots]
    a.master = torch.randn(n, device=DEV) * 0.02
    a.lp = torch.empty(n, device=DEV, dtype=torch.bfloat16)
    opt = FusedAdafactor(a, lr=1e-2, weight_decay=1e-5)
    opt._steps = 2

    def af(i):
        opt.apply_table(table)

    def sgd(i):
        _native.sgd_momentum_mt(a.master, None, a.lp, table, lr=1e-3, mu=0.0, dampening=0.0, wd=0.0)

    recs = [timed("K2-af adafactor mlp bf16-grad (%d tensors, %d params, 3 launches)" % (len(slots), n_real), af,
                  1, 20 * n_real, iters, "20 B/param", graph=True)]
    # per pass: device time of each kernel under torch.profiler, in a window of its own
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(iters):
            af(i)
        torch.cuda.synchronize()
    passes = {"stats": ("af_stats_kernel", 6), "norm": ("af_update_kernel<false", 2),
              "apply": ("af_update_kernel<true", 12)}          # name, bytes/param of the pass
    for ev in prof.key_averages():
        for pname, (key, bpp) in passes.items():
            if key in ev.key and ev.count:
                us = ev.device_time_total / ev.count
                gbs = bpp * n_real / us / 1e3
                rec = {"kernel": "K2-af %s pass (%s)" % (pname, ev.key[:60]), "us": round(us, 2),
                       "bytes": bpp * n_real, "GBps": round(gbs, 1), "frac_of_measured_hbm": round(gbs / peak_gbs(), 3),
                       "launches": ev.count, "note": "%d B/param, torch.profiler" % bpp}
                print(json.dumps(rec), flush=True)
                recs.append(rec)
    return recs + [
            timed("K2-mt sgd mlp bf16-grad (%d tensors, %d params)" % (len(slots), n_real), sgd, 1,
                  10 * n_real, iters, "10 B/param (no momentum)", graph=True)]


def bench_k10(iters):
    """K10 gradient accumulation over the headline MLP's 10 tensors (54.7 M parameters) as the solver
    builds it: one segment table over the arena's slots, bf16 gradients in the arena, an fp32
    accumulator, timed from a CUDA graph.  Gradients (109 MB) and accumulator (219 MB) are far larger
    than L2, so every launch streams from HBM.  Bytes per parameter: first = 1 reads g and writes acc
    (6); first = 0 reads g and acc and writes acc (10)."""
    from frl_b200.multi_tensor import GradSegTable

    class Slot:
        def __init__(self, index, offset, numel):
            self.index, self.offset, self.numel = index, offset, numel

    sizes = [4096 * 4096, 4096] * 3 + [1000 * 4096, 1000, 64 * 4096, 64]
    slots, off = [], 0
    for i, n in enumerate(sizes):
        slots.append(Slot(i, off, n))
        off = (off + n + 7) // 8 * 8
    n, n_real = off, sum(sizes)
    grad = torch.randn(n, device=DEV).bfloat16()
    table = GradSegTable(slots, DEV)
    for s in slots:
        table.point(s, grad.data_ptr() + 2 * s.offset, grad.dtype)
    table.upload()
    acc = torch.zeros(n, device=DEV)
    out = []
    for first, bpp in ((True, 6), (False, 10)):
        out.append(timed("K10 grad_accumulate_mt mlp bf16-grad first=%d (%d tensors, %d params)"
                         % (first, len(slots), n_real),
                         lambda i, first=first: _native.grad_accumulate_mt(acc, table, w=1.0, first=first),
                         1, bpp * n_real, iters, "accumulator %d MB" % (4 * n >> 20), graph=True))
    return out


def bench_k11(iters):
    """K11 weight EMA over the headline MLP's model range (54.7 M parameters, its arena as the solver
    lays it out), timed from a CUDA graph.  Two operand sets (EMA + master, 438 MB each) alternate,
    so every launch streams from HBM with L2 cold.  Bytes per parameter: read ema and p, write ema
    (12)."""
    sizes = [4096 * 4096, 4096] * 3 + [1000 * 4096, 1000, 64 * 4096, 64]
    n = 0
    for s in sizes:
        n = (n + s + 7) // 8 * 8
    ns = sets_for(8 * n)
    sets = [(torch.randn(n, device=DEV), torch.randn(n, device=DEV)) for _ in range(ns)]
    return [timed("K11 weight_ema mlp model range (%d elems)" % n,
                  lambda i: _native.weight_ema(sets[i][0], sets[i][1], 1e-4), ns, 12 * n, iters,
                  "%d rotating sets of %d MB" % (ns, 8 * n >> 20), graph=True)]


def bench_k3(iters):
    n = 54_703_144
    out = []
    for dt in (torch.bfloat16, torch.float32):
        ns = sets_for(n * (2 if dt == torch.bfloat16 else 4))
        gs = [torch.randn(n, device=DEV).to(dt) for _ in range(ns)]
        out3 = torch.zeros(3, device=DEV)
        scratch = torch.zeros((_native.reduce_scratch_bytes() + 3) // 4, dtype=torch.int32, device=DEV)
        out.append(timed("K3 sumsq_clip %s (%d elems)" % (str(dt).replace("torch.", ""), n),
                         lambda i: _native.grad_sumsq_clip(gs[i], n, pre_scale=1.0, max_norm=1.0,
                                                           out3=out3, scratch=scratch),
                         ns, n * gs[0].element_size(), iters))
        del gs
    return out


def bench_k4(iters):
    B, C, R = 4096, 1000, 64
    out = []
    for dt in (torch.bfloat16, torch.float32):
        esz = 2 if dt == torch.bfloat16 else 4
        per = B * C * esz + B * R * esz + B * R * 4 + B * 8
        ns = sets_for(per)
        mods = [torch.nn.CrossEntropyLoss(), torch.nn.MSELoss()]
        sets = []
        for _ in range(ns):
            lo = torch.randn(B, C, device=DEV).to(dt).requires_grad_(True)
            ro = torch.randn(B, R, device=DEV).to(dt).requires_grad_(True)
            sets.append((lo, ro, torch.randint(0, C, (B,), device=DEV), torch.randn(B, R, device=DEV)))
        held = {}

        def fwd(i):
            lo, ro, y, r = sets[i]
            held[i] = criteria.fused_task_losses(mods, [lo, ro], [(y,), (r,)], [1.0, 1.0])

        name = str(dt).replace("torch.", "")
        out.append(timed("K4 criteria forward %s [4096,1000] CE + [4096,64] MSE" % name, fwd, ns, per, iters))
        for i in range(ns):
            fwd(i)

        def bwd(i):
            held[i][0].backward(retain_graph=True)
            sets[i][0].grad = sets[i][1].grad = None

        # backward reads logits + lse and writes dlogits (+ the small head)
        out.append(timed("K4 criteria backward %s (includes autograd dispatch)" % name, bwd, ns,
                         2 * (B * C * esz + B * R * esz) + B * R * 4 + B * 12, iters))
    return out


def bench_k5(iters):
    out = []
    n = 4096 * 4096
    ns = sets_for(n * 6)
    src = [torch.randn(n, device=DEV) for _ in range(ns)]
    dst = [torch.empty(n, device=DEV, dtype=torch.bfloat16) for _ in range(ns)]
    sc, bi = torch.tensor([2.0], device=DEV), torch.tensor([-1.0], device=DEV)
    out.append(timed("K5 preproc_affine f32->bf16 [4096,4096] (1 channel)",
                     lambda i: _native.preproc_affine(src[i], dst[i], inner=n, channels=1, scale=sc, bias=bi),
                     ns, n * 6, iters))
    out.append(timed("K5 cast_scale f32->bf16 [4096,4096]",
                     lambda i: _native.cast_scale(src[i], dst[i], 1.0), ns, n * 6, iters))
    del src, dst
    B, Cc, H = 256, 3, 224
    n = B * Cc * H * H
    ns = sets_for(n * 3)
    src = [torch.randint(0, 256, (n,), device=DEV, dtype=torch.uint8) for _ in range(ns)]
    dst = [torch.empty(n, device=DEV, dtype=torch.bfloat16) for _ in range(ns)]
    sc, bi = torch.rand(3, device=DEV), torch.rand(3, device=DEV)
    out.append(timed("K5 preproc_affine u8->bf16 [256,3,224,224] per-channel",
                     lambda i: _native.preproc_affine(src[i], dst[i], inner=H * H, channels=Cc, scale=sc, bias=bi),
                     ns, n * 3, iters))
    return out


def _taps_touched(crop, out):
    """Distinct source lines one axis of a ``crop`` -> ``out`` bilinear resize reads (K5a's taps)."""
    import numpy as np
    s = np.float64(np.float32(crop) / np.float32(out))          # fmaf: exact product, one rounding
    src = np.maximum((s * (np.arange(out) + 0.5) - 0.5).astype(np.float32), np.float32(0))
    i0 = np.minimum(src.astype(np.int64), crop - 1)
    return np.unique(np.concatenate([i0, np.minimum(i0 + 1, crop - 1)])).size


def bench_k5a(iters):
    """K5a at the ImageNet training shape: batch 256, 3 x 256 x 256 uint8 -> 3 x 224 x 224 bf16,
    random resized crop + flip + per-channel affine, timed from a CUDA graph over rotating sets.
    ``bytes`` = the bf16 output plus, per sample, the source rows x columns its taps touch (from
    the drawn boxes); the rest of each stored image is never read."""
    B, Cc, S, O = 256, 3, 256, 224
    ns = sets_for(B * Cc * (S * S + 2 * O * O))
    src = [torch.randint(0, 256, (B, Cc, S, S), device=DEV, dtype=torch.uint8) for _ in range(ns)]
    dst = [torch.empty(B, Cc, O, O, device=DEV, dtype=torch.bfloat16) for _ in range(ns)]
    idx = [torch.arange(B, device=DEV, dtype=torch.int64) + i * B for i in range(ns)]
    sc, bi = torch.rand(Cc, device=DEV), torch.rand(Cc, device=DEV)
    params = torch.empty(B, 5, dtype=torch.int32, device=DEV)
    read = 0
    for i in range(ns):
        _native.augment_images(src[i], idx[i], dst[i], seed=0, epoch=1, mode=_native.AUG_RRC, scale=sc, bias=bi,
                               params_out=params)
        read += sum(Cc * _taps_touched(int(h), O) * _taps_touched(int(w), O) for h, w in params[:, 2:4].tolist())
    nbytes = read // ns + B * Cc * O * O * 2

    def fn(i):
        _native.augment_images(src[i], idx[i], dst[i], seed=0, epoch=1, mode=_native.AUG_RRC, scale=sc, bias=bi)

    return [timed("K5a augment_images RRC u8 [256,3,256,256] -> bf16 [256,3,224,224]", fn, ns, nbytes, iters,
                  "bytes: touched source lines of the drawn boxes + output", graph=True)]


def bench_k5m(iters):
    """K5a alone, fused with Mixup and fused with CutMix (frl_augment_mix_images) at the K5a shape,
    same sets and boxes: the mix reads both samples' taps in one CTA per pair, so its bytes are
    K5a's (each sample's taps are read once, each output written once)."""
    B, Cc, S, O = 256, 3, 256, 224
    ns = sets_for(B * Cc * (S * S + 2 * O * O))
    src = [torch.randint(0, 256, (B, Cc, S, S), device=DEV, dtype=torch.uint8) for _ in range(ns)]
    dst = [torch.empty(B, Cc, O, O, device=DEV, dtype=torch.bfloat16) for _ in range(ns)]
    idx = [torch.arange(B, device=DEV, dtype=torch.int64) + i * B for i in range(ns)]
    sc, bi = torch.rand(Cc, device=DEV), torch.rand(Cc, device=DEV)
    params = torch.empty(B, 5, dtype=torch.int32, device=DEV)
    read = 0
    for i in range(ns):
        _native.augment_images(src[i], idx[i], dst[i], seed=0, epoch=1, mode=_native.AUG_RRC, scale=sc, bias=bi,
                               params_out=params)
        read += sum(Cc * _taps_touched(int(h), O) * _taps_touched(int(w), O) for h, w in params[:, 2:4].tolist())
    nbytes = read // ns + B * Cc * O * O * 2
    kw = dict(seed=0, epoch=1, mode=_native.AUG_RRC, scale=sc, bias=bi)
    out = [timed("K5a augment_images RRC u8 [256,3,256,256] -> bf16 [256,3,224,224]",
                 lambda i: _native.augment_images(src[i], idx[i], dst[i], **kw), ns, nbytes, iters,
                 "bytes: touched source lines of the drawn boxes + output", graph=True)]
    out.append(timed("K5a + Mixup augment_mix_images (lam 0.7), same shape",
                     lambda i: _native.augment_mix_images(src[i], idx[i], dst[i], mix_mode=_native.MIX_MIXUP,
                                                          lam=0.7, **kw), ns, nbytes, iters, "bytes as K5a",
                     graph=True))
    out.append(timed("K5a + CutMix augment_mix_images (box 112x112), same shape",
                     lambda i: _native.augment_mix_images(src[i], idx[i], dst[i], mix_mode=_native.MIX_CUTMIX,
                                                          lam=0.75, box=(56, 168, 56, 168), **kw),
                     ns, nbytes, iters, "bytes as K5a", graph=True))
    return out


def bench_k4s(iters):
    """K4 forward + backward at [4096, 1000] bf16 logits: class indices with eps = 0 and eps = 0.1,
    fp32 probability targets; beside them the composed torch ops label smoothing took before
    (F.cross_entropy forward + autograd backward).  Bytes: logits read twice (forward, backward),
    gradient written once, targets read once per pass (8 B labels or a 4 B-per-class row)."""
    B, C = 4096, 1000
    out = []
    import torch.nn.functional as F
    for label, eps, prob in (("eps=0", 0.0, False), ("eps=0.1", 0.1, False), ("fp32 probabilities", 0.0, True)):
        tb = B * C * 4 if prob else B * 8
        per = 3 * B * C * 2 + 2 * tb + B * 8
        ns = sets_for(per)
        mods = [torch.nn.CrossEntropyLoss(label_smoothing=eps)]
        sets = []
        for _ in range(ns):
            lo = torch.randn(B, C, device=DEV).to(torch.bfloat16).requires_grad_(True)
            tgt = (torch.rand(B, C, device=DEV).softmax(1) if prob else torch.randint(0, C, (B,), device=DEV))
            sets.append((lo, tgt))

        def step(i):
            lo, tgt = sets[i]
            criteria.fused_task_losses(mods, [lo], [(tgt,)])[0].backward()
            lo.grad = None

        out.append(timed("K4 forward+backward bf16 [4096,1000] CE %s" % label, step, ns, per, iters,
                         "includes autograd dispatch"))
        if eps > 0:
            def composed(i):
                lo, tgt = sets[i]
                F.cross_entropy(lo, tgt, label_smoothing=eps).backward()
                lo.grad = None
            out.append(timed("composed torch F.cross_entropy forward+backward bf16 [4096,1000] %s" % label,
                             composed, ns, per, iters, "the path label smoothing took before K4 handled it"))
    return out


def bench_k6(iters):
    out = []
    rows = cols = 4096
    ns = sets_for(rows * cols * 2 * 3)
    dy = [torch.randn(rows, cols, device=DEV).bfloat16() for _ in range(ns)]
    act = [torch.randn(rows, cols, device=DEV).bfloat16() for _ in range(ns)]
    dz = [torch.empty(rows, cols, device=DEV, dtype=torch.bfloat16) for _ in range(ns)]
    db = torch.empty(cols, device=DEV, dtype=torch.bfloat16)
    out.append(timed("K6 colsum bf16 [4096,4096]", lambda i: _native.colsum(dy[i], db), ns,
                     rows * cols * 2 + cols * 2, iters))
    out.append(timed("K6b drelu_colsum bf16 [4096,4096]",
                     lambda i: _native.drelu_colsum(dy[i], act[i], dz[i], db), ns,
                     rows * cols * 2 * 3 + cols * 2, iters))
    dy1 = [torch.randn(rows, 1000, device=DEV).bfloat16() for _ in range(ns)]
    db1 = torch.empty(1000, device=DEV, dtype=torch.bfloat16)
    out.append(timed("K6 colsum bf16 [4096,1000]", lambda i: _native.colsum(dy1[i], db1), ns,
                     rows * 1000 * 2 + 2000, iters))
    return out


def bench_k8(iters):
    out = []
    n_rows, width, B = 16384, 4096, 4096
    src = torch.randn(n_rows, width).pin_memory()
    dst = torch.empty(B, width, device=DEV)
    idx = torch.randperm(n_rows, device=DEV)[:B].contiguous()
    for blocks in (8, 16, 32):
        out.append(timed("K8 gather_rows (LSU) pinned host -> HBM, %d CTAs" % blocks,
                         lambda i: _native.gather_rows(src, idx, dst, max_blocks=blocks), 1,
                         B * width * 4, max(iters // 2, 2), "PCIe-bound, not HBM"))
    out.append(timed("K8 gather_rows_tma pinned host -> HBM, 2 CTAs",
                     lambda i: _native.gather_rows_tma(src, idx, dst, max_blocks=2), 1, B * width * 4,
                     max(iters // 2, 2), "PCIe-bound"))
    return out


def bench_k8t(iters):
    """K8t at batch 4096 over a 256 MB seeded corpus in pinned memory (line lengths: a mixture
    with means of 120 B and 2 KB, so rows are padded and cut), next to K8 at the same batch and
    row bytes rounded up to 16 (the fixed-row ceiling).  ``bytes`` = rows delivered to HBM."""
    import tempfile
    import numpy as np
    from frl_b200 import synthetic, text_dataset
    from frl_b200.types import Split
    out = []
    B = 4096
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "corpus.txt")
        synthetic.write_mixed_text_corpus(path, 256 << 20, 0)
        for row_len in (257, 1025):
            ds = text_dataset.TextDataset(Split.TRAIN, path, lambda raw, split: raw, row_len - 1)
            field = ds.pinned_fields["line"]
            addr, starts = field.corpus.pin(), field.starts_on(DEV)
            g = torch.Generator().manual_seed(row_len)
            idx = [torch.randint(0, len(ds), (B,), generator=g).to(DEV) for _ in range(8)]
            lens = np.minimum(np.maximum(np.diff(ds._sample_indices) - 1, 0), row_len)
            payload = np.mean([lens[i.cpu().numpy()].sum() for i in idx])
            dst = torch.empty(B, row_len, dtype=torch.uint8, device=DEV)
            out.append(timed("K8t gather_lines row_len=%d, 8 CTAs" % row_len,
                             lambda i: _native.gather_lines(addr, field.corpus.n_bytes, field.corpus.alloc_bytes,
                                                            starts, idx[i % 8], dst, max_blocks=8),
                             1, B * row_len, iters, "line payload %.0f B/batch; PCIe-bound" % payload))
            rb = (row_len + 15) // 16 * 16
            src = torch.zeros((256 << 20) // rb, rb, dtype=torch.uint8, pin_memory=True)
            ridx = torch.randint(0, src.shape[0], (B,), generator=g).to(DEV)
            rdst = torch.empty(B, rb, dtype=torch.uint8, device=DEV)
            out.append(timed("K8 gather_rows row_bytes=%d, 8 CTAs (fixed-row ceiling)" % rb,
                             lambda i: _native.gather_rows(src, ridx, rdst, max_blocks=8), 1, B * rb, iters,
                             "PCIe-bound"))
            del ds, field, src
    return out


def bench_k9(iters):
    """K9 at the trunk's 4096 x 4096 operand: amax, then the quantise pass writing both layouts
    (what a weight or an activation in training takes) or only the row-major copy (eval).  Timed
    from a CUDA graph of the launches: each takes less time on the device than its issue."""
    out = []
    rows = cols = 4096
    n = rows * cols
    for dt in (torch.bfloat16, torch.float32):
        esz = torch.empty((), dtype=dt).element_size()
        ns = sets_for(n * esz + 2 * n)
        src = [torch.randn(rows, cols, device=DEV).to(dt) for _ in range(ns)]
        q = [torch.empty(rows, cols, device=DEV, dtype=torch.float8_e4m3fn) for _ in range(ns)]
        qt = [torch.empty(cols, rows, device=DEV, dtype=torch.float8_e4m3fn) for _ in range(ns)]
        sc = torch.zeros(2, device=DEV)
        _native.fp8_amax(src[0], sc[:1])
        name = str(dt).replace("torch.", "")
        out.append(timed("K9 fp8_amax %s [4096,4096]" % name,
                         lambda i: _native.fp8_amax(src[i], sc[:1]), ns, n * esz, iters, graph=True))
        out.append(timed("K9 fp8_quantize %s -> e4m3 [4096,4096] row-major + transposed" % name,
                         lambda i: _native.fp8_quantize(src[i], sc[:1], _native.FP8_E4M3, q[i], qt[i], sc[1:]),
                         ns, n * esz + 2 * n, iters, graph=True))
        out.append(timed("K9 fp8_quantize %s -> e4m3 [4096,4096] row-major only" % name,
                         lambda i: _native.fp8_quantize(src[i], sc[:1], _native.FP8_E4M3, q[i], None, sc[1:]),
                         ns, n * esz + n, iters, graph=True))
        del src, q, qt
    return out


def bench_k13(iters):
    """K13 against what it replaces, torch.mm then K6b, and against torch.mm alone: L2-cold (rotating
    operand sets), each arm timed from a CUDA graph, the three arms alternated over 3 rounds."""
    out = []
    B, N = 4096, 4096
    for K in (4096, 1064):
        per = (B * K + K * N + 3 * B * N) * 2
        ns = sets_for(per)
        ld = -(-K // _native.DX_DRELU_ROW_ALIGN) * _native.DX_DRELU_ROW_ALIGN   # the step's row stride
        dz_up = [torch.randn(B, ld, device=DEV).bfloat16()[:, :K] for _ in range(ns)]
        w = [torch.randn(K, N, device=DEV).bfloat16() for _ in range(ns)]
        act = [torch.randn(B, N, device=DEV).relu().bfloat16() for _ in range(ns)]
        dz = [torch.empty(B, N, device=DEV, dtype=torch.bfloat16) for _ in range(ns)]
        dx = [torch.empty(B, N, device=DEV, dtype=torch.bfloat16) for _ in range(ns)]
        db = torch.empty(N, device=DEV, dtype=torch.bfloat16)

        def k13(i):
            _native.dx_gemm_drelu(dz_up[i], w[i], act[i], dz[i], db)

        def mm(i):
            torch.mm(dz_up[i], w[i], out=dx[i])

        def mm_k6b(i):
            mm(i)
            _native.drelu_colsum(dx[i], act[i], dz[i], db)

        shape = "[%d,%d]x[%d,%d]" % (B, K, K, N)
        for _ in range(3):
            out.append(timed("K13 dx_gemm_drelu " + shape, k13, ns, per, iters, graph=True))
            out.append(timed("torch.mm + K6b drelu_colsum " + shape, mm_k6b, ns, per + 4 * B * N, iters,
                             graph=True))
            out.append(timed("torch.mm " + shape, mm, ns, per - 2 * B * N, iters, graph=True))
        del dz_up, w, act, dz, dx
    return out


def _muon_case(shapes):
    """A FusedMuon over 2-D weights of ``shapes`` (plus one bias), bf16 gradients in place."""
    import torch.nn as nn
    from frl_b200 import fused_optim
    from frl_b200.arena import ParamArena
    from frl_b200.multi_tensor import GradSegTable
    from frl_b200.types import Precision
    params = [nn.Parameter(torch.randn(sh) * 0.02) for sh in shapes] + [nn.Parameter(torch.zeros(64))]
    arena = ParamArena(params, device=DEV, precision=Precision.BF16)
    opt = fused_optim.FusedMuon(arena, lr=1e-3, weight_decay=1e-5)
    table = GradSegTable(arena.slots, DEV)
    grads = [torch.randn(s.shape, device=DEV).bfloat16() for s in arena.slots]
    for s, g in zip(arena.slots, grads):
        table.point(s, g.data_ptr(), g.dtype)
    table.upload()
    return opt, table, grads


def bench_k14(iters):
    """K14 (Muon) phase by phase at [4096, 4096] and [1000, 4096]: the kernels' device times from
    torch.profiler over ``iters`` updates captured in a CUDA graph (each update's last NS launch is
    the weight-writing update), against torch.mm / torch.addmm computing the same bf16 products
    from a graph.  TFLOP/s counts the full product and, for gram and poly, the tiles K14 computes
    (on or above the diagonal); the whole update is L2-warm after the first product."""
    from torch.profiler import ProfilerActivity, profile
    out = []
    for R, C in ((4096, 4096), (1000, 4096)):
        m, n = min(R, C), max(R, C)
        tm, tn = -(-m // 128), -(-m // 256)
        frac = sum(max(tn - a // 2, 0) for a in range(tm)) / (tm * tn)
        flops = {"gram": 2.0 * m * m * n, "poly": 2.0 * m * m * m, "update": 2.0 * m * m * n,
                 "last update": 2.0 * m * m * n}
        opt, table, grads = _muon_case([(R, C)])
        for _ in range(WARMUP):
            opt.apply_table(table)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for _ in range(iters):
                opt.apply_table(table)
        g.replay()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            g.replay()
            torch.cuda.synchronize()
        evs = sorted([e for e in prof.events() if e.device_type.name == "CUDA" and "muon" in e.name],
                     key=lambda e: e.time_range.start)
        times = {}
        ns_per_update = 3 * 5
        per_update = 2 + ns_per_update
        for i, e in enumerate(evs):
            j = i % per_update
            name = ("prologue" if j == 0 else "normalise" if j == 1 else
                    ("gram", "poly", "update")[(j - 2) % 3])
            if j == per_update - 1:
                name = "last update"
            times.setdefault(name, []).append(e.time_range.elapsed_us())
        x = torch.randn(m, n, device=DEV).bfloat16()
        a = torch.randn(m, m, device=DEV).bfloat16()
        o_mm = torch.empty(m, m, device=DEV, dtype=torch.bfloat16)
        o_x = torch.empty(m, n, device=DEV, dtype=torch.bfloat16)
        refs = {"gram": lambda i: torch.mm(x, x.T, out=o_mm),
                "poly": lambda i: torch.addmm(a, a, a, beta=-4.775, alpha=2.0315, out=o_mm),
                "update": lambda i: torch.addmm(x, a, x, beta=3.4445, out=o_x)}
        shape = "[%d,%d]" % (R, C)
        for name in ("prologue", "normalise", "gram", "poly", "update", "last update"):
            ts = times.get(name, [])
            if not ts:
                continue
            us = sum(ts) / len(ts)
            rec = {"kernel": "K14 %s %s" % (name, shape), "us": round(us, 2), "launches": len(ts)}
            if name in flops:
                f = flops[name] * (frac if name in ("gram", "poly") else 1.0)
                rec["TFLOPs_full_product"] = round(flops[name] / us / 1e6, 1)
                rec["TFLOPs_tiles_computed"] = round(f / us / 1e6, 1)
            print(json.dumps(rec), flush=True)
            out.append(rec)
        for name, fn in refs.items():
            rec = timed("torch %s %s (bf16, cuBLAS)" % ("mm" if name == "gram" else "addmm", name + " " + shape),
                        fn, 1, 0, iters, graph=True)
            rec["TFLOPs"] = round(flops[name] / rec["us"] / 1e6, 1)
            print(json.dumps({"kernel": rec["kernel"], "TFLOPs": rec["TFLOPs"]}), flush=True)
            out.append(rec)
        total = sum(sum(v) for v in times.values()) / iters
        print(json.dumps({"kernel": "K14 whole update %s" % shape, "us": round(total, 1)}), flush=True)
        del opt, table, grads, g
    return out


def bench_k5nhwc(iters):
    """K5 and K5a into channels_last against their NCHW forms, alternating, same sets: K5 u8 ->
    bf16 [256, 3, 224, 224] per channel, and K5a RRC u8 [256, 3, 256, 256] -> bf16 [256, 3, 224, 224]
    (bytes as bench_k5a).  Every form is timed from a CUDA graph over rotating L2-cold sets."""
    B, Cc, H = 256, 3, 224
    n = B * Cc * H * H
    ns = sets_for(n * 3)
    src = [torch.randint(0, 256, (B, Cc, H, H), device=DEV, dtype=torch.uint8) for _ in range(ns)]
    fmt = {"NCHW": torch.contiguous_format, "NHWC": torch.channels_last}
    dst = {k: [torch.empty(B, Cc, H, H, device=DEV, dtype=torch.bfloat16, memory_format=f) for _ in range(ns)]
           for k, f in fmt.items()}
    sc, bi = torch.rand(Cc, device=DEV), torch.rand(Cc, device=DEV)
    k5 = {"NCHW": lambda i: _native.preproc_affine(src[i], dst["NCHW"][i], inner=H * H, channels=Cc, scale=sc, bias=bi),
          "NHWC": lambda i: _native.preproc_affine_nhwc(src[i], dst["NHWC"][i], scale=sc, bias=bi)}
    out = []
    for rep in range(2):
        for k in ("NCHW", "NHWC"):
            out.append(timed("K5 preproc_affine%s u8->bf16 [256,3,224,224] per-channel, %s out (round %d)"
                             % ("_nhwc" if k == "NHWC" else "", k, rep), k5[k], ns, n * 3, iters, graph=True))
    del src, dst
    S, O = 256, 224
    ns = sets_for(B * Cc * (S * S + 2 * O * O))
    src = [torch.randint(0, 256, (B, Cc, S, S), device=DEV, dtype=torch.uint8) for _ in range(ns)]
    dst = {k: [torch.empty(B, Cc, O, O, device=DEV, dtype=torch.bfloat16, memory_format=f) for _ in range(ns)]
           for k, f in fmt.items()}
    idx = [torch.arange(B, device=DEV, dtype=torch.int64) + i * B for i in range(ns)]
    params = torch.empty(B, 5, dtype=torch.int32, device=DEV)
    read = 0
    for i in range(ns):
        _native.augment_images(src[i], idx[i], dst["NCHW"][i], seed=0, epoch=1, mode=_native.AUG_RRC, scale=sc,
                               bias=bi, params_out=params)
        read += sum(Cc * _taps_touched(int(h), O) * _taps_touched(int(w), O) for h, w in params[:, 2:4].tolist())
    nbytes = read // ns + B * Cc * O * O * 2
    kw = dict(seed=0, epoch=1, mode=_native.AUG_RRC, scale=sc, bias=bi)
    for rep in range(2):
        for k in ("NCHW", "NHWC"):
            out.append(timed("K5a augment_images%s RRC u8 [256,3,256,256] -> bf16 [256,3,224,224] %s (round %d)"
                             % ("_nhwc" if k == "NHWC" else "", k, rep),
                             lambda i, k=k: _native.augment_images(src[i], idx[i], dst[k][i], **kw), ns, nbytes,
                             iters, "bytes: touched source lines of the drawn boxes + output", graph=True))
    return out


def bench_k2g(iters):
    """Grouped K2-mt (``frl_*_mt_grouped``) against ungrouped K2-mt on the headline MLP's arena (10
    tensors, 54.7 M parameters) for SGD-momentum and AdamW: bf16 gradients in the arena, bf16 shadow,
    fp32 state, each timed from a CUDA graph; the arena (1.1 / 1.5 GB of traffic per launch) is far
    larger than L2, so every launch streams from HBM.  Three groups: the tensors with ndim <= 1 at
    wd 0, the trunk at half the lr, the heads at the default.  Five rounds, ungrouped and grouped
    alternating; the last record per rule is the medians (min-max) and grouped / ungrouped, against
    the target of 1.02 at the same bytes per parameter."""
    from frl_b200.multi_tensor import GradSegTable

    class Slot:
        def __init__(self, index, offset, shape):
            self.index, self.offset, self.shape = index, offset, shape
            self.numel = 1
            for d in shape:
                self.numel *= d
            self.is_model = True

    shapes = [(4096, 4096), (4096,)] * 3 + [(1000, 4096), (1000,), (64, 4096), (64,)]
    slots, off = [], 0
    for i, sh in enumerate(shapes):
        slots.append(Slot(i, off, sh))
        off = (off + slots[-1].numel + 7) // 8 * 8
    n, n_real = off, sum(s.numel for s in slots)
    grad = torch.randn(n, device=DEV).bfloat16()
    table = GradSegTable(slots, DEV)
    for s in slots:
        table.point(s, grad.data_ptr() + 2 * s.offset, grad.dtype)
    table.upload()
    seg_group = [0 if len(s.shape) <= 1 else (1 if i < 6 else 2) for i, s in enumerate(slots)]
    p = torch.randn(n, device=DEV) * 0.02
    lp = torch.empty(n, device=DEV, dtype=torch.bfloat16)
    m, v = torch.randn(n, device=DEV) * 1e-3, torch.rand(n, device=DEV) * 1e-6
    lr, wd, step = 1e-3, 1e-2, 3
    out = []
    for rule, bpp in (("sgd", 20), ("adamw", 28)):
        rows = torch.zeros(3, _native.GROUP_DYN_COLS)
        for gi, (glr, gwd) in enumerate(((lr, 0.0), (0.5 * lr, wd), (lr, wd))):
            if rule == "sgd":
                rows[gi, 0] = glr
            else:
                rows[gi, 0] = -(glr / (1 - 0.9 ** step))
                rows[gi, 1] = (1 - 0.999 ** step) ** 0.5
                rows[gi, 2] = 1 - glr * gwd
            rows[gi, 4] = gwd
        rows.view(torch.int32)[:, 3] = step
        groups = _native.SegGroups(seg_group, [_native.LW_CLIPPED] * len(slots), rows.to(DEV))
        if rule == "sgd":
            fns = {"ungrouped": lambda i: _native.sgd_momentum_mt(p, m, lp, table, lr=lr, mu=0.9, dampening=0.0,
                                                                  wd=wd, first_step=False),
                   "grouped": lambda i: _native.sgd_momentum_mt_grouped(p, m, lp, table, groups, mu=0.9,
                                                                        dampening=0.0, first_step=False)}
        else:
            fns = {"ungrouped": lambda i: _native.adamw_mt(p, m, v, None, lp, table, lr=lr, beta1=0.9, beta2=0.999,
                                                           eps=1e-8, wd=wd, step=step),
                   "grouped": lambda i: _native.adamw_mt_grouped(p, m, v, None, lp, table, groups, beta1=0.9,
                                                                 beta2=0.999, eps=1e-8)}
        times = {"ungrouped": [], "grouped": []}
        for r in range(5):
            for form in ("ungrouped", "grouped"):
                rec = timed("K2-mt %s %s mlp bf16-grad (%d tensors, %d params, 3 groups) round %d"
                            % (rule, form, len(slots), n_real, r), fns[form], 1, bpp * n_real, iters,
                            "%d B/param" % bpp, graph=True)
                times[form].append(rec["us"])
                out.append(rec)
        med = {k: sorted(t)[len(t) // 2] for k, t in times.items()}
        summary = {"kernel": "K2-mt %s grouped vs ungrouped, median of 5 (min-max)" % rule,
                   "ungrouped_us": "%.1f (%.1f-%.1f)" % (med["ungrouped"], min(times["ungrouped"]),
                                                        max(times["ungrouped"])),
                   "grouped_us": "%.1f (%.1f-%.1f)" % (med["grouped"], min(times["grouped"]), max(times["grouped"])),
                   "grouped_over_ungrouped": round(med["grouped"] / med["ungrouped"], 4),
                   "within_2pct": med["grouped"] <= 1.02 * med["ungrouped"]}
        print(json.dumps(summary), flush=True)
        out.append(summary)
    return out


BENCHES = {"k2": bench_k2, "k2mt": bench_k2mt, "k2lw": bench_k2lw, "k3": bench_k3, "k4": bench_k4, "k5": bench_k5, "k5a": bench_k5a,
           "k5m": bench_k5m, "k4s": bench_k4s, "k6": bench_k6,
           "k8": bench_k8, "k8t": bench_k8t, "k9": bench_k9, "k10": bench_k10, "k11": bench_k11,
           "k2q8": bench_k2q8, "k2af": bench_k2af, "k13": bench_k13, "k14": bench_k14, "k2w": bench_k2w,
           "k5nhwc": bench_k5nhwc, "k2lion": bench_k2lion, "k2g": bench_k2g}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default="k2,k2mt,k3,k4,k5,k6,k8,k9")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--json", default=None)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--max-sets", type=int, default=0)
    args = ap.parse_args()
    global WARMUP, MAX_SETS
    WARMUP, MAX_SETS = args.warmup, args.max_sets
    torch.cuda.set_device(0)
    recs = []
    for key in args.only.split(","):
        recs += BENCHES[key](args.iters)
        torch.cuda.empty_cache()
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"peak_hbm_gbs": peak_gbs(), "kernels": recs}, f, indent=1)


if __name__ == "__main__":
    main()
