#!/usr/bin/env python
"""Micro-benchmark of every hand-written kernel at the BASELINE shapes (1 GPU).

    python tools/kernel_bench.py [--only k2,k2lw,k3,k5a,...] [--iters 20] [--json out.json]

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


BENCHES = {"k2": bench_k2, "k2mt": bench_k2mt, "k2lw": bench_k2lw, "k3": bench_k3, "k4": bench_k4, "k5": bench_k5, "k5a": bench_k5a,
           "k5m": bench_k5m, "k4s": bench_k4s, "k6": bench_k6,
           "k8": bench_k8, "k8t": bench_k8t, "k9": bench_k9, "k10": bench_k10, "k11": bench_k11}


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
