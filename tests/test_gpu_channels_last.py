"""channels_last training on the GPU.

* K5 and K5a into channels_last (``frl_preproc_affine_nhwc``, ``frl_augment_images_nhwc``,
  ``frl_augment_mix_images_nhwc``) write the NCHW kernels' values bit for bit, permuted.
* The small conv Problem of test_gpu_resnet.py with ``channels_last=True`` against the stock-torch
  loop on a channels_last copy of its model on the same GPU: parameters keep channels_last strides and
  every conv weight gradient is read in place.
* ResNet-18 in bf16 with channels_last tracks the CPU oracle.
* Resume bit for bit NHWC -> NHWC, and NCHW <-> NHWC checkpoint loads, for Adam, 8-bit state, LARS,
  Muon, EMA and gradient accumulation; every tensor of the files is contiguous.
* ``testIO`` samples of an NHWC run equal an NCHW run's; the MLP's ``--dump-outputs`` do not change.
* Two ranks over gloo on one GPU agree bit for bit (tests/run_channels_last_mp.py).
"""
import copy
import io
import os
import random
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch
import torch.nn as nn

import frl_b200  # noqa: F401
from frl_b200 import _native, multi_tensor, synthetic
from frl_b200.ema import EMA_STATE_KEY
from frl_b200.grad_sync import accumulation_plan
from frl_b200.solver import Solver, SolverWorkerArgs
from frl_b200.types import Device, LayerAdaptation, Mode, OptimizerState, Precision, Split
from oracle import ref_loop

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = torch.device("cuda", 0)
CL = torch.channels_last
SEED = 3


# ---- K5 / K5a -------------------------------------------------------------------------------------------

@pytest.mark.parametrize("C", [1, 3, 4])
@pytest.mark.parametrize("hw", [(7, 9), (8, 12)])           # odd plane: one pixel per thread; else four
@pytest.mark.parametrize("src_dtype", [torch.uint8, torch.float32, torch.bfloat16])
@pytest.mark.parametrize("dst_dtype", [torch.float32, torch.bfloat16])
def test_k5_nhwc_is_k5_permuted(C, hw, src_dtype, dst_dtype):
    from test_channels_last_host import k5_nhwc_np
    g = torch.Generator(device=DEV).manual_seed(C)
    B = 5
    if src_dtype == torch.uint8:
        src = torch.randint(0, 256, (B, C) + hw, generator=g, device=DEV, dtype=torch.uint8)
    else:
        src = (torch.randn((B, C) + hw, generator=g, device=DEV) * 40).to(src_dtype)
    scale = torch.tensor([1 / (255 * (0.2 + 0.05 * c)) for c in range(C)], device=DEV)
    bias = torch.tensor([-0.5 + 0.1 * c for c in range(C)], device=DEV)
    for sc, bi in ((scale, bias), (None, bias), (scale, None), (None, None)):
        want = torch.empty(src.shape, dtype=dst_dtype, device=DEV)
        _native.preproc_affine(src, want, inner=hw[0] * hw[1], channels=C, scale=sc, bias=bi)
        got = torch.empty(src.shape, dtype=dst_dtype, device=DEV, memory_format=CL)
        _native.preproc_affine_nhwc(src, got, scale=sc, bias=bi)
        assert got.is_contiguous(memory_format=CL)
        stored = got.permute(0, 2, 3, 1)
        assert torch.equal(stored.view(torch.int16 if dst_dtype == torch.bfloat16 else torch.int32),
                           want.permute(0, 2, 3, 1).contiguous().view(
                               torch.int16 if dst_dtype == torch.bfloat16 else torch.int32))
        ref = k5_nhwc_np(src.float().cpu().numpy(), None if sc is None else sc.cpu().tolist(),
                         None if bi is None else bi.cpu().tolist(), dst_dtype)
        assert torch.equal(stored.cpu(), ref)


def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)


@pytest.mark.parametrize("C", [1, 3, 4])
@pytest.mark.parametrize("dst_dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("B", [5, 8])
def test_k5a_nhwc_is_k5a_permuted(C, dst_dtype, B):
    g = torch.Generator(device=DEV).manual_seed(B * C)
    src = torch.randint(0, 256, (B, C, 37, 41), generator=g, device=DEV, dtype=torch.uint8)
    idx = torch.arange(B, device=DEV, dtype=torch.int64) * 7 + 3
    sc = torch.rand(C, device=DEV) * 0.02
    bi = torch.rand(C, device=DEV) - 0.5
    out = (24, 20)
    modes = [_native.AUG_RRC, _native.AUG_PAD_CROP, _native.AUG_CENTER_RESIZE, _native.AUG_CENTER_CROP]
    mixes = [None, (_native.MIX_MIXUP, 0.7, (0, 0, 0, 0)), (_native.MIX_CUTMIX, 0.75, (3, 15, 4, 12))]
    for mode in modes:
        for mix in mixes:
            res = []
            for fmt in (torch.contiguous_format, CL):
                dst = torch.empty((B, C) + out, dtype=dst_dtype, device=DEV, memory_format=fmt)
                params = torch.zeros(B, 5, dtype=torch.int32, device=DEV)
                kw = dict(seed=11, epoch=2, mode=mode, pad=4, scale=sc, bias=bi, params_out=params)
                if mix is None:
                    _native.augment_images(src, idx, dst, **kw)
                else:
                    _native.augment_mix_images(src, idx, dst, mix_mode=mix[0], lam=mix[1], box=mix[2], **kw)
                res.append((dst, params))
            (a, pa), (b, pb) = res
            assert b.is_contiguous(memory_format=CL)
            assert torch.equal(pa, pb)
            assert torch.equal(_bits(b.permute(0, 2, 3, 1)), _bits(a.permute(0, 2, 3, 1).contiguous())), (mode, mix)


def test_device_transforms_honour_the_memory_format():
    from frl_b200.transform import DeviceImageAugment
    aug = DeviceImageAugment("x", ["y"], mode="rrc", out_size=16, scale=(0.01,) * 3, bias=(-0.5,) * 3)
    x = torch.randint(0, 256, (6, 3, 20, 20), device=DEV, dtype=torch.uint8)
    idx = torch.arange(6, device=DEV)
    a = aug.augment(x, idx, Split.TRAIN, torch.bfloat16)
    aug.memory_format = CL
    b = aug.augment(x, idx, Split.TRAIN, torch.bfloat16)
    assert a.is_contiguous() and _native.is_nhwc(b) and torch.equal(a, b)
    t = synthetic._channel_affine_device_transform((0.1, 0.2, 0.3), (1.0, 2.0, 3.0), ["y"])
    raw = {"x": x, "y": idx}
    (a,), _ = t.apply(raw, Split.TRAIN, torch.float32)
    t.memory_format = CL
    (b,), _ = t.apply(raw, Split.TRAIN, torch.float32)
    assert a.is_contiguous() and _native.is_nhwc(b) and torch.equal(a, b)


def test_cast_and_window_gather_keep_channels_last():
    """_cast_inputs casts a channels_last fp32 batch in its storage order; K8w gathers retained
    channels_last batches as their NHWC rows, without a copy of the window."""
    from frl_b200.solver_worker import SamplerState, SolverWorker
    x = torch.randn(6, 3, 5, 7, device=DEV).to(memory_format=CL)
    w = SolverWorker.__new__(SolverWorker)
    w.precision = Precision.BF16
    (lp,) = w._cast_inputs([x])
    assert _native.is_nhwc(lp) and torch.equal(lp, x.to(torch.bfloat16))
    batches = [torch.randn(4, 3, 5, 7, device=DEV).to(memory_format=CL) for _ in range(3)]
    idx = torch.tensor([0, 5, 11, 7], device=DEV)
    rows = SamplerState._gather_rows(batches, idx)
    assert _native.is_nhwc(rows) and torch.equal(rows, torch.cat(batches)[idx])


# ---- the small conv Problem against stock torch ---------------------------------------------------------

def _conv_problem(ns, save_dir, n=64, uint8=False, pinned=False):
    Reg, Cls = synthetic._task_classes(ns)
    tasks = [Cls(32, 10, 1.0, field="y_cls", name="cls"), Reg(32, 4, 1.0, field="y_reg", name="reg")]
    heads = [("cls", 10, "y_cls", "cls"), ("reg", 4, "y_reg", "reg")]

    def base():
        return nn.Sequential(ns.model.ListSelect(sel_index=0, num_elements=1),
                             nn.Conv2d(3, 16, 3, padding=1), nn.ReLU(), nn.Conv2d(16, 32, 3, stride=2, padding=1),
                             nn.ReLU(), nn.AdaptiveAvgPool2d(1), nn.Flatten())
    fields = [(ns.Split.TRAIN, synthetic.resnet_fields(n, 16, heads, 0, uint8))]
    return synthetic._problem_class(ns)(tasks, [], fields, save_dir, shift=0.0, scale=1.0, base_factory=base,
                                        pinned=pinned,
                                        channel_affine=synthetic.U8_CHANNEL_AFFINE if uint8 else None)


class _Deterministic:
    def __init__(self, monkeypatch):
        monkeypatch.setenv("FRL_B200_CUDNN_BENCHMARK", "0")

    def __enter__(self):
        self.old = (torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic,
                    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
        torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic = False, True
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False

    def __exit__(self, *exc):
        (torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic,
         torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32) = self.old


def _solve_capturing(run_opts, problem, **kw):
    captured = {}
    orig = Solver.build_worker.__func__

    def spy(cls, args):
        worker, sched, ckpt = orig(cls, args)
        captured["worker"] = worker
        return worker, sched, ckpt

    Solver.build_worker = classmethod(spy)
    try:
        list(Solver.solve(run_opts, problem, group_name=None, init_method="file:///tmp/unused", **kw))
    finally:
        Solver.build_worker = classmethod(orig)
    return captured["worker"]


@pytest.mark.parametrize("graph", ["0", "1"])
@pytest.mark.parametrize("clip", [0.0, 0.5])
def test_conv_problem_channels_last_matches_stock_torch(ns, monkeypatch, graph, clip):
    monkeypatch.setenv("FRL_B200_CUDA_GRAPH", graph)
    decisions = []
    orig_in_place = multi_tensor.grad_usable_in_place

    def recording(g, slot):
        ok = orig_in_place(g, slot)
        if len(slot.shape) == 4:
            decisions.append((tuple(g.stride()), ok))
        return ok

    monkeypatch.setattr(multi_tensor, "grad_usable_in_place", recording)
    t = ns.types
    run_opts = t.RunOpts(optim=t.OptimOpts(algo=t.OptAlgorithm.SGD, lr=0.05, gradientClip=clip), batchSize=8,
                         nEpochs=1, numThreads=0, singleThreaded=True, numVisualizedSamples=0)
    with _Deterministic(monkeypatch):
        torch.manual_seed(SEED)
        ref_problem = _conv_problem(ns, "/tmp/unused")
        ref_model = ref_problem.get_model().to(memory_format=CL)
        crit = ref_problem.get_criterion()
        spec = ref_loop.RunSpec(optim=ref_loop.OptimSpec(algo="sgd", lr=0.05, gradient_clip=clip), batch_size=8,
                                n_epochs=1)
        trace = ref_loop.train(ref_model, list(crit.loss_modules), list(crit.loss_weights), list(crit.loss_names),
                               [(d.data_type.value, d) for d in ref_problem.datasets], spec, device=DEV)
        save_dir = tempfile.mkdtemp(prefix="frl_b200_cl_conv_")
        torch.manual_seed(SEED)
        worker = _solve_capturing(run_opts, _conv_problem(ns, save_dir), channels_last=True)
    convs = [s for s in worker.arena.slots if len(s.shape) == 4]
    assert len(convs) == 2 and worker.arena.n_channels_last == 2
    for s in convs:
        assert s.param.is_contiguous(memory_format=CL) and not s.param.is_contiguous()
    assert decisions and all(ok for _, ok in decisions), decisions
    if graph == "1":
        assert worker.graphed is not None and len(worker.graphed._graphs) == 1
    rows = np.concatenate([r for _, _, r in worker.loss_history])
    want = np.concatenate([trace.losses[k] for k in sorted(trace.losses)])
    assert rows.shape == want.shape == (8, 3)
    np.testing.assert_allclose(rows, want, rtol=1e-4, atol=1e-6)
    final = torch.load(os.path.join(save_dir, "final_model.pth"), weights_only=False)["state_dict"]
    for k, v in ref_model.state_dict().items():
        assert final[k].is_contiguous(), k
        peak = float(v.abs().max())
        assert float((final[k] - v.cpu()).abs().max()) <= 1e-4 * peak, k


def test_resnet18_bf16_channels_last_tracks_the_oracle(ns):
    """test_resnet18_bf16_mode_tracks_the_oracle's bounds, channels_last."""
    t = ns.types
    problem = synthetic.make_resnet_problem(ns, "/tmp/unused", "resnet18", image=64, n_train=16)
    spec = ref_loop.RunSpec(optim=ref_loop.OptimSpec(algo="sgd", lr=0.01), batch_size=8, n_epochs=1)
    torch.manual_seed(SEED)
    model = problem.get_model()
    crit = problem.get_criterion()
    trace = ref_loop.train(model, list(crit.loss_modules), list(crit.loss_weights), list(crit.loss_names),
                           [(d.data_type.value, d) for d in problem.datasets], spec)
    run_opts = t.RunOpts(optim=t.OptimOpts(algo=t.OptAlgorithm.SGD, lr=0.01), batchSize=8, nEpochs=1,
                         numThreads=0, singleThreaded=True, numVisualizedSamples=0)
    save_dir = tempfile.mkdtemp(prefix="frl_b200_cl_r18_")
    torch.manual_seed(SEED)
    worker = _solve_capturing(run_opts, synthetic.make_resnet_problem(ns, save_dir, "resnet18", image=64, n_train=16),
                              precision=Precision.BF16, channels_last=True)
    assert worker.arena.n_channels_last == 20
    rows = np.concatenate([r for _, _, r in worker.loss_history])
    want = np.concatenate([trace.losses[k] for k in sorted(trace.losses)])
    np.testing.assert_allclose(rows[0], want[0], rtol=1e-2, atol=1e-2)
    np.testing.assert_allclose(rows[1], want[1], rtol=3e-2, atol=3e-2)
    assert np.isfinite(rows).all()


# ---- checkpoints across layouts -----------------------------------------------------------------------------

RESUME_CASES = {
    # name: (algo, lr, SolverWorkerArgs extras)
    "adam": ("adam", 1e-3, {}),
    "adam_8bit": ("adam", 1e-3, {"optimizer_state": OptimizerState.Q8}),
    "lars": ("sgd", 0.5, {"layer_adaptation": LayerAdaptation.LARS}),
    "muon": ("adam", 1e-3, {"muon": True}),
    "adam_ema": ("adam", 1e-3, {"ema_decay": 0.9}),
    "sgd_accum": ("sgd", 0.05, {"grad_accumulation": 2}),
}
STEPS, HALF = 8, 4


def _worker(ns, case, channels_last, seed):
    algo, lr, extra = RESUME_CASES[case]
    t = ns.types
    save_dir = tempfile.mkdtemp(prefix="frl_b200_cl_resume_")
    torch.manual_seed(seed)
    problem = _conv_problem(ns, save_dir)
    run_opts = t.RunOpts(optim=t.OptimOpts(algo=t.OptAlgorithm(algo), lr=lr, weightDecay=1e-4), batchSize=8,
                         nEpochs=1, numThreads=0, singleThreaded=True, numVisualizedSamples=0)
    args = SolverWorkerArgs(run_opts=run_opts, problem=problem, save_dir=save_dir, run_device=Device.GPU,
                            node_idx=0, node_count=1, rank=0, local_rank=0, world_size=1, group_name=None,
                            init_method="", precision=Precision.FP32, channels_last=channels_last, **extra)
    worker, _, _ = Solver.build_worker(args)
    worker.model.train()
    worker.criterion.train()
    return worker


def _batches():
    g = torch.Generator().manual_seed(1234)
    return [(torch.randn(8, 3, 16, 16, generator=g), torch.randint(0, 10, (8,), generator=g),
             torch.randn(8, 4, generator=g)) for _ in range(STEPS)]


def _train(worker, batches, start):
    plan = accumulation_plan(STEPS, worker.pipeline.accumulation, 8) if worker.pipeline.accumulation > 1 else None
    rows = []
    for i in range(start, start + len(batches)):
        x, y, r = batches[i - start]
        if plan is not None:
            mb = plan[i]
            worker.pipeline.set_microbatch(first=mb.first, closes=mb.closes, weight=mb.weight,
                                           group_scale=8 / mb.group_rows)
        _, total, _, _ = worker._pass_one_minibatch(i, Split.TRAIN, [x.to(DEV)], [(y.to(DEV),), (r.to(DEV),)])
        rows.append(float(total.detach()))
        del total
    torch.cuda.synchronize()
    return rows


def _files(worker):
    """The model and optimizer-state bytes a checkpoint is written from, loaded back."""
    frac = worker._get_worker_performance_summary({})
    model = torch.load(io.BytesIO(frac.modelBuffer), weights_only=False)
    opt = torch.load(io.BytesIO(frac.optimizerStateBuffer), weights_only=False)
    return model.state_dict(), opt


def _tensors(obj):
    if torch.is_tensor(obj):
        yield obj
    elif isinstance(obj, dict):
        for v in obj.values():
            yield from _tensors(v)
    elif isinstance(obj, (list, tuple)):
        for v in obj:
            yield from _tensors(v)


def _resume(worker, model_sd, opt):
    opt = copy.deepcopy(opt)
    ema = opt.pop(EMA_STATE_KEY, None)
    with torch.no_grad():
        worker.model.load_state_dict(model_sd)
    worker.arena.refresh_shadow()
    worker.optimizer.load_state_dict(opt)
    if ema is not None:
        worker.ema.load_state_dict(ema)


@pytest.mark.parametrize("case", sorted(RESUME_CASES))
def test_resume_and_cross_layout_checkpoints(ns, case, monkeypatch):
    with _Deterministic(monkeypatch):
        batches = _batches()
        runs = {}
        for cl in (False, True):
            a = _worker(ns, case, cl, SEED)
            if cl:
                assert a.arena.n_channels_last == 2
            _train(a, batches[:HALF], 0)
            model_sd, opt = _files(a)
            assert all(t.is_contiguous() for t in _tensors((model_sd, opt))), case
            rows = _train(a, batches[HALF:], HALF)
            runs[cl] = (model_sd, opt, rows, a.arena.master.clone(), _files(a))
        # the two layouts write files of the same keys, shapes, dtypes and strides
        for x, y in zip(_tensors(runs[False][:2]), _tensors(runs[True][:2])):
            assert x.shape == y.shape and x.dtype == y.dtype and x.stride() == y.stride()
        # NHWC -> NHWC: bit for bit
        b = _worker(ns, case, True, SEED + 4)
        _resume(b, *runs[True][:2])
        assert _train(b, batches[HALF:], HALF) == runs[True][2]
        assert torch.equal(b.arena.master, runs[True][3])
        # NCHW -> NHWC and NHWC -> NCHW: the other layout's convolutions, same run
        loose = 1e-2 if case == "adam_8bit" else 1e-3      # 8-bit blocks group other elements in NHWC
        for src, dst in ((False, True), (True, False)):
            c = _worker(ns, case, dst, SEED + 5)
            _resume(c, *runs[src][:2])
            rows = _train(c, batches[HALF:], HALF)
            np.testing.assert_allclose(rows, runs[dst][2], rtol=loose, atol=1e-6, err_msg="%s %s->%s" % (case, src, dst))
            got, want = _files(c)[0], runs[dst][4][0]
            for k, v in want.items():
                peak = float(v.abs().max()) or 1.0
                assert float((got[k] - v).abs().max()) <= 10 * loose * peak, (case, k)


# ---- testIO, the MLP's outputs, two ranks ---------------------------------------------------------------------

def test_testio_samples_of_nhwc_and_nchw_runs_agree(ns):
    t = ns.types
    picked = {}
    for cl in (False, True):
        save_dir = tempfile.mkdtemp(prefix="frl_b200_cl_testio_")
        torch.manual_seed(SEED)
        random.seed(5)
        problem = _conv_problem(ns, save_dir, n=48, uint8=True, pinned=True)
        run_opts = t.RunOpts(optim=t.OptimOpts(algo=t.OptAlgorithm.SGD, lr=0.05), batchSize=8, nEpochs=1,
                             numThreads=0, singleThreaded=True, numVisualizedSamples=4, mode=Mode.EVAL)
        args = SolverWorkerArgs(run_opts=run_opts, problem=problem, save_dir=save_dir, run_device=Device.GPU,
                                node_idx=0, node_count=1, rank=0, local_rank=0, world_size=1, group_name=None,
                                init_method="", precision=Precision.FP32, channels_last=cl)
        fracs = list(Solver._run_solver_worker(args))
        picked[cl] = fracs[-1].performance[Split.TRAIN].testIO
    assert len(picked[True]) == len(picked[False]) > 0
    for a, b in zip(picked[False], picked[True]):
        for x, y in zip(a.data, b.data):
            assert x.shape == y.shape and x.is_contiguous() and y.is_contiguous() and torch.equal(x, y)
        for x, y in zip(a.output, b.output):
            torch.testing.assert_close(x, y, rtol=1e-4, atol=1e-5)


def test_mlp_dump_outputs_do_not_change(tmp_path):
    out = {}
    for flag in ("0", "1"):
        d = str(tmp_path / flag)
        env = dict(os.environ, FRL_B200_CHANNELS_LAST=flag, PYTHONPATH=REPO)
        res = subprocess.run([sys.executable, os.path.join(REPO, "bench.py"), "--gpus", "1", "--steps", "3",
                              "--warmup", "2", "--batch", "512", "--no-torch-baseline", "--no-cpu-baseline",
                              "--no-e2e", "--dump-outputs", d], env=env, capture_output=True, text=True,
                             cwd=str(tmp_path), timeout=900)
        assert res.returncode == 0, res.stderr[-3000:]
        out[flag] = {f: np.load(os.path.join(d, f)) for f in sorted(os.listdir(d))}
    assert out["0"].keys() == out["1"].keys() and out["0"]
    for f in out["0"]:
        assert np.array_equal(out["0"][f], out["1"][f]), f


def test_two_gloo_ranks_agree_bit_for_bit():
    res = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nproc-per-node", "2",
                          os.path.join(REPO, "tests", "run_channels_last_mp.py")],
                         capture_output=True, text=True, timeout=600, cwd=REPO)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    assert res.stdout.count("CHANNELS_LAST_MP_OK") == 2, res.stdout
