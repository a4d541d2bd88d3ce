"""End-to-end parity of the H100 training step against the reference's CPU Solver.

The golden files hold what the UNMODIFIED reference produced on the toy 2-task Problem
(per-step losses of every split, learning rates, served sample order, first gradients, final
weights; see oracle/make_golden.py).  Here the same Problem and seed run through
``Solver.solve`` on cuda:0.  Bounds (BASELINE.json): indices bit-exact, losses/grads 1e-5 rel
in fp32, 1e-2 in bf16."""
import os
import tempfile

import numpy as np
import pytest
import torch

import frl_b200  # noqa: F401
from frl_b200 import _native, synthetic
from frl_b200.solver import Solver, SolverWorkerArgs
from frl_b200.types import Device, Precision
from oracle.make_golden import BATCH, CONFIGS, SEED

pytestmark = pytest.mark.gpu


def _run_opts(ns, cfg, **over):
    algo, lr, sched, n_epochs, clip, amsgrad, kind = cfg
    t = ns.types
    optim = t.OptimOpts(algo=t.OptAlgorithm(algo), lr=lr,
                        lr_scheduler=t.LRSchedulerOpts(algo=t.LRSchedulerAlgorithm(sched)),
                        gradientClip=clip, amsgrad=amsgrad)
    kw = dict(optim=optim, batchSize=BATCH, nEpochs=n_epochs, numThreads=0, singleThreaded=True,
              numVisualizedSamples=4)
    kw.update(over)
    return t.RunOpts(**kw)


def _solve_and_capture(ns, cfg, precision=Precision.FP32, **over):
    save_dir = tempfile.mkdtemp(prefix="frl_b200_test_")
    problem = synthetic.make_toy_problem(ns, save_dir, criterion_kind=cfg[6])
    run_opts = _run_opts(ns, cfg, **over)
    captured = {}
    orig = Solver.build_worker.__func__

    def spy(cls, args):
        worker, sched, ckpt = orig(cls, args)
        captured["worker"] = worker
        return worker, sched, ckpt

    Solver.build_worker = classmethod(spy)
    try:
        torch.manual_seed(SEED)
        summaries = list(Solver.solve(run_opts, problem, group_name=None, init_method="file:///tmp/unused",
                                      precision=precision))
    finally:
        Solver.build_worker = classmethod(orig)
    return summaries, captured["worker"], problem, save_dir


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_solver_matches_reference_solver(ns, golden_dir, name):
    g = np.load(os.path.join(golden_dir, name + ".npz"))
    before = _native.launch_count()
    summaries, worker, problem, save_dir = _solve_and_capture(ns, CONFIGS[name])
    assert _native.launch_count() - before >= len(g["rows"])         # our kernels did the work
    rows = np.concatenate([r for _, _, r in worker.loss_history])
    assert rows.shape == g["rows"].shape
    np.testing.assert_allclose(rows, g["rows"], rtol=1e-5, atol=1e-6)
    # sample order: exact
    assert problem.datasets[0].served == list(g["served_train"])
    assert problem.datasets[1].served == list(g["served_test"])
    # final weights written by the parent, standard fp32 state_dict
    final = torch.load(os.path.join(save_dir, "final_model.pth"), weights_only=False)
    assert final["epoch"] == CONFIGS[name][3]
    names = list(g["param_names"])
    assert list(final["state_dict"].keys()) == names
    # RMSprop divides by sqrt(v)+1e-8: elements with a tiny second moment amplify fp32 rounding
    ptol = 1e-3 if name == "toy_rmsprop" else 2e-4
    for i, k in enumerate(names):
        np.testing.assert_allclose(final["state_dict"][k].numpy(), g["param_%02d" % i],
                                   rtol=ptol, atol=ptol * 1e-2)
    # epoch means reported through the public summaries = unweighted mean of the step losses
    last = summaries[-1]
    assert last.epoch == CONFIGS[name][3]
    train_rows = g["rows"][(g["epoch"] == last.epoch) & g["is_train"]]
    got = last.performance[ns.Split.TRAIN].losses
    for j, loss_name in enumerate(worker.criterion.loss_names):
        assert got[loss_name] == pytest.approx(train_rows[:, 1 + j].mean(), rel=1e-5)
    for suffix in ("", ".model", ".test_data", ".annotate_param"):
        assert os.path.exists(os.path.join(save_dir, "final_model.pth" + suffix))
    whole = torch.load(os.path.join(save_dir, "final_model.pth.model"), weights_only=False)
    assert all(p.dtype == torch.float32 and p.device.type == "cpu" for p in whole.parameters())


def test_first_step_gradients_match_reference(ns, golden_dir):
    g = np.load(os.path.join(golden_dir, "toy_sgd.npz"))
    cfg = CONFIGS["toy_sgd"]
    save_dir = tempfile.mkdtemp(prefix="frl_b200_test_")
    torch.manual_seed(SEED)
    problem = synthetic.make_toy_problem(ns, save_dir)
    args = SolverWorkerArgs(run_opts=_run_opts(ns, cfg), problem=problem, save_dir=save_dir,
                            run_device=Device.GPU, node_idx=0, node_count=1, rank=0, local_rank=0,
                            world_size=1, group_name=None, init_method="")
    worker, _, _ = Solver.build_worker(args)
    ds = problem.datasets[0]
    batch = torch.utils.data.default_collate([ds[int(i)] for i in g["served_train"][:BATCH]])
    data = [t.cuda() for t in batch[0]]
    target = [tuple(t.cuda() for t in head) for head in batch[1]]
    worker.model.train()
    worker._pass_one_minibatch(0, ns.Split.TRAIN, data, target)
    torch.cuda.synchronize()
    # parameter order (ArenaSlot.index), not arena order: the task heads' weights are laid out
    # back to back (ParamArena(adjacent=...)) so the heads can run as one backward unit
    for i, s in enumerate(sorted((s for s in worker.arena.slots if s.is_model), key=lambda s: s.index)):
        got = worker.arena.grad_view(s).cpu().numpy()
        np.testing.assert_allclose(got, g["grad_%02d" % i], rtol=1e-5, atol=1e-7)


def test_resume_from_checkpoint_continues_identically(ns, golden_dir):
    """Stop after epoch 5 of 6 (checkpoint cadence), resume, and land on the same weights."""
    cfg = ("sgd", 0.01, "drop", 6, 0.0, False, "parallel")
    _, worker_full, _, dir_full = _solve_and_capture(ns, cfg)
    save_dir = tempfile.mkdtemp(prefix="frl_b200_test_")
    problem = synthetic.make_toy_problem(ns, save_dir)
    torch.manual_seed(SEED)
    gen = Solver.solve(_run_opts(ns, cfg), problem, group_name=None, init_method="file:///tmp/unused")
    for summary in gen:
        if summary.epoch == 5:
            break
    gen.close()
    assert os.path.exists(os.path.join(save_dir, ".checkpoint.pth"))
    ckpt = torch.load(os.path.join(save_dir, ".checkpoint.pth"), weights_only=False)
    assert ckpt["epoch"] == 5 and "momentum_buffer" in ckpt["optimizer"]["state"][0]
    problem2 = synthetic.make_toy_problem(ns, save_dir)
    rest = list(Solver.solve(_run_opts(ns, cfg), problem2, group_name=None, init_method="file:///tmp/unused"))
    assert [s.epoch for s in rest] == [6]
    # data order after a resume differs (global RNG), so compare against a stock torch.optim
    # continuation from the same checkpoint instead: the checkpoint must be loadable there
    ref_model = problem2.get_model()
    ref_model.load_state_dict(ckpt["state_dict"])
    ref_opt = torch.optim.SGD(ref_model.parameters(), lr=0.01, momentum=0.9, weight_decay=1e-5)
    ref_opt.load_state_dict(ckpt["optimizer"])
    assert ref_opt.state_dict()["state"][0]["momentum_buffer"].shape == ckpt["optimizer"]["state"][0]["momentum_buffer"].shape


def test_nan_loss_raises_floating_point_error(ns):
    cfg = ("sgd", 1e30, "drop", 1, 0.0, False, "parallel")       # diverges to NaN within a few steps
    with pytest.raises(FloatingPointError, match="Losses become NaN for dataset training at iteration 1"):
        _solve_and_capture(ns, cfg)


def test_bf16_mode_tracks_fp32_reference_within_tolerance(ns, golden_dir):
    g = np.load(os.path.join(golden_dir, "toy_sgd.npz"))
    _, worker, _, _ = _solve_and_capture(ns, CONFIGS["toy_sgd"], precision=Precision.BF16)
    rows = np.concatenate([r for _, _, r in worker.loss_history])
    np.testing.assert_allclose(rows, g["rows"], rtol=1e-2, atol=1e-3)
    assert worker.arena.lp is not None and worker.arena.grad.dtype == torch.bfloat16
    assert all(p.dtype == torch.bfloat16 for p in worker.model.parameters())


def test_multiprocess_entry_point_with_pipes(tmp_path):
    """Solver.solve in its default mode: one forked process per GPU, results over a pipe."""
    import subprocess
    import sys
    script = os.path.join(os.path.dirname(__file__), "run_solver_mp.py")
    out = subprocess.run([sys.executable, script, str(tmp_path)], capture_output=True, text=True,
                         timeout=600)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
    assert "MP_SOLVE_OK" in out.stdout


def test_multi_gpu_pipeline_matches_oracle(tmp_path):
    """>= 2 GPUs only: real kernels + NCCL bucket all-reduce vs the CPU oracle on the global batch."""
    import subprocess
    import sys
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs 2 GPUs")
    script = os.path.join(os.path.dirname(__file__), "run_ddp_vs_oracle.py")
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1",
                          "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port",
                          "29533", script], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
    assert out.stdout.count("DDP_PARITY_OK") == (8 if "NVLS_AVAILABLE True" in out.stdout else 4)


@pytest.mark.parametrize("name", ["toy_sgd", "toy_adam_clip", "toy_uncertainty"])
def test_cuda_graph_replay_matches_reference_solver(ns, golden_dir, name, monkeypatch):
    """Same parity bar with the step replayed from a CUDA graph (captured after 2 eager steps)."""
    monkeypatch.setenv("FRL_B200_CUDA_GRAPH", "1")
    g = np.load(os.path.join(golden_dir, name + ".npz"))
    _, worker, problem, save_dir = _solve_and_capture(ns, CONFIGS[name])
    assert worker.graphed is not None and len(worker.graphed._graphs) == 1
    rows = np.concatenate([r for _, _, r in worker.loss_history])
    np.testing.assert_allclose(rows, g["rows"], rtol=1e-5, atol=1e-6)
    final = torch.load(os.path.join(save_dir, "final_model.pth"), weights_only=False)
    for i, k in enumerate(list(g["param_names"])):
        np.testing.assert_allclose(final["state_dict"][k].numpy(), g["param_%02d" % i],
                                   rtol=2e-4, atol=2e-6)


@pytest.mark.parametrize("path", ["host", "tma", "kernel"])
def test_device_batch_loader_path_matches_reference_solver(ns, golden_dir, monkeypatch, path):
    """Same Problem with its dataset in pinned host memory: the loop uses DeviceBatchLoader
    (native host gather + DMA, or GPU-side row gather, + device transform) instead of per-sample
    __getitem__/collate.  Sample order and arithmetic must not change: per-step losses still
    match the reference run."""
    import frl_b200.synthetic as syn
    monkeypatch.setenv("FRL_B200_INPUT_PATH", path)
    g = np.load(os.path.join(golden_dir, "toy_sgd.npz"))
    orig = syn.make_toy_problem
    monkeypatch.setattr(syn, "make_toy_problem",
                        lambda ns_, save_dir, **kw: orig(ns_, save_dir, pinned=True, **kw))
    # depth 2 < metricAmortizationSchedule: retained targets must survive slot recycling
    summaries, worker, problem, _ = _solve_and_capture(ns, CONFIGS["toy_sgd"], metricAmortizationSchedule=5)
    assert problem.datasets[0].served == []            # the per-sample path was never used
    rows = np.concatenate([r for _, _, r in worker.loss_history])
    np.testing.assert_allclose(rows, g["rows"], rtol=1e-5, atol=1e-6)
    # the amortised per-sample metrics (Problem.compute_batch_metrics on retained batches) equal
    # those of the per-sample DataLoader path
    monkeypatch.setattr(syn, "make_toy_problem", orig)
    plain, _, _, _ = _solve_and_capture(ns, CONFIGS["toy_sgd"], metricAmortizationSchedule=5)
    for split in (ns.Split.TRAIN, ns.Split.TEST):
        want = plain[-1].performance[split].metrics
        got = summaries[-1].performance[split].metrics
        assert set(got) == set(want) and len(want) >= 2
        for k in want:
            assert got[k] == pytest.approx(want[k], rel=1e-5, abs=1e-7), (split, k)


def test_indexed_files_feed_the_loop_through_the_host_pool(ns, golden_dir, monkeypatch, tmp_path):
    """The toy Problem's datasets written as .idx/.bin files (this repo's writer,
    byte-identical to the reference's) and served from the memory-mapped files — the host gather
    pool copies each minibatch's frames from the page cache into pinned staging, one DMA per field,
    transform on the device.  Same samples in the same order => the golden per-step losses."""
    import frl_b200.synthetic as syn
    g = np.load(os.path.join(golden_dir, "toy_sgd.npz"))
    orig = syn.make_toy_problem
    monkeypatch.setattr(syn, "make_toy_problem",
                        lambda ns_, save_dir, **kw: orig(ns_, save_dir, indexed_dir=str(tmp_path), **kw))
    summaries, worker, problem, _ = _solve_and_capture(ns, CONFIGS["toy_sgd"])
    assert sorted(os.listdir(tmp_path / "training")) == ["x.bin", "x.idx", "y_cls.bin", "y_cls.idx",
                                                          "y_reg.bin", "y_reg.idx"]
    assert not any(t.is_pinned() for t in problem.datasets[0].pinned_fields.values())
    rows = np.concatenate([r for _, _, r in worker.loss_history])
    np.testing.assert_allclose(rows, g["rows"], rtol=1e-5, atol=1e-6)
    # and the per-sample protocol over the same files equals the in-memory dataset's
    plain = orig(ns, "/tmp/unused")
    for i in (0, 17, 511):
        a, b = problem.datasets[0][i], plain.datasets[0][i]
        assert torch.equal(a[0][0], b[0][0]) and torch.equal(a[1][0][0], b[1][0][0])
        assert torch.equal(a[1][1][0], b[1][1][0]) and int(a[2]["index"]) == int(b[2]["index"]) == i


def test_bf16_wire_format_of_the_host_input_path(ns, golden_dir, monkeypatch):
    """FRL_B200_INPUT_WIRE=bf16: in a bf16-compute run the host gather threads round the model
    inputs to bf16 (bit-identical to the device cast) so PCIe carries half the bytes; targets stay
    exact.  The run stays within the bf16 bound of the fp32 reference, and the wire dtype is
    really used."""
    import frl_b200.synthetic as syn
    from frl_b200 import device_loader
    g = np.load(os.path.join(golden_dir, "toy_sgd.npz"))
    orig = syn.make_toy_problem
    monkeypatch.setattr(syn, "make_toy_problem",
                        lambda ns_, save_dir, **kw: orig(ns_, save_dir, pinned=True, **kw))
    monkeypatch.setenv("FRL_B200_INPUT_PATH", "host")
    monkeypatch.setenv("FRL_B200_INPUT_WIRE", "bf16")
    seen = []
    real_init = device_loader.DeviceBatchLoader.__init__

    def spy(self, *a, **kw):
        real_init(self, *a, **kw)
        seen.append(dict(self._wire_dtype))

    monkeypatch.setattr(device_loader.DeviceBatchLoader, "__init__", spy)
    _, worker, problem, _ = _solve_and_capture(ns, CONFIGS["toy_sgd"], precision=Precision.BF16)
    assert seen and all(w["x"] == torch.bfloat16 and w["y_reg"] == torch.float32
                        and w["y_cls"] == torch.int64 for w in seen)
    rows = np.concatenate([r for _, _, r in worker.loss_history])
    np.testing.assert_allclose(rows, g["rows"], rtol=1e-2, atol=1e-3)
    # fp32 runs ignore the switch: parity mode never rounds its inputs
    seen.clear()
    _, worker, _, _ = _solve_and_capture(ns, CONFIGS["toy_sgd"])
    assert seen and all(w["x"] == torch.float32 for w in seen)
    rows = np.concatenate([r for _, _, r in worker.loss_history])
    np.testing.assert_allclose(rows, g["rows"], rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("path", ["host", "kernel", "tma"])
def test_batched_input_path_with_a_ragged_last_batch(ns, monkeypatch, path):
    """512 and 128 samples at batch 48: the last minibatch of every split is short.  The batched
    path must serve exactly what the per-sample DataLoader path serves (same solver underneath):
    identical per-step losses, sample counts and amortised metrics."""
    import frl_b200.synthetic as syn
    cfg = CONFIGS["toy_sgd"]
    plain, w_plain, _, _ = _solve_and_capture(ns, cfg, batchSize=48, nEpochs=1, metricAmortizationSchedule=3)
    orig = syn.make_toy_problem
    monkeypatch.setattr(syn, "make_toy_problem",
                        lambda ns_, save_dir, **kw: orig(ns_, save_dir, pinned=True, **kw))
    monkeypatch.setenv("FRL_B200_INPUT_PATH", path)
    fast, w_fast, problem, _ = _solve_and_capture(ns, cfg, batchSize=48, nEpochs=1, metricAmortizationSchedule=3)
    assert problem.datasets[0].served == []
    a = np.concatenate([r for _, _, r in w_plain.loss_history])
    b = np.concatenate([r for _, _, r in w_fast.loss_history])
    assert a.shape == b.shape == (11 + 3, 3)
    np.testing.assert_allclose(b, a, rtol=1e-6, atol=1e-7)
    for split in (ns.Split.TRAIN, ns.Split.TEST):
        pa, pb = plain[-1].performance[split], fast[-1].performance[split]
        assert set(pa.metrics) == set(pb.metrics) and len(pa.metrics) >= 2
        for k in pa.metrics:
            assert pb.metrics[k] == pytest.approx(pa.metrics[k], rel=1e-6, abs=1e-8)


@pytest.mark.parametrize("graph", ["0", "1"])
def test_fused_linear_relu_units_keep_reference_parity(ns, golden_dir, monkeypatch, graph):
    """FRL_B200_FUSE_RELU=1 (the default): the toy trunk's two Linear+ReLU pairs run as cuBLASLt bias+ReLU
    GEMMs with dReLU folded into the bias-gradient pass; same parity bar against the reference
    run, eager and under CUDA-graph replay, and the checkpointed module is a plain one."""
    monkeypatch.setenv("FRL_B200_FUSE_RELU", "1")
    monkeypatch.setenv("FRL_B200_CUDA_GRAPH", graph)
    g = np.load(os.path.join(golden_dir, "toy_sgd.npz"))
    _, worker, problem, save_dir = _solve_and_capture(ns, CONFIGS["toy_sgd"])
    assert sum(s.relu is not None for s in worker.pipeline.linear_sites) == 2
    rows = np.concatenate([r for _, _, r in worker.loss_history])
    np.testing.assert_allclose(rows, g["rows"], rtol=1e-5, atol=1e-6)
    final = torch.load(os.path.join(save_dir, "final_model.pth"), weights_only=False)
    for i, k in enumerate(list(g["param_names"])):
        np.testing.assert_allclose(final["state_dict"][k].numpy(), g["param_%02d" % i], rtol=2e-4, atol=2e-6)
    whole = torch.load(os.path.join(save_dir, "final_model.pth.model"), weights_only=False)
    x = torch.rand(5, 64)
    with torch.no_grad():
        out = whole([x])                                   # pickled module: stock forward, ReLUs active
    assert all("forward" not in m.__dict__ for m in whole.modules())
    assert len(out) == 2 and out[0].shape == (5, 4)


@pytest.mark.parametrize("config", ["err_MSE_DESC", "score_ASC", "score_DESC"])
def test_device_side_sampler_state_matches_reference_fixture(golden_dir, config):
    """The Problem's hook returns DEVICE tensors; per-sample metrics stay in HBM
    columns, the worst-k set is a running device buffer merged with topk per window, everything is
    read back once at the end of the split.  Same fixtures as the numpy-returning hook: the reference's own
    SamplerState on the same scenario (oracle/make_sampler_state_golden.py)."""
    import json
    import random
    import frl_b200.solver_worker as sw
    from frl_b200.problem import Ordering
    from oracle import make_sampler_state_golden as gen
    want = json.load(open(os.path.join(golden_dir, "sampler_state.json")))[config]
    name, ordering = config.rsplit("_", 1)
    batches, total = gen.scenario()
    dev = torch.device("cuda", 0)
    cuda_batches = [dict(meta={k: v.to(dev) for k, v in b["meta"].items()},
                         data=[t.to(dev) for t in b["data"]],
                         outputs=[t.to(dev) for t in b["outputs"]],
                         targets=[tuple(t.to(dev) for t in h) for h in b["targets"]]) for b in batches]
    random.seed(gen.PY_SEED)
    mine = sw.SamplerState(gen.make_problem(Ordering, name, ordering, as_numpy=False), total, total, dev,
                           gen.N_VIS)
    gen.drive(mine, cuda_batches)
    assert mine.metrics_on_device and mine._runner is None        # no worker thread, no host read so far
    assert not mine.random_samples and not mine.worst_samples
    mine.finish()
    for k, v in want["metrics"].items():
        np.testing.assert_allclose(np.asarray(mine.data_metric[k], dtype=np.float64), np.asarray(v),
                                   rtol=1e-6, atol=1e-7)
    assert [int(s.meta["index"]) for s in mine.random_samples] == want["random_ids"]
    assert sorted(int(s.meta["index"]) for s in mine.worst_samples) == want["worst_ids"]
    # the captured samples are the scenario's rows, bit for bit
    rows = {int(i): (b["data"][0][j], b["outputs"][0][j], b["targets"][1][0][j])
            for b in batches for j, i in enumerate(b["meta"]["index"])}
    for s in mine.random_samples + mine.worst_samples:
        d, o, t = rows[int(s.meta["index"])]
        assert torch.equal(s.data[0], d) and torch.equal(s.output[0], o) and torch.equal(s.target[1][0], t)
        assert not s.data[0].is_cuda
