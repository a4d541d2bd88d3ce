"""K13 on the H100: the data-gradient GEMM with the lower unit's ReLU backward and bias gradient in
its epilogue (``frl_dx_gemm_drelu``).

* dZ against float64: where act > 0 (or NaN), |dZ - P| <= K 2^-24 (|dZ_up| |W|) + 2^-8 |P| for the
  float64 product P -- the first term bounds any fp32 summation order over K terms, the second the
  single bf16 rounding (half an ulp, 2^-9 relative, doubled for the fp32 error it is applied to);
  where act <= 0, dZ is +0 exactly.
* db against the float64 column sum S of K13's own dZ: |db - S| <= B 2^-24 sum_r |dZ| + 2^-8 |S|
  (an fp32 sum of B terms in any order, then one bf16 rounding).
* against cuBLAS + K6b at 4096^3: every dZ element within one bf16 ulp of the product.
* NaN/inf, the accumulate flag, byte-identical launches, graph replay, refused shapes.
* wiring: the bench-shape MLP with FRL_B200_FUSED_DRELU_DX 1 against 0, and FP32 / FP8 runs, which
  K13 does not serve, bit-identical with the switch on and off.
"""
import tempfile

import pytest
import torch

import frl_b200  # noqa: F401
from frl_b200 import _native, synthetic
from frl_b200.solver import Solver, SolverWorkerArgs
from frl_b200.types import Device, Precision

pytestmark = pytest.mark.gpu


def _operands(rows, k, cols, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    dz_up = (torch.randn(rows, k, device="cuda", generator=g) / 8).to(torch.bfloat16)
    w = (torch.randn(k, cols, device="cuda", generator=g) / 8).to(torch.bfloat16)
    act = torch.randn(rows, cols, device="cuda", generator=g).relu().to(torch.bfloat16)
    return dz_up, w, act


def _run(dz_up, w, act, db=None, accumulate=False):
    dz = torch.full_like(act, float("nan"))
    db = torch.full((act.shape[1],), float("nan"), device="cuda", dtype=torch.bfloat16) if db is None else db
    _native.dx_gemm_drelu(dz_up, w, act, dz, db, accumulate=accumulate)
    return dz, db


def _check_db(dz, db, base=None):
    s = dz.double().sum(0) + (0 if base is None else base.double())
    bound = dz.shape[0] * 2.0 ** -24 * dz.double().abs().sum(0) + 2.0 ** -8 * s.abs()
    assert ((db.double() - s).abs() <= bound).all()


@pytest.mark.parametrize("rows,k,cols", [(4096, 4096, 4096), (4096, 1064, 4096), (256, 72, 512)])
def test_dz_and_db_against_float64(rows, k, cols):
    dz_up, w, act = _operands(rows, k, cols)
    dz, db = _run(dz_up, w, act)
    p = dz_up.double() @ w.double()
    bound = k * 2.0 ** -24 * (dz_up.double().abs() @ w.double().abs()) + 2.0 ** -8 * p.abs()
    keep = act > 0
    assert ((dz.double() - p).abs() <= bound)[keep].all()
    assert (dz[~keep].view(torch.int16) == 0).all()
    _check_db(dz, db)


def test_against_cublas_and_k6b():
    dz_up, w, act = _operands(4096, 4096, 4096, seed=3)
    dz, db = _run(dz_up, w, act)
    prod = torch.mm(dz_up, w)
    ref = torch.empty_like(prod)
    db_ref = torch.empty_like(db)
    _native.drelu_colsum(prod, act, ref, db_ref)
    diff = dz != ref
    frac = diff.double().mean().item()
    print("K13 vs cuBLAS + K6b: %.4f %% of dZ elements differ" % (100 * frac))
    mag = torch.maximum(dz.float().abs(), ref.float().abs())
    ulp = torch.where(mag > 0, torch.exp2(torch.floor(torch.log2(mag)) - 7), torch.zeros_like(mag))
    assert ((dz.float() - ref.float()).abs() <= ulp)[diff].all()
    torch.testing.assert_close(db.float(), db_ref.float(), rtol=2e-2, atol=2e-2 * db_ref.float().abs().max().item())


def test_nan_inf_follow_threshold_backward():
    rows, k, cols = 128, 72, 256
    dz_up, w, act = _operands(rows, k, cols, seed=5)
    act[0, :5] = torch.tensor([float("nan"), float("inf"), -float("inf"), 0.0, -0.0], dtype=torch.bfloat16)
    dz_up[7, 3] = float("nan")          # row 7 of the product NaN
    w[11, 20] = float("inf")            # column 20 of the product +-inf (or NaN)
    act[7, :8] = torch.tensor([1, -1, 0, float("nan"), 2, -0.0, 3, -2], dtype=torch.bfloat16)
    dz, _ = _run(dz_up, w, act)
    want = torch.ops.aten.threshold_backward((dz_up.double() @ w.double()).float().to(torch.bfloat16), act, 0)
    assert torch.equal(dz.isnan(), want.isnan())
    assert torch.equal(dz.isinf(), want.isinf())
    assert torch.equal(dz[dz.isinf()], want[want.isinf()])
    assert torch.isnan(dz[7, 0]) and torch.isnan(dz[7, 3]) and dz[7, 1] == 0 and dz[7, 2] == 0
    assert torch.isfinite(dz[0, 0]) and dz[0, 2] == 0 and dz[0, 3] == 0 and dz[0, 4] == 0
    fin = want.isfinite()
    torch.testing.assert_close(dz[fin].float(), want[fin].float(), rtol=2 ** -7, atol=1e-3)


def test_accumulate_flag():
    dz_up, w, act = _operands(512, 256, 512, seed=7)
    dz, db = _run(dz_up, w, act)
    _, db0 = _run(dz_up, w, act, db=torch.zeros_like(db), accumulate=True)
    assert torch.equal(db0, db)                                # 0 + s == s
    base = torch.randn(512, device="cuda").to(torch.bfloat16)
    _, db1 = _run(dz_up, w, act, db=base.clone(), accumulate=True)
    _check_db(dz, db1, base)


def test_repeated_launches_and_graph_replay_are_byte_identical():
    dz_up, w, act = _operands(1024, 1064, 1024, seed=9)
    dz_a, db_a = _run(dz_up, w, act)
    dz_b, db_b = _run(dz_up, w, act)
    assert torch.equal(dz_a.view(torch.int16), dz_b.view(torch.int16))
    assert torch.equal(db_a.view(torch.int16), db_b.view(torch.int16))
    dz = torch.empty_like(act)
    db = torch.empty_like(db_a)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s), torch.cuda.graph(graph, stream=s):
        _native.dx_gemm_drelu(dz_up, w, act, dz, db, accumulate=False)
    torch.cuda.current_stream().wait_stream(s)
    for _ in range(3):
        dz.zero_()
        db.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(dz.view(torch.int16), dz_a.view(torch.int16))
        assert torch.equal(db.view(torch.int16), db_a.view(torch.int16))


@pytest.mark.parametrize("rows,k,cols", [(100, 64, 256), (128, 64, 200), (128, 70, 256)])
def test_shapes_off_the_tile_are_refused(rows, k, cols):
    dz_up = torch.zeros(rows, k, device="cuda", dtype=torch.bfloat16)
    w = torch.zeros(k, cols, device="cuda", dtype=torch.bfloat16)
    act = torch.zeros(rows, cols, device="cuda", dtype=torch.bfloat16)
    db = torch.zeros(cols, device="cuda", dtype=torch.bfloat16)
    assert not _native.dx_drelu_fits(dz_up, w, act, db)
    with pytest.raises(_native.NativeLibraryError):
        _native.dx_gemm_drelu(dz_up, w, act, torch.empty_like(act), db)


# ---- wiring -------------------------------------------------------------------------------------

def _mlp_run(monkeypatch, fused, precision=Precision.BF16, width=4096, batch=4096, steps=5):
    monkeypatch.setenv("FRL_B200_FUSED_DRELU_DX", fused)
    ns = synthetic.api_namespace("frl_b200")
    t = ns.types
    save_dir = tempfile.mkdtemp(prefix="frl_b200_dx_")
    torch.manual_seed(0)
    problem = synthetic.make_mlp_problem(ns, save_dir, n_train=8, width=width, n_classes=1000, reg_dim=64, depth=3)
    run_opts = t.RunOpts(optim=t.OptimOpts(algo=t.OptAlgorithm.SGD, lr=0.01, momentum=0.9),
                         batchSize=batch, nEpochs=1, numThreads=0, singleThreaded=True, numVisualizedSamples=0)
    args = SolverWorkerArgs(run_opts=run_opts, problem=problem, save_dir=save_dir, run_device=Device.GPU,
                            node_idx=0, node_count=1, rank=0, local_rank=0, world_size=1, group_name=None,
                            init_method="", precision=precision)
    worker, _, _ = Solver.build_worker(args)
    worker.model.train()
    worker.criterion.train()
    g = torch.Generator().manual_seed(1234)
    losses = []
    for i in range(steps):
        x = torch.randn(batch, width, generator=g).cuda()
        y = torch.randint(0, 1000, (batch,), generator=g).cuda()
        r = torch.randn(batch, 64, generator=g).cuda()
        _, total, _, _ = worker._pass_one_minibatch(i, t.Split.TRAIN, [x], [(y,), (r,)])
        losses.append(float(total.detach()))
        del total
    torch.cuda.synchronize()
    return worker.pipeline, worker.arena.master.clone(), losses


def test_bench_shape_mlp_with_and_without_k13(monkeypatch):
    calls = []
    real = _native.dx_gemm_drelu
    monkeypatch.setattr(_native, "dx_gemm_drelu", lambda *a, **k: (calls.append(1), real(*a, **k))[1])
    pipe, w_on, l_on = _mlp_run(monkeypatch, "1")
    assert sum(s.consumer is not None for s in pipe.linear_sites) == 3
    assert pipe.fused_dw_update and len(pipe.dw_updated) == 3
    assert calls                                                   # eager steps before capture
    pipe0, w_off, l_off = _mlp_run(monkeypatch, "0")
    assert all(s.consumer is None for s in pipe0.linear_sites)
    torch.testing.assert_close(torch.tensor(l_on), torch.tensor(l_off), rtol=1e-2, atol=0)
    rel = (w_on - w_off).norm() / w_off.norm()
    assert rel < 1e-2, rel


@pytest.mark.parametrize("precision", [Precision.FP32, Precision.FP8], ids=["fp32", "fp8"])
def test_precisions_k13_does_not_serve_are_unchanged(monkeypatch, precision):
    _, w_on, l_on = _mlp_run(monkeypatch, "1", precision=precision, width=512, batch=256)
    _, w_off, l_off = _mlp_run(monkeypatch, "0", precision=precision, width=512, batch=256)
    assert l_on == l_off
    assert torch.equal(w_on, w_off)
