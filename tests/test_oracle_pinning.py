"""The oracle (oracle/ref_loop.py, optim_np.py, criteria_np.py) against the committed golden
vectors recorded from the live reference, against the reference itself (live where it is
present, else its recorded side under tests/golden/live), and against torch's own ops."""
import json
import os
import re

import numpy as np
import pytest
import torch

from oracle import criteria_np, optim_np, ref_loop
from oracle.live_golden import plain, reference_side, tensors_equal
from oracle.make_golden import BATCH, CONFIGS, SEED, run_oracle


def _golden_rows(golden_dir, name):
    return np.load(os.path.join(golden_dir, name + ".npz"), allow_pickle=False)


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_ref_loop_reproduces_reference_run(golden_dir, name):
    g = _golden_rows(golden_dir, name)
    trace, problem = run_oracle(name, CONFIGS[name])
    rows = np.concatenate([trace.losses[k] for k in sorted(
        trace.losses, key=lambda ek: (ek[0], 0 if ek[1] == "training" else 1))])
    # bit-exact on the machine that made the fixture; other CPUs may pick different SIMD paths
    np.testing.assert_allclose(rows, g["rows"], rtol=2e-6, atol=1e-7)
    served = sum((trace.indices[k] for k in sorted(trace.indices) if k[1] == "training"), [])
    assert served == list(g["served_train"])            # sample order: exact
    n_param = len([k for k in g.files if k.startswith("param_") and k != "param_names"])
    for i in range(n_param):
        np.testing.assert_allclose(trace.params[i], g["param_%02d" % i], rtol=2e-5, atol=2e-7)
    lrs = [lr for lr, e in zip(g["lr"], g["epoch"])]
    for lr, epoch in zip(lrs, g["epoch"]):
        assert lr == pytest.approx(trace.lrs[epoch - 1], rel=1e-12)


def test_lr_closed_forms_match_reference_tables(golden_dir):
    table = json.load(open(os.path.join(golden_dir, "lr_schedules.json")))
    for key, lrs in table.items():
        if key.startswith("kat_"):
            continue
        sched, n = key.split("_n")
        got = [ref_loop.lr_at_epoch(0.1, e, int(n), sched) for e in range(1, int(n) + 1)]
        assert got == pytest.approx(lrs, rel=1e-12)
    # the reference's own known-answer test (tests/test_solver.py:17-34)
    assert table["kat_resume60_adam_lr0.01_n75"] == [pytest.approx(0.001)]
    assert ref_loop.lr_at_epoch(0.01, 61, 75, "drop") == pytest.approx(0.001)


def test_sampler_restatement_matches_reference_lists(golden_dir):
    table = json.load(open(os.path.join(golden_dir, "samplers.json")))
    assert table["randperm_n10_w4_nodes1_e1"] == [[5, 0, 7], [6, 8, 4], [1, 9, 5], [2, 3, 6]]
    for key, per_rank in table.items():
        m = re.fullmatch(r"(\w+)_n(\d+)_w(\d+)_nodes(\d+)_e(\d+)", key)
        kind = m.group(1)
        n, w, nodes, e = (int(m.group(i)) for i in (2, 3, 4, 5))
        for rank, expect in enumerate(per_rank):
            node_size = w // nodes
            got = ref_loop.rank_indices(n, e, rank, w, kind, node_idx=rank // node_size,
                                        node_count=nodes)
            assert got == expect, key


def test_ref_loop_equals_live_reference_bitwise():
    name = "toy_sgd"

    def reference():
        from oracle.make_golden import run_live_reference
        run = run_live_reference(name, CONFIGS[name])
        return plain({"rows": run["rows"], "param_00": run["param_00"]})

    want, live = reference_side("ref_loop_" + name, reference)
    trace, _ = run_oracle(name, CONFIGS[name])
    rows = np.concatenate([trace.losses[k] for k in sorted(
        trace.losses, key=lambda ek: (ek[0], 0 if ek[1] == "training" else 1))])
    assert tensors_equal(plain(rows), want["rows"], live)
    assert tensors_equal(plain(trace.params[0]), want["param_00"], live)


# ---- numpy update rules vs torch.optim (what the reference actually calls) --------------------

def _torch_steps(opt_cls, kwargs, p0, grads):
    p = torch.nn.Parameter(torch.from_numpy(p0.copy()))
    opt = opt_cls([p], **kwargs)
    for g in grads:
        p.grad = torch.from_numpy(g.copy())
        opt.step()
    return p.detach().numpy()


def test_numpy_rules_match_torch_optim():
    rs = np.random.RandomState(3)
    p0 = rs.randn(257).astype(np.float32)
    grads = [rs.randn(257).astype(np.float32) for _ in range(5)]
    # SGD momentum
    want = _torch_steps(torch.optim.SGD, dict(lr=0.01, momentum=0.9, weight_decay=1e-5), p0, grads)
    p, buf = p0.copy(), np.zeros_like(p0)
    for i, g in enumerate(grads):
        p, buf = optim_np.sgd_step(p, g, buf, lr=0.01, mu=0.9, dampening=0.0, wd=1e-5,
                                   first_step=(i == 0))
    np.testing.assert_allclose(p, want, rtol=1e-6, atol=1e-7)
    # Adam (+amsgrad)
    for ams in (False, True):
        want = _torch_steps(torch.optim.Adam, dict(lr=1e-3, weight_decay=1e-5, eps=1e-8,
                                                   amsgrad=ams), p0, grads)
        p, m, v = p0.copy(), np.zeros_like(p0), np.zeros_like(p0)
        vmax = np.zeros_like(p0) if ams else None
        for i, g in enumerate(grads):
            p, m, v, vmax = optim_np.adam_step(p, g, m, v, vmax, lr=1e-3, beta1=0.9, beta2=0.999,
                                               eps=1e-8, wd=1e-5, step=i + 1)
        np.testing.assert_allclose(p, want, rtol=2e-6, atol=1e-7)
    # RMSprop with and without momentum
    for mu in (0.9, 0.0):
        want = _torch_steps(torch.optim.RMSprop, dict(lr=1e-3, momentum=mu, weight_decay=1e-5),
                            p0, grads)
        p, sq, buf = p0.copy(), np.zeros_like(p0), np.zeros_like(p0)
        for g in grads:
            p, sq, buf = optim_np.rmsprop_step(p, g, sq, buf, lr=1e-3, alpha=0.99, eps=1e-8,
                                               wd=1e-5, mu=mu)
        np.testing.assert_allclose(p, want, rtol=2e-6, atol=1e-7)


def test_numpy_criteria_match_torch_losses():
    rs = np.random.RandomState(5)
    out = rs.randn(33, 7).astype(np.float32)
    tgt = rs.randn(33, 7).astype(np.float32)
    lab = rs.randint(0, 7, size=33)
    lab[3] = -100
    to, tt, tl = (torch.tensor(out, requires_grad=True), torch.tensor(tgt), torch.tensor(lab))
    l = torch.nn.functional.mse_loss(to, tt)
    l.backward()
    loss, grad = criteria_np.mse(out, tgt)
    assert loss == pytest.approx(l.item(), rel=1e-6)
    np.testing.assert_allclose(grad, to.grad.numpy(), rtol=1e-5, atol=1e-8)
    to.grad = None
    l = torch.nn.functional.cross_entropy(to, tl)
    l.backward()
    loss, grad = criteria_np.cross_entropy(out, lab)
    assert loss == pytest.approx(l.item(), rel=1e-6)
    np.testing.assert_allclose(grad, to.grad.numpy(), rtol=1e-5, atol=1e-8)
    # masked variants against the reference's gather formulation
    mask = rs.rand(33) > 0.5
    ref = ref_loop.masked_loss(torch.nn.MSELoss(), torch.tensor(out), torch.tensor(tgt),
                               torch.tensor(mask))
    assert criteria_np.mse(out, tgt, mask)[0] == pytest.approx(ref.item(), rel=1e-6)
    empty = np.zeros(33, dtype=bool)
    ref0 = ref_loop.masked_loss(torch.nn.CrossEntropyLoss(), torch.tensor(out), torch.tensor(lab).clamp(min=0),
                                torch.tensor(empty))
    assert criteria_np.cross_entropy(out, lab, empty)[0] == pytest.approx(ref0.item(), rel=1e-6)
    assert criteria_np.mse(out, tgt, empty)[0] == 0.0


def test_bf16_round_matches_torch():
    x = np.random.RandomState(1).randn(4097).astype(np.float32) * 3
    want = torch.from_numpy(x).to(torch.bfloat16).to(torch.float32).numpy()
    assert np.array_equal(optim_np.bf16_round(x), want)


# ------------------------------------------------------------------------------------------------
# SamplerState (retained minibatches -> per-sample metrics, random picks, worst-k)
# against the live reference class on identical inputs
# ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("metric_name,ordering", [("err_MSE", "DESC"), ("score", "ASC"), ("score", "DESC")])
def test_sampler_state_matches_live_reference(metric_name, ordering):
    import random
    from typing import NamedTuple
    import frl_b200  # noqa: F401
    import frl_b200.solver_worker as my_sw
    from frl_b200.problem import Ordering as MyOrdering

    class Meta(NamedTuple):
        index: object = None

    def make_problem(Ordering):
        class P:
            def refine_batch_meta(self, meta):
                return Meta(**meta)

            def compute_batch_metrics(self, meta, target, output, device):
                err = ((output[0] - target[0][0]) ** 2).mean(1).numpy()
                score = (output[1][:, 0] - target[1][0].float()).numpy()      # signed, tie-free
                return {"err_MSE": err, "score": score}

            def get_rankable_metric(self):
                return metric_name, Ordering[ordering]
        return P()

    g = torch.Generator().manual_seed(11)
    sizes = [16, 16, 16, 16, 9]                       # ragged last minibatch
    batches, start = [], 0
    for n in sizes:
        batches.append(dict(
            meta={"index": torch.arange(start, start + n)},
            data=[torch.randn(n, 5, generator=g)],
            outputs=[torch.randn(n, 4, generator=g), torch.randn(n, 3, generator=g)],
            targets=[(torch.randn(n, 4, generator=g),), (torch.randint(0, 3, (n,), generator=g),)]))
        start += n
    total = start

    class FakeLoader:
        sampler = list(range(total))

    dev = torch.device("cpu")

    def feed(s):
        for k, b in enumerate(batches):
            if k % 2 == 0:                            # amortisation: fold every second minibatch
                s.compute_metrics()
            s.append_sample(b["meta"], b["data"], outputs=b["outputs"], targets=b["targets"])
        s.compute_metrics()
        return s

    def ids(samples):
        return [int(s.meta["index"]) for s in samples]

    def summary(s):
        return plain({"n_samples": s.n_samples,
                      "data_metric": {k: np.asarray(s.data_metric[k]) for k in ("err_MSE", "score")},
                      "random": ids(s.random_samples), "worst": ids(s.worst_samples),
                      "samples": {int(x.meta["index"]): {"data": list(x.data), "output": list(x.output),
                                                         "target": [t[0] for t in x.target],
                                                         "metric": {k: float(v) for k, v in x.metric.items()}}
                                  for x in s.worst_samples + s.random_samples}})

    def reference():
        from oracle.ref_shim import import_reference
        import_reference()
        import frldistml.scaffold.solver_worker as ref_sw
        from frldistml.scaffold.problem import Ordering as RefOrdering
        random.seed(5)
        return summary(feed(ref_sw.SamplerState(make_problem(RefOrdering), FakeLoader, list(range(total)), dev, 6)))

    ref, live = reference_side("sampler_state_%s_%s" % (metric_name, ordering), reference)
    random.seed(5)
    mine = feed(my_sw.SamplerState(make_problem(MyOrdering), total, total, dev, 6))
    mine.finish()
    mine = summary(mine)

    assert mine["n_samples"] == ref["n_samples"] == total
    for k in ("err_MSE", "score"):
        assert tensors_equal(mine["data_metric"][k], ref["data_metric"][k], live), k

    assert mine["random"] == ref["random"] and len(ref["random"]) == 6
    assert sorted(mine["worst"]) == sorted(ref["worst"])
    assert len(ref["worst"]) == 6
    for i, s in mine["samples"].items():
        r = ref["samples"][i]
        assert all(torch.equal(a, b) for a, b in zip(s["data"], r["data"]))
        assert all(torch.equal(a, b) for a, b in zip(s["output"], r["output"]))
        assert all(torch.equal(a, b) for a, b in zip(s["target"], r["target"]))
        assert s["metric"] == (r["metric"] if live else pytest.approx(r["metric"], rel=2e-6, abs=1e-7))


# ------------------------------------------------------------------------------------------------
# the criterion classes' own composition (what runs for arbitrary user losses,
# and what the fused kernels are checked against on the GPU) against the live reference classes
# ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kind", ["parallel", "uncertainty", "gradnorm", "masked"])
def test_criterion_classes_match_live_reference(kind):
    import frl_b200  # noqa: F401
    import frl_b200.criteria as my_c
    import frl_b200.model as my_m
    import frl_b200.types as my_t

    def build(c, m, t):
        torch.manual_seed(3)
        trunk = torch.nn.Sequential(m.ListSelect(sel_index=0, num_elements=1), torch.nn.Linear(6, 8),
                                    torch.nn.ReLU(), torch.nn.Linear(8, 8), torch.nn.ReLU())
        model = m.MultiTaskModel(trunk, [torch.nn.Linear(8, 3), torch.nn.Linear(8, 5)])
        mods = [torch.nn.MSELoss(), torch.nn.CrossEntropyLoss()]
        names, weights = ["reg", "cls"], [0.5, 2.0]
        if kind == "parallel":
            crit = c.ParallelCriterion(mods, weights, names)
        elif kind == "uncertainty":
            crit = c.UncertaintyWeightedCriterion(
                mods, [t.LossType.MSE, t.LossType.CrossEntropy], names, weights)
        elif kind == "gradnorm":
            crit = c.GradNormWeightedCriterion(mods, names, alpha=1.5, base_weights=weights)
        else:
            crit = c.ParallelCriterion([c.MaskedLoss(torch.nn.MSELoss()), torch.nn.CrossEntropyLoss()],
                                       weights, names)
        return model, crit

    g = torch.Generator().manual_seed(4)
    steps = []
    for k in range(4):
        x = torch.randn(12, 6, generator=g)
        y_reg, y_cls = torch.randn(12, 3, generator=g), torch.randint(0, 5, (12,), generator=g)
        mask = (torch.rand(12, 3, generator=g) > 0.4) if k != 2 else torch.zeros(12, 3, dtype=torch.bool)
        steps.append((x, y_reg, y_cls, mask))

    def run(c, m, t):
        model, crit = build(c, m, t)
        params = list(model.parameters()) + list(crit.parameters())
        opt = torch.optim.SGD(params, lr=0.05, momentum=0.9)
        trace = []
        for x, y_reg, y_cls, mask in steps:
            out = model([x])
            if kind == "gradnorm":
                crit.set_shared_params(model.final_shared_params(out))
            tgt = [(y_reg, mask) if kind == "masked" else (y_reg,), (y_cls,)]
            total, sub = crit(out, tgt)
            opt.zero_grad()
            total.backward()
            trace.append((total.detach().clone(), {k: v.detach().clone() for k, v in sub.items()},
                          [p.grad.detach().clone() for p in params]))
            opt.step()
        return trace, [p.detach().clone() for p in params]

    def reference():
        from oracle.ref_shim import import_reference
        import_reference()
        import frldistml.scaffold.criteria as ref_c
        import frldistml.scaffold.model as ref_m
        import frldistml.scaffold.types as ref_t
        return plain(run(ref_c, ref_m, ref_t))

    (ref_trace, ref_params), live = reference_side("criterion_" + kind, reference)
    my_trace, my_params = run(my_c, my_m, my_t)
    assert len(my_trace) == len(ref_trace) and len(my_params) == len(ref_params)
    for (rt, rs, rg), (mt, ms, mg) in zip(ref_trace, my_trace):
        assert tensors_equal(mt, rt, live)
        assert list(ms) == list(rs) and all(tensors_equal(ms[k], rs[k], live) for k in rs)
        assert len(mg) == len(rg) and all(tensors_equal(a, b, live) for a, b in zip(mg, rg))
    assert all(tensors_equal(a, b, live) for a, b in zip(my_params, ref_params))


# ------------------------------------------------------------------------------------------------
# parent-side aggregation of the per-rank epoch summaries (reference solver.py:457-526): sample-
# weighted means over ranks, MSE -> RMSE renaming, invalid (negative) metrics passed through
# ------------------------------------------------------------------------------------------------

def test_rank_aggregation_matches_live_reference():
    import frl_b200  # noqa: F401
    import frl_b200.solver as my_solver
    import frl_b200.solver_worker as my_sw
    import frl_b200.types as my_t

    per_rank = [   # (nSamples, losses, metrics) per split, three ranks with unequal sample counts
        {"training": (100, {"reg": 0.5, "cls": 2.25}, {"reg_MSE": 0.04, "cls_err": 0.25, "pose_MSE_deg": 9.0}),
         "testing": (10, {"reg": 0.7, "cls": 2.0}, {"reg_MSE": 0.09, "cls_err": 0.5, "pose_MSE_deg": -1.0})},
        {"training": (60, {"reg": 0.25, "cls": 1.75}, {"reg_MSE": 0.01, "cls_err": 0.125, "pose_MSE_deg": 4.0}),
         "testing": (30, {"reg": 0.1, "cls": 3.0}, {"reg_MSE": 0.16, "cls_err": 0.75, "pose_MSE_deg": -1.0})},
        {"training": (7, {"reg": 1.5, "cls": 0.5}, {"reg_MSE": 0.25, "cls_err": 1.0, "pose_MSE_deg": 1.0}),
         "testing": (3, {"reg": 0.3, "cls": 1.0}, {"reg_MSE": 0.0, "cls_err": 0.0, "pose_MSE_deg": -1.0})},
    ]

    def run(solver_mod, sw_mod, t):
        class DS:
            def __init__(self, split):
                self.data_type = split

        class P:
            datasets = [DS(t.Split.TRAIN), DS(t.Split.TEST)]

        fracs = []
        for rank in per_rank:
            perf = {t.Split(name): sw_mod.FractionalEpochSplitPerformanceSummary(
                        nSamples=n, losses=dict(losses), metrics=dict(metrics), samples=[],
                        worstSamples=[], testIO=[])
                    for name, (n, losses, metrics) in rank.items()}
            fracs.append(sw_mod.FractionalPerformanceSummary(
                epoch=3, modelBuffer=b"", optimizerStateBuffer=b"", performance=perf))
        ro = t.RunOpts(optim=t.OptimOpts(algo=t.OptAlgorithm.SGD), batchSize=4)
        out = solver_mod.Solver._aggregate_fractional_results(ro, P(), fracs)
        return {split.value: (dict(s.losses), dict(s.metrics)) for split, s in out.items()}

    def reference():
        from oracle.ref_shim import import_reference
        import_reference()
        import frldistml.scaffold.solver as ref_solver
        import frldistml.scaffold.solver_worker as ref_sw
        import frldistml.scaffold.types as ref_t
        return plain(run(ref_solver, ref_sw, ref_t))

    want, _ = reference_side("rank_aggregation", reference)
    got = plain(run(my_solver, my_sw, my_t))
    assert got == want
    assert set(want["training"][1]) == {"reg_RMSE", "cls_err", "pose_RMSE_deg"}
    assert want["testing"][1]["pose_RMSE_deg"] == -1.0          # invalid metric: not square-rooted


# ------------------------------------------------------------------------------------------------
# checkpoint files written by the parent (reference solver.py:565-651): same four files, same
# contents, and each side's loader reads the other's checkpoint
# ------------------------------------------------------------------------------------------------

def test_checkpoint_files_match_live_reference(tmp_path):
    import io
    from typing import NamedTuple
    import frl_b200  # noqa: F401
    import frl_b200.solver as my_solver
    import frl_b200.solver_worker as my_sw
    import frl_b200.types as my_t

    torch.manual_seed(1)
    model = torch.nn.Sequential(torch.nn.Linear(6, 5), torch.nn.BatchNorm1d(5), torch.nn.ReLU(),
                                torch.nn.Linear(5, 3))
    opt = torch.optim.SGD(model.parameters(), lr=0.1, momentum=0.9, weight_decay=1e-5)
    for _ in range(3):
        opt.zero_grad()
        model(torch.randn(8, 6)).square().mean().backward()
        opt.step()
    model.eval()
    buf = io.BytesIO()
    torch.save(model, buf)
    model_bytes = buf.getvalue()
    buf = io.BytesIO()
    torch.save(opt.state_dict(), buf)
    optim_bytes = buf.getvalue()
    samples = [dict(data=[torch.randn(6)], target=[(torch.randn(3),)], meta={"index": torch.tensor(i)},
                    output=[torch.randn(3)], metric={"m": 0.5}) for i in range(2)]

    class Anno(NamedTuple):
        scale: float = 2.0
        names: tuple = ("a", "b")

    class P:
        anno_param = Anno()

    def write(solver_mod, sw_mod, t, save_dir):
        io_samples = [sw_mod.SingleSample(**s) for s in samples]
        perf = {t.Split.TRAIN: sw_mod.FractionalEpochSplitPerformanceSummary(
                    nSamples=10, losses={}, metrics={}, samples=[], worstSamples=[], testIO=[]),
                t.Split.TEST: sw_mod.FractionalEpochSplitPerformanceSummary(
                    nSamples=4, losses={}, metrics={}, samples=[], worstSamples=[], testIO=io_samples)}
        frac = sw_mod.FractionalPerformanceSummary(epoch=7, modelBuffer=model_bytes,
                                                   optimizerStateBuffer=optim_bytes, performance=perf)
        ro = t.RunOpts(optim=t.OptimOpts(algo=t.OptAlgorithm.SGD), batchSize=4)
        solver_mod.Solver._save_checkpoint(7, save_dir, ro, P(), [frac], ".checkpoint.pth")

    ref_dir, my_dir = tmp_path / "ref", tmp_path / "mine"
    ref_dir.mkdir()
    my_dir.mkdir()

    def reference():
        from oracle.ref_shim import import_reference
        import_reference()
        import frldistml.scaffold.solver as ref_solver
        import frldistml.scaffold.solver_worker as ref_sw
        import frldistml.scaffold.types as ref_t
        from frldistml.scaffold.storage import StoragePath
        write(ref_solver, ref_sw, ref_t, StoragePath(str(ref_dir)))
        return {n: torch.frombuffer(bytearray(open(os.path.join(ref_dir, n), "rb").read()), dtype=torch.uint8)
                for n in sorted(os.listdir(ref_dir))}

    ref_files, live = reference_side("checkpoint_files", reference)
    if not live:
        for n, data in ref_files.items():
            open(os.path.join(ref_dir, n), "wb").write(data.numpy().tobytes())
    write(my_solver, my_sw, my_t, str(my_dir))
    names = sorted(os.listdir(ref_dir))
    assert sorted(os.listdir(my_dir)) == names == [".checkpoint.pth", ".checkpoint.pth.annotate_param",
                                                   ".checkpoint.pth.model", ".checkpoint.pth.test_data"]

    def same(a, b):
        if torch.is_tensor(a):
            return torch.is_tensor(b) and a.dtype == b.dtype and tensors_equal(a, b, live)
        if isinstance(a, dict):
            return isinstance(b, dict) and list(a) == list(b) and all(same(a[k], b[k]) for k in a)
        if isinstance(a, (list, tuple)):
            return type(a) is type(b) and len(a) == len(b) and all(same(x, y) for x, y in zip(a, b))
        return a == b

    for n in (".checkpoint.pth", ".checkpoint.pth.test_data", ".checkpoint.pth.annotate_param"):
        a = torch.load(os.path.join(ref_dir, n), weights_only=False)
        b = torch.load(os.path.join(my_dir, n), weights_only=False)
        assert same(a, b), n
    whole_ref = torch.load(os.path.join(ref_dir, ".checkpoint.pth.model"), weights_only=False)
    whole_mine = torch.load(os.path.join(my_dir, ".checkpoint.pth.model"), weights_only=False)
    assert same(dict(whole_ref.state_dict()), dict(whole_mine.state_dict()))
    # each loader reads the other side's file (the reference's loader where it is present)
    with open(os.path.join(ref_dir, ".checkpoint.pth"), "rb") as f:
        back = my_solver.Solver._load_checkpoint(f)
    got = back
    if live:
        import frldistml.scaffold.solver as ref_solver
        with open(os.path.join(my_dir, ".checkpoint.pth"), "rb") as f:
            got = ref_solver.Solver._load_checkpoint(f)
    assert got.epoch == back.epoch == 7
    assert same(dict(got.modelState), dict(back.modelState)) and same(got.optimizerState, back.optimizerState)
    torch.optim.SGD(whole_mine.parameters(), lr=0.1, momentum=0.9).load_state_dict(got.optimizerState)


def test_initial_model_loading_matches_live_reference(tmp_path, capsys):
    """``initialModelPath`` (reference solver.py:122-159): strict load, and the partial load that
    copies what matches in name and shape and reports the rest — same weights, same messages."""
    import frl_b200  # noqa: F401
    import frl_b200.solver as my_solver

    def net(width):
        torch.manual_seed(width)
        return torch.nn.Sequential(torch.nn.Linear(4, width), torch.nn.ReLU(), torch.nn.Linear(width, 2))

    donor = net(5)
    state = dict(donor.state_dict())
    state["extra.weight"] = torch.ones(3)
    state["0.weight"] = torch.nn.Parameter(state["0.weight"].clone())      # legacy serialised Parameter
    path = str(tmp_path / "init.pth")
    torch.save({"state_dict": state}, path)

    def load_with(mod):
        target = net(5)
        del_key = net(7)                       # different width: shape mismatches on every tensor but one
        mod._load_model_state(target, path, strict=False)
        mod._load_model_state(del_key, path, strict=False)
        out = capsys.readouterr().out
        lines = [l for l in out.splitlines() if l.startswith("Warning")]
        with pytest.raises(RuntimeError):
            mod._load_model_state(net(5), path, strict=True)               # unexpected key "extra.weight"
        capsys.readouterr()
        return plain((dict(target.state_dict()), dict(del_key.state_dict()), lines))

    def reference():
        from oracle.ref_shim import import_reference
        import_reference()
        import frldistml.scaffold.solver as ref_solver
        return load_with(ref_solver)

    (ra, rb, rl), live = reference_side("initial_model_loading", reference)
    ma, mb, ml = load_with(my_solver)
    assert list(ra) == list(ma) and list(rb) == list(mb)
    assert all(tensors_equal(ra[k], ma[k], live) for k in ra) and all(tensors_equal(rb[k], mb[k], live) for k in rb)
    assert ml == rl and len(rl) >= 4
    assert torch.equal(ma["0.weight"], donor.state_dict()["0.weight"])


def test_multitask_problem_plumbing_matches_live_reference():
    """The same synthetic MultiTaskProblem source instantiated against this package and against
    the reference (Problem/MultiTaskProblem/MultiTaskTransform/Task/MultiTaskModel):
    per-sample items, model structure and initial weights, criterion composition, merged metric
    hooks and rankable metric must coincide."""
    import frl_b200  # noqa: F401
    from frl_b200 import synthetic

    def build(pkg):
        ns = synthetic.api_namespace(pkg)
        problem = synthetic.make_toy_problem(ns, "/tmp/unused")
        torch.manual_seed(21)
        model = problem.get_model()
        crit = problem.get_criterion()
        items = [problem.datasets[0][i] for i in (0, 5, 511)] + [problem.datasets[1][3]]
        g = torch.Generator().manual_seed(2)
        out = [torch.randn(6, 4, generator=g), torch.randn(6, 10, generator=g)]
        tgt = [(torch.randn(6, 4, generator=g),), (torch.randint(0, 10, (6,), generator=g),)]
        meta = problem.refine_batch_meta({"index": torch.arange(6)})
        metrics = problem.compute_batch_metrics(meta=meta, target=tgt, output=out, device=torch.device("cpu"))
        with torch.no_grad():
            y = model([torch.ones(2, 64)])
        return plain(dict(
            model_type=type(model).__name__, crit_type=type(crit).__name__,
            state={k: v.clone() for k, v in model.state_dict().items()},
            names=list(crit.loss_names), weights=[float(w) for w in crit.loss_weights],
            loss_mods=[type(m).__name__ for m in crit.loss_modules], items=items,
            metrics={k: np.asarray(v) for k, v in metrics.items()},
            rank=(problem.get_rankable_metric()[0], problem.get_rankable_metric()[1].name),
            epoch=problem.summarize_epoch_metrics({k: np.asarray(v) for k, v in metrics.items()}),
            meta_fields=meta._fields, y=[t.clone() for t in y],
            splits=[d.data_type.value for d in problem.datasets], lens=[len(d) for d in problem.datasets]))

    def reference():
        from oracle.ref_shim import import_reference
        import_reference()
        return build("frldistml.scaffold")

    ref, live = reference_side("multitask_problem_plumbing", reference)
    mine = build("frl_b200")
    for k in ("model_type", "crit_type", "names", "weights", "loss_mods", "rank", "epoch", "meta_fields",
              "splits", "lens"):
        assert mine[k] == ref[k], k
    assert list(mine["state"]) == list(ref["state"])
    assert all(tensors_equal(mine["state"][k], ref["state"][k], live) for k in ref["state"])
    assert len(mine["y"]) == len(ref["y"]) and all(tensors_equal(a, b, live) for a, b in zip(mine["y"], ref["y"]))
    assert list(mine["metrics"]) == list(ref["metrics"])
    assert all(tensors_equal(mine["metrics"][k], ref["metrics"][k], live) for k in ref["metrics"])
    for a, b in zip(mine["items"], ref["items"]):
        assert len(a) == len(b) == 3
        assert all(torch.equal(x, y) for x, y in zip(a[0], b[0]))                      # data list
        assert all(torch.equal(x[0], y[0]) for x, y in zip(a[1], b[1]))                # target tuples
        assert list(a[2]) == list(b[2]) and all(torch.equal(torch.as_tensor(a[2][k]), torch.as_tensor(b[2][k]))
                                                 for k in a[2])
