"""SamplerState folds every window the same way whatever the Problem's metric hook returns: the
shared scenario (oracle/make_sampler_state_golden.py), with a bf16 input field, a bf16 target, a
list meta field and a None meta field added, gives the same ``SingleSample``s — values, dtypes,
meta types and order — from a hook returning numpy arrays and from one returning tensors."""
import random
from typing import NamedTuple

import numpy as np
import pytest
import torch

import frl_b200.solver_worker as sw
from frl_b200.problem import Ordering
from oracle import make_sampler_state_golden as gen


class Meta(NamedTuple):
    index: object = None
    name: object = None
    missing: object = None


def extended_scenario():
    batches, total = gen.scenario()
    g = torch.Generator().manual_seed(12)
    for b in batches:
        n = len(b["meta"]["index"])
        b["meta"]["name"] = ["s%d" % i for i in b["meta"]["index"].tolist()]
        b["data"].append(torch.randn(n, 3, generator=g).to(torch.bfloat16))
        b["targets"][1] += (torch.randn(n, 2, generator=g).to(torch.bfloat16),)
    return batches, total


def make_problem(metric_name, ordering, as_numpy,
                 metrics=lambda meta, output, target: gen.metrics(output, target)):
    class P:
        def refine_batch_meta(self, meta):
            return Meta(**meta)

        def compute_batch_metrics(self, meta, target, output, device):
            m = metrics(meta, output, target)
            return {k: v.numpy() for k, v in m.items()} if as_numpy else m

        def get_rankable_metric(self):
            return metric_name, Ordering[ordering]
    return P()


def fold(problem, batches, total):
    random.seed(gen.PY_SEED)
    state = sw.SamplerState(problem, total, total, torch.device("cpu"), gen.N_VIS)
    gen.drive(state, batches)
    state.finish()
    return state


def assert_same_value(a, b):
    assert type(a) is type(b)
    if torch.is_tensor(a):
        assert a.dtype == b.dtype and a.shape == b.shape and torch.equal(a, b)
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b)
        for x, y in zip(a, b):
            assert_same_value(x, y)
    elif isinstance(a, np.generic):
        assert a.dtype == b.dtype and a == b
    else:
        assert a == b


def assert_same_samples(xs, ys):
    assert len(xs) == len(ys)
    for x, y in zip(xs, ys):
        for field in ("data", "target", "output"):
            assert_same_value(getattr(x, field), getattr(y, field))
        assert list(x.meta) == list(y.meta) == ["index", "name", "missing"]
        for k in x.meta:
            assert_same_value(x.meta[k], y.meta[k])
        assert list(x.metric) == list(y.metric)
        for k in x.metric:
            assert_same_value(x.metric[k], y.metric[k])


@pytest.mark.parametrize("config", ["err_MSE_DESC", "score_ASC", "score_DESC"])
def test_numpy_and_tensor_hooks_give_the_same_samples(config):
    name, ordering = config.rsplit("_", 1)
    batches, total = extended_scenario()
    host = fold(make_problem(name, ordering, as_numpy=True), batches, total)
    tens = fold(make_problem(name, ordering, as_numpy=False), batches, total)

    assert list(host.data_metric) == list(tens.data_metric)
    for k in host.data_metric:
        assert host.data_metric[k].dtype == tens.data_metric[k].dtype == np.float32
        np.testing.assert_array_equal(host.data_metric[k], tens.data_metric[k])
    assert len(host.random_samples) == gen.N_VIS and len(host.worst_samples) == gen.N_VIS
    assert_same_samples(host.random_samples, tens.random_samples)
    assert_same_samples(host.worst_samples, tens.worst_samples)

    rows = {int(i): (b["data"][1][j], b["targets"][1][1][j])
            for b in batches for j, i in enumerate(b["meta"]["index"])}
    for s in host.random_samples + host.worst_samples:
        i = int(s.meta["index"])
        assert s.meta["index"].dim() == 0 and s.meta["index"].dtype == torch.int64
        assert s.meta["name"] == "s%d" % i and s.meta["missing"] is None
        d, t = rows[i]
        assert s.data[1].dtype == torch.bfloat16 and torch.equal(s.data[1], d)
        assert s.target[1][1].dtype == torch.bfloat16 and torch.equal(s.target[1][1], t)
        assert s.output[0].dtype == torch.float32

    # ascending by rank score: the most extreme sample last
    rank = host.data_metric[name] * (-1 if ordering == "DESC" else 1)
    scores = [rank[int(s.meta["index"])] for s in host.worst_samples]
    assert scores == sorted(scores)


@pytest.mark.parametrize("as_numpy", [True, False])
def test_a_valid_metric_that_ranks_as_minus_inf_is_kept(as_numpy):
    """err_MSE ranks only non-negative values; DESC ranks +inf as -inf.  With fewer valid samples
    than the worst-k set holds, every valid one is kept — that one too — and no invalid one."""
    batches, total = extended_scenario()
    table = torch.full((total,), -1.0)                 # negative: invalid for an MSE metric
    table[3], table[40], table[70] = 0.5, float("inf"), 2.0

    def metrics(meta, output, target):
        return {"err_MSE": table[meta.index]}

    state = fold(make_problem("err_MSE", "DESC", as_numpy, metrics), batches, total)
    assert [int(s.meta["index"]) for s in state.worst_samples] == [40, 70, 3]
    assert np.isinf(state.worst_samples[0].metric["err_MSE"])
