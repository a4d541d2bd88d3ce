"""The Adafactor path catalogue (``adafactor_oracle.AF_PATHS``) on the host.

* Every branch in ``AF_BRANCHES`` is reached by some case, read off the library's own band table
  (``_native.adafactor_plan``); each case reaches the branches it is named for.
* On every case the band table covers each element of each tensor exactly once and places the
  partials where the kernels expect them.
* On every case the float64 restatement ``adafactor_step``, which the GPU tests of
  tests/test_gpu_adafactor_paths.py lean on for their preconditions, equals float64
  ``torch.optim.Adafactor`` (foreach=False).
"""
import numpy as np
import pytest
import torch

import frl_b200  # noqa: F401
from frl_b200 import _native
import adafactor_oracle as af
from adafactor_oracle import AF_BRANCHES, AF_PATHS

EPS1 = 2.0 ** -23


def _reached():
    out = {}
    for name, case in AF_PATHS.items():
        for b in af.case_branches(case):
            out.setdefault(b, []).append(name)
    return out


@pytest.mark.parametrize("branch", AF_BRANCHES)
def test_catalogue_reaches_branch(branch):
    reached = _reached()
    assert branch in reached, f"no case of AF_PATHS reaches branch {branch!r}"


@pytest.mark.parametrize("name", list(AF_PATHS))
def test_case_reaches_the_branches_it_is_named_for(name):
    case = AF_PATHS[name]
    assert set(case.reaches) <= set(AF_BRANCHES), name
    missing = set(case.reaches) - af.case_branches(case)
    assert not missing, f"{name} does not reach {sorted(missing)}"


@pytest.mark.parametrize("name", list(AF_PATHS))
def test_band_table_covers_each_element_once(name):
    shape = af.case_shape_tensor(AF_PATHS[name])
    work, seg_info = _native.adafactor_plan(shape)
    work, seg_info = work.numpy(), seg_info.numpy()
    assert seg_info[0, 0] == 0 and seg_info[-1, 1] == work.shape[0]
    assert (seg_info[1:, 0] == seg_info[:-1, 1]).all()
    part = 0
    for i, (B, R, C) in enumerate(shape.tolist()):
        bands = work[seg_info[i, 0]:seg_info[i, 1]]
        assert (bands[:, 0] == i).all()
        if R == 0:
            seen = np.zeros(C, dtype=np.int64)
            for _, _, e0, _ in bands:
                assert e0 % af.AF_CHUNK == 0
                seen[e0:e0 + af.AF_CHUNK] += 1
            assert (seen == 1).all(), (i, C)
            continue
        n_rb, n_cb = -(-R // af.AF_ROWS), -(-C // af.AF_COLS)
        seen = np.zeros((B, R, C), dtype=np.int64)
        for _, b, r0, c0 in bands:
            assert r0 % af.AF_ROWS == 0 and c0 % af.AF_COLS == 0
            seen[b, r0:r0 + af.AF_ROWS, c0:c0 + af.AF_COLS] += 1
        assert (seen == 1).all(), (i, B, R, C)
        assert bands.shape[0] == B * n_rb * n_cb
        assert seg_info[i, 2] == part                    # row sums, column sums, row means
        part += B * R * n_cb + B * n_rb * C + B
    n_segs = shape.shape[0]
    want = (4 * n_segs + 15) // 16 * 16 + 8 * (2 * work.shape[0] + 2 * n_segs + part)
    assert _native.adafactor_scratch_bytes(shape) == want


@pytest.mark.parametrize("name", list(AF_PATHS))
def test_restatement_equals_torch_adafactor_on_the_case(name):
    case = AF_PATHS[name]
    gen = torch.Generator().manual_seed(sum(map(ord, name)))
    params = [torch.nn.Parameter(torch.randn(s, generator=gen, dtype=torch.float64)) for s in case.shapes]
    ref = torch.optim.Adafactor(params, lr=1e-2, weight_decay=0.1, eps=(EPS1, 1e-3), foreach=False)
    ps = [p.detach().numpy().ravel().copy() for p in params]
    states = [af.zero_state(s) for s in case.shapes]
    for t in range(1, 3):
        for i, p in enumerate(params):
            if p.numel() == 0:                           # torch divides by numel: no gradient
                continue
            g = torch.randn(p.shape, generator=gen, dtype=torch.float64) * 10.0 ** (t - 2)
            p.grad = g
            ps[i] = af.adafactor_step(ps[i], g.numpy().ravel(), states[i], p.shape, lr=1e-2, t=t, wd=0.1)
        ref.step()
        for i, p in enumerate(params):
            if p.numel() == 0:
                continue
            np.testing.assert_allclose(ps[i], p.detach().numpy().ravel(), rtol=1e-10, atol=1e-12,
                                       err_msg=f"{name} {tuple(p.shape)} step {t}")
            for k, v in states[i].items():
                np.testing.assert_allclose(v.ravel(), ref.state[p][k].numpy().ravel(), rtol=1e-12, atol=0,
                                           err_msg=f"{name} {tuple(p.shape)} {k} step {t}")
