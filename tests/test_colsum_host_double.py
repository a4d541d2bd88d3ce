"""The CPU stand-ins for K6 / K6b that the host-logic tests run on
(``oracle.optim_np.KernelDouble.colsum`` / ``drelu_colsum``) pinned to torch: dZ is
``threshold_backward(dy, act, 0)`` bit for bit, NaN positions included, and the column sums are the
float64 sum (plus the old ``out`` when accumulating) rounded once to the output dtype.  Integer
inputs keep every finite fp32 sum exact; NaN and +-inf sit in dy at live and dead units, and the
activations include NaN, -0.0, +0.0, the smallest positive subnormal and +-inf."""
import pytest
import torch

from oracle.optim_np import KernelDouble

F32, BF16 = torch.float32, torch.bfloat16
NAN, INF = float("nan"), float("inf")


def _specials(dt):
    gen = torch.Generator().manual_seed(0)
    dy = torch.randint(-8, 9, (8, 16), generator=gen).to(dt)
    act = torch.ones(8, 16, dtype=dt)
    act[1] = -1.0                                        # row 1 dead, the others live
    dy[0, 0], dy[1, 1] = NAN, NAN                        # NaN dy: live, dead
    dy[0, 2], dy[1, 3] = INF, INF                        # +inf: live, dead
    dy[0, 4], dy[1, 5] = -INF, -INF                      # -inf: live, dead
    dy[0, 6], dy[2, 6] = INF, -INF                       # +inf and -inf in one column
    act[0, 7] = NAN                                      # NaN activation, finite dy
    act[0, 8] = -0.0
    act[0, 9] = 0.0
    act[0, 10] = torch.finfo(dt).smallest_normal * torch.finfo(dt).eps
    act[0, 11], dy[0, 11] = NAN, NAN
    act[0, 12], act[0, 13] = INF, -INF
    dy[3, 14] = -3.0
    act[3, 14] = 0.0                                     # dead unit with negative dy: dZ is +0.0
    return dy, act


def _same(got, want):
    assert got.dtype == want.dtype
    assert torch.equal(torch.isnan(got), torch.isnan(want))
    keep = ~torch.isnan(want)
    bits = torch.int32 if got.dtype == F32 else torch.int16
    assert torch.equal(got[keep].view(bits), want[keep].view(bits))


@pytest.mark.parametrize("xdt,odt", [(F32, F32), (BF16, BF16), (BF16, F32), (F32, BF16)])
@pytest.mark.parametrize("accumulate", [False, True])
def test_host_double_matches_threshold_backward_and_the_float64_sum(xdt, odt, accumulate):
    dy, act = _specials(xdt)
    old = torch.arange(16, dtype=odt) - 8
    want_dz = torch.ops.aten.threshold_backward(dy, act, 0)
    assert want_dz[0, 7] == dy[0, 7] and want_dz[0, 10] == dy[0, 10] and torch.isnan(want_dz[0, 11])
    assert want_dz[0, 8] == 0 and want_dz[1, 3] == 0 and not torch.signbit(want_dz[3, 14])
    k = KernelDouble()
    for name, src in (("colsum", dy), ("drelu_colsum", want_dz)):
        out = old.clone()
        dz = torch.full_like(dy, 7.0)
        if name == "colsum":
            k.colsum(dy, out, accumulate=accumulate)
        else:
            k.drelu_colsum(dy, act, dz, out, accumulate=accumulate)
            _same(dz, want_dz)
        want = src.double().sum(0) + (old.double() if accumulate else 0)
        _same(out, want.to(odt))
    assert [c[0] for c in k.calls] == ["colsum", "drelu_colsum"]
