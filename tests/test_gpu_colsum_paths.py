"""The bias-gradient kernels K6 (``frl_colsum``) and K6b (``frl_drelu_colsum``) on every
instantiation against float64 torch, and the arena ``nn.Linear`` sites that call them.

References.  The column sum is ``x.double().sum(0)``, plus ``out.double()`` when accumulating,
rounded once to the output dtype.  K6b's dZ is ``torch.ops.aten.threshold_backward(dy, act, 0)``,
stock ReLU backward: dy unless ``act <= 0``, so a NaN activation passes dy through.

Exact inputs.  Integers in [-8, 8] are exact in bf16, and with fewer than 2^21 rows every partial
sum stays below 2^24, so every fp32 sum of them is exact in any order.  The kernel's output must
then equal the float64 reference rounded once to the output dtype, bit for bit: a dropped, doubled
or misplaced row or column, a bad split fold, a skipped accumulate or a ticket left set shows.

Random normals.  The kernel's fold order for one column c, with S row splits (``colsum_splits``,
restated as ``splits`` below) and 8 warps per CTA:

    lane      the thread of (split s, warp w) adds rows s*8 + w + k*8S, k = 0, 1, ..., in sequence
              onto 0.f: at most d = ceil(rows / 8S) terms, the first add exact -> d - 1 roundings
    warps     the CTA adds its 8 warps' partials in order onto 0.f            -> 7 roundings
    splits    the last CTA of the tile adds the S split partials onto 0.f    -> S - 1 roundings
    old out   accumulate: one more add                                       -> 1 rounding
    output    fp32: nothing more;  bf16: one rounding to nearest even

Every input reaches the result through at most h = d + S + 6 fp32 additions, so by the standard
bound for summation trees

    |fp32 result - exact| <= E = gamma_h * mag,   gamma_h = h*U / (1 - h*U),   U = 2^-24,

where mag = sum_r |x_rc| (+ |old out_c|) in float64.  A bf16 output adds one rounding of relative
size at most 2^-8:  |out - exact| <= E + 2^-8 * (|exact| + E).  No subnormal term is needed: the
normals are far from the subnormal range.

Rows in flight.  The kernel is instantiated for 1, 2 and 4 rows a warp keeps in flight; the
default picks 4 for K6 and 2 for K6b, and ``FRL_B200_COLSUM_ROWS`` (read once per process)
selects the others.  ``run_colsum_rows.py`` runs the exact cases at each setting, the default
included, in a process of its own and lists the instantiations ``torch.profiler`` saw launch;
together they are all 48 (2 input dtypes x 2 output dtypes x vector/scalar x K6/K6b x 1/2/4 rows).
The profiling stays in those processes: a profiling session in the test process would change what
a later session there sees.

Dense Linear+ReLU sites run their forward through ``torch._addmm_activation`` (the cuBLASLt
bias+ReLU epilogue).  On an H100 with torch 2.11 that epilogue maps a NaN pre-activation to
NaN, as stock ``torch.relu`` does (``test_nan_activation_passes_dy_through_a_dense_unit``).
"""
import functools
import json
import os
import subprocess
import sys

import pytest
import torch
import torch.nn as nn

import frl_b200  # noqa: F401
from frl_b200 import _native, arena_linear, fused_optim, grad_sync
from frl_b200.arena import ParamArena
from frl_b200.model import MultiTaskModel
from frl_b200.types import OptAlgorithm, OptimOpts, Precision

pytestmark = pytest.mark.gpu
DEV = "cuda"

U = 2.0 ** -24
U_BF16 = 2.0 ** -8
F32, BF16 = torch.float32, torch.bfloat16
PAIRS = [(F32, F32), (BF16, BF16), (BF16, F32), (F32, BF16)]
PAIR_IDS = ["f32-f32", "bf16-bf16", "bf16-f32", "f32-bf16"]
CAP = 8192 * 128                 # one column tile at this many rows runs 128 splits of 1024 rows / lane
GUARD = 96.0                     # the value around ``out`` that no launch may touch
G = 5                            # guard elements on each side: ``out`` starts 5 elements into its buffer

# exact cases: rows 0, 1, 7, 63/64/65 and CAP +- 1; cols 1, 7, 8, 255, 256, 257, 4104; the headline
# MLP's trunk (64 and 4096 rows x 4096) and its heads' concatenated 1000 + 64 columns
EXACT_SHAPES = [(0, 8), (0, 7), (1, 1), (1, 8), (7, 7), (7, 255), (63, 256), (64, 256), (65, 256), (65, 257),
                (7, 4104), (64, 4096), (4096, 4096), (4096, 1064), (CAP - 1, 256), (CAP + 1, 256), (CAP + 1, 7)]
# aligned: vector path when cols % 8 == 0; offset: every operand one element into its storage (scalar
# path at any cols); act / dz: only that K6b operand misaligned; inplace: K6b's dz aliases dy
LAYOUTS = {"k6": ("aligned", "offset"), "k6b": ("aligned", "offset", "act", "dz", "inplace")}


@functools.lru_cache(None)
def sm_count() -> int:
    return int(_native.lib().frl_device_sm_count())


def splits(rows: int, cols: int) -> int:
    """``colsum_splits`` of colsum.cu at its defaults (4 CTAs per SM, >= 64 rows per split)."""
    tiles = -(-cols // 256)
    want = min(-(-sm_count() * 4 // tiles), -(-rows // 64))
    return max(1, min(want, 128))


def _ints(shape, lo, hi, dtype, gen):
    return torch.randint(lo, hi + 1, shape, generator=gen, device=DEV).to(dtype)


def _matrix(rows, cols, dtype, offset):
    """(storage, [rows, cols] view ``offset`` elements into it); the storage is NaN-filled."""
    store = torch.full((rows * cols + offset,), float("nan"), dtype=dtype, device=DEV)
    return store, store[offset:].view(rows, cols)


def _guarded(init):
    """``out`` as a slice of a larger buffer with GUARD on both sides, as an arena bias slice is."""
    buf = torch.full((init.numel() + 2 * G,), GUARD, dtype=init.dtype, device=DEV)
    buf[G:G + init.numel()] = init
    return buf, buf[G:G + init.numel()]


def _bits(t):
    return t.view(torch.int32) if t.dtype == F32 else t.view(torch.int16)


def assert_bits(got, want, what=""):
    assert got.dtype == want.dtype and got.shape == want.shape, what
    bad = (_bits(got) != _bits(want)).nonzero().flatten()
    assert bad.numel() == 0, "%s: %d elements differ, first at %s: got %r, want %r" % (
        what, bad.numel(), bad[:4].tolist(), got.flatten()[bad[:4]].tolist(), want.flatten()[bad[:4]].tolist())


def assert_nan_aware(got, want, what=""):
    """Same NaN positions; everything else bit-identical."""
    assert got.dtype == want.dtype and got.shape == want.shape, what
    assert torch.equal(torch.isnan(got), torch.isnan(want)), "%s: NaN positions differ" % what
    keep = ~torch.isnan(want)
    assert_bits(got[keep], want[keep], what)


def launch(kind, x, act, dz, out, accumulate=False):
    if kind == "k6":
        _native.colsum(x, out, accumulate=accumulate)
    else:
        _native.drelu_colsum(x, act, dz, out, accumulate=accumulate)


# ---- exact inputs ------------------------------------------------------------------------------------

def check_exact(kind, xdt, odt, rows, cols, layout, seed=0):
    """One exact case: store, then accumulate, into a guarded ``out``; dZ and its storage checked too."""
    gen = torch.Generator(device=DEV).manual_seed(seed * 1000003 + rows * 31 + cols)
    what = "%s %s->%s [%d, %d] %s" % (kind, xdt, odt, rows, cols, layout)
    off = {name: int(layout == "offset" or layout == name) for name in ("x", "act", "dz")}
    xs, x = _matrix(rows, cols, xdt, off["x"])
    x.copy_(_ints((rows, cols), -8, 8, xdt, gen))
    act = dz = dzs = None
    want_dz = x
    if kind == "k6b":
        _, act = _matrix(rows, cols, xdt, off["act"])
        act.copy_(_ints((rows, cols), -2, 2, xdt, gen))
        act[::3] *= -1                                   # -0.0 among the dead units
        want_dz = torch.ops.aten.threshold_backward(x, act, 0)
        if layout == "inplace":
            dzs, dz = xs, x
        else:
            dzs, dz = _matrix(rows, cols, xdt, off["dz"])
    old = _ints((cols,), -64, 64, odt, gen)
    buf, out = _guarded(old)
    snapshot = buf.clone()
    total = want_dz.double().sum(0)
    launch(kind, x, act, dz, out)
    assert_bits(out, total.to(odt), what + " store")
    if kind == "k6b":
        assert_bits(dz, want_dz, what + " dz")
        if off["dz"]:
            assert torch.isnan(dzs[0]), what + ": dz's storage before the view was written"
    out.copy_(old)                                       # in place, x now holds dZ, whose dZ is itself
    launch(kind, x, act, dz, out, accumulate=True)
    assert_bits(out, (total + old.double()).to(odt), what + " accumulate")
    assert_bits(buf[:G], snapshot[:G], what + " guard before out")
    assert_bits(buf[G + cols:], snapshot[G + cols:], what + " guard after out")


def exact_cases(shapes=EXACT_SHAPES, layouts=LAYOUTS):
    cases = []
    for kind in ("k6", "k6b"):
        for (xdt, odt), pid in zip(PAIRS, PAIR_IDS):
            for rows, cols in shapes:
                for layout in layouts[kind]:
                    if rows > 65536 and layout in ("act", "dz", "inplace"):
                        continue                         # the long cases: one vector and one scalar layout
                    cases.append(pytest.param(kind, xdt, odt, rows, cols, layout,
                                              id="%s-%s-%dx%d-%s" % (kind, pid, rows, cols, layout)))
    return cases


@pytest.mark.parametrize("kind,xdt,odt,rows,cols,layout", exact_cases())
def test_exact_sums_equal_float64_rounded_once(kind, xdt, odt, rows, cols, layout):
    check_exact(kind, xdt, odt, rows, cols, layout)


def test_exact_shapes_reach_every_split_regime():
    s = {shape: splits(*shape) for shape in EXACT_SHAPES}
    assert s[(63, 256)] == s[(64, 256)] == 1 and s[(65, 256)] == 2       # the 64-rows-per-split threshold
    assert s[(CAP - 1, 256)] == s[(CAP + 1, 256)] == s[(CAP + 1, 7)] == 128
    assert s[(0, 8)] == 1 and 1 < s[(4096, 4096)] < 128
    # CAP +- 1 straddle a whole number of rows per lane at 128 splits
    assert -(-(CAP - 1) // (8 * 128)) == 1024 and -(-(CAP + 1) // (8 * 128)) == 1025


# ---- rows in flight: every instantiation ------------------------------------------------------------

RIF_SHAPES = [(0, 8), (7, 7), (65, 257), (5000, 256), (5001, 264), (CAP + 1, 8)]


def _template_args(name):
    """``void frl::colsum_kernel<float, __nv_bfloat16, true, false, 4>(...)`` -> a normalised tuple."""
    inner = name.split("colsum_kernel<", 1)[1].split(">(", 1)[0]
    parts = [p.strip() for p in inner.split(",")]
    dt = ["bf16" if "bfloat16" in p else "f32" for p in parts[:2]]
    return (dt[0], dt[1], parts[2], parts[3], int(parts[4]))


ALL_INSTANTIATIONS = sorted((x, o, v, m, r) for x in ("f32", "bf16") for o in ("f32", "bf16")
                            for v in ("true", "false") for m in ("true", "false") for r in (1, 2, 4))


@functools.lru_cache(None)
def _run_rows(rif):
    """The exact cases of RIF_SHAPES in a process of its own at ``FRL_B200_COLSUM_ROWS=rif`` (None:
    unset, the default); the sorted instantiations it launched.  The profiler runs there too, so
    this process never starts a profiling session of its own."""
    script = os.path.join(os.path.dirname(os.path.abspath(__file__)), "run_colsum_rows.py")
    env = {k: v for k, v in os.environ.items() if k != "FRL_B200_COLSUM_ROWS"}
    if rif is not None:
        env["FRL_B200_COLSUM_ROWS"] = str(rif)
    res = subprocess.run([sys.executable, script], env=env, capture_output=True, text=True, timeout=900)
    assert res.returncode == 0 and "COLSUM_ROWS_OK" in res.stdout, res.stdout[-3000:] + res.stderr[-3000:]
    line = [ln for ln in res.stdout.splitlines() if ln.startswith("INSTANTIATIONS ")][-1]
    return sorted(tuple(t) for t in json.loads(line[len("INSTANTIATIONS "):]))


@pytest.mark.parametrize("rif", [None, 1, 2, 4], ids=["default", "1", "2", "4"])
def test_exact_cases_at_every_rows_in_flight_setting(rif):
    seen = _run_rows(rif)
    # the default keeps 4 rows in flight for K6 and 2 for K6b (two loads per row)
    want = {rif} if rif is not None else {2, 4}
    assert len(seen) == 16 and {t[4] for t in seen} == want, seen
    if rif is None:
        assert all(t[4] == (2 if t[3] == "true" else 4) for t in seen), seen


def test_every_colsum_instantiation_is_launched():
    seen = set()
    for rif in (None, 1, 2, 4):
        seen |= set(_run_rows(rif))
    assert sorted(seen) == ALL_INSTANTIATIONS and len(ALL_INSTANTIATIONS) == 48


# ---- random normals against the rounding envelope ---------------------------------------------------

ENVELOPE_SHAPES = [(64, 4096), (4096, 4096), (4096, 1064), (65, 257), (20000, 7), (CAP + 1, 256)]


def test_envelope_shapes_reach_one_some_and_the_maximum_split_count():
    s = [splits(r, c) for r, c in ENVELOPE_SHAPES]
    assert 1 in s and 128 in s and any(1 < v < 128 for v in s), s


def envelope(rows, cols, mag, exact, odt):
    S = splits(rows, cols)
    h = -(-rows // (8 * S)) + S + 6
    err = h * U / (1 - h * U) * mag
    if odt == BF16:
        err = err + U_BF16 * (exact.abs() + err)
    return err


@pytest.mark.parametrize("kind", ["k6", "k6b"])
@pytest.mark.parametrize("xdt,odt", PAIRS, ids=PAIR_IDS)
@pytest.mark.parametrize("rows,cols", ENVELOPE_SHAPES)
def test_random_sums_stay_inside_the_rounding_envelope(kind, xdt, odt, rows, cols):
    gen = torch.Generator(device=DEV).manual_seed(rows + cols)
    x = torch.randn(rows, cols, generator=gen, device=DEV).to(xdt)
    act = dz = None
    want_dz = x
    if kind == "k6b":
        act = torch.randn(rows, cols, generator=gen, device=DEV).relu().to(xdt)
        dz = torch.empty_like(x)
        want_dz = torch.ops.aten.threshold_backward(x, act, 0)
    old = (torch.randn(cols, generator=gen, device=DEV) * 10).to(odt)
    for accumulate in (False, True):
        buf, out = _guarded(old)
        launch(kind, x, act, dz, out, accumulate=accumulate)
        exact = want_dz.double().sum(0)
        mag = want_dz.double().abs().sum(0)
        if accumulate:
            exact, mag = exact + old.double(), mag + old.double().abs()
        dist = (out.double() - exact).abs()
        bound = envelope(rows, cols, mag, exact, odt)
        worst = int(torch.argmax(dist - bound))
        assert bool((dist <= bound).all()), "column %d: |%r - %r| > %r" % (
            worst, float(out[worst]), float(exact[worst]), float(bound[worst]))
        assert bool((buf[:G] == GUARD).all() and (buf[G + cols:] == GUARD).all())
        if kind == "k6b":
            assert_bits(dz, want_dz, "dz")


# ---- non-finite values, bf16 overflow --------------------------------------------------------------

def _specials(rows, cols, xdt, gen):
    """Integer dy / act with non-finite values planted column by column (rows >= 4)."""
    nan, inf = float("nan"), float("inf")
    dy = _ints((rows, cols), -8, 8, xdt, gen)
    act = _ints((rows, cols), -2, 2, xdt, gen)
    tiny = torch.finfo(xdt).smallest_normal * torch.finfo(xdt).eps      # the smallest positive subnormal
    act[:, :16] = 1.0
    act[1, :16] = -1.0                                   # row 1 dead, the others live
    dy[0, 0] = nan                                       # NaN dy at a live unit
    dy[1, 1] = nan                                       # NaN dy at a dead unit
    dy[0, 2] = inf                                       # +inf live
    dy[1, 3] = inf                                       # +inf dead
    dy[0, 4] = -inf                                      # -inf live
    dy[1, 5] = -inf                                      # -inf dead
    dy[0, 6], dy[2, 6] = inf, -inf                       # +inf and -inf in one column
    act[0, 7] = nan                                      # NaN activations, finite dy
    act[0, 8], act[2, 8] = nan, nan
    act[0, 9] = -0.0
    act[0, 10] = 0.0
    act[0, 11] = tiny
    act[0, 12], dy[0, 12] = nan, nan                     # NaN activation and NaN dy
    act[0, 13] = inf
    act[0, 14] = -inf
    dy[0, 15] = 0.0
    assert float(act[0, 11]) > 0 and float(act[0, 11]) < torch.finfo(xdt).smallest_normal
    return dy, act


@pytest.mark.parametrize("xdt,odt", PAIRS, ids=PAIR_IDS)
@pytest.mark.parametrize("cols", [64, 63], ids=["vector", "scalar"])
def test_non_finite_values_follow_threshold_backward_and_the_float64_sum(xdt, odt, cols):
    gen = torch.Generator(device=DEV).manual_seed(cols)
    rows = 40
    dy, act = _specials(rows, cols, xdt, gen)
    old = _ints((cols,), -64, 64, odt, gen)
    want_dz = torch.ops.aten.threshold_backward(dy, act, 0)
    assert not torch.isnan(want_dz[0, 7]) and want_dz[0, 7] == dy[0, 7]        # stock: NaN act passes dy
    for kind, src in (("k6", dy), ("k6b", want_dz)):
        for accumulate in (False, True):
            buf, out = _guarded(old)
            dz = torch.full_like(dy, 7.0) if kind == "k6b" else None
            launch(kind, dy, act, dz, out, accumulate=accumulate)
            want = src.double().sum(0) + (old.double() if accumulate else 0)
            assert_nan_aware(out, want.to(odt), "%s accumulate=%s" % (kind, accumulate))
            assert bool((buf[:G] == GUARD).all() and (buf[G + cols:] == GUARD).all())
            if kind == "k6b":
                assert_nan_aware(dz, want_dz, "dz")
    # in place
    dz = dy.clone()
    _, out = _guarded(old)
    _native.drelu_colsum(dz, act, dz, out)
    assert_nan_aware(dz, want_dz, "dz in place")
    assert_nan_aware(out, want_dz.double().sum(0).to(odt), "in place")


@pytest.mark.parametrize("kind", ["k6", "k6b"])
@pytest.mark.parametrize("xdt", [F32, BF16])
def test_bf16_output_overflows_to_inf_as_a_bf16_cast_does(kind, xdt):
    top = torch.finfo(BF16).max                          # (2 - 2^-7) * 2^127
    x = torch.zeros(2, 8, dtype=xdt, device=DEV)
    x[:, 0] = torch.tensor([top, 2.0 ** 119])            # (2 - 2^-8) * 2^127: a tie, rounds to even = inf
    x[:, 1] = torch.tensor([top, 2.0 ** 118])            # below the tie: bf16 max
    x[:, 2] = torch.tensor([-top, -2.0 ** 119])          # -inf
    x[:, 3] = torch.tensor([2.0 ** 119, 0.0])            # with the old out below: inf
    act = torch.ones_like(x)
    old = torch.tensor([0, 0, 0, top, -top, 1, 2, 3], dtype=BF16, device=DEV)
    for accumulate in (False, True):
        _, out = _guarded(old)
        dz = torch.empty_like(x) if kind == "k6b" else None
        launch(kind, x, act, dz, out, accumulate=accumulate)
        tot = x.double().sum(0) + (old.double() if accumulate else 0)
        assert tot.float().double().equal(tot)           # exact in fp32: one rounding to bf16 remains
        want = tot.float().to(BF16)
        assert_bits(out, want, "accumulate=%s" % accumulate)
        assert torch.isinf(out[0]) and torch.isinf(out[2]) and out[1] == top
        assert torch.isinf(out[3]) == accumulate


# ---- repeats and CUDA-graph replay ------------------------------------------------------------------

@pytest.mark.parametrize("xdt,odt", PAIRS, ids=PAIR_IDS)
def test_back_to_back_launches_repeat_and_replay_from_a_graph_bit_for_bit(xdt, odt):
    """K6, K6b, K6 with the same cols (one cached scratch, one ticket per tile) and 32, 1 and 6
    splits: each right on its own, the same bits again, and the same bits from a graph replay."""
    cols = 4104
    gen = torch.Generator(device=DEV).manual_seed(7)
    x1 = _ints((4096, cols), -8, 8, xdt, gen)
    dy, act = _ints((64, cols), -8, 8, xdt, gen), _ints((64, cols), -2, 2, xdt, gen)
    x3 = _ints((333, cols), -8, 8, xdt, gen)
    old3 = _ints((cols,), -64, 64, odt, gen)
    assert [splits(4096, cols), splits(64, cols), splits(333, cols)] == [32, 1, 6]
    outs = [torch.empty(cols, dtype=odt, device=DEV) for _ in range(3)]
    dz = torch.empty_like(dy)

    def sequence():
        _native.colsum(x1, outs[0])
        _native.drelu_colsum(dy, act, dz, outs[1])
        outs[2].copy_(old3)
        _native.colsum(x3, outs[2], accumulate=True)

    want_dz = torch.ops.aten.threshold_backward(dy, act, 0)
    want = [x1.double().sum(0).to(odt), want_dz.double().sum(0).to(odt),
            (x3.double().sum(0) + old3.double()).to(odt)]
    sequence()
    eager = [o.clone() for o in outs]
    for got, w, name in zip(eager, want, ("k6", "k6b", "k6 accumulate")):
        assert_bits(got, w, name)
    assert_bits(dz, want_dz, "dz")
    for _ in range(3):
        sequence()
        for got, w in zip(outs, eager):
            assert_bits(got, w, "repeat")
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        sequence()
    for _ in range(2):
        for o in outs:
            o.fill_(float("nan"))
        dz.fill_(float("nan"))
        graph.replay()
        torch.cuda.synchronize()
        for got, w in zip(outs, eager):
            assert_bits(got, w, "replay")
        assert_bits(dz, want_dz, "dz replay")


# ---- through the Linear sites -----------------------------------------------------------------------

class _Trunk(nn.Module):
    """Two Linear+ReLU units (the second applied twice per forward) and a plain Linear, on a 3-D
    input; every unit output is tapped with a tensor hook (module hooks would stop the fusion)."""

    def __init__(self):
        super().__init__()
        self.u1 = nn.Sequential(nn.Linear(32, 64), nn.ReLU())
        self.u2 = nn.Sequential(nn.Linear(64, 64), nn.ReLU())
        self.plain = nn.Linear(64, 48)
        self.taps = []
        self.edits = {}              # tap name -> fn(dy, y) -> dy: rewrites the gradient arriving there

    def _tap(self, name, y):
        rec = [name, y.detach().clone(), None]
        self.taps.append(rec)
        if y.requires_grad:
            def hook(g, rec=rec):
                edit = self.edits.get(rec[0])
                if edit is not None:
                    g = edit(g, rec[1])
                rec[2] = g.detach().clone()
                return g
            y.register_hook(hook)
        return y

    def forward(self, x):
        h = self._tap("u1", self.u1(x))
        h = self._tap("u2", self.u2(h))
        h = self._tap("u2", self.u2(h))
        o = self._tap("plain", self.plain(h))
        return o.reshape(-1, o.shape[-1])


def _net(heads):
    torch.manual_seed(0)
    return MultiTaskModel(_Trunk(), [nn.Linear(48, n) for n in heads]).to(DEV)


def _pipeline(net, precision):
    arena = ParamArena(net.parameters(), device=DEV, precision=precision,
                       adjacent=arena_linear.head_layout_groups(net))
    opt = fused_optim.create_fused_optimizer(arena, OptimOpts(algo=OptAlgorithm.SGD, lr=0.05))
    pipe = grad_sync.GradBucketPipeline(arena, opt, eager_update=False)
    assert pipe.patch_linears(net) == 3 + len(net.additional_layers)
    return arena, pipe


def _run(net, x, weights):
    """Forward, tapping the head outputs too; returns the loss sum_i <out_i, w_i>."""
    net.model_base.taps = []
    outs = net(x)
    for i, o in enumerate(outs):
        net.model_base._tap("head%d" % i, o)
    return sum((o.float() * w).sum() for o, w in zip(outs, weights))


def _bias_references(net):
    """Per bias parameter name: (float64 sum over every application of threshold_backward(dY, y, 0)
    (plain sites: dY), float64 sum of its magnitudes, rows per application)."""
    names = {"u1": "model_base.u1.0.bias", "u2": "model_base.u2.0.bias", "plain": "model_base.plain.bias"}
    ref = {}
    for name, y, dy in net.model_base.taps:
        dz = torch.ops.aten.threshold_backward(dy, y, 0) if name in ("u1", "u2") else dy
        dz = dz.reshape(-1, dz.shape[-1]).double()
        key = names.get(name) or "additional_layers.%s.bias" % name[len("head"):]
        s, m, _ = ref.get(key, (0, 0, 0))
        ref[key] = (s + dz.sum(0), m + dz.abs().sum(0), dz.shape[0])
    return ref


def _assert_close_nan_aware(got, want, tol, what):
    got = got.double()
    assert torch.equal(torch.isnan(got), torch.isnan(want)), what
    inf = torch.isinf(want)
    assert torch.equal(got[inf], want[inf]), what
    fin = torch.isfinite(want)
    dist = (got[fin] - want[fin]).abs()
    assert bool((dist <= tol[fin]).all()), "%s: worst %r over %r" % (what, float(dist.max()), float(tol[fin].max()))


def _check_arena_biases(net, arena):
    refs = _bias_references(net)
    assert len(refs) == 3 + len(net.additional_layers)
    for name, p in net.named_parameters():
        if not name.endswith("bias"):
            continue
        want, mag, rows = refs[name]
        got = arena.grad_view(arena.slot_of(p))
        # two applications (u2) round twice: twice the single-launch envelope
        tol = 2 * envelope(rows, got.numel(), mag, mag, got.dtype)
        _assert_close_nan_aware(got, want, tol, name)


HEADS = {"adjacent": (16, 24), "ragged": (10, 5)}


@pytest.mark.parametrize("heads", list(HEADS))
@pytest.mark.parametrize("precision", ["fp32", "bf16", "fp8"])
def test_step_writes_every_bias_slot_as_threshold_backward_plus_a_float64_sum(precision, heads):
    prec = Precision(precision)
    net = _net(HEADS[heads])
    arena, pipe = _pipeline(net, prec)
    sites = {s.module: s for s in pipe.linear_sites}
    trunk = net.model_base
    assert sites[trunk.u1[0]].relu is trunk.u1[1] and sites[trunk.u2[0]].relu is trunk.u2[1]
    assert sites[trunk.plain].relu is None
    assert [sites[m].fp8 for m in (trunk.u1[0], trunk.u2[0], trunk.plain)] == [prec is Precision.FP8] * 3
    msite = sites[net.additional_layers[0]].multihead
    assert msite is not None and (msite.grad_bias_cat() is not None) == (heads == "adjacent")
    dt = F32 if prec is Precision.FP32 else BF16
    gen = torch.Generator(device=DEV).manual_seed(3)
    x = torch.randn(4, 16, 32, generator=gen, device=DEV).to(dt)
    weights = [torch.randn(64, n, generator=gen, device=DEV) for n in HEADS[heads]]
    net.train()
    for _ in range(2):                                    # the second step re-stores every slot
        pipe.begin_step()
        _run(net, x, weights).backward()
        torch.cuda.synchronize()
        assert [t[0] for t in trunk.taps] == ["u1", "u2", "u2", "plain", "head0", "head1"]
        assert all(t[2] is not None for t in trunk.taps)
        _check_arena_biases(net, arena)
        pipe.finish_step()
    pipe.remove_hooks()


def _plant_non_finite(live):
    """Rewrite dY at u1: +inf and NaN at dead units, and, if ``live``, NaN and -inf at live ones."""
    def edit(g, y):
        g = g.clone()
        y2, g2 = y.reshape(-1, y.shape[-1]), g.view(-1, g.shape[-1])
        dead, alive = (y2 <= 0), (y2 > 0)
        for col, val, mask in ((0, float("inf"), dead), (1, float("nan"), dead), (2, float("nan"), alive),
                               (3, -float("inf"), alive)):
            rows = mask[:, col].nonzero().flatten()
            if rows.numel() and (live or mask is dead):
                g2[rows[0], col] = val
        return g
    return edit


def test_step_with_non_finite_dy_matches_threshold_backward():
    net = _net(HEADS["adjacent"])
    arena, pipe = _pipeline(net, Precision.FP32)
    net.model_base.edits["u1"] = _plant_non_finite(live=True)
    gen = torch.Generator(device=DEV).manual_seed(4)
    x = torch.randn(4, 16, 32, generator=gen, device=DEV)
    weights = [torch.randn(64, n, generator=gen, device=DEV) for n in HEADS["adjacent"]]
    net.train()
    pipe.begin_step()
    _run(net, x, weights).backward()
    torch.cuda.synchronize()
    b = arena.grad_view(arena.slot_of(net.model_base.u1[0].bias))
    assert torch.isfinite(b[:2]).all() and torch.isnan(b[2]) and b[3] == -float("inf")
    _check_arena_biases(net, arena)
    pipe.finish_step()
    pipe.remove_hooks()


@pytest.mark.parametrize("non_finite", [False, True])
def test_outside_a_step_the_sites_return_stock_gradients(non_finite):
    """``torch.autograd.grad`` (GradNorm, debugGrad) through the patched net against the stock one;
    with ``non_finite``, +inf and NaN reach u1 at dead units, where stock ReLU backward zeroes them."""
    stock, net = _net(HEADS["ragged"]), _net(HEADS["ragged"])
    _, pipe = _pipeline(net, Precision.FP32)
    gen = torch.Generator(device=DEV).manual_seed(5)
    x = torch.randn(4, 16, 32, generator=gen, device=DEV).requires_grad_(True)
    weights = [torch.randn(64, n, generator=gen, device=DEV) for n in HEADS["ragged"]]
    grads = []
    for m in (stock, net):
        if non_finite:
            m.model_base.edits["u1"] = _plant_non_finite(live=False)
        m.train()
        grads.append(torch.autograd.grad(_run(m, x, weights), [x] + list(m.parameters())))
    names = ["x"] + [n for n, _ in net.named_parameters()]
    for name, got, want in zip(names, grads[1], grads[0]):
        assert torch.isfinite(want).all(), name
        torch.testing.assert_close(got, want, rtol=1e-5, atol=1e-5, msg=name)
    pipe.remove_hooks()


def test_nan_activation_passes_dy_through_a_dense_unit():
    """A NaN input row makes u1's pre-activations NaN.  The loss is linear in the heads' outputs, so
    every dY stays finite, and u2's bias gradient keeps the rows where its activation is NaN."""
    net = _net(HEADS["adjacent"])
    arena, pipe = _pipeline(net, Precision.FP32)
    gen = torch.Generator(device=DEV).manual_seed(6)
    x = torch.randn(4, 16, 32, generator=gen, device=DEV)
    x[0, 0, 0] = float("nan")
    weights = [torch.randn(64, n, generator=gen, device=DEV) for n in HEADS["adjacent"]]
    net.train()
    pipe.begin_step()
    _run(net, x, weights).backward()
    torch.cuda.synchronize()
    taps = net.model_base.taps
    y_u1 = taps[0][1].reshape(-1, 64)
    nan_kept = bool(torch.isnan(y_u1[0]).all())
    print("cuBLASLt bias+ReLU epilogue keeps a NaN pre-activation:", nan_kept)
    assert nan_kept                                       # as torch.relu does (module docstring)
    assert not torch.isnan(y_u1[1:]).any()
    for name, _, dy in taps:
        assert torch.isfinite(dy).all(), name
    _check_arena_biases(net, arena)
    assert torch.isfinite(arena.grad_view(arena.slot_of(net.model_base.u2[0].bias))).all()
    # the rule matters here: dropping the NaN rows (act > 0 ? dy : 0) lands outside the envelope
    want, mag, rows = _bias_references(net)["model_base.u2.0.bias"]
    dropped = sum(torch.where(y > 0, dy, 0).reshape(-1, 64).double().sum(0) for n, y, dy in taps if n == "u2")
    assert bool(((dropped - want).abs() > 2 * envelope(rows, 64, mag, mag, F32)).any())
    pipe.finish_step()
    pipe.remove_hooks()
