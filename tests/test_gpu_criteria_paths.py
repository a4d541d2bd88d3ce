"""K4 (the fused criterion, csrc/criteria.cu) and K3 (global gradient norm and clip coefficient,
csrc/reduce.cu) on every code path, against float64 torch: F.cross_entropy and F.mse_loss, the
reference MaskedLoss formula (out[mask], or out - out when the mask selects nothing) written out
here, autograd for the gradients, and clip_grad_norm_ followed by torch.optim.SGD for K3.  Nothing
here goes through the numpy oracle, so a blind spot the oracle shares with a kernel cannot hide.

Every cross-entropy case states the branch it exists for and first asserts, from the launch
geometry restated below, that the kernels take it.  Tolerances are written at each check:
  * losses: 1e-5 relative.  bf16 outputs are compared against float64 torch on the bf16-rounded
    inputs: the kernels widen them exactly and then compute in fp32, as for fp32 outputs;
  * gradients: an absolute bound per element, scaled by |upstream * weight| / (selected count).
"""
import math

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import frl_b200  # noqa: F401
from frl_b200 import _native, criteria
from frl_b200.criteria import MaskedLoss

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
EPS32 = 2.0 ** -23
BF16_STORE = 2.0 ** -8          # relative error bound of a value rounded to bf16 (twice the half-ulp)

# K4 launch geometry (csrc/criteria.cu), restated to tell which branch a case takes
K4_MAX_BLOCKS = 528             # CTAs per task at most
K4_WARPS = 8                    # one CE row per warp of a 256-thread CTA
K4_ROW_CHUNK = 1024             # a CE row this long or shorter is held in registers
K4_MSE_PER_CTA = 256 * 8        # MSE elements per CTA before the CTA count is capped
CE_ROWS_ONE_PASS = K4_MAX_BLOCKS * K4_WARPS       # 4224: more rows and a warp strides over rows
MSE_FULL_GRID = K4_MAX_BLOCKS * 256               # 135 168: one element per thread of 528 CTAs
MSE_CAPPED = K4_MAX_BLOCKS * K4_MSE_PER_CTA       # 1 081 344: more and the CTA count is capped

# K3 launch geometry (csrc/reduce.cu)
K3_PER_CTA = 256 * 4 * 4        # elements one CTA covers before the grid strides
K3_MAX_PARTIALS = 132 * 8


def _ce_path(out: torch.Tensor, C: int) -> str:
    """The forward and backward branch K4 takes for a CE output as the kernels see it (the
    backward's gradient buffer is a fresh allocation, so it is always aligned)."""
    vec = C % 4 == 0 and out.data_ptr() % (4 * out.element_size()) == 0
    if not vec:
        return "scalar"
    return "register" if C <= K4_ROW_CHUNK else "online"


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


@pytest.fixture(autouse=True)
def _release_cached_memory():
    """The device is shared: hand the float64 reference copies back after every case."""
    yield
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------
# tasks, the kernel run, the float64 reference
# ------------------------------------------------------------------------------------------------

class _Task:
    """One criterion task.  The output lives in a flat leaf `storage` (at `offset` elements, so a
    view can be misaligned); the kernels see `out()`, a view of it, and its gradient lands in
    storage.grad."""

    def __init__(self, module, values, dtype, targets, weight=1.0, offset=0):
        self.module = module
        self.shape = tuple(values.shape)
        self.offset = offset
        self.storage = torch.empty(values.numel() + offset, dtype=dtype, device=DEV)
        with torch.no_grad():
            self.storage[offset:].copy_(values.reshape(-1))
        self.storage.requires_grad_(True)
        self.targets = tuple(targets)
        self.weight = weight

    def out(self):
        return self.storage[self.offset:].view(self.shape)

    @property
    def inner(self):
        return self.module.loss_layer if isinstance(self.module, MaskedLoss) else self.module

    @property
    def mask(self):
        return self.targets[1] if isinstance(self.module, MaskedLoss) else None

    @property
    def is_ce(self):
        return isinstance(self.inner, nn.CrossEntropyLoss)


def _run_k4(tasks, upstream, sink=None, nan_flag=None):
    """[total, w_i L_i] and d(upstream . losses)/d out_i through the fused kernels."""
    outs = [t.out() for t in tasks]
    res = criteria.fused_task_losses([t.module for t in tasks], outs, [t.targets for t in tasks],
                                     [t.weight for t in tasks], sink, nan_flag)
    assert res is not None, "the tasks should be inside the kernels' domain"
    res.backward(upstream)
    grads = []
    for t in tasks:
        g = t.storage.grad
        grads.append(torch.zeros(t.shape, device=DEV) if g is None else g[t.offset:].view(t.shape).clone())
        t.storage.grad = None
    return res.detach(), grads


def _ref_loss(t, x):
    """The task's loss in float64 torch, as the reference evaluates it."""
    tgt = t.targets[0]
    if t.is_ce:
        def fn(a, b):
            return F.cross_entropy(a, b, ignore_index=t.inner.ignore_index)
    else:
        tgt = tgt.double()
        fn = F.mse_loss
    if t.mask is None:
        return fn(x, tgt)
    m = t.mask.bool()
    if not bool(m.any()):
        return fn(x - x, tgt - tgt)          # reference MaskedLoss with an empty mask
    return fn(x[m], tgt[m])


def _ref_k4(tasks, upstream):
    xs = [t.out().detach().double().requires_grad_(True) for t in tasks]
    subs = [t.weight * _ref_loss(t, x) for t, x in zip(tasks, xs)]
    total = 0.0
    for s in subs:
        total = total + s
    losses = torch.stack([total] + subs)
    grads = torch.autograd.grad(losses, xs, grad_outputs=upstream.double(), allow_unused=True)
    return losses.detach(), [torch.zeros_like(x) if g is None else g for x, g in zip(xs, grads)]


def _count(t):
    """Rows (CE) or elements (MSE) the task's mean divides by."""
    if t.is_ce:
        valid = t.targets[0] != t.inner.ignore_index
        if t.mask is not None:
            valid = valid & t.mask.bool()
        return int(valid.sum())
    if t.mask is None:
        return t.out().numel()
    return int(t.mask.bool().sum()) * (t.out().numel() // max(t.mask.numel(), 1))


def _grad_bound(t, upstream, i):
    """Absolute bound on |kernel - float64| per gradient element: a multiple of fp32 (or bf16
    storage) rounding, times |(g_total + g_i) * w_i| / count.  CE: the kernels form
    exp(x - lse) with an fp32 lse, whose rounding grows with |lse| (logits scaled by 1e4)."""
    x = t.out().detach().double()
    unit = abs(float(upstream[0]) + float(upstream[1 + i])) * abs(t.weight) / max(_count(t), 1)
    store = BF16_STORE if t.storage.dtype == torch.bfloat16 else 8 * EPS32
    if t.is_ce:
        lse = torch.logsumexp(x, dim=1, keepdim=True).nan_to_num(0.0)
        return unit * (store + 8 * EPS32 * (1.0 + lse.abs()))
    diff = (x - t.targets[0].double()).abs().nan_to_num(0.0)
    return unit * (2.0 * diff * store + EPS32)


def _assert_close(got, want, bound, what):
    """|got - want| <= bound elementwise; NaN and inf only where the other side has them."""
    want = want.double()
    assert got.shape == want.shape, (what, got.shape, want.shape)
    gn, wn = torch.isnan(got), torch.isnan(want)
    assert torch.equal(gn, wn), (f"{what}: NaN at {int((gn & ~wn).sum())} unexpected and "
                                 f"{int((wn & ~gn).sum())} missing entries")
    gi, wi = got.isinf(), want.isinf()
    assert torch.equal(gi, wi) and torch.equal(got[gi].double(), want[wi]), f"{what}: infinities differ"
    err = got.to(torch.float64, copy=True).sub_(want).abs_().masked_fill_(wn | wi, 0.0)
    bound = torch.as_tensor(bound, dtype=torch.float64, device=err.device).expand_as(err)
    bad = err > bound
    if bool(bad.any()):
        k = int((err - bound).flatten().argmax())
        raise AssertionError(f"{what}: {int(bad.sum())} of {err.numel()} entries out of bound; worst at flat "
                             f"index {k}: got {got.flatten()[k].item()!r} want {want.flatten()[k].item()!r} "
                             f"bound {bound.flatten()[k].item():.3g}")


def _check_k4(tasks, upstream, sink=None, nan_flag=None):
    got, grads = _run_k4(tasks, upstream, sink, nan_flag)
    want, want_grads = _ref_k4(tasks, upstream)
    _assert_close(got, want, 1e-5 * want.abs(), "losses [total, w_i L_i]")
    for i, t in enumerate(tasks):
        _assert_close(grads[i], want_grads[i], _grad_bound(t, upstream, i), f"task {i} gradient")
    return got, grads


def _ce_values(rows, C, seed, ignore_index=-100):
    """Logits with the edges that matter: labels 0 and C-1 (the last partial vector or chunk),
    rows scaled by 1e4 (the max subtraction carries the row), rows with -inf logits (never at
    the label) and ignored rows."""
    g = _gen(seed)
    x = torch.randn(rows, C, device=DEV, generator=g) * 2
    y = torch.randint(0, C, (rows,), device=DEV, generator=g)
    y[0] = C - 1
    if rows > 1:
        y[1] = 0
        y[-1] = C - 1
    r = torch.arange(rows, device=DEV)
    x[r % 8 == 3] *= 1e4
    ninf = r[r % 8 == 5]
    if len(ninf):
        x[ninf[:, None], torch.tensor([1, C // 2, C - 2], device=DEV)] = -math.inf
        x[ninf, y[ninf]] = torch.randn(len(ninf), device=DEV, generator=g)
    y[r % 11 == 6] = ignore_index
    return x, y


# ------------------------------------------------------------------------------------------------
# K4: cross-entropy on every forward / backward branch
# ------------------------------------------------------------------------------------------------

# (C, rows, branch of an aligned output, whether a warp strides over rows)
CE_SHAPES = [
    (1023, 7, "scalar", False), (1023, 4225, "scalar", True),
    (1024, 1, "register", False), (1024, 4224, "register", False), (1024, 20011, "register", True),
    (1025, 7, "scalar", False),
    (1028, 4225, "online", True), (1028, 20011, "online", True),
    (2048, 7, "online", False), (2052, 33, "online", False), (4096, 4225, "online", True),
    (32000, 7, "online", False),
    (50257, 7, "scalar", False),
]


def _ce_params():
    for C, rows, path, strided in CE_SHAPES:
        tag = "-strided" if strided else ""
        yield pytest.param(C, rows, 0, path, strided, id=f"C{C}-rows{rows}-{path}{tag}")
        if C % 4 == 0:
            # a view one element into its buffer: C % 4 == 0 but the vector loads are not allowed
            yield pytest.param(C, rows, 1, "scalar", strided, id=f"C{C}-rows{rows}-misaligned-scalar{tag}")


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("C,rows,offset,path,strided", list(_ce_params()))
def test_cross_entropy_paths_match_torch(C, rows, offset, path, strided, dtype):
    x, y = _ce_values(rows, C, seed=C * 7 + rows)
    t = _Task(nn.CrossEntropyLoss(), x, dtype, (y,), weight=1.3, offset=offset)
    out = t.out()
    assert _ce_path(out, C) == path
    assert (out.data_ptr() % (4 * out.element_size()) != 0) == bool(offset)
    assert (rows > CE_ROWS_ONE_PASS) == strided
    _check_k4([t], torch.tensor([0.75, -1.5], device=DEV))


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("C", [256, 1028])
def test_per_position_cross_entropy_with_ignore_index_zero(C, dtype):
    """The text layout: logits [N, C, L], labels [N, L], padding label 0 ignored."""
    N, L = 3, 343
    g = _gen(C)
    x = torch.randn(N, C, L, device=DEV, generator=g) * 3
    y = torch.randint(1, C, (N, L), device=DEV, generator=g)
    y[:, -100:] = 0                       # padded tail of every line
    y[0, 0], y[1, 0] = C - 1, 1
    t = _Task(nn.CrossEntropyLoss(ignore_index=0), x, dtype, (y,), weight=0.9)
    _check_k4([t], torch.tensor([1.0, 0.25], device=DEV))


# ------------------------------------------------------------------------------------------------
# K4: MSE, grid-stride loops, the CTA cap, target dtypes, masks
# ------------------------------------------------------------------------------------------------

f32, bf16 = torch.float32, torch.bfloat16
# (output shape, output dtype, target dtype, mask: None | "rows" ([B, L] over [B, L, D]) |
#  "first" (over dim 0) | "elems" (full shape) | "empty" (selects nothing))
MSE_CASES = [
    ((1,), f32, f32, None), ((7,), bf16, f32, None),
    ((MSE_FULL_GRID - 1,), f32, f32, None), ((MSE_FULL_GRID + 1,), f32, bf16, None),
    ((MSE_CAPPED - 1,), f32, f32, None), ((MSE_CAPPED + 1,), bf16, bf16, None),
    ((1000, 3001), f32, f32, None), ((1000, 3001), bf16, f32, None),
    ((6, 37, 129), f32, f32, "rows"), ((6, 37, 129), bf16, bf16, "rows"),
    ((64, 129, 160), f32, f32, "rows"), ((64, 129, 160), bf16, f32, "elems"),
    ((33, 40), f32, f32, "first"), ((1000, 3001), f32, bf16, "first"),
    ((6, 37, 129), f32, f32, "empty"), ((6, 37, 129), bf16, bf16, "empty"),
]


def _mse_id(case):
    shape, od, td, mask = case
    return "x".join(map(str, shape)) + f"-{str(od)[6:]}-tgt_{str(td)[6:]}-{mask or 'unmasked'}"


@pytest.mark.parametrize("shape,out_dtype,tgt_dtype,mask_kind", MSE_CASES, ids=[_mse_id(c) for c in MSE_CASES])
def test_mse_paths_match_torch(shape, out_dtype, tgt_dtype, mask_kind):
    g = _gen(sum(shape))
    o = torch.randn(shape, device=DEV, generator=g) * 1.5
    tgt = torch.randn(shape, device=DEV, generator=g).to(tgt_dtype)
    n = o.numel()
    if mask_kind is None:
        mod, targets = nn.MSELoss(), (tgt,)
    else:
        mshape = {"rows": shape[:2], "first": shape[:1], "elems": shape, "empty": shape[:2]}[mask_kind]
        mask = torch.rand(mshape, device=DEV, generator=g) > 0.4
        if mask_kind == "empty":
            mask.zero_()
        mod, targets = MaskedLoss(nn.MSELoss()), (tgt, mask)
        inner = n // mask.numel()            # elements of `out` one mask entry covers
        assert inner == {"rows": shape[-1], "first": n // shape[0], "elems": 1, "empty": shape[-1]}[mask_kind]
        if mask_kind == "rows":
            assert inner not in (1, n // shape[0])       # neither per element nor per row
    t = _Task(mod, o, out_dtype, targets, weight=0.6)
    got, grads = _check_k4([t], torch.tensor([1.25, 0.5], device=DEV))
    if mask_kind == "empty":
        assert got[1].item() == 0.0 and not bool(grads[0].any())


# ------------------------------------------------------------------------------------------------
# K4: masks that select nothing
# ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("ignore_index", [-100, 0, 3])
def test_empty_mask_matches_the_reference_formula(ignore_index):
    """inner(out - out, tgt - tgt): every CE label becomes 0, so ignore_index == 0 ignores every
    row and gives NaN (raising the NaN flag); otherwise log C.  MSE gives 0.  Zero gradients."""
    g = _gen(11)
    B, C = 64, 1028
    none = torch.zeros(B, dtype=torch.bool, device=DEV)
    y = torch.randint(0, C, (B,), device=DEV, generator=g)
    tasks = [_Task(MaskedLoss(nn.CrossEntropyLoss(ignore_index=ignore_index)),
                   torch.randn(B, C, device=DEV, generator=g), f32, (y, none), weight=1.5),
             _Task(MaskedLoss(nn.MSELoss()), torch.randn(B, 7, device=DEV, generator=g), bf16,
                   (torch.randn(B, 7, device=DEV, generator=g), none), weight=2.0)]
    flag = torch.zeros(1, dtype=torch.int32, pin_memory=True)
    sink = torch.full((3,), -1.0, pin_memory=True)
    got, grads = _check_k4(tasks, torch.tensor([1.0, 0.5, 0.5], device=DEV), sink, flag)
    torch.cuda.synchronize()
    if ignore_index == 0:
        assert math.isnan(got[1].item())
    else:
        assert got[1].item() == pytest.approx(1.5 * math.log(C), rel=1e-6)
    assert got[2].item() == 0.0
    assert all(not bool(gr.any()) for gr in grads)
    assert flag.item() == int(ignore_index == 0)
    assert torch.equal(sink.isnan(), got.cpu().isnan())


# ------------------------------------------------------------------------------------------------
# K4: eight tasks in one launch, and the composed path for a ninth
# ------------------------------------------------------------------------------------------------

def _eight_tasks(with_empty):
    g = _gen(2024)

    def rn(*shape, s=1.0):
        return torch.randn(*shape, device=DEV, generator=g) * s

    x1, y1 = _ce_values(4500, 1028, seed=1)
    x2, y2 = _ce_values(257, 1000, seed=2, ignore_index=5)
    x4, y4 = _ce_values(70, 4097, seed=4)
    m2 = torch.rand(257, device=DEV, generator=g) > 0.3
    m3 = torch.rand(33, 40, device=DEV, generator=g) > 0.5
    m6 = torch.rand(1000, 9, device=DEV, generator=g) > 0.5
    x7 = rn(64, 10)
    t5_shape = (0, 3) if with_empty else (5, 3)
    return [
        _Task(nn.MSELoss(), rn(300, 17), f32, (rn(300, 17),), weight=0.5),
        _Task(nn.CrossEntropyLoss(), x1, f32, (y1,), weight=2.0),
        _Task(MaskedLoss(nn.CrossEntropyLoss(ignore_index=5)), x2, bf16, (y2, m2), weight=0.25),
        _Task(MaskedLoss(nn.MSELoss()), rn(33, 40, 12), bf16, (rn(33, 40, 12), m3), weight=1.5),
        _Task(nn.CrossEntropyLoss(), x4, bf16, (y4,), weight=1.0),
        _Task(nn.MSELoss(), rn(*t5_shape), f32, (rn(*t5_shape),), weight=0.75),
        _Task(MaskedLoss(nn.MSELoss()), rn(1000, 9), f32, (rn(1000, 9).to(bf16), m6), weight=3.0),
        _Task(MaskedLoss(nn.CrossEntropyLoss()), x7, f32,
              (torch.randint(0, 10, (64,), device=DEV, generator=g),
               torch.zeros(64, dtype=torch.bool, device=DEV)), weight=1.25),
    ]


EIGHT_UPSTREAM = [0.5, 1.0, -2.0, 0.25, 3.0, -0.5, 1.5, 2.0, -1.0]


@pytest.mark.parametrize("with_empty", [False, True], ids=["all_rows", "task5_rows0"])
def test_eight_tasks_in_one_launch(with_empty):
    """Mixed kinds, dtypes and masks in one launch: every task's CTA range, partial slots and
    lse offset.  A task with no rows is a mean over nothing: NaN, as torch, and so is the total."""
    tasks = _eight_tasks(with_empty)
    assert len(tasks) == _native.MAX_TASKS
    assert (tasks[5].out().shape[0] == 0) == with_empty
    got, grads = _check_k4(tasks, torch.tensor(EIGHT_UPSTREAM, device=DEV))
    assert math.isnan(got[0].item()) == with_empty and math.isnan(got[6].item()) == with_empty
    assert not any(math.isnan(v) for i, v in enumerate(got.tolist()) if i not in (0, 6))


def test_eight_tasks_are_deterministic():
    tasks = _eight_tasks(False)
    up = torch.tensor(EIGHT_UPSTREAM, device=DEV)
    a, ga = _run_k4(tasks, up)
    b, gb = _run_k4(tasks, up)
    assert torch.equal(a, b)
    assert all(torch.equal(p, q) for p, q in zip(ga, gb))


def test_nine_tasks_take_the_composed_path():
    """More tasks than one launch holds: ParallelCriterion composes the loss modules one by one
    (masked tasks still through K4, one task per launch) and must give the same values."""
    tasks = _eight_tasks(False)
    g = _gen(9)
    tasks.append(_Task(nn.MSELoss(), torch.randn(20, 4, device=DEV, generator=g), f32,
                       (torch.randn(20, 4, device=DEV, generator=g),), weight=0.3))
    mods, outs = [t.module for t in tasks], [t.out() for t in tasks]
    tgts, weights = [t.targets for t in tasks], [t.weight for t in tasks]
    assert criteria._plan_for(mods, outs, tgts, weights) is None
    assert criteria._plan_for(mods[:8], outs[:8], tgts[:8], weights[:8]) is not None
    pc = criteria.ParallelCriterion(mods, weights, [f"t{i}" for i in range(9)])
    total, split = pc(outs, tgts)
    want, _ = _ref_k4(tasks, torch.ones(10, device=DEV))
    for i, t in enumerate(tasks):
        # an unmasked bf16 task runs torch's own bf16 loss here, which rounds its result to bf16
        tol = 1e-2 if (t.storage.dtype == bf16 and t.mask is None) else 1e-5
        assert split[f"t{i}"].item() == pytest.approx(want[1 + i].item(), rel=tol), i
    assert total.item() == pytest.approx(want[0].item(), rel=1e-2)
    fused, _ = _run_k4(tasks[:8], torch.ones(9, device=DEV))
    for i in range(8):
        tol = 1e-2 if (tasks[i].storage.dtype == bf16 and tasks[i].mask is None) else 2e-5
        assert split[f"t{i}"].item() == pytest.approx(fused[1 + i].item(), rel=tol), i


# ------------------------------------------------------------------------------------------------
# K4: the NaN flag and the loss sink
# ------------------------------------------------------------------------------------------------

NAN_TASKS = {"ce-register": 1000, "ce-online": 1028, "ce-scalar": 1025, "mse": None}


@pytest.mark.parametrize("where", ["masked_out", "selected"])
@pytest.mark.parametrize("kind", list(NAN_TASKS))
def test_nan_flag_follows_the_selected_entries(kind, where):
    """A NaN the mask drops changes nothing; a selected one makes that loss and the total NaN and
    raises the flag.  The NaN sits in the last partial vector / chunk of its row."""
    g = _gen(5)
    selected = where == "selected"
    C = NAN_TASKS[kind]
    if C is not None:
        x = torch.randn(64, C, device=DEV, generator=g)
        y = torch.randint(0, C, (64,), device=DEV, generator=g)
        y[3] = C - 1
        x[3, C - 2] = math.nan
        mask = torch.ones(64, dtype=torch.bool, device=DEV)
        mask[10] = False
        mask[3] = selected
        task = _Task(MaskedLoss(nn.CrossEntropyLoss()), x, f32, (y, mask), weight=1.5)
        assert _ce_path(task.out(), C) == kind[3:]
    else:
        o = torch.randn(40, 6, device=DEV, generator=g)
        o[3, 4] = math.nan
        mask = torch.rand(40, 6, device=DEV, generator=g) > 0.3
        mask[3, 4] = selected
        task = _Task(MaskedLoss(nn.MSELoss()), o, bf16, (torch.randn(40, 6, device=DEV, generator=g), mask))
    clean = _Task(nn.MSELoss(), torch.randn(32, 5, device=DEV, generator=g), f32,
                  (torch.randn(32, 5, device=DEV, generator=g),), weight=0.5)
    flag = torch.zeros(1, dtype=torch.int32, pin_memory=True)
    sink = torch.full((3,), -1.0, pin_memory=True)
    got, _ = _check_k4([task, clean], torch.tensor([1.0, 0.5, -0.5], device=DEV), sink, flag)
    torch.cuda.synchronize()
    assert flag.item() == int(selected)
    assert [math.isnan(v) for v in got.tolist()] == [selected, selected, False]
    _assert_close(sink, got.cpu(), 0.0, "sink")


def test_nan_in_an_ignored_row_leaves_loss_and_flag_clean():
    """A NaN row whose label is ignore_index does not enter the loss.  Torch's gradient of that row
    is NaN (log_softmax's backward multiplies the row's softmax by 0); the kernels write 0 there."""
    g = _gen(6)
    x = torch.randn(64, 1028, device=DEV, generator=g)
    y = torch.randint(0, 1028, (64,), device=DEV, generator=g)
    y[3] = 7
    x[3, 5] = math.nan
    task = _Task(nn.CrossEntropyLoss(ignore_index=7), x, f32, (y,), weight=1.0)
    flag = torch.zeros(1, dtype=torch.int32, pin_memory=True)
    up = torch.tensor([1.0, 0.5], device=DEV)
    got, grads = _run_k4([task], up, None, flag)
    want, want_grads = _ref_k4([task], up)
    torch.cuda.synchronize()
    assert flag.item() == 0
    _assert_close(got, want, 1e-5 * want.abs(), "losses")
    keep = torch.arange(64, device=DEV) != 3
    _assert_close(grads[0][keep], want_grads[0][keep], _grad_bound(task, up, 0)[keep], "gradient")
    assert not bool(grads[0][3].any())


# ------------------------------------------------------------------------------------------------
# K3: global norm and clip coefficient against clip_grad_norm_
# ------------------------------------------------------------------------------------------------

def _k3(g, pre_scale, max_norm, scratch=None):
    out3 = torch.full((3,), -1.0, device=DEV)
    if scratch is None:
        scratch = torch.zeros((_native.reduce_scratch_bytes() + 3) // 4, dtype=torch.int32, device=DEV)
    _native.grad_sumsq_clip(g, g.numel(), pre_scale=pre_scale, max_norm=max_norm, out3=out3, scratch=scratch)
    return out3


def _torch_clip(g, pre_scale, max_norm, p0=None, pieces=3):
    """clip_grad_norm_ over float64 copies of pre_scale * g split into several tensors; returns
    torch's norm, the coefficient it multiplies in (its clamp(max=1) formula) and the parameters,
    whose .grad are the clipped gradients."""
    gg = g.double() * pre_scale
    params = []
    for i, chunk in enumerate(torch.tensor_split(gg, pieces)):
        if p0 is None:
            # clip_grad_norm_ only reads and scales .grad: a zero-stride stand-in costs no memory
            p = torch.zeros((), dtype=torch.float64, device=DEV).expand(chunk.shape)
        else:
            p = torch.tensor_split(p0.double(), pieces)[i].clone()
        p.grad = chunk
        params.append(p)
    norm = torch.nn.utils.clip_grad_norm_(params, max_norm)
    coef = torch.clamp(max_norm / (norm + 1e-6), max=1.0)
    return norm, coef, params


def _assert_out3(out3, norm, coef):
    want = torch.stack([norm * norm, norm, coef]).to(DEV)
    _assert_close(out3, want, torch.tensor([2e-5, 1e-5, 1e-5], dtype=torch.float64, device=DEV) * want.abs(),
                  "K3 [sum g^2, norm, coefficient]")


K3_CAPPED = 1056 * K3_PER_CTA + K3_PER_CTA + 3      # more work than 132 x 8 CTAs, and a scalar tail
K3_SIZES = [(1, False), (3, False), (4, False), (5, False), (1023 * 4 + 1, False),
            (K3_CAPPED, True), (54_703_144, True)]


@pytest.mark.parametrize("dt", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("n,capped", K3_SIZES, ids=[str(n) for n, _ in K3_SIZES])
def test_norm_and_coefficient_on_both_sides_of_one(n, capped, dt):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert (-(-n // K3_PER_CTA) > min(sms * 8, K3_MAX_PARTIALS)) == capped
    g = torch.randn(n, device=DEV, generator=_gen(n))
    g[0] = 1.5                                       # keeps the norm well above the 1e-6 guard
    g = g.to(dt)
    scratch = torch.zeros((_native.reduce_scratch_bytes() + 3) // 4, dtype=torch.int32, device=DEV)
    norm1 = math.sqrt(sum(c.double().square().sum().item() for c in torch.split(g, 1 << 22)))
    for pre_scale, side in ((0.37, "below"), (1.0, "above")):
        max_norm = pre_scale * norm1 * (1 - 2e-4 if side == "below" else 1 + 2e-4)
        out3 = _k3(g, pre_scale, max_norm, scratch)        # second launch: the ticket was reset
        norm, coef, _ = _torch_clip(g, pre_scale, max_norm)
        assert (coef.item() < 1.0) == (side == "below")
        _assert_out3(out3, norm, coef)


@pytest.mark.parametrize("dt", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("n", [5, K3_CAPPED])
def test_all_zero_gradients(n, dt):
    g = torch.zeros(n, dtype=dt, device=DEV)
    out3 = _k3(g, 0.5, 0.3)
    norm, coef, _ = _torch_clip(g, 0.5, 0.3)
    assert out3.tolist() == [0.0, 0.0, 1.0]
    _assert_out3(out3, norm, coef)


NONFINITE = [("finite", None), ("nan", "body"), ("nan", "tail"), ("inf", "body"), ("inf", "tail")]


@pytest.mark.parametrize("dt", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("kind,pos", NONFINITE, ids=[f"{k}-{p}" if p else k for k, p in NONFINITE])
def test_clipped_sgd_step_matches_torch(kind, pos, dt):
    """K3's coefficient fed to K2 SGD against clip_grad_norm_ + torch.optim.SGD.  A NaN gradient
    makes every updated weight NaN; an inf one makes the coefficient 0 and only its own weight
    NaN.  `tail` puts the bad element in K3's scalar tail."""
    n = 100_003
    g = torch.randn(n, device=DEV, generator=_gen(3)) * 0.1
    bad = {"body": 4099, "tail": n - 1}.get(pos)
    if kind != "finite":
        g[bad] = math.nan if kind == "nan" else math.inf
    g = g.to(dt)
    p0 = torch.randn(n, device=DEV, generator=_gen(4))
    pre_scale = 0.5
    max_norm = 0.5 * torch.linalg.vector_norm(g.double() * pre_scale).item() if kind == "finite" else 1.0
    out3 = _k3(g, pre_scale, max_norm)
    norm, coef, params = _torch_clip(g, pre_scale, max_norm, p0=p0)
    _assert_out3(out3, norm, coef)
    if kind == "nan":
        assert math.isnan(out3[2].item())
    elif kind == "inf":
        assert out3[2].item() == 0.0
    else:
        assert 0.45 < out3[2].item() < 0.55

    p, buf = p0.clone(), torch.zeros(n, device=DEV)
    _native.sgd_momentum(p, g, buf, None, n, lr=0.1, mu=0.9, dampening=0.0, wd=1e-4, grad_scale=pre_scale,
                         grad_scale_dev=out3[2:], first_step=True)
    torch.optim.SGD(params, lr=0.1, momentum=0.9, weight_decay=1e-4).step()
    want = torch.cat([q.detach() for q in params])
    _assert_close(p, want, 1e-6 * (1.0 + want.abs().nan_to_num(0.0)), "weights after the clipped SGD step")
    if kind == "nan":
        assert bool(p.isnan().all())
    elif kind == "inf":
        assert p.isnan().nonzero().flatten().tolist() == [bad]
