"""K2-af (Adafactor) on the H100 across the path catalogue ``adafactor_oracle.AF_PATHS``.

Every case runs several steps, each checked by ``test_gpu_adafactor._check_step``: a float64
``torch.optim.Adafactor`` started from the kernel's own state, weights within 1e-4 of the
tensor's largest step plus 2 ulp of |p|, ``row_var`` / ``col_var`` / ``variance`` at rtol 1e-5,
the bf16 shadow equal to the master rounded (the bounds are derived in that file).

The branch tests check their preconditions in the float64 restatement ``adafactor_step`` fed
the kernel's state, so none of them can pass by taking one side only:
  * alpha = eps2 * rho (all-zero and tiny weights) beside alpha = RMS(p) * rho;
  * update clipping, RMS(u) / d above 1 and below 1 in one table, and with d raised, nowhere;
  * the eps1 clamp of the row mean and the eps1^2 clamp of vhat, with an all-zero matrix in a
    B > 1 tensor;
  * a NaN and an inf in one matrix of B > 1 tensors: the non-finite pattern of every tensor is
    fp32 torch's, and every other matrix and tensor is bit for bit a clean run's;
  * two launches and a CUDA-graph replay over the catalogue's largest band table agree bit for
    bit, with more bands than the device holds CTAs.

No case disagreed with torch: the kernel and the planner were left as they were.
"""
import pytest
import torch

import frl_b200  # noqa: F401
from frl_b200 import _native, fused_optim
from frl_b200.multi_tensor import GradSegTable
import adafactor_oracle as af
from adafactor_oracle import AF_PATHS, AfCase
import test_gpu_adafactor as T

pytestmark = pytest.mark.gpu
DEV = "cuda"
EPS1, EPS2 = T.EPS


class _PathCase(T._Case):
    """``test_gpu_adafactor._Case`` over an ``AfCase``: its model flags, gradient dtypes and
    gradient offsets; ``weights`` (per slot, a tensor or None) replaces the randn masters."""

    def __init__(self, case, lp=True, seed=0, lr=1e-2, wd=1e-2, d=1.0, weights=None, make=None):
        self.case = case
        self.arena = a = T._Arena(case.shapes, lp, seed)
        for i, s in enumerate(a.slots):
            s.is_model = case.slot_model(i)
        if weights is not None:
            for s, w in zip(a.slots, weights):
                if w is not None:
                    a.master[s.offset:s.end] = w.reshape(-1).to(DEV)
            if a.lp is not None:
                a.lp = a.master.to(torch.bfloat16)
        self.opt = fused_optim.FusedAdafactor(a, lr=lr, weight_decay=wd, d=d)
        self.table = GradSegTable(a.slots, a.device)
        self.make = make
        self.t = 0
        self.new_grads()

    def values(self, i, s):
        """This step's gradient of slot i, float32 on the CPU: ``make(i, slot, t)``, else randn
        * 0.1 * exp(randn) as in test_gpu_adafactor."""
        v = self.make(i, s, self.t) if self.make is not None else None
        if v is None:
            gen = self.arena.gen
            v = torch.randn(s.numel, generator=gen) * 0.1 * torch.exp(torch.randn(s.numel, generator=gen))
        return v.reshape(-1).float()

    def new_grads(self, edit=None):
        a, off = self.arena, self.case.g_offset
        self.t += 1
        self.grads = []
        for i, s in enumerate(a.slots):
            buf = torch.zeros(s.numel + off + 8, dtype=self.case.slot_gdt(i), device=DEV)
            buf[off:off + s.numel] = self.values(i, s).to(buf.dtype).to(DEV)
            self.grads.append(buf[off:off + s.numel])
        if edit is not None:
            edit(self.grads)
        for s, g in zip(a.slots, self.grads):
            self.table.point(s, g.data_ptr(), g.dtype)
        self.table.upload()


def _restated(case, gs=1.0, coef=1.0):
    """Per slot, what the float64 restatement reports (``adafactor_step``'s ``info``) for the
    step about to run, from the kernel's weights and state; None for a slot without elements."""
    a, opt, h = case.arena, case.opt, case.opt.hyper
    out = []
    for s, g in zip(a.slots, case.g_eff(gs, coef)):
        if s.numel == 0:
            out.append(None)
            continue
        B, R, C = af.adafactor_shape(s.shape)
        v = {k: x.double().cpu().numpy() for k, x in opt._slot_state(s).items()}
        st = {"row_var": v["row_var"].reshape(B, R), "col_var": v["col_var"].reshape(B, C)} if R else \
            {"variance": v["variance"].reshape(-1)}
        info = {}
        af.adafactor_step(a.master[s.offset:s.end].double().cpu().numpy(), g.cpu().numpy(), st, s.shape,
                          lr=h["lr"], t=opt._steps + 1, beta2_decay=h["beta2_decay"], eps1=EPS1, eps2=h["eps"][1],
                          d=h["d"], wd=h["weight_decay"], info=info)
        out.append(info)
    return out


# ---- the catalogue ----------------------------------------------------------------------------------

@pytest.mark.parametrize("name", list(AF_PATHS))
def test_case_matches_torch_adafactor(name):
    case = _PathCase(AF_PATHS[name], seed=sum(map(ord, name)))
    for t in range(3):
        T._check_step(case, gs=0.5, coef=0.7 if t % 2 else 1.0)
        case.new_grads()


# ---- alpha: RMS(p) below and above eps2 ------------------------------------------------------------

def test_both_alpha_branches_in_one_table():
    shapes = ((40, 70), (3, 33, 1030), (5000,), (300,), (64, 64), (2, 20, 9), (37, 130), ())
    kind = ("zero", "tiny", "zero", "tiny", "randn", "zero", "randn", "zero")
    gen = torch.Generator().manual_seed(21)
    weights = [torch.zeros(sh) if k == "zero" else torch.randn(sh, generator=gen) * 1e-5 if k == "tiny" else None
               for sh, k in zip(shapes, kind)]
    case = _PathCase(AfCase(shapes, gdt=(torch.float32, torch.bfloat16)), seed=21, weights=weights)
    for _ in range(3):
        for k, info in zip(kind, _restated(case)):
            assert (info["rms_p"] < EPS2) == (k != "randn"), (k, info["rms_p"])
        T._check_step(case, gs=1.0, coef=1.0)
        case.new_grads()


# ---- update clipping: RMS(u) / d above and below 1 -------------------------------------------------

_CLIP_SHAPES = ((37, 130), (3, 40, 50), (2000,), (64, 256), (2, 33, 70), (48, 80), (500,))
_CLIP_KIND = ("decaying", "decaying", "decaying", "outlier", "outlier", "heavy_tailed", "growing")


def _clip_grads(i, s, t):
    gen = torch.Generator().manual_seed(1000 * t + i)
    k = _CLIP_KIND[i]
    if k == "decaying":                 # 10x smaller each step: vhat remembers the larger past
        return torch.randn(s.numel, generator=gen) * 0.1 * 10.0 ** -t
    if k == "growing":
        return torch.randn(s.numel, generator=gen) * 0.1 * 10.0 ** t
    if k == "heavy_tailed":
        return torch.randn(s.numel, generator=gen) * torch.exp(3 * torch.randn(s.numel, generator=gen))
    g = torch.randn(s.numel, generator=gen) * 1e-3
    g[int(torch.randint(s.numel, (1,), generator=gen))] = 1e3
    return g


def test_both_sides_of_the_clipping_threshold():
    case = _PathCase(AfCase(_CLIP_SHAPES, gdt=(torch.float32, torch.bfloat16)), seed=23, make=_clip_grads)
    for t in range(1, 4):
        x = {k: [] for k in _CLIP_KIND}
        for k, info in zip(_CLIP_KIND, _restated(case)):
            x[k].append(info["x"])
        assert min(x["outlier"] + x["heavy_tailed"]) > 1.0, (t, x)
        if t > 1:
            assert max(x["decaying"]) < 1.0 < min(x["growing"]), (t, x)
        T._check_step(case, gs=1.0, coef=1.0)
        case.new_grads()


def test_nothing_clips_with_d_raised():
    case = _PathCase(AfCase(_CLIP_SHAPES, gdt=(torch.bfloat16, torch.float32)), seed=23, d=1e4, make=_clip_grads)
    for _ in range(3):
        assert max(info["x"] for info in _restated(case)) < 1.0
        T._check_step(case, gs=1.0, coef=1.0)
        case.new_grads()


# ---- the eps1 clamps: row mean below eps1, vhat below eps1^2 ----------------------------------------

_EPS_SHAPES = ((40, 70), (3, 33, 50), (2, 64, 20), (300,), (37, 130))


def _eps_grads(i, s, t):
    gen = torch.Generator().manual_seed(100 * t + i)
    g = torch.randn(s.numel, generator=gen)
    if i == 0:
        return g * 1e-4                               # row mean ~1e-8 < eps1
    if i == 1:
        g = (g * 1e-8).view(s.shape)                  # vhat ~1e-25 < eps1^2; matrix 1 all zero
        g[1] = 0
        return g
    if i == 2:
        g = (g * 0.1).view(s.shape)                   # a zero row and a zero column in each matrix
        g[:, 5, :] = 0
        g[:, :, 7] = 0
        return g
    if i == 3:
        return g * 1e-8                               # variance ~1e-16 < eps1^2
    return g * 0.1


def test_both_eps1_clamps():
    case = _PathCase(AfCase(_EPS_SHAPES, gdt=(torch.float32, torch.bfloat16)), seed=25, make=_eps_grads)
    for _ in range(3):
        info = _restated(case)
        assert info[0]["row_mean"].max() < EPS1 and info[0]["vhat_min"] > EPS1 ** 2
        assert info[1]["vhat_min"] < EPS1 ** 2 and info[1]["row_mean"][1] == 0.0
        assert info[2]["vhat_min"] == 0.0 and info[2]["row_mean"].min() > EPS1
        assert info[3]["vhat_min"] < EPS1 ** 2
        assert info[4]["row_mean"].min() > EPS1 and info[4]["vhat_min"] > EPS1 ** 2
        T._check_step(case, gs=1.0, coef=1.0)
        case.new_grads()


# ---- non-finite gradients stay in their matrix -------------------------------------------------------

_NF_SHAPES = ((4, 33, 40), (3, 70, 1030), (37, 130), (1000,), (2, 5, 6))
_NAN_AT = (0, 2, (2, 5, 7))            # slot, matrix, (matrix, row, column)
_INF_AT = (1, 1, (1, 66, 1027))        # band b = 1, rb = 1, cb = 1


def _poison(grads):
    for (slot, _, idx), v in ((_NAN_AT, float("nan")), (_INF_AT, float("inf"))):
        grads[slot].view(_NF_SHAPES[slot])[idx] = v


def test_nonfinite_gradient_stays_in_its_matrix():
    d = 1e4                             # no clean tensor clips: a poisoned one's denominator, max(1, nan), is 1 too
    clean = _PathCase(AfCase(_NF_SHAPES), lp=False, seed=27, d=d)
    bad = _PathCase(AfCase(_NF_SHAPES), lp=False, seed=27, d=d)
    bad.grads = [g.clone() for g in clean.grads]
    _poison(bad.grads)
    for s, g in zip(bad.arena.slots, bad.grads):
        bad.table.point(s, g.data_ptr(), g.dtype)
    bad.table.upload()
    assert max(info["x"] for info in _restated(clean)) < 1.0
    params = [torch.nn.Parameter(bad.arena.master[s.offset:s.end].view(s.shape).cpu().clone())
              for s in bad.arena.slots]
    ref = torch.optim.Adafactor(params, lr=1e-2, weight_decay=1e-2, d=d, foreach=False)
    for p, g in zip(params, bad.grads):
        p.grad = g.view(p.shape).cpu().clone()
    ref.step()
    clean.step()
    bad.step()
    torch.cuda.synchronize()
    poisoned = {_NAN_AT[0]: _NAN_AT[1], _INF_AT[0]: _INF_AT[1]}
    for i, (s, p) in enumerate(zip(bad.arena.slots, params)):
        got = bad.arena.master[s.offset:s.end].view(s.shape)
        want = clean.arena.master[s.offset:s.end].view(s.shape)
        assert torch.equal(torch.isfinite(got).cpu(), torch.isfinite(p.detach())), s.shape
        st_got, st_want = bad.opt._slot_state(s), clean.opt._slot_state(s)
        if i not in poisoned:
            assert torch.equal(got, want), s.shape
            for k in st_got:
                assert torch.equal(st_got[k], st_want[k]), (s.shape, k)
            continue
        b = poisoned[i]
        assert not bool(torch.isfinite(got[b]).all()), s.shape
        keep = [m for m in range(s.shape[0]) if m != b]
        assert torch.equal(got[keep], want[keep]), s.shape
        for k in st_got:
            assert torch.equal(st_got[k][keep], st_want[k][keep]), (s.shape, k)


# ---- the ticket reset over the largest table --------------------------------------------------------

def _largest():
    return max(AF_PATHS, key=lambda n: _native.adafactor_plan(af.case_shape_tensor(AF_PATHS[n]))[0].shape[0])


def _refill(case, t):
    """New gradient values written into the same allocations, so a captured graph reads them."""
    gen = torch.Generator().manual_seed(t)
    for g in case.grads:
        g.copy_((torch.randn(g.numel(), generator=gen) * 0.1).to(g.dtype))


def test_two_launches_and_graph_replay_identical_bytes_over_the_largest_table():
    name = _largest()
    spec = AfCase(AF_PATHS[name].shapes, gdt=(torch.float32, torch.bfloat16), model=(True, False))
    prop = torch.cuda.get_device_properties(0)
    n_work = _native.adafactor_plan(af.case_shape_tensor(spec))[0].shape[0]
    assert n_work > prop.multi_processor_count * prop.max_threads_per_multi_processor // 256, (name, n_work)
    a, b, c = (_PathCase(spec, seed=29) for _ in range(3))
    for case in (b, c):
        for s, g in zip(case.arena.slots, a.grads):
            case.table.point(s, g.data_ptr(), g.dtype)
        case.table.upload()
    coef = torch.tensor([0.7], device=DEV)
    c.opt.enable_dynamic_scalars()
    c.opt._af_plan(c.table)
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(st):
        with torch.cuda.graph(graph, stream=st):
            c.opt.apply_table(c.table, grad_scale=0.5, clip_coef_dev=coef)
    torch.cuda.current_stream().wait_stream(st)
    torch.cuda.synchronize()
    for t in range(4):
        _refill(a, t)
        for case in (a, b, c):
            case.opt.hyper["lr"] = 1e-2 / (t + 1)
        a.step(0.5, coef)
        b.step(0.5, coef)
        c.opt.begin_step()
        graph.replay()
        c.opt.end_step()
        torch.cuda.synchronize()
        for x, y, z in zip(T._snapshot(a), T._snapshot(b), T._snapshot(c)):
            assert torch.equal(x, y) and torch.equal(x, z), t
