"""The layer-wise trust-ratio update K2-lw (``csrc/layerwise.cu``: ``lw_stats_kernel`` and
``lw_apply_kernel``, LARS and LAMB) on every instantiation and runtime branch against float64 on
the same GPU.

Reference.  ``LayerwiseTorch`` (tests/layerwise_oracle.py) in float64, one tensor at a time, fed
exactly the gradient the kernel reads: bf16-rounded where the gradient is bf16, times
``grad_scale``, times the clip coefficient on FRL_LW_CLIPPED segments only.  Every step starts the
reference from the kernel's own fp32 state (master weights, ``momentum_buffer`` unless it is a
first step, ``exp_avg``, ``exp_avg_sq`` and step = t-1), so one comparison covers one update.

Tolerance (``layerwise_oracle.update_envelope``): per element of the weights and every state vector

    |got - ref| <= c * (U * mag + ETA),    U = 2^-24,  ETA = 2^-150,

with ``mag`` the float64 sum of the magnitudes of the terms the rule adds up to that value, and for
the trust ratio a relative bound ``c_r * U * kappa``.  ``c`` and ``c_r`` count roundings on the
longest chain (a square counts its operand's error twice, a square root halves it):

  ratio     the squares and every partial sum are double: 16 fma per thread, 5 shuffle levels and
            3 block levels per tile, the fold over the tensor's tiles and the square root add up
            to < 2^-40 relative, far below U.  What remains is fp32: LARS g^ = g * scale (1),
            eta = 1e-3f (1), wd (1), the final rounding of the ratio (1): c_r = 4, doubled to 8.
            LAMB: ||u|| carries u's own error (below, about 18 U relative to mag(u)), so the
            ratio is held to c_r = 24 times kappa = ||mag(u)|| / ||u||.
  LARS 16   d: g^ 1, wd 1, fma 1, ratio c_r, r * (..) 1;  buffer: mu 1, fma 1;  weights: lr 1, fma 1.
  LAMB 24   K2's Adam chain without the L2 term: g^ 1;  exp_avg 3;  exp_avg_sq 2*1 + 5;  u: m * inv_bc1
            2, sqrt(v) and / bc2_sqrt 5 + 3, + eps 2, / 1, lam, fma 2 (about 18);  weights: lr * r
            (2 + the ratio's c_r * kappa, carried as kappa * |u| in mag), fma 1.

The data keep |g| in [0.5, 2) * scale and |w| <= 3 with wd <= 1e-2, as the K2 tests do.  The
learning rates (LARS 5, LAMB 1e-2) make one step move a weight by about 1e-3 of its value, so a
dropped weight-decay term (1e-2 of the step) is far outside the envelope.

Known differences from float64:
  * LAMB at |g| ~ 1e30: (1-beta2) * g^2 overflows fp32, so exp_avg_sq is +inf and u is lam * w
    (ratio 1/wd, or 1 with wd = 0), exactly as fp32 torch computes it; that edge is compared with
    ``LayerwiseTorch`` in fp32.
  * exp_avg uses the lerp formula for weight < 0.5 only (beta1 = 0.9), as in K2.
"""
import json
import os
import subprocess
import sys

import pytest
import torch

import frl_b200  # noqa: F401
from frl_b200 import _native, fused_optim
from frl_b200.arena import ParamArena
from frl_b200.multi_tensor import GradSegTable
from frl_b200.types import Precision
from layerwise_oracle import BETAS, LAMB_EPS, check_update
from test_gpu_optim_paths import _grad, _weights, assert_shadow

pytestmark = pytest.mark.gpu
DEV = "cuda"

ADAPTED, CLIPPED = _native.LW_ADAPTED, _native.LW_CLIPPED
FLAG_COMBOS = (ADAPTED | CLIPPED, ADAPTED, CLIPPED, 0)
PLACES = ("arena_f32", "f32", "arena_bf16", "bf16")   # where a listed slot's gradient lies
SCALE = 0.375                                         # grad_scale (x clip coefficient) by value
LR = {"lars": 5.0, "lamb": 1e-2}
LR_SCALE = (1.0, 0.6, 0.3, 0.8, 0.45)                 # lr of consecutive steps
# variant -> (mode, momentum, first step t)
VARIANTS = {"lars": ("lars", 0.0, 1), "lars_momentum": ("lars", 0.9, 1), "lamb": ("lamb", 0.0, 1),
            "lamb_late": ("lamb", 0.0, 10 ** 6)}
RATIO_GUARD = -3.5                                    # ratio entries past n_segs


class _Slot:
    def __init__(self, index, offset, numel):
        self.index, self.offset, self.numel = index, offset, numel
        self.is_model = True

    @property
    def end(self):
        return self.offset + self.numel


def dyn_block(mode, lr, step):
    """The kernel's ``dyn`` layout: LARS [lr], LAMB [lr, 1/(1-beta1^t), sqrt(1-beta2^t)]."""
    vals = [lr] if mode == "lars" else [lr, 1.0 / (1.0 - BETAS[0] ** step), (1.0 - BETAS[1] ** step) ** 0.5]
    return torch.tensor(vals + [0.0] * (4 - len(vals)), dtype=torch.float32)


class _LwCase:
    """Arena-shaped master, state and shadow vectors with a K2-lw table over some of the slots
    (``layout``: (numel, listed)); each listed slot has its own flags and gradient place."""

    def __init__(self, variant, layout, flags, places, lp, seed):
        self.mode, self.mu, self.t0 = VARIANTS[variant]
        gen = self.gen = torch.Generator(device=DEV).manual_seed(seed)
        slots, off = [], 0
        for i, (n, listed) in enumerate(layout):
            slots.append((_Slot(i, off, n), listed))
            off = (off + n + 7) // 8 * 8
        self.total = total = off
        self.listed = [s for s, listed in slots if listed]
        self.flag_list = list(flags)
        self.flags = torch.tensor(self.flag_list, dtype=torch.int32, device=DEV)
        arena_g = {torch.float32: torch.zeros(total, device=DEV),
                   torch.bfloat16: torch.zeros(total, dtype=torch.bfloat16, device=DEV)}
        self.table = GradSegTable(self.listed, torch.device(DEV))
        self.grads = []
        for s, place in zip(self.listed, places):
            dt = torch.bfloat16 if place.endswith("bf16") else torch.float32
            t = arena_g[dt][s.offset:s.end] if place.startswith("arena") else torch.empty(s.numel, dtype=dt, device=DEV)
            self.table.point(s, t.data_ptr(), dt)
            self.grads.append(t)
        self.table.upload()
        n_segs = self.table.n_segs
        self.ratio = torch.full((n_segs + 2,), RATIO_GUARD, device=DEV)
        nbytes = _native.layerwise_scratch_bytes(self.table.n_tiles, n_segs)
        self.scratch = torch.zeros((nbytes + 15) // 16 * 4, dtype=torch.int32, device=DEV)
        cover = torch.zeros(total, dtype=torch.bool, device=DEV)
        data = torch.zeros(total, dtype=torch.bool, device=DEV)
        for s in self.listed:
            cover[s.offset:(s.end + 7) // 8 * 8] = True
            data[s.offset:s.end] = True
        self.pad, self.outside = cover & ~data, ~cover
        self.p = _weights(total, gen)
        if self.mode == "lars":        # a first step must ignore whatever the buffer holds
            self.states = [torch.randn(total, device=DEV, generator=gen) * 0.1] if self.mu else []
        elif self.t0 == 1:
            self.states = [torch.zeros(total, device=DEV), torch.zeros(total, device=DEV)]
        else:                          # mid-training moments
            self.states = [torch.randn(total, device=DEV, generator=gen) * 0.1,
                           torch.rand(total, device=DEV, generator=gen) * 0.01 + 1e-4]
        self.shadow = torch.randn(total, device=DEV, generator=gen).to(torch.bfloat16) if lp else None
        for v in self.vectors():
            v[self.pad] = 0            # arena padding is zero
        self.before = [v.clone() for v in self.vectors()]

    def vectors(self):
        return [v for v in [self.p, self.shadow] + self.states if v is not None]

    def scales(self, clipped):
        """Effective gradient scale of each segment: by value alone, or 0.5 x the coefficient 0.75
        on FRL_LW_CLIPPED segments."""
        return [SCALE if not clipped else 0.5 * (0.75 if f & CLIPPED else 1.0) for f in self.flag_list]

    def new_grads(self, scale=1.0):
        for t in self.grads:
            t.copy_(_grad(t.numel(), self.gen, scale))

    def launch(self, *, lr, step, wd, coef=None, dyn=None):
        gs, gs_dev = (SCALE, None) if coef is None else (0.5, coef)
        if self.mode == "lars":
            _native.lars_mt(self.p, self.states[0] if self.mu else None, self.shadow, self.table, self.flags,
                            self.ratio, self.scratch, lr=lr, mu=self.mu, wd=wd, grad_scale=gs,
                            grad_scale_dev=gs_dev, first_step=step == 1, dyn=dyn)
        else:
            _native.lamb_mt(self.p, self.states[0], self.states[1], self.shadow, self.table, self.flags,
                            self.ratio, self.scratch, lr=lr, beta1=BETAS[0], beta2=BETAS[1], eps=LAMB_EPS,
                            wd=wd, step=step, grad_scale=gs, grad_scale_dev=gs_dev, dyn=dyn)

    def step_and_check(self, *, lr, step, wd, clipped=False, dyn_wrong=False, what="", dtype=torch.float64):
        """One launch (with ``dyn`` and wrong by-value scalars if ``dyn_wrong``), then every listed
        tensor against float64, the shadow, the padding and the slots outside the table."""
        coef = torch.tensor([0.75], device=DEV) if clipped else None
        w0 = [self.p[s.offset:s.end].clone() for s in self.listed]
        s0 = [[v[s.offset:s.end].clone() for v in self.states] for s in self.listed]
        if dyn_wrong:
            dyn = dyn_block(self.mode, lr, step).to(DEV)
            self.launch(lr=123.0, step=step if self.mode == "lars" else step + 7, wd=wd, coef=coef, dyn=dyn)
        else:
            self.launch(lr=lr, step=step, wd=wd, coef=coef)
        ratios = self.ratio.cpu().tolist()
        for j, (s, sc) in enumerate(zip(self.listed, self.scales(clipped))):
            check_update(self.mode, self.p[s.offset:s.end], [v[s.offset:s.end] for v in self.states], ratios[j],
                         w0[j], self.grads[j].double() * sc, s0[j], adapted=bool(self.flag_list[j] & ADAPTED),
                         lr=lr, mu=self.mu, wd=wd, step=step, what="%s seg %d (n=%d)" % (what, j, s.numel),
                         dtype=dtype)
            if self.shadow is not None:
                assert_shadow(self.shadow[s.offset:s.end], self.p[s.offset:s.end], "%s seg %d" % (what, j))
        assert ratios[self.table.n_segs:] == [RATIO_GUARD] * 2, what + ": ratio written past n_segs"
        self.assert_pad_and_outside(what)
        return ratios

    def assert_pad_and_outside(self, what):
        for v, b in zip(self.vectors(), self.before):
            bits = torch.int16 if v.dtype == torch.bfloat16 else torch.int32
            assert torch.all(v[self.pad] == 0), what + ": padding written"
            assert torch.equal(v[self.outside].view(bits), b[self.outside].view(bits)), \
                what + ": slot outside the table written"


# ---- every instantiation and runtime branch ------------------------------------------------------

# listed: 1, 3, 4, 5 (scalar tails only), 4095 / 4096 / 4097 (kTileElems = 4096) and three tiles + 3,
# interleaved with slots the table leaves alone
LAYOUT = [(7, False), (1, True), (3, True), (4, True), (11, False), (5, True), (4095, True), (4096, True),
          (4100, False), (4097, True), (3 * 4096 + 3, True), (13, False)]


@pytest.mark.parametrize("rot", range(4))
@pytest.mark.parametrize("lp", [False, True], ids=["no_shadow", "shadow"])
@pytest.mark.parametrize("wd", [0.0, 1e-2], ids=["wd0", "wd"])
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_table_update_matches_float64(variant, wd, lp, rot):
    """Each rotation moves every flag combination (adapted x clipped) across the sizes and the
    gradient places (fp32 / bf16, in the arena / outside it).  Step 1: grad_scale by value; step 2:
    x grad_scale_dev, and ``dyn`` with deliberately wrong by-value lr and step; step 3: x
    grad_scale_dev, ``dyn`` NULL."""
    n = sum(listed for _, listed in LAYOUT)
    case = _LwCase(variant, LAYOUT, [FLAG_COMBOS[(j + rot) % 4] for j in range(n)],
                   [PLACES[j % 4] for j in range(n)], lp, seed=100 + rot)
    for k in range(3):
        step = case.t0 + k
        case.new_grads()
        case.step_and_check(lr=LR[case.mode] * LR_SCALE[k], step=step, wd=wd, clipped=k > 0, dyn_wrong=k == 1,
                            what="step %d" % step)


def test_more_tiles_and_segments_than_one_resident_wave():
    """One segment with more tiles than any resident grid holds (SMs x 8 CTAs), and a table of more
    segments than that, so a CTA folds several segments on later grid-stride iterations."""
    wave = _native.lib().frl_device_sm_count() * 8
    sizes = [(wave + 3) * 4096 + 5] + [1 + (37 * k) % 4100 for k in range(wave + 64)]
    layout = [(n, True) for n in sizes]
    for variant in ("lars_momentum", "lamb"):
        case = _LwCase(variant, layout, [FLAG_COMBOS[j % 4] for j in range(len(sizes))],
                       [PLACES[j % 4] for j in range(len(sizes))], True, seed=5)
        assert case.table.n_tiles > 2 * wave and case.table.n_segs > wave
        for k in range(2):
            case.new_grads()
            case.step_and_check(lr=LR[case.mode] * LR_SCALE[k], step=1 + k, wd=1e-2, clipped=k == 1,
                                dyn_wrong=k == 1, what="%s step %d" % (variant, 1 + k))


# ---- ratio 1 and numeric edges --------------------------------------------------------------------

EDGE_LAYOUT = [(4096 + 7, True), (3, True), (4097, True), (5, True)]
EDGE_FLAGS = [ADAPTED | CLIPPED, 0, ADAPTED, ADAPTED | CLIPPED]
EDGE_PLACES = ["arena_f32", "f32", "bf16", "arena_bf16"]


@pytest.mark.parametrize("wd", [0.0, 1e-2], ids=["wd0", "wd"])
@pytest.mark.parametrize("variant", ["lars_momentum", "lamb"])
def test_ratio_is_exactly_one_where_the_rule_says(variant, wd):
    """Not adapted; ||w|| = 0; ||g^|| = 0 (LARS) or, with zero state, zero gradient and wd = 0,
    ||u|| = 0 (LAMB): ratio exactly 1.0, and every tensor still matches float64."""
    case = _LwCase(variant, EDGE_LAYOUT, EDGE_FLAGS, EDGE_PLACES, True, seed=9)
    case.new_grads()
    s0, s2 = case.listed[0], case.listed[2]
    case.grads[0].zero_()                             # tensor 0: zero gradient
    case.p[s2.offset:s2.end] = 0                      # tensor 2: zero weights
    ratios = case.step_and_check(lr=LR[case.mode], step=1, wd=wd, what="ratio 1")
    assert ratios[1] == 1.0 and ratios[2] == 1.0
    if case.mode == "lars" or wd == 0:
        assert ratios[0] == 1.0
    assert ratios[3] != 1.0
    # zero gradient: only the weight-decay term moves the weights
    assert bool((case.p[s0.offset:s0.end] == case.before[0][s0.offset:s0.end]).all()) == (wd == 0)


SCALES = [1e-30, 1e-20, 1.0, 1e17, 1e20, 1e30]


@pytest.mark.parametrize("scale", SCALES)
@pytest.mark.parametrize("wd", [0.0, 1e-2], ids=["wd0", "wd"])
@pytest.mark.parametrize("variant", ["lars", "lars_momentum", "lamb"])
def test_gradient_scale_edges_match_float64(variant, wd, scale):
    """LARS is invariant to the gradient's scale, and its ratio, norms aside, is an ordinary float
    at every scale here: squares of |g| ~ 1e20 overflow fp32, of |g| ~ 1e-20 are subnormal and of
    |g| ~ 1e-30 underflow to zero.  LAMB's u ~ 1e-25 at |g| ~ 1e-30 has squares that underflow fp32
    too.  Two steps each."""
    case = _LwCase(variant, EDGE_LAYOUT, EDGE_FLAGS, EDGE_PLACES, True, seed=11)
    dtype = torch.float32 if case.mode == "lamb" and scale >= 1e30 else torch.float64
    for k in range(2):
        case.new_grads(scale)
        case.step_and_check(lr=LR[case.mode] * LR_SCALE[k], step=1 + k, wd=wd, what="|g|~%g step %d" % (scale, 1 + k),
                            dtype=dtype)
    if dtype == torch.float32:
        assert all(bool(torch.isposinf(case.states[1][s.offset:s.end]).all()) for s in case.listed)


@pytest.mark.parametrize("bad", [float("nan"), float("inf"), float("-inf")], ids=["nan", "inf", "-inf"])
@pytest.mark.parametrize("variant", ["lars_momentum", "lamb"])
def test_nonfinite_gradient_stays_in_its_tensor(variant, bad):
    """One non-finite gradient element: that tensor's weights go non-finite (where float64 puts the
    non-finite values), every other tensor still matches float64."""
    case = _LwCase(variant, EDGE_LAYOUT, EDGE_FLAGS, EDGE_PLACES, True, seed=13)
    case.new_grads()
    case.grads[2][2049] = bad
    case.step_and_check(lr=LR[case.mode], step=1, wd=1e-2, what="g[2049] = %r" % bad)
    for j, s in enumerate(case.listed):
        finite = bool(torch.isfinite(case.p[s.offset:s.end]).all())
        assert finite == (j != 2), (j, finite)


# ---- CUDA graphs -------------------------------------------------------------------------------

@pytest.mark.parametrize("variant", ["lars_momentum", "lamb"])
def test_graph_replay_with_dyn_equals_eager_launches(variant):
    """Both launches captured once with ``dyn``, replayed over 5 steps while lr (and LAMB's bias
    corrections) change in the device block: bit for bit the eager launches."""
    n = sum(listed for _, listed in LAYOUT)
    flags, places = [FLAG_COMBOS[j % 4] for j in range(n)], [PLACES[j % 4] for j in range(n)]
    eager, replayed = (_LwCase(variant, LAYOUT, flags, places, True, seed=17) for _ in range(2))
    replayed.table, replayed.grads = eager.table, eager.grads     # both read the same gradients
    mode = eager.mode
    coef = torch.tensor([0.75], device=DEV)
    graph_dyn = torch.zeros(4, device=DEV)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):                     # LARS's first_step is by value: capture a later step
        replayed.launch(lr=1.0, step=2 if mode == "lars" else 1, wd=1e-2, coef=coef, dyn=graph_dyn)
    for step in range(1, 6):
        lr = LR[mode] * LR_SCALE[step - 1]
        eager.new_grads()
        eager.launch(lr=lr, step=step, wd=1e-2, coef=coef)
        if mode == "lars" and step == 1:
            replayed.launch(lr=lr, step=step, wd=1e-2, coef=coef)
        else:
            graph_dyn.copy_(dyn_block(mode, lr, step))
            graph.replay()
        torch.cuda.synchronize()
        for a, b in zip(eager.vectors() + [eager.ratio], replayed.vectors() + [replayed.ratio]):
            assert torch.equal(a, b), "step %d" % step


# ---- optimizer classes ---------------------------------------------------------------------------

@pytest.mark.parametrize("precision", [Precision.FP32, Precision.BF16])
@pytest.mark.parametrize("mode", ["lars", "lamb"])
def test_optimizer_classes_match_float64(mode, precision):
    """``FusedLars`` / ``FusedLamb`` through ``apply_table`` with device-resident scalars and lr
    changing every step, 5 steps, clip coefficient on model parameters only: every slot against
    float64 from the optimizer's own state, ratios from ``last_ratios``."""
    gen = torch.Generator(device=DEV).manual_seed(23)
    model = [torch.nn.Parameter(_weights(33 * 17, gen).view(33, 17)), torch.nn.Parameter(_weights(5, gen)),
             torch.nn.Parameter(_weights(4099 * 2, gen).view(2, 4099))]
    crit = [torch.nn.Parameter(_weights(7, gen)), torch.nn.Parameter(_weights(6, gen).view(2, 3))]
    arena = ParamArena(model, crit, device=DEV, precision=precision)
    if mode == "lars":
        opt = fused_optim.FusedLars(arena, lr=LR[mode], momentum=0.9, weight_decay=1e-2)
        names, mu = ("momentum_buffer",), 0.9
    else:
        opt = fused_optim.FusedLamb(arena, lr=LR[mode], betas=BETAS, eps=LAMB_EPS, weight_decay=1e-2)
        names, mu = ("exp_avg", "exp_avg_sq"), 0.0
    opt.enable_dynamic_scalars()
    slots = list(arena.slots)
    table = GradSegTable(slots, arena.device)
    g = arena.grad
    for s in slots:
        table.point(s, g.data_ptr() + s.offset * g.element_size(), g.dtype)
    table.upload()
    coef = torch.tensor([0.75], device=DEV)
    for k in range(5):
        step = k + 1
        opt.hyper["lr"] = lr = LR[mode] * LR_SCALE[k]
        for s in slots:
            g[s.offset:s.end].copy_(_grad(s.numel, gen))
        w0 = [arena.master[s.offset:s.end].clone() for s in slots]
        s0 = [[opt._vec[n][s.offset:s.end].clone() if n in opt._vec else torch.zeros(s.numel, device=DEV)
               for n in names] for s in slots]
        opt.begin_step()
        opt.apply_table(table, grad_scale=0.5, clip_coef_dev=coef)
        opt.end_step()
        ratios = opt.last_ratios(table).cpu().tolist()
        for j, s in enumerate(slots):
            check_update(mode, arena.master[s.offset:s.end], [opt._vec[n][s.offset:s.end] for n in names], ratios[j],
                         w0[j], g[s.offset:s.end].double() * 0.5 * (0.75 if s.is_model else 1.0), s0[j],
                         adapted=fused_optim.is_adapted(s), lr=lr, mu=mu, wd=1e-2, step=step,
                         what="step %d slot %d %s" % (step, s.index, s.shape))
            if arena.lp is not None and s.is_model:
                assert_shadow(arena.lp[s.offset:s.end], arena.master[s.offset:s.end], "step %d" % step)


# ---- every instantiation is launched ---------------------------------------------------------------

LW_INSTANTIATIONS = sorted(
    ["lw_stats_kernel:false,frl::LarsParams", "lw_stats_kernel:true,frl::LambParams"]
    + ["lw_apply_kernel:%s,%s,frl::%s" % (lamb, lp, p) for lamb, p in (("false", "LarsParams"), ("true", "LambParams"))
       for lp in ("false", "true")])


def test_every_layerwise_instantiation_is_launched():
    """All six instantiations launch, each update checked against float64.  The profiler runs in a
    process of its own (tests/run_layerwise_instantiations.py), so this process never starts a
    profiling session: one that ended here would hide kernels from later sessions."""
    script = os.path.join(os.path.dirname(os.path.abspath(__file__)), "run_layerwise_instantiations.py")
    res = subprocess.run([sys.executable, script], capture_output=True, text=True, timeout=600)
    assert res.returncode == 0 and "LAYERWISE_INSTANTIATIONS_OK" in res.stdout, res.stdout[-3000:] + res.stderr[-3000:]
    line = [ln for ln in res.stdout.splitlines() if ln.startswith("INSTANTIATIONS ")][-1]
    seen = json.loads(line[len("INSTANTIATIONS "):])
    assert seen == LW_INSTANTIATIONS and len(seen) == 6, seen
