"""The fused optimizer update (K2 ``update_kernel``, K2-mt ``update_mt_kernel``) on every
instantiation against float64 ``torch.optim`` on the same GPU.

Reference.  ``torch.optim.SGD`` / ``Adam`` / ``RMSprop`` with ``foreach=False`` on float64 copies,
fed exactly the gradient the kernel reads: bf16-rounded when the gradient is bf16, times
``grad_scale`` and the device clip coefficient.  Every step starts the reference from the
kernel's own fp32 state (master weights and every state vector), so one comparison covers one
update and the bound below does not have to grow with the step count.

Tolerance: an fp32 rounding envelope, per element of the weights and of every state vector,

    |got - ref| <= c * (U * mag + ETA),    U = 2^-24,  ETA = 2^-150,

U bounds the relative error of one rounding to fp32, ETA its absolute error in the subnormal
range (squares of |g| ~ 1e-30 underflow to zero).  ``mag`` is the float64 sum of the magnitudes of
the terms the rule adds up to that value (``_envelope``), so a sum that cancels is held to the
error of its parts; for the weights it is |ref| + lr * (magnitude of the step's update).  ``c``
counts the fp32 roundings on the rule's longest chain, the fp32 conversions of the
hyper-parameters included (a square counts its operand's error twice, a square root halves it):

    SGD      8   g*scale, wd*p + g, wd -> 3;  (1-dampening)*d, mu*buf + .., mu, 1-dampening -> 4;
                 -lr*buf + p, lr -> 2, shared with the buffer's last rounding
    RMSprop 16   gradient 3;  square_avg 2*3 + 4 = 10, halved by sqrt -> 5, sqrt, +eps -> 2;
                 g / avg 1;  mu*buf + upd, mu 2;  -lr*upd + p, lr 2;  rounded up
    Adam    24   gradient 3;  exp_avg: g - m, 1-beta1, fma 3;  exp_avg_sq 2*3 + 4 = 10, halved 5,
                 sqrt, / bc2_sqrt, bc2_sqrt, +eps 4;  m / denom 1;  step_size, fma 2;
                 with headroom for |m| / mag(m) < 1 and weight-decay terms in the squares

The data keep |g| >= 0.19 > wd * |p| (|p| <= 3, wd <= 1e-2), so weight decay never cancels the
gradient: near such a cancellation the first Adam / RMSprop step divides a rounding error by
|g| itself, and no fp32 envelope holds there.

Second reference: ``torch.optim`` in its default form (foreach, fp32) on the same GPU, from the
same fp32 state and the same fp32 gradient, 4 steps of 2^20 + 3 elements, weights and every
state vector.  Measured on an H100 80GB HBM3 (SXM, 700 W power limit) with torch 2.11:

    rule               elements differing   largest distance   in units of U * mag
    SGD                        0                   0 ulps              0     bit-identical
    SGD, momentum        1360310              773494 ulps              2.000
    Adam                  771745                6554 ulps              3.331
    Adam, amsgrad        1534919                6554 ulps              3.331
    RMSprop               821695               41943 ulps              3.323
    RMSprop, momentum    2148194              134626 ulps              3.971

The ulp counts come from values that cancel to far below their terms (a weight crossing zero);
measured against the magnitude of the terms, as the envelope measures, torch's fp32 result is
within 4 roundings of the kernel's.  SGD with momentum differs because torch rounds
``buf * mu`` before adding the gradient where the kernel uses one fmaf.  The test pins bit
equality for SGD and these distances (rounded up to a half unit) for the others.

Known differences from float64 torch:
  * squares that overflow fp32 (|g| ~ 1e30): exp_avg_sq / square_avg become +inf and the step
    becomes 0 (Adam) or 0 / the momentum's decay (RMSprop), exactly as fp32 torch.optim does; the
    edge test compares those cases with fp32 torch.
  * ``exp_avg.lerp_`` always uses the ``weight < 0.5`` formula (beta1 > 0.5); torch switches to
    ``end - (end - self) * (1 - weight)`` for beta1 <= 0.5.  A rounding difference only.
"""
import math
import tempfile

import pytest
import torch

import frl_b200  # noqa: F401
from frl_b200 import _native, fused_optim, synthetic
from frl_b200.arena import ParamArena
from frl_b200.multi_tensor import GradSegTable
from frl_b200.solver import Solver, SolverWorkerArgs
from frl_b200.types import Device, OptAlgorithm, OptimOpts, Precision

pytestmark = pytest.mark.gpu
DEV = "cuda"

U = 2.0 ** -24
ETA = 2.0 ** -150
C = {"sgd": 8, "rmsprop": 16, "adam": 24}

# one entry per state count of each rule: (rule, hyper-parameters besides lr and weight decay)
VARIANTS = {
    "sgd": ("sgd", dict(momentum=0.0, dampening=0.0)),
    "sgd_momentum": ("sgd", dict(momentum=0.9, dampening=0.1)),
    "adam": ("adam", dict(betas=(0.9, 0.999), eps=1e-8, amsgrad=False)),
    "adam_amsgrad": ("adam", dict(betas=(0.9, 0.999), eps=1e-8, amsgrad=True)),
    "rmsprop": ("rmsprop", dict(alpha=0.99, eps=1e-8, momentum=0.0)),
    "rmsprop_momentum": ("rmsprop", dict(alpha=0.99, eps=1e-8, momentum=0.9)),
}
STATE_NAMES = {"sgd": (), "sgd_momentum": ("momentum_buffer",), "adam": ("exp_avg", "exp_avg_sq"),
               "adam_amsgrad": ("exp_avg", "exp_avg_sq", "max_exp_avg_sq"), "rmsprop": ("square_avg",),
               "rmsprop_momentum": ("square_avg", "momentum_buffer")}
NONNEG = {"exp_avg_sq", "max_exp_avg_sq", "square_avg"}
BASE_LR = {"sgd": 0.05, "adam": 1e-2, "rmsprop": 1e-2}
LR_SCALE = (1.0, 0.6, 0.3, 0.8, 0.45)            # lr of steps 1..5
SCALE = 0.375                                    # grad_scale (x clip coefficient) of every test

# largest |kernel - fp32 torch.optim (foreach)| / (U * mag + ETA) over weights and states, as
# measured (module docstring); 0 means bit-identical
DISTANCE_TO_FP32_TORCH = {"sgd": 0.0, "sgd_momentum": 2.5, "adam": 3.5, "adam_amsgrad": 3.5, "rmsprop": 3.5,
                          "rmsprop_momentum": 4.0}


# ---- kernel entry points ---------------------------------------------------------------------------

def _kernel_kw(variant, lr, wd, step):
    rule, hp = VARIANTS[variant]
    if rule == "sgd":
        return dict(lr=lr, mu=hp["momentum"], dampening=hp["dampening"], wd=wd, first_step=step == 1)
    if rule == "adam":
        return dict(lr=lr, beta1=hp["betas"][0], beta2=hp["betas"][1], eps=hp["eps"], wd=wd, step=step)
    return dict(lr=lr, alpha=hp["alpha"], eps=hp["eps"], wd=wd, mu=hp["momentum"])


def _state_args(variant, states):
    """The kernel's positional state arguments (None where the instantiation has no state)."""
    s = list(states) + [None] * 3
    return s[:{"sgd": 1, "adam": 3, "rmsprop": 2}[VARIANTS[variant][0]]]


def _scale_args(coef):
    """grad_scale and grad_scale_dev with the product SCALE: by value alone, or 0.5 x coefficient."""
    return (SCALE, None) if coef is None else (0.5, coef)


def launch_flat(variant, p, g, states, lp, n, *, lr, wd, step, coef=None, dyn=None):
    fn = {"sgd": _native.sgd_momentum, "adam": _native.adam, "rmsprop": _native.rmsprop}[VARIANTS[variant][0]]
    gs, gs_dev = _scale_args(coef)
    fn(p, g, *_state_args(variant, states), lp, n, grad_scale=gs, grad_scale_dev=gs_dev, dyn=dyn,
       **_kernel_kw(variant, lr, wd, step))


def launch_mt(variant, p, states, lp, table, *, lr, wd, step, coef=None, dyn=None):
    fn = {"sgd": _native.sgd_momentum_mt, "adam": _native.adam_mt,
          "rmsprop": _native.rmsprop_mt}[VARIANTS[variant][0]]
    gs, gs_dev = _scale_args(coef)
    fn(p, *_state_args(variant, states), lp, table, grad_scale=gs, grad_scale_dev=gs_dev, dyn=dyn,
       **_kernel_kw(variant, lr, wd, step))


def dyn_block(variant, lr, step):
    """The kernel's ``dyn`` layout (what ``FusedArenaOptimizer._dyn_values`` uploads)."""
    rule, hp = VARIANTS[variant]
    vals = [lr]
    if rule == "adam":
        b1, b2 = hp["betas"]
        vals = [-(lr / (1.0 - b1 ** step)), (1.0 - b2 ** step) ** 0.5]
    return torch.tensor(vals + [0.0] * (4 - len(vals)), dtype=torch.float32)


# ---- reference and envelope ------------------------------------------------------------------------

def _torch_optimizer(variant, params, lr, wd, foreach=False):
    rule, hp = VARIANTS[variant]
    cls = {"sgd": torch.optim.SGD, "adam": torch.optim.Adam, "rmsprop": torch.optim.RMSprop}[rule]
    return cls(params, lr=lr, weight_decay=wd, foreach=foreach, **hp)


def reference_step(variant, p, g, states, *, lr, wd, step, dtype=torch.float64, foreach=False):
    """One ``torch.optim`` step in ``dtype`` from the state (p, states) with gradient ``g``."""
    rule = VARIANTS[variant][0]
    param = torch.nn.Parameter(p.to(dtype, copy=True))
    opt = _torch_optimizer(variant, [param], lr, wd, foreach)
    if not (rule == "sgd" and step == 1):          # SGD's first step starts its buffer from g
        st = opt.state[param]
        for name, s in zip(STATE_NAMES[variant], states):
            st[name] = s.to(dtype, copy=True)
        if rule != "sgd":
            st["step"] = torch.tensor(float(step - 1))
    param.grad = g.to(dtype)
    opt.step()
    return param.detach(), [opt.state[param][name] for name in STATE_NAMES[variant]]


def _envelope(variant, p0, g, s0, ref_p, ref_s, *, lr, wd, step):
    """c * (U * mag + ETA) for the weights and every state vector (float64)."""
    rule, hp = VARIANTS[variant]
    mag_g = g.abs() + wd * p0.abs()
    if rule == "sgd":
        upd, mags = mag_g, []
        if hp["momentum"]:
            if step > 1:
                upd = hp["momentum"] * s0[0].abs() + (1 - hp["dampening"]) * mag_g
            mags = [upd]
        step_mag = lr * upd
    elif rule == "adam":
        b1, b2 = hp["betas"]
        mag_m = s0[0].abs() + (1 - b1) * (mag_g + s0[0].abs())
        mag_v = b2 * s0[1].abs() + (1 - b2) * mag_g * mag_g
        mags = [mag_m, mag_v] + ([torch.maximum(s0[2].abs(), mag_v)] if hp["amsgrad"] else [])
        denom = ref_s[-1].sqrt() / math.sqrt(1 - b2 ** step) + hp["eps"]
        step_mag = lr / (1 - b1 ** step) * mag_m / denom
    else:
        avg = ref_s[0].sqrt() + hp["eps"]
        mags = [hp["alpha"] * s0[0].abs() + (1 - hp["alpha"]) * mag_g * mag_g]
        upd = mag_g / avg
        if hp["momentum"]:
            upd = hp["momentum"] * s0[1].abs() + upd
            mags.append(upd)
        step_mag = lr * upd
    c = C[rule]
    return [c * (U * (ref_p.abs() + step_mag) + ETA)] + [c * (U * m + ETA) for m in mags]


def assert_within(got, ref, bound, what):
    """Non-finite values exactly where the reference has them; finite ones inside the bound."""
    got = got.double()
    for kind in (torch.isnan, torch.isposinf, torch.isneginf):
        diff = kind(got) != kind(ref)
        assert not diff.any(), "%s: %s differs at %s" % (what, kind.__name__, diff.nonzero().flatten()[:8].tolist())
    out = torch.isfinite(ref) & ~((got - ref).abs() <= bound)
    if out.any():
        i = int(out.nonzero()[0])
        raise AssertionError("%s: %d elements outside the envelope, first [%d]: got %r ref %r bound %r"
                             % (what, int(out.sum()), i, got[i].item(), ref[i].item(), bound[i].item()))


def check_step(variant, got_p, got_s, p0, g, s0, *, lr, wd, step, what, dtype=torch.float64):
    """The kernel's update (got_*) from (p0, s0) with effective gradient g against torch.optim in
    ``dtype`` (fp32 only where fp32 itself overflows; both sides then carry their own error)."""
    ref_p, ref_s = reference_step(variant, p0, g, s0, lr=lr, wd=wd, step=step, dtype=dtype)
    ref_p, ref_s = ref_p.double(), [s.double() for s in ref_s]
    bounds = _envelope(variant, p0.double(), g.double(), [s.double() for s in s0], ref_p, ref_s,
                       lr=lr, wd=wd, step=step)
    if dtype != torch.float64:
        bounds = [2 * b for b in bounds]
    assert_within(got_p, ref_p, bounds[0], what + " weights")
    for name, got, ref, b in zip(STATE_NAMES[variant], got_s, ref_s, bounds[1:]):
        assert_within(got, ref, b, "%s %s" % (what, name))


def assert_shadow(lp, p, what):
    """The bf16 shadow is RNE-bf16 of the master, bit for bit (NaN where the master is NaN)."""
    want = p.to(torch.bfloat16)
    nan = torch.isnan(p)
    assert torch.equal(torch.isnan(lp), nan), what + " shadow NaN"
    assert torch.equal(lp[~nan].view(torch.int16), want[~nan].view(torch.int16)), what + " shadow"


# ---- data ------------------------------------------------------------------------------------------

def _grad(n, gen, scale=1.0):
    """|g| in [0.5, 2) * scale, random sign."""
    mag = torch.rand(n, device=DEV, generator=gen, dtype=torch.float64) * 1.5 + 0.5
    sign = torch.randint(0, 2, (n,), device=DEV, generator=gen).double() * 2 - 1
    return (mag * sign * scale).float()


def _weights(n, gen):
    return torch.randn(n, device=DEV, generator=gen).clamp_(-3, 3)


def _state_values(name, n, gen):
    """A mid-training state vector (non-negative where the rule keeps squares)."""
    if name in NONNEG:
        return torch.rand(n, device=DEV, generator=gen) * 0.01 + 1e-4
    return torch.randn(n, device=DEV, generator=gen) * 0.1


PAD = 8                                           # keeps the slice 16-byte aligned in bf16 and fp32
SENTINEL = -7.25


def _padded(n, dtype, fill):
    buf = torch.full((n + 2 * PAD,), fill, dtype=dtype, device=DEV)
    return buf, buf[PAD:PAD + n]


def _assert_sentinels(buf, n, what):
    edges = torch.cat([buf[:PAD], buf[PAD + n:]]).float()
    assert torch.all(edges == SENTINEL), what + ": write outside the launched range"


def _three_waves():
    """Elements of three resident waves of the flat kernel: SMs x 8 CTAs/SM x one 4096-element tile each."""
    return 3 * _native.lib().frl_device_sm_count() * 8 * 4096 + 3


# ---- flat K2: every instantiation -------------------------------------------------------------------

# scalar tail only; one vector; one tile; one tile + 1..3; a partial second tile; three waves
LENGTHS = [1, 2, 3, 4, 4096, 4097, 4098, 4099, 4096 + 2500 + 2, "three_waves"]


@pytest.mark.parametrize("length", LENGTHS)
@pytest.mark.parametrize("lp", [False, True], ids=["no_shadow", "shadow"])
@pytest.mark.parametrize("gdt", [torch.float32, torch.bfloat16], ids=["g_f32", "g_bf16"])
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_flat_update_matches_float64_torch_optim(variant, gdt, lp, length):
    i = LENGTHS.index(length)
    n = _three_waves() if length == "three_waves" else length
    wd = (0.0, 1e-2)[i % 2]
    coef = torch.tensor([0.75], device=DEV) if (i // 2) % 2 else None
    rule = VARIANTS[variant][0]
    gen = torch.Generator(device=DEV).manual_seed(1000 + i)
    pbuf, p = _padded(n, torch.float32, SENTINEL)
    p.copy_(_weights(n, gen))
    sbufs = [_padded(n, torch.float32, SENTINEL) for _ in STATE_NAMES[variant]]
    states = [s for _, s in sbufs]
    for name, s in zip(STATE_NAMES[variant], states):
        # SGD's first step must ignore whatever its buffer holds; the other rules start from zero
        s.copy_(_state_values(name, n, gen) if rule == "sgd" else torch.zeros_like(s))
    lbuf, shadow = _padded(n, torch.bfloat16, SENTINEL) if lp else (None, None)
    gbuf, g = _padded(n, gdt, float("nan"))
    for step in range(1, 5):
        lr = BASE_LR[rule] * LR_SCALE[step - 1]
        g.copy_(_grad(n, gen))
        p0, s0 = p.clone(), [s.clone() for s in states]
        launch_flat(variant, p, g, states, shadow, n, lr=lr, wd=wd, step=step, coef=coef)
        check_step(variant, p, states, p0, g.double() * SCALE, s0, lr=lr, wd=wd, step=step,
                   what="n=%d step %d" % (n, step))
        if lp:
            assert_shadow(shadow, p, "step %d" % step)
    for name, buf in [("weights", pbuf), ("shadow", lbuf)] + list(zip(STATE_NAMES[variant], (b for b, _ in sbufs))):
        if buf is not None:
            _assert_sentinels(buf, n, name)


# ---- flat K2: numeric edges -------------------------------------------------------------------------

EDGE_N = 4096 + 7                                 # one tile and a 3-element scalar tail
NONFINITE = {0: float("nan"), 1: float("inf"), 2049: float("-inf"), 4100: float("inf"),
             4101: float("-inf"), 4102: float("nan")}
EDGES = ([(v, e) for v in VARIANTS for e in ("zero", "zero_decay", "tiny", "huge", "nonfinite")]
         + [(v, e) for v in ("adam", "adam_amsgrad") for e in ("step_1", "step_1e6")]
         + [("adam_amsgrad", "vmax_holds")])


@pytest.mark.parametrize("variant,edge", EDGES)
def test_flat_update_edges_match_float64_torch_optim(variant, edge):
    rule = VARIANTS[variant][0]
    n = EDGE_N
    gen = torch.Generator(device=DEV).manual_seed(7)
    p = _weights(n, gen)
    names = STATE_NAMES[variant]
    states = [_state_values(name, n, gen) for name in names]
    shadow = torch.empty(n, dtype=torch.bfloat16, device=DEV)
    first = {"step_1": 1, "step_1e6": 10 ** 6}.get(edge, 3)
    if edge in ("step_1", "vmax_holds"):
        first = 1
        for s in states:
            s.zero_()
    wd = 1e-2 if edge in ("zero_decay", "nonfinite", "step_1", "step_1e6") else 0.0
    # fp32 squares of |g| ~ 1e30 overflow to +inf in the kernel and in fp32 torch alike
    dtype = torch.float32 if (edge == "huge" and rule != "sgd") else torch.float64
    scales = {"tiny": 1e-30, "huge": 1e30}
    for k in range(5 if edge == "vmax_holds" else 2):
        step = first + k
        lr = BASE_LR[rule] * LR_SCALE[k]
        if edge in ("zero", "zero_decay"):
            g = torch.zeros(n, device=DEV)
        elif edge == "vmax_holds":                # large gradients, then small: v falls below vmax
            g = _grad(n, gen, 1.0 if k < 2 else 1e-2)
        else:
            g = _grad(n, gen, scales.get(edge) or 1.0)
        if edge == "nonfinite" and k == 0:
            for j, x in NONFINITE.items():
                g[j] = x
        p0, s0 = p.clone(), [s.clone() for s in states]
        launch_flat(variant, p, g, states, shadow, n, lr=lr, wd=wd, step=step)
        check_step(variant, p, states, p0, g.double() * SCALE, s0, lr=lr, wd=wd, step=step,
                   what="%s step %d" % (edge, step), dtype=dtype)
        assert_shadow(shadow, p, "%s step %d" % (edge, step))
    if edge == "huge" and rule != "sgd":
        assert torch.isposinf(states[1 if rule == "adam" else 0]).all()
    if edge == "vmax_holds":
        assert bool((states[2] > states[1]).all())
    if edge == "nonfinite":
        bad = torch.zeros(n, dtype=torch.bool, device=DEV)
        bad[list(NONFINITE)] = True
        assert bool(torch.isfinite(p[~bad]).all()) and not bool(torch.isfinite(p[bad]).any())


# ---- K2-mt ------------------------------------------------------------------------------------------

class _Slot:
    def __init__(self, index, offset, numel):
        self.index, self.offset, self.numel = index, offset, numel

    @property
    def end(self):
        return self.offset + self.numel


# (numel, listed in the table): the listed sizes interleaved with slots the table leaves alone
MT_LAYOUT = [(7, False), (1, True), (2, True), (11, False), (3, True), (5, True), (4096, True),
             (4100, False), (4097, True), (3 * 4096 + 3, True), (13, False)]
PLACES = ("arena_f32", "f32", "arena_bf16", "bf16")   # where each listed slot's gradient lies


class _MtCase:
    """Arena vectors with a segment table over some of its slots; gradients fp32 and bf16, in the
    arena's gradient vectors and in tensors of their own."""

    def __init__(self, variant, lp, seed):
        gen = self.gen = torch.Generator(device=DEV).manual_seed(seed)
        slots, off = [], 0
        for i, (n, listed) in enumerate(MT_LAYOUT):
            slots.append((_Slot(i, off, n), listed))
            off = (off + n + 7) // 8 * 8
        self.total = total = off
        self.listed = [s for s, listed in slots if listed]
        arena_g = {torch.float32: torch.zeros(total, device=DEV),
                   torch.bfloat16: torch.zeros(total, dtype=torch.bfloat16, device=DEV)}
        self.table = GradSegTable(self.listed, torch.device(DEV))
        self.grads = []
        for j, s in enumerate(self.listed):
            place = PLACES[j % len(PLACES)]
            dt = torch.bfloat16 if place.endswith("bf16") else torch.float32
            t = arena_g[dt][s.offset:s.end] if place.startswith("arena") else torch.empty(s.numel, dtype=dt, device=DEV)
            self.table.point(s, t.data_ptr(), dt)
            self.grads.append(t)
        self.table.upload()
        self.arena_g = arena_g
        self.idx = torch.cat([torch.arange(s.offset, s.end, device=DEV) for s in self.listed])
        cover = torch.zeros(total, dtype=torch.bool, device=DEV)
        for s in self.listed:
            cover[s.offset:(s.end + 7) // 8 * 8] = True
        data = torch.zeros(total, dtype=torch.bool, device=DEV)
        data[self.idx] = True
        self.pad, self.outside = cover & ~data, ~cover
        self.p = _weights(total, gen)
        self.states = [_state_values(name, total, gen) for name in STATE_NAMES[variant]]
        self.shadow = torch.randn(total, device=DEV, generator=gen).to(torch.bfloat16) if lp else None
        for v in [self.p, self.shadow] + self.states:
            if v is not None:
                v[self.pad] = 0                  # arena padding is zero
        self.before = [v.clone() for v in [self.p, self.shadow] + self.states if v is not None]

    def new_grads(self):
        for t in self.grads:
            t.copy_(_grad(t.numel(), self.gen))
        return torch.cat([t.double() for t in self.grads]) * SCALE

    def vectors(self):
        return [v for v in [self.p, self.shadow] + self.states if v is not None]

    def assert_pad_and_outside(self, what):
        for v, b in zip(self.vectors(), self.before):
            assert torch.all(v[self.pad] == 0), what + ": padding written"
            assert torch.equal(v[self.outside].view(torch.int16 if v.dtype == torch.bfloat16 else torch.int32),
                               b[self.outside].view(torch.int16 if b.dtype == torch.bfloat16 else torch.int32)), \
                what + ": slot outside the table written"


@pytest.mark.parametrize("lp", [False, True], ids=["no_shadow", "shadow"])
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_mt_update_matches_float64_torch_optim(variant, lp):
    case = _MtCase(variant, lp, seed=21)
    rule = VARIANTS[variant][0]
    coef = torch.tensor([0.75], device=DEV)
    idx = case.idx
    for step in range(1, 5):
        lr = BASE_LR[rule] * LR_SCALE[step - 1]
        g = case.new_grads()
        p0, s0 = case.p[idx].clone(), [s[idx].clone() for s in case.states]
        launch_mt(variant, case.p, case.states, case.shadow, case.table, lr=lr, wd=1e-2, step=step, coef=coef)
        check_step(variant, case.p[idx], [s[idx] for s in case.states], p0, g, s0, lr=lr, wd=1e-2, step=step,
                   what="mt step %d" % step)
        if lp:
            assert_shadow(case.shadow[idx], case.p[idx], "mt step %d" % step)
        case.assert_pad_and_outside("mt step %d" % step)


# ---- device-resident scalars (dyn) and CUDA-graph replay ---------------------------------------------

@pytest.mark.parametrize("form", ["flat", "mt"])
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_dyn_block_and_graph_replay_equal_by_value_launches(variant, form):
    """(a) deliberately wrong by-value lr / step with a correct ``dyn`` block == the by-value launch;
    (b) one launch captured in a CUDA graph, replayed over steps 1..5 with the scalars uploaded
    before each replay == eager launches.  Bit for bit."""
    rule = VARIANTS[variant][0]
    coef = torch.tensor([0.75], device=DEV)
    if form == "flat":
        n = 3 * 4096 + 3
        gen = torch.Generator(device=DEV).manual_seed(5)
        g = torch.empty(n, device=DEV)
        p = _weights(n, gen)
        states = [_state_values(name, n, gen) for name in STATE_NAMES[variant]]
        # (weights, states..., shadow) of the eager, the dyn and the replayed launches
        eager, via_dyn, replayed = ([p.clone()] + [s.clone() for s in states]
                                    + [torch.zeros(n, dtype=torch.bfloat16, device=DEV)] for _ in range(3))

        def launch(v, lr, step, dyn=None):
            launch_flat(variant, v[0], g, v[1:-1], v[-1], n, lr=lr, wd=1e-2, step=step, coef=coef, dyn=dyn)

        def new_grads():
            g.copy_(_grad(n, gen))
    else:
        cases = [_MtCase(variant, True, seed=33) for _ in range(3)]      # three identical copies
        table = cases[0].table                   # one table: every copy reads the same gradients
        eager, via_dyn, replayed = ([c.p] + c.states + [c.shadow] for c in cases)

        def launch(v, lr, step, dyn=None):
            launch_mt(variant, v[0], v[1:-1], v[-1], table, lr=lr, wd=1e-2, step=step, coef=coef, dyn=dyn)

        def new_grads():
            cases[0].new_grads()

    dyn, graph_dyn = (torch.zeros(4, device=DEV) for _ in range(2))
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):                 # SGD's graph is a later step: first_step is by value
        launch(replayed, 1.0, 2 if rule == "sgd" else 1, dyn=graph_dyn)
    for step in range(1, 6):
        lr = BASE_LR[rule] * LR_SCALE[step - 1]
        new_grads()
        launch(eager, lr, step)
        dyn.copy_(dyn_block(variant, lr, step))
        wrong_step = step if rule == "sgd" else step + 7
        launch(via_dyn, 123.0, wrong_step, dyn=dyn)
        if rule == "sgd" and step == 1:
            launch(replayed, lr, step)
        else:
            graph_dyn.copy_(dyn_block(variant, lr, step))
            graph.replay()
        torch.cuda.synchronize()
        for a, b, c in zip(eager, via_dyn, replayed):
            assert torch.equal(a, b), "dyn, step %d" % step
            assert torch.equal(a, c), "graph replay, step %d" % step


# ---- second reference: fp32 torch.optim in its default (foreach) form --------------------------------

def _ulps(a, b):
    """Distance in fp32 units in the last place (finite values)."""
    def key(x):
        i = x.contiguous().view(torch.int32).long()
        return torch.where(i < 0, -(i & 0x7FFFFFFF), i)
    return (key(a) - key(b)).abs()


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_distance_to_fp32_torch_optim(variant):
    rule = VARIANTS[variant][0]
    n = (1 << 20) + 3
    gen = torch.Generator(device=DEV).manual_seed(3)
    p = _weights(n, gen)
    states = [torch.zeros(n, device=DEV) for _ in STATE_NAMES[variant]]
    worst, differ, worst_env = 0, 0, 0.0
    for step in range(1, 5):
        lr = BASE_LR[rule] * LR_SCALE[step - 1]
        g = _grad(n, gen)
        p0, s0 = p.clone(), [s.clone() for s in states]
        launch_flat(variant, p, g, states, None, n, lr=lr, wd=1e-2, step=step)
        g32 = g * SCALE                           # the fp32 product the kernel forms
        ref_p, ref_s = reference_step(variant, p0, g32, s0, lr=lr, wd=1e-2, step=step,
                                      dtype=torch.float32, foreach=True)
        bounds = _envelope(variant, p0.double(), g32.double(), [s.double() for s in s0], ref_p.double(),
                           [s.double() for s in ref_s], lr=lr, wd=1e-2, step=step)
        for got, ref, b in zip([p] + states, [ref_p] + ref_s, bounds):
            worst = max(worst, int(_ulps(got, ref).max()))
            differ += int((got != ref).sum())
            worst_env = max(worst_env, float(((got.double() - ref.double()).abs() / (b / C[rule])).max()))
    print("fp32 torch.optim (foreach) vs kernel: %s max %d ulps, %d elements differ, max |diff| / (U mag + ETA) "
          "%.3f" % (variant, worst, differ, worst_env))
    if DISTANCE_TO_FP32_TORCH[variant] == 0:
        assert differ == 0 and worst == 0
    assert worst_env <= DISTANCE_TO_FP32_TORCH[variant], (variant, worst_env)


# ---- optimizer classes: apply_range and torch-format state dicts ---------------------------------------

CLASS_KINDS = {
    "sgd_momentum": lambda a: fused_optim.FusedSGD(a, lr=0.05, momentum=0.9, dampening=0.1, weight_decay=1e-2),
    "adam_amsgrad": lambda a: fused_optim.FusedAdam(a, lr=1e-2, weight_decay=1e-2, amsgrad=True),
    "rmsprop_momentum": lambda a: fused_optim.FusedRMSprop(a, lr=1e-2, momentum=0.9, weight_decay=1e-2),
}


@pytest.mark.parametrize("precision", [Precision.FP32, Precision.BF16])
@pytest.mark.parametrize("variant", list(CLASS_KINDS))
def test_optimizer_classes_round_trip_state_dicts_through_torch_optim(variant, precision):
    """Each step: the fused optimizer's ``state_dict()`` loads into float64 torch.optim, torch's
    ``state_dict()`` loads back unchanged, both step (clip coefficient on model parameters only,
    ``apply_range`` split at ``model_end``) and agree within the envelope."""
    rule = VARIANTS[variant][0]
    gen = torch.Generator(device=DEV).manual_seed(11)
    model = [torch.nn.Parameter(_weights(33 * 17, gen).view(33, 17)), torch.nn.Parameter(_weights(5, gen)),
             torch.nn.Parameter(_weights(4099, gen))]
    crit = [torch.nn.Parameter(_weights(7, gen)), torch.nn.Parameter(_weights(6, gen).view(2, 3))]
    arena = ParamArena(model, crit, device=DEV, precision=precision)
    assert 0 < arena.model_end < arena.numel
    opt = CLASS_KINDS[variant](arena)
    slots = sorted(arena.slots, key=lambda s: s.index)
    refs = [torch.nn.Parameter(arena.master[s.offset:s.end].view(s.shape).double()) for s in slots]
    ref_opt = _torch_optimizer(variant, refs, 1.0, 1e-2)
    coef = torch.tensor([0.75], device=DEV)
    for step in range(1, 5):
        lr = BASE_LR[rule] * LR_SCALE[step - 1]
        opt.hyper["lr"] = lr
        for s in slots:
            arena.grad[s.offset:s.end].copy_(_grad(s.numel, gen))
        sd = opt.state_dict()
        ref_opt.load_state_dict(sd)
        ref_opt.param_groups[0]["foreach"] = False
        assert ref_opt.param_groups[0]["lr"] == lr
        for r, s in zip(refs, slots):
            r.data.copy_(arena.master[s.offset:s.end].view(s.shape))
        vec_before = {k: v.clone() for k, v in opt._vec.items()}
        steps_before = opt._steps
        opt.load_state_dict(ref_opt.state_dict())
        for k, v in vec_before.items():
            assert torch.equal(opt._vec[k], v), "state %s changed by the round trip" % k
        if rule != "sgd":
            assert opt._steps == steps_before == step - 1
        assert (opt._steps == 0) == (step == 1)          # SGD's first-step flag survives
        p0 = torch.cat([r.detach().flatten().clone() for r in refs])
        s0 = [torch.cat([ref_opt.state[r][name].flatten() if ref_opt.state[r] else torch.zeros(r.numel(), device=DEV,
                                                                                            dtype=torch.float64)
                         for r in refs]) for name in STATE_NAMES[variant]]
        g_eff = []
        for r, s in zip(refs, slots):
            g = arena.grad[s.offset:s.end].double() * 0.5 * (0.75 if s.is_model else 1.0)
            r.grad = g.view(s.shape)
            g_eff.append(g)
        opt.begin_step()
        opt.apply_range(0, arena.numel, grad_scale=0.5, clip_coef_dev=coef)
        opt.end_step()
        ref_opt.step()
        got_p = torch.cat([arena.master[s.offset:s.end] for s in slots])
        got_s = [torch.cat([opt._vec[name][s.offset:s.end] for s in slots]) for name in STATE_NAMES[variant]]
        ref_p = torch.cat([r.detach().flatten() for r in refs])
        ref_s = [torch.cat([ref_opt.state[r][name].flatten() for r in refs]) for name in STATE_NAMES[variant]]
        bounds = _envelope(variant, p0, torch.cat(g_eff), s0, ref_p, ref_s, lr=lr, wd=1e-2, step=step)
        assert_within(got_p, ref_p, bounds[0], "step %d weights" % step)
        for name, got, ref, b in zip(STATE_NAMES[variant], got_s, ref_s, bounds[1:]):
            assert_within(got, ref, b, "step %d %s" % (step, name))
        if arena.lp is not None:
            for s in slots:
                if s.is_model:
                    assert_shadow(arena.lp[s.offset:s.end], arena.master[s.offset:s.end], "step %d" % step)


# ---- end to end: graph-replayed steps equal eager steps ---------------------------------------------------

E2E_OPTS = {
    "rmsprop_momentum": OptimOpts(algo=OptAlgorithm.RMSPROP, lr=1e-3, momentum=0.9, weightDecay=1e-4),
    "adam_amsgrad": OptimOpts(algo=OptAlgorithm.ADAM, lr=1e-3, weightDecay=1e-4, amsgrad=True),
}
E2E_STEPS = 8


def _run_mlp(variant, graph):
    ns = synthetic.api_namespace("frl_b200")
    t = ns.types
    save_dir = tempfile.mkdtemp(prefix="frl_b200_optim_paths_")
    torch.manual_seed(0)
    problem = synthetic.make_mlp_problem(ns, save_dir, n_train=8, width=256, n_classes=10, reg_dim=8, depth=2)
    run_opts = t.RunOpts(optim=E2E_OPTS[variant], batchSize=32, nEpochs=1, numThreads=0, singleThreaded=True,
                         numVisualizedSamples=0)
    args = SolverWorkerArgs(run_opts=run_opts, problem=problem, save_dir=save_dir, run_device=Device.GPU,
                            node_idx=0, node_count=1, rank=0, local_rank=0, world_size=1, group_name=None,
                            init_method="", precision=Precision.FP32, graph_step=graph)
    worker, _, _ = Solver.build_worker(args)
    worker.model.train()
    worker.criterion.train()
    gen = torch.Generator().manual_seed(1234)
    rows = []
    for i in range(E2E_STEPS):
        x, y, r = torch.randn(32, 256, generator=gen), torch.randint(0, 10, (32,), generator=gen), \
            torch.randn(32, 8, generator=gen)
        worker.optimizer.hyper["lr"] = E2E_OPTS[variant].lr * LR_SCALE[i % len(LR_SCALE)]
        _, total, _, _ = worker._pass_one_minibatch(i, t.Split.TRAIN, [x.cuda()], [(y.cuda(),), (r.cuda(),)])
        rows.append(float(total.detach()))
        del total
    torch.cuda.synchronize()
    return worker, rows


@pytest.mark.parametrize("variant", list(E2E_OPTS))
def test_graph_replayed_steps_equal_eager_steps(variant):
    """RMSprop (momentum) and Adam-amsgrad through ``Solver.build_worker``: steps replayed from the
    captured graph read lr (and Adam's bias corrections) from the device block, and must equal the
    eager run's steps bit for bit while lr changes every step."""
    eager_w, eager = _run_mlp(variant, False)
    graph_w, graphed = _run_mlp(variant, True)
    opt = graph_w.optimizer
    assert type(opt) is type(eager_w.optimizer) is {"rmsprop_momentum": fused_optim.FusedRMSprop,
                                                    "adam_amsgrad": fused_optim.FusedAdam}[variant]
    assert graph_w.graphed is not None and len(graph_w.graphed._graphs) == 1 and opt._dyn is not None
    assert eager == graphed and eager[0] != eager[-1]
    assert torch.equal(graph_w.arena.master, eager_w.arena.master)
    assert opt._vec.keys() == eager_w.optimizer._vec.keys() == set(STATE_NAMES[variant])
    for k, v in opt._vec.items():
        assert torch.equal(v, eager_w.optimizer._vec[k]), k


# ---- every instantiation is launched -----------------------------------------------------------------

FLAT_INSTANTIATIONS = sorted(
    "frl::%s,frl::%s,%d,%s" % (rule, gv, ns, lp)
    for rule, ns in (("SgdRule", 0), ("SgdRule", 1), ("AdamRule<false>", 2), ("AdamRule<true>", 3),
                     ("RmspropRule<false>", 1), ("RmspropRule<true>", 2))
    for gv in ("f32x4", "bf16x4") for lp in ("false", "true"))
MT_INSTANTIATIONS = sorted(
    "frl::%s,%d,%s" % (rule, ns, lp)
    for rule, ns in (("SgdRule", 0), ("SgdRule", 1), ("AdamRule<false>", 2), ("AdamRule<true>", 3),
                     ("RmspropRule<false>", 1), ("RmspropRule<true>", 2))
    for lp in ("false", "true"))


def _template_args(name, kernel):
    """``frl::update_kernel<A, B<C>, D>(...)`` -> ``A,B<C>,D`` (spaces dropped)."""
    rest = name.split(kernel + "<", 1)[1]
    depth = 0
    for i, ch in enumerate(rest):
        depth += ch == "<"
        if ch == ">":
            if depth == 0:
                return rest[:i].replace(" ", "")
            depth -= 1
    raise ValueError(name)


def test_every_update_instantiation_is_launched():
    from torch.profiler import ProfilerActivity, profile
    n = 4099
    case = {lp: _MtCase(v, lp, seed=3) for v in ("adam_amsgrad",) for lp in (False, True)}
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for variant in VARIANTS:
            names = STATE_NAMES[variant]
            for gdt in (torch.float32, torch.bfloat16):
                for lp in (False, True):
                    states = [torch.zeros(n, device=DEV) for _ in names]
                    shadow = torch.zeros(n, dtype=torch.bfloat16, device=DEV) if lp else None
                    launch_flat(variant, torch.zeros(n, device=DEV), torch.zeros(n, dtype=gdt, device=DEV), states,
                                shadow, n, lr=0.1, wd=0.0, step=1)
            for lp in (False, True):
                c = case[lp]
                launch_mt(variant, c.p, c.states[:len(names)], c.shadow, c.table, lr=0.1, wd=0.0, step=1)
        torch.cuda.synchronize()
    flat, mt = set(), set()
    for e in prof.events():
        if "frl::update_kernel<" in e.name:
            flat.add(_template_args(e.name, "frl::update_kernel"))
        elif "frl::update_mt_kernel<" in e.name:
            mt.add(_template_args(e.name, "frl::update_mt_kernel"))
    print("flat", sorted(flat), "mt", sorted(mt))
    assert sorted(flat) == FLAT_INSTANTIATIONS and len(flat) == 24
    assert sorted(mt) == MT_INSTANTIATIONS and len(mt) == 12
