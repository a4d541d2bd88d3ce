"""The hand-written sm_90a GEMMs (K12 ``dw_gemm``, K13 ``dx_gemm_drelu``, K14 Muon's Gram, poly and
update products) element by element against float64, at the shapes that reach each path of their
shared skeleton (csrc/gemm_sm90.cuh): one k-block, exactly ``kStages`` and one more, a single
tile, the grouped tile walk with 16 row blocks and with 17, CTAs holding 2 and 3 tiles, padded
leading dimensions, partial columns, mirrored Gram tiles, and plans mixing many matrices.

Bound.  Every output is bf16, rounded once from an fp32 accumulator.  For the float64 product
P = A B over K terms:

    |out - P| <= K 2^-24 (|A| |B|) + 2^-8 |P|

An fp32 sum of K products of bf16 values (each exact in fp32), in any order, is off by at most
K u sum|a b| with u = 2^-24 (the first-order bound of recursive summation; pairwise and
tensor-core orders do better).  The bf16 rounding of that fp32 value is at most half an ulp,
2^-9 relative; 2^-8 |P| covers it together with the fp32 error it is applied to.

K14's poly and update products fold an addend into the accumulator before the bf16 rounding:
out = bf16(fmaf(alpha, Add, beta * acc)).  The accumulator error is scaled by |beta|; beta * acc
and the FMA each round once in fp32 (2^-24 relative each, of values bounded by |beta A B| and
|alpha Add| + |beta A B|), which 2^-23 (|alpha Add| + |beta| |A| |B|) covers:

    |out - P| <= |beta| K 2^-24 (|A| |B|) + 2^-23 (|alpha Add| + |beta| |A| |B|) + 2^-8 |P|

for P = alpha Add + beta A B in float64.  K14's products are checked against the kernel's own
operands (its X0, its A, its B), so each product is held to this bound on its own rather than
through the end-to-end Newton-Schulz result, which pulls errors back toward the orthogonal factor.

Untouched memory.  Outputs and K14's workspace start filled with a bf16 NaN pattern; everything
the kernel may not write (padding columns, bytes between buffers, what lies past the last one) must
still hold it afterwards, and nothing inside a logical extent may.

References run in float64 on the GPU.  Shapes come from the device's SM count.
"""
import collections
import math

import pytest
import torch

import frl_b200  # noqa: F401
from frl_b200 import _native
from frl_b200.fused_optim import MUON_NS_COEFFICIENTS
from frl_b200.multi_tensor import GradSegTable
import gemm_sm90_oracle as go

pytestmark = pytest.mark.gpu
DEV = "cuda"
CANARY = 0x7FA5                        # a bf16 NaN no kernel computes
BF = torch.bfloat16


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _canary(shape, dtype=BF):
    t = torch.empty(shape, dtype=dtype, device=DEV)
    t.view(torch.int16).fill_(CANARY)
    return t


def _is_canary(t):
    return t.contiguous().view(torch.int16) == CANARY


def _assert_within(out, p, bound, what):
    out = out.double()
    assert not torch.isnan(out).any(), "%s: %d NaN" % (what, int(torch.isnan(out).sum()))
    bad = (out - p).abs() > bound
    if bad.any():
        i = tuple(bad.nonzero()[0].tolist())
        raise AssertionError("%s: %d of %d elements out of bound, first %s: got %r want %r bound %r"
                             % (what, int(bad.sum()), bad.numel(), i, out[i].item(), p[i].item(), bound[i].item()))


# ---- K12: dW = dZ^T X --------------------------------------------------------------------------

def _k12_operands(rows, out, inp, pad, seed=0):
    """dz [rows, out] and x [rows, inp], row strides out + pad and inp + pad, NaN in the padding"""
    g = _gen(seed)
    dz = torch.full((rows, out + pad), float("nan"), device=DEV, dtype=BF)
    x = torch.full((rows, inp + pad), float("nan"), device=DEV, dtype=BF)
    dz[:, :out] = torch.randn(rows, out, device=DEV, generator=g).to(BF)
    x[:, :inp] = torch.randn(rows, inp, device=DEV, generator=g).to(BF)
    return dz[:, :out], x[:, :inp]


def _check_gw(gw, dz, x, what):
    a, b = dz.double().t(), x.double()
    p = a @ b
    _assert_within(gw, p, go.gemm_bound(a, b, p, dz.shape[0]), what)


@pytest.mark.parametrize("pad", [0, 40], ids=["dense", "padded"])
@pytest.mark.parametrize("path", go.K12_PATHS)
def test_k12_gradient_every_element_against_float64(path, pad):
    rows, out, inp = go.k12_shapes(_sms())[path]
    dz, x = _k12_operands(rows, out, inp, pad)
    buf = _canary(out * inp + 64)                       # gw, then a canary
    gw = buf[:out * inp].view(out, inp)
    _native.dw_gemm(dz, x, gw)
    torch.cuda.synchronize()
    _check_gw(gw, dz, x, "K12 %s" % path)
    assert _is_canary(buf[out * inp:]).all()


@pytest.mark.parametrize("path", ["one_kblock", "tiles_m_17_just_above_sms", "two_sms_plus_one_tiles"])
def test_k12_update_mode_writes_the_same_gradient_and_nothing_past_the_slices(path):
    rows, out, inp = go.k12_shapes(_sms())[path]
    dz, x = _k12_operands(rows, out, inp, 24, seed=1)
    n = out * inp
    g = _gen(2)
    p = torch.randn(n + 16, device=DEV, generator=g)
    mom = torch.randn(n + 16, device=DEV, generator=g)
    lp = _canary(n + 64)
    tails = (p[n:].clone(), mom[n:].clone())
    gw = _canary(n + 64)
    _native.dw_gemm_sgd(dz, x, gw[:n].view(out, inp), p, mom, lp, lr=0.01, mu=0.9, dampening=0.0, wd=1e-4)
    ref = _canary(n)
    _native.dw_gemm(dz, x, ref.view(out, inp))
    torch.cuda.synchronize()
    assert torch.equal(gw[:n].view(torch.int16), ref.view(torch.int16))
    _check_gw(gw[:n].view(out, inp), dz, x, "K12 update %s" % path)
    assert _is_canary(gw[n:]).all() and _is_canary(lp[n:]).all()
    assert torch.equal(p[n:], tails[0]) and torch.equal(mom[n:], tails[1])
    assert not _is_canary(lp[:n]).any()


# ---- K13: dZ = [act > 0] bf16(dZ_up W), db (+)= colsum(dZ) ------------------------------------------

def _k13_operands(rows, k, cols, ld_up=None, ld_act=None, seed=0):
    g = _gen(seed)
    up_full = torch.full((rows, ld_up or k), float("nan"), device=DEV, dtype=BF)
    up_full[:, :k] = (torch.randn(rows, k, device=DEV, generator=g) / 8).to(BF)
    w = (torch.randn(k, cols, device=DEV, generator=g) / 8).to(BF)
    act_full = torch.full((rows, ld_act or cols), float("nan"), device=DEV, dtype=BF)
    act_full[:, :cols] = torch.randn(rows, cols, device=DEV, generator=g).relu().to(BF)
    return up_full[:, :k], w, act_full[:, :cols]


def _check_dz(dz, dz_up, w, act, what):
    a, b = dz_up.double(), w.double()
    p = a @ b
    keep = act > 0
    bound = go.gemm_bound(a, b, p, dz_up.shape[1])
    _assert_within(dz.double()[keep], p[keep], bound[keep], what)
    assert (dz[~keep].view(torch.int16) == 0).all(), what


def _check_db(dz, db, base=None):
    """db against the float64 column sum of this launch's own dZ: an fp32 sum of B terms in any
    order, then one bf16 rounding"""
    s = dz.double().sum(0) + (0 if base is None else base.double())
    bound = dz.shape[0] * 2.0 ** -24 * dz.double().abs().sum(0) + 2.0 ** -8 * s.abs()
    _assert_within(db, s, bound, "db")


def _k13(dz_up, w, act, ld_dz=None, db=None, accumulate=False):
    rows, cols = act.shape
    full = _canary((rows, ld_dz or cols))
    dz = full[:, :cols]
    dz.fill_(float("nan"))
    db = torch.full((cols,), float("nan"), device=DEV, dtype=BF) if db is None else db
    _native.dx_gemm_drelu(dz_up, w, act, dz, db, accumulate=accumulate)
    torch.cuda.synchronize()
    return full, dz, db


K13_PATHS = {
    "k8": (256, 8, 512), "k24": (256, 24, 512), "k32": (256, 32, 512), "k40": (256, 40, 512),
    "k1064": (256, 1064, 512), "single_tile": (128, 72, 256), "one_strip_128_row_tiles": (16384, 72, 256),
}


@pytest.mark.parametrize("path", list(K13_PATHS) + ["tiles_m_16", "tiles_m_17"])
def test_k13_dz_and_db_against_float64(path):
    rows, k, cols = K13_PATHS.get(path) or go.k13_tiles_shapes(_sms())[path]
    dz_up, w, act = _k13_operands(rows, k, cols)
    _, dz, db = _k13(dz_up, w, act)
    _check_dz(dz, dz_up, w, act, "K13 %s" % path)
    _check_db(dz, db)


def test_k13_heads_row_stride_with_nan_past_k():
    """the heads' K = 1064 dZ_up rows at the production stride (DX_DRELU_ROW_ALIGN), NaN in
    columns 1064..1087 that must not be read"""
    k = 1064
    ld = go.up(k, _native.DX_DRELU_ROW_ALIGN)
    assert ld == 1088
    dz_up, w, act = _k13_operands(512, k, 768, ld_up=ld, seed=3)
    assert dz_up.stride(0) == ld and torch.isnan(dz_up.as_strided((512, ld), (ld, 1))[:, k:]).all()
    _, dz, db = _k13(dz_up, w, act)
    _check_dz(dz, dz_up, w, act, "K13 K=1064 ld=1088")
    _check_db(dz, db)


def test_k13_padded_act_and_dz_rows():
    rows, k, cols = 384, 72, 512
    dz_up, w, act = _k13_operands(rows, k, cols, ld_act=cols + 264, seed=4)
    full, dz, db = _k13(dz_up, w, act, ld_dz=cols + 72)
    _check_dz(dz, dz_up, w, act, "K13 padded")
    _check_db(dz, db)
    assert _is_canary(full[:, cols:]).all()


def test_k13_scratch_reused_across_rows():
    """one scratch per (device, cols): rows 4096 -> 128 -> 2176, then accumulate; each db from its
    own launch's dZ (a ticket left non-zero or a stale partial would show)"""
    cols = 768
    for i, (rows, acc) in enumerate([(4096, False), (128, False), (2176, False), (2176, True)]):
        dz_up, w, act = _k13_operands(rows, 40, cols, seed=10 + i)
        base = torch.randn(cols, device=DEV, generator=_gen(20 + i)).to(BF) if acc else None
        _, dz, db = _k13(dz_up, w, act, db=None if base is None else base.clone(), accumulate=acc)
        _check_dz(dz, dz_up, w, act, "K13 rows %d" % rows)
        _check_db(dz, db, base)
        if i == 0:
            scratch = _native._dx_drelu_scratch[(act.device.index, cols)]
    assert _native._dx_drelu_scratch[(act.device.index, cols)] is scratch      # one buffer served all four


# ---- K14: Muon's Newton-Schulz products ----------------------------------------------------------

A_NS, B_NS, C_NS = (float(torch.tensor(v, dtype=torch.float32)) for v in MUON_NS_COEFFICIENTS)
LR, EPS = 0.02, 1e-7
MUON_SHAPES = ((1, 512), (7, 9), (8, 64), (127, 129), (128, 128), (129, 300), (255, 257), (256, 256),
               (257, 1000), (300, 700), (700, 300), (383, 385), (1000, 4096), (4096, 1000), (4096, 4096))
Slot = collections.namedtuple("Slot", "index offset numel shape")


class _Muon:
    """Muon matrices in an arena this test owns: K14 planned over them with a workspace and an
    exp_avg_sq vector allocated here, so the intermediates can be read where build_plan puts them."""

    def __init__(self, shapes):
        self.rows, off = [], 0
        for i, (R, C) in enumerate(shapes):
            self.rows.append((i, off, R, C))
            off += go.up(R * C, 8)
        self.total = off
        self.layout, ws_bytes = go.muon_layout(self.rows)
        shape = torch.tensor(self.rows, dtype=torch.int64).reshape(-1, 4)
        assert _native.muon_plan_bytes(shape)[2] == ws_bytes
        self.ws = torch.empty(ws_bytes + 256, dtype=torch.uint8, device=DEV)
        self.state = torch.empty(self.total + 64, dtype=torch.float32, device=DEV)
        self.plan = _native.muon_plan(shape, self.state, self.ws)
        self.slots = [Slot(i, o, R * C, (R, C)) for i, o, R, C in self.rows]
        self.table = GradSegTable(self.slots, torch.device(DEV))
        # bf16 elements of the workspace and of exp_avg_sq the kernels may write
        self.ws_ok = torch.zeros(self.ws.numel() // 2, dtype=torch.bool, device=DEV)
        self.state_ok = torch.zeros(self.state.numel() * 2, dtype=torch.bool, device=DEV)
        for L in self.layout:
            x_ok = self.ws_ok if L.x_in_ws else self.state_ok
            for ok, off_, ld, cols in ((self.ws_ok, L.ga_off, L.ld_g, L.m), (self.ws_ok, L.gb_off, L.ld_g, L.m),
                                       (x_ok, L.x_off[0], L.ld_x, L.n), (x_ok, L.x_off[1], L.ld_x, L.n)):
                ok[off_ // 2:off_ // 2 + L.m * ld].view(L.m, ld)[:, :cols] = True
        self.lp_ok = torch.zeros(self.total + 64, dtype=torch.bool, device=DEV)
        for s in self.slots:
            self.lp_ok[s.offset:s.offset + s.numel] = True

    def grads(self, seed):
        g = torch.Generator(device=DEV).manual_seed(seed)
        return [torch.randn(s.shape, device=DEV, generator=g) for s in self.slots]

    def run(self, grads, *, ns_steps, momentum=0.0, nesterov=False, buf=None, p=None, wd=0.0):
        self.ws.view(torch.int16).fill_(CANARY)
        self.state.view(torch.int16).fill_(CANARY)
        self.p = torch.zeros(self.total + 64, device=DEV) if p is None else p.clone()
        self.buf = torch.zeros(self.total + 64, device=DEV) if buf is None else buf.clone()
        self.lp = _canary(self.total + 64)
        for s, g in zip(self.slots, grads):
            self.table.point(s, g.data_ptr(), g.dtype)
        self.table.upload()
        _native.muon_mt(self.p, self.buf, self.lp, self.table, self.plan, lr=LR, wd=wd, momentum=momentum,
                        nesterov=nesterov, ns_coefficients=MUON_NS_COEFFICIENTS, ns_steps=ns_steps, eps=EPS,
                        adjust_lr_fn="match_rms_adamw")
        torch.cuda.synchronize()
        assert _is_canary(self.ws[:self.ws_ok.numel() * 2])[~self.ws_ok].all(), "workspace written out of bounds"
        assert _is_canary(self.state)[~self.state_ok].all(), "exp_avg_sq written out of bounds"
        assert _is_canary(self.lp)[~self.lp_ok].all() and not _is_canary(self.lp)[self.lp_ok].any()

    # intermediates of matrix i, logical extent only, as float64
    def x(self, k, i):
        L = self.layout[i]
        return go.read_x(k, self.ws, self.state, L)[:, :L.n]

    def ga(self, i):
        L = self.layout[i]
        return go.read_ga(self.ws, L)[:, :L.m]

    def gb(self, i):
        L = self.layout[i]
        return go.read_gb(self.ws, L)[:, :L.m]

    def p_of(self, i):
        s = self.slots[i]
        return self.p[s.offset:s.offset + s.numel].view(s.shape)

    def lp_of(self, i):
        s = self.slots[i]
        return self.lp[s.offset:s.offset + s.numel].view(s.shape)

    def buf_of(self, buf, i):
        s = self.slots[i]
        return buf[s.offset:s.offset + s.numel].view(s.shape)

    def adj(self, i):
        R, C = self.slots[i].shape
        return torch.tensor(0.2 * math.sqrt(max(R, C)), dtype=torch.float32, device=DEV) * \
            torch.tensor(LR, dtype=torch.float32, device=DEV)


def _expected_x0(g, buf0, momentum, nesterov):
    """(X0 in the kernel's [m, n] layout, the new momentum buffer), restating the prologue and the
    normalisation bit for bit: fp32 lerps, bf16(u), the bf16 of the float64 norm clamped at bf16(eps),
    then bf16(bf16(u) / nrm) with an IEEE fp32 division"""
    buf = go.lerp32(buf0, g, 1.0 - momentum)
    u = go.lerp32(g, buf, momentum) if nesterov else buf
    xb = u.to(BF)
    ss = float((xb.double() ** 2).sum())
    nrm = torch.tensor(math.sqrt(ss), dtype=torch.float64).float().to(BF).float()
    eps_bf = torch.tensor(EPS, dtype=torch.float32).to(BF).float()
    nrm = torch.maximum(nrm, eps_bf).to(DEV)
    x0 = (xb.float() / nrm).to(BF)
    return (x0.t() if g.shape[0] > g.shape[1] else x0), buf


def _check_x0(M, i, g, buf0, momentum, nesterov, what):
    want, buf = _expected_x0(g, M.buf_of(buf0, i) if buf0 is not None else torch.zeros_like(g), momentum, nesterov)
    differ = int((M.x(0, i).view(torch.int16) != want.contiguous().view(torch.int16)).sum())
    assert differ == 0, "%s: X0 differs in %d elements" % (what, differ)
    assert torch.equal(M.buf_of(M.buf, i).view(torch.int32), buf.view(torch.int32)), what + ": momentum buffer"


def _check_gram(x, ga, what):
    xd = x.double()
    p = xd @ xd.t()
    _assert_within(ga, p, go.gemm_bound(xd, xd.t(), p, xd.shape[1]), what + " gram")


def _check_poly(ga, gb, what):
    a = ga.double()
    p = B_NS * a + C_NS * (a @ a)
    _assert_within(gb, p, go.gemm_bound(a, a, p, a.shape[0], alpha_add=B_NS * a, beta=C_NS), what + " poly")


def _check_update(x, gb, out, what):
    xd, b = x.double(), gb.double()
    p = A_NS * xd + b @ xd
    _assert_within(out, p, go.gemm_bound(b, xd, p, b.shape[0], alpha_add=A_NS * xd), what + " update")


def _o_from_last_update(M, i, what):
    """the bf16 O the last update applied, from p = -adj O (p was 0, wd 0), in X's [m, n] layout;
    p must be exactly the fp32 -adj O and the shadow exactly bf16(p)"""
    adj = M.adj(i)
    p = M.p_of(i)
    o = (-p / adj).to(BF)
    assert (p == -adj * o.float()).all(), what + ": p is not -adj * bf16 O"
    assert torch.equal(M.lp_of(i).view(torch.int16), p.to(BF).view(torch.int16)), what + ": shadow"
    return o.t() if M.layout[i].trans else o


def _check_one_step(M, i, g, what):
    """ns_steps = 1, momentum 0, p = 0, wd = 0: X0, then each product against the kernel's own operands"""
    _check_x0(M, i, g, None, 0.0, False, what)
    x0 = M.x(0, i)
    _check_gram(x0, M.ga(i), what)
    _check_poly(M.ga(i), M.gb(i), what)
    o = _o_from_last_update(M, i, what)
    _check_update(x0, M.gb(i), o, what)
    return o


def _ulp32(x):
    x = x.abs()
    return torch.nextafter(x, torch.full_like(x, float("inf"))) - x


@pytest.mark.parametrize("shape", MUON_SHAPES, ids=lambda s: "%dx%d" % s)
def test_k14_products_against_float64(shape):
    M = _Muon([shape])
    grads = M.grads(0)
    g = grads[0]
    what = "K14 %dx%d" % shape

    M.run(grads, ns_steps=1)
    o = _check_one_step(M, 0, g, what)
    x0, b0 = M.x(0, 0).clone(), M.gb(0).clone()

    # the same O applied to p != 0 with weight decay: p = fmaf(-adj, O, p decay)
    p0 = torch.randn(M.total + 64, device=DEV, generator=_gen(1))
    wd = 0.1
    M.run(grads, ns_steps=1, p=p0, wd=wd)
    f32 = lambda v: float(torch.tensor(v, dtype=torch.float32))            # noqa: E731
    decay = torch.tensor(1.0 - f32(LR) * f32(wd), dtype=torch.float32, device=DEV)   # fp32 of the double 1 - lr wd
    s = M.slots[0]
    ot = o.t() if M.layout[0].trans else o
    want = go.fma32(-M.adj(0).expand(s.shape), ot.float(), p0[s.offset:s.offset + s.numel].view(s.shape) * decay)
    got = M.p_of(0)
    assert ((got - want).abs() <= _ulp32(want)).all(), what + ": p with weight decay"
    assert torch.equal(M.lp_of(0).view(torch.int16), got.to(BF).view(torch.int16))

    # two steps: X1 through the non-last update (masked partial columns), then the second Gram
    M.run(grads, ns_steps=2)
    assert torch.equal(M.x(0, 0).view(torch.int16), x0.view(torch.int16))
    x1 = M.x(1, 0)
    _check_update(x0, b0, x1, what + " step 1")
    _check_gram(x1, M.ga(0), what + " step 2")

    # momentum 0.95, Nesterov, a non-zero buffer: the prologue's lerps
    buf0 = torch.randn(M.total + 64, device=DEV, generator=_gen(2))
    M.run(grads, ns_steps=1, momentum=0.95, nesterov=True, buf=buf0)
    _check_x0(M, 0, g, buf0, 0.95, True, what + " nesterov")


def _mixed_shapes(n, seed):
    g = torch.Generator().manual_seed(seed)
    shapes = []
    for j in range(n):
        if j % 10 == 0:
            shapes.append((int(torch.randint(1, 9, (1,), generator=g)), int(torch.randint(1, 1500, (1,), generator=g))))
        else:
            shapes.append(tuple(int(v) for v in torch.randint(1, 640, (2,), generator=g)))
    return shapes


def test_k14_one_plan_over_mixed_matrices_and_a_second_launch():
    """~150 matrices in one plan: a CTA's consecutive tiles belong to different matrices with
    different K; a second launch of the same plan (tickets back at 0) again gives every X0 and
    every product of its own inputs"""
    shapes = _mixed_shapes(150, 5)
    M = _Muon(shapes)
    assert M.plan.n_mat == 150
    for launch in range(2):
        grads = M.grads(100 + launch)
        M.run(grads, ns_steps=1)
        for i, sh in enumerate(shapes):
            _check_one_step(M, i, grads[i], "K14 mixed launch %d matrix %d %dx%d" % ((launch, i) + sh))
