"""Host checks for the layout the sm_90a GEMM tests read K14's intermediates through.

``tests/gemm_sm90_oracle.muon_layout`` restates where ``build_plan`` (csrc/muon.cu) puts each
matrix's Gram buffers and iterates.  If it disagreed with the library, the GPU test would compare
the wrong bytes; ``frl_muon_plan_bytes`` needs no device, so the workspace and scratch sizes are
pinned here for every shape list the GPU test uses and for random lists.  The fma32 helper the
prologue check relies on is held against exact rational arithmetic.
"""
import random
from fractions import Fraction

import numpy as np
import pytest
import torch

import frl_b200  # noqa: F401
from frl_b200 import _native
import gemm_sm90_oracle as go

MUON_SHAPES = ((1, 512), (7, 9), (8, 64), (127, 129), (128, 128), (129, 300), (255, 257), (256, 256),
               (257, 1000), (300, 700), (700, 300), (383, 385), (1000, 4096), (4096, 1000), (4096, 4096))


def _rows(shapes):
    rows, off = [], 0
    for i, (R, C) in enumerate(shapes):
        rows.append((i, off, R, C))
        off += go.up(R * C, 8)
    return rows


def _check(rows):
    _, scratch, ws = _native.muon_plan_bytes(torch.tensor(rows, dtype=torch.int64).reshape(-1, 4))
    layout, ws_mine = go.muon_layout(rows)
    assert ws_mine == ws
    assert go.muon_scratch_bytes(rows) == scratch
    end = 0
    for L in layout:                     # buffers back to back, 128-byte aligned, inside the workspace
        assert L.ga_off == end and L.ga_off % 128 == 0 and L.gb_off % 128 == 0
        end = L.gb_off + go.up(2 * L.m * L.ld_g, 128)
        if L.x_in_ws:
            assert L.x_off[0] == end and L.x_off[1] % 128 == 0
            end = L.x_off[1] + go.up(2 * L.m * L.ld_x, 128)
        else:
            assert L.n % 8 == 0 and L.x_off == (4 * L.arena_off, 4 * L.arena_off + 2 * L.m * L.n)
    assert end == ws


@pytest.mark.parametrize("shape", MUON_SHAPES, ids=lambda s: "%dx%d" % s)
def test_layout_matches_the_library_per_shape(shape):
    _check(_rows([shape]))


def test_layout_matches_the_library_for_the_whole_list():
    _check(_rows(MUON_SHAPES))


@pytest.mark.parametrize("seed", range(8))
def test_layout_matches_the_library_for_random_lists(seed):
    rnd = random.Random(seed)
    n = rnd.choice([1, 3, 40, 150])
    shapes = [(rnd.randint(1, 700), rnd.randint(1, 700)) if rnd.random() < 0.9 else
              (rnd.randint(1, 9), rnd.randint(1, 4100)) for _ in range(n)]
    _check(_rows(shapes))


def test_gpu_test_shapes_cover_the_tile_walk():
    for sms in (78, 114, 132):
        s = go.k12_shapes(sms)
        rows, out, inp = s["tiles_m_17_just_above_sms"]
        assert out // go.BM == 17 and sms < 17 * (inp // go.BN) <= sms + 17
        rows, out, inp = s["two_sms_plus_one_tiles"]
        assert (out // go.BM) * (inp // go.BN) == 2 * sms + 1 and (out // go.BM) % 16
        rows, out, inp = s["tiles_m_16_two_per_cta"]
        assert out // go.BM == 16 and 2 * sms < 16 * (inp // go.BN) < 3 * sms
        assert [s[k][0] // go.K12_BK for k in ("one_kblock", "kstages_kblocks", "kstages_plus_one")] == \
            [1, go.K_STAGES, go.K_STAGES + 1]
        for name, (rows, k, cols) in go.k13_tiles_shapes(sms).items():
            tm, tn = rows // go.BM, cols // go.BN
            assert tm == int(name[-2:]) and sms < tm * tn <= sms + tm


def test_fma32_rounds_once():
    g = torch.Generator().manual_seed(0)
    a = torch.randn(20000, generator=g)
    b = torch.randn(20000, generator=g)
    c = -(a.double() * b.double()).float() + torch.randn(20000, generator=g) * 1e-6     # heavy cancellation
    # the float64 sum lands exactly halfway between two fp32 values while the exact sum does not:
    # ties-to-even on the float64 sum would round the wrong way in both
    u = 2.0 ** -23
    a = torch.cat([a, torch.tensor([1 + u, -(1 + u), 2.0 ** -12])])
    b = torch.cat([b, torch.tensor([2.0 ** -24 * (1 - u), 2.0 ** -24 * (1 - u), 2.0 ** -12])])
    c = torch.cat([c, torch.tensor([1 + u, 1 + u, 1.0])])
    got = go.fma32(a, b, c)
    for x, y, z, r in zip(a.tolist(), b.tolist(), c.tolist(), got.tolist()):
        exact = Fraction(x) * Fraction(y) + Fraction(z)
        lo = float(np.float32(float(exact)))
        # the correctly rounded fp32 of the exact value: the nearer of the two fp32 around it
        cands = [np.float32(lo), np.nextafter(np.float32(lo), np.float32(np.inf)),
                 np.nextafter(np.float32(lo), np.float32(-np.inf))]
        best = min(cands, key=lambda v: (abs(Fraction(float(v)) - exact), int(np.float32(v).view(np.int32)) & 1))
        assert r == float(best), (x, y, z, r, float(best))
