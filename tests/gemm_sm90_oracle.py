"""TEST INFRASTRUCTURE for the hand-written sm_90a GEMMs (K12, K13, K14).

* ``muon_layout``: where K14 keeps each matrix's Newton-Schulz intermediates, restated from
  ``build_plan`` in csrc/muon.cu, so a test can read them out of the workspace and the
  ``exp_avg_sq`` vector it owns.  Per matrix [R, C], m = min(R, C), n = max(R, C): the Gram
  buffers ``ga`` and ``gb``, each [m, up(m, 8)] bf16 in ``up(2 m up(m, 8), 128)`` bytes, back to back
  in the workspace from offset 0; then, when n % 8 != 0, the two iterates X0 and X1, each
  [m, up(n, 8)] bf16 in ``up(2 m up(n, 8), 128)`` bytes; otherwise X0 and X1 are [m, n] bf16, one
  after the other in the matrix's own fp32 ``exp_avg_sq`` slot (4 bytes per element).
* ``muon_scratch_bytes``: tickets, norms and per-prologue-tile partials.
* ``fma32``: fmaf(a, b, c) of fp32 tensors, rounded once, for the kernels' fp32 lerp.
* ``gemm_bound``: the float64 bound every bf16 GEMM output is held to.
* tile-table shapes derived from the SM count.

Never imported by the product.
"""
import dataclasses
from typing import List, Sequence, Tuple

import torch

BM, BN = 128, 256          # output tile of all three kernels
PT = 64                    # K14's prologue tile edge
K_STAGES = 6               # depth of the k-block ring
K12_BK = 32                # K12's k-block (rows of dZ and X)


def up(x: int, a: int) -> int:
    return (x + a - 1) // a * a


@dataclasses.dataclass
class MatLayout:
    R: int
    C: int
    arena_off: int
    m: int
    n: int
    trans: bool
    ld_g: int
    ga_off: int            # byte offsets into the workspace
    gb_off: int
    ld_x: int
    x_in_ws: bool
    x_off: Tuple[int, int]  # byte offsets into the workspace (x_in_ws) or into exp_avg_sq


def muon_layout(shape: Sequence[Sequence[int]]) -> Tuple[List[MatLayout], int]:
    """Per-matrix layout and the workspace bytes of rows (segment, arena offset, R, C)."""
    out, off = [], 0
    for _, arena_off, R, C in shape:
        m, n = min(R, C), max(R, C)
        ld_g = up(m, 8)
        gbytes = up(2 * m * ld_g, 128)
        ga_off, gb_off = off, off + gbytes
        off += 2 * gbytes
        if n % 8 == 0:
            ld_x, x_in_ws = n, False
            base = 4 * arena_off
            x_off = (base, base + 2 * m * n)
        else:
            ld_x, x_in_ws = up(n, 8), True
            xbytes = up(2 * m * ld_x, 128)
            x_off = (off, off + xbytes)
            off += 2 * xbytes
        out.append(MatLayout(R, C, arena_off, m, n, R > C, ld_g, ga_off, gb_off, ld_x, x_in_ws, x_off))
    return out, off


def muon_scratch_bytes(shape: Sequence[Sequence[int]]) -> int:
    n_mat = len(shape)
    n_pro = sum(-(-R // PT) * -(-C // PT) for _, _, R, C in shape)
    return 2 * up(4 * n_mat, 16) + up(8 * n_pro, 128)


def _bf16(buf: torch.Tensor, off: int, rows: int, ld: int) -> torch.Tensor:
    return buf.view(torch.uint8)[off:off + 2 * rows * ld].view(torch.bfloat16).view(rows, ld)


def read_ga(ws: torch.Tensor, L: MatLayout) -> torch.Tensor:
    """[m, ld_g] bf16 view of the Gram matrix A (padding columns included)."""
    return _bf16(ws, L.ga_off, L.m, L.ld_g)


def read_gb(ws: torch.Tensor, L: MatLayout) -> torch.Tensor:
    """[m, ld_g] bf16 view of the polynomial B."""
    return _bf16(ws, L.gb_off, L.m, L.ld_g)


def read_x(k: int, ws: torch.Tensor, state: torch.Tensor, L: MatLayout) -> torch.Tensor:
    """[m, ld_x] bf16 view of iterate X_k (k = 0, 1)."""
    return _bf16(ws if L.x_in_ws else state, L.x_off[k], L.m, L.ld_x)


def fma32(a: torch.Tensor, b: torch.Tensor, c: torch.Tensor) -> torch.Tensor:
    """fmaf(a, b, c) elementwise for fp32 tensors: one rounding of the exact a b + c.

    a b is exact in float64 (48 significant bits).  The float64 sum s = a b + c is exact up to a
    remainder e (TwoSum); rounding s to fp32 is the correct rounding of s + e except when s lies
    exactly halfway between two fp32 values and e != 0, where e's sign picks the neighbour."""
    p = a.double() * b.double()
    c = c.double()
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)
    r = s.float()
    other = torch.nextafter(r, torch.where(s > r.double(), torch.full_like(r, float("inf")),
                                           torch.full_like(r, -float("inf"))))
    half = (s - r.double()).abs() == (other.double() - s).abs()
    toward_other = (e != 0) & ((e > 0) == (other.double() > s))
    return torch.where(half & (e != 0), torch.where(toward_other, other, r), r)


def lerp32(e: torch.Tensor, x: torch.Tensor, w: float) -> torch.Tensor:
    """torch's fp32 lerp as the kernels compute it (``muon_oracle._lerp32`` with fused
    multiply-adds): |w| < 0.5 ? fmaf(w, x - e, e) : fmaf(-(x - e), 1 - w, x)."""
    e, x = e.float(), x.float()
    w32 = torch.tensor(w, dtype=torch.float32, device=e.device)
    d = x - e
    if abs(float(w32)) < 0.5:
        return fma32(w32.expand_as(d), d, e)
    return fma32(-d, (1 - w32).expand_as(d), x)


def gemm_bound(a: torch.Tensor, b: torch.Tensor, p: torch.Tensor, k: int, alpha_add=None, beta: float = 1.0):
    """Largest |out - P| a bf16 GEMM output may show, in float64 (see the GPU test's docstring).

    ``a @ b`` is the float64 product over k terms, ``p`` the float64 reference; ``alpha_add`` the
    float64 alpha * addend of an epilogue that folds one in with an fp32 FMA (P = alpha Add + beta
    A B)."""
    ab = a.abs() @ b.abs()
    bound = abs(beta) * k * 2.0 ** -24 * ab + 2.0 ** -8 * p.abs()
    if alpha_add is not None:
        bound = bound + 2.0 ** -23 * (alpha_add.abs() + abs(beta) * ab)
    return bound


K12_PATHS = ("one_kblock", "kstages_kblocks", "kstages_plus_one", "many_kblocks", "single_tile",
             "tiles_m_16_two_per_cta", "tiles_m_17_just_above_sms", "two_sms_plus_one_tiles")


def k12_shapes(sms: int):
    """K12 shapes (rows, out, in) that reach each path of the tile walk on ``sms`` SMs."""
    just_above = -(-(sms + 1) // 17)              # tiles_n with 17 row blocks and > sms tiles
    t = 2 * sms + 1
    tm = next((d for d in range(2, t + 1) if t % d == 0 and d % 16), t)
    return {
        "one_kblock": (32, 256, 512),
        "kstages_kblocks": (K_STAGES * K12_BK, 256, 512),
        "kstages_plus_one": ((K_STAGES + 1) * K12_BK, 256, 512),
        "many_kblocks": (4096, 256, 512),
        "single_tile": (224, BM, BN),
        "tiles_m_16_two_per_cta": (224, 16 * BM, 2 * sms // 16 * BN + BN),
        "tiles_m_17_just_above_sms": (4096, 17 * BM, just_above * BN),
        "two_sms_plus_one_tiles": (192, tm * BM, t // tm * BN),
    }


def k13_tiles_shapes(sms: int):
    """K13 shapes (rows, k, cols) with 16 and 17 row blocks, tile counts just above ``sms``."""
    return {
        "tiles_m_16": (16 * BM, 72, -(-(sms + 1) // 16) * BN),
        "tiles_m_17": (17 * BM, 72, -(-(sms + 1) // 17) * BN),
    }
