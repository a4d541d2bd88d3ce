"""TEST INFRASTRUCTURE for Adafactor (K2-af).

* ``adafactor_step``: a float64 numpy restatement of one step of one tensor, written from the rule
  in include/frl_b200.h (K2-af), which is ``torch.optim.Adafactor``'s with foreach=False.
* ``AdafactorKernelDouble``: ``oracle.optim_np.KernelDouble`` plus a CPU stand-in for
  ``_native.adafactor_mt`` that reads each gradient where the segment table points, so the host
  logic (and multi-rank runs under gloo) needs no GPU.  The band table comes from the library's
  host planner.
* ``AF_PATHS``: named segment tables that together reach every branch of the kernels' band
  walk listed in ``AF_BRANCHES``; ``case_branches`` reads off the library's band table which ones
  a case reaches.

Never imported by the product.
"""
import dataclasses
from typing import Tuple

import numpy as np
import torch

from frl_b200 import _native
from frl_b200.fused_optim import adafactor_kernel_shape, adafactor_shape
from oracle.optim_np import KernelDouble
from adam8_oracle import _read


def _lerp(e, x, w):
    return e + w * (x - e) if abs(w) < 0.5 else x - (x - e) * (1.0 - w)


def _pymax(lo, x):
    return x if x > lo else lo


def adafactor_step(p, g, state, shape, *, lr, t, beta2_decay=-0.8, eps1=2.0 ** -23, eps2=1e-3, d=1.0, wd=0.0,
                   info=None):
    """One step of one tensor in float64.  ``p``, ``g``: flat arrays; ``state``: dict with ``row_var``
    [B, R] and ``col_var`` [B, C], or ``variance`` [numel].  Returns the new p; updates ``state``.
    ``info``, a dict, receives which side of each branch the step took: ``rms_p`` (alpha is
    eps2 * rho below eps2), ``x`` = RMS(u) / d (the update is clipped above 1), ``row_mean`` [B]
    before its eps1 clamp (factored only) and ``vhat_min``, the smallest vhat before its eps1^2
    clamp."""
    p = np.asarray(p, dtype=np.float64).copy()
    g = np.asarray(g, dtype=np.float64)
    B, R, C = adafactor_shape(shape)
    w = float(t) ** beta2_decay
    rho = min(lr, 1.0 / float(t) ** 0.5)
    with np.errstate(invalid="ignore", over="ignore"):
        rms_p = float(np.sqrt((p * p).sum())) / p.size ** 0.5
        alpha = _pymax(eps2, rms_p) * rho
        p *= 1.0 - lr * wd
        if R:
            g3 = g.reshape(B, R, C)
            rv = state["row_var"] = _lerp(state["row_var"], (g3 * g3).sum(axis=2) / C, w)
            cv = state["col_var"] = _lerp(state["col_var"], (g3 * g3).sum(axis=1) / R, w)
            m = rv.mean(axis=1)
            den = np.where(m < eps1, eps1, m)
            vhat = (rv[:, :, None] * cv[:, None, :] / den[:, None, None]).ravel()
        else:
            vhat = state["variance"] = _lerp(state["variance"], g * g, w)
        u = 1.0 / np.sqrt(np.where(vhat < eps1 * eps1, eps1 * eps1, vhat)) * g
        x = float(np.sqrt((u * u).sum())) / (u.size ** 0.5 * d)
        denom = _pymax(1.0, x)
    if info is not None:
        info.update(rms_p=rms_p, x=x, vhat_min=float(vhat.min()))
        if R:
            info["row_mean"] = m
    return p + (-alpha / denom) * u


def zero_state(shape):
    B, R, C = adafactor_shape(shape)
    if R:
        return {"row_var": np.zeros((B, R)), "col_var": np.zeros((B, C))}
    return {"variance": np.zeros(C)}


class AdafactorKernelDouble(KernelDouble):
    LW_ADAPTED, LW_CLIPPED = 1, 2

    adafactor_plan = staticmethod(_native.adafactor_plan)
    adafactor_scratch_bytes = staticmethod(_native.adafactor_scratch_bytes)

    def adafactor_mt(self, p, state, p_lp, table, plan, *, lr, beta2_decay, eps1, eps2, d, wd, step,
                     grad_scale=1.0, grad_scale_dev=None, dyn=None):
        self.calls.append(("adafactor_mt", table.n_segs))
        shape_dev, off, flags, _, _, _, _ = plan
        c = float(grad_scale_dev.item()) if grad_scale_dev is not None else 1.0
        fl, offs = flags.tolist(), off.tolist()
        for i, s in enumerate(table.slots):
            if s.numel == 0:
                continue
            row = table._segs[i]
            g = _read(row.g, s.numel, row.g_dtype).astype(np.float32) * np.float32(grad_scale)
            if fl[i] & self.LW_CLIPPED:
                g = g * np.float32(c)
            B, R, C = adafactor_shape(s.shape)
            o = offs[i]
            if R:
                st = {"row_var": state[o:o + B * R].double().numpy().reshape(B, R),
                      "col_var": state[o + B * R:o + B * (R + C)].double().numpy().reshape(B, C)}
            else:
                st = {"variance": state[o:o + C].double().numpy()}
            w = adafactor_step(p[s.offset:s.end].double().numpy(), g, st, s.shape, lr=lr, t=step,
                               beta2_decay=beta2_decay, eps1=eps1, eps2=eps2, d=d, wd=wd)
            p[s.offset:s.end] = torch.from_numpy(w).float()
            flat = np.concatenate([st["row_var"].ravel(), st["col_var"].ravel()]) if R else st["variance"]
            state[o:o + flat.size] = torch.from_numpy(flat).float()
            if p_lp is not None and s.is_model:
                p_lp[s.offset:s.end] = torch.from_numpy(w).to(p_lp.dtype)


# ---- the path catalogue ----------------------------------------------------------------------------

AF_ROWS, AF_COLS = 64, 1024          # kAfRows, kAfCols: a band is up to 64 rows x 1024 columns
AF_CHUNK = 16 * AF_COLS              # kAfChunk: elements per chunk of a 0/1-D tensor
# Most CTAs of 256 threads an H100 SXM holds at once (132 SMs x 2048 threads): a table with more
# bands than this makes every CTA of the launch grid-stride.
H100_RESIDENT_CTAS = 132 * (2048 // 256)


@dataclasses.dataclass(frozen=True)
class AfCase:
    """One segment table for K2-af.  ``shapes``: the parameters, in arena order.  ``gdt``: the
    gradient dtype of each slot, cycled.  ``g_offset``: each gradient is a view at this element
    offset into a larger allocation (0: an allocation of its own, 16-byte aligned).  ``model``:
    whether each slot is a model parameter, which takes the clip coefficient, cycled.
    ``reaches``: the branches of ``AF_BRANCHES`` the case exists for."""
    shapes: Tuple[Tuple[int, ...], ...]
    reaches: Tuple[str, ...] = ()
    gdt: Tuple[torch.dtype, ...] = (torch.float32,)
    g_offset: int = 0
    model: Tuple[bool, ...] = (True,)

    def slot_gdt(self, i):
        return self.gdt[i % len(self.gdt)]

    def slot_model(self, i):
        return self.model[i % len(self.model)]


def _hundreds_of_matrices():
    rng = np.random.default_rng(2024)
    shapes = [tuple(int(x) for x in rng.integers(1, 81, size=2)) for _ in range(400)]
    shapes += [(2,) + tuple(int(x) for x in rng.integers(1, 41, size=2)) for _ in range(80)]
    return tuple(shapes) + ((600, 2, 3), (4096,))


AF_BRANCHES = (
    "band_b_rb_cb_all_positive",     # column partial at B*R*n_cb + (b*n_rb + rb)*C + c with all three > 0
    "row_mean_R_below_32",           # each matrix's row mean summed by one thread
    "row_mean_R_32_or_more",         # ... by the whole CTA
    "last_row_band_short",           # a matrix's last row band has fewer than 64 rows, after others
    "last_col_band_short",           # ... its last column band fewer than 1024 columns
    "thread_cols_partial",           # C % 4 != 0: a thread owns 1 to 3 columns
    "last_chunk_short",              # a 0/1-D tensor's last chunk is short, after full ones
    "chunk_exactly_full",            # ... ends exactly on a chunk edge
    "single_short_chunk",            # ... is one short chunk
    "zero_dim",
    "zero_element_segments",         # segments without a band amid ones with bands
    "hundreds_of_segments",          # several hundred segments share the ticket array
    "n_work_above_resident_grid",    # more bands than H100_RESIDENT_CTAS: every CTA grid-strides
    "mixed_grad_dtypes",             # fp32 and bf16 gradients in one table
    "scalar_rows_f32",               # C % 4 == 0 but the gradient misaligned for a 16-byte load
    "scalar_rows_bf16",              # ... for an 8-byte load
    "vector_rows",                   # C % 4 == 0 and aligned: the vector loads and stores
    "clip_on_some_segments",         # the clip coefficient reaches some segments only
)

AF_PATHS = {
    "b1_row_and_col_bands": AfCase(((130, 2100),), ("last_row_band_short", "last_col_band_short", "vector_rows")),
    "batched_row_and_col_bands": AfCase(((3, 130, 2100), (2, 2, 65, 1025)),
                                        ("band_b_rb_cb_all_positive", "thread_cols_partial")),
    "rows_around_32_and_64": AfCase(tuple((r, 40) for r in (1, 31, 32, 33, 63, 64, 65)) + ((4, 31, 12), (4, 32, 12),
                                                                                           (128, 8)),
                                    ("row_mean_R_below_32", "row_mean_R_32_or_more", "last_row_band_short")),
    "cols_around_4_and_1024": AfCase(tuple((6, c) for c in (1, 3, 4, 1023, 1024, 1025)) + ((2, 3, 2049),),
                                     ("thread_cols_partial", "last_col_band_short")),
    "tall_skinny": AfCase(((70001, 3),), ("last_row_band_short", "thread_cols_partial", "n_work_above_resident_grid")),
    "wide_single_row": AfCase(((1, 100000),), ("last_col_band_short", "row_mean_R_below_32")),
    "vector_chunks": AfCase(((16383,), (16384,), (16385,), (40000,), ()),
                            ("last_chunk_short", "chunk_exactly_full", "single_short_chunk", "zero_dim")),
    "zero_element_tensors": AfCase(((0, 7), (5, 6), (3, 0, 2), (0,), (9,), (2, 0)), ("zero_element_segments",)),
    "hundreds_of_matrices": AfCase(_hundreds_of_matrices(), ("hundreds_of_segments", "n_work_above_resident_grid")),
    "mixed_grad_dtypes": AfCase(((37, 130), (64, 1024), (2, 33, 1025), (1000,), (16385,), (5, 4)), ("mixed_grad_dtypes",),
                                gdt=(torch.float32, torch.bfloat16)),
    "scalar_rows_f32": AfCase(((40, 1024), (3, 65, 8), (64, 4), (100,)), ("scalar_rows_f32",), g_offset=1),
    "scalar_rows_bf16": AfCase(((40, 1024), (3, 65, 8), (64, 4), (100,)), ("scalar_rows_bf16",),
                               gdt=(torch.bfloat16,), g_offset=1),
    "clip_on_some_segments": AfCase(((37, 130), (2, 70, 20), (1000,), (8, 4, 3, 3)), ("clip_on_some_segments",),
                                    model=(True, False)),
}


def case_shape_tensor(case):
    """The kernel's (B, R, C) rows of the case's slots, as ``FusedAdafactor`` builds them."""
    return torch.tensor([adafactor_kernel_shape(s) for s in case.shapes], dtype=torch.int64)


def case_branches(case):
    """The branches of ``AF_BRANCHES`` the case's table reaches, read off the library's band table."""
    shape = case_shape_tensor(case)
    work, seg_info = _native.adafactor_plan(shape)
    work = work.numpy()
    sh = shape.numpy()
    out = set()
    if work.shape[0] > H100_RESIDENT_CTAS:
        out.add("n_work_above_resident_grid")
    if len(case.shapes) >= 300:
        out.add("hundreds_of_segments")
    if len({case.slot_gdt(i) for i, s in enumerate(case.shapes) if np.prod(s, dtype=np.int64)}) > 1:
        out.add("mixed_grad_dtypes")
    if len({case.slot_model(i) for i in range(len(case.shapes))}) > 1:
        out.add("clip_on_some_segments")
    for i, s in enumerate(case.shapes):
        B, R, C = (int(x) for x in sh[i])
        w0, w1 = (int(x) for x in seg_info[i, :2])
        bands = work[w0:w1]
        if w0 == w1:
            out.add("zero_element_segments")
            continue
        if len(s) == 0:
            out.add("zero_dim")
        if R == 0:
            e0 = bands[:, 2]
            last = C - e0.max()
            if e0.max() > 0 and last < AF_CHUNK:
                out.add("last_chunk_short")
            if last == AF_CHUNK:
                out.add("chunk_exactly_full")
            if C < AF_CHUNK:
                out.add("single_short_chunk")
            continue
        out.add("row_mean_R_below_32" if R < 32 else "row_mean_R_32_or_more")
        b, r0, c0 = bands[:, 1], bands[:, 2], bands[:, 3]
        if ((b > 0) & (r0 > 0) & (c0 > 0)).any():
            out.add("band_b_rb_cb_all_positive")
        if ((r0 > 0) & (R - r0 < AF_ROWS)).any():
            out.add("last_row_band_short")
        if ((c0 > 0) & (C - c0 < AF_COLS)).any():
            out.add("last_col_band_short")
        if C % 4:
            out.add("thread_cols_partial")
            continue
        dt = case.slot_gdt(i)
        nbytes, align = (4, 16) if dt == torch.float32 else (2, 8)
        if case.g_offset * nbytes % align:
            out.add("scalar_rows_f32" if dt == torch.float32 else "scalar_rows_bf16")
        else:
            out.add("vector_rows")
    return out
