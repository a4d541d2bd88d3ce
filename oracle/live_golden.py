"""TEST INFRASTRUCTURE — the reference side of the tests that compare this package with the
reference on identical inputs.

Where the reference can be imported (``ref_shim.reference_available()``) the reference side is
computed live; with ``FRL_RECORD_GOLDEN=1`` it is also stored under ``tests/golden/live/``:

    FRL_RECORD_GOLDEN=1 python -m pytest tests/test_oracle_pinning.py tests/test_indexed_dataset.py

Elsewhere the stored recording is returned, so those tests run from the repository alone.
Recordings hold plain containers, strings, numbers and tensors only (``torch.load`` with
``weights_only=True``).
"""
import os

import torch

from oracle.ref_shim import reference_available

LIVE_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "live")


def reference_side(name, compute):
    """``(value, live)``: ``compute()`` run against the reference and ``True`` where it is
    present, else the recording of that value and ``False``."""
    path = os.path.join(LIVE_DIR, name + ".pt")
    if reference_available():
        value = compute()
        if os.environ.get("FRL_RECORD_GOLDEN") == "1":
            os.makedirs(LIVE_DIR, exist_ok=True)
            torch.save(value, path)
        return value, True
    return torch.load(path, weights_only=True), False


def plain(x):
    """``x`` with numpy arrays as tensors, numpy scalars as Python numbers and named tuples as
    tuples, so both sides of a comparison have the form a recording can hold."""
    import numpy as np
    if isinstance(x, np.ndarray):
        return torch.from_numpy(np.array(x, order="C", copy=True))
    if isinstance(x, np.generic):
        return x.item()
    if torch.is_tensor(x):
        return x.detach().clone()
    if isinstance(x, dict):
        return {k: plain(v) for k, v in x.items()}
    if isinstance(x, (list, tuple)):
        return type(x)(plain(v) for v in x) if type(x) in (list, tuple) else tuple(plain(v) for v in x)
    return x


def tensors_equal(a, b, live):
    """Bitwise where both sides ran on this machine; across machines, float results of the
    same ops may differ in the last bits (other SIMD paths), as for the other golden vectors."""
    if a.shape != b.shape:
        return False
    if live or not (a.is_floating_point() or b.is_floating_point()):
        return torch.equal(a, b)
    return torch.allclose(a.double(), b.double(), rtol=2e-6, atol=1e-7)
