"""TEST INFRASTRUCTURE — numpy restatement of stochastic rounding to bf16 (K2-sr, include/frl_b200.h):
the 16 random bits of arena element i at update t and the rounding (bits(x) + r) >> 16.  Never
imported by the product."""
import numpy as np

from oracle.augment_np import philox4x32_10

SR_TAG = 0x53520000


def sr_bits(idx, t: int, seed: int) -> np.ndarray:
    """uint32 array: the 16 random bits (low half) of the arena elements ``idx`` at update ``t``."""
    idx = np.asarray(idx, dtype=np.int64).astype(np.uint64)
    q = idx >> np.uint64(2)
    words = philox4x32_10((q & np.uint64(0xFFFFFFFF), q >> np.uint64(32), np.uint64(t), np.uint64(SR_TAG)),
                          (seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF))
    w = np.stack(words, axis=-1)
    return (w[np.arange(w.shape[0]), (idx & np.uint64(3)).astype(np.int64)] & np.uint32(0xFFFF)).astype(np.uint32)


def sr_round(x, r) -> np.ndarray:
    """uint16 bf16 bit patterns of fp32 ``x`` rounded with the 16 random bits ``r``."""
    u = np.asarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    r = np.asarray(r, dtype=np.uint64) & np.uint64(0xFFFF)
    out = ((u + r) >> np.uint64(16)).astype(np.uint32) & np.uint32(0xFFFF)
    nan = (u & np.uint64(0x7FFFFFFF)) > np.uint64(0x7F800000)
    return np.where(nan, np.uint32(0x7FC0), out).astype(np.uint16)


def bf16_to_f32(bits) -> np.ndarray:
    return (np.asarray(bits, dtype=np.uint32) << np.uint32(16)).view(np.float32)


def sr_arena(x, lo: int, t: int, seed: int) -> np.ndarray:
    """SR of the fp32 values ``x`` of arena elements ``[lo, lo + len(x))`` at update ``t``: uint16."""
    x = np.asarray(x, dtype=np.float32).ravel()
    return sr_round(x, sr_bits(np.arange(lo, lo + x.size), t, seed))
