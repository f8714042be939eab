"""numpy statement of the tagged scrub gate's address tags.

ORACLE — TEST INFRASTRUCTURE ONLY.  Restates `tag_word` of
k8s_cc_manager_b200/csrc/scrub_kernels.cuh independently of the CUDA code:

    the 4-byte word at device address a (i = a >> 2) holds
        lo32(i) * 0x9E3779B1  ^  hi32(i) * 0x85EBCA77  ^  seed      (mod 2**32)
    the byte at address x is byte (x & 3), little-endian, of the word at x & ~3.

The tagged check counts, byte by byte, what differs from these tags, then zeroes.
"""
from __future__ import annotations

import numpy as np

K1 = 0x9E3779B1
K2 = 0x85EBCA77
BLOCK = 64 << 20  # bytes per numpy block in the counting helpers


def tag_word_py(seed: int, addr: int) -> int:
    """Pure-Python tag of the word containing address `addr` (small cases)."""
    i = addr >> 2
    return (((i & 0xFFFFFFFF) * K1) ^ ((i >> 32) * K2) ^ seed) & 0xFFFFFFFF


def tag_bytes(seed: int, addr: int, n: int) -> np.ndarray:
    """The n tag bytes of [addr, addr + n) as uint8."""
    if n == 0:
        return np.zeros(0, np.uint8)
    w0 = addr & ~3
    w1 = (addr + n + 3) & ~3
    i = np.arange(w0 >> 2, w1 >> 2, dtype=np.uint64)
    lo = (i & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    hi = (i >> np.uint64(32)).astype(np.uint32)
    words = (lo * np.uint32(K1)) ^ (hi * np.uint32(K2)) ^ np.uint32(seed & 0xFFFFFFFF)
    return words.astype("<u4").view(np.uint8)[addr - w0: addr - w0 + n]


def mismatch_count(buf: np.ndarray, seed: int, addr: int) -> int:
    """Bytes of `buf`, read at device address `addr`, that differ from their tags."""
    b = buf.view(np.uint8).reshape(-1)
    return sum(int(np.count_nonzero(b[o:o + BLOCK] != tag_bytes(seed, addr + o, min(BLOCK, b.size - o))))
               for o in range(0, b.size, BLOCK))


def wrong_seed_count(seed_written: int, seed_checked: int, addr: int, n: int) -> int:
    """Mismatches of a check with `seed_checked` over [addr, addr + n) holding the tags of `seed_written`."""
    return sum(int(np.count_nonzero(tag_bytes(seed_written, addr + o, min(BLOCK, n - o))
                                    != tag_bytes(seed_checked, addr + o, min(BLOCK, n - o))))
               for o in range(0, n, BLOCK))


def alias_counts(seed: int, base: int, n0: int) -> tuple:
    """Mismatch counts of the tagged gate when [base + n0, base + 2 n0) is a second view of [base, base + n0).

    Both views are tagged in address order, so the physical bytes hold the second view's tags T2 when the
    checks start.  Returns (exact, low, high):
      exact      the two views checked by separate launches, the first view first: the first view reads T2
                 (counts T2 != T1) and zeroes, the second view reads zeros (counts T2 != 0);
      low, high  both views inside ONE launch, in any interleaving: a byte counts [T2 != T1] (both read T2),
                 [T2 != T1] + [T2 != 0] (the first view reads first) or [T1 != 0] (the second view does).
    """
    exact = low = high = 0
    for o in range(0, n0, BLOCK):
        m = min(BLOCK, n0 - o)
        t1 = tag_bytes(seed, base + o, m)
        t2 = tag_bytes(seed, base + n0 + o, m)
        a = (t2 != t1).astype(np.int64)
        b = a + (t2 != 0)
        c = (t1 != 0).astype(np.int64)
        exact += int(b.sum())
        low += int(np.minimum(a, c).sum())
        high += int(np.maximum(b, c).sum())
    return exact, low, high
