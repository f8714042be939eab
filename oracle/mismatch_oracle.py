"""Where a tagged check found bytes off their tags: the mismatch report of include/ccm.h (ccm_mismatch_report),
restated in numpy from the bytes as the check read them.

ORACLE — TEST INFRASTRUCTURE ONLY.  The buffer starts at device address `addr`; a window is a 16-byte, 16-aligned
ADDRESS window, so the first and the last may stick out of the buffer (bytes outside it are neither compared nor
reported: they read as 0 and count as holding their tags).  `ranges` is what the call mapped, as (lo, hi) addresses;
the ALIAS search covers exactly them (default: the buffer).

Each mismatched window gets the first kind that fits:
    zero     every byte of it inside the buffer reads 0;
    alias    its bytes are exactly the tags of `seed` of ANOTHER 16-aligned window, every source byte inside
             `ranges`.  Decoded from the first whole word w at position k: for every hi = hi32(a >> 2) the ranges
             span, lo = (w ^ seed ^ hi * K2) * K1^-1 mod 2^32 and the candidate is 4 * (hi << 32 | lo) - 4 k;
             the ascending hi values are tried in order and the first candidate that fits wins;
    partial  some byte still holds its own tag;
    foreign  anything else.
"""
from __future__ import annotations

import numpy as np

from tag_oracle import K1, K2, tag_bytes, tag_word_py

RECORDS = 64                    # include/ccm.h: CCM_DIRT_RECORDS
K1_INV = pow(K1, -1, 1 << 32)


def tag_byte_py(seed: int, x: int) -> int:
    return (tag_word_py(seed, x & ~3) >> (8 * (x & 3))) & 0xFF


def _mapped(a: int, ranges) -> bool:
    return any(lo <= a < hi for lo, hi in ranges)


def decode_alias(seed: int, w: int, data: bytes, present: int, ranges):
    """Source address of an ALIAS window at address w (data: its 16 bytes, present: bit i = byte w + i is in the
    buffer), or None."""
    k = next((k for k in range(4) if (present >> (4 * k)) & 0xF == 0xF), None)
    if k is None:
        return None
    word = int.from_bytes(data[4 * k: 4 * k + 4], "little")
    his = sorted({h for lo, hi in ranges if hi > lo for h in range(lo >> 34, ((hi - 1) >> 34) + 1)})
    for h in his:
        lo32 = ((word ^ seed ^ (h * K2)) * K1_INV) & 0xFFFFFFFF
        src = 4 * (h << 32 | lo32) - 4 * k
        if src % 16 or src == w:
            continue
        if all(_mapped(src + i, ranges) and data[i] == tag_byte_py(seed, src + i) for i in range(16) if present >> i & 1):
            return src
    return None


def classify(seed: int, w: int, data: bytes, present: int, ranges):
    """(kind, source address or None) of one window."""
    idx = [i for i in range(16) if present >> i & 1]
    if all(data[i] == 0 for i in idx):
        return "zero", None
    src = decode_alias(seed, w, data, present, ranges)
    if src is not None:
        return "alias", src
    if any(data[i] == tag_byte_py(seed, w + i) for i in idx):
        return "partial", None
    return "foreign", None


def report(buf: np.ndarray, addr: int, seed: int, ranges=None, classify_limit: int = 4096) -> dict:
    """The exact report of `buf` (1-D uint8, as read) at `addr` checked against the tags of `seed`: counts, first /
    last mismatched byte (offsets from addr), and every mismatched window as a dict (offset, mask, zero, kind,
    source_offset, bytes hex), ascending.  Windows are classified only when there are at most `classify_limit`
    of them (kind None otherwise).  The library keeps at most RECORDS windows."""
    buf = np.ascontiguousarray(buf, dtype=np.uint8).ravel()
    n = buf.size
    ranges = [(addr, addr + n)] if ranges is None else list(ranges)
    diff = np.flatnonzero(buf != tag_bytes(seed, addr, n)).astype(np.int64)
    out = {"mismatch_bytes": int(diff.size), "mismatch_windows": 0, "zero_windows": 0, "first_offset": None,
           "last_offset": None, "truncated": False, "windows": []}
    if diff.size == 0:
        return out
    a16 = addr % 16
    win, inv = np.unique((diff + a16) >> 4, return_inverse=True)
    mask = np.zeros(win.size, dtype=np.int64)
    np.bitwise_or.at(mask, inv, np.left_shift(1, (diff + a16) & 15))
    start = win * 16 - a16
    idx = start[:, None] + np.arange(16)[None, :]
    inside = (idx >= 0) & (idx < n)
    data = np.where(inside, buf[np.clip(idx, 0, n - 1)], 0).astype(np.uint8)
    zero = ~np.any(data != 0, axis=1)
    present = (inside * (1 << np.arange(16))[None, :]).sum(axis=1)
    out.update(mismatch_windows=int(win.size), zero_windows=int(zero.sum()), first_offset=int(diff[0]),
               last_offset=int(diff[-1]), truncated=bool(win.size > RECORDS))
    do_kind = win.size <= classify_limit
    for i in range(win.size):
        kind, src = (classify(seed, addr + int(start[i]), data[i].tobytes(), int(present[i]), ranges)
                     if do_kind else (None, None))
        out["windows"].append({"offset": int(start[i]), "mask": int(mask[i]), "zero": bool(zero[i]), "kind": kind,
                               "source_offset": (src - addr) if src is not None else 0,
                               "bytes": data[i].tobytes().hex()})
    return out
