"""Where the non-zero bytes of a buffer are: the dirt report of include/ccm.h (ccm_dirt_report), restated in numpy.

A dirty window is a 16-byte, 16-aligned ADDRESS window that holds at least one non-zero byte of the buffer; the
buffer starts at device address `base`, so its first and last windows may stick out of it.  Offsets are relative
to `base` (a window that starts before the buffer has a negative offset); bytes outside the buffer count as zero.
"""
from __future__ import annotations

import numpy as np

RECORDS = 64   # include/ccm.h: CCM_DIRT_RECORDS


def report(buf: np.ndarray, base: int) -> dict:
    """The exact report of `buf` (1-D uint8) placed at address `base`: counts, first / last non-zero byte, and
    EVERY dirty window as (offset, mask, bytes hex), ascending.  The library keeps at most RECORDS of them."""
    buf = np.ascontiguousarray(buf, dtype=np.uint8).ravel()
    n = buf.size
    nz = np.flatnonzero(buf).astype(np.int64)
    out = {"nonzero_bytes": int(nz.size), "dirty_windows": 0, "first_offset": None, "last_offset": None,
           "truncated": False, "windows": []}
    if nz.size == 0:
        return out
    addr = nz + (base % 16)                      # address minus the 16-aligned address below `base`
    win, inv = np.unique(addr >> 4, return_inverse=True)
    mask = np.zeros(win.size, dtype=np.int64)
    np.bitwise_or.at(mask, inv, np.left_shift(1, addr & 15))
    start = win * 16 - (base % 16)               # window offsets relative to base
    idx = start[:, None] + np.arange(16)[None, :]
    inside = (idx >= 0) & (idx < n)
    data = np.where(inside, buf[np.clip(idx, 0, n - 1)], 0).astype(np.uint8)
    out.update(dirty_windows=int(win.size), first_offset=int(nz[0]), last_offset=int(nz[-1]),
               truncated=bool(win.size > RECORDS),
               windows=[(int(o), int(m), data[i].tobytes().hex()) for i, (o, m) in enumerate(zip(start, mask))])
    return out


def window_count(base: int, n: int) -> int:
    """Windows a buffer of n bytes at `base` touches (every one is dirty when every byte is)."""
    return 0 if n == 0 else ((base + n - 1) >> 4) - (base >> 4) + 1
