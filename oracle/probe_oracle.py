"""numpy statement of the zero gate's alias probe (include/ccm.h: ccm_scrub_probe).

ORACLE — TEST INFRASTRUCTURE ONLY.  Restates, independently of the CUDA code, what the three probe steps find:

    a probe window is the 32-byte sector at every address that is a multiple of 4096 and lies entirely inside one
    mapped chunk; the windows of a chunk [a, a + n) start at w0 = roundup(a, 4096), and there are
    (a + n - 32 - w0) // 4096 + 1 of them when w0 + 32 <= a + n, none otherwise.

Each step runs over every chunk in mapping order before the next step starts:
    P1  the tags of `seed` (tag_oracle) into every window;
    "probe_mismatch" = k XORs the first byte of each of the first k windows (in launch order) with 0xA5;
    P2  every window compared with its tags, the bytes that differ counted and booked as 16-byte windows, then zeroed;
    "probe_dirt" = k XORs the same bytes with 0xA5;
    P3  every window's non-zero bytes counted.

An alias (`alias` = (view2, view1, n0)): [view2, view2 + n0) is a second virtual view of [view1, view1 + n0).  The window
at view2 + x and the one at view1 + x are the same physical sector (x is a multiple of 4096 in both, since both views
start on a page).  This oracle works per window on arrays of addresses and their physical sector; the CPU test holds it
against a byte-level model of pages and a page table.
"""
from __future__ import annotations

import numpy as np

import mismatch_oracle as MO
import tag_oracle as TO

STRIDE = 4096            # include/ccm.h: CCM_PROBE_STRIDE
WINDOW = 32              # include/ccm.h: CCM_PROBE_WINDOW
PAGE = 2 << 20           # include/ccm.h: CCM_PAGE_BYTES
XOR = 0xA5


def chunk_windows(addr: int, n: int) -> tuple:
    """(w0, count) of the windows of the chunk [addr, addr + n)."""
    w0 = -(-addr // STRIDE) * STRIDE
    return w0, ((addr + n - WINDOW - w0) // STRIDE + 1) if w0 + WINDOW <= addr + n else 0


def windows(chunks) -> np.ndarray:
    """Addresses of every window, in launch order: chunk by chunk ((addr, bytes) in mapping order), ascending inside."""
    parts = []
    for a, n in chunks:
        w0, k = chunk_windows(a, n)
        parts.append(w0 + STRIDE * np.arange(k, dtype=np.uint64))
    return np.concatenate(parts).astype(np.uint64) if parts else np.zeros(0, np.uint64)


def expected(chunks, seed: int, va_base: int, alias=None, probe_mismatch: int = 0, probe_dirt: int = 0,
             ranges=None, classify_limit: int = 4096) -> dict:
    """What the probe of `chunks` finds: windows, P2's bytes, its 16-byte windows (offset from va_base, mask, the bytes
    as read, kind and source offset; kinds only when there are at most `classify_limit` windows) and its page map
    {page: bytes}, and P3's bytes.  `ranges`: what the ALIAS search covers (default: the chunks).

    A window whose sector no other window shares, and that no drill touches, reads back exactly its own tags and then
    zero: only the others are followed, in launch order."""
    w = windows(chunks)
    nw = w.size
    phys = w.copy()
    if alias is not None:
        view2, view1, n0 = alias
        inside = (w >= view2) & (w < view2 + n0)
        phys[inside] = w[inside] - np.uint64(view2 - view1)
    _, inv, counts = np.unique(phys, return_inverse=True, return_counts=True)
    followed = counts[inv] > 1
    followed[:min(max(probe_mismatch, probe_dirt), nw)] = True
    idx = np.flatnonzero(followed)
    sector = {}
    for i in idx:                                   # P1, in launch order: the last writer of a sector wins
        sector[int(phys[i])] = bytearray(TO.tag_bytes(seed, int(w[i]), WINDOW).tobytes())
    for i in range(min(probe_mismatch, nw)):
        sector[int(phys[i])][0] ^= XOR
    read = {}
    for i in idx:                                   # P2, in launch order: read the sector, then zero it
        s = sector[int(phys[i])]
        read[int(i)] = bytes(s)
        s[:] = bytes(WINDOW)
    for i in range(min(probe_dirt, nw)):
        sector[int(phys[i])][0] ^= XOR
    p3 = sum(sum(1 for b in sector[int(phys[i])] if b) for i in idx)
    ranges = [(a, a + n) for a, n in chunks] if ranges is None else ranges
    recs, pages, total = [], {}, 0
    for i in idx:
        tags = TO.tag_bytes(seed, int(w[i]), WINDOW).tobytes()
        got = read[int(i)]
        for h in (0, 1):
            mask = sum(1 << b for b in range(16) if got[16 * h + b] != tags[16 * h + b])
            if not mask:
                continue
            off = int(w[i]) + 16 * h - va_base
            nbytes = bin(mask).count("1")
            total += nbytes
            pages[off // PAGE] = pages.get(off // PAGE, 0) + nbytes
            recs.append({"offset": off, "mask": mask, "bytes": got[16 * h:16 * h + 16].hex(), "kind": None,
                         "source_offset": 0})
    if len(recs) <= classify_limit:
        for r in recs:
            r["kind"], r["source_offset"] = classify(r, seed, va_base, ranges)
    recs.sort(key=lambda r: r["offset"])
    return {"windows": nw, "bytes_probed": nw * WINDOW, "mismatch_bytes": total, "mismatch_windows": len(recs),
            "zero_windows": sum(1 for r in recs if not any(bytes.fromhex(r["bytes"]))), "records": recs,
            "pages": pages, "reread_nonzero_bytes": p3}


def classify(rec: dict, seed: int, va_base: int, ranges) -> tuple:
    """(kind, source offset from va_base) of one record of `expected` (mismatch_oracle's classes)."""
    kind, src = MO.classify(seed, va_base + rec["offset"], bytes.fromhex(rec["bytes"]), 0xFFFF, ranges)
    return kind, (src - va_base) if src is not None else 0
