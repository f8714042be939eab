"""The coverage ledger's expected per-slot counts, restated in plain Python (include/ccm.h: ccm_cover_ledger).

Every pass of a proving call counts, per 128 KiB slot from the call's va_base, the bytes each of its threads addressed.
A clean call counts min(128 KiB, mapped - s * 128 KiB) on slot s of every pass that ran.  Three drills change one
launch of one pass (which launch: tests/cover_oracle.py, first_launch):
  cover_skip k       the launch never takes the first k chunks it would grab (the read-back: the last k);
  cover_repeat k     the first launch of the pass whose range starts on a page boundary of the map and holds at least a
                     page runs as [a, a + page - k chunks), [a + page, end) and [a, a + k chunks) again: the slots of
                     chunks 0..k-1 of that page count twice, those of chunks 16-k..15 not at all;
  cover_lane_drop t  thread t skips its share of the launch's first chunk: PER_THREAD x 16 bytes fewer on its slot
                     (256 for the scrub, census and tag kernels, 128 for the read-back), whatever t is.
"""
from __future__ import annotations

import cover_oracle as CO

SLOT = 128 << 10
PAGE = CO.PAGE
PASSES = CO.PASSES
SHARE = {"first": 16 * 16, "check": 16 * 16, "readback": 8 * 16}   # PER_THREAD x 16 bytes of one thread's share


def expected(mapped: int, nslots: int | None = None) -> list[int]:
    """Bytes every pass that ran must count on each slot (nslots: the ledger's slots, past the mapping 0)."""
    want = [min(SLOT, mapped - s) for s in range(0, mapped, SLOT)]
    return want + [0] * ((nslots or len(want)) - len(want))


def add(counts: list[int], lo: int, hi: int, sign: int) -> None:
    """Adds sign x the bytes of offsets [lo, hi) to the slots they lie on."""
    for s in range(lo // SLOT, -(-hi // SLOT)):
        counts[s] += sign * max(0, min(hi, (s + 1) * SLOT) - max(lo, s * SLOT))


def first_repeat_launch(pass_: str, tagged: bool, ranges, mappings, interleave: bool, mapped: int):
    """(offset, bytes) of the launch "cover_repeat" acts on: the pass's first launch that starts on a page boundary and
    holds at least a page (None: no such launch)."""
    if pass_ == "check":
        src = ranges if tagged else []
    elif pass_ == "first":
        src = mappings if tagged else ranges
    else:
        src = ranges if interleave else ([(0, mapped)] if mapped else [])
    return next(((o, n) for o, n in src if o % PAGE == 0 and n >= PAGE), None)


def ledger(mapped: int, tagged: bool, drill: tuple | None = None, nslots: int | None = None) -> dict:
    """The ledger's rows and inexact slots of a call that mapped `mapped` bytes (va_base 128-aligned, every launch's
    range 128-aligned).  drill = (name, pass, value, offset, bytes) of the drilled launch, name one of "skip", "repeat",
    "drop"; None for a clean call."""
    ran = {"first": True, "check": tagged, "readback": True}
    want = expected(mapped, nslots)
    got = {p: list(want) for p in PASSES}
    if drill is not None and ran[drill[1]]:
        name, pass_, value, off, n = drill
        c = got[pass_]
        if name == "skip":
            lo, hi = CO.skipped(off, off, n, value, pass_ == "readback")
            add(c, lo, hi, -1)
        elif name == "repeat":
            add(c, off, off + value * SLOT, +1)
            add(c, off + PAGE - value * SLOT, off + PAGE, -1)
        elif name == "drop":
            head, _, _ = CO.split_region(off, n)
            c[(off + head) // SLOT] -= SHARE[pass_]
    rows, slots = {}, []
    for p in PASSES:
        if not ran[p]:
            rows[p] = {"ran": 0}
            continue
        short = [i for i, (g, w) in enumerate(zip(got[p], want)) if g < w]
        over = [i for i, (g, w) in enumerate(zip(got[p], want)) if g > w]
        rows[p] = {"ran": 1, "slots_short": len(short), "slots_over": len(over),
                   "bytes_missing": sum(w - g for g, w in zip(got[p], want) if g < w),
                   "bytes_extra": sum(g - w for g, w in zip(got[p], want) if g > w), "bytes_outside": 0,
                   "first_short_slot": short[0] if short else 0, "first_over_slot": over[0] if over else 0}
    for i, w in enumerate(want):
        if any(ran[p] and got[p][i] != w for p in PASSES):
            c = [got[p][i] if ran[p] else 0 for p in PASSES]
            slots.append({"slot": i, "expected": w, "first": c[0], "check": c[1], "readback": c[2]})
    exact = all(rows[p].get("bytes_missing", 0) == 0 and rows[p].get("bytes_extra", 0) == 0 for p in PASSES)
    return {"exact": int(exact), "slots_mapped": -(-mapped // SLOT), "passes": rows, "slots": slots}
