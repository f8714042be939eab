"""The coverage proof's expected per-page counts, restated in plain Python (include/ccm.h: ccm_scrub_prove).

Every pass of a proving call counts the bytes its kernels processed on each 2 MiB page from the call's va_base.  A
clean call counts min(2 MiB, mapped - p * 2 MiB) on page p of every pass that ran.  The "cover_skip" drill writes k
into the grab word of the first launch of one pass: that launch's kernel then never takes the first k chunks it would
grab.  Its chunks are 128 KiB of the range's body, where the body is what split_region (scrub_kernels.cuh) leaves
between the ragged head (up to the next 128-byte boundary) and the vectors after the last whole chunk; the scrub,
census, tag fill and tag check grab them upwards, the read-back downwards.  So the skipped bytes are the first k
chunks of the body (the read-back: the last k), and nothing else of the call changes.

Which launch is first in each pass follows the plan of tests/product_plan.py (call_launches): the first pass (scrub
or census) and the tagged check run one launch per enqueued range; the tag fill runs one per mapping (main chunk or tail granule; the
fallback: segment); the read-back one per enqueued range when it is interleaved, else one over the whole mapping.
"""
from __future__ import annotations

import product_plan as PP

PAGE = 2 << 20
CHUNK = 128 << 10
ALIGN = 128
PASSES = ("first", "check", "readback")
DRILL_PASS = {0: "readback", 1: "first", 2: "check", 3: "readback"}   # sim key "cover_pass"


def split_region(addr: int, n: int) -> tuple[int, int, int]:
    """(head, body_vecs, tail) of split_region(p, n, 16, 128) for a range at address `addr`."""
    mis = addr & (ALIGN - 1)
    head = min(ALIGN - mis if mis else 0, n)
    body_vecs = (n - head) // 16
    return head, body_vecs, n - head - body_vecs * 16


def skipped(addr: int, off: int, n: int, k: int, descending: bool) -> tuple[int, int]:
    """[lo, hi) offsets (from va_base) a launch over [off, off + n) at address `addr` skips when its grab word starts
    at k."""
    head, body_vecs, _ = split_region(addr, n)
    nchunks = body_vecs * 16 // CHUNK
    k = min(k, nchunks)
    body = off + head
    if descending:
        return body + (nchunks - k) * CHUNK, body + nchunks * CHUNK
    return body, body + k * CHUNK


def expected(mapped: int) -> list[int]:
    """Bytes every pass that ran must count on each page of a call that mapped `mapped` bytes."""
    return [min(PAGE, mapped - p) for p in range(0, mapped, PAGE)]


def counts(mapped: int, skip: tuple[int, int] | None = None) -> list[int]:
    """Per-page counts of one pass that walked [0, mapped) except the offsets [lo, hi) of `skip`."""
    out = expected(mapped)
    if skip:
        lo, hi = skip
        for p in range(lo // PAGE, -(-hi // PAGE)):
            out[p] -= max(0, min(hi, (p + 1) * PAGE) - max(lo, p * PAGE))
    return out


def first_launch(pass_: str, tagged: bool, ranges: list[tuple[int, int]], mappings: list[tuple[int, int]],
                 interleave: bool, mapped: int) -> tuple[int, int] | None:
    """(offset, bytes) of the first launch of `pass_` in a call whose enqueued ranges are `ranges` and whose mappings
    (main chunks and tail granules, or fallback segments) are `mappings`; None when the pass does not run."""
    if pass_ == "check":
        return ranges[0] if tagged and ranges else None
    if pass_ == "first":
        src = mappings if tagged else ranges
        return src[0] if src else None
    if not interleave:
        return (0, mapped) if mapped else None
    return ranges[0] if ranges else None


def call_launches(nbytes: int, env: dict) -> tuple[list[tuple[int, int]], list[tuple[int, int]], bool, int]:
    """(enqueued ranges, mappings, interleave, mapped) of a call for `nbytes` (> 0) under the plan knobs `env`, from
    tests/product_plan.py: the VMM path's ranges and chunks, or (CCM_PIPELINE=0) the fallback's segments, which the
    fallback scrubs and reads back one by one."""
    if env.get("CCM_PIPELINE") == "0":
        segs = PP.arena_segments(nbytes, nbytes, env)
        return segs, segs, True, sum(n for _, n in segs)
    plan = PP.plan(nbytes, nbytes, PP.H100_GRAN, env)
    run = PP.simulate(plan, None)
    return run.ranges(plan), run.chunks, plan.interleave, run.mapped


def report(mapped: int, tagged: bool, drill: tuple[str, int, int, int] | None = None) -> dict:
    """The cover report's rows and inexact pages for a call that mapped `mapped` bytes at a va_base aligned to 128
    bytes.  drill = (pass, k, offset, bytes) of the drilled launch (first_launch), or None."""
    ran = {"first": True, "check": tagged, "readback": True}
    want = expected(mapped)
    got = {p: list(want) for p in PASSES}
    if drill is not None and ran[drill[0]]:
        pass_, k, off, n = drill
        got[pass_] = counts(mapped, skipped(off, off, n, k, pass_ == "readback"))
    rows, pages = {}, []
    for p in PASSES:
        if not ran[p]:
            rows[p] = {"ran": 0}
            continue
        short = [i for i, (g, w) in enumerate(zip(got[p], want)) if g < w]
        rows[p] = {"ran": 1, "bytes_counted": sum(got[p]), "bytes_missing": sum(want) - sum(got[p]),
                   "pages_short": len(short), "first_short_page": short[0] if short else 0}
    for i, w in enumerate(want):
        c = [got[p][i] if ran[p] else 0 for p in PASSES]
        if any(ran[p] and got[p][i] != w for p in PASSES):
            pages.append({"page": i, "expected": w, "first": c[0], "check": c[1], "readback": c[2]})
    return {"covered": all(rows[p].get("bytes_missing", 0) == 0 for p in PASSES), "passes": rows, "pages": pages}
