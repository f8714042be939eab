"""The dirt triage restated (include/ccm.h: ccm_scrub_triage): its runs, and the class of every page of a dirt page
map under the two triage drills.

After a failed read-back the triage takes every page of the dirt page map, intersects it with what the call mapped
(the mapping, or each cudaMalloc segment of the fallback: `spans`, as (offset, bytes) from the dirt report's va_base,
ascending) and merges adjacent pieces inside one span into maximal runs.  It re-zeroes every run (T1), re-reads it
(T2), holds, and re-reads it again (T3).  On memory that keeps what is stored, only the drills leave bytes for T2 and
T3: "triage_stay" = k XORs the first byte of each of the first k dirt pages with 0xA5 between T1 and T2,
"triage_return" = k the same bytes between T2 and T3.  So that byte reads non-zero at T2 when its page is among the
first `stay` pages, and at T3 when it is among exactly one of the first `stay` and the first `ret` pages.

    runs(pages, spans)                      [(offset, bytes, span index)] the runs of a dirt page map
    classify(entries, stay, ret)            [(page, chunk, class, dirt bytes, T2 bytes, T3 bytes)] per dirt page
    report(entries, spans, stay, ret)       the exact fields of ccm_triage_report
    brute_runs(pages, spans, unit)          runs() one `unit` of memory at a time (the definition, for tests)
"""
from __future__ import annotations

PAGE_BYTES = 2 << 20
STAYS, RETURNS, CLEARS = "stays", "returns", "clears"


def _page_list(pages) -> list:
    """Ascending page numbers of a dirt page map given as pages or (page, bytes, chunk) entries."""
    return sorted(p[0] if isinstance(p, tuple) else int(p) for p in pages)


def runs(pages, spans) -> list:
    """(offset, bytes, span) of every maximal run: each dirt page intersected with each span, adjacent pieces inside
    one span merged.  Launches of each triage step = len(runs(...))."""
    out: list = []
    for p in _page_list(pages):
        lo, hi = p * PAGE_BYTES, (p + 1) * PAGE_BYTES
        for k, (so, sn) in enumerate(spans):
            a, b = max(lo, so), min(hi, so + sn)
            if a >= b:
                continue
            if out and out[-1][2] == k and out[-1][0] + out[-1][1] == a:
                out[-1] = (out[-1][0], out[-1][1] + b - a, k)
            else:
                out.append((a, b - a, k))
    return out


def brute_runs(pages, spans, unit: int) -> list:
    """runs() by walking every `unit` bytes of every span (unit divides every page, span offset and length): a unit is
    examined when its page is dirty, and consecutive examined units of one span form a run."""
    dirty = set(_page_list(pages))
    out: list = []
    for k, (so, sn) in enumerate(spans):
        assert so % unit == 0 and sn % unit == 0 and PAGE_BYTES % unit == 0
        start = None
        for o in range(so, so + sn + unit, unit):
            inside = o < so + sn and o // PAGE_BYTES in dirty
            if inside and start is None:
                start = o
            elif not inside and start is not None:
                out.append((start, o - start, k))
                start = None
    return sorted(out)


def classify(entries, stay: int = 0, ret: int = 0) -> list:
    """(page, chunk, class, dirt bytes, T2 bytes, T3 bytes) of every (page, bytes, chunk) entry of a dirt page map,
    ascending, on memory that keeps what is stored, with the drills "triage_stay" = stay and "triage_return" = ret."""
    out = []
    for i, (page, nbytes, chunk) in enumerate(sorted(entries)):
        t2 = int(i < stay)
        t3 = int((i < stay) != (i < ret))
        cls = STAYS if t2 else RETURNS if t3 else CLEARS
        out.append((page, chunk, cls, nbytes, t2, t3))
    return out


def report(entries, spans, stay: int = 0, ret: int = 0) -> dict:
    """The exact fields of ccm_triage_report (all but the offsets' base, the times and the hold)."""
    rows = classify(entries, stay, ret)
    rs = runs(entries, spans)
    out = {"pages_examined": len(rows), "bytes_examined": sum(n for _, n, _ in rs), "runs": len(rs),
           "t2_bytes": sum(r[4] for r in rows), "t3_bytes": sum(r[5] for r in rows)}
    for cls, key in ((STAYS, "stay"), (RETURNS, "return"), (CLEARS, "clear")):
        out[f"{key}_pages"] = sum(1 for r in rows if r[2] == cls)
        out[f"{key}_bytes"] = sum(r[3] for r in rows if r[2] == cls)
    for t, col in (("t2", 4), ("t3", 5)):
        hit = [r[0] * PAGE_BYTES for r in rows if r[col]]
        out[f"{t}_first_offset"] = min(hit) if hit else 0
        out[f"{t}_last_offset"] = max(hit) if hit else 0
    return out


def drill_xors(entries, stay: int = 0, ret: int = 0) -> int:
    """xor_byte_kernel launches the two drills add."""
    n = len(list(entries))
    return min(stay, n) + min(ret, n)
