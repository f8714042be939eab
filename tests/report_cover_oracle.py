"""What the report proof of a failed product call must count (include/ccm.h: ccm_report_cover), restated in plain
Python.

A proven call that located dirt or triaged runs the proving twin of every kernel of its locate pass and of each triage
step it runs.  Each step counts the bytes it walked on the 2 MiB page of their offset from the dirt or mismatch
report's va_base:
  LOCATE             every span of what the call holds (the mapping, or the cudaMalloc segments at their offsets);
  DIRT_T1..T3        the runs of the dirt page map (oracle/triage_oracle.py: runs), with the same spans;
  MISMATCH_T1..T3    the runs of the mismatch page map.
So page p of a step must count the bytes of its pieces on p, and their total is the step's bytes_expected (a triage's
bytes_examined).

The drill "report_skip" = k, "report_skip_step" = s writes k into the grab word of the first launch of step s: the
first span of the locate pass, or the first run of a triage.  That launch's kernel then never takes the first k
128 KiB chunks of its range's body (tests/cover_oracle.py: skipped, upwards), and nothing else of the call changes.
"""
from __future__ import annotations

import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
for _p in (ROOT / "oracle", ROOT / "tests"):
    if str(_p) not in sys.path:
        sys.path.insert(0, str(_p))

import cover_oracle as CO  # noqa: E402
import probe_oracle as PO  # noqa: E402
import triage_oracle as TO  # noqa: E402

PAGE = 2 << 20           # include/ccm.h: CCM_PAGE_BYTES
STEPS = ("LOCATE", "DIRT_T1", "DIRT_T2", "DIRT_T3", "MISMATCH_T1", "MISMATCH_T2", "MISMATCH_T3")


def pieces(step: str, spans: list[tuple[int, int]], dirt_pages=(), mismatch_pages=()) -> list[tuple[int, int]]:
    """(offset, bytes) of what step `step` walks, in launch order: the spans, or the runs of its triage's page map."""
    if step == "LOCATE":
        return list(spans)
    pages = dirt_pages if step.startswith("DIRT") else mismatch_pages
    return [(o, n) for o, n, _ in TO.runs(pages, spans)]


def per_page(parts: list[tuple[int, int]], skip: tuple[int, int] | None = None, base: int = 0) -> dict[int, int]:
    """Bytes of `parts` on each page from `base` (pages before it are negative), less the offsets [lo, hi) of
    `skip`."""
    out: dict[int, int] = {}
    for o, n in parts:
        a = o - base
        while a < o - base + n:
            b = min(o - base + n, (a // PAGE + 1) * PAGE)
            out[a // PAGE] = out.get(a // PAGE, 0) + b - a
            a = b
    if skip:
        lo, hi = skip
        for p in range(lo // PAGE, -(-hi // PAGE)):
            out[p] -= max(0, min(hi, (p + 1) * PAGE) - max(lo, p * PAGE))
    return out


def skipped(parts: list[tuple[int, int]], k: int) -> tuple[int, int] | None:
    """[lo, hi) offsets the first launch over `parts` skips when its grab word starts at k (ranges 128-byte aligned)."""
    if not parts or k == 0:
        return None
    o, n = parts[0]
    return CO.skipped(o, o, n, k, False)


def step_report(parts: list[tuple[int, int]], k: int = 0) -> dict:
    """The fields of ccm_report_cover_step for a step over `parts` whose first launch was drilled with k, and its
    inexact pages as (page, expected, counted)."""
    want = per_page(parts)
    got = per_page(parts, skipped(parts, k))
    short = sorted(p for p in want if got[p] < want[p])
    return {"launches": len(parts), "bytes_expected": sum(n for _, n in parts), "bytes_counted": sum(got.values()),
            "bytes_missing": sum(want[p] - got[p] for p in short), "bytes_extra": 0, "bytes_outside": 0,
            "pages_short": len(short), "pages_over": 0, "first_short_page": short[0] if short else 0,
            "pages": [(p, want[p], got[p]) for p in short]}


def brute_counts(parts: list[tuple[int, int]], unit: int, skip: tuple[int, int] | None = None,
                 base: int = 0) -> dict[int, int]:
    """per_page() one `unit` of memory at a time (the definition, for tests)."""
    out: dict[int, int] = {}
    for o, n in parts:
        for a in range(o, o + n, unit):
            if skip and skip[0] <= a < skip[1]:
                continue
            out[(a - base) // PAGE] = out.get((a - base) // PAGE, 0) + unit
    return out


# ---------------------------------------------------------------------------------- caller-owned maps (ccm_region_prove)
def cover_map(parts: list[tuple[int, int]], base: int, pages: int) -> list[int]:
    """The cover map a proving kernel fills walking `parts` ((address, bytes)) into a map of `pages` page words with
    page 0 at `base` (any base), and the outside slot last: every byte before base or on a page >= pages."""
    out = [0] * (pages + 1)
    for p, b in per_page(parts, base=base).items():
        out[p if 0 <= p < pages else pages] += b
    return out


def probe_parts(chunks: list[tuple[int, int]]) -> list[tuple[int, int]]:
    """What a probe step walks over `chunks` ((address, bytes), in launch order): CCM_PROBE_WINDOW bytes per window
    (oracle/probe_oracle.py: chunk_windows)."""
    out = []
    for a, n in chunks:
        w0, k = PO.chunk_windows(a, n)
        out += [(w0 + i * PO.STRIDE, PO.WINDOW) for i in range(k)]
    return out


def map_base(addr: int, n: int, run: int) -> tuple[int, int]:
    """(base, pages) of a map for one armed pass over [addr, addr + n), so that page boundaries cut it where the
    proving kernels split their counts.  A region longer than a page and two chunks gets every whole page that fits:
    its last boundary cuts the tail window (the last byte, or two when that boundary would fall on a chunk boundary,
    lie past it), so base is as unaligned as the region's end, and every other boundary cuts a 128 KiB chunk; the
    bytes before base, the ragged head with them, and those past the last page count outside.  A shorter region gets
    one boundary, chosen by `run` among: inside the ragged head, inside the first chunk, inside a leftover vector and
    before the last byte; with the bytes before it outside or (every other round of cuts) those from it on."""
    head = min((CO.ALIGN - addr % CO.ALIGN) % CO.ALIGN, n)
    nchunks = (n - head) // CO.CHUNK
    last = n - 1 if (n - 1 - head) % CO.CHUNK else n - 2
    if n >= PAGE + 2 * CO.CHUNK + head:
        pages = (last - head) // PAGE
        return addr + last - pages * PAGE, pages
    cuts = [c for c in (head // 2 + 1, head + CO.CHUNK // 2 + 3, head + nchunks * CO.CHUNK + 5, n - 1) if 0 < c < n]
    if not cuts:
        return addr, 1
    cut = addr + cuts[run % len(cuts)]
    return (cut, 1) if run // len(cuts) % 2 == 0 else (cut - PAGE, 1)
