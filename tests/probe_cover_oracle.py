"""What the probe proof of a product call must count (include/ccm.h: ccm_probe_cover), restated in plain Python.

A call both proven and probed runs the proving twin of each probe step.  Each counts CCM_PROBE_WINDOW (32) bytes for
every window it took, on the 2 MiB page of the window's offset, where a window at address w of a chunk
(addr, bytes, offset) lies at offset `offset + (w - addr)`: for the VMM path the chunks are the mapping loop's
iterations from tests/product_plan.py, with offset = their place in the reserved range; on the cudaMalloc fallback
they are the segments, with offset = the bytes of the segments before them.  A window that crosses a page boundary
splits its bytes there (only possible on chunk offsets that are not multiples of 32).

The drill "probe_skip" = k, "probe_skip_step" = s: the first launch of step s (the first chunk with windows) starts
k windows later and takes k fewer, so step s misses exactly the first min(k, windows of that chunk) windows.
"""
from __future__ import annotations

STRIDE = 4096            # include/ccm.h: CCM_PROBE_STRIDE
WINDOW = 32              # include/ccm.h: CCM_PROBE_WINDOW
PAGE = 2 << 20           # include/ccm.h: CCM_PAGE_BYTES
STEPS = ("P1", "P2", "P3")


def chunk_windows(addr: int, n: int) -> tuple[int, int]:
    """(w0, count) of the probe windows of the chunk [addr, addr + n)."""
    w0 = -(-addr // STRIDE) * STRIDE
    return w0, ((addr + n - WINDOW - w0) // STRIDE + 1) if w0 + WINDOW <= addr + n else 0


def vmm_chunks(va_base: int, chunks: list[tuple[int, int]]) -> list[tuple[int, int, int]]:
    """The mapping loop's (offset, bytes) chunks as (address, bytes, offset)."""
    return [(va_base + off, n, off) for off, n in chunks]


def arena_chunks(segments: list[tuple[int, int]]) -> list[tuple[int, int, int]]:
    """The fallback's (address, bytes) segments as (address, bytes, offset into the concatenated segments)."""
    out, off = [], 0
    for a, n in segments:
        out.append((a, n, off))
        off += n
    return out


def _add(pages: dict, off: int, n: int) -> None:
    while n:
        p = off // PAGE
        take = min(n, (p + 1) * PAGE - off)
        pages[p] = pages.get(p, 0) + take
        off, n = off + take, n - take


def _count(chunks, skip_first: int = 0) -> dict:
    """{page: bytes} of the windows of `chunks`, the first `skip_first` windows of the first chunk with any left out."""
    pages: dict = {}
    pending = skip_first
    for a, n, off in chunks:
        w0, k = chunk_windows(a, n)
        if k == 0:
            continue
        s = min(pending, k)
        pending = 0
        o0 = off + (w0 - a) + s * STRIDE
        k -= s
        # whole runs of windows that start and end on one page, page by page
        i = 0
        while i < k:
            o = o0 + i * STRIDE
            p = o // PAGE
            last = min(k, i + ((p + 1) * PAGE - o + STRIDE - 1) // STRIDE)   # first window past page p
            if o0 + (last - 1) * STRIDE + WINDOW <= (p + 1) * PAGE:
                pages[p] = pages.get(p, 0) + (last - i) * WINDOW
            else:
                pages[p] = pages.get(p, 0) + (last - 1 - i) * WINDOW
                _add(pages, o0 + (last - 1) * STRIDE, WINDOW)
            i = last
    return {p: b for p, b in pages.items() if b}


def expected(chunks) -> dict:
    """{page: bytes} every step of a call over `chunks` must count."""
    return _count(chunks)


def windows(chunks) -> int:
    return sum(chunk_windows(a, n)[1] for a, n, _ in chunks)


def report(chunks, probe_skip: int = 0, probe_skip_step: int = 2) -> dict:
    """The probe proof of a call over `chunks` with the drill: per step the windows counted and missing, the pages short
    and the first short page, the inexact pages {page: (expected, [P1, P2, P3])}, and `covered`."""
    step = 2 if probe_skip_step == 0 else probe_skip_step
    want = expected(chunks)
    counted = [(_count(chunks, probe_skip) if k + 1 == step else want) for k in range(3)]
    steps = []
    for c in counted:
        short = sorted(p for p in want if c.get(p, 0) < want[p])
        missing = sum(want[p] - c.get(p, 0) for p in short)
        steps.append({"windows_counted": sum(c.values()) // WINDOW, "windows_missing": -(-missing // WINDOW),
                      "windows_extra": 0, "windows_outside": 0, "pages_short": len(short), "pages_over": 0,
                      "first_short_page": short[0] if short else 0})
    pages = {p: (want[p], [c.get(p, 0) for c in counted]) for p in sorted(want)
             if any(c.get(p, 0) != want[p] for c in counted)}
    return {"windows_expected": windows(chunks), "steps": steps, "pages": pages,
            "covered": int(all(s["windows_missing"] == 0 for s in steps))}
