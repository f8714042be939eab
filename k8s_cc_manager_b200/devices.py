"""Duck-typed device objects over libccm.so.

The reference manager never sees a C ABI: it calls methods on objects handed out by
`pci.devices.find_gpus()` of NVIDIA/gpu-admin-tools (reference main.py:38-40,155).
This module rebuilds exactly the attributes the reference touches (SURVEY.md §8b)
on top of include/ccm.h, and adds the one new capability, `scrub_and_verify()`.

    find_gpus() -> (devices, count)          reference main.py:155,164,174,203,275,473
    dev.bdf, dev.name                        main.py:187,191,210,239,280
    dev.is_gpu(), dev.is_nvswitch()          main.py:165,175
    dev.is_cc_query_supported  (attribute)   main.py:186
    dev.is_ppcie_query_supported (attribute) main.py:205,477
    dev.query_cc_mode() / set_cc_mode(m)     main.py:441,505,511,524
    dev.query_ppcie_mode() / set_ppcie_mode  main.py:310,340,345,353,359,373,479,482,495
    dev.reset_with_os() / wait_for_boot()    main.py:346-347,368,372,490,494,519,523
    GpuError                                 main.py:40,380,531

Errors: every non-zero ccm_status becomes a GpuError carrying `.status`.
"""
from __future__ import annotations

import ctypes as C
import dataclasses
from dataclasses import dataclass, field
from typing import List, Optional, Sequence, Tuple

from . import _native as N


class GpuError(Exception):
    """Raised for any failed device operation (reference: gpu.GpuError).  A scrub that read back dirt
    carries its DirtReport as `.dirt`; a tagged scrub whose check found bytes off their tags carries its
    MismatchReport as `.mismatch`; a census call carries its ResidueReport (what the first pass erased) as
    `.residue`; a triage call that read back dirt carries its TriageReport (what kind of dirt) as `.triage`; a mismatch
    triage call whose tagged check failed carries its TriageReport (what kind of mismatch) as `.mismatch_triage`; a
    proving call carries its CoverReport (how many bytes each pass walked on every page) as `.cover` and its
    CoverLedger (how many bytes every thread of each pass addressed on every 128 KiB slot) as `.ledger`; a probing call
    carries its ProbeReport (what the alias probe found) as `.probe`; a call both proving and probing carries its
    ProbeCoverReport (how many windows each probe step took on every page) as `.probe_cover`; a proving call that
    located dirt or triaged carries its ReportCoverReport (how many bytes the locate pass and each triage step walked on
    every page) as `.report_cover`; a call armed for the HBM health report carries its HbmHealth (the GPU's ECC and
    row-remapping state before and after the call) as `.health`."""

    def __init__(self, message: str, status: int = N.ERR_IO):
        super().__init__(message)
        self.status = status
        for attr, _ in _REPORTS:
            setattr(self, attr, None)


def _error(rc: int, what: str, bdf: str = "") -> "Optional[GpuError]":
    if rc == N.OK:
        return None
    detail = N.last_error()
    where = f" on {bdf}" if bdf else ""
    return GpuError(f"{what}{where}: {N.strerror(rc)}" + (f" ({detail})" if detail else ""), rc)


def _check(rc: int, what: str, bdf: str = "") -> None:
    err = _error(rc, what, bdf)
    if err is not None:
        raise err


def _signed64(x: int) -> int:
    return x - (1 << 64) if x >= 1 << 63 else x


PAGE_BYTES = N.PAGE_BYTES
PAGE_RUNS = 64      # runs a PageDigest keeps


@dataclass(frozen=True)
class PageRun:
    """A maximal stretch of consecutive 2 MiB pages in one chunk that all hold booked bytes."""
    first_page: int      # offset of its first byte from the report's va_base = first_page * PAGE_BYTES
    pages: int
    chunk: int
    bytes: int

    def describe(self) -> str:
        lo, hi = self.first_page * PAGE_BYTES, (self.first_page + self.pages) * PAGE_BYTES - 1
        return f"+{lo:#x}..+{hi:#x} chunk {self.chunk} {self.bytes} B"


@dataclass(frozen=True)
class ChunkPages:
    """The booked bytes of one chunk (physical allocation), and on how many of its pages they lie."""
    chunk: int
    pages: int
    bytes: int


@dataclass
class PageDigest:
    """What a report carries of its page map (its `pages` field, and its JSON): the page count, exact totals per chunk,
    and the first PAGE_RUNS runs."""
    pages: int                   # pages holding at least one booked byte
    bytes: int                   # booked bytes on them: the report's exact count
    nruns: int                   # runs of consecutive pages in one chunk (all of them)
    runs_truncated: int          # nruns > len(runs)
    by_chunk: List[ChunkPages] = field(default_factory=list)   # ascending chunk
    runs: List[PageRun] = field(default_factory=list)          # ascending, the first PAGE_RUNS

    @classmethod
    def from_json(cls, d: dict) -> "PageDigest":
        return cls(**{**d, "by_chunk": [ChunkPages(**c) for c in d["by_chunk"]],
                      "runs": [PageRun(**r) for r in d["runs"]]})

    def summary(self, first: int = 4) -> str:
        """One line for an operator: how many pages, the bytes of each chunk, and the first few runs."""
        chunks = ", ".join(f"chunk {c.chunk}: {c.bytes} B on {c.pages} pages" for c in self.by_chunk)
        more = f" (+{self.nruns - first} more)" if self.nruns > first else ""
        return (f"{self.bytes} bytes on {self.pages} 2 MiB pages in {self.nruns} runs; {chunks}; runs: "
                + "; ".join(r.describe() for r in self.runs[:first]) + more)


class PageMap:
    """The booked bytes of every 2 MiB page behind one report (include/ccm.h: ccm_last_page_map), ascending."""

    def __init__(self, entries):
        """entries: (page, bytes, chunk) tuples or ccm_page_entry structures."""
        rows = [(e.page, e.bytes, e.chunk) if hasattr(e, "page") else tuple(e) for e in entries]
        self.entries: List[Tuple[int, int, int]] = sorted((int(p), int(b), int(c)) for p, b, c in rows)

    def __len__(self) -> int:
        return len(self.entries)

    @property
    def bytes(self) -> int:
        return sum(b for _, b, _ in self.entries)

    def by_chunk(self) -> dict:
        """{chunk: booked bytes}: exact, per physical allocation."""
        out: dict = {}
        for _, b, c in self.entries:
            out[c] = out.get(c, 0) + b
        return dict(sorted(out.items()))

    def runs(self) -> List[PageRun]:
        """Maximal stretches of consecutive pages in one chunk, with their bytes, ascending."""
        runs: List[PageRun] = []
        for p, b, c in self.entries:
            last = runs[-1] if runs else None
            if last is not None and last.chunk == c and last.first_page + last.pages == p:
                runs[-1] = PageRun(last.first_page, last.pages + 1, c, last.bytes + b)
            else:
                runs.append(PageRun(p, 1, c, b))
        return runs

    def digest(self, keep: int = PAGE_RUNS) -> PageDigest:
        runs = self.runs()
        pages: dict = {}
        for _, _, c in self.entries:
            pages[c] = pages.get(c, 0) + 1
        chunks = [ChunkPages(c, pages[c], b) for c, b in self.by_chunk().items()]
        return PageDigest(len(self.entries), self.bytes, len(runs), int(len(runs) > keep), chunks, runs[:keep])

    def summary(self) -> str:
        return self.digest().summary()


def last_page_map(cuda_ordinal: int, book: int) -> "Optional[PageMap]":
    """The page map behind the last report of `book` (N.BOOK_DIRT / BOOK_MISMATCH / BOOK_RESIDUE) on a CUDA device
    (include/ccm.h: ccm_last_page_map); None when it cannot be read."""
    entries = _read_pages("ccm_last_page_map", N.PageEntry, cuda_ordinal, book)
    return PageMap(entries) if entries is not None else None


def _read_pages(fn: str, ctype: type, cuda_ordinal: int, *args) -> "Optional[list]":
    """The entries (`ctype`) the library's page reader `fn`(cuda_ordinal, *args, out, cap, n) gives; None if unread."""
    n = C.c_uint64(0)
    if cuda_ordinal < 0 or getattr(N.lib(), fn)(cuda_ordinal, *args, None, 0, C.byref(n)) != N.OK:
        return None
    buf = (ctype * max(1, n.value))()
    if getattr(N.lib(), fn)(cuda_ordinal, *args, buf, n.value, C.byref(n)) != N.OK:
        return None
    return buf[:n.value]


class _WindowReport:
    """What the three window reports share: their JSON and the chunks their records lie in.  Each report is a
    dataclass with a `records` field of its WINDOW type and, last, a `pages` field (a PageDigest, or None)."""
    WINDOW: type

    @classmethod
    def from_json(cls, d: dict):
        pages = d.get("pages")
        return cls(**{**d, "records": [cls.WINDOW(**r) for r in d["records"]],
                      "pages": PageDigest.from_json(pages) if pages is not None else None})

    def as_json(self) -> dict:
        return dataclasses.asdict(self)

    @property
    def chunks(self) -> List[int]:
        return sorted({r.chunk for r in self.records})


def _last_report(cuda_ordinal: int, getter: str, native: type, report: type):
    """The report `getter` (ccm_scrub_last_dirt / ccm_scrub_last_mismatch) gives for the last product call on a CUDA
    device; None when it cannot be read."""
    out = native()
    if cuda_ordinal < 0 or getattr(N.lib(), getter)(cuda_ordinal, C.byref(out)) != N.OK:
        return None
    return report.from_native(out)


@dataclass
class DirtWindow:
    """One dirty 16-byte, 16-aligned window (include/ccm.h: ccm_dirt_record)."""
    offset: int      # first byte of the window from the report's va_base (negative only for the head window
                     # of a raw region that does not start 16-aligned)
    chunk: int       # physical allocation behind it, in creation order (fallback: segment index)
    mask: int        # bit i: byte i is non-zero
    bytes: str       # the 16 bytes as read, hex

    def describe(self) -> str:
        return f"+{self.offset:#x} chunk {self.chunk} mask {self.mask:04x} [{self.bytes}]"


@dataclass
class DirtReport(_WindowReport):
    """Where the read-back of a failed scrub found its non-zero bytes (include/ccm.h: ccm_dirt_report).
    Every field but the choice of `records` is exact; records are distinct windows sorted by offset, all of
    them unless `truncated`."""
    WINDOW = DirtWindow
    BOOK, WINDOWS = N.BOOK_DIRT, "dirty_windows"
    nonzero_bytes: int       # the locate pass's own recount
    dirty_windows: int
    first_offset: int        # first / last non-zero byte, from va_base
    last_offset: int
    va_base: int
    ms_locate: float
    located: int             # 0: no locate pass ran (the call read back clean)
    truncated: int
    records: List[DirtWindow] = field(default_factory=list)
    pages: Optional[PageDigest] = None   # its page map, when it booked a window (last_page_map)

    @classmethod
    def from_native(cls, d: N.DirtReport) -> "DirtReport":
        recs = [DirtWindow(_signed64(r.offset), r.chunk, r.mask, bytes(r.bytes).hex())
                for r in d.records[:d.nrecords]]
        return cls(d.nonzero_bytes, d.dirty_windows, d.first_offset, d.last_offset, d.va_base, d.ms_locate,
                   d.located, d.truncated, recs)

    def summary(self, first: int = 4) -> str:
        """One line for an operator: extent, window count, chunks involved and the first few windows."""
        more = " (records truncated)" if self.truncated else ""
        recs = "; ".join(r.describe() for r in self.records[:first])
        return (f"non-zero bytes at offsets {self.first_offset:#x}..{self.last_offset:#x} of va {self.va_base:#x}, "
                f"{self.nonzero_bytes} bytes in {self.dirty_windows} dirty 16-byte windows{more}, "
                f"chunks {self.chunks}; first windows: {recs}")


def last_dirt(cuda_ordinal: int) -> "Optional[DirtReport]":
    """The dirt report of the last product call on a CUDA device (include/ccm.h: ccm_scrub_last_dirt);
    None when it cannot be read."""
    return _last_report(cuda_ordinal, "ccm_scrub_last_dirt", N.DirtReport, DirtReport)


@dataclass
class MismatchWindow:
    """One 16-byte, 16-aligned window that did not hold its tags (include/ccm.h: ccm_mismatch_record)."""
    offset: int          # from the report's va_base (negative only for the head window of an unaligned raw region)
    chunk: int           # physical allocation behind it, in creation order (fallback: segment index)
    mask: int            # bit i: byte i differs from its tag
    kind: str            # "zero" | "alias" | "partial" | "foreign" (include/ccm.h: ccm_mismatch_kind)
    source_offset: int   # alias: the window whose tags these are; otherwise 0
    source_chunk: int    # alias: the allocation behind that window; otherwise 0
    bytes: str           # the 16 bytes as the check read them, hex

    def describe(self) -> str:
        return f"+{self.offset:#x} chunk {self.chunk} mask {self.mask:04x} [{self.bytes}]"


@dataclass
class MismatchReport(_WindowReport):
    """Where a failed tagged check found bytes that did not hold their tags (include/ccm.h: ccm_mismatch_report).
    mismatch_bytes, mismatch_windows, zero_windows, first_offset and last_offset are exact.  The split between
    alias, partial and foreign windows is known for the records only; records are distinct windows sorted by
    offset, all of them unless `truncated`."""
    WINDOW = MismatchWindow
    BOOK, WINDOWS = N.BOOK_MISMATCH, "mismatch_windows"
    mismatch_bytes: int
    mismatch_windows: int
    zero_windows: int        # mismatched windows whose bytes all read 0
    first_offset: int        # first / last mismatched byte, from va_base
    last_offset: int
    va_base: int
    seed: int
    located: int             # 0: the last call's tagged check was clean (or it was not tagged)
    truncated: int
    records: List[MismatchWindow] = field(default_factory=list)
    pages: Optional[PageDigest] = None   # its page map, when it booked a window (last_page_map)

    @classmethod
    def from_native(cls, m: N.MismatchReport) -> "MismatchReport":
        recs = [MismatchWindow(_signed64(r.offset), r.chunk, r.mask, N.MISMATCH_KINDS.get(r.kind, str(r.kind)),
                               _signed64(r.source_offset), r.source_chunk, bytes(r.bytes).hex())
                for r in m.records[:m.nrecords]]
        return cls(m.mismatch_bytes, m.mismatch_windows, m.zero_windows, m.first_offset, m.last_offset, m.va_base,
                   m.seed, m.located, m.truncated, recs)

    def by_kind(self) -> dict:
        out: dict = {}
        for r in self.records:
            out.setdefault(r.kind, []).append(r)
        return out

    def summary(self, first: int = 2) -> str:
        """One line for an operator: extent, exact window counts, then the records grouped by kind.  Alias records
        are given as the distinct source - offset deltas with the chunk pairs (chunk <- source chunk)."""
        more = " (records truncated)" if self.truncated else ""
        parts = []
        groups = self.by_kind()
        for kind in ("alias", "zero", "partial", "foreign"):
            recs = groups.get(kind, [])
            if not recs:
                continue
            if kind == "alias":
                deltas: dict = {}
                for r in recs:
                    deltas.setdefault(r.source_offset - r.offset, []).append(r)
                for delta, rs in sorted(deltas.items()):
                    lo, hi = min(r.offset for r in rs), max(r.offset for r in rs)
                    pairs = ", ".join(f"chunk {c} \u2190 chunk {s}" for c, s in sorted({(r.chunk, r.source_chunk) for r in rs}))
                    sign = "-" if delta < 0 else ""
                    parts.append(f"alias: +{lo:#x}..+{hi:#x} hold the tags of +{lo + delta:#x}.. "
                                 f"(delta {sign}{abs(delta):#x}, {pairs}; {len(rs)} records)")
            else:
                chunks = sorted({r.chunk for r in recs})
                parts.append(f"{kind}: {len(recs)} records, chunks {chunks}; "
                             + "; ".join(r.describe() for r in recs[:first]))
        return (f"bytes off their tags at offsets {self.first_offset:#x}..{self.last_offset:#x} of va {self.va_base:#x}, "
                f"{self.mismatch_bytes} bytes in {self.mismatch_windows} 16-byte windows, {self.zero_windows} of them "
                f"all zero{more}; " + " | ".join(parts))


def last_mismatch(cuda_ordinal: int) -> "Optional[MismatchReport]":
    """The mismatch report of the last product call on a CUDA device (include/ccm.h: ccm_scrub_last_mismatch);
    None when it cannot be read."""
    return _last_report(cuda_ordinal, "ccm_scrub_last_mismatch", N.MismatchReport, MismatchReport)


@dataclass
class ResidueWindow:
    """One 16-byte, 16-aligned window that held non-zero bytes when the census read it (include/ccm.h:
    ccm_residue_record).  It carries no bytes: they were the previous tenant's data."""
    offset: int      # from the report's va_base (negative only for the head window of an unaligned raw region)
    chunk: int       # physical allocation behind it, in creation order (fallback: segment index)
    mask: int        # bit i: byte i was non-zero

    def describe(self) -> str:
        return f"+{self.offset:#x} chunk {self.chunk} mask {self.mask:04x}"


@dataclass
class ResidueReport(_WindowReport):
    """What a census call's first pass found in the memory it mapped, before it erased it (include/ccm.h:
    ccm_residue_report).  residue_bytes, residue_windows, first_offset and last_offset are exact; records are distinct
    windows sorted by offset, all of them unless `truncated`."""
    WINDOW = ResidueWindow
    BOOK, WINDOWS = N.BOOK_RESIDUE, "residue_windows"
    residue_bytes: int
    residue_windows: int
    first_offset: int        # first / last non-zero byte, from va_base (0 when there is none)
    last_offset: int
    bytes_examined: int      # == bytes_scrubbed
    va_base: int
    located: int             # 1: a census ran over everything the call mapped
    truncated: int
    records: List[ResidueWindow] = field(default_factory=list)
    pages: Optional[PageDigest] = None   # its page map, when it booked a window (last_page_map)

    @classmethod
    def from_native(cls, r: N.ResidueReport) -> "ResidueReport":
        recs = [ResidueWindow(_signed64(w.offset), w.chunk, w.mask) for w in r.records[:r.nrecords]]
        return cls(r.residue_bytes, r.residue_windows, r.first_offset, r.last_offset, r.bytes_examined, r.va_base,
                   r.located, r.truncated, recs)

    def summary(self, first: int = 4) -> str:
        """One line for an operator: "none", or the count, extent, chunks and first windows."""
        if not self.located:
            return "no census ran"
        if self.residue_bytes == 0:
            return f"none: all {self.bytes_examined} bytes examined were zero at first touch"
        more = " (records truncated)" if self.truncated else ""
        recs = "; ".join(r.describe() for r in self.records[:first])
        return (f"{self.residue_bytes} of {self.bytes_examined} bytes were non-zero at first touch, in "
                f"{self.residue_windows} 16-byte windows at offsets {self.first_offset:#x}..{self.last_offset:#x} of va "
                f"{self.va_base:#x}{more}, chunks {self.chunks}; first windows: {recs}")


TRIAGE_PAGES = 64       # pages that did not clear a TriageReport keeps
TRIAGE_HOLD_MS = 100    # default hold between the triage's two re-reads


@dataclass(frozen=True)
class TriagePage:
    """The class of one page of the dirt page map after the triage (include/ccm.h: ccm_triage_page)."""
    page: int            # offset of the page from the report's va_base = page * PAGE_BYTES
    chunk: int           # physical allocation behind its first byte (as PageEntry.chunk)
    cls: str             # "stays" | "returns" | "clears"
    dirt_bytes: int      # the dirt page map's bytes on it
    t2_bytes: int        # non-zero bytes the re-read right after the re-zero found on it
    t3_bytes: int        # non-zero bytes the re-read after the hold found on it

    def describe(self) -> str:
        return (f"+{self.page * PAGE_BYTES:#x} chunk {self.chunk} {self.cls} ({self.dirt_bytes} B dirt, "
                f"{self.t2_bytes} B at once, {self.t3_bytes} B after the hold)")


def last_triage_pages(cuda_ordinal: int) -> "Optional[List[TriagePage]]":
    """The pages of the last triage on a CUDA device (include/ccm.h: ccm_last_triage_pages), ascending; None when they
    cannot be read."""
    return _triage_pages(cuda_ordinal, "ccm_last_triage_pages")


def last_mismatch_triage_pages(cuda_ordinal: int) -> "Optional[List[TriagePage]]":
    """The pages of the last mismatch triage on a CUDA device (include/ccm.h: ccm_last_mismatch_triage_pages), one per
    page of the mismatch page map, ascending (`dirt_bytes`: that map's bytes on the page); None when they cannot be
    read."""
    return _triage_pages(cuda_ordinal, "ccm_last_mismatch_triage_pages")


def _triage_pages(cuda_ordinal: int, fn: str) -> "Optional[List[TriagePage]]":
    pages = _read_pages(fn, N.TriagePage, cuda_ordinal)
    return None if pages is None else [TriagePage(p.page, p.chunk, N.TRIAGE_CLASSES.get(p.cls, str(p.cls)),
                                                  p.dirt_bytes, p.t2_bytes, p.t3_bytes) for p in pages]


@dataclass
class TriageReport:
    """What kind of dirt a failed read-back found (include/ccm.h: ccm_triage_report): the dirty pages re-zeroed and
    re-read at once and after a hold.  A page "stays" when zero stored over it does not read back as zero, "returns"
    when it reads back zero at once but not after the hold (something is still writing this GPU's memory), and
    "clears" otherwise.  Every count is exact; `suspect_pages` are the first TRIAGE_PAGES pages that did not clear."""
    pages_examined: int
    bytes_examined: int
    stay_pages: int
    stay_bytes: int          # the dirt report's bytes on the pages of each class
    return_pages: int
    return_bytes: int
    clear_pages: int
    clear_bytes: int
    t2_bytes: int            # non-zero bytes found at once (T2) and after the hold (T3)
    t3_bytes: int
    t2_first_offset: int     # first / last of them, from va_base (0 when there is none)
    t2_last_offset: int
    t3_first_offset: int
    t3_last_offset: int
    va_base: int
    ms_hold: float           # the hold actually waited
    ms_triage: float
    hold_ms: int             # the hold asked for
    runs: int                # contiguous runs the dirty pages make
    triaged: int
    suspect_pages: List[TriagePage] = field(default_factory=list)
    suspect_truncated: int = 0

    @classmethod
    def from_native(cls, t: N.TriageReport, pages: "Optional[List[TriagePage]]" = None) -> "TriageReport":
        suspect = [p for p in pages or () if p.cls != "clears"]
        return cls(*(getattr(t, name) for name, _ in N.TriageReport._fields_ if name != "reserved"),
                   suspect_pages=suspect[:TRIAGE_PAGES], suspect_truncated=int(len(suspect) > TRIAGE_PAGES))

    @classmethod
    def from_json(cls, d: dict) -> "TriageReport":
        return cls(**{**d, "suspect_pages": [TriagePage(**p) for p in d["suspect_pages"]]})

    def as_json(self) -> dict:
        return dataclasses.asdict(self)

    def summary(self, first: int = 4) -> str:
        """One line for an operator: pages and runs, the count of each class, the hold, and the first few pages that
        did not clear."""
        line = (f"{self.pages_examined} pages in {self.runs} runs: {self.stay_pages} stay, {self.return_pages} return, "
                f"{self.clear_pages} clear (hold {self.hold_ms} ms)")
        if self.suspect_pages:
            more = " (+more)" if self.suspect_truncated or len(self.suspect_pages) > first else ""
            line += "; " + "; ".join(p.describe() for p in self.suspect_pages[:first]) + more
        return line


def last_triage(cuda_ordinal: int) -> "Optional[TriageReport]":
    """The triage report of the last product call on a CUDA device (include/ccm.h: ccm_scrub_last_triage), with the
    pages that did not clear; None when it cannot be read."""
    out = N.TriageReport()
    if cuda_ordinal < 0 or N.lib().ccm_scrub_last_triage(cuda_ordinal, C.byref(out)) != N.OK:
        return None
    return TriageReport.from_native(out, last_triage_pages(cuda_ordinal) if out.triaged else None)


def last_mismatch_triage(cuda_ordinal: int) -> "Optional[TriageReport]":
    """The mismatch triage report of the last product call on a CUDA device (include/ccm.h:
    ccm_scrub_last_mismatch_triage), with the pages that did not clear; None when it cannot be read.  Its byte counts
    are bytes of the mismatch page map, and its va_base is the mismatch report's."""
    out = N.TriageReport()
    if cuda_ordinal < 0 or N.lib().ccm_scrub_last_mismatch_triage(cuda_ordinal, C.byref(out)) != N.OK:
        return None
    return TriageReport.from_native(out, last_mismatch_triage_pages(cuda_ordinal) if out.triaged else None)


def _arm_triage(cuda_ordinal: int, hold_ms: int) -> bool:
    """Arms (hold_ms > 0) or disarms (0) the triage on a CUDA device; False when the library refused."""
    return cuda_ordinal >= 0 and N.lib().ccm_scrub_triage(cuda_ordinal, hold_ms) == N.OK


def _arm_mismatch_triage(cuda_ordinal: int, hold_ms: int) -> bool:
    """Arms (hold_ms > 0) or disarms (0) the mismatch triage on a CUDA device; False when the library refused."""
    return cuda_ordinal >= 0 and N.lib().ccm_scrub_mismatch_triage(cuda_ordinal, hold_ms) == N.OK


def _mismatch_triage_check(mismatch_triage: bool, check: str) -> None:
    """The mismatch triage triages what the tagged check found: it needs check="tagged"."""
    if mismatch_triage and check != "tagged":
        raise ValueError(f"mismatch_triage needs check='tagged', not {check!r}")


def _triage_hold(hold_ms: int) -> int:
    if not 0 < hold_ms <= N.TRIAGE_MAX_HOLD_MS:
        raise ValueError(f"triage hold must be 1..{N.TRIAGE_MAX_HOLD_MS} ms, not {hold_ms}")
    return int(hold_ms)


COVER_PAGES = 64   # inexact pages a CoverReport, ProbeCoverReport or ReportCoverReport keeps


class _ProofReport:
    """What the three proof reports share: their C struct, their JSON and the inexact pages they keep.  Each report is a
    dataclass whose fields are those of its C struct, then its rows (ROWS, the struct's array of the same name: a ROW
    per name of NAMES), `pages` (a list of PAGE) and `pages_truncated`."""
    ROWS: str
    ROW: type
    NAMES: Tuple[str, ...]
    PAGE: type

    @classmethod
    def from_native(cls, r, pages=None):
        """The report of the C struct `r`, with the first COVER_PAGES of its inexact pages `pages`."""
        rows = [cls.ROW(name=name, **{f: getattr(row, f) for f, _ in row._fields_ if f != "reserved"})
                for name, row in zip(cls.NAMES, getattr(r, cls.ROWS))]
        pages = pages or []
        return cls(**{f.name: getattr(r, f.name) for f in dataclasses.fields(cls)[:-3]}, **{cls.ROWS: rows},
                   pages=pages[:COVER_PAGES], pages_truncated=int(len(pages) > COVER_PAGES))

    @classmethod
    def _last(cls, cuda_ordinal: int, getter: str, native: type, read_pages):
        """As _last_report, with the inexact pages (read_pages) of a report that proved and was not covered."""
        out = native()
        if cuda_ordinal < 0 or getattr(N.lib(), getter)(cuda_ordinal, C.byref(out)) != N.OK:
            return None
        return cls.from_native(out, read_pages(cuda_ordinal) if out.proved and not out.covered else None)

    @classmethod
    def from_json(cls, d: dict):
        return cls(**{**d, cls.ROWS: [cls.ROW(**r) for r in d[cls.ROWS]], "pages": [cls.PAGE(**p) for p in d["pages"]]})

    def as_json(self) -> dict:
        return dataclasses.asdict(self)

    def _with_pages(self, line: str, first: int) -> str:
        """`line`, then the first `first` inexact pages kept, and "(+more)" when there are others."""
        if not self.pages:
            return line
        more = " (+more)" if self.pages_truncated or len(self.pages) > first else ""
        return line + "; " + "; ".join(p.describe() for p in self.pages[:first]) + more


@dataclass
class CoverPage:
    """One page some pass of a proving call did not count exactly (include/ccm.h: ccm_cover_page)."""
    page: int
    chunk: int
    expected: int      # bytes every pass that ran had to count on it
    first: int         # bytes the first pass, the tagged check and the read-back counted
    check: int
    readback: int

    def describe(self) -> str:
        return (f"page {self.page} (chunk {self.chunk}): expected {self.expected}, first {self.first}, "
                f"check {self.check}, read-back {self.readback}")


@dataclass
class CoverPass:
    """What one pass counted against what the call mapped (include/ccm.h: ccm_cover_pass)."""
    name: str          # "first", "check" or "readback"
    ran: int
    bytes_counted: int
    bytes_missing: int
    bytes_extra: int
    bytes_outside: int
    pages_short: int
    pages_over: int
    first_short_page: int


@dataclass
class CoverReport(_ProofReport):
    """The coverage proof of one product call (include/ccm.h: ccm_cover_report): every pass counted on the device the
    bytes its kernels processed on each 2 MiB page, and `covered` says each pass that ran walked every mapped byte
    exactly once.  `pages` are the first COVER_PAGES inexact pages."""
    bytes_mapped: int
    pages_mapped: int
    va_base: int
    ms_prove: float
    proved: int
    covered: int
    passes: List[CoverPass] = field(default_factory=list)
    pages: List[CoverPage] = field(default_factory=list)
    pages_truncated: int = 0
    ROWS, ROW, NAMES, PAGE = "passes", CoverPass, N.COVER_PASSES, CoverPage

    def short_pass(self) -> "Optional[CoverPass]":
        """The first pass that ran and did not count every page exactly (None when covered)."""
        return next((p for p in self.passes if p.ran and (p.bytes_missing or p.bytes_extra)), None)

    def summary(self, first: int = 4) -> str:
        """One line for an operator: what was mapped and, when a pass was short, which one and on which pages."""
        line = f"{self.bytes_mapped} bytes on {self.pages_mapped} pages"
        bad = self.short_pass()
        if bad is None:
            return line + ": every pass covered every byte once (" + ", ".join(p.name for p in self.passes if p.ran) + ")"
        line += (f": the {bad.name} pass counted {bad.bytes_counted} bytes ({bad.bytes_missing} missing, "
                 f"{bad.bytes_extra} extra) with {bad.pages_short} pages short")
        return self._with_pages(line, first)


def last_cover_pages(cuda_ordinal: int) -> "Optional[List[CoverPage]]":
    """The inexact pages of the last proving call on a CUDA device (include/ccm.h: ccm_last_cover_pages), ascending;
    None when they cannot be read."""
    pages = _read_pages("ccm_last_cover_pages", N.CoverPage, cuda_ordinal)
    return None if pages is None else [CoverPage(p.page, p.chunk, p.expected, *p.count) for p in pages]


def last_cover(cuda_ordinal: int) -> "Optional[CoverReport]":
    """The coverage report of the last product call on a CUDA device (include/ccm.h: ccm_scrub_last_cover), with its
    first inexact pages; None when it cannot be read."""
    return CoverReport._last(cuda_ordinal, "ccm_scrub_last_cover", N.CoverReport, last_cover_pages)


LEDGER_SLOTS = 64   # inexact slots a CoverLedger keeps


@dataclass
class LedgerSlot:
    """One 128 KiB slot some pass of a proving call did not count exactly (include/ccm.h: ccm_ledger_slot)."""
    slot: int
    chunk: int
    expected: int      # bytes every pass that ran had to count on it
    first: int         # bytes the first pass, the tagged check and the read-back counted
    check: int
    readback: int

    def describe(self) -> str:
        return (f"slot {self.slot} (chunk {self.chunk}): expected {self.expected}, first {self.first}, "
                f"check {self.check}, read-back {self.readback}")


@dataclass
class LedgerPass:
    """What one pass counted per slot against what the call mapped (include/ccm.h: ccm_ledger_pass)."""
    name: str          # "first", "check" or "readback"
    ran: int
    slots_short: int
    slots_over: int
    bytes_missing: int
    bytes_extra: int
    bytes_outside: int
    first_short_slot: int
    first_over_slot: int


@dataclass
class CoverLedger:
    """The coverage ledger of one proving call (include/ccm.h: ccm_cover_ledger): every thread of every pass counted on
    the device the bytes it addressed on each 128 KiB slot, and `exact` says each pass that ran walked every slot
    exactly once.  A call can fail on its ledger while its CoverReport is covered (a chunk walked twice and another on
    the same page skipped).  `slots` are the first LEDGER_SLOTS inexact slots."""
    bytes_mapped: int
    slots_mapped: int
    va_base: int
    ms_ledger: float
    proved: int
    exact: int
    passes: List[LedgerPass] = field(default_factory=list)
    slots: List[LedgerSlot] = field(default_factory=list)
    slots_truncated: int = 0

    @classmethod
    def from_native(cls, r, slots=None) -> "CoverLedger":
        passes = [LedgerPass(name, **{f: getattr(p, f) for f, _ in p._fields_ if f != "reserved"})
                  for name, p in zip(N.COVER_PASSES, r.passes)]
        slots = slots or []
        return cls(r.bytes_mapped, r.slots_mapped, r.va_base, r.ms_ledger, r.proved, r.exact, passes,
                   slots[:LEDGER_SLOTS], int(len(slots) > LEDGER_SLOTS))

    @classmethod
    def from_json(cls, d: dict) -> "CoverLedger":
        return cls(**{**d, "passes": [LedgerPass(**p) for p in d["passes"]],
                      "slots": [LedgerSlot(**x) for x in d["slots"]]})

    def as_json(self) -> dict:
        return dataclasses.asdict(self)

    def inexact_pass(self) -> "Optional[LedgerPass]":
        """The first pass that ran and did not count every slot exactly (None when exact)."""
        return next((p for p in self.passes if p.ran and (p.bytes_missing or p.bytes_extra)), None)

    def summary(self, first: int = 4) -> str:
        """One line for an operator: what was mapped and, when a pass was inexact, which one and on which slots."""
        line = f"{self.bytes_mapped} bytes on {self.slots_mapped} slots of 128 KiB"
        bad = self.inexact_pass()
        if bad is None:
            return line + ": every pass walked every slot once (" + ", ".join(p.name for p in self.passes if p.ran) + ")"
        line += (f": the {bad.name} pass has {bad.slots_short} slots short and {bad.slots_over} over "
                 f"({bad.bytes_missing} bytes missing, {bad.bytes_extra} extra, {bad.bytes_outside} outside)")
        if not self.slots:
            return line
        more = " (+more)" if self.slots_truncated or len(self.slots) > first else ""
        return line + "; " + "; ".join(x.describe() for x in self.slots[:first]) + more


def last_ledger_slots(cuda_ordinal: int) -> "Optional[List[LedgerSlot]]":
    """The inexact slots of the last proving call on a CUDA device (include/ccm.h: ccm_last_ledger_slots), ascending;
    None when they cannot be read."""
    slots = _read_pages("ccm_last_ledger_slots", N.LedgerSlot, cuda_ordinal)
    return None if slots is None else [LedgerSlot(x.slot, x.chunk, x.expected, *x.count) for x in slots]


def last_ledger(cuda_ordinal: int) -> "Optional[CoverLedger]":
    """The coverage ledger of the last product call on a CUDA device (include/ccm.h: ccm_scrub_last_ledger), with its
    first inexact slots; None when it cannot be read."""
    out = N.CoverLedger()
    if cuda_ordinal < 0 or N.lib().ccm_scrub_last_ledger(cuda_ordinal, C.byref(out)) != N.OK:
        return None
    return CoverLedger.from_native(out, last_ledger_slots(cuda_ordinal) if out.proved and not out.exact else None)


def _attach_ledger(rep: "ScrubReport", cuda_ordinal: int) -> bool:
    """Attaches the coverage ledger of a proving call as `.ledger`; False when it cannot be read or did not run (the
    call then fails with ERR_UNCOVERED, as a probe proof that did not run does).  A stand-in library without
    ccm_scrub_last_ledger has no ledger to give."""
    if not hasattr(N.lib(), "ccm_scrub_last_ledger"):
        return True
    ledger = last_ledger(cuda_ordinal)
    rep.ledger = ledger if ledger is not None and ledger.proved else None
    return rep.ledger is not None


def _arm_prove(cuda_ordinal: int, on: bool) -> int:
    """Arms or disarms the coverage proof on a CUDA device; the library's status (a call that asked for the proof and
    could not arm it fails with it: it is never run unproven)."""
    return N.lib().ccm_scrub_prove(cuda_ordinal, int(on)) if cuda_ordinal >= 0 else N.ERR_NO_CUDA


@dataclass
class ProbeReport:
    """The alias probe of one product call (include/ccm.h: ccm_probe_report): one 32-byte window per 4 KiB page of
    every mapped chunk was tagged (P1), checked and zeroed (P2), and read for zeros (P3).  A page mapped twice shows as
    bytes off their tags (mismatch_bytes; where they are comes as the call's `.mismatch`)."""
    windows: int
    bytes_probed: int
    mismatch_bytes: int
    mismatch_windows: int      # 16-byte windows of the mismatch report
    reread_nonzero_bytes: int
    seed: int
    launches: int
    va_base: int
    ms_probe: float
    probed: int

    @classmethod
    def from_native(cls, r: N.ProbeReport) -> "ProbeReport":
        return cls(*(getattr(r, f) for f, _ in N.ProbeReport._fields_ if f != "reserved"))

    @classmethod
    def from_json(cls, d: dict) -> "ProbeReport":
        return cls(**d)

    def as_json(self) -> dict:
        return dataclasses.asdict(self)

    @property
    def held(self) -> bool:
        """Every window held its tags and read back zero."""
        return self.mismatch_bytes == 0 and self.reread_nonzero_bytes == 0

    def summary(self) -> str:
        """One line for an operator."""
        line = f"{self.windows} windows ({self.bytes_probed} bytes) in {self.ms_probe:.2f} ms"
        if self.held:
            return line + ": every window held its tags and read back zero"
        return (line + f": {self.mismatch_bytes} bytes off their tags in {self.mismatch_windows} 16-byte windows, "
                f"{self.reread_nonzero_bytes} non-zero bytes after the zeroing")


def last_probe(cuda_ordinal: int) -> "Optional[ProbeReport]":
    """The alias probe report of the last product call on a CUDA device (include/ccm.h: ccm_scrub_last_probe); None
    when it cannot be read."""
    out = N.ProbeReport()
    if cuda_ordinal < 0 or N.lib().ccm_scrub_last_probe(cuda_ordinal, C.byref(out)) != N.OK:
        return None
    return ProbeReport.from_native(out)


def _arm_probe(cuda_ordinal: int, on: bool) -> int:
    """Arms or disarms the alias probe on a CUDA device; the library's status."""
    return N.lib().ccm_scrub_probe(cuda_ordinal, int(on)) if cuda_ordinal >= 0 else N.ERR_NO_CUDA


def _probe_check(probe: bool, check: str) -> None:
    """The alias probe is a check of the zero gate: the tagged check already covers every window."""
    if probe and check == "tagged":
        raise ValueError("probe=True is for check='zero': the tagged check already covers every probe window")


@dataclass
class ProbeCoverPage:
    """One page some step of a proven probe did not count exactly (include/ccm.h: ccm_probe_cover_page)."""
    page: int
    chunk: int
    expected: int      # bytes (PROBE_WINDOW per window) every step had to count on it
    p1: int            # bytes P1, P2 and P3 counted
    p2: int
    p3: int

    def describe(self) -> str:
        return (f"page {self.page} (chunk {self.chunk}): expected {self.expected}, P1 {self.p1}, P2 {self.p2}, "
                f"P3 {self.p3}")


@dataclass
class ProbeCoverStep:
    """What one probe step counted against the call's windows (include/ccm.h: ccm_probe_cover_step)."""
    name: str          # "P1", "P2" or "P3"
    ran: int
    windows_counted: int
    windows_missing: int
    windows_extra: int
    windows_outside: int
    pages_short: int
    pages_over: int
    first_short_page: int


@dataclass
class ProbeCoverReport(_ProofReport):
    """The probe proof of one product call both proven and probed (include/ccm.h: ccm_probe_cover): every probe step
    counted on the device the windows it took on each 2 MiB page, and `covered` says each took every probe window of
    the call exactly once.  `pages` are the first COVER_PAGES inexact pages."""
    windows_expected: int
    va_base: int
    ms_prove: float
    proved: int
    covered: int
    steps: List[ProbeCoverStep] = field(default_factory=list)
    pages: List[ProbeCoverPage] = field(default_factory=list)
    pages_truncated: int = 0
    ROWS, ROW, NAMES, PAGE = "steps", ProbeCoverStep, N.PROBE_STEPS, ProbeCoverPage

    def short_step(self) -> "Optional[ProbeCoverStep]":
        """The first step that did not count every page exactly (None when covered)."""
        return next((p for p in self.steps if p.ran and (p.windows_missing or p.windows_extra)), None)

    def summary(self, first: int = 4) -> str:
        """One line for an operator: how many windows the probe had and, when a step was short, which one and where."""
        line = f"{self.windows_expected} probe windows"
        bad = self.short_step()
        if bad is None:
            return line + ": every step took every window once (" + ", ".join(p.name for p in self.steps if p.ran) + ")"
        line += (f": step {bad.name} counted {bad.windows_counted} windows ({bad.windows_missing} missing, "
                 f"{bad.windows_extra} extra) with {bad.pages_short} pages short, first short page "
                 f"{bad.first_short_page}")
        return self._with_pages(line, first)


def last_probe_cover_pages(cuda_ordinal: int) -> "Optional[List[ProbeCoverPage]]":
    """The inexact pages of the last proven probe on a CUDA device (include/ccm.h: ccm_last_probe_cover_pages),
    ascending; None when they cannot be read."""
    pages = _read_pages("ccm_last_probe_cover_pages", N.ProbeCoverPage, cuda_ordinal)
    return None if pages is None else [ProbeCoverPage(p.page, p.chunk, p.expected, *p.count) for p in pages]


def last_probe_cover(cuda_ordinal: int) -> "Optional[ProbeCoverReport]":
    """The probe proof of the last product call on a CUDA device (include/ccm.h: ccm_scrub_last_probe_cover), with
    its first inexact pages; None when it cannot be read."""
    return ProbeCoverReport._last(cuda_ordinal, "ccm_scrub_last_probe_cover", N.ProbeCover, last_probe_cover_pages)


def _attach_probe(rep: "ScrubReport", cuda_ordinal: int, prove: bool = False) -> bool:
    """The probe report of a call that probed, and where its tags were wrong when they were; for a proving call that
    probed, the probe proof.  False for a proving call that probed and has no proof that ran: none could be read, or
    the one read did not run.  (A stand-in library without ccm_scrub_last_probe_cover has no proof to give, and
    its verdict stands; _native.lib() loads no libccm without it.)"""
    report = last_probe(cuda_ordinal)
    rep.probe = report if report is not None and report.probed else None
    if rep.probe is not None and rep.probe.mismatch_bytes:
        rep.mismatch = last_mismatch(cuda_ordinal)
        if rep.mismatch is not None and rep.mismatch.mismatch_windows:
            pages = last_page_map(cuda_ordinal, rep.mismatch.BOOK)
            rep.mismatch.pages = pages.digest() if pages is not None else None
    if prove and rep.probe is not None:
        if not hasattr(N.lib(), "ccm_scrub_last_probe_cover"):
            return True
        pc = last_probe_cover(cuda_ordinal)
        rep.probe_cover = pc if pc is not None and pc.proved else None
        return rep.probe_cover is not None
    return True


@dataclass
class ReportCoverPage:
    """One page one step of a proven locate pass or triage did not count exactly (include/ccm.h:
    ccm_report_cover_page)."""
    page: int
    chunk: int
    step: str          # N.REPORT_STEPS
    expected: int      # bytes the step had to count on it
    counted: int       # bytes it counted

    def describe(self) -> str:
        return f"page {self.page} (chunk {self.chunk}): {self.step} counted {self.counted} of {self.expected} bytes"


@dataclass
class ReportCoverStep:
    """What one step of a proven locate pass or triage counted (include/ccm.h: ccm_report_cover_step)."""
    name: str          # N.REPORT_STEPS
    ran: int
    launches: int
    bytes_expected: int
    bytes_counted: int
    bytes_missing: int
    bytes_extra: int
    bytes_outside: int
    pages_short: int
    pages_over: int
    first_short_page: int


# The report each step of the report proof walks for: the locate pass the dirt report, the triage steps their triage.
REPORT_STEP_OF = {"LOCATE": "dirt", "DIRT_T1": "triage", "DIRT_T2": "triage", "DIRT_T3": "triage",
                  "MISMATCH_T1": "mismatch_triage", "MISMATCH_T2": "mismatch_triage", "MISMATCH_T3": "mismatch_triage"}


@dataclass
class ReportCoverReport(_ProofReport):
    """The report proof of one proven product call that failed (include/ccm.h: ccm_report_cover): its locate pass and
    every triage step it ran counted on the device the bytes they walked on each 2 MiB page, and `covered` says each
    walked every byte of its reports exactly once.  It never changes the call's verdict: a short step says only which
    pages of the dirt and triage reports rest on a kernel that missed bytes.  `pages` are the first COVER_PAGES
    inexact (step, page) entries."""
    va_base: int
    ms_prove: float
    proved: int
    covered: int
    steps: List[ReportCoverStep] = field(default_factory=list)
    pages: List[ReportCoverPage] = field(default_factory=list)
    pages_truncated: int = 0
    ROWS, ROW, NAMES, PAGE = "steps", ReportCoverStep, N.REPORT_STEPS, ReportCoverPage

    def short_steps(self) -> "List[ReportCoverStep]":
        """The steps that ran and did not count every page exactly."""
        return [p for p in self.steps if p.ran and (p.bytes_missing or p.bytes_extra)]

    def unproven_pages(self, report: str) -> "List[int]":
        """The pages (of those kept) on which a step behind `report` ("dirt", "triage" or "mismatch_triage") was
        inexact, ascending."""
        return sorted({p.page for p in self.pages if REPORT_STEP_OF[p.step] == report})

    def summary(self, first: int = 4) -> str:
        """One line for an operator: which steps ran and, when one was short, which and where."""
        ran = [p.name for p in self.steps if p.ran]
        bad = self.short_steps()
        if not bad:
            return "every step walked every byte of its reports once (" + ", ".join(ran) + ")"
        line = "; ".join(f"step {p.name} counted {p.bytes_counted} of {p.bytes_expected} bytes ({p.bytes_missing} "
                         f"missing, {p.bytes_extra} extra) with {p.pages_short} pages short, first short page "
                         f"{p.first_short_page}" for p in bad)
        return self._with_pages(line, first)


def last_report_cover_pages(cuda_ordinal: int) -> "Optional[List[ReportCoverPage]]":
    """The inexact (step, page) entries of the last proven locate pass and triages on a CUDA device (include/ccm.h:
    ccm_last_report_cover_pages), by step then page; None when they cannot be read."""
    pages = _read_pages("ccm_last_report_cover_pages", N.ReportCoverPage, cuda_ordinal)
    return None if pages is None else [ReportCoverPage(p.page, p.chunk, N.REPORT_STEPS[p.step - 1], p.expected,
                                                       p.counted) for p in pages]


def last_report_cover(cuda_ordinal: int) -> "Optional[ReportCoverReport]":
    """The report proof of the last product call on a CUDA device (include/ccm.h: ccm_scrub_last_report_cover), with
    its first inexact pages; None when it cannot be read."""
    return ReportCoverReport._last(cuda_ordinal, "ccm_scrub_last_report_cover", N.ReportCover, last_report_cover_pages)


def _attach_report_cover(rep: "ScrubReport", cuda_ordinal: int) -> None:
    """For a proving call that ran a locate pass or a triage, their proof.  (A stand-in library without
    ccm_scrub_last_report_cover has none to give.)  Never changes the call's status."""
    if not hasattr(N.lib(), "ccm_scrub_last_report_cover"):
        return
    report = last_report_cover(cuda_ordinal)
    rep.report_cover = report if report is not None and report.proved else None


@dataclass
class HbmSnapshot:
    """One NVML snapshot of a GPU's ECC and row-remapping state (include/ccm.h: ccm_hbm_state).  A query that did not
    answer has its bit clear in `available`, its fields 0 and its NVML return code in `nvml_rc`."""
    dram_corrected: int
    dram_uncorrected: int
    sram_corrected: int
    sram_uncorrected: int
    ecc_current: int
    ecc_pending: int
    rows_corrected: int
    rows_uncorrected: int
    remap_pending: int
    remap_failure: int
    hist_max: int
    hist_high: int
    hist_partial: int
    hist_low: int
    hist_none: int
    available: int
    nvml_rc: List[int]
    ms_query: float

    @classmethod
    def from_native(cls, s: N.HbmState) -> "HbmSnapshot":
        return cls(**{f: (list(getattr(s, f)) if f == "nvml_rc" else getattr(s, f))
                      for f, _ in N.HbmState._fields_ if f != "reserved"})

    def answered(self, query: str) -> bool:
        """Whether the query (a name of N.HBM_QUERIES) answered."""
        return bool(self.available >> N.HBM_QUERIES.index(query) & 1)

    def unanswered(self) -> List[str]:
        return [q for q in N.HBM_QUERIES if not self.answered(q)]


def _delta(d: int, answered: bool) -> str:
    return f"{d:+d}" if answered else "?"


@dataclass
class HbmHealth:
    """The HBM health report of one armed product call (include/ccm.h: ccm_hbm_health): the GPU's ECC and row-remapping
    state through NVML before the call mapped anything and after its reports, and the rule's verdict on the pair
    (N.HBM_FIT, N.HBM_UNFIT, N.HBM_UNKNOWN) with its reasons (names of N.HBM_REASONS)."""
    before: HbmSnapshot
    after: HbmSnapshot
    d_dram_corrected: int
    d_dram_uncorrected: int
    d_sram_corrected: int
    d_sram_uncorrected: int
    ms_health: float
    mode: int
    verdict: int
    reasons: List[str]
    missing_queries: List[str]

    @classmethod
    def from_native(cls, h: N.HbmHealth) -> "HbmHealth":
        names = lambda bits, table: [n for k, n in enumerate(table) if bits >> k & 1]   # noqa: E731
        return cls(HbmSnapshot.from_native(h.before), HbmSnapshot.from_native(h.after), h.d_dram_corrected,
                   h.d_dram_uncorrected, h.d_sram_corrected, h.d_sram_uncorrected, h.ms_health, h.mode, h.verdict,
                   names(h.reasons, N.HBM_REASONS), names(h.missing_queries, N.HBM_QUERIES))

    @classmethod
    def from_json(cls, d: dict) -> "HbmHealth":
        return cls(**{**d, "before": HbmSnapshot(**d["before"]), "after": HbmSnapshot(**d["after"])})

    def as_json(self) -> dict:
        return dataclasses.asdict(self)

    @property
    def fit(self) -> bool:
        return self.verdict == N.HBM_FIT

    @property
    def verdict_name(self) -> str:
        return {N.HBM_FIT: "fit", N.HBM_UNFIT: "unfit", N.HBM_UNKNOWN: "unknown"}.get(self.verdict, "not judged")

    def why(self) -> List[str]:
        """The reasons of a report that is not fit, one phrase each, for an operator."""
        a = self.after
        phrases = {
            "dram_uncorrected": f"uncorrected DRAM errors {self.d_dram_uncorrected:+d} during the gate",
            "sram_uncorrected": f"uncorrected SRAM errors {self.d_sram_uncorrected:+d} during the gate",
            "remap_pending": "a row remap is pending: the GPU must be reset before release",
            "remap_failure": f"a row remap failed ({a.rows_uncorrected} rows remapped for uncorrected errors, "
                             f"{a.hist_none} banks without spare rows): the GPU should go to RMA",
            "ecc_off": "ECC is off",
            "no_answer": "NVML did not answer " + ", ".join(
                f"{q} ({self.before.nvml_rc[N.HBM_QUERIES.index(q)] or self.after.nvml_rc[N.HBM_QUERIES.index(q)]})"
                for q in self.missing_queries),
            "went_down": "an error counter went down between the snapshots (a reset in between)",
        }
        return [phrases[r] for r in self.reasons]

    def summary(self) -> str:
        """One line for an operator: ECC, the counter deltas over the gate and the remap state after it; then the
        verdict's reasons when it is not fit."""
        a, both = self.after, lambda q: self.before.answered(q) and self.after.answered(q)
        ecc = ("on" if a.ecc_current else "off") if a.answered("ecc_mode") else "unknown"
        line = (f"ECC {ecc}; DRAM corrected {_delta(self.d_dram_corrected, both('dram_corrected'))}, uncorrected "
                f"{_delta(self.d_dram_uncorrected, both('dram_uncorrected'))} during the gate")
        if self.d_sram_corrected or self.d_sram_uncorrected:
            line += f"; SRAM corrected {self.d_sram_corrected:+d}, uncorrected {self.d_sram_uncorrected:+d}"
        if a.answered("remapped_rows"):
            line += (f"; rows remapped {a.rows_corrected}/{a.rows_uncorrected}, "
                     f"{'remap pending' if a.remap_pending else 'none pending'}, "
                     f"{'remap FAILED' if a.remap_failure else 'no failure'}")
        else:
            line += "; row remapping unknown"
        if not self.fit:
            line += f"; {self.verdict_name.upper()}: " + "; ".join(self.why())
        return line


def hbm_snapshot(dev) -> HbmSnapshot:
    """One NVML snapshot of a GPU's ECC and row-remapping state (include/ccm.h: ccm_hbm_snapshot); `dev` is a device of
    find_gpus() or its index.  Needs no CUDA context and changes nothing on the device.  A snapshot whose queries did
    not all answer is returned as it is (see `available`); GpuError for an unknown device."""
    index = dev if isinstance(dev, int) else dev.index
    out = N.HbmState()
    rc = N.lib().ccm_hbm_snapshot(index, C.byref(out))
    if rc in (N.ERR_NO_DEVICE, N.ERR_INVALID):
        _check(rc, "hbm_snapshot")
    return HbmSnapshot.from_native(out)


def last_health(cuda_ordinal: int) -> "Optional[HbmHealth]":
    """The HBM health report of the last product call on a CUDA device (include/ccm.h: ccm_scrub_last_health); None
    when it cannot be read or the call was not armed."""
    out = N.HbmHealth()
    if cuda_ordinal < 0 or N.lib().ccm_scrub_last_health(cuda_ordinal, C.byref(out)) != N.OK or not out.mode:
        return None
    return HbmHealth.from_native(out)


def _health_mode(health: str) -> int:
    """ccm_scrub_health's mode for 'off' / 'report' / 'require'; ValueError for anything else."""
    if health not in N.HBM_HEALTH_MODES:
        raise ValueError(f"HBM health must be 'off', 'report' or 'require', not {health!r}")
    return N.HBM_HEALTH_MODES[health]


def _arm_health(cuda_ordinal: int, mode: int) -> int:
    """Arms (mode 1 or 2) or disarms (0) the HBM health report on a CUDA device; the library's status."""
    return N.lib().ccm_scrub_health(cuda_ordinal, mode) if cuda_ordinal >= 0 else N.ERR_NO_CUDA


def _attach_health(rep: "ScrubReport", cuda_ordinal: int, mode: int) -> None:
    """The health report of an armed call; under 'require', a call that returned OK without one fails with
    ERR_HBM_HEALTH (a report that was asked for and is missing is no evidence of health)."""
    rep.health = last_health(cuda_ordinal)
    if mode == N.HBM_HEALTH_MODES["require"] and rep.health is None and rep.status == N.OK:
        rep.status = N.ERR_HBM_HEALTH


def _mib(n: int) -> str:
    return f"{n / 2**20:.1f} MiB"


@dataclass
class RelayReport:
    """What the relayed whole-HBM gate (ccm-scrub --relay, DESIGN.md §5n) reached on one GPU, in bytes: the inputs each
    leg measured, the accounting rule's outputs (csrc/ccm_relay.h) and the phase times.  Leg A's gate ran in a first
    process; this process's context was created while A's still existed, then A exited and leg B scrubbed what was free,
    A's footprint included.  `first` is leg A's report for the GPU (a ScrubReport)."""
    total: int
    a_free_before: int
    a_unreached: int
    b_free_held: int
    b_free_settled: int
    b_free_before: int
    b_unreached: int
    marked: int
    footprint_a: int      # total - a_free_before: what the device held beside leg A's mapping
    freed: int            # b_free_settled - b_free_held: what A's exit gave back
    held: int             # footprint_a - freed: memory neither leg could map
    growth: int           # b_free_settled - b_free_before: what leg B's process allocated after the hand-over
    unreached: int        # held + growth + a_unreached + b_unreached
    coverage: float       # 1 - unreached / total
    settled: int
    settle_polls: int
    ms_first: float       # leg A started .. its HBM back with the driver
    ms_handover: float    # this leg's context created and armed, A reaped
    ms_settle: float      # A reaped .. its memory back
    ms_second: float      # leg B's time to verdict
    first: "Optional[ScrubReport]" = None

    @classmethod
    def from_json(cls, d: dict) -> "RelayReport":
        first = d.get("first")
        return cls(**{**d, "first": ScrubReport.from_json(first) if first is not None else None})

    def as_json(self) -> dict:
        d = {f.name: getattr(self, f.name) for f in dataclasses.fields(self)}
        d["first"] = self.first.as_json() if self.first is not None else None
        return d

    def summary(self) -> str:
        """One line for an operator: the relay's coverage, where A's footprint went, what each leg left unreached and
        how long each phase took."""
        return (f"coverage {self.coverage:.5f} of {self.total / 2**30:.1f} GiB ({_mib(self.unreached)} unreached); "
                f"first context's footprint {_mib(self.footprint_a)}, freed {_mib(self.freed)}, held {_mib(self.held)}, "
                f"growth {_mib(self.growth)}; unmappable A {_mib(self.a_unreached)}, B {_mib(self.b_unreached)}"
                + (f"; marker {_mib(self.marked)}" if self.marked else "")
                + (f"; free memory did not settle in {self.settle_polls} reads" if not self.settled else "")
                + f"; first leg {self.ms_first:.0f} ms, hand-over {self.ms_handover:.0f} ms, settle "
                f"{self.ms_settle:.0f} ms, second leg {self.ms_second:.0f} ms")


def reports_from_payload(payload: dict) -> "List[ScrubReport]":
    """The reports of a scrub worker's JSON line.  A relayed line (ccm-scrub --relay) also holds leg A's line under
    "first": each report's relay gets leg A's report for its GPU."""
    reports = [ScrubReport.from_json(r) for r in payload["reports"]]
    first = {r["bdf"]: r for r in (payload.get("first") or {}).get("reports", [])}
    for rep in reports:
        if rep.relay is not None and rep.bdf in first:
            rep.relay.first = ScrubReport.from_json(first[rep.bdf])
    return reports


# The reports a call can carry, as (attribute of ScrubReport and GpuError, report class), in JSON order.
_REPORTS = (("dirt", DirtReport), ("mismatch", MismatchReport), ("residue", ResidueReport), ("triage", TriageReport),
            ("mismatch_triage", TriageReport), ("cover", CoverReport), ("probe", ProbeReport),
            ("probe_cover", ProbeCoverReport), ("report_cover", ReportCoverReport), ("health", HbmHealth),
            ("ledger", CoverLedger), ("relay", RelayReport))
# The JSON key of a report whose attribute is not its key.
_JSON_KEYS = {"health": "hbm_health", "ledger": "cover_ledger"}


@dataclass
class ScrubReport:
    """Outcome of one GPU's HBM scrub-and-verify (include/ccm.h: ccm_scrub_result)."""
    bdf: str
    bytes_requested: int
    bytes_scrubbed: int
    device_total_bytes: int
    nonzero_bytes: int
    ms_acquire: float
    ms_scrub: float
    ms_verify: float
    ms_release: float
    ms_total: float
    segments: int
    status: int
    release_deferred: int = 0        # 1: the HBM is handed back by libccm's background reaper
    device_free_before: int = 0      # free HBM when the call started
    bytes_unreached: int = 0         # free HBM that could not be mapped (hence not scrubbed)
    ms_release_wait: float = 0.0     # waited for the previous call's deferred release
    ms_gpu_span: float = 0.0         # first scrub launch .. last verify done
    # tagged gate only (check="tagged"; include/ccm.h: ccm_tag_result)
    check: str = "zero"
    tag_seed: int = 0                # seed of the address tags this call wrote
    mismatch_bytes: int = 0          # bytes that did not hold their tag
    ms_tag: float = 0.0              # tag-fill kernels
    ms_check: float = 0.0            # check-and-zero kernels
    # Where the dirt is (a DirtReport), set for every report with nonzero_bytes != 0.  Not a dataclass field,
    # so positional construction, the field list and the JSON of a clean report stay as they were.
    dirt = None
    # Where the tags were wrong (a MismatchReport), set for every report with mismatch_bytes != 0.  Not a dataclass
    # field either, for the same reason.
    mismatch = None
    # What the first pass found before it erased it (a ResidueReport), set for every report of a census call
    # (residue=True).  Not a dataclass field either.
    residue = None
    # What kind of dirt it is (a TriageReport), set for every report of a triage call (triage=True) that triaged: one
    # whose read-back found non-zero bytes.  Not a dataclass field either.
    triage = None
    # What kind of mismatch it is (a TriageReport of the mismatch page map), set for every report of a mismatch triage
    # call (mismatch_triage=True) that triaged: one whose tagged check found bytes off their tags.  Not a dataclass
    # field either.
    mismatch_triage = None
    # How many bytes each pass walked on every page (a CoverReport), set for every report of a proving call
    # (prove=True) whose passes finished.  Not a dataclass field either.
    cover = None
    # What the alias probe found (a ProbeReport), set for every report of a probing call (probe=True) that probed: one
    # whose read-back was clean.  Not a dataclass field either.
    probe = None
    # How many windows each probe step took on every page (a ProbeCoverReport), set for every report of a call both
    # proving and probing (prove=True, probe=True) that probed.  Not a dataclass field either.
    probe_cover = None
    # How many bytes the locate pass and each triage step walked on every page (a ReportCoverReport), set for every
    # report of a proving call (prove=True) that located dirt or triaged.  Not a dataclass field either.
    report_cover = None
    # The GPU's ECC and row-remapping state before and after the call (an HbmHealth), set for every report of a call
    # armed for it (health="report" or "require").  Not a dataclass field either; its JSON key is "hbm_health".
    health = None
    # How many bytes every thread of each pass addressed on every 128 KiB slot (a CoverLedger), set for every report of
    # a proving call (prove=True) whose passes finished.  Not a dataclass field either; its JSON key is "cover_ledger".
    ledger = None
    # What the relayed gate reached on this GPU (a RelayReport, with leg A's report as its `first`), set for every report
    # of a relayed call (ccm-scrub --relay) whose relay was computed.  Not a dataclass field either.
    relay = None

    @property
    def clean(self) -> bool:
        return self.status == N.OK and self.nonzero_bytes == 0 and self.mismatch_bytes == 0

    @property
    def coverage(self) -> float:
        """Scrubbed fraction of the DEVICE's memory (the rest is the CUDA context's own
        footprint, driver reservations and whatever other contexts hold)."""
        return self.bytes_scrubbed / self.device_total_bytes if self.device_total_bytes else 0.0

    @property
    def coverage_of_free(self) -> float:
        """Scrubbed fraction of what was free when the call started (1.0 = every reachable byte)."""
        return self.bytes_scrubbed / self.device_free_before if self.device_free_before else 0.0

    @property
    def scrub_gbs(self) -> float:
        return self.bytes_scrubbed / self.ms_scrub / 1e6 if self.ms_scrub > 0 else 0.0

    @property
    def verify_gbs(self) -> float:
        return self.bytes_scrubbed / self.ms_verify / 1e6 if self.ms_verify > 0 else 0.0

    @classmethod
    def from_native(cls, bdf: str, r: N.ScrubResult, tag: "N.TagResult | None" = None) -> "ScrubReport":
        rep = cls(bdf, r.bytes_requested, r.bytes_scrubbed, r.device_total_bytes, r.nonzero_bytes,
                  r.ms_acquire, r.ms_scrub, r.ms_verify, r.ms_release, r.ms_total, r.segments, r.status,
                  r.release_deferred, r.device_free_before, r.bytes_unreached, r.ms_release_wait, r.ms_gpu_span)
        if tag is not None:
            rep.check, rep.tag_seed, rep.mismatch_bytes = "tagged", tag.seed, tag.mismatch_bytes
            rep.ms_tag, rep.ms_check = tag.ms_tag, tag.ms_check
        return rep

    def as_json(self) -> dict:
        """The report as the scrub workers print it: the tagged-gate fields only for a tagged call, "dirt",
        "mismatch", "residue", "triage" and "mismatch_triage" only when that report is attached."""
        d = dataclasses.asdict(self)
        if self.check == "zero":
            for name in TAG_FIELDS:
                del d[name]
        for attr, _ in _REPORTS:
            if getattr(self, attr) is not None:
                d[_JSON_KEYS.get(attr, attr)] = getattr(self, attr).as_json()
        return d

    @classmethod
    def from_json(cls, d: dict) -> "ScrubReport":
        """Inverse of as_json."""
        d = dict(d)
        found = [(attr, kind, d.pop(_JSON_KEYS.get(attr, attr), None)) for attr, kind in _REPORTS]
        rep = cls(**d)
        for attr, kind, js in found:
            if js is not None:
                setattr(rep, attr, kind.from_json(js))
        return rep


def _attach_reports(rep: ScrubReport, cuda_ordinal: int, census: "N.ResidueReport | None",
                    triage: bool = False, mismatch_triage: bool = False, prove: bool = False) -> None:
    """Attaches to the report of a call what that call found: the census's report, and the device's last dirt /
    mismatch report when the call counted non-zero / mismatched bytes; each report that booked a window with its page
    map's digest; for a triage call whose read-back found non-zero bytes, the triage report when it ran; and for a
    mismatch triage call whose tagged check found bytes off their tags, the mismatch triage report when it ran."""
    if census is not None:
        rep.residue = ResidueReport.from_native(census)
    if rep.nonzero_bytes:
        rep.dirt = last_dirt(cuda_ordinal)
    if rep.mismatch_bytes:
        rep.mismatch = last_mismatch(cuda_ordinal)
    if triage and rep.nonzero_bytes:
        report = last_triage(cuda_ordinal)
        rep.triage = report if report is not None and report.triaged else None
    if mismatch_triage and rep.mismatch_bytes:
        report = last_mismatch_triage(cuda_ordinal)
        rep.mismatch_triage = report if report is not None and report.triaged else None
    if prove:
        report = last_cover(cuda_ordinal)
        rep.cover = report if report is not None and report.proved else None
    for attr, _ in _REPORTS:
        report = getattr(rep, attr)
        if isinstance(report, _WindowReport) and getattr(report, report.WINDOWS):
            pages = last_page_map(cuda_ordinal, report.BOOK)
            report.pages = pages.digest() if pages is not None else None


# ScrubReport fields that only a tagged call reports
TAG_FIELDS = ("check", "tag_seed", "mismatch_bytes", "ms_tag", "ms_check")
CHECKS = ("zero", "tagged")


def _check_mode(check: str) -> bool:
    """True for the tagged gate; ValueError for anything but 'zero' / 'tagged'."""
    if check not in CHECKS:
        raise ValueError(f"scrub check must be 'zero' or 'tagged', not {check!r}")
    return check == "tagged"


class NvidiaDevice:
    """One NVIDIA PCI function (GPU or NVSwitch) behind the C ABI."""

    def __init__(self, info: N.DevInfo):
        self.index = int(info.index)
        self.bdf = info.bdf.decode()
        self.name = info.name.decode()
        self.kind = int(info.kind)
        self.is_cc_query_supported = bool(info.cc_query_supported)
        self.is_ppcie_query_supported = bool(info.ppcie_query_supported)
        self.cuda_ordinal = int(info.cuda_ordinal)
        self.hbm_total_bytes = int(info.hbm_total_bytes)

    def __repr__(self) -> str:
        return f"<{type(self).__name__} {self.bdf} {self.name!r}>"

    def is_gpu(self) -> bool:
        return self.kind == N.KIND_GPU

    def is_nvswitch(self) -> bool:
        return self.kind == N.KIND_NVSWITCH

    # -- CC mode -------------------------------------------------------------
    def query_cc_mode(self) -> str:
        mode = C.c_int(-1)
        _check(N.lib().ccm_query_cc_mode(self.index, C.byref(mode)), "query_cc_mode", self.bdf)
        return N.CC_MODE_NAMES[mode.value]

    def set_cc_mode(self, mode: str) -> None:
        if mode not in N.CC_MODES:
            raise GpuError(f"invalid CC mode {mode!r} for {self.bdf}", N.ERR_INVALID)
        _check(N.lib().ccm_set_cc_mode(self.index, N.CC_MODES[mode]), "set_cc_mode", self.bdf)

    # -- PPCIe mode ------------------------------------------------------------
    def query_ppcie_mode(self) -> str:
        mode = C.c_int(-1)
        _check(N.lib().ccm_query_ppcie_mode(self.index, C.byref(mode)), "query_ppcie_mode", self.bdf)
        return N.PPCIE_MODE_NAMES[mode.value]

    def set_ppcie_mode(self, mode: str) -> None:
        if mode not in N.PPCIE_MODES:
            raise GpuError(f"invalid PPCIe mode {mode!r} for {self.bdf}", N.ERR_INVALID)
        _check(N.lib().ccm_set_ppcie_mode(self.index, N.PPCIE_MODES[mode]), "set_ppcie_mode", self.bdf)

    # -- reset / boot ----------------------------------------------------------
    def reset_with_os(self) -> None:
        _check(N.lib().ccm_reset(self.index), "reset_with_os", self.bdf)

    def wait_for_boot(self, timeout_ms: int = 0) -> None:
        _check(N.lib().ccm_wait_for_boot(self.index, timeout_ms), "wait_for_boot", self.bdf)

    # -- NEW: HBM scrub-and-verify ---------------------------------------------
    def scrub_and_verify(self, nbytes: int = 0, check: str = "zero", residue: bool = False, triage: bool = False,
                         triage_hold_ms: int = TRIAGE_HOLD_MS, mismatch_triage: bool = False,
                         prove: bool = False, probe: bool = False, health: str = "off") -> ScrubReport:
        """Zero-fills and reads back this GPU's HBM (nbytes=0: all the context can map).
        check="tagged" first writes and checks an address-tagged known answer
        (include/ccm.h: ccm_scrub_verify_tagged).  residue=True runs the census in the first pass and attaches what
        it found as `.residue` (include/ccm.h: ccm_scrub_verify_residue); it never changes the verdict.
        triage=True arms the dirt triage for this call (include/ccm.h: ccm_scrub_triage): when the read-back finds
        non-zero bytes, the dirty pages are re-zeroed and re-read at once and after `triage_hold_ms`, and what
        kind of dirt it is comes attached as `.triage`; it never changes the verdict either.
        mismatch_triage=True (check="tagged" only, else ValueError) arms the mismatch triage for this call
        (include/ccm.h: ccm_scrub_mismatch_triage): when the tagged check finds bytes off their tags, those pages are
        re-tagged, checked and zeroed, held for `triage_hold_ms` and read for zeros, and what kind of mismatch it is
        comes attached as `.mismatch_triage`; it never changes the verdict either.
        prove=True arms the coverage proof for this call (include/ccm.h: ccm_scrub_prove): every pass counts on the
        device the bytes it walked on each page, the report comes attached as `.cover`, and a pass that missed or
        repeated a byte fails the call with ERR_UNCOVERED.  A device that cannot be armed fails the call.
        probe=True (check="zero" only, else ValueError) arms the alias probe for this call (include/ccm.h:
        ccm_scrub_probe): after a clean read-back, one 32-byte window per 4 KiB page is tagged, checked and zeroed and
        read for zeros; the report comes attached as `.probe`, and a window off its tags (a page mapped twice) fails
        the call with ERR_MISMATCH and attaches where as `.mismatch`.  A device that cannot be armed fails the call.
        prove=True with probe=True also proves the probe: each probe step counts on the device the windows it took on
        each page, the report comes attached as `.probe_cover`, and a step that missed or repeated a window fails the
        call with ERR_UNCOVERED.  A proving call that fails and locates its dirt or triages also proves its locate pass
        and triage steps: the report comes attached as `.report_cover`, and never changes the verdict.
        health="report" or "require" arms the HBM health report for this call (include/ccm.h: ccm_scrub_health): the
        GPU's ECC counters and row-remapping state are read through NVML before the call maps anything and after its
        reports, and the report comes attached as `.health`.  Under "require" a GPU whose uncorrected count rose, whose
        remap is pending or failed, whose ECC is off, or whose state could not be read fails the call with
        ERR_HBM_HEALTH; "report" never changes the verdict.  A device that cannot be armed fails the call.

        Raises GpuError if the scrub cannot run (no CUDA device, no HBM, CUDA error),
        if any byte reads back non-zero, or (tagged) if any byte did not hold its tag.  When the read-back
        found non-zero bytes, the report (or the GpuError, as `.dirt`) carries where they are; when the tagged check
        found bytes off their tags, it carries where those are as `.mismatch`.
        """
        res, tag, census = N.ScrubResult(), None, None
        if _check_mode(check):
            tag = N.TagResult()
        _mismatch_triage_check(mismatch_triage, check)
        _probe_check(probe, check)
        hold = _triage_hold(triage_hold_ms) if triage or mismatch_triage else 0
        hmode = _health_mode(health)
        armed = marmed = False
        try:
            if hmode:
                _check(_arm_health(self.cuda_ordinal, hmode), "scrub_and_verify (HBM health)", self.bdf)
            if prove:
                _check(_arm_prove(self.cuda_ordinal, True), "scrub_and_verify (coverage proof)", self.bdf)
            if probe:
                _check(_arm_probe(self.cuda_ordinal, True), "scrub_and_verify (alias probe)", self.bdf)
            armed = triage and _arm_triage(self.cuda_ordinal, hold)
            marmed = mismatch_triage and _arm_mismatch_triage(self.cuda_ordinal, hold)
            if residue:
                census = N.ResidueReport()
                rc = N.lib().ccm_scrub_verify_residue(self.index, nbytes, C.byref(tag) if tag is not None else None,
                                                      C.byref(census), C.byref(res))
            elif tag is not None:
                rc = N.lib().ccm_scrub_verify_tagged(self.index, nbytes, C.byref(tag), C.byref(res))
            else:
                rc = N.lib().ccm_scrub_verify(self.index, nbytes, C.byref(res))
            err = _error(rc, "scrub_and_verify", self.bdf)   # the library's error text, before anything else runs
        finally:
            if armed:
                _arm_triage(self.cuda_ordinal, 0)
            if marmed:
                _arm_mismatch_triage(self.cuda_ordinal, 0)
            if prove:
                _arm_prove(self.cuda_ordinal, False)
            if probe:
                _arm_probe(self.cuda_ordinal, False)
            if hmode:
                _arm_health(self.cuda_ordinal, 0)
        rep = ScrubReport.from_native(self.bdf, res, tag)
        _attach_reports(rep, self.cuda_ordinal, census, armed, marmed, prove)
        probe_proved = _attach_probe(rep, self.cuda_ordinal, prove) if probe else True
        if prove:
            _attach_report_cover(rep, self.cuda_ordinal)
        if err is None and prove and rep.cover is None:   # a proof that was asked for and did not run
            err = GpuError(f"scrub_and_verify on {self.bdf}: the coverage proof did not run", N.ERR_UNCOVERED)
        ledger_ok = _attach_ledger(rep, self.cuda_ordinal) if prove else True
        if err is None and not probe_proved:
            err = GpuError(f"scrub_and_verify on {self.bdf}: the probe proof did not run", N.ERR_UNCOVERED)
        if err is None and not ledger_ok:
            err = GpuError(f"scrub_and_verify on {self.bdf}: the coverage ledger did not run", N.ERR_UNCOVERED)
        if hmode:
            _attach_health(rep, self.cuda_ordinal, hmode)
            if err is None and rep.status == N.ERR_HBM_HEALTH:   # a report that was asked for and is missing
                err = GpuError(f"scrub_and_verify on {self.bdf}: the HBM health report is missing", N.ERR_HBM_HEALTH)
        if err is not None:
            for attr, _ in _REPORTS:
                setattr(err, attr, getattr(rep, attr))
            raise err
        return rep

    def wait_scrub_released(self) -> Tuple[float, float]:
        """Blocks until the HBM of the last scrub_and_verify() is back with the driver (libccm
        hands it back on a background thread so the verdict is not held up by cuMemUnmap /
        cuMemRelease).  Returns (ms the release took, ms this call waited)."""
        rel, waited = C.c_double(0.0), C.c_double(0.0)
        _check(N.lib().ccm_scrub_release_wait(self.index, C.byref(rel), C.byref(waited)), "wait_scrub_released", self.bdf)
        return rel.value, waited.value

    def release_cuda_context(self) -> None:
        """Give back everything libccm holds on this GPU, including its CUDA primary context
        (include/ccm.h: ccm_device_release).  Call it when the scrub gate is done."""
        _check(N.lib().ccm_device_release(self.index), "release_cuda_context", self.bdf)


class Gpu(NvidiaDevice):
    pass


class NvSwitch(NvidiaDevice):
    pass


def find_gpus() -> Tuple[List[NvidiaDevice], int]:
    """All NVIDIA PCI functions (GPUs AND NVSwitches), freshly enumerated.

    Mirrors pci.devices.find_gpus() as the reference uses it (main.py:144-155): the
    second element is the device count.
    """
    lib = N.lib()
    n = C.c_int(0)
    _check(lib.ccm_enumerate(None, 0, C.byref(n)), "enumerate")
    infos = (N.DevInfo * max(1, n.value))()
    _check(lib.ccm_enumerate(infos, n.value, C.byref(n)), "enumerate")
    devices: List[NvidiaDevice] = []
    for i in range(n.value):
        cls = Gpu if infos[i].kind == N.KIND_GPU else NvSwitch
        devices.append(cls(infos[i]))
    return devices, len(devices)


def scrub_and_verify_many(devices: Sequence[NvidiaDevice], nbytes: int = 0,
                          check: str = "zero", residue: bool = False, triage: bool = False,
                          triage_hold_ms: int = TRIAGE_HOLD_MS,
                          mismatch_triage: bool = False, prove: bool = False,
                          probe: bool = False, health: str = "off") -> Tuple[List[ScrubReport], float]:
    """Concurrent multi-context scrub of several GPUs through ONE native call
    (ccm_scrub_verify_many: one host thread + primary context + stream per GPU, no
    peer access, no collective; check="tagged": ccm_scrub_verify_many_tagged; residue=True:
    ccm_scrub_verify_many_residue, each report with its `.residue`; triage=True: every GPU armed for the dirt
    triage, as in NvidiaDevice.scrub_and_verify; mismatch_triage=True: every GPU armed for the mismatch triage, as
    there; prove=True: every GPU armed for the coverage proof, and a GPU that cannot be armed is not scrubbed: its
    report carries the arming's status; probe=True: every GPU armed for the alias probe, likewise; health="report" or
    "require": every GPU armed for the HBM health report, likewise, each report with its `.health`).  Returns
    (reports, wall_ms); never raises for a per-device failure — inspect report.status /
    report.clean."""
    tagged = _check_mode(check)
    _mismatch_triage_check(mismatch_triage, check)
    _probe_check(probe, check)
    hmode = _health_mode(health)
    if prove or probe or hmode:
        # every check asked for is armed on a device before it is scrubbed; a device that refuses one is not scrubbed
        # (its report carries that arming's status, and no report of a call that did not run)
        arm_health = lambda ordinal, on: _arm_health(ordinal, hmode if on else 0)   # noqa: E731
        arms = [arm for on, arm in ((prove, _arm_prove), (probe, _arm_probe), (hmode, arm_health)) if on]
        refused, armed = {}, []
        try:
            for d in devices:
                for arm in arms:
                    rc = arm(d.cuda_ordinal, True)
                    if rc != N.OK:
                        refused[d.index] = ScrubReport.from_native(d.bdf, N.ScrubResult(status=rc))
                        break
                    armed.append((d, arm))
            ran = [d for d in devices if d.index not in refused]
            reports, wall = scrub_and_verify_many(ran, nbytes, check, residue, triage, triage_hold_ms, mismatch_triage)
        finally:
            for d, arm in armed:
                arm(d.cuda_ordinal, False)
        it = iter(reports)
        reports = [refused[d.index] if d.index in refused else next(it) for d in devices]
        for rep, d in zip(reports, devices):
            if d.index in refused:
                continue
            if prove:
                report = last_cover(d.cuda_ordinal)
                rep.cover = report if report is not None and report.proved else None
                if rep.status == N.OK and rep.cover is None:   # a proof that was asked for and did not run
                    rep.status = N.ERR_UNCOVERED
                if not _attach_ledger(rep, d.cuda_ordinal) and rep.status == N.OK:
                    rep.status = N.ERR_UNCOVERED   # a ledger that was asked for and did not run
            if probe and not _attach_probe(rep, d.cuda_ordinal, prove) and rep.status == N.OK:
                rep.status = N.ERR_UNCOVERED   # a probe proof that was asked for and did not run
            if prove:
                _attach_report_cover(rep, d.cuda_ordinal)
            if hmode:
                _attach_health(rep, d.cuda_ordinal, hmode)
        return reports, wall
    n = len(devices)
    if n == 0:
        return [], 0.0
    hold = _triage_hold(triage_hold_ms) if triage or mismatch_triage else 0
    idx = (C.c_int * n)(*[d.index for d in devices])
    res = (N.ScrubResult * n)()
    wall = C.c_double(0.0)
    tags = (N.TagResult * n)() if tagged else None
    census = (N.ResidueReport * n)() if residue else None
    armed = {d.cuda_ordinal for d in devices if triage and _arm_triage(d.cuda_ordinal, hold)}
    marmed = {d.cuda_ordinal for d in devices if mismatch_triage and _arm_mismatch_triage(d.cuda_ordinal, hold)}
    try:
        if residue:
            N.lib().ccm_scrub_verify_many_residue(n, idx, nbytes, tags, census, res, C.byref(wall))
        elif tagged:
            N.lib().ccm_scrub_verify_many_tagged(n, idx, nbytes, tags, res, C.byref(wall))
        else:
            N.lib().ccm_scrub_verify_many(n, idx, nbytes, res, C.byref(wall))
    finally:
        for ordinal in armed:
            _arm_triage(ordinal, 0)
        for ordinal in marmed:
            _arm_mismatch_triage(ordinal, 0)
    reports = [ScrubReport.from_native(d.bdf, res[i], tags[i] if tagged else None) for i, d in enumerate(devices)]
    for i, (rep, d) in enumerate(zip(reports, devices)):
        _attach_reports(rep, d.cuda_ordinal, census[i] if residue else None, d.cuda_ordinal in armed,
                        d.cuda_ordinal in marmed)
    return reports, wall.value


def release_cuda_contexts(devices: Sequence[NvidiaDevice]) -> float:
    """Concurrent ccm_device_release for several GPUs (one native thread each): joins each
    engine's deferred HBM release, then resets its CUDA primary context.  Returns wall ms."""
    n = len(devices)
    if n == 0:
        return 0.0
    idx = (C.c_int * n)(*[d.index for d in devices])
    wall = C.c_double(0.0)
    _check(N.lib().ccm_device_release_many(n, idx, C.byref(wall)), "release_cuda_contexts")
    return wall.value


def select_backend(name: str) -> None:
    """Explicit backend choice ('sim' | 'cudasim' | 'sysfs'); rebuilds the device table."""
    if name not in N.BACKENDS:
        raise ValueError(f"unknown backend {name!r}")
    _check(N.lib().ccm_init(N.BACKENDS[name]), f"ccm_init({name})")


class ScrubbingProxy:
    """Wraps a device object from ANOTHER device library (e.g. the real gpu-admin-tools `Gpu`)
    and adds the one capability it lacks: `scrub_and_verify()`, served by libccm.so on the CUDA
    device with the same PCI address.  Every other attribute is forwarded untouched, so the
    manager keeps using that library's register access for query/set/reset/wait_for_boot
    (arrangement (1) of INTEGRATION.md §D)."""

    def __init__(self, foreign, native: "NvidiaDevice | None"):
        object.__setattr__(self, "_foreign", foreign)
        object.__setattr__(self, "_native", native)

    def __getattr__(self, name):
        return getattr(object.__getattribute__(self, "_foreign"), name)

    def __setattr__(self, name, value):
        setattr(object.__getattribute__(self, "_foreign"), name, value)

    def __repr__(self):
        return f"<ScrubbingProxy {self._foreign!r} scrub={'libccm' if self._native else 'unavailable'}>"

    def release_cuda_context(self) -> None:
        native = object.__getattribute__(self, "_native")
        if native is not None:
            native.release_cuda_context()

    def wait_scrub_released(self):
        native = object.__getattribute__(self, "_native")
        return native.wait_scrub_released() if native is not None else (0.0, 0.0)

    def scrub_and_verify(self, nbytes: int = 0, check: str = "zero", residue: bool = False, triage: bool = False,
                         triage_hold_ms: int = TRIAGE_HOLD_MS, mismatch_triage: bool = False,
                         prove: bool = False, probe: bool = False, health: str = "off") -> ScrubReport:
        native = object.__getattribute__(self, "_native")
        _mismatch_triage_check(mismatch_triage, check)
        _probe_check(probe, check)
        _health_mode(health)
        if native is None:
            raise GpuError(f"no CUDA device with PCI address {self._foreign.bdf}: HBM scrub cannot run", N.ERR_NO_CUDA)
        if health != "off":
            return native.scrub_and_verify(nbytes, check=check, residue=residue, triage=triage,
                                           triage_hold_ms=triage_hold_ms, mismatch_triage=mismatch_triage, prove=prove,
                                           probe=probe, health=health)
        if probe:
            return native.scrub_and_verify(nbytes, check=check, residue=residue, triage=triage,
                                           triage_hold_ms=triage_hold_ms, mismatch_triage=mismatch_triage, prove=prove,
                                           probe=True)
        if prove:
            return native.scrub_and_verify(nbytes, check=check, residue=residue, triage=triage,
                                           triage_hold_ms=triage_hold_ms, mismatch_triage=mismatch_triage, prove=True)
        if mismatch_triage:
            return native.scrub_and_verify(nbytes, check=check, residue=residue, triage=triage,
                                           triage_hold_ms=triage_hold_ms, mismatch_triage=True)
        if triage:
            return native.scrub_and_verify(nbytes, check=check, residue=residue, triage=True,
                                           triage_hold_ms=triage_hold_ms)
        if residue:
            return native.scrub_and_verify(nbytes, check=check, residue=True)
        if check == "zero":
            return native.scrub_and_verify(nbytes)   # exactly the call a zero-only device takes
        return native.scrub_and_verify(nbytes, check=check)


def _norm_bdf(bdf: str) -> str:
    bdf = bdf.strip().lower()
    return bdf if bdf.count(":") == 2 else "0000:" + bdf


def with_scrub(foreign_find_gpus):
    """Turns another library's `find_gpus()` into a device source for CCManager whose GPUs can be
    scrubbed: `CCManager(..., device_source=with_scrub(pci.devices.find_gpus))`."""
    def source():
        devices, _ = foreign_find_gpus()
        by_bdf = {_norm_bdf(d.bdf): d for d in find_gpus()[0] if d.is_gpu() and d.cuda_ordinal >= 0}
        wrapped = [ScrubbingProxy(d, by_bdf.get(_norm_bdf(d.bdf))) if d.is_gpu() else d for d in devices]
        return wrapped, len(wrapped)
    return source
