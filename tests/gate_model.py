"""One composed model of a product scrub gate call (include/ccm.h), in plain Python and numpy, no CUDA.

A product call is a composition: a gate kind (zero, tagged, census, census_tagged), a path (VMM pipelined, VMM
map-first, whole HBM with its tail zone, or the cudaMalloc fallback; each with or without the interleaved read-back),
up to four armings (prove, probe, dirt triage, mismatch triage) and any subset of the sim drills of ScrubDrill.  The
per-feature oracles each restate one of these; this module composes them into one prediction of everything the call
returns and leaves, so that a seeded random scenario (tests/gate_scenarios.py) can be checked field for field.

    predict(scenario, record)   the observables of the call (observe() of what it should return)
    observe(record)             the same observables of what tests/report_cover_calls.py recorded

A scenario is a call dict of tests/report_cover_calls.py.  The model takes from the record only what it cannot know in
advance: how much a whole-HBM call mapped and what was free, the granularity's consequence on fallback sizes, va_base
and the random tag and probe seeds.

Memory is kept sparse (`Mem`): runs of one content (a byte value, the tags of a seed, or unknown) over physical offsets,
and a virtual-to-physical map that the "scrub_alias" drill bends.  A whole-HBM flood is one run.  Only small ranges are
ever expanded into numpy arrays (tag comparisons), and reading unknown memory raises `Unpredictable`: the scenario
generator must never produce such a call.

The rules, each from the header line it restates:
* Drill order (ccm.h ccm_sim_set; csrc/ccm_scrub.cu GateRun): per mapping, "scrub_poison" then "scrub_residue" then
  the tag fill or tagged census (held); per enqueued range, "tag_flood" then "tag_inject", then the check, census or
  scrub, then "scrub_flood" then "scrub_inject", then (interleaved) the read-back; then the read-back of everything
  (not interleaved); then the probe P1, "probe_mismatch", P2, "probe_dirt", P3; then the locate pass, the dirt triage
  and the mismatch triage ("triage_stay" between T1 and T2, "triage_return" between T2 and T3 of each).
* What each pass overwrites: every pass writes the bytes it walks (a tag fill erases poison, the check-and-zero erases
  "tag_inject" bytes before the read-back); the census books the bytes it reads first (poison or residue) and then
  writes; a pass whose first launch was drilled with "cover_skip" leaves its skipped 128 KiB chunks as they were.
* Where budgets are spent: "scrub_inject" and "tag_inject" per enqueued range, "scrub_residue" per mapping, both in
  enqueue order (ccm.h: "each once, in enqueue order"; "each mapping ... in mapping order").
* Gating: a call whose read-back found dirt does not probe; a tagged call never probes (ccm.h ccm_scrub_probe); the
  fallback ignores "scrub_alias"; the triages need a located report with pages.
* Precedence (ccm.h ccm_scrub_prove / ccm_probe_cover / ccm_scrub_verify_tagged / ccm_scrub_probe): pass-proof
  UNCOVERED, probe-proof UNCOVERED, tag MISMATCH, probe MISMATCH, DIRTY.
"""
from __future__ import annotations

import bisect
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
for _p in (ROOT / "oracle", ROOT / "tests"):
    if str(_p) not in sys.path:
        sys.path.insert(0, str(_p))

import cover_oracle as CO  # noqa: E402
import probe_cover_oracle as PCO  # noqa: E402
import product_plan as PP  # noqa: E402
import report_cover_oracle as RO  # noqa: E402
import tag_oracle as TAG  # noqa: E402
import triage_oracle as TO  # noqa: E402

PAGE = 2 << 20               # include/ccm.h: CCM_PAGE_BYTES
RECORDS = 64                 # include/ccm.h: CCM_DIRT_RECORDS
STRIDE, WINDOW = 4096, 32    # include/ccm.h: CCM_PROBE_STRIDE, CCM_PROBE_WINDOW
GATHER_LIMIT = 64 << 20      # most bytes the model expands into numpy at once
OK, DIRTY, MISMATCH, UNCOVERED = 0, -8, -13, -14
ZERO, ALIAS, PARTIAL, FOREIGN = 1, 2, 3, 4   # include/ccm.h: ccm_mismatch_kind
CLASS_ID = {TO.STAYS: 1, TO.RETURNS: 2, TO.CLEARS: 3}
KINDS = ("zero", "tagged", "census", "census_tagged")
# Every drill key of ScrubDrill (csrc/ccm_internal.h), as ccm_sim_set names it.
DRILL_KEYS = ("scrub_inject", "scrub_poison", "scrub_flood", "tag_inject", "scrub_alias", "scrub_residue",
              "triage_stay", "triage_return", "tag_flood", "cover_skip", "cover_pass", "probe_mismatch", "probe_dirt",
              "probe_skip", "probe_skip_step", "report_skip", "report_skip_step")
# The verdicts from the highest precedence down (csrc/ccm_scrub.cu engine_scrub_verify).
PRECEDENCE = ("pass_uncovered", "probe_uncovered", "tag_mismatch", "probe_mismatch", "dirty")


class Unpredictable(Exception):
    """The call would read memory whose content the model cannot know (what the driver handed back)."""


# ------------------------------------------------------------------------------------------------ sparse memory
class Mem:
    """The bytes a call holds: runs [lo, hi, content] over physical offsets, content ("b", v), ("t", seed, delta) -- the
    byte at physical p holds the tag byte of address va + p + delta -- or ("u",).  `pieces` maps virtual offsets to
    physical ones: (vlo, vhi, plo)."""

    def __init__(self, n: int, va: int, alias: int = 0):
        self.n, self.va = n, va
        self.pieces = [(0, alias, 0), (alias, 2 * alias, 0), (2 * alias, n, 2 * alias)] if alias else [(0, n, 0)]
        self.lo, self.runs = [0], [[0, n, ("u",)]]

    def phys(self, vlo: int, vhi: int):
        for a, b, p in self.pieces:
            lo, hi = max(a, vlo), min(b, vhi)
            if lo < hi:
                yield lo, hi, p + lo - a

    def _split(self, x: int) -> int:
        i = bisect.bisect_right(self.lo, x) - 1
        if i < 0 or x >= self.runs[i][1] or x == self.runs[i][0]:
            return i if i >= 0 and x == self.runs[i][0] else i + 1
        lo, hi, c = self.runs[i]
        self.runs[i:i + 1] = [[lo, x, c], [x, hi, c]]
        self.lo[i:i + 1] = [lo, x]
        return i + 1

    def _set(self, plo: int, phi: int, content) -> None:
        if plo >= phi:
            return
        i = self._split(plo)
        j = self._split(phi)
        self.runs[i:j] = [[plo, phi, content]]
        self.lo[i:j] = [plo]

    def write(self, vlo: int, vhi: int, value: int) -> None:
        for lo, hi, p in self.phys(vlo, vhi):
            self._set(p, p + hi - lo, ("b", value))

    def tag(self, vlo: int, vhi: int, seed: int) -> None:
        for lo, hi, p in self.phys(vlo, vhi):
            self._set(p, p + hi - lo, ("t", seed, lo - p))

    def segments(self, vlo: int, vhi: int):
        """(vlo, vhi, content, v - p) of every run under [vlo, vhi)."""
        for lo, hi, p in self.phys(vlo, vhi):
            d = lo - p
            i = max(0, bisect.bisect_right(self.lo, p) - 1)
            while i < len(self.runs) and self.runs[i][0] < p + hi - lo:
                a, b, c = self.runs[i]
                s, e = max(a, p), min(b, p + hi - lo)
                if s < e:
                    yield s + d, e + d, c, d
                i += 1

    def values(self, vlo: int, vhi: int) -> np.ndarray:
        if vhi - vlo > GATHER_LIMIT:
            raise Unpredictable(f"would expand {vhi - vlo} bytes")
        out = np.zeros(max(0, vhi - vlo), np.uint8)
        for a, b, c, d in self.segments(vlo, vhi):
            if c[0] == "u":
                raise Unpredictable(f"reads what the driver handed back at [{a}, {b})")
            if c[0] == "b":
                out[a - vlo:b - vlo] = c[1]
            else:
                out[a - vlo:b - vlo] = TAG.tag_bytes(c[1], self.va + a - d + c[2], b - a)
        return out

    def xor(self, v: int) -> None:
        b = int(self.values(v, v + 1)[0]) ^ 0xA5
        self.write(v, v + 1, b)

    def booked(self, ranges, seed: int | None = None) -> list[tuple[int, int, np.ndarray | None, np.ndarray | None]]:
        """The booked bytes of `ranges` (non-zero, or with a seed off their tags) as (lo, hi, mask, values): mask None
        means every byte of [lo, hi) is booked.  With a seed, each gathered piece is widened to whole 16-byte windows
        inside its range, so that a window's bytes are all in one piece."""
        out = []
        for lo, hi in ranges:
            todo = []
            for a, b, c, d in self.segments(lo, hi):
                if c == ("b", 0) and seed is None:
                    continue
                if seed is not None and c[0] == "t" and c[1] == seed and c[2] == d:
                    continue   # the bytes hold their own tags
                if seed is None and c[0] == "b":
                    out.append((a, b, None, None))
                    continue
                a, b = (max(lo, a & ~15), min(hi, (b + 15) & ~15)) if seed is not None else (a, b)
                if todo and a <= todo[-1][1]:
                    todo[-1][1] = max(todo[-1][1], b)
                else:
                    todo.append([a, b])
            for a, b in todo:
                got = self.values(a, b)
                want = TAG.tag_bytes(seed, self.va + a, b - a) if seed is not None else np.zeros(b - a, np.uint8)
                m = got != want
                if m.any():
                    out.append((a, b, m, got))
        return out


def book(mem: Mem, ranges, seed: int | None = None, chunk_of=lambda o: 0, zero_windows: bool = False) -> dict:
    """A window book over `ranges` (include/ccm.h: the dirt, mismatch and residue reports and their page maps): exact
    counts, first and last booked byte, the page map, and the records when there are at most RECORDS windows."""
    parts = mem.booked(ranges, seed)
    nbytes, pages, first, last = 0, {}, None, None
    wins: list[tuple[int, int]] = []     # window index intervals [a, b]
    zero = 0
    for a, b, m, got in parts:
        if m is None:
            nbytes += b - a
            lo, hi = a, b - 1
            for p in range(a // PAGE, (b - 1) // PAGE + 1):
                pages[p] = pages.get(p, 0) + min(b, (p + 1) * PAGE) - max(a, p * PAGE)
            wins.append((a >> 4, (b - 1) >> 4))
        else:
            idx = np.flatnonzero(m).astype(np.int64) + a
            nbytes += idx.size
            lo, hi = int(idx[0]), int(idx[-1])
            pg, cnt = np.unique(idx // PAGE, return_counts=True)
            for p, k in zip(pg.tolist(), cnt.tolist()):
                pages[p] = pages.get(p, 0) + k
            w = np.unique(idx >> 4)
            cut = np.flatnonzero(np.diff(w) != 1)
            starts = np.concatenate(([0], cut + 1))
            ends = np.concatenate((cut, [w.size - 1]))
            wins += [(int(w[s]), int(w[e])) for s, e in zip(starts, ends)]
            if zero_windows:   # booked windows whose bytes inside the piece all read 0
                wid = (np.arange(a, b, dtype=np.int64) >> 4) - (a >> 4)
                nzw = np.zeros(int(wid[-1]) + 1, bool)
                np.logical_or.at(nzw, wid, got != 0)
                bkw = np.zeros_like(nzw)
                bkw[(idx >> 4) - (a >> 4)] = True
                zero += int((bkw & ~nzw).sum())
        first = lo if first is None else min(first, lo)
        last = hi if last is None else max(last, hi)
    wins.sort()
    merged: list[list[int]] = []
    for a, b in wins:
        if merged and a <= merged[-1][1] + 1:
            merged[-1][1] = max(merged[-1][1], b)
        else:
            merged.append([a, b])
    nwin = sum(b - a + 1 for a, b in merged)
    out = {"bytes": nbytes, "windows": nwin, "first": first or 0, "last": last or 0,
           "pages": [(p, k, chunk_of(p * PAGE)) for p, k in sorted(pages.items())], "records": None}
    region = [(lo, hi) for lo, hi in ranges]

    def window(w: int):
        lo, hi = w * 16, w * 16 + 16
        got = np.zeros(16, np.uint8)
        inside = np.zeros(16, bool)
        for a, b in region:
            s, e = max(lo, a), min(hi, b)
            if s < e:
                got[s - lo:e - lo] = mem.values(s, e)
                inside[s - lo:e - lo] = True
        return got, inside

    if zero_windows:
        out["zero_windows"] = zero
    if nwin <= RECORDS:
        recs = []
        for a, b in merged:
            for w in range(a, b + 1):
                got, inside = window(w)
                want = TAG.tag_bytes(seed, mem.va + w * 16, 16) if seed is not None else np.zeros(16, np.uint8)
                mask = sum(1 << i for i in range(16) if inside[i] and got[i] != want[i])
                rec = {"offset": w * 16, "chunk": chunk_of(w * 16), "mask": mask, "bytes": got.tobytes().hex()}
                if seed is not None:
                    rec["kind"] = (ZERO if not got[inside].any() else
                                   PARTIAL if any(inside[i] and got[i] == want[i] for i in range(16)) else FOREIGN)
                recs.append(rec)
        out["records"] = recs
    return out


def cut(ranges, skip):
    """`ranges` less the offsets [lo, hi) of `skip`."""
    if not skip or skip[0] >= skip[1]:
        return list(ranges)
    out = []
    for a, b in ranges:
        for s, e in ((a, min(b, skip[0])), (max(a, skip[1]), b)):
            if s < e:
                out.append((s, e))
    return out


# ------------------------------------------------------------------------------------------------ the call's layout
class Layout:
    """What a call maps and how it walks it, from tests/product_plan.py: the mappings (held spans), the enqueued ranges
    and the order GateRun takes them in, the read-back's spans, the chunk behind each offset and the probe's chunks."""

    def __init__(self, sc: dict, rec: dict):
        env, nbytes = sc.get("env", {}), sc["bytes"]
        res0 = rec["results"][-1]
        self.va = rec["va_base"]
        self.fallback = env.get("CCM_PIPELINE") == "0"
        self.alias = 0
        if self.fallback:
            # the fallback holds every segment, then enqueues them all at once, and reads back after its last drill
            segs = PP.arena_segments(nbytes, res0["device_free_before"], env)
            self.mapped = sum(n for _, n in segs)
            self.mappings = [(o, o + n) for o, n in segs]
            self.held, self.enqueue = [self.mappings], [self.mappings]
            self.order = [("held", 0), ("enqueue", 0)]
            self.interleave = False
            self.spans = list(self.mappings)
            self.chunk_lo, self.chunks = [o for o, _ in segs], list(range(len(segs)))
            self.segments = len(segs)
            return
        plan = PP.plan(nbytes, res0["device_free_before"], PP.H100_GRAN, env, node_fanout=sc.get("many", 0) > 1)
        run = PP.simulate(plan, res0["bytes_scrubbed"] if nbytes == 0 else None)
        self.mapped, self.interleave = run.mapped, plan.interleave
        tagged = sc.get("kind", "zero") in ("tagged", "census_tagged")
        # "scrub_alias" (ccm.h): the second main-zone chunk starts with a view of the first when it is at least as large
        if sc.get("drill", {}).get("scrub_alias") and len(run.main) >= 2 and run.main[1][1] >= run.main[0][1]:
            self.alias = run.main[0][1]
        self.chunk_lo, self.chunks, handle = [], [], 0
        for i, (o, n) in enumerate(run.chunks):
            if i == 1 and self.alias:
                self.chunk_lo.append(o)
                self.chunks.append(0)          # the aliased view reports handle 0
                if n == self.alias:
                    continue
                o += self.alias
            self.chunk_lo.append(o)
            self.chunks.append(handle)
            handle += 1
        self.segments = handle
        self.mappings = [(o, o + n) for o, n in run.chunks]
        ranges = [(o, o + n) for o, n in run.ranges(plan)]
        # GateRun order (csrc/ccm_scrub.cu scrub_verify_pipelined): each mapping is held as it is mapped; a main-zone
        # chunk is enqueued right after (a tagged call: after the last mapping), the tail granules as one range after
        # the loop, or everything as one range when the call maps first.
        self.held, self.enqueue = [[m] for m in self.mappings], [[r] for r in ranges]
        main = {(o, o + n) for o, n in run.main}
        order, deferred = [], []
        for i, m in enumerate(self.mappings):
            order.append(("held", i))
            if m in main and not plan.map_first:
                (deferred if tagged else order).append(("enqueue", ranges.index(m)))
        order += deferred
        if plan.map_first and ranges:
            order.append(("enqueue", 0))
        elif run.tail:
            order.append(("enqueue", len(ranges) - 1))
        self.order = order
        self.spans = [(0, self.mapped)]

    def chunk_of(self, off: int) -> int:
        return self.chunks[bisect.bisect_right(self.chunk_lo, off) - 1]


def merge(books: list[dict], chunk_of) -> dict | None:
    """One book from the books of several launches over disjoint ranges (None when nothing was booked)."""
    books = [b for b in books if b["bytes"]]
    if not books:
        return None
    pages: dict = {}
    for b in books:
        for p, k, _ in b["pages"]:
            pages[p] = pages.get(p, 0) + k
    nwin = sum(b["windows"] for b in books)
    recs = None
    if nwin <= RECORDS:
        recs = sorted((r for b in books for r in b["records"]), key=lambda r: r["offset"])
    out = {"bytes": sum(b["bytes"] for b in books), "windows": nwin, "first": min(b["first"] for b in books),
           "last": max(b["last"] for b in books), "records": recs,
           "pages": [(p, k, chunk_of(p * PAGE)) for p, k in sorted(pages.items())]}
    if "zero_windows" in books[0]:
        out["zero_windows"] = sum(b["zero_windows"] for b in books)
    return out


# ------------------------------------------------------------------------------------------------ the call
def predict(sc: dict, rec: dict) -> dict:
    """The observables (observe()) the call of scenario `sc` must return, given what the model takes from `rec`."""
    kind = sc.get("kind", "zero")
    tagged, census = kind in ("tagged", "census_tagged"), kind.startswith("census")
    d = {k: int(sc.get("drill", {}).get(k, 0)) for k in DRILL_KEYS}
    prove = bool(sc.get("prove"))
    L = Layout(sc, rec)
    mem = Mem(L.mapped, L.va, L.alias)
    chunk_of = L.chunk_of
    seed = rec["tags"][-1]["seed"] if tagged else None
    # "cover_skip" (ccm.h): pending for the first launch of the pass "cover_pass" chooses (0 and 3: the read-back)
    skip_pass = CO.DRILL_PASS[d["cover_pass"]]
    pending = {p: d["cover_skip"] if p == skip_pass else 0 for p in CO.PASSES}
    first_launch: dict = {}

    def launch(pass_: str, lo: int, hi: int) -> list:
        """What one launch of `pass_` over [lo, hi) walks: all of it, or less the chunks its drilled grab word skips
        (the read-back grabs downwards)."""
        first_launch.setdefault(pass_, (lo, hi - lo))
        k, pending[pass_] = pending[pass_], 0
        return cut([(lo, hi)], CO.skipped(lo, lo, hi - lo, k, pass_ == "readback") if k else None)

    def spend(lo: int, hi: int, budget: int, op) -> int:
        for o in PP.inject_offsets([(lo, hi - lo)], budget):
            op(o)
            budget -= 1
        return budget

    inject, tag_inject, residue = d["scrub_inject"], d["tag_inject"], d["scrub_residue"]
    census_books, check_books, readback = [], [], 0
    for what, i in L.order:
        if what == "held":
            for lo, hi in L.held[i]:
                if d["scrub_poison"]:
                    mem.write(lo, hi, d["scrub_poison"])
                if d["scrub_residue"]:     # every mapping is zero-filled; the budget only limits the 0xA5 bytes
                    mem.write(lo, hi, 0)
                    residue = spend(lo, hi, residue, lambda o: mem.write(o, o + 1, 0xA5))
            if tagged:
                for lo, hi in L.held[i]:
                    for a, b in launch("first", lo, hi):
                        if census:
                            census_books.append(book(mem, [(a, b)], chunk_of=chunk_of))
                        mem.tag(a, b, seed)
            continue
        spans = L.enqueue[i]
        if tagged:
            for lo, hi in spans:
                if d["tag_flood"]:
                    mem.write(lo, hi, d["tag_flood"])
                tag_inject = spend(lo, hi, tag_inject, mem.xor)
        for lo, hi in spans:
            for a, b in launch("check" if tagged else "first", lo, hi):
                if tagged:
                    check_books.append(book(mem, [(a, b)], seed, chunk_of, zero_windows=True))
                elif census:
                    census_books.append(book(mem, [(a, b)], chunk_of=chunk_of))
                mem.write(a, b, 0)
        for lo, hi in spans:
            if d["scrub_flood"]:
                mem.write(lo, hi, d["scrub_flood"])
            inject = spend(lo, hi, inject, lambda o: mem.write(o, o + 1, 0xA5))
        if L.interleave:
            for lo, hi in spans:
                readback += book(mem, launch("readback", lo, hi))["bytes"]
    if not L.interleave:
        for lo, hi in L.spans:
            readback += book(mem, launch("readback", lo, hi))["bytes"]

    check = merge(check_books, chunk_of)
    mismatch_bytes = check["bytes"] if check else 0
    nonzero = readback
    # ---- the probe (ccm.h ccm_scrub_probe): an armed zero gate whose passes finished and whose read-back was clean
    probe, pcover, mrep = {"probed": 0}, {"proved": 0}, None
    if sc.get("probe") and not tagged and nonzero == 0 and L.mapped:
        probe, mrep, nonzero = run_probe(mem, L, d, rec["probe"]["seed"])
        if prove:
            pcover = PCO.report([(L.va + a, b - a, a) for a, b in L.mappings], d["probe_skip"], d["probe_skip_step"])
            pcover["proved"] = 1
    # ---- the coverage proof (ccm.h ccm_scrub_prove)
    cover = {"proved": 0}
    if prove:
        drill = None
        if d["cover_skip"] and skip_pass in first_launch:
            drill = (skip_pass, d["cover_skip"], *first_launch[skip_pass])
        cover = CO.report(L.mapped, tagged, drill)
        cover["proved"] = 1
    if tagged and check:
        mrep = check
    residue_book = merge(census_books, chunk_of) if census else None
    # ---- the locate pass and the triages (ccm.h ccm_scrub_last_dirt, ccm_scrub_triage, ccm_scrub_mismatch_triage)
    rskip = {s: 0 for s in RO.STEPS}
    rskip[RO.STEPS[(d["report_skip_step"] or 4) - 1]] = d["report_skip"]   # 0 selects CCM_REPORT_DIRT_T3
    steps: dict = {}
    dirt = triage = mtriage = None
    if nonzero:
        dirt = book(mem, cut(L.spans, RO.skipped([(a, b - a) for a, b in L.spans], rskip["LOCATE"])), chunk_of=chunk_of)
        steps["LOCATE"] = RO.step_report([(a, b - a) for a, b in L.spans], rskip["LOCATE"])
        if sc.get("triage") and dirt["pages"]:
            triage = run_triage(mem, L, d, dirt["pages"], rskip, steps, "DIRT", None, sc["triage"])
    if tagged and check and sc.get("mismatch_triage"):
        mtriage = run_triage(mem, L, d, check["pages"], rskip, steps, "MISMATCH", seed, sc["mismatch_triage"])
    # ---- the verdict (csrc/ccm_scrub.cu engine_scrub_verify; include/ccm.h as cited in PRECEDENCE)
    fails = {"pass_uncovered": bool(prove and not cover["covered"]),
             "probe_uncovered": bool(pcover["proved"] and not pcover["covered"]),
             "tag_mismatch": bool(mismatch_bytes),
             "probe_mismatch": bool(probe["probed"] and probe["mismatch_bytes"]),
             "dirty": bool(nonzero)}
    failed = [n for n in PRECEDENCE if fails[n]]
    rc = {"pass_uncovered": UNCOVERED, "probe_uncovered": UNCOVERED, "tag_mismatch": MISMATCH,
          "probe_mismatch": MISMATCH, "dirty": DIRTY}[failed[0]] if failed else OK
    count = max(1, sc.get("many", 0))
    env = sc.get("env", {})
    res = {"status": rc, "bytes_scrubbed": L.mapped, "nonzero_bytes": nonzero, "segments": L.segments,
           "scrub_variant": 1, "verify_variant": 1,
           "release_deferred": int(not L.fallback and env.get("CCM_ASYNC_RELEASE", "1") != "0")}
    return {"rc": rc, "fails": failed, "results": [res] * count,
            "tags": [mismatch_bytes] * count if tagged else None,
            "residue": [[residue_book["bytes"], residue_book["windows"]] if residue_book else [0, 0]] * count
            if census else None,
            "dirt": _dirt_obs(dirt), "mismatch": _mismatch_obs(mrep),
            "pages1": [list(p) for p in dirt["pages"]] if dirt else [],
            "pages2": [list(p) for p in mrep["pages"]] if mrep else [],
            # the residue page map is the last census call's (ccm.h ccm_last_page_map): only a census call replaces it
            "pages3": ([list(p) for p in residue_book["pages"]] if residue_book else []) if census else None,
            "triage": triage or _untriaged(), "mismatch_triage": mtriage or _untriaged(),
            "cover": _cover_obs(cover, chunk_of), "probe": probe, "probe_cover": _pcover_obs(pcover),
            "report_cover": _rcover_obs(prove, steps)}


# ------------------------------------------------------------------------------------------------ the alias probe
def run_probe(mem: Mem, L: Layout, d: dict, seed: int):
    """P1, "probe_mismatch", P2, "probe_dirt", P3 (ccm.h ccm_scrub_probe) over every window of every mapping (the
    fallback: segment), in launch order.  Windows over memory that holds zero and that no drill touches end as they
    began and book nothing, so only the others are walked one by one: the drills' first windows, the skipped ones,
    both views of an alias, and those over non-zero memory.  Returns (probe report, mismatch book, P3 count)."""
    chunks = [(lo, PCO.chunk_windows(L.va + lo, hi - lo)) for lo, hi in L.mappings]
    total = sum(n for _, (_, n) in chunks)
    starts = [w0 - L.va for _, (w0, _) in chunks]
    counts = [n for _, (_, n) in chunks]

    def nth(i: int) -> int:
        for s, n in zip(starts, counts):
            if i < n:
                return s + i * STRIDE
            i -= n
        raise IndexError(i)

    first = next((k for k, n in enumerate(counts) if n), None)
    skipped = set()
    if d["probe_skip"] and first is not None:
        skipped = {starts[first] + i * STRIDE for i in range(min(d["probe_skip"], counts[first]))}
    step = d["probe_skip_step"] or 2
    special = set(skipped)
    special |= {nth(i) for i in range(min(total, max(d["probe_mismatch"], d["probe_dirt"])))}
    if L.alias:
        special |= {w for s, n in zip(starts, counts) for w in range(s, s + n * STRIDE, STRIDE) if w < 2 * L.alias}
    for a, b, c, _ in mem.segments(0, L.mapped):
        if c != ("b", 0):
            if b - a > GATHER_LIMIT:
                raise Unpredictable("a probe over a large dirty span")
            for s, n in zip(starts, counts):
                lo = max(0, -(-(a - WINDOW + 1 - s) // STRIDE))
                hi = min(n, (b - 1 - s) // STRIDE + 1)
                special |= {s + i * STRIDE for i in range(lo, hi)}
    wins = sorted(special)
    for w in wins:                                           # P1
        if not (step == 1 and w in skipped):
            mem.tag(w, w + WINDOW, seed)
    xor_first = [nth(i) for i in range(min(total, d["probe_mismatch"]))]
    for w in xor_first:
        mem.xor(w)
    books = []
    for w in wins:                                           # P2
        if not (step == 2 and w in skipped):
            books.append(book(mem, [(w, w + WINDOW)], seed, L.chunk_of, zero_windows=True))
            mem.write(w, w + WINDOW, 0)
    for i in range(min(total, d["probe_dirt"])):
        mem.xor(nth(i))
    p3 = sum(book(mem, [(w, w + WINDOW)])["bytes"] for w in wins if not (step == 3 and w in skipped))
    m = merge(books, L.chunk_of)
    launched = sum(1 for n in counts if n)
    rep = {"probed": 1, "windows": total, "mismatch_bytes": m["bytes"] if m else 0,
           "mismatch_windows": m["windows"] if m else 0, "reread_nonzero_bytes": p3,
           "launches": 3 * launched + min(total, d["probe_mismatch"]) + min(total, d["probe_dirt"])}
    return rep, m, p3


# ------------------------------------------------------------------------------------------------ the triages
TRIAGE_FIELDS = ("pages_examined", "bytes_examined", "stay_pages", "stay_bytes", "return_pages", "return_bytes",
                 "clear_pages", "clear_bytes", "t2_bytes", "t3_bytes", "t2_first_offset", "t2_last_offset",
                 "t3_first_offset", "t3_last_offset", "hold_ms", "runs", "triaged")


def run_triage(mem: Mem, L: Layout, d: dict, pages, rskip: dict, steps: dict, which: str, seed, hold: int) -> dict:
    """A triage (ccm.h ccm_scrub_triage, or ccm_scrub_mismatch_triage when `seed` is given) over the runs of its page
    map `pages`: T1 (re-zero, or re-tag), "triage_stay", T2 (re-read, or check-and-zero), "triage_return", T3 (re-read),
    each step over every run, its first launch less what a "report_skip" of it skips."""
    runs = TO.runs(pages, [(a, b - a) for a, b in L.spans])
    parts = [(o, n) for o, n, _ in runs]
    names = [f"{which}_T{k}" for k in (1, 2, 3)]

    def walk(name: str) -> list:
        steps[name] = RO.step_report(parts, rskip[name])
        first = RO.skipped(parts, rskip[name])
        return [r for o, n in parts for r in cut([(o, o + n)], first)]

    def xor_pages(k: int) -> None:
        for p, _, _ in pages[:k]:
            o = p * PAGE
            if any(a <= o < a + n for a, n in parts):
                mem.xor(o)

    for a, b in walk(names[0]):
        mem.tag(a, b, seed) if seed is not None else mem.write(a, b, 0)
    xor_pages(d["triage_stay"])
    t2_walk = walk(names[1])
    t2 = merge([book(mem, [r], seed, L.chunk_of) for r in t2_walk], L.chunk_of)
    if seed is not None:
        for a, b in t2_walk:
            mem.write(a, b, 0)
    xor_pages(d["triage_return"])
    t3 = merge([book(mem, [r], None, L.chunk_of) for r in walk(names[2])], L.chunk_of)
    on2 = {p: k for p, k, _ in (t2["pages"] if t2 else [])}
    on3 = {p: k for p, k, _ in (t3["pages"] if t3 else [])}
    rows = []
    for p, k, c in pages:
        cls = 1 if on2.get(p) else 2 if on3.get(p) else 3
        rows.append([p, c, cls, k, on2.get(p, 0), on3.get(p, 0)])
    rep = {"pages_examined": len(pages), "bytes_examined": sum(parts[i][1] for i in range(len(parts))),
           "t2_bytes": t2["bytes"] if t2 else 0, "t3_bytes": t3["bytes"] if t3 else 0,
           "t2_first_offset": t2["first"] if t2 else 0, "t2_last_offset": t2["last"] if t2 else 0,
           "t3_first_offset": t3["first"] if t3 else 0, "t3_last_offset": t3["last"] if t3 else 0,
           "hold_ms": hold, "runs": len(runs), "triaged": 1}
    for cls, key in ((1, "stay"), (2, "return"), (3, "clear")):
        rep[f"{key}_pages"] = sum(1 for r in rows if r[2] == cls)
        rep[f"{key}_bytes"] = sum(r[3] for r in rows if r[2] == cls)
    return {"report": [rep[f] for f in TRIAGE_FIELDS], "pages": rows}


def _untriaged() -> dict:
    return {"report": [0] * len(TRIAGE_FIELDS), "pages": []}


# ------------------------------------------------------------------------------------------------ observables
def _dirt_obs(b) -> list:
    if not b:
        return [0, 0, 0, 0, 0, 0, []]
    recs = None if b["records"] is None else [[r["offset"], r["chunk"], r["mask"], r["bytes"]] for r in b["records"]]
    return [b["bytes"], b["windows"], b["first"], b["last"], min(b["windows"], RECORDS), 1, recs]


def _mismatch_obs(b) -> list:
    if not b:
        return [0, 0, 0, 0, 0, 0, []]
    recs = None if b["records"] is None else [[r["offset"], r["chunk"], r["mask"], r["kind"]] for r in b["records"]]
    return [b["bytes"], b["windows"], b["zero_windows"], b["first"], b["last"], min(b["windows"], RECORDS), recs]


PASS_KEYS = ("ran", "bytes_counted", "bytes_missing", "pages_short", "first_short_page")


def _cover_obs(c: dict, chunk_of) -> dict:
    if not c["proved"]:
        return {"proved": 0}
    return {"proved": 1, "covered": int(c["covered"]),
            "passes": {p: {k: c["passes"][p].get(k, 0) for k in PASS_KEYS} for p in CO.PASSES},
            "pages": [[p["page"], chunk_of(p["page"] * PAGE), p["expected"], p["first"], p["check"], p["readback"]]
                      for p in c["pages"]]}


PSTEP_KEYS = ("windows_counted", "windows_missing", "pages_short", "first_short_page")


def _pcover_obs(c: dict) -> dict:
    if not c["proved"]:
        return {"proved": 0}
    return {"proved": 1, "covered": c["covered"], "windows_expected": c["windows_expected"],
            "steps": [{k: s[k] for k in PSTEP_KEYS} for s in c["steps"]]}


RSTEP_KEYS = ("launches", "bytes_expected", "bytes_counted", "bytes_missing", "pages_short", "first_short_page")


def _rcover_obs(prove: bool, steps: dict) -> dict:
    if not prove or not steps:
        return {"proved": 0}
    return {"proved": 1, "covered": int(all(s["bytes_missing"] == 0 for s in steps.values())),
            "steps": {n: ({"ran": 1, **{k: steps[n][k] for k in RSTEP_KEYS}} if n in steps else {"ran": 0})
                      for n in RO.STEPS},
            "pages": [[n, p, e, g] for n in RO.STEPS if n in steps for p, e, g in steps[n]["pages"]]}


def observe(rec: dict) -> dict:
    """The observables of a call tests/report_cover_calls.py recorded, in predict()'s form."""
    r = rec["reports"]
    fail_rc = rec["rc"]
    dirt = list(r["dirt"])
    dirt[6] = None if dirt[1] > RECORDS else [list(x) for x in dirt[6]]
    mism = list(r["mismatch"])
    mism[6] = None if mism[1] > RECORDS else [list(x) for x in mism[6]]
    tri = {}
    for key, fn, pages in (("triage", "ccm_scrub_last_triage", "ccm_last_triage_pages"),
                           ("mismatch_triage", "ccm_scrub_last_mismatch_triage", "ccm_last_mismatch_triage_pages")):
        rep = dict(zip(TRIAGE_FIELDS_ALL, r[fn]))
        tri[key] = {"report": [rep[f] for f in TRIAGE_FIELDS], "pages": [list(p) for p in r[pages]]}
    cv = rec["cover"]
    cover = {"proved": 0}
    if cv["proved"]:
        cover = {"proved": 1, "covered": cv["covered"],
                 "passes": {p: ({k: cv["passes"][p][k] for k in PASS_KEYS} if cv["passes"][p]["ran"] else
                                {k: 0 for k in PASS_KEYS}) for p in CO.PASSES},
                 "pages": [[p["page"], p["chunk"], p["expected"], p["first"], p["check"], p["readback"]]
                           for p in rec["cover_pages"]]}
    pc = rec["probe_cover"]
    pcover = {"proved": 0} if not pc["proved"] else {
        "proved": 1, "covered": pc["covered"], "windows_expected": pc["windows_expected"],
        "steps": [{k: s[k] for k in PSTEP_KEYS} for s in pc["steps"]]}
    rc_ = rec["report_cover"]
    rcover = {"proved": 0} if not rc_["proved"] else {
        "proved": 1, "covered": rc_["covered"],
        "steps": {n: ({"ran": 1, **{k: rc_["steps"][n][k] for k in RSTEP_KEYS}} if rc_["steps"][n]["ran"]
                      else {"ran": 0}) for n in RO.STEPS},
        "pages": [[p["step"], p["page"], p["expected"], p["counted"]] for p in rc_["pages"]]}
    p = rec["probe"]
    probe = {"probed": 0} if not p["probed"] else {
        "probed": 1, **{k: p[k] for k in ("windows", "mismatch_bytes", "mismatch_windows", "reread_nonzero_bytes",
                                          "launches")}}
    return {"rc": fail_rc, "results": [{k: x[k] for k in RESULT_KEYS} for x in rec["results"]],
            "tags": [t["mismatch_bytes"] for t in rec["tags"]] if rec.get("tags") else None,
            "residue": [[x["residue_bytes"], x["residue_windows"]] for x in rec["residue"]] if rec.get("residue")
            else None,
            "dirt": dirt, "mismatch": mism, "pages1": [list(x) for x in r["pages1"]],
            "pages2": [list(x) for x in r["pages2"]],
            "pages3": [list(x) for x in r["pages3"]] if rec["call"].get("kind", "zero").startswith("census") else None,
            **tri,
            "cover": cover, "probe": probe, "probe_cover": pcover, "report_cover": rcover}


RESULT_KEYS = ("status", "bytes_scrubbed", "nonzero_bytes", "segments", "scrub_variant", "verify_variant",
               "release_deferred")
# ccm_triage_report as tests/cover_proof_calls.py records it (no times, no va_base)
TRIAGE_FIELDS_ALL = TRIAGE_FIELDS + ("reserved",)


def first_difference(want, got, path: str = ""):
    """(path, expected, returned) of the first field where `got` differs from `want`, or None."""
    if isinstance(want, dict) and isinstance(got, dict):
        for k in want:
            if k not in got:
                return f"{path}.{k}", want[k], "<absent>"
            diff = first_difference(want[k], got[k], f"{path}.{k}")
            if diff:
                return diff
        return None
    if isinstance(want, (list, tuple)) and isinstance(got, (list, tuple)):
        if len(want) != len(got):
            return f"{path}[len]", len(want), len(got)
        for i, (a, b) in enumerate(zip(want, got)):
            diff = first_difference(a, b, f"{path}[{i}]")
            if diff:
                return diff
        return None
    return None if want == got else (path, want, got)


def compare(sc: dict, rec: dict):
    """first_difference of the model's prediction and what the call returned (the verdict list is the model's own)."""
    want = predict(sc, rec)
    want.pop("fails")
    return first_difference(want, observe(rec))
