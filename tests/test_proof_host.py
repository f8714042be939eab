"""The host comparison of the coverage, probe and report proofs (csrc/ccm_proof.h) on the CPU: a driver over the
header fills the ABI structs from cover maps the oracles give (tests/cover_oracle.py, tests/probe_cover_oracle.py,
tests/report_cover_oracle.py), and every field and inexact page must be the oracle's.  Also what the oracles never
produce: pages counted twice, bytes in the outside slot, the probe's rounding up to whole windows, and the span
expectation against min(2 MiB, mapped - page offset).  And the Python reports built from the C structs, field by
name."""
from __future__ import annotations

import bisect
import json
import subprocess
from pathlib import Path

import pytest

import cover_oracle as CO
import probe_cover_oracle as PCO
import report_cover_oracle as RO
import test_probe_cover as TP
import test_report_cover as TR
from k8s_cc_manager_b200 import _native as N
from k8s_cc_manager_b200 import devices as D

ROOT = Path(__file__).resolve().parents[1]
MiB = 1 << 20
PAGE = CO.PAGE
VA = (3 << 34) + (5 << 21)   # an address

DRIVER = r'''
#include <cinttypes>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>
#include "ccm_proof.h"

struct Span { uint64_t addr, bytes, offset; };
struct Piece { uint64_t offset, bytes; };

static uint64_t u() { unsigned long long v = 0; if (scanf("%llu", &v) != 1) throw 1; return v; }
static std::vector<Span> spans() { std::vector<Span> v(u()); for (Span& s : v) { s.addr = u(); s.bytes = u(); s.offset = u(); } return v; }
static std::vector<Piece> pieces() { std::vector<Piece> v(u()); for (Piece& p : v) { p.offset = u(); p.bytes = u(); } return v; }
static ccm_proof::ChunkTable table() {
  ccm_proof::ChunkTable t(u());
  for (auto& c : t) { c.first = u(); c.second = (uint32_t)u(); }
  return t;
}
static std::vector<uint32_t> words(uint64_t n) { std::vector<uint32_t> v(n); for (uint32_t& w : v) w = (uint32_t)u(); return v; }
static void list(const std::vector<uint32_t>& v) {
  printf("[");
  for (size_t i = 0; i < v.size(); ++i) printf("%s%u", i ? "," : "", v[i]);
  printf("]\n");
}

int main() {
  ccm_report_cover rcover;
  memset(&rcover, 0, sizeof rcover);
  std::vector<ccm_report_cover_page> rpages;
  char cmd[32];
  while (scanf("%31s", cmd) == 1) {
    const std::string c = cmd;
    if (c == "cover") {
      const uint64_t np = u();
      const std::vector<Span> s = spans();
      const uint64_t mapped = u(), va_base = u();
      const bool ran[3] = {u() != 0, u() != 0, u() != 0};
      const ccm_proof::ChunkTable t = table();
      const std::vector<uint32_t> maps = words(3 * (np + 1));
      ccm_cover_report r;
      std::vector<ccm_cover_page> pages;
      ccm_proof::fill_cover(maps.data(), np, s, mapped, va_base, ran, t, &r, &pages);
      printf("{\"bytes_mapped\":%" PRIu64 ",\"pages_mapped\":%" PRIu64 ",\"va_base\":%" PRIu64 ",\"proved\":%d,"
             "\"covered\":%d,\"passes\":[", r.bytes_mapped, r.pages_mapped, r.va_base, r.proved, r.covered);
      for (int k = 0; k < 3; ++k) {
        const ccm_cover_pass& p = r.pass[k];
        printf("%s{\"ran\":%d,\"bytes_counted\":%" PRIu64 ",\"bytes_missing\":%" PRIu64 ",\"bytes_extra\":%" PRIu64
               ",\"bytes_outside\":%" PRIu64 ",\"pages_short\":%" PRIu64 ",\"pages_over\":%" PRIu64
               ",\"first_short_page\":%" PRIu64 "}", k ? "," : "", p.ran, p.bytes_counted, p.bytes_missing,
               p.bytes_extra, p.bytes_outside, p.pages_short, p.pages_over, p.first_short_page);
      }
      printf("],\"pages\":[");
      for (size_t i = 0; i < pages.size(); ++i)
        printf("%s[%" PRIu64 ",%u,%u,%u,%u,%u]", i ? "," : "", pages[i].page, pages[i].chunk, pages[i].expected,
               pages[i].count[0], pages[i].count[1], pages[i].count[2]);
      printf("]}\n");
    } else if (c == "probe") {
      const uint64_t np = u();
      const std::vector<Span> s = spans();
      const uint64_t va_base = u();
      const ccm_proof::ChunkTable t = table();
      const std::vector<uint32_t> maps = words(3 * (np + 1));
      ccm_probe_cover r;
      std::vector<ccm_probe_cover_page> pages;
      ccm_proof::fill_probe_cover(maps.data(), np, s, va_base, t, &r, &pages);
      printf("{\"windows_expected\":%" PRIu64 ",\"va_base\":%" PRIu64 ",\"proved\":%d,\"covered\":%d,\"steps\":[",
             r.windows_expected, r.va_base, r.proved, r.covered);
      for (int k = 0; k < 3; ++k) {
        const ccm_probe_cover_step& p = r.step[k];
        printf("%s{\"ran\":%d,\"windows_counted\":%" PRIu64 ",\"windows_missing\":%" PRIu64 ",\"windows_extra\":%" PRIu64
               ",\"windows_outside\":%" PRIu64 ",\"pages_short\":%" PRIu64 ",\"pages_over\":%" PRIu64
               ",\"first_short_page\":%" PRIu64 "}", k ? "," : "", p.ran, p.windows_counted, p.windows_missing,
               p.windows_extra, p.windows_outside, p.pages_short, p.pages_over, p.first_short_page);
      }
      printf("],\"pages\":[");
      for (size_t i = 0; i < pages.size(); ++i)
        printf("%s[%" PRIu64 ",%u,%u,%u,%u,%u]", i ? "," : "", pages[i].page, pages[i].chunk, pages[i].expected,
               pages[i].count[0], pages[i].count[1], pages[i].count[2]);
      printf("]}\n");
    } else if (c == "report") {   // one take; the first of a call starts the report proved and covered
      const uint64_t np = u();
      const int first = (int)u(), n = (int)u();
      const std::vector<Piece> p = pieces();
      const std::vector<uint32_t> l32 = words(CCM_REPORT_STEPS);
      const std::vector<uint64_t> launches(l32.begin(), l32.end());
      const ccm_proof::ChunkTable t = table();
      const std::vector<uint32_t> maps = words(n * (np + 1));
      if (!rcover.proved) {
        rcover.proved = 1;
        rcover.covered = 1;
      }
      ccm_proof::fill_report_steps(maps.data(), np, first, n, p, launches.data(), t, &rcover, &rpages);
    } else if (c == "report_out") {
      printf("{\"covered\":%d,\"steps\":[", rcover.covered);
      for (unsigned k = 0; k < CCM_REPORT_STEPS; ++k) {
        const ccm_report_cover_step& p = rcover.step[k];
        printf("%s{\"ran\":%d,\"launches\":%" PRIu64 ",\"bytes_expected\":%" PRIu64 ",\"bytes_counted\":%" PRIu64
               ",\"bytes_missing\":%" PRIu64 ",\"bytes_extra\":%" PRIu64 ",\"bytes_outside\":%" PRIu64
               ",\"pages_short\":%" PRIu64 ",\"pages_over\":%" PRIu64 ",\"first_short_page\":%" PRIu64 "}", k ? "," : "",
               p.ran, p.launches, p.bytes_expected, p.bytes_counted, p.bytes_missing, p.bytes_extra, p.bytes_outside,
               p.pages_short, p.pages_over, p.first_short_page);
      }
      printf("],\"pages\":[");
      for (size_t i = 0; i < rpages.size(); ++i)
        printf("%s[%" PRIu64 ",%u,%d,%u,%u]", i ? "," : "", rpages[i].page, rpages[i].chunk, rpages[i].step,
               rpages[i].expected, rpages[i].counted);
      printf("]}\n");
      memset(&rcover, 0, sizeof rcover);
      rpages.clear();
    } else if (c == "pieces") {
      const uint64_t np = u();
      list(ccm_proof::piece_bytes(pieces(), np));
    } else if (c == "probe_bytes") {
      const uint64_t np = u();
      list(ccm_proof::probe_bytes(spans(), np));
    } else if (c == "chunk") {
      const ccm_proof::ChunkTable t = table();
      printf("%u\n", ccm_proof::chunk_of(t, u()));
    } else {
      return 2;
    }
  }
  return 0;
}
'''


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    d = tmp_path_factory.mktemp("proof")
    (d / "driver.cpp").write_text(DRIVER)
    subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-Werror", "-I", str(ROOT / "k8s_cc_manager_b200" / "csrc"),
                    "-I", str(ROOT / "include"), str(d / "driver.cpp"), "-o", str(d / "driver")], check=True)

    def run(*commands) -> list:
        text = "\n".join(" ".join(str(int(x)) if not isinstance(x, str) else x for x in cmd) for cmd in commands)
        out = subprocess.run([str(d / "driver")], input=text + "\n", capture_output=True, text=True, check=True).stdout
        return [json.loads(line) for line in out.splitlines()]
    return run


def flat(pairs) -> list:
    return [len(pairs), *(x for p in pairs for x in p)]


def chunk_of(table, offset: int) -> int:
    """The chunk of the last allocation that starts at or before offset (the first when none does)."""
    i = bisect.bisect_right([o for o, _ in table], offset)
    return table[max(i - 1, 0)][1]


def as_map(per_page, np_: int, outside: int = 0) -> list[int]:
    """np page words from a list or a {page: bytes} dict, then the outside slot."""
    words = [0] * np_
    for p, b in (per_page.items() if isinstance(per_page, dict) else enumerate(per_page)):
        words[p] += b
    return words + [outside]


# ---------------------------------------------------------------------------------- coverage proof
ONE_RANGE = {"CCM_MAP_FIRST": "1", "CCM_INTERLEAVE_VERIFY": "1"}
TWO_RANGES = {"CCM_MAP_FIRST": "0", "CCM_INTERLEAVE_VERIFY": "0"}
FALLBACK = {"CCM_PIPELINE": "0", "CCM_ARENA_MAX_SEGMENT_MB": "3"}
CALLS = [(256 * MiB, ONE_RANGE), (1536 * MiB, TWO_RANGES), (10 * MiB + 777, FALLBACK)]


def cover_layout(nbytes: int, env: dict):
    """(ranges, mappings, interleave, mapped, spans, chunk table) of a call: the VMM path holds one span from va_base;
    the fallback holds its segments at their concatenated offsets, at addresses of their own."""
    ranges, mappings, interleave, mapped = CO.call_launches(nbytes, env)
    if env.get("CCM_PIPELINE") == "0":
        spans = [(VA + 3 * off + 4096 * i, n, off) for i, (off, n) in enumerate(mappings)]
    else:
        spans = [(VA, mapped, 0)]
    return ranges, mappings, interleave, mapped, spans, [(off, i) for i, (off, _) in enumerate(mappings)]


def cover_maps(mapped: int, tagged: bool, drill, np_: int) -> list[int]:
    """The three passes' maps a call leaves, as the oracle counts them; a pass that did not run leaves junk, which
    must never be compared."""
    maps = []
    for p in CO.PASSES:
        if p == "check" and not tagged:
            maps += [7] * (np_ + 1)
            continue
        skip = None
        if drill is not None and drill[0] == p:
            _, k, off, n = drill
            skip = CO.skipped(off, off, n, k, p == "readback")
        maps += as_map(CO.counts(mapped, skip), np_)
    return maps


@pytest.mark.parametrize("nbytes,env", CALLS)
@pytest.mark.parametrize("tagged", [False, True])
@pytest.mark.parametrize("drill", [None, (1, 1), (1, 9), (2, 2), (3, 1), (3, 3), (0, 10 ** 6)])
def test_cover_fill_matches_the_oracle(driver, nbytes, env, tagged, drill):
    ranges, mappings, interleave, mapped, spans, table = cover_layout(nbytes, env)
    np_ = -(-mapped // PAGE) + 3
    d = None
    if drill is not None:
        name = CO.DRILL_PASS[drill[0]]
        first = CO.first_launch(name, tagged, ranges, mappings, interleave, mapped)
        d = (name, drill[1], *first) if first else None
    want = CO.report(mapped, tagged, d)
    [got] = driver(("cover", np_, *flat(spans), mapped, VA, 1, int(tagged), 1, *flat(table),
                    *cover_maps(mapped, tagged, d, np_)))
    assert (got["bytes_mapped"], got["pages_mapped"], got["va_base"], got["proved"]) == (mapped, -(-mapped // PAGE), VA, 1)
    assert got["covered"] == int(want["covered"])
    for p, row in zip(CO.PASSES, got["passes"]):
        if not want["passes"][p]["ran"]:
            assert row == {**{k: 0 for k in row}, "ran": 0}, p
            continue
        assert {k: row[k] for k in want["passes"][p]} == want["passes"][p], p
        assert row["bytes_extra"] == row["bytes_outside"] == row["pages_over"] == 0, p
    assert [{"page": pg, "expected": e, "first": a, "check": b, "readback": c} for pg, _, e, a, b, c in got["pages"]] \
        == want["pages"]
    assert [ch for _, ch, *_ in got["pages"]] == [chunk_of(table, pg * PAGE) for pg, *_ in got["pages"]]


def test_cover_fill_counts_pages_over_and_the_outside_slot(driver):
    """A chunk counted twice on page 1 of the first pass, 5 bytes outside the read-back's map: extra bytes, pages over,
    no page entry for the outside slot, and not covered."""
    mapped, np_ = 5 * MiB + 7, 4
    exact = as_map(CO.expected(mapped), np_)
    first = list(exact)
    first[1] += CO.CHUNK
    readback = exact[:-1] + [5]
    [got] = driver(("cover", np_, 1, VA, mapped, 0, mapped, VA, 1, 0, 1, 1, 0, 0, *first, *[0] * (np_ + 1), *readback))
    f, _, r = got["passes"]
    assert f == {"ran": 1, "bytes_counted": mapped + CO.CHUNK, "bytes_missing": 0, "bytes_extra": CO.CHUNK,
                 "bytes_outside": 0, "pages_short": 0, "pages_over": 1, "first_short_page": 0}
    assert r == {"ran": 1, "bytes_counted": mapped + 5, "bytes_missing": 0, "bytes_extra": 5, "bytes_outside": 5,
                 "pages_short": 0, "pages_over": 0, "first_short_page": 0}
    assert got["pages"] == [[1, 0, PAGE, PAGE + CO.CHUNK, 0, PAGE]] and got["covered"] == 0
    [alone] = driver(("cover", np_, 1, VA, mapped, 0, mapped, VA, 1, 0, 1, 1, 0, 0, *exact, *[0] * (np_ + 1), *readback))
    assert alone["covered"] == 0 and alone["pages"] == []


@pytest.mark.parametrize("tiling", [[5 * MiB + 7], [3 * MiB, 3 * MiB, 1], [PAGE, 1, PAGE - 1, 17], [1] * 5, [0]])
def test_span_expectation_is_min_of_a_page_and_what_is_left(driver, tiling):
    offs = [sum(tiling[:i]) for i in range(len(tiling))]
    mapped = sum(tiling)
    np_ = -(-mapped // PAGE) + 2
    [got] = driver(("pieces", np_, *flat([(o, n) for o, n in zip(offs, tiling)])))
    assert got == [min(PAGE, mapped - p * PAGE) if p * PAGE < mapped else 0 for p in range(np_)]


def test_chunk_of_takes_the_last_allocation_at_or_before_an_offset(driver):
    table = [(0, 4), (3 * MiB, 5), (9 * MiB, 6)]
    offsets = [0, 3 * MiB - 1, 3 * MiB, 20 * MiB, (1 << 64) - 5]   # the last: a head window 5 bytes before base
    got = driver(*(("chunk", *flat(table), o) for o in offsets))
    assert got == [4, 4, 5, 6, 4]


# ---------------------------------------------------------------------------------- probe proof
@pytest.mark.parametrize("name", list(TP.GEOMETRIES))
@pytest.mark.parametrize("step", [0, 1, 2, 3])
@pytest.mark.parametrize("skip", [0, 1, 5, 700])
def test_probe_fill_matches_the_oracle(driver, name, step, skip):
    chunks = TP.GEOMETRIES[name]
    want = PCO.report(chunks, skip, step)
    exp = PCO.expected(chunks)
    np_ = max(exp) + 3
    hit = (2 if step == 0 else step) - 1
    maps = []
    for k in range(3):
        maps += as_map(PCO._count(chunks, skip) if k == hit else exp, np_)
    table = [(off, i) for i, (_, _, off) in enumerate(sorted(chunks, key=lambda c: c[2]))]
    [got] = driver(("probe", np_, *flat(chunks), VA, *flat(table), *maps))
    assert (got["windows_expected"], got["va_base"], got["proved"], got["covered"]) \
        == (want["windows_expected"], VA, 1, want["covered"])
    assert got["steps"] == [{"ran": 1, **s} for s in want["steps"]]
    assert {pg: (e, [a, b, c]) for pg, _, e, a, b, c in got["pages"]} == want["pages"]
    assert [pg for pg, *_ in got["pages"]] == sorted(want["pages"])
    assert [ch for _, ch, *_ in got["pages"]] == [chunk_of(table, pg * PAGE) for pg, *_ in got["pages"]]


def test_probe_bytes_split_a_window_across_a_page(driver):
    chunks = TP.GEOMETRIES["window_across_a_page"]   # offset 16 bytes short of a 32-byte multiple
    [got] = driver(("probe_bytes", 3, *flat(chunks)))
    assert got == [PCO.expected(chunks).get(p, 0) for p in range(3)] and got[0] % 32 == 16 and got[1] % 32 == 16


def test_probe_fill_rounds_up_to_whole_windows(driver):
    """Counts that are not whole windows: one byte missing, 33 bytes over, 5 bytes outside."""
    chunks = TP.GEOMETRIES["vmm"]
    exp = PCO.expected(chunks)
    np_ = max(exp) + 2
    m = [as_map(exp, np_) for _ in range(3)]
    m[0][2] -= 1
    m[1][1] += 33
    m[2][np_] = 5
    [got] = driver(("probe", np_, *flat(chunks), VA, 1, 0, 0, *m[0], *m[1], *m[2]))
    total = PCO.windows(chunks)
    p1, p2, p3 = got["steps"]
    assert (p1["windows_counted"], p1["windows_missing"], p1["windows_extra"], p1["pages_short"]) == (total, 1, 0, 1)
    assert p1["first_short_page"] == 2
    assert (p2["windows_counted"], p2["windows_extra"], p2["pages_over"], p2["windows_missing"]) == (total + 2, 2, 1, 0)
    assert (p3["windows_counted"], p3["windows_extra"], p3["windows_outside"], p3["pages_over"]) == (total + 1, 1, 1, 0)
    assert got["covered"] == 0
    assert [pg[0] for pg in got["pages"]] == [1, 2]


# ---------------------------------------------------------------------------------- report proof
def report_take(step: str, parts, k_of: dict, np_: int, table, outside: int = 0):
    """The `report` command of one take: the locate pass alone, or the three steps of a triage, each with its drill."""
    first = RO.STEPS.index(step) + 1
    names = RO.STEPS[first - 1: first + (0 if step == "LOCATE" else 2)]
    maps = []
    for s in names:
        maps += as_map(RO.per_page(parts, RO.skipped(parts, k_of.get(s, 0))), np_, outside)
    launches = [len(parts)] * len(RO.STEPS)
    return ("report", np_, first, len(names), *flat(parts), *launches, *flat(table), *maps)


@pytest.mark.parametrize("layout", sorted(TR.LAYOUTS))
@pytest.mark.parametrize("drilled", RO.STEPS)
@pytest.mark.parametrize("k", [0, 1, 3, 100])
def test_report_fill_matches_the_oracle(driver, layout, drilled, k):
    """The locate pass, the dirt triage and the mismatch triage of one call, in that order, one step drilled."""
    spans = TR.LAYOUTS[layout]
    np_ = -(-sum(n for _, n in spans) // PAGE) + 2
    table = [(o, i) for i, (o, _) in enumerate(spans)]
    takes, want_steps, want_pages = [], [], []
    for step in ("LOCATE", "DIRT_T1", "MISMATCH_T1"):
        parts = RO.pieces(step, spans, TR.DIRT, TR.MISMATCH)
        takes.append(report_take(step, parts, {drilled: k}, np_, table))
    for s in RO.STEPS:
        rep = RO.step_report(RO.pieces(s, spans, TR.DIRT, TR.MISMATCH), k if s == drilled else 0)
        want_steps.append({"ran": 1, **{f: v for f, v in rep.items() if f != "pages"}})
        want_pages += [[p, chunk_of(table, p * PAGE), RO.STEPS.index(s) + 1, e, c] for p, e, c in rep["pages"]]
    [got] = driver(*takes, ("report_out",))
    assert got["steps"] == want_steps
    assert got["pages"] == want_pages
    assert got["covered"] == int(not want_pages)


def test_report_fill_counts_pages_over_and_the_outside_slot(driver):
    """A triage whose three steps each count 9 bytes outside: extra, not covered, and no page entries; a locate pass
    that counts one page twice: one entry."""
    spans = TR.LAYOUTS["vmm"]
    np_ = 8
    runs = RO.pieces("DIRT_T1", spans, TR.DIRT, TR.MISMATCH)
    [got] = driver(report_take("DIRT_T1", runs, {}, np_, [(0, 0)], outside=9), ("report_out",))
    assert got["covered"] == 0 and got["pages"] == []
    total = sum(n for _, n in runs)
    for row in got["steps"][1:4]:
        assert (row["bytes_counted"], row["bytes_extra"], row["bytes_outside"], row["pages_over"]) == (total + 9, 9, 9, 0)
    m = as_map(RO.per_page(spans), np_)
    m[3] += 100
    [over] = driver(("report", np_, 1, 1, *flat(spans), *[1] * 7, 1, 0, 0, *m), ("report_out",))
    assert over["steps"][0]["pages_over"] == 1 and over["steps"][0]["bytes_extra"] == 100
    assert over["pages"] == [[3, 0, 1, PAGE, PAGE + 100]] and over["covered"] == 0
    assert [s["ran"] for s in over["steps"]] == [1, 0, 0, 0, 0, 0, 0]


# ---------------------------------------------------------------------------------- the Python reports
@pytest.mark.parametrize("report,native", [(D.CoverReport, N.CoverReport), (D.ProbeCoverReport, N.ProbeCover),
                                           (D.ReportCoverReport, N.ReportCover)])
def test_reports_take_every_field_of_their_struct_by_name(report, native):
    r = native()
    heads = [f for f, _ in native._fields_ if f != report.ROWS]
    for i, f in enumerate(heads):
        setattr(r, f, 1000 + i)
    for k, row in enumerate(getattr(r, report.ROWS)):
        for i, (f, _) in enumerate(row._fields_):
            setattr(row, f, 100 * k + i + 1)
    got = report.from_native(r, [None] * (D.COVER_PAGES + 1))
    assert [getattr(got, f) for f in heads] == [getattr(r, f) for f in heads]
    for name, row, want in zip(report.NAMES, getattr(got, report.ROWS), getattr(r, report.ROWS)):
        assert row.name == name
        assert all(getattr(row, f) == getattr(want, f) for f, _ in want._fields_ if f != "reserved"), (name, row)
    assert len(got.pages) == D.COVER_PAGES and got.pages_truncated == 1
