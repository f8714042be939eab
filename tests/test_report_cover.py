"""The report proof on the CPU: the oracle against a walk of every 4 KiB of small mappings (VMM and fallback spans,
runs of a dirt page map, the drill on each step); the C ABI without a CUDA device (exports, layouts from a C99
compile, drill keys); the locate twin's resource usage; ReportCoverReport in ScrubReport's and GpuError's JSON; the
device calls, the worker and the CLI; and the manager's report proof line and the unproven pages it marks on the dirt
and triage lines."""
from __future__ import annotations

import ctypes as C
import json
import logging
import re
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

import report_cover_oracle as RO
import scenarios as SC
import test_cover_proof as TC
import test_dirt_locate as TD
import test_dirt_triage as TT
from k8s_cc_manager_b200 import _native as N
from k8s_cc_manager_b200 import devices as D
from k8s_cc_manager_b200.devices import GpuError, ReportCoverPage, ReportCoverReport, ReportCoverStep, ScrubReport

ROOT = Path(__file__).resolve().parents[1]
MiB = 1 << 20
PAGE = RO.PAGE
UNIT = 4096

# (offset, bytes) spans of what a call holds: one mapping, or cudaMalloc segments at their concatenated offsets
LAYOUTS = {
    "vmm": [(0, 12 * MiB)],
    "vmm_ragged": [(0, 9 * MiB + 3 * UNIT)],
    "fallback_3mib": [(o, min(3 * MiB, 10 * MiB - o)) for o in range(0, 10 * MiB, 3 * MiB)],
    "fallback_odd": [(0, 5 * MiB), (5 * MiB, MiB), (6 * MiB, 7 * MiB + 5 * UNIT)],
}
DIRT = [(0, 10, 0), (1, 3, 0), (2, 1, 0), (4, 7, 1)]
MISMATCH = [(3, 16, 0), (5, 9, 1)]


# ---------------------------------------------------------------------------------- oracle against a walk
@pytest.mark.parametrize("layout", sorted(LAYOUTS))
@pytest.mark.parametrize("step", RO.STEPS)
@pytest.mark.parametrize("k", [0, 1, 3, 100])
def test_oracle_matches_a_walk_of_every_unit(layout, step, k):
    spans = LAYOUTS[layout]
    parts = RO.pieces(step, spans, DIRT, MISMATCH)
    assert parts, (layout, step)
    skip = RO.skipped(parts, k)
    got = {p: v for p, v in RO.per_page(parts, skip).items() if v}
    assert got == RO.brute_counts(parts, UNIT, skip)
    rep = RO.step_report(parts, k)
    assert rep["bytes_expected"] == sum(n for _, n in parts) == sum(RO.brute_counts(parts, UNIT).values())
    assert rep["launches"] == len(parts)
    o, n = parts[0]
    body = n // RO.CO.CHUNK   # the first launch's whole chunks (its range starts 128-byte aligned)
    assert rep["bytes_missing"] == min(k, body) * RO.CO.CHUNK
    assert rep["bytes_counted"] == rep["bytes_expected"] - rep["bytes_missing"]
    assert [p for p, _, _ in rep["pages"]] == sorted({a // PAGE for a in range(o, o + min(k, body) * RO.CO.CHUNK, UNIT)})


def test_locate_walks_the_spans_and_the_triages_the_runs_of_their_own_map():
    spans = LAYOUTS["fallback_3mib"]
    assert RO.pieces("LOCATE", spans) == spans
    # dirt pages 0, 1, 2, 4 cut at the 3 MiB segment boundaries; adjacent pieces inside one segment merged
    assert RO.pieces("DIRT_T2", spans, DIRT, MISMATCH) == [(0, 3 * MiB), (3 * MiB, 3 * MiB), (8 * MiB, MiB), (9 * MiB, MiB)]
    assert RO.pieces("MISMATCH_T1", spans, DIRT, MISMATCH) == [(6 * MiB, 2 * MiB)]
    assert sum(RO.per_page(RO.pieces("LOCATE", spans)).values()) == 10 * MiB


# ---------------------------------------------------------------------------------- caller-owned maps (ccm_region_prove)
def byte_walk_map(parts: list[tuple[int, int]], base: int, pages: int) -> list[int]:
    """The map, one byte at a time: each byte's page from base, or the outside slot."""
    m = np.zeros(pages + 1, np.int64)
    for a, n in parts:
        page = (np.arange(a, a + n, dtype=np.int64) - base) // PAGE
        np.add.at(m, np.where((page >= 0) & (page < pages), page, pages), 1)
    return m.tolist()


A = 1 << 40   # an address
MAP_CASES = [([(A + 5, 5 * MiB + 77)], A + 3 * MiB + 11, 1),               # below base, page 0, past it
             ([(A + 5, 5 * MiB + 77)], A - PAGE + 9, 2),                      # the whole region inside, unaligned base
             ([(A, 6 * MiB)], A, 3),                                          # exactly the map
             ([(A + 100, 40)], A + 120, 0),                                   # no page: everything outside
             ([(A + 7, 300), (A + 3 * PAGE - 17, 64), (A + 9 * MiB, 2 * MiB)], A + 1, 4)]


@pytest.mark.parametrize("parts,base,pages", MAP_CASES)
def test_cover_map_matches_a_byte_walk(parts, base, pages):
    assert RO.cover_map(parts, base, pages) == byte_walk_map(parts, base, pages)
    assert sum(RO.cover_map(parts, base, pages)) == sum(n for _, n in parts)
    assert {p: v for p, v in RO.per_page(parts, base=base).items() if v} == RO.brute_counts(parts, 1, base=base)


@pytest.mark.parametrize("chunk", [(A + 100, 4 * MiB), (A + 4096 - 9, 3 * 4096), (A + 4095, 2), (A, 31)])
def test_probe_map_is_32_bytes_per_window(chunk):
    w0, k = RO.PO.chunk_windows(*chunk)
    parts = RO.probe_parts([chunk])
    assert parts == [(w0 + 4096 * i, 32) for i in range(k)]
    for base in (w0 + 7, w0 + 4096 * (k // 2) + 7, chunk[0] - PAGE + 1):
        m = RO.cover_map(parts, base, 1)
        assert m == byte_walk_map(parts, base, 1) and sum(m) == 32 * k, base


def test_map_bases_cut_where_the_kernels_split():
    """A region longer than a page and two chunks: base and every page boundary but the last cut a chunk of the body,
    the last cuts the tail, and bytes lie before base and past the last page.  A shorter one: each cut on each side."""
    CH = RO.CO.CHUNK
    for addr in (A, A + 1, A + 17, A + 127):
        for n in (PAGE + 2 * CH + 200, 16 * MiB + 3, (1 << 34) - 8, 3 * PAGE + 1 - (addr - A)):
            head = (128 - addr % 128) % 128
            base, pages = RO.map_base(addr, n, 0)
            assert pages >= 1 and base > addr + head and (base - addr - head) % CH != 0, (addr, n)
            assert addr + n - 2 <= base + pages * PAGE < addr + n, (addr, n)
            m = RO.cover_map([(addr, n)], base, pages)
            assert m[-1] == (base - addr) + (addr + n - base - pages * PAGE) and 0 < min(m[:-1]), (addr, n)
        n = 3 * CH + 77
        seen = {RO.map_base(addr, n, run) for run in range(8)}
        assert len(seen) == 8 and {p for _, p in seen} == {1}, addr
        for base, _ in seen:
            assert addr < base < addr + n or addr < base + PAGE < addr + n


# ---------------------------------------------------------------------------------- the C ABI
ENTRY_POINTS = ("ccm_scrub_last_report_cover", "ccm_last_report_cover_pages")


def test_region_prove_is_exported_and_refuses_a_missing_device(native):
    lib = N.lib()
    nm = subprocess.run(["nm", "-D", "--defined-only", str(N.LIB_PATH)], capture_output=True, text=True,
                        check=True).stdout
    assert "ccm_region_prove" in N.EXPORTED_SYMBOLS and re.search(r" T ccm_region_prove$", nm, re.M)
    header = (ROOT / "include" / "ccm.h").read_text()
    assert re.search(r"^int ccm_region_prove\(int cuda_ordinal, uint32_t\* map, uint64_t base, uint32_t pages\);",
                     header, re.M)
    words = (C.c_uint32 * 4)()
    for ordinal in (-1, 1 << 12):
        assert lib.ccm_region_prove(ordinal, C.cast(words, C.c_void_p), 0, 3) == N.ERR_NO_CUDA
        assert lib.ccm_region_prove(ordinal, None, 0, 0) == N.ERR_NO_CUDA


def test_entry_points_are_exported_and_refuse_what_they_must(native):
    lib = N.lib()
    nm = subprocess.run(["nm", "-D", "--defined-only", str(N.LIB_PATH)], capture_output=True, text=True,
                        check=True).stdout
    for fn in ENTRY_POINTS:
        assert fn in N.EXPORTED_SYMBOLS and re.search(rf" T {fn}$", nm, re.M), fn
    for ordinal in (-1, 1 << 12):
        rep = N.ReportCover(proved=7)
        assert lib.ccm_scrub_last_report_cover(ordinal, C.byref(rep)) == N.ERR_NO_CUDA and rep.proved == 0
        n = C.c_uint64(7)
        assert lib.ccm_last_report_cover_pages(ordinal, None, 0, C.byref(n)) == N.ERR_NO_CUDA and n.value == 0
    assert lib.ccm_scrub_last_report_cover(0, None) == N.ERR_INVALID
    assert lib.ccm_last_report_cover_pages(0, None, 0, None) == N.ERR_INVALID
    n = C.c_uint64()
    assert lib.ccm_last_report_cover_pages(0, None, 3, C.byref(n)) == N.ERR_INVALID
    assert "ccm_last_report_cover_pages: cap 3" in N.last_error()
    assert D.last_report_cover(-1) is None and D.last_report_cover_pages(-1) is None
    header = (ROOT / "include" / "ccm.h").read_text()
    for fn in ENTRY_POINTS:
        assert re.search(rf"^int {fn}\(", header, re.M), fn
    assert '"report_skip"' in header and '"report_skip_step"' in header
    for k, name in enumerate(N.REPORT_STEPS):
        assert re.search(rf"CCM_REPORT_{name} = {k + 1},?$", header, re.M), name
    assert N.REPORT_STEPS == RO.STEPS


LAYOUT_C = r"""
#include <stddef.h>
#include <stdio.h>
#include "ccm.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu\n", sizeof(ccm_report_cover_step), sizeof(ccm_report_cover),
         sizeof(ccm_report_cover_page), offsetof(ccm_report_cover, ms_prove), offsetof(ccm_report_cover, proved),
         offsetof(ccm_report_cover, covered), offsetof(ccm_report_cover, step), offsetof(ccm_report_cover_step, ran),
         offsetof(ccm_report_cover_step, first_short_page), offsetof(ccm_report_cover_page, step),
         offsetof(ccm_report_cover_page, expected), offsetof(ccm_report_cover_page, counted));
  return 0;
}
"""


def test_struct_layouts_match_a_c99_compile(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "layout.c"
    src.write_text(LAYOUT_C)
    subprocess.run([cc, "-std=c99", "-Wall", "-Werror", "-I", str(ROOT / "include"), str(src), "-o",
                    str(tmp_path / "layout")], check=True)
    got = [int(x) for x in subprocess.run([str(tmp_path / "layout")], capture_output=True, text=True,
                                          check=True).stdout.split()]
    want = [C.sizeof(N.ReportCoverStep), C.sizeof(N.ReportCover), C.sizeof(N.ReportCoverPage),
            N.ReportCover.ms_prove.offset, N.ReportCover.proved.offset, N.ReportCover.covered.offset,
            N.ReportCover.steps.offset, N.ReportCoverStep.ran.offset, N.ReportCoverStep.first_short_page.offset,
            N.ReportCoverPage.step.offset, N.ReportCoverPage.expected.offset, N.ReportCoverPage.counted.offset]
    assert got == want == [80, 584, 24, 8, 16, 20, 24, 72, 64, 12, 16, 20]


def test_drill_keys_round_trip_and_refuse_what_they_must(native):
    lib = N.lib()
    assert lib.ccm_sim_topology(2, 0) == 0
    assert lib.ccm_sim_set(-1, b"cuda_ordinal", -1) == 0
    v = C.c_int64(-1)
    assert lib.ccm_sim_get(0, b"report_skip", C.byref(v)) == 0 and v.value == 0
    assert lib.ccm_sim_get(0, b"report_skip_step", C.byref(v)) == 0 and v.value == N.REPORT_DIRT_T3
    assert lib.ccm_sim_set(0, b"report_skip", 9) == 0 and lib.ccm_sim_get(0, b"report_skip", C.byref(v)) == 0
    assert v.value == 9
    for value, stored in [(s, s) for s in range(1, 8)] + [(0, N.REPORT_DIRT_T3)]:
        assert lib.ccm_sim_set(0, b"report_skip_step", value) == 0
        assert lib.ccm_sim_get(0, b"report_skip_step", C.byref(v)) == 0 and v.value == stored
    for bad in (-1, 8, 1 << 40):
        assert lib.ccm_sim_set(0, b"report_skip_step", bad) == N.ERR_INVALID
        assert "sim key 'report_skip_step' takes 0..7" in N.last_error()
    assert lib.ccm_sim_get(1, b"report_skip", C.byref(v)) == 0 and v.value == 0
    assert lib.ccm_sim_set(0, b"report_skip", 0) == 0


def test_locate_twin_has_no_spills_no_stack_and_one_cta_per_sm():
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not Path(cuobjdump).exists():
        pytest.skip("cuobjdump is not installed")
    out = subprocess.run([cuobjdump, "--dump-resource-usage", str(N.LIB_PATH)], capture_output=True, text=True,
                         check=True).stdout
    lines = out.splitlines()
    usage = [lines[i + 1] for i, line in enumerate(lines) if re.search(r"Function \S*cover_locate_pass\S*:", line)]
    assert len(usage) == 1
    assert re.search(r"STACK:0\b", usage[0]) and re.search(r"LOCAL:0\b", usage[0]), usage
    regs = int(re.search(r"REG:(\d+)", usage[0]).group(1))
    assert 512 * regs <= 65536, regs   # a 512-thread CTA still fits one SM's register file


# ---------------------------------------------------------------------------------- reports and JSON
def sample_report_cover(covered=1) -> ReportCoverReport:
    steps = [ReportCoverStep(name, int(name in ("LOCATE", "DIRT_T1", "DIRT_T2", "DIRT_T3")), 1, 6 * MiB if
                             name == "LOCATE" else 2 * MiB, 6 * MiB if name == "LOCATE" else 2 * MiB, 0, 0, 0, 0, 0, 0)
             for name in N.REPORT_STEPS]
    steps = [s if s.ran else ReportCoverStep(s.name, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0) for s in steps]
    pages = []
    if not covered:
        steps[3] = ReportCoverStep("DIRT_T3", 1, 1, 2 * MiB, 2 * MiB - (1 << 17), 1 << 17, 0, 0, 1, 0, 2)
        pages = [ReportCoverPage(2, 0, "DIRT_T3", 2 * MiB, 2 * MiB - (1 << 17))]
    return ReportCoverReport(0x7F0000000000, 0.1, 1, covered, steps, pages)


def test_json_carries_the_report_only_when_a_proof_ran():
    rep = TC.zero_report("0000:01:00.0")
    assert "report_cover" not in rep.as_json()
    rep.report_cover = sample_report_cover(0)
    d = rep.as_json()
    assert d["report_cover"]["steps"][3]["bytes_missing"] == 1 << 17
    back = ScrubReport.from_json(json.loads(json.dumps(d)))
    assert back.report_cover == sample_report_cover(0)
    assert GpuError("x").report_cover is None


def test_summary_names_the_short_step_and_its_pages():
    assert sample_report_cover(1).summary() == \
        "every step walked every byte of its reports once (LOCATE, DIRT_T1, DIRT_T2, DIRT_T3)"
    s = sample_report_cover(0).summary()
    assert "step DIRT_T3 counted 1966080 of 2097152 bytes (131072 missing, 0 extra) with 1 pages short, first short " \
           "page 2" in s
    assert "page 2 (chunk 0): DIRT_T3 counted 1966080 of 2097152 bytes" in s
    assert sample_report_cover(0).unproven_pages("triage") == [2]
    assert sample_report_cover(0).unproven_pages("dirt") == sample_report_cover(0).unproven_pages("mismatch_triage") == []


def test_native_report_converts():
    r = N.ReportCover(va_base=5, ms_prove=0.5, proved=1, covered=0)
    r.steps[3].ran, r.steps[3].bytes_missing, r.steps[3].launches = 1, 7, 2
    rep = ReportCoverReport.from_native(r, [ReportCoverPage(1, 0, "DIRT_T3", 9, 2)] * (D.COVER_PAGES + 1))
    assert [s.name for s in rep.steps] == list(N.REPORT_STEPS)
    assert rep.steps[3].bytes_missing == 7 and rep.steps[3].launches == 2 and rep.short_steps() == [rep.steps[3]]
    assert len(rep.pages) == D.COVER_PAGES and rep.pages_truncated == 1


def test_cli_prints_the_keys_the_worker_prints():
    src = (ROOT / "k8s_cc_manager_b200" / "csrc" / "ccm_scrub_cli.cpp").read_text()
    body = src[src.index("static void print_rcover"):src.index('// The "probe" object')]
    printed = set(re.findall(r'\\"(\w+)\\":', body))
    assert printed == ({"report_cover"} | set(ReportCoverReport.__dataclass_fields__)
                       | set(ReportCoverStep.__dataclass_fields__) | set(ReportCoverPage.__dataclass_fields__))
    assert "prove && ccm_scrub_last_report_cover(ordinals[i], &rc) == CCM_OK && rc.proved" in src


def test_worker_prints_the_key_only_for_a_proven_call_that_proved_its_reports(monkeypatch, capsys):
    from k8s_cc_manager_b200 import scrub_worker

    def fake_many(devs, n, check="zero", residue=False, triage=False, triage_hold_ms=D.TRIAGE_HOLD_MS,
                  mismatch_triage=False, prove=False, probe=False):
        rep = TC.zero_report(devs[0].bdf, N.ERR_DIRTY)
        rep.nonzero_bytes = 3
        rep.cover = TC.sample_cover(1) if prove else None
        rep.report_cover = sample_report_cover(0) if prove else None
        return [rep], 1.0
    monkeypatch.setattr(D, "find_gpus", lambda: ([TC._Dev("0000:01:00.0")], 1))
    monkeypatch.setattr(D, "scrub_and_verify_many", fake_many)
    for argv, key in ((["--prove", "--triage"], True), (["--triage"], False), ([], False)):
        assert scrub_worker.main(["--bdf", "0000:01:00.0", *argv]) == 3
        rep = json.loads(capsys.readouterr().out.strip().splitlines()[-1])["reports"][0]
        assert ("report_cover" in rep) == key
        if key:
            assert rep["status"] == N.ERR_DIRTY
            assert ReportCoverReport.from_json(rep["report_cover"]) == sample_report_cover(0)


def test_device_calls_attach_the_proof_and_never_change_the_status(monkeypatch):
    monkeypatch.setattr(D, "_arm_prove", lambda o, on: N.OK)
    monkeypatch.setattr(D, "last_cover", lambda o: TC.sample_cover(1))
    proof = {"value": sample_report_cover(0)}
    monkeypatch.setattr(D, "last_report_cover", lambda o: proof["value"])
    lib = type("Lib", (), {"ccm_scrub_verify_many": staticmethod(lambda n, idx, nbytes, res, wall: 0),
                           "ccm_scrub_last_report_cover": staticmethod(lambda o, out: N.OK)})()
    monkeypatch.setattr(N, "lib", lambda: lib)
    devs = [type("Dev", (), {"index": 0, "cuda_ordinal": 0, "bdf": "0000:01:00.0"})()]
    reports, _ = D.scrub_and_verify_many(devs, prove=True)
    assert reports[0].status == 0 and reports[0].report_cover == sample_report_cover(0)
    reports, _ = D.scrub_and_verify_many(devs)
    assert reports[0].report_cover is None
    # a proof that did not run (a clean call) or cannot be read attaches nothing, and fails nothing
    for value in (ReportCoverReport(0, 0.0, 0, 0), None):
        proof["value"] = value
        reports, _ = D.scrub_and_verify_many(devs, prove=True)
        assert reports[0].report_cover is None and reports[0].status == 0


def test_a_single_device_call_carries_it_on_its_error(native, monkeypatch):
    lib = native.lib()
    assert lib.ccm_sim_topology(1, 0) == 0
    gpu = [d for d in D.find_gpus()[0] if d.is_gpu()][0]
    monkeypatch.setattr(D, "_arm_prove", lambda o, on: N.OK)
    monkeypatch.setattr(D, "last_cover", lambda o: TC.sample_cover(1))
    monkeypatch.setattr(D, "last_dirt", lambda o: TD.sample_dirt())
    monkeypatch.setattr(D, "last_report_cover", lambda o: sample_report_cover(0))
    real = N.lib()

    def dirty(index, nbytes, res):
        res._obj.nonzero_bytes, res._obj.status = 3, N.ERR_DIRTY
        return N.ERR_DIRTY
    fake = type("Lib", (), {"__getattr__": lambda self, name: getattr(real, name),
                            "ccm_scrub_verify": staticmethod(dirty)})()
    monkeypatch.setattr(N, "lib", lambda: fake)
    with pytest.raises(GpuError) as err:
        gpu.scrub_and_verify(prove=True)
    assert err.value.status == N.ERR_DIRTY and err.value.report_cover == sample_report_cover(0)
    assert err.value.dirt == TD.sample_dirt()


# ---------------------------------------------------------------------------------- manager
def report_lines(caplog, prefix):
    return [(r.levelno, r.getMessage()) for r in caplog.records if r.getMessage().startswith(prefix)]


@pytest.mark.parametrize("covered", [1, 0])
def test_manager_logs_the_proof_and_marks_the_unproven_triage_pages(monkeypatch, caplog, covered):
    bdf = SC.GPU_BDFS[0]
    mgr, _ = TD.manager_for([], monkeypatch, scrub_proof="require", scrub_triage="report")
    holder = GpuError("dirty", N.ERR_DIRTY)
    holder.dirt, holder.triage, holder.report_cover = TD.sample_dirt(), TT.sample_triage(), sample_report_cover(covered)
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        mgr._note_reports(bdf, holder)
    assert mgr.last_transition["scrub_report_cover"] == {bdf: sample_report_cover(covered)}
    level = logging.INFO if covered else logging.ERROR
    assert report_lines(caplog, "HBM report proof on ") == [
        (level, f"HBM report proof on {bdf}: {sample_report_cover(covered).summary()}")]
    triage = report_lines(caplog, "HBM dirt triage on ")
    assert len(triage) == 1 and triage[0][1].startswith(f"HBM dirt triage on {bdf}: {TT.sample_triage().summary()}")
    assert ("(unproven on pages 2: a step of the report proof was short there)" in triage[0][1]) == (not covered)
    dirt = report_lines(caplog, f"HBM dirt on {bdf}")
    assert len(dirt) == 1 and "unproven" not in dirt[0][1]
    # the report proof is a report: the labels and the verdict are the gate's own
    assert "scrub_cover" not in mgr.last_transition


def test_manager_without_a_proof_logs_no_proof_line(monkeypatch, caplog):
    mgr, _ = TD.manager_for([], monkeypatch, scrub_triage="report")
    holder = GpuError("dirty", N.ERR_DIRTY)
    holder.dirt, holder.triage = TD.sample_dirt(), TT.sample_triage()
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        mgr._note_reports(SC.GPU_BDFS[0], holder)
    assert report_lines(caplog, "HBM report proof on ") == []
    assert "scrub_report_cover" not in mgr.last_transition
