"""The page maps on the CPU: the numpy oracle against a window-by-window restatement, PageMap's runs and per-chunk totals,
the JSON of reports that carry pages (a whole-HBM-sized sparse map included), the CLI's and the worker's keys, the
manager's page lines beside the report lines, and the C ABI of ccm_last_page_map without a CUDA device."""
from __future__ import annotations

import ctypes as C
import json
import logging
import re
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

import scenarios as SC
import test_dirt_locate as TD
from k8s_cc_manager_b200 import _native as N
from k8s_cc_manager_b200 import devices as D
from k8s_cc_manager_b200.devices import (ChunkPages, MismatchReport, MismatchWindow, PageDigest, PageMap,
                                         PageRun, ResidueReport, ResidueWindow, ScrubReport)

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "oracle"))
import page_oracle as PO  # noqa: E402
import tag_oracle as TO  # noqa: E402

MiB = 1 << 20
PAGE = PO.PAGE_BYTES


# ---------------------------------------------------------------------------------- oracle
@pytest.mark.parametrize("seed", range(4))
def test_oracle_matches_the_window_by_window_definition(seed):
    """Regions that start anywhere in a window, straddle page boundaries of their base and begin before it."""
    rng = np.random.default_rng(seed)
    ptr0 = 0x7F00_0000_0000
    for n in (0, 1, 15, 17, 100, 3000):
        for mis in (0, 1, 8, 15):
            ptr = ptr0 + 2 * PAGE - 40 + mis        # the region crosses the page boundary 2 pages past ptr0
            for base in (ptr, ptr0, ptr0 + 2 * PAGE - 1500, ptr + 3):
                buf = np.where(rng.random(n) < (0.05, 0.5, 1.0, 0.01)[seed], rng.integers(1, 256, n), 0).astype(np.uint8)
                assert PO.page_map(buf, ptr, base) == PO.brute_page_map(buf, ptr, base), (n, mis, base)
                tags = TO.tag_bytes(0x1234, ptr, n)
                flip = np.where(rng.random(n) < 0.1, buf, 0).astype(np.uint8)
                assert PO.check_page_map(tags ^ flip, ptr, 0x1234, base) == \
                    PO.brute_page_map(tags ^ flip, ptr, base, seed=0x1234), (n, mis, base)


def test_oracle_properties():
    ptr = 0x7F00_0000_0003                 # the head window starts 3 bytes before the region: page 0
    buf = np.zeros(3 * PAGE, dtype=np.uint8)
    buf[[0, PAGE - 4, PAGE - 3, 2 * PAGE + 5]] = 1
    got = PO.page_map(buf, ptr)
    # byte 2 PAGE + 5 lies on page 2 of the region, but its window starts 8 bytes earlier: offset 2 PAGE - 3, page 1
    assert got == {0: 3, 1: 1} and sum(got.values()) == np.count_nonzero(buf)
    full = np.ones(PAGE, dtype=np.uint8)
    assert PO.page_map(full, 0x1000_0000) == {0: PAGE}                       # a fully booked page: 2^21 in one word
    assert PO.entries({3: 5, 1: 2}, lambda o: o // (2 * PAGE)) == [(1, 2, 0), (3, 5, 1)]


# ---------------------------------------------------------------------------------- PageMap
def test_runs_and_per_chunk_totals():
    pm = PageMap([(5, 10, 1), (0, 3, 0), (1, 4, 0), (3, 1, 0), (4, 2, 1), (6, 7, 1), (7, 1, 2), (9, PAGE, 2)])
    assert len(pm) == 8 and pm.bytes == 3 + 4 + 1 + 2 + 10 + 7 + 1 + PAGE
    assert pm.by_chunk() == {0: 8, 1: 19, 2: 1 + PAGE}
    assert pm.runs() == [PageRun(0, 2, 0, 7), PageRun(3, 1, 0, 1), PageRun(4, 3, 1, 19), PageRun(7, 1, 2, 1),
                         PageRun(9, 1, 2, PAGE)]
    dg = pm.digest()
    assert (dg.pages, dg.bytes, dg.nruns, dg.runs_truncated) == (8, pm.bytes, 5, 0)
    assert dg.by_chunk == [ChunkPages(0, 3, 8), ChunkPages(1, 3, 19), ChunkPages(2, 2, 1 + PAGE)]
    line = dg.summary()
    assert "on 8 2 MiB pages in 5 runs" in line and "chunk 1: 19 B on 3 pages" in line
    assert "+0x0..+0x3fffff chunk 0 7 B" in line and "(+1 more)" in line
    # ctypes entries build the same map
    arr = (N.PageEntry * 2)(N.PageEntry(2, 5, 1), N.PageEntry(1, 4, 1))
    assert PageMap(arr).runs() == [PageRun(1, 2, 1, 9)]
    assert PageMap([]).digest() == PageDigest(0, 0, 0, 0, [], [])


def whole_hbm_sparse(seed=1) -> PageMap:
    """About 40 300 pages (80 GB) in 6 chunks, a sparse scatter with some stretches."""
    rng = np.random.default_rng(seed)
    npages = 40_300
    pages = sorted(set(rng.choice(npages, size=3000, replace=False).tolist()) | set(range(100, 400)))
    chunk_of = lambda p: min(p // 8192, 5)   # noqa: E731
    return PageMap([(p, int(rng.integers(PAGE // 2, PAGE + 1)), chunk_of(p)) for p in pages])


def test_whole_hbm_sparse_map_digest_round_trips_through_json():
    pm = whole_hbm_sparse()
    dg = pm.digest()
    assert dg.runs_truncated and len(dg.runs) == D.PAGE_RUNS and dg.runs == pm.runs()[:D.PAGE_RUNS]
    assert sum(c.bytes for c in dg.by_chunk) == pm.bytes == dg.bytes and sum(c.pages for c in dg.by_chunk) == len(pm)
    assert dg.bytes > 1 << 32                                   # the totals are not 32-bit
    js = json.loads(json.dumps(D.dataclasses.asdict(dg)))
    assert PageDigest.from_json(js) == dg


# ---------------------------------------------------------------------------------- reports
def sample_mismatch() -> MismatchReport:
    return MismatchReport(2, 2, 0, 0x10, 0x400011, 0x7F00_0000_0000, 7, 1, 0,
                          [MismatchWindow(0x10, 0, 1, "partial", 0, 0, "00" * 16),
                           MismatchWindow(0x400010, 2, 3, "foreign", 0, 0, "11" * 16)])


def sample_residue() -> ResidueReport:
    return ResidueReport(3, 2, 0x10, 0x2011, 1 << 30, 0x7F00_0000_0000, 1, 0,
                         [ResidueWindow(0x10, 0, 1), ResidueWindow(0x2010, 0, 3)])


def test_reports_keep_their_positional_form_and_round_trip_with_pages():
    for rep in (TD.sample_dirt(), sample_mismatch(), sample_residue()):
        kind = type(rep)
        assert rep.pages is None and list(kind.__dataclass_fields__)[-1] == "pages"
        assert kind.from_json(json.loads(json.dumps(rep.as_json()))) == rep
        rep.pages = whole_hbm_sparse(3).digest()
        js = json.loads(json.dumps(rep.as_json()))
        assert set(js["pages"]) == set(PageDigest.__dataclass_fields__)
        assert kind.from_json(js) == rep and kind.from_json(js).pages == rep.pages
        old = dict(js)
        del old["pages"]                      # a report written before the pages existed
        assert kind.from_json(old).pages is None
    sr = TD.report(nonzero=3)
    sr.dirt = TD.sample_dirt()
    sr.dirt.pages = PageMap([(0, 1, 0), (1, 2, 3)]).digest()
    js = json.loads(json.dumps(sr.as_json()))
    assert set(js) - {"dirt"} == set(TD.report().as_json()) and ScrubReport.from_json(js).dirt == sr.dirt


# ---------------------------------------------------------------------------------- CLI and worker
def test_cli_prints_the_keys_the_worker_prints():
    """The CLI's pages object has PageDigest's keys, each run PageRun's and each chunk ChunkPages'; each report printer
    prints a "pages" member."""
    src = (ROOT / "k8s_cc_manager_b200" / "csrc" / "ccm_scrub_cli.cpp").read_text()
    pages = src[src.index("static void print_pages"):src.index("static void print_dirt")]
    printed = set(re.findall(r'\\"(\w+)\\":', pages))
    assert printed == (set(PageDigest.__dataclass_fields__) | set(PageRun.__dataclass_fields__)
                       | set(ChunkPages.__dataclass_fields__))
    assert "keep = 64" in pages and D.PAGE_RUNS == 64
    for fn, book, nxt in (("print_dirt", "CCM_BOOK_DIRT", "static void print_mismatch"),
                          ("print_mismatch", "CCM_BOOK_MISMATCH", "static void print_residue"),
                          ("print_residue", "CCM_BOOK_RESIDUE", "static int usage")):
        body = src[src.index(f"static void {fn}"):src.index(nxt)]
        assert '\\"pages\\": ' in body and f"print_pages(ordinal, {book}," in body, fn


def test_worker_prints_pages_as_the_cli_does(monkeypatch):
    """Worker JSON of a report with pages: the same nested keys as the CLI prints, null when there are none."""
    from k8s_cc_manager_b200 import scrub_worker

    def fake_many(devs, nbytes=0, check="zero", residue=False):
        reps = []
        for d in devs:
            r = TD.report(d.bdf, nonzero=3)
            r.dirt = TD.sample_dirt()
            r.dirt.pages = PageMap([(0, 1, 0), (1, 2, 3)]).digest()
            r.residue = sample_residue()
            reps.append(r)
        return reps, 1.0

    class Dev:
        bdf = SC.GPU_BDFS[0]
        def is_gpu(self): return True
    monkeypatch.setattr(D, "find_gpus", lambda: ([Dev()], 1))
    monkeypatch.setattr(D, "scrub_and_verify_many", fake_many)
    out = json.loads(json.dumps(scrub_worker.run([SC.GPU_BDFS[0]], 4096, "zero", True)))
    rep = out["reports"][0]
    assert set(rep["dirt"]["pages"]) == set(PageDigest.__dataclass_fields__) and rep["residue"]["pages"] is None
    assert set(rep["dirt"]["pages"]["runs"][0]) == set(PageRun.__dataclass_fields__)


# ---------------------------------------------------------------------------------- manager
def test_manager_logs_a_page_line_beside_each_report_line(monkeypatch, caplog):
    dirt = TD.sample_dirt()
    dirt.pages = PageMap([(0, 1, 0), (1, 2, 3)]).digest()
    devs = [TD.FakeGpu(SC.GPU_BDFS[0]), TD.FakeGpu(SC.GPU_BDFS[1], dirt=dirt)]
    mgr, c = TD.manager_for(devs, monkeypatch)
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is False
    bdf = SC.GPU_BDFS[1]
    TD.assert_dirt_logged(mgr, c, caplog, bdf, dirt)          # the report line, as before
    msgs = [r.getMessage() for r in caplog.records]
    pages = [m for m in msgs if m.startswith(f"HBM dirt pages on {bdf}: ")]
    assert pages == [f"HBM dirt pages on {bdf}: {dirt.pages.summary()}"]
    assert msgs.index(pages[0]) == msgs.index(next(m for m in msgs if m.startswith(f"HBM dirt on {bdf}: "))) + 1


def test_manager_logs_no_page_line_without_pages(monkeypatch, caplog):
    devs = [TD.FakeGpu(SC.GPU_BDFS[0], dirt=TD.sample_dirt())]
    mgr, _ = TD.manager_for(devs, monkeypatch)
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is False
    assert not any(" pages on " in r.getMessage() for r in caplog.records)
    from k8s_cc_manager_b200 import manager
    assert set(manager.CCManager._PAGE_NOTES) == {a for a, *_ in manager.CCManager._REPORT_NOTES}
    for attr, _, _, line in manager.CCManager._REPORT_NOTES:
        assert manager.CCManager._PAGE_NOTES[attr] == line.replace(" on %s", " pages on %s")


# ---------------------------------------------------------------------------------- C ABI
def test_page_entry_layout_and_constants_match_the_header(tmp_path):
    src = tmp_path / "pages.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "ccm.h"\nint main(void){'
                   'printf("%zu %zu %zu %zu %u %d %d %d\\n", sizeof(ccm_page_entry), offsetof(ccm_page_entry,page),'
                   'offsetof(ccm_page_entry,bytes), offsetof(ccm_page_entry,chunk), CCM_PAGE_BYTES,'
                   'CCM_BOOK_DIRT, CCM_BOOK_MISMATCH, CCM_BOOK_RESIDUE);return 0;}')
    exe = tmp_path / "pages"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-pedantic", "-I", str(ROOT / "include"), str(src), "-o",
                    str(exe)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    E = N.PageEntry
    assert got == [C.sizeof(E), E.page.offset, E.bytes.offset, E.chunk.offset, N.PAGE_BYTES, N.BOOK_DIRT,
                   N.BOOK_MISMATCH, N.BOOK_RESIDUE]
    assert C.sizeof(E) == 16 and N.PAGE_BYTES == PAGE == 2 * MiB


def test_last_page_map_is_exported_and_needs_a_cuda_device(native):
    lib = native.lib()
    assert "ccm_last_page_map" in native.EXPORTED_SYMBOLS
    nm = subprocess.run(["nm", "-D", "--defined-only", str(native.LIB_PATH)], capture_output=True, text=True,
                        check=True).stdout
    assert re.search(r" T ccm_last_page_map$", nm, re.M)
    n = C.c_uint64(7)
    for ordinal in (-1, 1 << 12):
        assert lib.ccm_last_page_map(ordinal, native.BOOK_DIRT, None, 0, C.byref(n)) == native.ERR_NO_CUDA
        assert n.value == 0
    for book in (0, 4, -1):
        assert lib.ccm_last_page_map(0, book, None, 0, C.byref(n)) == native.ERR_INVALID
    assert lib.ccm_last_page_map(0, native.BOOK_DIRT, None, 0, None) == native.ERR_INVALID
    assert lib.ccm_last_page_map(0, native.BOOK_DIRT, None, 5, C.byref(n)) == native.ERR_INVALID
    assert D.last_page_map(-1, native.BOOK_DIRT) is None
