"""The page maps on one H100: the locate pass, the tag check and both censuses against the numpy page oracle on raw
regions (every start offset of tests/window_book_cases.py, page boundaries inside a grab, a fully booked page, a flood
past 2^32 bytes), and the product call's maps under every fault drill in every mapping mode, on the fallback and
through the fan-out, against what tests/product_plan.py predicts.  Every report is checked against its map: the
pages add up to its exact count, its first and last byte lie on the first and last page, and every record's page is
there with at least its mask's bytes."""
from __future__ import annotations

import ctypes as C
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "oracle"))
import page_oracle as PO  # noqa: E402
import product_gate_calls as PGC  # noqa: E402
import product_plan as PP  # noqa: E402
import tag_oracle as TO  # noqa: E402
import test_window_books_gpu as WBG  # noqa: E402
import window_book_cases as WB  # noqa: E402
from k8s_cc_manager_b200 import _native as N  # noqa: E402
from k8s_cc_manager_b200 import devices as D  # noqa: E402

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

GiB, MiB = 1 << 30, 1 << 20
PAGE = PO.PAGE_BYTES
SEED = WBG.SEED
BOOK = {"locate": N.BOOK_DIRT, "check": N.BOOK_MISMATCH, "census0": N.BOOK_RESIDUE, "census1": N.BOOK_RESIDUE}
DRILL_KEYS = WBG.DRILL_KEYS


@pytest.fixture(scope="module")
def lib():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return PGC.open_lib()


@pytest.fixture(autouse=True)
def _own_stream():
    if not torch.cuda.is_available():
        yield
        return
    with torch.cuda.stream(torch.cuda.Stream()):
        yield
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def page_map(book: int) -> dict:
    pm = D.last_page_map(0, book)
    assert pm is not None
    return {p: b for p, b, _ in pm.entries}


def page_entries(book: int) -> list:
    return D.last_page_map(0, book).entries


# ------------------------------------------------------------------------------------ the invariants
def count_of(rep) -> int:
    return {D.DirtReport: "nonzero_bytes", D.MismatchReport: "mismatch_bytes", D.ResidueReport: "residue_bytes"}[type(rep)]


def window_page(va_base: int, off: int) -> int:
    """The page of the window that holds the byte at offset `off` from va_base."""
    w = ((va_base + off) & ~15) - va_base
    return 0 if w < 0 else w // PAGE


def assert_report_invariants(rep, pages: dict, what):
    """Σ page bytes == the report's exact count; the first and last page hold its first and last byte's windows; every
    record's page is present with at least popc(mask) bytes (and, with records for every window, exactly them)."""
    count = getattr(rep, count_of(rep))
    assert sum(pages.values()) == count, what
    windows = getattr(rep, type(rep).WINDOWS)
    if windows == 0:
        assert pages == {}, what
        return
    assert min(pages) == window_page(rep.va_base, rep.first_offset), what
    assert max(pages) == window_page(rep.va_base, rep.last_offset), what
    per_page: dict = {}
    for r in rep.records:
        p = 0 if r.offset < 0 else r.offset // PAGE
        per_page[p] = per_page.get(p, 0) + bin(r.mask).count("1")
    for p, b in per_page.items():
        assert pages.get(p, 0) >= b, (what, p)
    if not rep.truncated and count_of(rep) != "mismatch_bytes":
        assert per_page == pages, what


# ------------------------------------------------------------------------------------ A. raw regions
def run_region(lib, rig, kind: str, off: int, region: np.ndarray, what, seed=SEED):
    """One region pass through tests/test_window_books_gpu.py's rig and checks (book against its oracle), then its
    page map against the page oracle and the report."""
    n = region.size
    ptr, _, _ = rig.place(off, region)
    if kind == "locate":
        rep = WBG.locate(lib, ptr, n)
        want = PO.page_map(region, ptr)
    elif kind == "check":
        rep = WBG.check_locate(lib, ptr, n, seed)
        want = PO.check_page_map(region, ptr, seed)
    else:
        rep = WBG.census(lib, ptr, n, kind == "census1", seed)
        want = PO.page_map(region, ptr)
    got = page_map(BOOK[kind])
    assert got == want, (kind, what)
    assert all(c == 0 for _, _, c in page_entries(BOOK[kind])), (kind, what)
    assert_report_invariants(rep, got, (kind, what))
    return rep, got


def boundary_content(kind, off, n, rng, rig, seed=SEED):
    """Dirt on both sides of every page boundary of the region (in region offsets and in window offsets), at its
    first and last bytes, and 300 more bytes anywhere."""
    pos = {0, n - 1} | set(rng.integers(0, n, size=300).tolist())
    for k in range(1, n // PAGE + 1):
        pos |= {k * PAGE + d for d in range(-40, 40) if 0 <= k * PAGE + d < n}
    wins = sorted({WB.window_of(off, r) for r in pos})
    masks = [int(rng.integers(1, 1 << 16)) & WB.in_region_mask(n, w) or WB.in_region_mask(n, w) for w in wins]
    return WBG.content_for(kind, off, n, wins, masks, rng, rig=rig, seed=seed)


def test_regions_at_every_offset_with_page_boundaries_inside_grabs(lib):
    """Every start offset the window-book cases cover; regions of 2 and 3 pages and a bit, whose page boundaries fall
    inside a grab (and inside a thread's batch) whenever the start is not 128-aligned."""
    lengths = (2 * PAGE + 3 * WB.CHUNK + 77, 3 * PAGE + 5)
    rig = WBG.Rig(max(lengths))
    rng = np.random.default_rng(11)
    for off in WB.OFFSETS:
        for n in lengths:
            for kind in WBG.PASSES:
                region = boundary_content(kind, off, n, rng, rig)
                run_region(lib, rig, kind, off, region, (off, n))


def test_small_placements_of_the_window_book_cases(lib):
    """The placements of tests/window_book_cases.py (head, tail, leftover and batch windows; every head-window count),
    sparse and dense: all on page 0, as the oracle says."""
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    g = WB.geometry(sm)
    rig = WBG.Rig(max(n for _, n in WB.placements(g)))
    rng = np.random.default_rng(19)
    for off, n in WB.placements(g)[::7]:
        ptr = rig.buf.data_ptr() + rig.lo + off
        for dense in (False, True):
            for kind in WBG.PASSES:
                region = WBG.placement_content(kind, g, off, n, ptr, dense, rng, SEED)
                run_region(lib, rig, kind, off, region, (off, n, dense))


def full_pages(n: int, mis: int) -> dict:
    """The page map of n booked bytes starting `mis` bytes past a 16-byte boundary: page p holds the bytes of the windows
    whose offsets lie in [p PAGE, (p + 1) PAGE) (page 0 also the head window, which starts before the region)."""
    first_window = lambda at: at + (-mis - at) % 16   # noqa: E731  (offset of the first window at or after `at`)
    out = {}
    for p in range(n // PAGE + 1):
        a, b = (0 if p == 0 else first_window(p * PAGE)), min(first_window((p + 1) * PAGE), n)
        if b > a:
            out[p] = b - a
    return out


def test_a_fully_booked_page_and_a_flood(lib):
    """Every byte booked: each whole page holds 2^21 in one counter, for all three books."""
    n = 3 * PAGE + 3 * WB.CHUNK + 9
    rig = WBG.Rig(n)
    for off in (0, 1, 17, 127):
        for kind in WBG.PASSES:
            ptr = rig.buf.data_ptr() + rig.lo + off
            region = np.full(n, 0xFF, dtype=np.uint8)
            if kind == "check":
                region = TO.tag_bytes(SEED, ptr, n) ^ np.uint8(0xFF)
            _, got = run_region(lib, rig, kind, off, region, ("flood", off))
            assert got == full_pages(n, ptr % 16) and got[1] == got[2] == PAGE, (kind, off)


def test_a_flood_past_2_to_the_32(lib):
    """A 4.5 GiB region of 0xFF: the pages add up past 2^32 (locate, then the census that zeroes it)."""
    n = 4 * GiB + GiB // 2 + 3
    buf = torch.full((n + 64,), 0xFF, dtype=torch.uint8, device="cuda")
    ptr = buf.data_ptr() + 1
    for kind in ("locate", "census0"):
        if kind == "locate":
            rep = WBG.locate(lib, ptr, n)
        else:
            rep = WBG.census(lib, ptr, n, False)
        got = page_map(BOOK[kind])
        assert got == full_pages(n, ptr % 16) and sum(got.values()) == n > 1 << 32, kind
        assert_report_invariants(rep, got, kind)
    del buf


def test_a_clean_call_after_a_dirty_one_costs_nothing_more(lib):
    """After a dirty pass, a clean one reports an empty map with exactly the launches of a clean pass; a second dirty
    pass shows only its own pages."""
    n = 3 * PAGE + 1000
    rig = WBG.Rig(n)
    rng = np.random.default_rng(23)
    for kind in WBG.PASSES:
        clean = TO.tag_bytes(SEED, rig.buf.data_ptr() + rig.lo + 5, n) if kind == "check" else np.zeros(n, np.uint8)
        run_region(lib, rig, kind, 5, clean, ("clean first", kind))
        l0 = lib.ccm_kernel_launches()
        run_region(lib, rig, kind, 5, clean, ("clean", kind))
        clean_launches = lib.ccm_kernel_launches() - l0
        run_region(lib, rig, kind, 5, boundary_content(kind, 5, n, rng, rig), ("dirty", kind))
        l0 = lib.ccm_kernel_launches()
        rep, got = run_region(lib, rig, kind, 5, clean, ("clean after dirty", kind))
        assert lib.ccm_kernel_launches() - l0 == clean_launches == 1, kind
        assert got == {} and getattr(rep, type(rep).WINDOWS) == 0, kind
        # two dirty passes: the second map is the second region's alone
        wins = [WB.window_of(5, PAGE + 100)]
        first = WBG.content_for(kind, 5, n, [WB.window_of(5, 2 * PAGE + 100)], [0xFFFF], rng, rig)
        run_region(lib, rig, kind, 5, first, ("dirty 1", kind))
        second = WBG.content_for(kind, 5, n, wins, [0x00F0], rng, rig)
        _, got = run_region(lib, rig, kind, 5, second, ("dirty 2", kind))
        assert list(got.values()) == [4], (kind, got)


# ------------------------------------------------------------------------------------ B. product calls
def product(lib, call: str, env: dict, drills: dict, nbytes: int = 0, many: bool = False):
    """One product call ("zero", "tagged", "census0", "census1") on device 0, through the fan-out when `many`.  Returns
    (rc, result, tag, residue report, dirt report, mismatch report, {book: page entries})."""
    with PGC.knobs(env):
        for k in DRILL_KEYS:
            assert lib.ccm_sim_set(0, k.encode(), int(drills.get(k, 0))) == 0
        try:
            res, rr = N.ScrubResult(), N.ResidueReport()
            tag = N.TagResult() if call in ("tagged", "census1") else None
            tag_p = C.byref(tag) if tag is not None else None
            devs, wall = (C.c_int * 1)(0), C.c_double()
            if call.startswith("census") and many:
                rc = lib.ccm_scrub_verify_many_residue(1, devs, nbytes, tag_p, C.byref(rr), C.byref(res), C.byref(wall))
            elif call.startswith("census"):
                rc = lib.ccm_scrub_verify_residue(0, nbytes, tag_p, C.byref(rr), C.byref(res))
            elif tag is not None and many:
                rc = lib.ccm_scrub_verify_many_tagged(1, devs, nbytes, tag_p, C.byref(res), C.byref(wall))
            elif tag is not None:
                rc = lib.ccm_scrub_verify_tagged(0, nbytes, tag_p, C.byref(res))
            elif many:
                rc = lib.ccm_scrub_verify_many(1, devs, nbytes, C.byref(res), C.byref(wall))
            else:
                rc = lib.ccm_scrub_verify(0, nbytes, C.byref(res))
        finally:
            for k in DRILL_KEYS:
                lib.ccm_sim_set(0, k.encode(), 0)
    d, m = N.DirtReport(), N.MismatchReport()
    assert lib.ccm_scrub_last_dirt(0, C.byref(d)) == 0 and lib.ccm_scrub_last_mismatch(0, C.byref(m)) == 0
    maps = {b: page_entries(b) for b in (N.BOOK_DIRT, N.BOOK_MISMATCH, N.BOOK_RESIDUE)}
    PGC.release_wait(lib)
    return (rc, res, tag, D.ResidueReport.from_native(rr), D.DirtReport.from_native(d),
            D.MismatchReport.from_native(m), maps)


def layout(env: dict, res, nbytes: int, many: bool):
    """(chunks, enqueued ranges) of the call: VMM chunks (one handle each) or fallback segments."""
    if env.get("CCM_PIPELINE") == "0":
        segs = PP.arena_segments(nbytes, res.device_free_before, env)
        return segs, segs
    p = PP.plan(nbytes, res.device_free_before, PP.H100_GRAN, env)     # one device: the fan-out maps as one call does
    run = PP.simulate(p, res.bytes_scrubbed if nbytes == 0 else None)
    assert run.mapped == res.bytes_scrubbed and len(run.chunks) == res.segments
    return run.chunks, run.ranges(p)


def chunk_of(chunks, o: int) -> int:
    return max(i for i, (co, _) in enumerate(chunks) if co <= o)


def predicted(chunks, offsets=None, full=False) -> list:
    """(page, bytes, chunk) entries: one byte at each of `offsets`, or (full) every mapped byte."""
    pages: dict = {}
    if full:
        total = sum(n for _, n in chunks)
        for p in range(-(-total // PAGE)):
            pages[p] = min(PAGE, total - p * PAGE)
    for o in offsets or ():
        pages[o // PAGE] = pages.get(o // PAGE, 0) + 1
    return PO.entries(pages, lambda o: chunk_of(chunks, o))


DRILL_CALLS = {                       # drill -> (call, sim drills, book of the report it fills)
    "scrub_inject": ("zero", {"scrub_inject": 1000}, N.BOOK_DIRT),
    "scrub_flood": ("zero", {"scrub_flood": PP.FLOOD}, N.BOOK_DIRT),
    "tag_inject": ("tagged", {"tag_inject": 1000}, N.BOOK_MISMATCH),
    "scrub_residue": ("census0", {"scrub_residue": 1000}, N.BOOK_RESIDUE),
    "scrub_poison": ("census1", {"scrub_poison": PP.POISON}, N.BOOK_RESIDUE),
}


def check_product(lib, drill: str, env: dict, nbytes: int = 0, many: bool = False):
    call, drills, _ = DRILL_CALLS[drill]
    return assert_product(drill, env, nbytes, many, product(lib, call, env, drills, nbytes, many))


def assert_product(drill: str, env: dict, nbytes: int, many: bool, out):
    """What one product() call under `drill` left: its report and page maps against product_plan."""
    _, _, book = DRILL_CALLS[drill]
    rc, res, tag, rr, dirt, mm, maps = out
    what = (drill, env, nbytes, many)
    chunks, ranges = layout(env, res, nbytes, many)
    if drill == "scrub_inject":
        want, rep = predicted(chunks, PP.inject_offsets(ranges, 1000)), dirt
    elif drill == "scrub_flood":
        want, rep = predicted(chunks, full=True), dirt
    elif drill == "tag_inject":
        want, rep = predicted(chunks, PP.inject_offsets(ranges, 1000)), mm
    elif drill == "scrub_residue":
        want, rep = predicted(chunks, PP.inject_offsets(chunks, 1000)), rr
    else:
        want, rep = predicted(chunks, full=True), rr
    assert rep.located, (what, rc)
    assert maps[book] == want, what
    pages = {p: b for p, b, _ in maps[book]}
    assert_report_invariants(rep, pages, what)
    by_chunk = D.PageMap(maps[book]).by_chunk()
    assert by_chunk == D.PageMap(want).by_chunk(), what
    for other in {N.BOOK_DIRT, N.BOOK_MISMATCH} - {book}:
        assert maps[other] == [], (what, other)         # the call's other report is clean: an empty map
    # the report as the device object hands it out carries the digest of the same map
    digest = D.PageMap(maps[book]).digest()
    assert digest.bytes == getattr(rep, count_of(rep)) and digest.pages == len(want)
    return rep


@pytest.mark.parametrize("mf,il", PP.MODES)
@pytest.mark.parametrize("drill", list(DRILL_CALLS))
def test_product_call_pages_at_whole_hbm(lib, drill, mf, il):
    check_product(lib, drill, PP.mode_env(mf, il))


@pytest.mark.parametrize("drill", list(DRILL_CALLS))
def test_product_call_pages_on_the_fallback(lib, drill):
    """Whole HBM in one cudaMalloc, then 64 MiB in 3 MiB segments: pages that span two segments carry the chunk of
    their first byte."""
    check_product(lib, drill, {"CCM_PIPELINE": "0"})
    check_product(lib, drill, {"CCM_PIPELINE": "0", "CCM_ARENA_MAX_SEGMENT_MB": "3"}, nbytes=64 * MiB)


@pytest.mark.parametrize("drill", ["scrub_inject", "scrub_flood", "tag_inject", "scrub_residue"])
def test_product_call_pages_through_the_fan_out(lib, drill):
    check_product(lib, drill, {}, many=True)
    check_product(lib, drill, {"CCM_MAP_FIRST": "1"}, many=True)   # as the fan-out maps several devices


@pytest.mark.parametrize("mf", [0, 1])
def test_scrub_alias_pages(lib, mf):
    """Two views of one physical range: the pages lie in the first chunk's offsets or the aliased view's, and every
    page carries the chunk its records carry."""
    assert_alias(mf, product(lib, "tagged", {"CCM_MAP_FIRST": str(mf)}, {"scrub_alias": 1}, nbytes=4 * GiB))


def assert_alias(mf: int, out):
    rc, res, tag, rr, dirt, mm, maps = out
    assert rc == N.ERR_MISMATCH and mm.located
    pages = {p: b for p, b, _ in maps[N.BOOK_MISMATCH]}
    assert_report_invariants(mm, pages, ("alias", mf))
    chunk = {p: c for p, _, c in maps[N.BOOK_MISMATCH]}
    assert all(p < 2 * GiB // PAGE for p in pages), sorted(pages)[-3:]      # the first chunk (1 GiB) and its view
    assert all(c == 0 for c in chunk.values())
    for r in mm.records:
        assert chunk[r.offset // PAGE] == r.chunk, r


def test_clean_product_call_after_a_dirty_one(lib):
    """A clean call after a dirty one: empty maps, and the launches of a clean call after a clean one."""
    env = {"CCM_MAP_FIRST": "0"}
    product(lib, "zero", env, {}, 4 * GiB)
    l0 = lib.ccm_kernel_launches()
    product(lib, "zero", env, {}, 4 * GiB)
    clean = lib.ccm_kernel_launches() - l0
    check_product(lib, "scrub_inject", env, nbytes=4 * GiB)
    l0 = lib.ccm_kernel_launches()
    rc, res, _, _, dirt, mm, maps = product(lib, "zero", env, {}, 4 * GiB)
    assert rc == 0 and lib.ccm_kernel_launches() - l0 == clean
    assert maps[N.BOOK_DIRT] == [] and maps[N.BOOK_MISMATCH] == [] and not dirt.located
    # the device object attaches no pages to a clean report, and the digest of a dirty one
    gpu = next(g for g in D.find_gpus()[0] if g.is_gpu() and g.cuda_ordinal == 0)
    with PGC.knobs(env):
        lib.ccm_sim_set(gpu.index, b"scrub_inject", 5)
        try:
            with pytest.raises(D.GpuError) as ei:
                gpu.scrub_and_verify(4 * GiB)
        finally:
            lib.ccm_sim_set(gpu.index, b"scrub_inject", 0)
    PGC.release_wait(lib)
    assert ei.value.dirt.pages is not None and ei.value.dirt.pages.bytes == ei.value.dirt.nonzero_bytes == 5
    rep = gpu.scrub_and_verify(4 * GiB, residue=True)
    PGC.release_wait(lib)
    assert rep.dirt is None and (rep.residue.pages is None) == (rep.residue.residue_windows == 0)
    assert rep.residue.pages is None or rep.residue.pages.bytes == rep.residue.residue_bytes
