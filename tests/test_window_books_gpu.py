"""The window books on one H100: the locate pass, the tag check and both censuses against the numpy oracles at every
placement of tests/window_book_cases.py, with every 16-bit mask on every place they book from, at the 64-record limit
(in single launches and in product calls on the pipelined and the fallback path), and across a seeded sequence of
region passes and product calls on one engine, with the census error path in it.  The placement matrix, every mask
and the head and tail windows run each pass once more armed (include/ccm.h: ccm_region_prove): the proving twin must
book, map and write exactly what the plain kernel did, and count every byte of the region on its page of a cover map
whose page boundaries cut the region (tests/report_cover_oracle.py: map_base)."""
from __future__ import annotations

import contextlib
import ctypes as C
import sys
from dataclasses import dataclass
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "oracle"))
import dirt_oracle as DO  # noqa: E402
import mismatch_oracle as MO  # noqa: E402
import product_gate_calls as PGC  # noqa: E402
import product_plan as PP  # noqa: E402
import region_cover_calls as RCC  # noqa: E402
import scrub_cases as CASES  # noqa: E402
import tag_oracle as TO  # noqa: E402
import window_book_cases as WB  # noqa: E402
from k8s_cc_manager_b200 import _native as N  # noqa: E402
from k8s_cc_manager_b200 import devices as D  # noqa: E402

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

GiB, MiB, KiB = 1 << 30, 1 << 20, 1 << 10
GUARD = 4 * KiB
GUARD_BYTE = 0xEE
SEED = 0x7A61B00C
DRILL_KEYS = PP.DRILL_KEYS + ("tag_inject", "scrub_alias", "scrub_residue")
PASSES = ("locate", "check", "census0", "census1")
PAGE_BOOK = {"locate": N.BOOK_DIRT, "check": N.BOOK_MISMATCH, "census0": N.BOOK_RESIDUE, "census1": N.BOOK_RESIDUE}
ARMED_RUNS = {}           # test -> armed passes it ran


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


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


# ------------------------------------------------------------------------------------ one book, as compared
@dataclass
class Book:
    count: int            # locate: non-zero bytes; check: mismatched bytes; census: residue bytes
    windows: int
    first: int | None
    last: int | None
    truncated: bool
    records: list         # tuples, ascending
    zero_windows: int = 0


def book_of(kind: str, rep) -> Book:
    if kind == "locate":
        return Book(rep.nonzero_bytes, rep.dirty_windows, rep.first_offset, rep.last_offset, bool(rep.truncated),
                    [(r.offset, r.mask, r.bytes) for r in rep.records])
    if kind == "check":
        return Book(rep.mismatch_bytes, rep.mismatch_windows, rep.first_offset, rep.last_offset, bool(rep.truncated),
                    [(r.offset, r.mask, r.bytes, r.kind, r.source_offset) for r in rep.records], rep.zero_windows)
    return Book(rep.residue_bytes, rep.residue_windows, rep.first_offset, rep.last_offset, bool(rep.truncated),
                [(r.offset, r.mask) for r in rep.records])


def oracle(kind: str, region: np.ndarray, ptr: int, seed: int = SEED) -> Book:
    if kind == "check":
        w = MO.report(region, ptr, seed)
        return Book(w["mismatch_bytes"], w["mismatch_windows"], w["first_offset"], w["last_offset"], w["truncated"],
                    [(x["offset"], x["mask"], x["bytes"], x["kind"], x["source_offset"]) for x in w["windows"]],
                    w["zero_windows"])
    w = DO.report(region, ptr)
    recs = [(o, m, b) if kind == "locate" else (o, m) for o, m, b in w["windows"]]
    return Book(w["nonzero_bytes"], w["dirty_windows"], w["first_offset"], w["last_offset"], w["truncated"], recs)


def assert_book(got: Book, want: Book, what):
    assert (got.count, got.windows, got.zero_windows) == (want.count, want.windows, want.zero_windows), what
    if want.windows:
        assert (got.first, got.last) == (want.first, want.last), what
    else:
        assert got.records == [] and not got.truncated, what
    if not want.truncated:
        assert not got.truncated and got.records == want.records, what
    else:
        # 64 distinct windows of the oracle's, sorted (the check's kinds are compared only when the oracle classified)
        key = (lambda r: r[:3]) if want.records and want.records[0][3:4] == (None,) else (lambda r: r)
        got_k = [key(r) for r in got.records]
        assert got.truncated and len(got_k) == WB.RECORDS == len(set(got_k)) and got_k == sorted(got_k), what
        assert set(got_k) <= {key(r) for r in want.records}, what


# ------------------------------------------------------------------------------------ running one pass
class Rig:
    """One device buffer with guards; a region is placed `offset` bytes past a 128-byte boundary."""

    def __init__(self, top: int):
        self.buf = torch.empty(GUARD + 128 + top + GUARD, dtype=torch.uint8, device="cuda")
        self.lo = GUARD + (-(self.buf.data_ptr() + GUARD) % 128)     # region start at offset 0 mod 128

    def place(self, offset: int, region: np.ndarray):
        """Uploads guards + region; returns (ptr, host image of the slice, slice bounds)."""
        n = region.size
        a, b = self.lo + offset - GUARD, self.lo + offset + n + GUARD
        host = np.full(b - a, GUARD_BYTE, dtype=np.uint8)
        host[GUARD:GUARD + n] = region
        self.buf[a:b].copy_(torch.from_numpy(host))
        ptr = self.buf.data_ptr() + self.lo + offset
        assert ptr % 128 == offset
        return ptr, host, (a, b)

    def read(self, bounds) -> np.ndarray:
        a, b = bounds
        return self.buf[a:b].cpu().numpy()


def locate(lib, ptr, n) -> D.DirtReport:
    d = N.DirtReport()
    assert lib.ccm_region_locate(0, C.c_void_p(ptr), n, stream(), C.byref(d)) == 0, N.last_error()
    assert d.located == 1
    return D.DirtReport.from_native(d)


def check_locate(lib, ptr, n, seed=SEED) -> D.MismatchReport:
    m = N.MismatchReport()
    assert lib.ccm_region_tag_check_locate(0, C.c_void_p(ptr), n, seed, stream(), C.byref(m)) == 0, N.last_error()
    assert m.located == 1 and m.seed == seed and m.va_base == ptr
    return D.MismatchReport.from_native(m)


def check_zero(lib, ptr, n, seed=SEED) -> int:
    mm = C.c_uint64()
    assert lib.ccm_region_tag_check_zero(0, C.c_void_p(ptr), n, seed, stream(), C.byref(mm), None) == 0
    return mm.value


def census(lib, ptr, n, tags, seed=SEED) -> D.ResidueReport:
    r = N.ResidueReport()
    assert lib.ccm_region_census(0, C.c_void_p(ptr), n, int(tags), seed, stream(), C.byref(r)) == 0, N.last_error()
    assert r.located == 1 and r.va_base == ptr and r.bytes_examined == n
    return D.ResidueReport.from_native(r)


def armed_map(lib, ptr: int, n: int, test: str) -> RCC.ArmedMap:
    """A cover map for the next armed pass of `test` over [ptr, ptr + n); counts the pass."""
    ARMED_RUNS[test] = ARMED_RUNS.get(test, 0) + 1
    return RCC.ArmedMap(lib, ptr, n, sum(ARMED_RUNS.values()))


def run_pass(lib, rig: Rig, kind: str, offset: int, region: np.ndarray, what, seed=SEED, zero_too=True,
             armed: str | None = None) -> Book:
    """Runs one pass over `region` placed at `offset`, compares its book with the oracle and the slice's end state
    (guards unchanged; the region unchanged by locate, zero after the check and the zero census, the tags after the
    tagged census).  For the check, the plain check-and-zero runs on the same input as well.  armed (the test's name):
    everything once more with the proving twins, which must give the same book and page map, and cover maps of the
    region."""
    n = region.size
    books, page_maps = [], []
    for arm_it in (False, True) if armed else (False,):
        ptr, host, bounds = rig.place(offset, region)
        want = oracle(kind, region, ptr, seed)
        arm = armed_map(lib, ptr, n, armed) if arm_it else contextlib.nullcontext()
        with arm:
            if kind == "locate":
                got = book_of(kind, locate(lib, ptr, n))
            elif kind == "check":
                got = book_of(kind, check_locate(lib, ptr, n, seed))
            else:
                got = book_of(kind, census(lib, ptr, n, kind == "census1", seed))
        if arm_it:
            assert arm.take() == [arm.want([(ptr, n)])], (kind, what, "cover map", arm.base - ptr, arm.pages)
        books.append(got)
        page_maps.append(D.last_page_map(0, PAGE_BOOK[kind]).entries)
        assert_book(got, want, (kind, arm_it) + tuple(what))
        after = rig.read(bounds)
        assert np.all(after[:GUARD] == GUARD_BYTE) and np.all(after[GUARD + n:] == GUARD_BYTE), (kind, what, "guards")
        end = after[GUARD:GUARD + n]
        if kind == "locate":
            assert np.array_equal(end, region), (kind, what, "locate wrote the region")
        elif kind == "census1":
            assert np.array_equal(end, TO.tag_bytes(seed, ptr, n)), (kind, what, "not the tags")
        else:
            assert not end.any(), (kind, what, "region not zeroed")
        if kind == "check" and zero_too:
            rig.place(offset, region)
            with arm:
                assert check_zero(lib, ptr, n, seed) == want.count, (what, "check_zero")
            if arm_it:
                assert arm.take() == [arm.want([(ptr, n)])], (what, "check_zero cover map", arm.base - ptr)
            after = rig.read(bounds)
            assert not after[GUARD:GUARD + n].any() and np.all(after[:GUARD] == GUARD_BYTE), (what, "check_zero end")
            assert np.all(after[GUARD + n:] == GUARD_BYTE), (what, "check_zero guards")
    # which 64 records a truncated book keeps is not fixed: the rest of it is
    same = [(b.count, b.windows, b.first, b.last, b.truncated, b.zero_windows, None if b.truncated else b.records)
            for b in books]
    assert all(x == same[0] for x in same) and all(m == page_maps[0] for m in page_maps), (kind, what, "armed")
    return books[0]


def content_for(kind: str, offset: int, n: int, windows, masks, rng, rig: Rig, seed=SEED) -> np.ndarray:
    """Region bytes that book exactly `masks[i]` in window `windows[i]` for the pass `kind`."""
    if kind == "check":
        ptr = rig.buf.data_ptr() + rig.lo + offset
        return WB.flip_content(TO.tag_bytes(seed, ptr, n), windows, masks, rng)
    return WB.dirt_content(offset, n, windows, masks, rng)


# ------------------------------------------------------------------------------------ A. placements
def placement_content(kind, g, off, n, ptr, dense, rng, seed):
    """Structural positions (CASES), one byte in every head and tail window, and (dense) 200 more.  For the check:
    those bytes XORed, and whole windows made zero, another window's tags (alias), random bytes or one byte off
    (partial), head windows included."""
    pos = set(CASES.structural_positions(g, off, n))
    head, body, tail = CASES.split(off, n, 16)
    edge_wins = sorted({WB.window_of(off, r) for r in range(0, head)} | {WB.window_of(off, r) for r in
                                                                         range(head + body, n)})
    for w in edge_wins:
        inside = WB.window_bytes(off, n, w)
        pos.add(inside[int(rng.integers(0, len(inside)))])
    if dense and n:
        pos |= set(rng.integers(0, n, size=200).tolist())
    pos = sorted(pos)
    if kind != "check":
        region = np.zeros(n, dtype=np.uint8)
        if pos:
            region[pos] = CASES.dirt_values(pos, n * 7 + off)
        return region
    region = TO.tag_bytes(seed, ptr, n).copy()
    for p in pos:
        region[p] ^= 0x5A
    first = head % 16                                      # the first whole window in the region
    aligned = (n - first) // 16 if n >= first else 0       # whole windows: first + 16 i, i < aligned
    picks = list(edge_wins)
    if aligned:
        picks += sorted(first + 16 * int(x) for x in rng.choice(aligned, size=min(aligned, 90 if dense else 6),
                                                                 replace=False))
    for j, w in enumerate(picks):
        inside = WB.window_bytes(off, n, w)
        k = j % 4
        if k == 0:
            region[inside] = 0
        elif k == 1 and aligned > 1:
            src = first + 16 * (aligned - 1) if w != first + 16 * (aligned - 1) else first
            t = TO.tag_bytes(seed, ptr + src, 16)
            region[inside] = t[[i - w for i in inside]]
        elif k == 2:
            region[inside] = rng.integers(0, 256, len(inside))
        else:
            region[inside[0]] ^= 0x33
    return region


def test_placement_matrix(lib):
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    g = WB.geometry(sm)
    assert (g.chunk, g.grabbers) == (WB.CHUNK, sm)
    top = max(n for _, n in WB.placements(g))
    rig = Rig(top)
    rng = np.random.default_rng(17)
    seen = set()
    for off, n in WB.placements(g):
        ptr = rig.buf.data_ptr() + rig.lo + off
        for dense in (False, True):
            for kind in PASSES:
                seed = (SEED ^ (n * 131 + off)) & 0xFFFFFFFF or 1
                region = placement_content(kind, g, off, n, ptr, dense, rng, seed)
                got = run_pass(lib, rig, kind, off, region, (off, n, dense), seed, armed="placements")
                seen.add((kind, "truncated" if got.truncated else "exact"))
                if kind == "check":
                    seen |= {("kind", r[3]) for r in got.records}
        # the fill alone, plain and armed: exactly the tags, nothing outside
        for arm in (contextlib.nullcontext(), armed_map(lib, ptr, n, "placements")):
            _, _, bounds = rig.place(off, np.zeros(n, dtype=np.uint8))
            with arm:
                assert lib.ccm_region_tag_fill(0, C.c_void_p(ptr), n, SEED, stream(), None) == 0, N.last_error()
            after = rig.read(bounds)
            assert np.array_equal(after[GUARD:GUARD + n], TO.tag_bytes(SEED, ptr, n)), (off, n, "tag fill")
            assert np.all(after[:GUARD] == GUARD_BYTE) and np.all(after[GUARD + n:] == GUARD_BYTE), (off, n, "guards")
            if isinstance(arm, RCC.ArmedMap):
                assert arm.take() == [arm.want([(ptr, n)])], (off, n, "tag fill cover map", arm.base - ptr, arm.pages)
    assert {(k, s) for k in PASSES for s in ("exact", "truncated")} <= seen, sorted(seen)
    print(f"\nplacement matrix: {ARMED_RUNS['placements']} armed passes")
    assert {("kind", k) for k in ("zero", "alias", "partial", "foreign")} <= seen, sorted(seen)


def test_every_kind_in_a_head_window(lib):
    """Zero, alias, partial and foreign windows in whole and partial head windows, each alone in its region."""
    rig = Rig(4 * WB.CHUNK)
    rng = np.random.default_rng(3)
    n = 3 * WB.CHUNK + 77
    seen = set()
    for off in (1, 16, 17, 97, 112, 127):
        ptr = rig.buf.data_ptr() + rig.lo + off
        head, _, _ = CASES.split(off, n, 16)
        for w in sorted({WB.window_of(off, r) for r in range(head)}):
            inside = WB.window_bytes(off, n, w)
            for k in ("zero", "alias", "partial", "foreign"):
                region = TO.tag_bytes(SEED, ptr, n).copy()
                if k == "zero":
                    region[inside] = 0
                elif k == "alias":
                    src = head + 16 * 1000
                    region[inside] = TO.tag_bytes(SEED, ptr + src, 16)[[i - w for i in inside]]
                elif k == "partial":
                    region[inside[-1]] ^= 0x81
                else:
                    region[inside] = TO.tag_bytes(SEED ^ 0x01010101, ptr, n)[inside]
                got = run_pass(lib, rig, "check", off, region, (off, w, k), zero_too=False)
                assert [r[0] for r in got.records] == [w]
                seen.add((len(inside) == 16, got.records[0][3]))
    assert {(whole, k) for whole in (True, False) for k in ("zero", "alias", "partial", "foreign")} <= seen, seen


# ------------------------------------------------------------------------------------ B. every mask
def mask_layout(path: str, i: int):
    """(offset, n, 64 windows) on the batch path (vector u = 0 on even calls, u = 15 on odd ones) or the
    leftover-vector path."""
    if path == "batch":
        lay = WB.batch_layout(64, 0 if i % 2 == 0 else WB.PER_THREAD - 1)
    else:
        lay = WB.leftover_layout(64)
    return lay.offset, lay.n, list(lay.windows)


@pytest.mark.parametrize("kind", PASSES)
@pytest.mark.parametrize("path", ["batch", "leftover"])
def test_every_mask(lib, kind, path):
    masks = WB.all_masks()
    rig = Rig(4 * WB.CHUNK + 4096)
    rng = np.random.default_rng(2 * PASSES.index(kind) + (path == "batch"))
    for i in range(0, len(masks), 64):
        ms = masks[i:i + 64]
        off, n, wins = mask_layout(path, i // 64)
        wins = wins[:len(ms)]
        region = content_for(kind, off, n, wins, ms, rng, rig=rig)
        got = run_pass(lib, rig, kind, off, region, (path, i), zero_too=False, armed=f"mask {kind} {path}")
        assert not got.truncated and [(r[0], r[1]) for r in got.records] == list(zip(wins, ms)), (kind, path, i)
    print(f"\nevery mask, {kind} on the {path} path: {ARMED_RUNS[f'mask {kind} {path}']} armed passes")


@pytest.mark.parametrize("kind", PASSES)
def test_every_edge_mask_in_head_and_tail_windows(lib, kind):
    """Offset 16: seven whole head windows, and a tail window of 15 bytes."""
    masks = WB.edge_masks()
    n = 112 + WB.CHUNK + 48 + 15
    heads, tail = [16 * k for k in range(7)], n - 15
    rig = Rig(n)
    rng = np.random.default_rng(29)
    for i in range(0, len(masks), 7):
        ms = masks[i:i + 7]
        tm = masks[(i // 7 * 5) % len(masks)] & 0x7FFF or 0x4000
        wins, all_ms = heads[:len(ms)] + [tail], ms + [tm]
        region = content_for(kind, 16, n, wins, all_ms, rng, rig=rig)
        got = run_pass(lib, rig, kind, 16, region, ("head/tail", i), zero_too=False, armed=f"head/tail {kind}")
        assert [(r[0], r[1]) for r in got.records] == list(zip(wins, all_ms)), (kind, i)
    print(f"\nhead and tail windows, {kind}: {ARMED_RUNS[f'head/tail {kind}']} armed passes")


@pytest.mark.parametrize("kind", PASSES)
def test_first_and_last_byte_of_a_batch(lib, kind):
    """A thread's batch booked only at u = 15, or at u = 0 and u = 15: every byte position of the first and the last
    booked byte, on the first and the last thread of a chunk."""
    rig = Rig(2 * WB.CHUNK)
    rng = np.random.default_rng(31)
    n = 2 * WB.CHUNK + 48
    for t in (0, WB.THREADS - 1):
        for c in (0, 1):
            w0 = c * WB.CHUNK + t * 16
            w15 = w0 + (WB.PER_THREAD - 1) * WB.STRIDE
            for b in range(16):
                for wins, ms in (([w15], [1 << b]), ([w0, w15], [1 << b, 1 << (15 - b)]),
                                 ([w0, w15], [1 << 15, 1 << 0])):
                    region = content_for(kind, 0, n, wins, ms, rng, rig=rig)
                    got = run_pass(lib, rig, kind, 0, region, (t, c, b, ms), zero_too=False)
                    first = wins[0] + (ms[0] & -ms[0]).bit_length() - 1
                    last = wins[-1] + ms[-1].bit_length() - 1
                    assert (got.first, got.last) == (first, last), (kind, t, c, b, ms)


# ------------------------------------------------------------------------------------ C. the record limit
@pytest.mark.parametrize("kind", PASSES)
@pytest.mark.parametrize("w", WB.LIMIT_COUNTS)
def test_record_limit(lib, kind, w):
    rng = np.random.default_rng(w * 7 + PASSES.index(kind))
    rig = Rig(max(lay.n for lay in WB.limit_layouts(w)))
    for lay in WB.limit_layouts(w):
        masks = [int(rng.integers(1, 1 << 16)) & WB.in_region_mask(lay.n, x) or WB.in_region_mask(lay.n, x)
                 for x in lay.windows]
        region = content_for(kind, lay.offset, lay.n, lay.windows, masks, rng, rig=rig)
        got = run_pass(lib, rig, kind, lay.offset, region, (lay.name, w))
        assert got.windows == w and got.truncated == (w > WB.RECORDS), (kind, lay.name)
        assert len(got.records) == min(w, WB.RECORDS), (kind, lay.name)
        if w <= WB.RECORDS:
            assert [(r[0], r[1]) for r in got.records] == list(zip(lay.windows, masks)), (kind, lay.name)


# -------------------------------------------------------------------- product calls at the limit
PIPELINED = {"CCM_MAP_FIRST": "0", "CCM_VMM_FIRST_CHUNK_MB": "2", "CCM_VMM_CHUNK_MB": "2"}
FALLBACK = {"CCM_PIPELINE": "0", "CCM_ARENA_MAX_SEGMENT_MB": "2"}
PRODUCT_BYTES = 64 * MiB


def product(lib, call: str, nbytes=PRODUCT_BYTES, env=None, drills=None):
    """call: "zero", "tagged", "census0" or "census1".  Returns (rc, result, tag, residue, dirt, mismatch); after a
    failed call, product.error holds the library's message."""
    drills = drills or {}
    with PGC.knobs(env or {}):
        for k in DRILL_KEYS:
            assert lib.ccm_sim_set(0, k.encode(), int(drills.get(k, 0))) == 0
        try:
            res, rr = N.ScrubResult(), N.ResidueReport()
            tag = N.TagResult() if call in ("tagged", "census1") else None
            tag_p = C.byref(tag) if tag is not None else None
            if call.startswith("census"):
                rc = lib.ccm_scrub_verify_residue(0, nbytes, tag_p, C.byref(rr), C.byref(res))
            elif tag is not None:
                rc = lib.ccm_scrub_verify_tagged(0, nbytes, tag_p, C.byref(res))
            else:
                rc = lib.ccm_scrub_verify(0, nbytes, C.byref(res))
            product.error = N.last_error() if rc else ""
        finally:
            for k in DRILL_KEYS:
                lib.ccm_sim_set(0, k.encode(), 0)
    d, m = N.DirtReport(), N.MismatchReport()
    assert lib.ccm_scrub_last_dirt(0, C.byref(d)) == 0 and lib.ccm_scrub_last_mismatch(0, C.byref(m)) == 0
    PGC.release_wait(lib)
    return (rc, res, tag, D.ResidueReport.from_native(rr), D.DirtReport.from_native(d),
            D.MismatchReport.from_native(m))


def mappings(env, res):
    """The product call's chunks (pipelined) or segments (fallback), (offset, bytes) in order."""
    if env.get("CCM_PIPELINE") == "0":
        return PP.arena_segments(PRODUCT_BYTES, res.device_free_before, env)
    return PP.simulate(PP.plan(PRODUCT_BYTES, res.device_free_before, PP.H100_GRAN, env), None).chunks


def chunk_at(chunks, o):
    return [i for i, (co, cn) in enumerate(chunks) if co <= o < co + cn]


def assert_single_byte_book(recs, offs, chunks, truncated_rule, what):
    """Records of one single-byte window per drilled byte: exactly all of them (k <= 64), else 64 distinct sorted
    ones of them; `truncated_rule` "first" pins the first 64 in mapping order."""
    want = [(o // 16 * 16, 1 << (o % 16)) for o in sorted(offs)]
    got = [(r.offset, r.mask) for r in recs]
    for r in recs:
        assert chunk_at(chunks, r.offset + r.mask.bit_length() - 1) == [r.chunk], (what, r)
    if len(offs) <= WB.RECORDS:
        assert got == want, what
    else:
        assert len(got) == WB.RECORDS == len(set(got)) and got == sorted(got) and set(got) <= set(want), what
        if truncated_rule == "first":
            assert got == want[:WB.RECORDS], what


def check_product_drill(lib, env, drill, k):
    """One product call with `drill` spending k bytes; its report against product_plan."""
    call, drills = {"residue0": ("census0", {"scrub_residue": k}), "residue1": ("census1", {"scrub_residue": k}),
                    "inject": ("zero", {"scrub_inject": k}), "tag_inject": ("tagged", {"tag_inject": k})}[drill]
    rc, res, tag, rr, dirt, mm = product(lib, call, env=env, drills=drills)
    chunks = mappings(env, res)
    assert res.segments == len(chunks) == 32, (env, drill)
    offs = PP.inject_offsets(chunks, k)
    assert len(offs) == k
    what = (env, drill, k)
    if drill.startswith("residue"):
        assert rc == 0 and res.nonzero_bytes == 0 and not dirt.located and not mm.located, what
        assert rr.located and rr.residue_bytes == rr.residue_windows == k and rr.truncated == (k > WB.RECORDS), what
        assert (rr.first_offset, rr.last_offset) == (min(offs), max(offs)), what
        assert_single_byte_book(rr.records, offs, chunks, None, what)
    elif drill == "inject":
        assert rc == N.ERR_DIRTY and res.nonzero_bytes == k and not mm.located, what
        assert dirt.located and dirt.nonzero_bytes == dirt.dirty_windows == k, what
        assert dirt.truncated == (k > WB.RECORDS) and (dirt.first_offset, dirt.last_offset) == (min(offs), max(offs))
        # The fallback locates segment by segment and keeps records while the report has room: the first 64 windows
        # in segment order.  The pipelined call locates its one mapping in one launch: any 64.
        rule = "first" if env is FALLBACK else None
        assert_single_byte_book(dirt.records, offs, chunks, rule, what)
        for r in dirt.records:
            o = r.offset + r.mask.bit_length() - 1
            assert bytes.fromhex(r.bytes) == bytes(0xA5 if i == o % 16 else 0 for i in range(16)), (what, r)
    else:
        assert rc == N.ERR_MISMATCH and tag.mismatch_bytes == k and not dirt.located, what
        assert mm.located and mm.mismatch_bytes == mm.mismatch_windows == k and mm.zero_windows == 0, what
        assert mm.truncated == (k > WB.RECORDS) and (mm.first_offset, mm.last_offset) == (min(offs), max(offs)), what
        assert all(r.kind == "partial" for r in mm.records), what
        assert_single_byte_book(mm.records, offs, chunks, None, what)
        if env is PIPELINED:                               # one contiguous mapping: the window is at va_base + offset
            for r in mm.records:
                o = r.offset + r.mask.bit_length() - 1
                t = TO.tag_bytes(tag.seed, tag.va_base + r.offset, 16)
                assert bytes.fromhex(r.bytes) == bytes(t[i] ^ (0xA5 if i == o % 16 else 0) for i in range(16)), what
    return rc


@pytest.mark.parametrize("env", [PIPELINED, FALLBACK], ids=["pipelined", "fallback"])
@pytest.mark.parametrize("drill", ["residue0", "residue1", "inject", "tag_inject"])
def test_record_limit_in_product_calls(lib, env, drill):
    for k in (63, 64, 65):
        check_product_drill(lib, env, drill, k)


# ------------------------------------------------------------------------------------ D. back to back
def region_windows_content(kind, off, n, count, rng, rig, seed=SEED):
    """Region content for the sequence: empty, sparse, exactly 64 / 65 windows, or flooded."""
    if count == "flood":
        wins = sorted({WB.window_of(off, r) for r in range(0, n, 16)} | {WB.window_of(off, n - 1)})
        ms = [0xFFFF] * len(wins)
    else:
        k = {"empty": 0, "sparse": 5, "64": 64, "65": 65}[count]
        first = WB.window_of(off, 0) % 16                   # the first whole window in the region
        wins = sorted(first + 16 * int(x) for x in rng.choice((n - first) // 16, size=k, replace=False))
        ms = [int(rng.integers(1, 1 << 16)) for _ in wins]
    return content_for(kind, off, n, wins, ms, rng, rig=rig, seed=seed)


def test_back_to_back_calls_on_one_engine(lib):
    rng = np.random.default_rng(2024)
    off, n = 33, 3 * WB.CHUNK + 100
    rig = Rig(n)
    region_kinds = ("locate", "check", "check_zero", "census0", "census1")
    contents = ("empty", "sparse", "64", "65", "flood")
    products = ("clean", "inject", "tag_inject", "residue0", "residue1")
    seen = set()
    for step in range(200):
        if rng.random() < 0.7:
            kind, count = region_kinds[rng.integers(len(region_kinds))], contents[rng.integers(len(contents))]
            pk = "check" if kind == "check_zero" else kind
            region = region_windows_content(pk, off, n, count, rng, rig)
            if kind == "check_zero":
                ptr, _, bounds = rig.place(off, region)
                assert check_zero(lib, ptr, n) == TO.mismatch_count(region, SEED, ptr), (step, count)
                assert not rig.read(bounds)[GUARD:GUARD + n].any(), step
            else:
                run_pass(lib, rig, kind, off, region, (step, count), zero_too=False)
            seen.add((kind, count))
        else:
            drill = products[rng.integers(len(products))]
            if drill == "clean":
                call = ("zero", "tagged")[rng.integers(2)]
                rc, res, tag, rr, dirt, mm = product(lib, call, env=PIPELINED)
                assert rc == 0 and res.nonzero_bytes == 0 and not dirt.located and not mm.located, step
                assert dirt.records == [] and mm.records == [], step
            else:
                k = int(rng.choice([1, 5, 63, 64, 65]))
                check_product_drill(lib, PIPELINED, drill, k)
            seen.add(drill)
    assert len(seen) >= 20, sorted(map(str, seen))


def test_census_error_leaves_an_empty_book(lib):
    """A census call that runs out of memory after it has censused earlier mappings (a request larger than what
    cudaMemGetInfo reports free) fails with CCM_ERR_NOMEM; the next region census and the next product census report
    exactly their own residue."""
    rig = Rig(2 * WB.CHUNK)
    rng = np.random.default_rng(5)
    n = 2 * WB.CHUNK - 3
    for call in ("census0", "census1"):
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        free, _ = torch.cuda.mem_get_info()
        rc, res, _, _, _, _ = product(lib, call, nbytes=free + 2 * GiB, env={"CCM_MAP_FIRST": "0"},
                                      drills={"scrub_residue": 1000})
        # the pipelined path ran out creating a mapping, after it had mapped and censused earlier ones
        assert rc == N.ERR_NOMEM and "cuMemCreate" in product.error, (call, rc, product.error)
        kind = call
        region = region_windows_content(kind, 5, n, "sparse", rng, rig)
        run_pass(lib, rig, kind, 5, region, (call, "after the error"))
        check_product_drill(lib, PIPELINED, "residue0" if call == "census0" else "residue1", 5)
