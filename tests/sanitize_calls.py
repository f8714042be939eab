"""A small, complete set of calls that launches every kernel entry of libccm.so, with every result checked exactly
against the oracles while it runs: a child process for tests/test_sanitizers_gpu.py, which runs it under each
compute-sanitizer tool (memcheck, racecheck, synccheck, initcheck) and once under torch.profiler to see that every
entry launched.  A tool perturbs timing and scheduling, so every count, book, page map, cover map and probe report must
still be exact.

  region    caller-owned regions, each flush against the END of its own cudaMalloc allocation (the region starts
            `offset` bytes past a 128-byte boundary, and nothing of the allocation lies past its last byte), then, in a
            second call, at the START of its own allocation.  The byte past the end belongs to no allocation, so
            memcheck sees any read or write there.  Below the start it does so only at the aligned starts of the
            second call: cudaMalloc returns aligned addresses, so a region that starts `offset` bytes past a 128-byte
            boundary keeps those bytes inside its allocation, and there only a write is seen (they must still hold
            FILL afterwards).  main() sets PYTORCH_NO_CUDA_MEMORY_CACHING=1 in this process before it loads torch, so
            every tensor is its own cudaMalloc of exactly its size; a caching allocator would hide an overrun inside
            its pool block.  Importing this module changes no environment.  Every byte a call reads is written first.
              * one launch shape of tests/scrub_cases.py per generic scrub / verify instantiation (generic_cases), at a
                misaligned start and lengths at its tiling edges: 0, 1, one short of a tile, a whole tile and one
                grab per grabber plus one byte;
              * the default-frame kernels (default scrub and verifier, tag fill, tag check, locate, both censuses),
                plain and armed (include/ccm.h: ccm_region_prove), where their proving twins run, at PLACEMENTS: head
                windows only, leftover vectors, a grab cut by a page boundary, 65 booked windows (one past the record
                limit) and a length at which every grabber takes two grabs (scrub_cases.big_length);
              * ccm_region_probe, plain and armed, at ragged lengths;
              * every byte value at each byte position of a word (all_byte_values), at a 128-byte boundary and one
                byte past it, through every generic verifier and the default verifier, locate, tag check and both
                censuses (unarmed: the cover maps do not depend on the bytes);
              * the arena: byte fill (0xA5, then 0x00), seeded pattern fill, default scrub and verify.
  product   product gate calls of a few 2 MiB chunks (PRODUCT_CALLS), each compared with the composed model
            (tests/gate_model.py): clean, inject (xor_byte_kernel), tagged, census, proven, probed (clean, and with
            the probe's mismatch and dirt drills), both triages on a dirty call, map-first and the cudaMalloc fallback.
            They read what earlier tenants left, by design, so initcheck runs the region phase only.

Run as `sanitize_calls.py --phase region|product|all [--kernels]`: it ends with ccm_device_release and prints one
`RESULT <json>` line with the calls run, the first mismatch (null when every result was exact), the number of results
that were not exact and the labels of their calls (`mismatches`, `failed`: tests/test_kernel_mutants.py reads which
checks a deliberately broken kernel fails).  An exception inside one call is that call's mismatch and the run goes on; a
call that returns CCM_ERR_CUDA or leaves a sticky CUDA error stops it, and RESULT says `"fault": true`.  With --kernels
the run is profiled and a `KERNELS <json>` line lists every kernel the process launched.  ENTRIES maps every kernel
entry to the part of the run that launches it; tests/test_sanitizers_gpu.py checks on the CPU that it names every entry
of the registry.  Not collected by pytest.
"""
from __future__ import annotations

import argparse
import contextlib
import ctypes as C
import json
import os
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
for p in (ROOT, ROOT / "tests", ROOT / "oracle"):
    if str(p) not in sys.path:
        sys.path.insert(0, str(p))

import numpy as np  # noqa: E402

import scrub_cases as SC  # noqa: E402
import window_book_cases as WB  # noqa: E402

MiB = 1 << 20
PAGE = 2 * MiB
FILL = 0xEE                          # what the bytes of an allocation outside its region hold
SEED = 0x5A17C0DE
FAST = ("scrub_st128_fast_kernel<512, 16, 0>", "verify_ld128_fast_kernel<1024, 8, 2>")   # ccm_default_kernels()


# ------------------------------------------------------------------------------------ the case table
def generic_cases() -> dict:
    """Generic instantiation -> the first launch shape of tests/scrub_cases.py that launches it (memset launches none)."""
    out = {}
    for case in SC.all_cases():
        name = SC.instantiation(case, FAST)
        if name is not None and not SC.is_fast(case):
            out.setdefault(name, case)
    return out


def schedule_cases() -> list:
    """(instantiation, case): the first generic launch shape of each kind, variant and schedule (static, per-CTA grabs,
    per-warp grabs) that generic_cases() does not already launch.  The schedule is a launch argument, not a template
    one, so one shape per instantiation would leave the others' loops (for_each_tile) unrun."""
    chosen = {id(c) for c in generic_cases().values()}
    seen = {(c.kind, c.variant, c.cfg[5]) for c in generic_cases().values()}
    out = []
    for case in SC.all_cases():
        name = SC.instantiation(case, FAST)
        key = (case.kind, case.variant, case.cfg[5] if case.cfg else None)
        if name is None or SC.is_fast(case) or id(case) in chosen or key in seen:
            continue
        seen.add(key)
        out.append((name, case))
    return out


# kernel entry (name<template arguments>) -> the part of this run that launches it
ENTRIES = {name: "generic" for name in generic_cases()}
ENTRIES.update({
    FAST[0]: "region scrub",
    FAST[1]: "region verify",
    "cover_zero_pass<512, 16, 0>": "region scrub, armed",
    "cover_read_pass<1024, 8, 2>": "region verify, armed",
    "tag_fill_kernel<512, 16>": "region fill",
    "cover_tag_fill_pass<512, 16>": "region fill, armed",
    "tag_check_zero_kernel<512, 16>": "region check",
    "cover_tag_check_pass<512, 16>": "region check, armed",
    "locate_dirt_kernel<512, 16>": "region locate",
    "cover_locate_pass<512, 16>": "region locate, armed",
    "census_zero_kernel<512, 16>": "region census0",
    "cover_census_zero_pass<512, 16>": "region census0, armed",
    "census_tag_fill_kernel<512, 16>": "region census1",
    "cover_census_tag_pass<512, 16>": "region census1, armed",
    "alias_probe_fill_pass<256, 4>": "region probe",
    "alias_probe_check_pass<256, 4>": "region probe",
    "alias_probe_reread_pass<256, 4>": "region probe",
    "cover_probe_fill_pass<256, 4>": "region probe, armed",
    "cover_probe_check_pass<256, 4>": "region probe, armed",
    "cover_probe_reread_pass<256, 4>": "region probe, armed",
    "fill_byte_kernel": "arena fill",
    "fill_pattern_kernel": "arena pattern",
    "xor_byte_kernel": "product inject",
})

BOOK_KINDS = ("scrub", "verify", "fill", "check", "locate", "census0", "census1")


def placements(g: SC.Geometry) -> list:
    """(name, offset, length) of the default-frame kernels' regions (g: their geometry at this SM count)."""
    return [("head windows", 17, 40),
            ("leftover vectors", 16, 112 + 3 * 16 + 5),
            ("page-cut grab", 17, 2 * PAGE + 3 * WB.CHUNK + 77),
            ("65 windows", WB.mixed_layout(65).offset, WB.mixed_layout(65).n),
            ("two grabs each", 1, SC.big_length(g)),
            ("64 windows in warp rounds", 0, WB.CHUNK)]


# 64 windows that warp 0 of the CTA holding the region's one chunk books in three rounds of its lanes (thread t takes
# vector u * THREADS + t in round u): 31, then 32, then 1.  The 64th record slot is claimed after the 63rd was, so a
# book that marks itself full one slot early keeps 63 records.
WARP_ROUNDS = [16 * t for t in range(31)] + [16 * (WB.THREADS + t) for t in range(32)] + [16 * 2 * WB.THREADS]


def word3_windows(content: np.ndarray, ptr: int) -> np.ndarray:
    """content with every seventh address window from the fourth on made 0 in its first 12 bytes and 0x5A in its last
    4: windows that hold a non-zero byte only in their last word."""
    starts = np.arange((-ptr) % 16 + 48, content.size - 15, 112)
    content[starts[:, None] + np.arange(12)] = 0
    content[starts[:, None] + np.arange(12, 16)] = 0x5A
    return content


# Every byte value at each of the four byte positions of a word: byte i of each 1024 is (i // 4 + 64 * (i % 4)) % 256.
# One grab of the default-frame kernels (128 KiB), leftover vectors and a ragged tail; placed at a 128-byte boundary
# and one byte past it (127 head bytes), so the chunk, vector and byte paths all read 0x01 and 0x80.
ALL_BYTES_LENGTH = 128 * 1024 + 4096 + 13
ALL_BYTES_KINDS = ("verify", "check", "locate", "census0", "census1")


def all_byte_values(n: int) -> np.ndarray:
    i = np.arange(n)
    return ((i % 1024 // 4 + 64 * (i % 4)) % 256).astype(np.uint8)


def generic_lengths(g: SC.Geometry, head: int) -> list:
    """0, 1, one short of a tile, a whole tile, and a grab per grabber and one byte, after `head` ragged bytes."""
    return [0, 1, head + g.tile - 1, head + g.tile, head + g.chunk * g.grabbers + 1]


PIPELINED = {"CCM_VMM_FIRST_CHUNK_MB": "2", "CCM_VMM_CHUNK_MB": "2"}
NBYTES = 6 * MiB + 1                 # four 2 MiB chunks, the last holding one byte
PRODUCT_CALLS = [
    {"bytes": NBYTES, "kind": "zero", "env": PIPELINED},
    {"bytes": NBYTES, "kind": "zero", "env": PIPELINED, "drill": {"scrub_inject": 5}},
    {"bytes": NBYTES, "kind": "tagged", "env": PIPELINED},
    {"bytes": NBYTES, "kind": "census", "env": PIPELINED, "drill": {"scrub_residue": 9}},
    {"bytes": NBYTES, "kind": "census_tagged", "env": PIPELINED, "drill": {"scrub_residue": 4}},
    {"bytes": NBYTES, "kind": "zero", "env": PIPELINED, "prove": 1},
    {"bytes": NBYTES, "kind": "tagged", "env": PIPELINED, "prove": 1},
    {"bytes": NBYTES, "kind": "census", "env": PIPELINED, "prove": 1, "drill": {"scrub_residue": 4}},
    {"bytes": NBYTES, "kind": "census_tagged", "env": PIPELINED, "prove": 1, "drill": {"scrub_residue": 1}},
    {"bytes": NBYTES, "kind": "zero", "env": PIPELINED, "probe": 1},
    {"bytes": NBYTES, "kind": "zero", "env": PIPELINED, "probe": 1, "prove": 1},
    {"bytes": NBYTES, "kind": "zero", "env": PIPELINED, "probe": 1, "prove": 1,
     "drill": {"probe_mismatch": 3, "probe_dirt": 2}},
    {"bytes": NBYTES, "kind": "tagged", "env": PIPELINED, "triage": 2, "mismatch_triage": 2,
     "drill": {"scrub_inject": 3, "tag_inject": 4, "triage_stay": 1, "triage_return": 1}},
    {"bytes": NBYTES, "kind": "tagged", "env": PIPELINED, "prove": 1, "triage": 2, "mismatch_triage": 2,
     "drill": {"scrub_inject": 3, "tag_inject": 4}},
    {"bytes": NBYTES, "kind": "zero", "env": {"CCM_MAP_FIRST": "1"}, "drill": {"scrub_inject": 4}},
    {"bytes": 10 * MiB + 777, "kind": "zero", "env": {"CCM_PIPELINE": "0", "CCM_ARENA_MAX_SEGMENT_MB": "3"},
     "drill": {"scrub_inject": 7}},
    {"bytes": 10 * MiB + 777, "kind": "tagged", "env": {"CCM_PIPELINE": "0"}, "prove": 1, "triage": 1,
     "drill": {"scrub_inject": 2}},
]


# ------------------------------------------------------------------------------------ running them
class Fault(Exception):
    """A call returned CCM_ERR_CUDA or left a sticky CUDA error: the context is not to be trusted, so the run stops."""


class Run:
    """The calls made so far, every result that was not exact (the labels of the first MAX_FAILED, and their total) and
    the first one's detail.  `sync` (torch.cuda.synchronize) tells a sticky CUDA error from an ordinary exception."""

    MAX_FAILED = 500

    def __init__(self, sync=None):
        self.calls = 0
        self.first = None
        self.failed = []
        self.mismatches = 0
        self.sync = sync

    def check(self, ok: bool, what, *detail) -> None:
        self.calls += 1
        if ok:
            return
        self.mismatches += 1
        if self.first is None:
            self.first = {"call": [str(x) for x in what], "detail": [str(x)[:2000] for x in detail]}
        if len(self.failed) < self.MAX_FAILED:
            self.failed.append([str(x) for x in what])

    def rc(self, rc: int, what) -> None:
        """Stops the run when a call returned CCM_ERR_CUDA."""
        from k8s_cc_manager_b200 import _native as N
        if rc == N.ERR_CUDA:
            raise Fault(f"{[str(x) for x in what]} returned CCM_ERR_CUDA: {N.last_error()}")

    @contextlib.contextmanager
    def call(self, what):
        """One call: an exception inside it is that call's mismatch and the run goes on (a wrong book must not hide
        the checks after it); a CUDA error, returned or sticky, stops the run."""
        try:
            yield
        except Fault:
            raise
        except Exception as exc:  # noqa: BLE001 -- any failure of one call is that call's result
            try:
                if self.sync is not None:
                    self.sync()
            except Exception as sticky:  # noqa: BLE001
                raise Fault(f"{[str(x) for x in what]}: {sticky}") from exc
            if "CCM_ERR_CUDA" in str(exc) or "CUDA error" in str(exc):
                raise Fault(f"{[str(x) for x in what]}: {exc}") from exc
            self.check(False, what, "exception", f"{type(exc).__name__}: {exc}")


def own(torch, at: str, offset: int, n: int):
    """(buffer, region address, index of the region in the buffer): an allocation of its own whose last byte is the
    region's (at "end"; the region starts `offset` past a 128-byte boundary) or whose first byte is (at "start")."""
    lo = offset if at == "end" else 0
    buf = torch.full((lo + n,), FILL, dtype=torch.uint8, device="cuda")
    assert buf.data_ptr() % 512 == 0
    return buf, buf.data_ptr() + lo, lo


def run_generic(lib, torch, run: Run, sms: int) -> None:
    from k8s_cc_manager_b200 import _native as N
    for name, case in list(generic_cases().items()) + schedule_cases():
        g = SC.geometry(case, sms)
        kw = case.cfg_kwargs()
        cfg = C.byref(N.launch_cfg(kw["ctas_per_sm"], kw["threads"], kw["tile_bytes"], kw["unroll"], kw["cache_policy"],
                                   kw["schedule"]))
        lengths = generic_lengths(g, 111)
        for at, offset, n in [("end", 17, n) for n in lengths] + [("start", 0, lengths[-1])]:
            what = (name, case.label(), at, offset, n)
            with run.call(what):
                if case.kind == "scrub":
                    buf, ptr, lo = own(torch, at, offset, n)
                    rc = lib.ccm_region_scrub(0, C.c_void_p(ptr), n, case.variant, cfg, None, None)
                    run.rc(rc, what)
                    torch.cuda.synchronize()
                    bad = int((buf[:lo] != FILL).sum()) + int(torch.count_nonzero(buf[lo:]))
                    run.check(rc == 0 and bad == 0, what, rc, N.last_error() if rc else "", f"{bad} bytes wrong")
                else:
                    pos = SC.structural_positions(g, offset, n)
                    buf, ptr, lo = own(torch, at, offset, n)
                    buf[lo:].zero_()
                    if pos:
                        buf[torch.tensor([lo + p for p in pos], device="cuda")] = torch.tensor(
                            SC.dirt_values(pos, n + offset), dtype=torch.uint8, device="cuda")
                    nz = C.c_uint64(1 << 63)
                    rc = lib.ccm_region_verify(0, C.c_void_p(ptr), n, case.variant, cfg, None, C.byref(nz), None)
                    run.rc(rc, what)
                    run.check(rc == 0 and nz.value == len(pos), what, rc, N.last_error() if rc else "", nz.value,
                              len(pos))
                del buf
        for at, offset in (("end", 1), ("start", 0)) if case.kind != "scrub" else ():
            n = ALL_BYTES_LENGTH
            what = (name, case.label(), "all bytes", at, offset, n)
            with run.call(what):
                buf, ptr, lo = own(torch, at, offset, n)
                buf[lo:].copy_(torch.from_numpy(all_byte_values(n)))
                nz = C.c_uint64(1 << 63)
                rc = lib.ccm_region_verify(0, C.c_void_p(ptr), n, case.variant, cfg, None, C.byref(nz), None)
                run.rc(rc, what)
                want = int(np.count_nonzero(all_byte_values(n)))
                run.check(rc == 0 and nz.value == want, what, rc, N.last_error() if rc else "", nz.value, want)
                del buf


def book_content(kind: str, name: str, offset: int, n: int, ptr: int, g, rng) -> np.ndarray:
    """What a default-frame pass reads: dirt (or, for the check, the tags with bytes flipped) at the structural
    positions and in every head and tail window; 65 windows in the record-limit placement; random bytes for the scrub,
    zeros for the fill, which only writes."""
    import tag_oracle as TO
    import test_window_books_gpu as WBG
    if kind == "scrub":
        return rng.integers(1, 256, n, dtype=np.uint8)
    if kind == "fill":
        return np.zeros(n, dtype=np.uint8)
    if name in ("65 windows", "64 windows in warp rounds"):
        windows = WB.mixed_layout(65).windows if name == "65 windows" else WARP_ROUNDS
        masks = [int(rng.integers(1, 1 << 16)) & WB.in_region_mask(n, w) or WB.in_region_mask(n, w) for w in windows]
        if kind == "check":
            return WB.flip_content(TO.tag_bytes(SEED, ptr, n), windows, masks, rng)
        return WB.dirt_content(offset, n, windows, masks, rng)
    content = WBG.placement_content("locate" if kind == "verify" else kind, g, offset, n, ptr, False, rng, SEED)
    if name == "page-cut grab":
        # bytes of the chunk that straddles the first page boundary (the body starts at the region's first 128-byte
        # boundary), on the page after it
        head = (-ptr) % 128
        content[2 * PAGE + head // 2:2 * PAGE + head // 2 + 4] ^= 0x5A
    return content


def run_book_pass(lib, torch, run: Run, kind: str, what, content, at: str, offset: int, n: int, armed: int) -> None:
    """One default-frame pass over the region content(address) gives, placed in an allocation of its own, compared with
    the oracles: its count or book, its page map, the bytes it leaves (and none outside the region), and armed, its
    cover map.  The check runs twice: with its book (ccm_region_tag_check_locate), then as the plain check-and-zero."""
    buf, ptr, lo = own(torch, at, offset, n)
    region = content(ptr)
    for step in (("book", "zero") if kind == "check" else ("book",)):
        label = what + (("check_zero",) if step == "zero" else ())
        with run.call(label):
            book_step(lib, torch, run, kind, step, label, buf, ptr, lo, region, n, armed)


def book_step(lib, torch, run: Run, kind: str, step: str, label, buf, ptr: int, lo: int, region, n: int,
              armed: int) -> None:
    """One step of run_book_pass: `region` into the buffer, the pass, and every check of its results."""
    import page_oracle as PG
    import region_cover_calls as RCC
    import tag_oracle as TO
    import test_window_books_gpu as WBG
    from k8s_cc_manager_b200 import _native as N
    from k8s_cc_manager_b200 import devices as D
    buf.fill_(FILL)
    if n:
        buf[lo:].copy_(torch.from_numpy(region))
    arm = RCC.ArmedMap(lib, ptr, n, armed) if armed else None
    got, rc = None, 0
    with arm or contextlib.nullcontext():
        if kind == "scrub":
            rc = lib.ccm_region_scrub(0, C.c_void_p(ptr), n, N.SCRUB_AUTO, None, None, None)
        elif kind == "fill":
            rc = lib.ccm_region_tag_fill(0, C.c_void_p(ptr), n, SEED, None, None)
        elif kind == "verify" or step == "zero":
            nz = C.c_uint64(1 << 63)
            rc = (lib.ccm_region_verify(0, C.c_void_p(ptr), n, N.VERIFY_AUTO, None, None, C.byref(nz), None)
                  if kind == "verify" else
                  lib.ccm_region_tag_check_zero(0, C.c_void_p(ptr), n, SEED, None, C.byref(nz), None))
            got = nz.value
        elif kind == "locate":
            got = WBG.book_of("locate", WBG.locate(lib, ptr, n))
        elif kind == "check":
            got = WBG.book_of("check", WBG.check_locate(lib, ptr, n, SEED))
        else:
            got = WBG.book_of("census", WBG.census(lib, ptr, n, kind == "census1", SEED))
    run.rc(rc, label)
    torch.cuda.synchronize()
    run.check(rc == 0, label, rc, N.last_error() if rc else "")
    if kind == "verify" or step == "zero":
        want = int(np.count_nonzero(region)) if kind == "verify" else TO.mismatch_count(region, SEED, ptr)
        run.check(got == want, label, "count", got, want)
    elif got is not None:
        want = WBG.oracle(kind, region, ptr, SEED)
        try:
            WBG.assert_book(got, want, label)
            run.check(True, label)
        except AssertionError:
            run.check(False, label, "book", got, want)
        book = {"locate": N.BOOK_DIRT, "check": N.BOOK_MISMATCH}.get(kind, N.BOOK_RESIDUE)
        pages = PG.check_page_map(region, ptr, SEED) if kind == "check" else PG.page_map(region, ptr)
        got_pages, want_pages = D.last_page_map(0, book).entries, PG.entries(pages)
        run.check(got_pages == want_pages, label, "page map", got_pages, want_pages)
    after = buf.cpu().numpy()
    end = after[lo:]
    if kind in ("locate", "verify"):
        ok_end = np.array_equal(end, region)
    elif kind in ("fill", "census1"):
        ok_end = np.array_equal(end, TO.tag_bytes(SEED, ptr, n))
    else:
        ok_end = not end.any()
    run.check(ok_end and bool(np.all(after[:lo] == FILL)), label, "bytes left")
    if arm:
        maps, want_map = arm.take(), arm.want([(ptr, n)] if n else [])
        run.check(maps == [want_map], label, "cover map", maps, want_map)


def run_books(lib, torch, run: Run, sms: int) -> None:
    g = WB.geometry(sms)
    rng = np.random.default_rng(SEED)
    armed = 0
    for name, offset, n in placements(g):
        for at in ("end", "start"):
            off = offset if at == "end" else 0
            for kind in BOOK_KINDS:
                for arm in (False, True):
                    armed += arm
                    run_book_pass(lib, torch, run, kind, (kind, name, at, off, n, "armed" if arm else "plain"),
                                  lambda ptr: book_content(kind, name, off, n, ptr, g, rng), at, off, n,
                                  armed if arm else 0)
    import tag_oracle as TO
    n = ALL_BYTES_LENGTH
    for at, off in (("end", 1), ("start", 0)):
        for kind in ALL_BYTES_KINDS:
            # the check reads every value as the difference from its tag, and windows that read 0 but in their last
            # word
            content = ((lambda ptr: word3_windows(TO.tag_bytes(SEED, ptr, n) ^ all_byte_values(n), ptr))
                       if kind == "check" else (lambda ptr: all_byte_values(n)))
            run_book_pass(lib, torch, run, kind, (kind, "all bytes", at, off, n, "plain"), content, at, off, n, 0)


def run_probe(lib, torch, run: Run) -> None:
    for at, offset, n in (("end", 100, 3 * 4096 - 100 + 31), ("end", 7, 5 * 4096 + 1000), ("start", 0, 4 * MiB + 33),
                          ("start", 0, 31)):
        for armed in (False, True):
            what = ("probe", at, offset, n, "armed" if armed else "plain")
            with run.call(what):
                probe_call(lib, torch, run, what, at, offset, n, armed)


def probe_call(lib, torch, run: Run, what, at: str, offset: int, n: int, armed: bool) -> None:
    """One ccm_region_probe over a clean region: its report, the bytes it leaves and, armed, its three cover maps."""
    import probe_oracle as PO
    import region_cover_calls as RCC
    import report_cover_oracle as RO
    from k8s_cc_manager_b200 import _native as N
    buf, ptr, lo = own(torch, at, offset, n)
    w0, k = PO.chunk_windows(ptr, n)
    arm = RCC.ArmedMap(lib, ptr, n, 0, steps=3, at=(w0 + PO.STRIDE * (k // 2) + 7, 1)) if armed else None
    rep, mm = N.ProbeReport(), N.MismatchReport()
    with arm or contextlib.nullcontext():
        rc = lib.ccm_region_probe(0, C.c_void_p(ptr), n, SEED, None, C.byref(rep), C.byref(mm))
    run.rc(rc, what)
    run.check(rc == 0, what, rc, N.last_error() if rc else "")
    got = (rep.probed, rep.windows, rep.bytes_probed, rep.seed, rep.mismatch_bytes, rep.reread_nonzero_bytes,
           rep.va_base, rep.launches, mm.located, mm.mismatch_bytes)
    want = (1, k, 32 * k, SEED, 0, 0, ptr, 3 if k else 0, 1, 0)
    run.check(got == want, what, "report", got, want)
    host = buf.cpu().numpy()
    expect = np.full(host.size, FILL, dtype=np.uint8)
    for i in range(k):
        o = w0 + 4096 * i - buf.data_ptr()
        expect[o:o + 32] = 0
    run.check(np.array_equal(host, expect), what, "bytes left")
    if arm:
        maps, want_map = arm.take(), arm.want(RO.probe_parts([(ptr, n)]))
        run.check(maps == [want_map] * 3, what, "cover maps", maps, want_map)


def run_arena(lib, run: Run) -> None:
    import scrub_oracle as SO
    from k8s_cc_manager_b200 import _native as N
    nbytes = 8 * MiB + 48
    ai = N.ArenaInfo()
    rc = lib.ccm_arena_acquire(0, nbytes, C.byref(ai))
    run.rc(rc, ("arena acquire",))
    run.check(rc == 0, ("arena acquire",), rc, N.last_error() if rc else "")
    if rc:
        return
    nz = C.c_uint64(1 << 63)

    def verify(what) -> int:
        rc = lib.ccm_arena_verify(0, N.VERIFY_AUTO, None, None, C.byref(nz), None)
        run.rc(rc, what)
        return rc

    try:
        with run.call(("arena fill",)):
            # 0xA5 in every byte, then 0x00: a fill that writes a wrong value shows as a count either way
            for value, want in ((0xA5, ai.bytes), (0x00, 0)):
                rc = lib.ccm_arena_fill(0, value, None)
                run.rc(rc, ("arena fill", value))
                rc |= verify(("arena fill", value))
                run.check(rc == 0 and nz.value == want, ("arena fill", value, "count"), nz.value, want)
        with run.call(("arena scrub",)):
            assert lib.ccm_arena_fill(0, 0xA5, None) == 0 and verify(("arena scrub",)) == 0, N.last_error()
            rc = lib.ccm_arena_scrub(0, N.SCRUB_AUTO, None, None, None)
            run.rc(rc, ("arena scrub",))
            rc |= verify(("arena scrub",))
            run.check(rc == 0 and nz.value == 0, ("arena scrub",), nz.value)
        with run.call(("arena step",)):
            # a default scrub-and-verify step: its scrub's last CTA clears the previous read-back's count
            assert lib.ccm_arena_fill(0, 0xA5, None) == 0 and verify(("arena step",)) == 0, N.last_error()
            rc = lib.ccm_arena_scrub_verify_async(0, N.SCRUB_AUTO, N.VERIFY_AUTO, None, None, None)
            run.rc(rc, ("arena step",))
            rc |= lib.ccm_arena_fetch_count(0, None, C.byref(nz))
            run.rc(rc, ("arena step",))
            run.check(rc == 0 and nz.value == 0, ("arena step",), rc, nz.value)
        with run.call(("arena pattern",)):
            rc = lib.ccm_arena_fill_random(0, SEED, None)
            run.rc(rc, ("arena pattern",))
            rc |= verify(("arena pattern",))
            want = SO.pattern_count_c(ai.bytes, SEED, 0)
            run.check(rc == 0 and nz.value == want, ("arena pattern",), nz.value, want)
            # the bytes too: a pattern shifted by a word has the same count, up to its two ends
            host = np.empty(ai.bytes, dtype=np.uint8)
            rc = lib.ccm_arena_read(0, 0, host.ctypes.data, ai.bytes)
            run.rc(rc, ("arena pattern", "bytes"))
            run.check(rc == 0 and ai.segments == 1 and np.array_equal(host, SO.pattern_np(ai.bytes, SEED, 0)),
                      ("arena pattern", "bytes"), rc, ai.segments)
    finally:
        rc = lib.ccm_arena_release(0)
        run.rc(rc, ("arena release",))
        run.check(rc == 0, ("arena release",), N.last_error())


def run_product(lib, run: Run) -> None:
    import gate_model as GM
    import report_cover_calls as RCALLS
    from k8s_cc_manager_b200 import _native as N
    for c in PRODUCT_CALLS:
        what = ("product", json.dumps(c))
        with run.call(what):
            rec = RCALLS.call(lib, c)
            if rec["rc"] == N.ERR_CUDA:
                raise Fault(f"{what}: {rec.get('error', '')}")
            diff = GM.compare(c, rec)
            run.check(diff is None, what, diff, rec.get("error", ""))


def kernel_names(prof) -> list:
    return sorted({e.name for e in prof.events() if str(e.device_type).endswith("CUDA") and e.name})


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--phase", choices=("region", "product", "all"), default="all")
    ap.add_argument("--kernels", action="store_true", help="profile the run and print the kernels it launched")
    args = ap.parse_args()
    # This process only, before torch initialises CUDA: one cudaMalloc per tensor, none cached.
    os.environ["PYTORCH_NO_CUDA_MEMORY_CACHING"] = "1"
    import torch
    assert not torch.cuda.is_initialized(), "CUDA came up before the allocator setting"

    import product_gate_calls as PGC
    from k8s_cc_manager_b200 import _native as N
    lib = PGC.open_lib()
    assert N.default_kernels() == FAST, N.default_kernels()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    run = Run(torch.cuda.synchronize)
    prof = None
    if args.kernels:
        from torch.profiler import ProfilerActivity, profile
        prof = profile(activities=[ProfilerActivity.CUDA])
        prof.__enter__()
    fault = None
    try:
        if args.phase in ("region", "all"):
            run_generic(lib, torch, run, sms)
            run_books(lib, torch, run, sms)
            run_probe(lib, torch, run)
            run_arena(lib, run)
        if args.phase in ("product", "all"):
            torch.cuda.synchronize()
            run_product(lib, run)
        torch.cuda.synchronize()
    except Fault as exc:
        fault = str(exc)[:2000]
    except RuntimeError as exc:   # a sticky CUDA error raised by torch outside any call
        if "CUDA" not in str(exc):
            raise
        fault = str(exc)[:2000]
    if fault is None:
        if prof is not None:
            prof.__exit__(None, None, None)
            print("KERNELS " + json.dumps(kernel_names(prof)), flush=True)
        rc = lib.ccm_device_release(0)
        run.check(rc == 0, ("device release",), rc)
    print("RESULT " + json.dumps({"phase": args.phase, "calls": run.calls, "first_mismatch": run.first,
                                  "mismatches": run.mismatches, "failed": run.failed, "fault": fault is not None,
                                  "fault_detail": fault}), flush=True)


if __name__ == "__main__":
    main()
