"""Launch-to-launch state of the default (compile-time-shape) kernels, and a child-process driver for
the programmatic-dependent-launch path.

The default scrub and verify kernels hand their grab and done words back zeroed (GrabCtl): a word left
non-zero would make the next launch start at chunk `grab` and skip chunk 0 (scrub) or the last chunks
(verify, which walks the chunks in descending order).  `launch_state_sequence` runs a fixed sequence of
default-kernel calls, alternating the engine stream and a torch stream, and after every call dirties
chunk 0 and the last whole chunk of the next region only.  Each region step runs every default-frame kernel that
has a grab word of its own: read-back, locate, census, scrub, tag fill and tag check.  An armed step runs their
proving twins (include/ccm.h: ccm_region_prove), which share the plain kernels' grab words, between plain steps,
and each twin's cover map must hold every byte of the region.

Run as a script (tests/test_scrub_exactness_gpu.py does, once with CCM_PDL=1 and once without — the
library latches CCM_PDL once per process) it also drives PDL-chained arena steps and a product call with
injected dirt, and prints one `RESULT <json>` line.  Not collected by pytest.
"""
from __future__ import annotations

import ctypes as C
import json
import os
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
for p in (ROOT, ROOT / "tests"):
    if str(p) not in sys.path:
        sys.path.insert(0, str(p))

from k8s_cc_manager_b200 import _native as N  # noqa: E402
from region_cover_calls import ArmedMap  # noqa: E402

CHUNK = 128 * 1024          # bytes per grab of the default kernels
MiB = 1 << 20
ARENA_SEGMENT_MB = 96
ARENA_BYTES = 300 * MiB     # -> segments of 96, 96, 96 and 12 MiB
OFFSET = 5                  # region start mod 128: a 123-byte ragged head in front of chunk 0


def ok(rc, what=""):
    assert rc == 0, f"{what}: {N.strerror(rc)}: {N.last_error()}"


def arena_segments() -> list[tuple[int, int]]:
    """(offset, bytes) of each arena segment: the acquire path takes CCM_ARENA_MAX_SEGMENT_MB pieces."""
    out, off, seg = [], 0, ARENA_SEGMENT_MB * MiB
    while off < ARENA_BYTES:
        n = min(seg, ARENA_BYTES - off)
        out.append((off, n))
        off += n
    return out


def dirt_offsets(n: int) -> list[int]:
    """Chunk 0 and the last whole chunk of a region at OFFSET (its first and its last byte), or the first
    and last byte when the region has no whole chunk."""
    head = min((128 - OFFSET) % 128, n)
    whole = (n - head) // 16 * 16 // CHUNK
    if whole == 0:
        return sorted({0, n - 1})
    return sorted({head, head + whole * CHUNK - 1})


def acquire_segmented_arena(lib) -> N.ArenaInfo:
    old = os.environ.get("CCM_ARENA_MAX_SEGMENT_MB")
    os.environ["CCM_ARENA_MAX_SEGMENT_MB"] = str(ARENA_SEGMENT_MB)
    try:
        ai = N.ArenaInfo()
        ok(lib.ccm_arena_acquire(0, ARENA_BYTES, C.byref(ai)), "arena_acquire")
    finally:
        if old is None:
            os.environ.pop("CCM_ARENA_MAX_SEGMENT_MB", None)
        else:
            os.environ["CCM_ARENA_MAX_SEGMENT_MB"] = old
    assert ai.bytes == ARENA_BYTES and ai.segments == len(arena_segments()), (ai.bytes, ai.segments)
    return ai


def dirty_arena_segments(lib, value: int = 0x5A) -> int:
    """Dirt in chunk 0 and in the last byte of every segment; returns the number of dirty bytes."""
    offs = sorted({o for off, n in arena_segments() for o in (off, off + n - 1)})
    for o in offs:
        ok(lib.ccm_arena_write(0, o, (C.c_uint8 * 1)(value), 1), "arena_write")
    return len(offs)


def region_step(lib, n: int, handle, armed: bool) -> list:
    """One region step over n bytes at OFFSET, dirt in chunk 0 and the last whole chunk (or the first and last byte):
    the read-back, the locate pass and the zero census each count it, the census and the scrub zero it, then the tag
    fill and the tag check (which zeroes the region again) count the same bytes XORed into the tags.  Returns
    [n or "armed n", [counted by each], [expected], bytes left non-zero after the zeroing passes, final read-back]."""
    import torch
    buf = torch.zeros(n + 256, dtype=torch.uint8, device="cuda")
    assert buf.data_ptr() % 128 == 0
    region = buf[OFFSET:OFFSET + n]
    offs = torch.tensor(dirt_offsets(n), device="cuda")
    region[offs] = 0xC3
    torch.cuda.synchronize()
    addr = region.data_ptr()
    ptr = C.c_void_p(addr)
    arm = ArmedMap(lib, addr, n, n) if armed else None
    torch.cuda.synchronize()   # the map is zero before any stream launches into it
    counted, left, maps = [], 0, []

    def run(call, what):
        """call() with the twins armed (and its map taken) when the step is armed."""
        if arm is None:
            return ok(call(), what)
        with arm:
            ok(call(), what)
        torch.cuda.synchronize()
        maps.append((what, arm.take()[0] == arm.want([(addr, n)])))
        torch.cuda.synchronize()

    nz = C.c_uint64(12345)
    run(lambda: lib.ccm_region_verify(0, ptr, n, N.VERIFY_AUTO, None, handle(), C.byref(nz), None), "region_verify")
    counted.append(nz.value)
    d = N.DirtReport()
    run(lambda: lib.ccm_region_locate(0, ptr, n, handle(), C.byref(d)), "region_locate")
    counted.append(d.nonzero_bytes)
    r = N.ResidueReport()
    run(lambda: lib.ccm_region_census(0, ptr, n, 0, 0, handle(), C.byref(r)), "region_census")
    counted.append(r.residue_bytes)
    torch.cuda.synchronize()
    left += int(torch.count_nonzero(region))
    region[offs] = 0xC3
    torch.cuda.synchronize()
    run(lambda: lib.ccm_region_scrub(0, ptr, n, N.SCRUB_AUTO, None, handle(), None), "region_scrub")
    torch.cuda.synchronize()
    left += int(torch.count_nonzero(region))
    run(lambda: lib.ccm_region_tag_fill(0, ptr, n, 0x600D, handle(), None), "region_tag_fill")
    torch.cuda.synchronize()
    region[offs] ^= 0xFF
    torch.cuda.synchronize()
    mm = C.c_uint64(12345)
    run(lambda: lib.ccm_region_tag_check_zero(0, ptr, n, 0x600D, handle(), C.byref(mm), None), "region_tag_check")
    counted.append(mm.value)
    torch.cuda.synchronize()
    left += int(torch.count_nonzero(region))
    run(lambda: lib.ccm_region_verify(0, ptr, n, N.VERIFY_AUTO, None, handle(), C.byref(nz), None), "region_verify")
    assert int(torch.count_nonzero(buf[:OFFSET])) == 0 and int(torch.count_nonzero(buf[OFFSET + n:])) == 0
    assert all(exact for _, exact in maps), (n, [what for what, exact in maps if not exact])
    return [f"armed {n}" if armed else n, counted, [offs.numel()] * 4, left, nz.value]


def launch_state_sequence(lib) -> list[list]:
    """Returns one [label, counted, expected, left after zeroing, verify after zeroing] row per step;
    raises on the first inexact result."""
    import torch
    stream = torch.cuda.Stream()
    handles = [None, C.c_void_p(stream.cuda_stream)]   # NULL = the engine's own stream
    calls = [0]

    def handle():
        h = handles[calls[0] % 2]
        calls[0] += 1
        return h

    rows = []
    # ("armed", n): the twins, each between plain launches on its grab word: no whole chunk, 1 byte, many chunks
    steps = [CHUNK - 1, ("armed", CHUNK - 1), 1, ("armed", 1), 9 * CHUNK + 12345, ("armed", 9 * CHUNK + 12345),
             "arena", CHUNK - 1, ("armed", 40 * MiB + 3), 40 * MiB + 3, 1, "arena", 9 * CHUNK + 12345]
    for step in steps:
        torch.cuda.synchronize()
        if step == "arena":
            acquire_segmented_arena(lib)
            try:
                want = dirty_arena_segments(lib)
                nz = C.c_uint64(12345)
                ok(lib.ccm_arena_verify(0, N.VERIFY_AUTO, None, handle(), C.byref(nz), None), "arena_verify")
                counted = nz.value
                h = handle()
                ok(lib.ccm_arena_scrub_verify_async(0, N.SCRUB_AUTO, N.VERIFY_AUTO, None, None, h), "step")
                ok(lib.ccm_arena_fetch_count(0, h, C.byref(nz)), "fetch_count")
                after = nz.value
                nsteps = C.c_int()                      # hands the step's event slot back, as bench.py does
                ok(lib.ccm_arena_step_times(0, 8, None, None, C.byref(nsteps)), "step_times")
                assert nsteps.value == 1, nsteps.value
                cfg = N.launch_cfg(schedule=1)          # generic kernel, independent of the grab words
                ok(lib.ccm_arena_verify(0, N.VERIFY_LD128, C.byref(cfg), handle(), C.byref(nz), None), "verify")
                left = nz.value
            finally:
                torch.cuda.synchronize()
                ok(lib.ccm_arena_release(0), "arena_release")
            rows.append(["arena", counted, want, left, after])
        else:
            armed = isinstance(step, tuple)
            rows.append(region_step(lib, step[1] if armed else step, handle, armed))
        label, counted, want, left, after = rows[-1]
        assert (counted, left, after) == (want, 0, 0), f"step {label}: counted {counted} of {want} dirty bytes, " \
                                                        f"{left} left after the scrub, re-verify {after}"
    return rows


def pdl_arena_steps(lib, steps: int = 4) -> list[list[int]]:
    """A poisoned segmented arena, then `steps` scrub -> verify steps on a torch stream (chained with
    programmatic dependent launch when CCM_PDL=1), each after fresh dirt in every segment."""
    import torch
    stream = torch.cuda.Stream()
    h = C.c_void_p(stream.cuda_stream)
    acquire_segmented_arena(lib)
    rows = []
    try:
        ok(lib.ccm_arena_fill(0, 0xA5, None), "arena_fill")
        for _ in range(steps):
            ndirt = dirty_arena_segments(lib)
            ok(lib.ccm_arena_scrub_verify_async(0, N.SCRUB_AUTO, N.VERIFY_AUTO, None, None, h), "step")
            nz = C.c_uint64(12345)
            ok(lib.ccm_arena_fetch_count(0, h, C.byref(nz)), "fetch_count")
            fetched = nz.value
            cfg = N.launch_cfg(schedule=2)              # generic kernel: launched without the PDL attribute
            ok(lib.ccm_arena_verify(0, N.VERIFY_LD256, C.byref(cfg), h, C.byref(nz), None), "verify")
            rows.append([ndirt, fetched, nz.value])
        s_ms, v_ms, n = (C.c_float * 8)(), (C.c_float * 8)(), C.c_int()
        ok(lib.ccm_arena_step_times(0, 8, s_ms, v_ms, C.byref(n)), "step_times")
        assert n.value == steps
    finally:
        stream.synchronize()
        ok(lib.ccm_arena_release(0), "arena_release")
    return rows


def product_call_with_dirt(lib, k: int = 1000) -> list[int]:
    lib.ccm_sim_set(0, b"scrub_inject", k)
    try:
        res = N.ScrubResult()
        rc = lib.ccm_scrub_verify(0, 2 << 30, C.byref(res))
    finally:
        lib.ccm_sim_set(0, b"scrub_inject", 0)
    return [rc, res.nonzero_bytes, res.bytes_scrubbed]


def main() -> None:
    lib = N.lib()
    ok(lib.ccm_init(N.BACKEND_CUDASIM), "init")
    out = {"arena_steps": pdl_arena_steps(lib),
           "sequence": launch_state_sequence(lib),
           "product_dirty": product_call_with_dirt(lib)}
    ms_release, waited = C.c_double(), C.c_double()
    ok(lib.ccm_scrub_release_wait(0, C.byref(ms_release), C.byref(waited)), "release_wait")
    print("RESULT " + json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
