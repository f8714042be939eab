"""The dirt report on one H100: the locate kernel against the numpy oracle at every edge of its tiling and above
2^32 bytes, the product call's report (records, chunk attribution) under injected dirt and floods in every mapping
mode, nothing added to clean calls, the tagged call, the arena fallback, the fan-out, the worker and the manager,
and the kernel's rate against a same-run verifier."""
from __future__ import annotations

import ctypes as C
import logging
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "oracle"))
import dirt_oracle as DO  # noqa: E402
import product_gate_calls as PGC  # noqa: E402
import product_plan as PP  # noqa: E402
import scenarios as SC  # noqa: E402
import scrub_cases as CASES  # noqa: E402
from k8s_cc_manager_b200 import _native as N  # noqa: E402
from k8s_cc_manager_b200 import devices as D  # noqa: E402

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

GiB, MiB, KiB = 1 << 30, 1 << 20, 1 << 10
GUARD = 256 * KiB
DRILL_KEYS = PP.DRILL_KEYS + ("tag_inject", "scrub_alias")
INJECTED = 0xA5                       # the byte value of the scrub_inject drill


@pytest.fixture(scope="module")
def lib():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return PGC.open_lib()


@pytest.fixture(autouse=True)
def _own_stream():
    """A torch stream of its own, handed to the library, so torch's fills and the library's launches are ordered."""
    if not torch.cuda.is_available():
        yield
        return
    with torch.cuda.stream(torch.cuda.Stream()):
        yield
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def locate(lib, ptr, n) -> D.DirtReport:
    d = N.DirtReport()
    assert lib.ccm_region_locate(0, C.c_void_p(ptr), n, stream(), C.byref(d)) == 0, N.last_error()
    assert d.located == 1
    return D.DirtReport.from_native(d)


def last_dirt(lib) -> D.DirtReport:
    d = N.DirtReport()
    assert lib.ccm_scrub_last_dirt(0, C.byref(d)) == 0, N.last_error()
    return D.DirtReport.from_native(d)


def assert_matches_oracle(rep: D.DirtReport, want: dict, what):
    assert rep.nonzero_bytes == want["nonzero_bytes"], what
    assert rep.dirty_windows == want["dirty_windows"], what
    if want["dirty_windows"]:
        assert (rep.first_offset, rep.last_offset) == (want["first_offset"], want["last_offset"]), what
    got = [(r.offset, r.mask, r.bytes) for r in rep.records]
    assert all(r.chunk == 0 for r in rep.records)
    if not want["truncated"]:
        assert not rep.truncated and got == want["windows"], what
    else:
        assert rep.truncated and len(got) == DO.RECORDS == len(set(got)) and got == sorted(got), what
        assert set(got) <= set(want["windows"]), what


# ------------------------------------------------------------------------- kernel exactness
def test_every_tiling_edge_matches_the_oracle(lib):
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    g = CASES.geometry(CASES.FAST_VERIFY, sm)             # 128 KiB per grab, one CTA per SM: locate's geometry too
    assert (g.chunk, g.grabbers) == (128 * KiB, sm)
    top = max(CASES.lengths(g)) + 128
    buf = torch.empty(GUARD + top + GUARD, dtype=torch.uint8, device="cuda")
    rng = np.random.default_rng(11)
    seen = {"exact": 0, "truncated": 0}
    for n in CASES.lengths(g):
        for off in CASES.OFFSETS:
            for dense in (False, True):
                buf.fill_(0xEE)                            # non-zero guards: never reported
                region = buf[GUARD + off: GUARD + off + n]
                region.zero_()
                pos = CASES.structural_positions(g, off, n)
                if dense:
                    pos = sorted(set(pos) | set(rng.integers(0, n, size=200).tolist()))
                region[torch.tensor(pos, device="cuda")] = torch.tensor(CASES.dirt_values(pos, n * 7 + off),
                                                                        dtype=torch.uint8, device="cuda")
                before = buf.cpu().numpy()
                ptr = buf.data_ptr() + GUARD + off
                rep = locate(lib, ptr, n)
                assert np.array_equal(buf.cpu().numpy(), before), (n, off, "the pass wrote memory")
                want = DO.report(before[GUARD + off: GUARD + off + n], ptr)
                assert_matches_oracle(rep, want, (n, off, dense))
                seen["truncated" if want["truncated"] else "exact"] += 1
    assert seen["exact"] and seen["truncated"], seen


def test_all_dirty_above_2_to_the_32(lib):
    n = 4 * GiB + 4 * MiB + 5
    buf = torch.full((n + 32,), 0x5A, dtype=torch.uint8, device="cuda")
    ptr = buf.data_ptr() + 3
    rep = locate(lib, ptr, n)
    assert rep.nonzero_bytes == n > 1 << 32
    assert rep.dirty_windows == DO.window_count(ptr, n)
    assert (rep.first_offset, rep.last_offset) == (0, n - 1) and rep.truncated
    offs = [r.offset for r in rep.records]
    assert len(offs) == DO.RECORDS == len(set(offs)) and offs == sorted(offs)
    for r in rep.records:
        assert (ptr + r.offset) % 16 == 0 and -16 < r.offset < n
        inside = [0 <= r.offset + i < n for i in range(16)]
        assert r.mask == sum(1 << i for i in range(16) if inside[i])
        assert bytes.fromhex(r.bytes) == bytes(0x5A if inside[i] else 0 for i in range(16))


# ------------------------------------------------------------------------------ product call
def product(lib, nbytes, env=None, drills=None, tagged=False):
    """One product call on device 0 with plan knobs and drills; returns (rc, result, launches, dirt report)."""
    drills = drills or {}
    with PGC.knobs(env or {}):
        for k in DRILL_KEYS:
            assert lib.ccm_sim_set(0, k.encode(), int(drills.get(k, 0))) == 0
        try:
            res = N.ScrubResult()
            l0 = lib.ccm_kernel_launches()
            if tagged:
                rc = lib.ccm_scrub_verify_tagged(0, nbytes, C.byref(N.TagResult()), C.byref(res))
            else:
                rc = lib.ccm_scrub_verify(0, nbytes, C.byref(res))
            launches = lib.ccm_kernel_launches() - l0
        finally:
            for k in DRILL_KEYS:
                lib.ccm_sim_set(0, k.encode(), 0)
    dirt = last_dirt(lib)
    PGC.release_wait(lib)
    return rc, res, launches, dirt


def inject_windows(offsets):
    return [(o // 16 * 16, 1 << (o % 16), bytes(INJECTED if i == o % 16 else 0 for i in range(16)).hex())
            for o in sorted(offsets)]


def ranges_from_records(offsets, mapped):
    """The enqueued ranges, read back from where scrub_inject put its bytes (4 per range: first, +17, middle + 3,
    last), for calls whose split the driver decided.  None when the records do not have that shape."""
    out, k, start = [], 0, 0
    while k + 3 < len(offsets) and offsets[k] == start:
        n = offsets[k + 3] - start + 1
        if offsets[k + 1:k + 4] != [start + 17, start + n // 2 + 3, start + n - 1]:
            return None
        out.append((start, n))
        start, k = start + n, k + 4
    return out if k == len(offsets) and start == mapped else None


def check_injected(rc, res, dirt, ranges, chunks=None):
    """Records == the windows of the drill's bytes; `chunks` (offset, bytes) in creation order, when known."""
    offs = PP.inject_offsets(ranges, PP.INJECT)
    assert rc == N.ERR_DIRTY and res.nonzero_bytes == len(offs) > 0
    assert dirt.located and dirt.nonzero_bytes == len(offs) == dirt.dirty_windows and not dirt.truncated
    assert (dirt.first_offset, dirt.last_offset) == (min(offs), max(offs))
    assert [(r.offset, r.mask, r.bytes) for r in dirt.records] == inject_windows(offs)
    assert dirt.va_base != 0 and dirt.ms_locate > 0
    ids = [r.chunk for r in dirt.records]
    assert ids == sorted(ids) and ids[0] == 0 and ids[-1] == res.segments - 1
    if chunks is not None:
        assert len(chunks) == res.segments
        for r in dirt.records:
            assert [i for i, (o, n) in enumerate(chunks) if o <= r.offset < o + n] == [r.chunk], r


@pytest.mark.parametrize("mf,il", PP.MODES)
def test_injected_dirt_is_located_at_every_requested_size(lib, mf, il):
    env = PP.mode_env(mf, il)
    for nbytes in PP.requested_sizes(PP.H100_GRAN):
        rc, res, _, dirt = product(lib, nbytes, env, PP.DRILLS["inject"])
        p = PP.plan(nbytes, res.device_free_before, PP.H100_GRAN, env)
        run = PP.simulate(p, None)
        assert res.bytes_scrubbed == run.mapped, nbytes
        check_injected(rc, res, dirt, run.ranges(p), run.chunks)


@pytest.mark.parametrize("tail_mb", PP.TAIL_MBS)
def test_injected_dirt_is_located_at_whole_hbm(lib, tail_mb):
    for env in PP.whole_hbm_cases(tail_mb):
        rc, res, _, dirt = product(lib, 0, env, PP.DRILLS["inject"])
        mapped = res.bytes_scrubbed
        p = PP.plan(0, res.device_free_before, PP.H100_GRAN, env)
        run = PP.simulate(p, mapped)
        if p.map_first or mapped >= p.main_end:
            ranges = run.ranges(p)
        elif dirt.truncated:
            # the main zone ran out of memory and halved its chunks into more than 16 ranges: the summary is
            # still exact, the records are 64 of the drill's bytes
            assert rc == N.ERR_DIRTY and dirt.nonzero_bytes == dirt.dirty_windows == res.nonzero_bytes > DO.RECORDS
            assert (dirt.first_offset, dirt.last_offset) == (0, mapped - 1)
            assert all(bin(r.mask).count("1") == 1 and r.bytes.replace("00", "") == f"{INJECTED:02x}"
                       for r in dirt.records)
            continue
        else:                                              # the driver chose the split: read it off the records
            ranges = ranges_from_records([r.offset + r.mask.bit_length() - 1 for r in dirt.records], mapped)
        assert ranges, (env, [r.offset for r in dirt.records])
        check_injected(rc, res, dirt, ranges)
        if mapped >= p.main_end:                           # main-zone chunks exact, tail granules after them
            for r in dirt.records:
                main = [i for i, (o, n) in enumerate(run.main) if o <= r.offset < o + n]
                assert main == [r.chunk] if main else len(run.main) <= r.chunk < res.segments, (env, r)


@pytest.mark.parametrize("nbytes", [4 * GiB, 0])
def test_flood_is_located_everywhere(lib, nbytes):
    rc, res, _, dirt = product(lib, nbytes, {}, PP.DRILLS["flood"])
    mapped = res.bytes_scrubbed
    assert rc == N.ERR_DIRTY and res.nonzero_bytes == mapped == dirt.nonzero_bytes
    assert (dirt.first_offset, dirt.last_offset) == (0, mapped - 1)
    assert dirt.dirty_windows == mapped // 16 and dirt.truncated
    offs = [r.offset for r in dirt.records]
    assert len(offs) == DO.RECORDS == len(set(offs)) and offs == sorted(offs)
    assert all(r.mask == 0xFFFF and r.bytes == f"{PP.FLOOD:02x}" * 16 and r.chunk < res.segments
               for r in dirt.records)


# ----------------------------------------------------------------------------------- clean calls
def test_clean_calls_launch_nothing_more_and_dirty_calls_one_kernel(lib):
    nbytes = 4 * GiB
    rc, _, plain, dirt = product(lib, nbytes)
    assert rc == 0 and not dirt.located
    for drills in ({"scrub_poison": PP.POISON}, {"scrub_alias": 1}):
        rc, _, launches, dirt = product(lib, nbytes, {}, drills)
        assert rc == 0 and launches == plain and not dirt.located and dirt.dirty_windows == 0, drills
    rc, _, launches, dirt = product(lib, nbytes, {}, {"scrub_inject": 3})
    assert rc == N.ERR_DIRTY and launches == plain + 1 and dirt.located and dirt.dirty_windows == 3
    # tagged: tag_inject's bytes fail the tag check, but the zero read-back is clean.  The drill launches one
    # XOR kernel per byte; nothing else is added.
    rc, _, tagged_plain, dirt = product(lib, nbytes, tagged=True)
    assert rc == 0 and not dirt.located
    rc, _, launches, dirt = product(lib, nbytes, {}, {"tag_inject": 3}, tagged=True)
    assert rc == N.ERR_MISMATCH and launches == tagged_plain + 3 and not dirt.located
    rc, _, _, dirt = product(lib, nbytes)                 # a later clean call clears the report
    assert rc == 0 and not dirt.located


# ----------------------------------------------------------------------------------- other paths
def test_tagged_call_locates_injected_dirt(lib):
    env = PP.mode_env(0, 1)
    rc, res, _, dirt = product(lib, 4 * GiB, env, PP.DRILLS["inject"], tagged=True)
    p = PP.plan(4 * GiB, res.device_free_before, PP.H100_GRAN, env)
    run = PP.simulate(p, None)
    check_injected(rc, res, dirt, run.ranges(p), run.chunks)


def test_arena_fallback_attributes_segments(lib):
    env = {"CCM_PIPELINE": "0", "CCM_ARENA_MAX_SEGMENT_MB": "96"}
    rc, res, _, dirt = product(lib, 300 * MiB, env, PP.DRILLS["inject"])
    segs = PP.arena_segments(300 * MiB, res.device_free_before, env)
    assert res.segments == len(segs) == 4
    check_injected(rc, res, dirt, segs, segs)


def test_fan_out_worker_and_device_carry_the_report(lib):
    from k8s_cc_manager_b200 import scrub_worker
    gpu = next(d for d in D.find_gpus()[0] if d.cuda_ordinal == 0)
    with PGC.knobs({}):
        lib.ccm_sim_set(gpu.index, b"scrub_inject", 1000)
        try:
            devs = (C.c_int * 2)(gpu.index, gpu.index)
            out = (N.ScrubResult * 2)()
            assert lib.ccm_scrub_verify_many(2, devs, GiB, out, None) == N.ERR_DIRTY
            dirt = last_dirt(lib)                          # map first: one range per call, 4 bytes
            assert dirt.dirty_windows == 4 and [r.offset for r in dirt.records][0] == 0
            PGC.release_wait(lib)
            reps, _ = D.scrub_and_verify_many([gpu], GiB)
            assert reps[0].dirt is not None and reps[0].dirt.dirty_windows == reps[0].nonzero_bytes == 4
            PGC.release_wait(lib)
            js = scrub_worker.run([gpu.bdf], GiB)["reports"][0]
            assert js["dirt"]["dirty_windows"] == 4 and D.ScrubReport.from_json(js).dirt == D.DirtReport.from_json(js["dirt"])
            PGC.release_wait(lib)
            with pytest.raises(D.GpuError) as ei:
                gpu.scrub_and_verify(GiB)
            assert ei.value.status == N.ERR_DIRTY and ei.value.dirt.dirty_windows == 4
            assert "non-zero bytes" in str(ei.value)
        finally:
            lib.ccm_sim_set(gpu.index, b"scrub_inject", 0)
            PGC.release_wait(lib)
    reps, _ = D.scrub_and_verify_many([gpu], GiB)
    assert reps[0].clean and reps[0].dirt is None and "dirt" not in reps[0].as_json()
    PGC.release_wait(lib)


def test_manager_transition_logs_and_keeps_the_report(lib, monkeypatch, caplog):
    import kubernetes
    from k8s_cc_manager_b200 import manager
    for k, v in dict(EVICT_OPERATOR_COMPONENTS="false", CC_RELEASE_CUDA_CONTEXT="false").items():
        monkeypatch.setenv(k, v)
    assert lib.ccm_init(N.BACKEND_CUDASIM) == 0
    lib.ccm_sim_set(-1, b"cc_mode", N.CC_MODES["off"])
    lib.ccm_sim_set(0, b"scrub_inject", 5)
    try:
        c = kubernetes.reset_cluster()
        c.add_node(SC.NODE, {})
        mgr = manager.CCManager(SC.NODE, "on", True, device_source=D.find_gpus, scrub_bytes=4 * GiB)
        with caplog.at_level(logging.ERROR, logger="k8s-cc-manager"):
            assert mgr.set_cc_mode("on") is False
        assert c.labels(SC.NODE).get("nvidia.com/cc.mode.state") == "failed"
        bdf = next(d.bdf for d in D.find_gpus()[0] if d.cuda_ordinal == 0)
        dirt = mgr.last_transition["scrub_dirt"][bdf]
        assert dirt.dirty_windows == 5 and dirt.first_offset == 0
        assert any(f"HBM dirt on {bdf}" in r.getMessage() for r in caplog.records)
    finally:
        lib.ccm_sim_set(0, b"scrub_inject", 0)
        for d in D.find_gpus()[0]:
            if d.is_gpu():
                d.wait_scrub_released()


# ------------------------------------------------------------------------------------- rate
def _best(fn, reps=5):
    ts = []
    for _ in range(reps + 1):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return min(ts[1:])


@pytest.mark.parametrize("dirt", ["sparse", "every_byte"])
def test_locate_keeps_up_with_the_verifier(lib, dirt):
    n = 32 * GiB
    buf = torch.zeros(n, dtype=torch.uint8, device="cuda")
    if dirt == "sparse":
        buf[torch.arange(0, n, n // 1000 + 7, device="cuda")] = 0x5A
    else:
        buf.fill_(0x5A)
    p, st = C.c_void_p(buf.data_ptr()), stream()
    d = N.DirtReport()
    t_verify = _best(lambda: lib.ccm_region_verify(0, p, n, N.VERIFY_AUTO, None, st, None, None))
    t_locate = _best(lambda: lib.ccm_region_locate(0, p, n, st, C.byref(d)))
    assert d.nonzero_bytes == (n if dirt == "every_byte" else len(range(0, n, n // 1000 + 7)))
    print(f"{dirt}: verify {n / t_verify / 1e6:.0f} GB/s, locate {n / t_locate / 1e6:.0f} GB/s")
    assert n / t_locate >= 0.85 * (n / t_verify)
