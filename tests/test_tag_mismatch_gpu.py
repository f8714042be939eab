"""The mismatch report on one H100: the check kernel's book against the numpy oracle at every tiling edge and above
2^32 bytes, the product call's report under tag_inject and scrub_alias in every mapping mode and on the fallback,
nothing added to clean calls, both reports on one call, the fan-out, the worker, the device and the manager, and the
kernel's rate against a same-run clean check."""
from __future__ import annotations

import ctypes as C
import logging
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "oracle"))
import mismatch_oracle as MO  # noqa: E402
import product_gate_calls as PGC  # noqa: E402
import product_plan as PP  # noqa: E402
import scenarios as SC  # noqa: E402
import tag_oracle as TO  # noqa: E402
from k8s_cc_manager_b200 import _native as N  # noqa: E402
from k8s_cc_manager_b200 import devices as D  # noqa: E402

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

GiB, MiB, KiB = 1 << 30, 1 << 20, 1 << 10
CHUNK = 128 * KiB
GUARD = 256 * KiB
DRILL_KEYS = PP.DRILL_KEYS + ("tag_inject", "scrub_alias")
N0 = GiB                               # scrub_alias: the first chunk (CCM_VMM_FIRST_CHUNK_MB default)


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


def fill(lib, ptr, n, seed):
    assert lib.ccm_region_tag_fill(0, C.c_void_p(ptr), n, seed, stream(), None) == 0, N.last_error()


def check_locate(lib, ptr, n, seed) -> D.MismatchReport:
    m = N.MismatchReport()
    assert lib.ccm_region_tag_check_locate(0, C.c_void_p(ptr), n, seed, stream(), C.byref(m)) == 0, N.last_error()
    assert m.located == 1 and m.seed == seed and m.va_base == ptr
    return D.MismatchReport.from_native(m)


def check_zero(lib, ptr, n, seed) -> int:
    mm = C.c_uint64()
    assert lib.ccm_region_tag_check_zero(0, C.c_void_p(ptr), n, seed, stream(), C.byref(mm), None) == 0
    return mm.value


def assert_matches_oracle(rep: D.MismatchReport, want: dict, what):
    assert rep.mismatch_bytes == want["mismatch_bytes"], what
    assert rep.mismatch_windows == want["mismatch_windows"], what
    assert rep.zero_windows == want["zero_windows"], what
    if want["mismatch_windows"]:
        assert (rep.first_offset, rep.last_offset) == (want["first_offset"], want["last_offset"]), what
    got = [(r.offset, r.mask, r.kind, r.source_offset, r.bytes) for r in rep.records]
    exp = [(w["offset"], w["mask"], w["kind"], w["source_offset"], w["bytes"]) for w in want["windows"]]
    assert all(r.chunk == 0 and r.source_chunk == 0 for r in rep.records)
    if not want["truncated"]:
        assert not rep.truncated and got == exp, what
    else:
        assert rep.truncated and len(got) == MO.RECORDS == len(set(got)) and got == sorted(got), what
        assert set(got) <= set(exp), what


def lengths(sm_count):
    return [1, 15, 16, 17, CHUNK - 1, CHUNK + 1, 2 * CHUNK * sm_count + 7]


OFFSETS = [0, 1, 3, 8, 15]


# ------------------------------------------------------------------------- kernel exactness
def test_every_tiling_edge_matches_the_oracle(lib):
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    top = max(lengths(sm)) + 32
    buf = torch.empty(GUARD + top + GUARD, dtype=torch.uint8, device="cuda")
    rng = np.random.default_rng(5)
    seen = set()
    for n in lengths(sm):
        for off in OFFSETS:
            for dense in (False, True):
                seed = (0x9E37 * (n + 1) + off * 7 + dense) & 0xFFFFFFFF or 1
                buf.fill_(0xEE)
                ptr = buf.data_ptr() + GUARD + off
                fill(lib, ptr, n, seed)
                host = buf.cpu().numpy()
                region = host[GUARD + off: GUARD + off + n]          # a view: edits go into `host`
                head = (128 - ptr % 128) % 128
                body_end = head + (n - head) // 16 * 16
                marks = sorted({m for m in (0, n - 1, head - 1, head, body_end - 1, body_end, head + CHUNK, n // 2)
                                if 0 <= m < n})
                for i, m in enumerate(marks):                       # single XORed bytes
                    region[m] ^= 0x5A
                aligned = [o for o in range((16 - ptr % 16) % 16, n - 15, 16)]
                if aligned:
                    picks = rng.choice(aligned, size=min(len(aligned), 6 if not dense else 90), replace=False)
                    for j, o in enumerate(sorted(int(x) for x in picks)):
                        kind = j % 3
                        if kind == 0:
                            region[o:o + 16] = 0                        # zero window
                        elif kind == 1:                                 # another window's tags (alias in the region)
                            src = aligned[(aligned.index(o) + 3) % len(aligned)]
                            region[o:o + 16] = TO.tag_bytes(seed, ptr + src, 16)
                        else:
                            region[o:o + 16] = rng.integers(0, 256, 16)  # random bytes
                buf.copy_(torch.from_numpy(host))
                before = host.copy()
                want = MO.report(before[GUARD + off: GUARD + off + n], ptr, seed)
                rep = check_locate(lib, ptr, n, seed)
                assert_matches_oracle(rep, want, (n, off, dense))
                after = buf.cpu().numpy()
                assert not after[GUARD + off: GUARD + off + n].any(), (n, off, "region not zeroed")
                assert np.all(after[:GUARD + off] == 0xEE) and np.all(after[GUARD + off + n:] == 0xEE), (n, off)
                # the plain check on the same input: the same count, and it leaves an empty book behind
                buf.copy_(torch.from_numpy(before))
                assert check_zero(lib, ptr, n, seed) == want["mismatch_bytes"]
                fill(lib, ptr, n, seed)
                clean = check_locate(lib, ptr, n, seed)
                assert clean.mismatch_windows == 0 and clean.records == [] and clean.mismatch_bytes == 0, (n, off)
                seen.add("truncated" if want["truncated"] else "exact")
                seen |= {w["kind"] for w in want["windows"]}
    assert {"exact", "truncated", "zero", "alias", "partial", "foreign"} <= seen, seen


def test_wrong_seed_above_2_to_the_32(lib):
    n = 17 * GiB + 5
    buf = torch.empty(n + 16, dtype=torch.uint8, device="cuda")
    ptr = buf.data_ptr() + 3
    written, checked = 0x0BADF00D, 0x1234ABCD
    fill(lib, ptr, n, written)
    rep = check_locate(lib, ptr, n, checked)
    assert TO.wrong_seed_count(written, checked, ptr, 64 * MiB) == 64 * MiB
    assert rep.mismatch_bytes > 1 << 32
    assert rep.mismatch_bytes == n                         # xor 0x19995BC0: every byte differs
    assert rep.mismatch_windows == ((ptr + n - 1) >> 4) - (ptr >> 4) + 1 == n // 16 + 1
    assert rep.truncated and len(rep.records) == MO.RECORDS
    assert all(r.kind == "foreign" for r in rep.records)
    del buf


def test_every_window_of_a_wrong_seed_is_counted(lib):
    n = 1 * GiB
    buf = torch.empty(n, dtype=torch.uint8, device="cuda")
    ptr = buf.data_ptr()
    fill(lib, ptr, n, 0x11111111)
    rep = check_locate(lib, ptr, n, 0x22222222)            # xor 0x33333333: every byte differs
    assert rep.mismatch_bytes == n and rep.mismatch_windows == n // 16 and rep.zero_windows == 0
    assert (rep.first_offset, rep.last_offset) == (0, n - 1)


# ------------------------------------------------------------------------------ product call
def product(lib, nbytes, env=None, drills=None):
    drills = drills or {}
    with PGC.knobs(env or {}):
        for k in DRILL_KEYS:
            assert lib.ccm_sim_set(0, k.encode(), int(drills.get(k, 0))) == 0
        try:
            tag, res = N.TagResult(), N.ScrubResult()
            l0 = lib.ccm_kernel_launches()
            rc = lib.ccm_scrub_verify_tagged(0, nbytes, C.byref(tag), C.byref(res))
            launches = lib.ccm_kernel_launches() - l0
        finally:
            for k in DRILL_KEYS:
                lib.ccm_sim_set(0, k.encode(), 0)
    m, d = N.MismatchReport(), N.DirtReport()
    assert lib.ccm_scrub_last_mismatch(0, C.byref(m)) == 0 and lib.ccm_scrub_last_dirt(0, C.byref(d)) == 0
    PGC.release_wait(lib)
    return rc, tag, res, launches, D.MismatchReport.from_native(m), D.DirtReport.from_native(d)


def check_tag_inject(rc, tag, res, mm, ranges, k, chunks, contiguous=True):
    offs = PP.inject_offsets(ranges, k)
    assert rc == N.ERR_MISMATCH and tag.mismatch_bytes == len(offs) > 0
    assert mm.located and mm.mismatch_bytes == mm.mismatch_windows == len(offs) and mm.zero_windows == 0
    assert mm.seed == tag.seed and mm.va_base == tag.va_base
    assert (mm.first_offset, mm.last_offset) == (min(offs), max(offs))
    if len(offs) > MO.RECORDS:
        assert mm.truncated and len(mm.records) == MO.RECORDS
    want = set(PP.inject_offsets(ranges, k))
    for r in mm.records:
        assert r.kind == "partial" and bin(r.mask).count("1") == 1, r
        o = r.offset + r.mask.bit_length() - 1
        assert o in want
        if contiguous:                                     # the window's address is va_base + offset
            got = bytes.fromhex(r.bytes)
            tags = TO.tag_bytes(tag.seed, tag.va_base + r.offset, 16)
            assert got[o - r.offset] == tags[o - r.offset] ^ 0xA5
            assert all(got[i] == tags[i] for i in range(16) if i != o - r.offset)
        if chunks is not None:
            assert [i for i, (co, cn) in enumerate(chunks) if co <= r.offset < co + cn] == [r.chunk], r


@pytest.mark.parametrize("mf,il", PP.MODES)
@pytest.mark.parametrize("k", [3, 1000])
def test_tag_inject_is_reported_as_partial_windows(lib, mf, il, k):
    env = PP.mode_env(mf, il)
    nbytes = 4 * GiB
    plain = product(lib, nbytes, env)[3]
    rc, tag, res, launches, mm, dirt = product(lib, nbytes, env, {"tag_inject": k})
    p = PP.plan(nbytes, res.device_free_before, PP.H100_GRAN, env)
    run = PP.simulate(p, None)
    ranges = run.ranges(p)
    check_tag_inject(rc, tag, res, mm, ranges, k, run.chunks)
    assert launches == plain + len(PP.inject_offsets(ranges, k)) and not dirt.located


@pytest.mark.parametrize("k", [3, 1000])
def test_tag_inject_on_the_fallback(lib, k):
    env = {"CCM_PIPELINE": "0", "CCM_ARENA_MAX_SEGMENT_MB": "96"}
    rc, tag, res, _, mm, _ = product(lib, 300 * MiB, env, {"tag_inject": k})
    segs = PP.arena_segments(300 * MiB, res.device_free_before, env)
    assert res.segments == len(segs) == 4
    check_tag_inject(rc, tag, res, mm, segs, k, segs, contiguous=False)


def check_alias_records(mm, map_first):
    for r in mm.records:
        if r.kind == "alias":
            assert r.offset < N0 and r.source_offset == r.offset + N0 and r.chunk == r.source_chunk == 0, r
        else:
            assert r.kind == "zero", r
            assert (r.offset < 2 * N0) if map_first else (N0 <= r.offset < 2 * N0), r


@pytest.mark.parametrize("nbytes", [4 * GiB, 0])
def test_scrub_alias_pipelined_names_the_second_view(lib, nbytes):
    rc, tag, res, _, mm, _ = product(lib, nbytes, {"CCM_MAP_FIRST": "0"}, {"scrub_alias": 1})
    assert rc == N.ERR_MISMATCH and mm.located and mm.mismatch_bytes == tag.mismatch_bytes
    assert mm.mismatch_windows == 2 * N0 // 16 and mm.zero_windows == N0 // 16
    assert mm.truncated and len(mm.records) == MO.RECORDS
    check_alias_records(mm, False)
    assert any(r.kind == "alias" for r in mm.records)
    assert "delta 0x40000000, chunk 0 ← chunk 0" in mm.summary()


def test_scrub_alias_map_first(lib):
    rc, tag, res, _, mm, _ = product(lib, 4 * GiB, {"CCM_MAP_FIRST": "1"}, {"scrub_alias": 1})
    assert rc == N.ERR_MISMATCH and mm.located
    assert N0 // 16 <= mm.mismatch_windows <= N0 // 8 and mm.zero_windows <= N0 // 16
    check_alias_records(mm, True)


@pytest.mark.parametrize("env", [{"CCM_MAP_FIRST": "0"}, {"CCM_MAP_FIRST": "1"}, {"CCM_PIPELINE": "0"}])
def test_clean_calls_leave_no_report(lib, env):
    rc, tag, res, _, mm, _ = product(lib, 4 * GiB, env, {"tag_inject": 2})
    assert rc == N.ERR_MISMATCH and mm.located
    rc, tag, res, _, mm, dirt = product(lib, 4 * GiB, env)
    assert rc == 0 and not mm.located and mm.records == [] and not dirt.located


def test_both_reports_on_one_call(lib):
    rc, tag, res, _, mm, dirt = product(lib, 4 * GiB, {}, {"tag_inject": 2, "scrub_inject": 5})
    assert rc == N.ERR_MISMATCH and tag.mismatch_bytes == 2 and res.nonzero_bytes == 5
    assert mm.located and mm.mismatch_windows == 2 and all(r.kind == "partial" for r in mm.records)
    assert dirt.located and dirt.dirty_windows == 5


# ----------------------------------------------------------------------------------- other paths
def test_fan_out_worker_and_device_carry_the_report(lib):
    from k8s_cc_manager_b200 import scrub_worker
    gpu = next(d for d in D.find_gpus()[0] if d.cuda_ordinal == 0)
    with PGC.knobs({}):
        lib.ccm_sim_set(gpu.index, b"scrub_alias", 1)
        try:
            reps, _ = D.scrub_and_verify_many([gpu], 4 * GiB, check="tagged")
            assert reps[0].mismatch is not None and reps[0].mismatch.mismatch_bytes == reps[0].mismatch_bytes > 0
            assert reps[0].dirt is None
            PGC.release_wait(lib)
            js = scrub_worker.run([gpu.bdf], 4 * GiB, "tagged")["reports"][0]
            assert js["mismatch"]["mismatch_windows"] > 0 and "dirt" not in js
            assert D.ScrubReport.from_json(js).mismatch == D.MismatchReport.from_json(js["mismatch"])
            PGC.release_wait(lib)
            with pytest.raises(D.GpuError) as ei:
                gpu.scrub_and_verify(4 * GiB, check="tagged")
            assert ei.value.status == N.ERR_MISMATCH and ei.value.mismatch.mismatch_windows == 2 * N0 // 16
        finally:
            lib.ccm_sim_set(gpu.index, b"scrub_alias", 0)
            PGC.release_wait(lib)
    reps, _ = D.scrub_and_verify_many([gpu], GiB, check="tagged")
    assert reps[0].clean and reps[0].mismatch is None and "mismatch" not in reps[0].as_json()
    PGC.release_wait(lib)


def test_manager_transition_logs_the_alias(lib, monkeypatch, caplog):
    import kubernetes
    from k8s_cc_manager_b200 import manager
    for k, v in dict(EVICT_OPERATOR_COMPONENTS="false", CC_RELEASE_CUDA_CONTEXT="false").items():
        monkeypatch.setenv(k, v)
    assert lib.ccm_init(N.BACKEND_CUDASIM) == 0
    lib.ccm_sim_set(-1, b"cc_mode", N.CC_MODES["off"])
    lib.ccm_sim_set(0, b"scrub_alias", 1)
    try:
        c = kubernetes.reset_cluster()
        c.add_node(SC.NODE, {})
        mgr = manager.CCManager(SC.NODE, "on", True, device_source=D.find_gpus, scrub_bytes=4 * GiB,
                                scrub_check="tagged")
        with caplog.at_level(logging.ERROR, logger="k8s-cc-manager"):
            assert mgr.set_cc_mode("on") is False
        bdf = next(d.bdf for d in D.find_gpus()[0] if d.cuda_ordinal == 0)
        mm = mgr.last_transition["scrub_mismatch"][bdf]
        assert mm.mismatch_windows == 2 * N0 // 16
        assert any(f"HBM tag mismatch on {bdf}" in r.getMessage() and "delta 0x40000000" in r.getMessage()
                   for r in caplog.records)
    finally:
        lib.ccm_sim_set(0, b"scrub_alias", 0)
        for d in D.find_gpus()[0]:
            if d.is_gpu():
                d.wait_scrub_released()


# ------------------------------------------------------------------------------------- rate
def _best(fn, prep, reps=5):
    ts = []
    for _ in range(reps + 1):
        prep()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return min(ts[1:])


@pytest.mark.parametrize("dirt", ["sparse", "every_byte"])
def test_mismatches_keep_up_with_a_clean_check(lib, dirt):
    n = 16 * GiB
    buf = torch.empty(n, dtype=torch.uint8, device="cuda")
    p, st, seed = buf.data_ptr(), stream(), 0xA11CE
    m = N.MismatchReport()
    step = 32 * MiB

    def prep_clean():
        fill(lib, p, n, seed)

    def prep_dirty():
        fill(lib, p, n, seed if dirt == "sparse" else seed ^ 0x5A5A5A5A)
        if dirt == "sparse":
            buf[torch.arange(0, n, step, device="cuda")] ^= 0xA5

    run = lambda: lib.ccm_region_tag_check_locate(0, C.c_void_p(p), n, seed, st, C.byref(m))  # noqa: E731
    t_clean = _best(run, prep_clean)
    assert m.mismatch_bytes == 0
    t_dirty = _best(run, prep_dirty)
    assert m.mismatch_bytes == (n // step if dirt == "sparse" else n)
    ratio = t_clean / t_dirty
    print(f"{dirt}: clean {n / t_clean / 1e6:.0f} GB/s, with mismatches {n / t_dirty / 1e6:.0f} GB/s ({ratio:.3f}x)")
    # A flood takes the booking branch in every batch: it reads each vector a second time (from L2) and books each
    # window one after another.  Measured on one H100 80GB HBM3 at 700 W: 0.56x (profiles/h100_tag_mismatch.json).
    assert ratio >= (0.95 if dirt == "sparse" else 0.5)
