"""The dirt triage on one H100, in every mapping mode, on the cudaMalloc fallback, through the fan-out, after the tagged
gate's dirty read-back and in a census call.  For each:

- an armed "scrub_inject" call equals the unarmed call in status, result, dirt report and dirt page map, and every
  dirt page clears;
- with the "triage_stay" / "triage_return" drills, every page's class and bytes equal oracle/triage_oracle.py;
- an armed dirty call launches what the unarmed one launches, plus one re-zero, one re-read and one more re-read per
  run, plus the drills' XORs; an armed clean call launches exactly what an unarmed clean call launches;
- the hold waited is at least the hold asked for, a later clean call empties the report, and the HBM still goes back.
"scrub_flood" makes the triage examine every mapped page."""
from __future__ import annotations

import ctypes as C
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "oracle"))
import product_gate_calls as PGC  # noqa: E402
import product_plan as PP  # noqa: E402
import triage_oracle as TR  # noqa: E402
from k8s_cc_manager_b200 import _native as N  # noqa: E402
from k8s_cc_manager_b200 import devices as D  # noqa: E402

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

GiB, MiB = 1 << 30, 1 << 20
PAGE = TR.PAGE_BYTES
HOLD_MS = 5
DRILL_KEYS = PP.DRILL_KEYS + ("tag_inject", "scrub_alias", "scrub_residue", "triage_stay", "triage_return")
# the result fields an armed call must leave as the unarmed call does
RESULT_FIELDS = ("status", "bytes_requested", "bytes_scrubbed", "device_total_bytes", "nonzero_bytes", "segments",
                 "scrub_variant", "verify_variant", "release_deferred", "bytes_unreached")
DIRT_FIELDS = ("nonzero_bytes", "dirty_windows", "first_offset", "last_offset", "located", "nrecords", "truncated")

# gate path -> (call, env, bytes, fan-out)
PATHS = {f"vmm-mf{mf}-il{il}": ("zero", PP.mode_env(mf, il), 4 * GiB, False) for mf, il in PP.MODES}
PATHS.update({
    "fallback": ("zero", {"CCM_PIPELINE": "0"}, 4 * GiB, False),
    "fallback-3MiB-segments": ("zero", {"CCM_PIPELINE": "0", "CCM_ARENA_MAX_SEGMENT_MB": "3"}, 64 * MiB, False),
    "fan-out": ("zero", {}, 4 * GiB, True),
    "tagged": ("tagged", {}, 4 * GiB, False),
    "census": ("census0", {}, 4 * GiB, False),
    "census-tagged-fallback": ("census1", {"CCM_PIPELINE": "0"}, 4 * GiB, False),
})


@pytest.fixture(scope="module")
def lib():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return PGC.open_lib()


def call(lib, kind: str, env: dict, drills: dict, nbytes: int, many: bool = False, hold: int = 0) -> dict:
    """One product call on device 0 (armed with `hold` ms when hold > 0) and what it left behind."""
    with PGC.knobs(env):
        for k in DRILL_KEYS:
            assert lib.ccm_sim_set(0, k.encode(), int(drills.get(k, 0))) == 0
        assert lib.ccm_scrub_triage(0, hold) == 0, N.last_error()
        try:
            res, rr, wall = N.ScrubResult(), N.ResidueReport(), C.c_double()
            tag = N.TagResult() if kind in ("tagged", "census1") else None
            tag_p = C.byref(tag) if tag is not None else None
            devs = (C.c_int * 1)(0)
            l0 = lib.ccm_kernel_launches()
            if kind.startswith("census"):
                rc = lib.ccm_scrub_verify_residue(0, nbytes, tag_p, C.byref(rr), C.byref(res))
            elif many:
                rc = lib.ccm_scrub_verify_many(1, devs, nbytes, C.byref(res), C.byref(wall))
            elif tag is not None:
                rc = lib.ccm_scrub_verify_tagged(0, nbytes, tag_p, C.byref(res))
            else:
                rc = lib.ccm_scrub_verify(0, nbytes, C.byref(res))
            launches = lib.ccm_kernel_launches() - l0
            err = N.last_error() if rc else ""
        finally:
            lib.ccm_scrub_triage(0, 0)
            for k in DRILL_KEYS:
                lib.ccm_sim_set(0, k.encode(), 0)
    d, t = N.DirtReport(), N.TriageReport()
    assert lib.ccm_scrub_last_dirt(0, C.byref(d)) == 0 and lib.ccm_scrub_last_triage(0, C.byref(t)) == 0
    out = {"rc": rc, "err": err, "res": res, "dirt": d, "triage": t, "launches": launches,
           "dirt_pages": D.last_page_map(0, N.BOOK_DIRT).entries, "triage_pages": D.last_triage_pages(0)}
    PGC.release_wait(lib)
    return out


def spans(env: dict, res, nbytes: int) -> list:
    """What the call mapped, as (offset, bytes) from the dirt report's va_base."""
    if env.get("CCM_PIPELINE") == "0":
        segs = PP.arena_segments(nbytes, res.device_free_before, env)
        assert sum(n for _, n in segs) == res.bytes_scrubbed and len(segs) == res.segments
        return segs
    return [(0, res.bytes_scrubbed)]


def assert_same_call(armed: dict, plain: dict, what):
    """Status, error text, result, dirt report and dirt page map as the unarmed call left them."""
    assert armed["rc"] == plain["rc"] and armed["err"] == plain["err"], what
    for f in RESULT_FIELDS:
        assert getattr(armed["res"], f) == getattr(plain["res"], f), (what, f)
    for f in DIRT_FIELDS:
        assert getattr(armed["dirt"], f) == getattr(plain["dirt"], f), (what, f)
    a, p = armed["dirt"], plain["dirt"]
    for i in range(a.nrecords):
        ra, rp = a.records[i], p.records[i]
        assert (ra.offset, ra.chunk, ra.mask, bytes(ra.bytes)) == (rp.offset, rp.chunk, rp.mask, bytes(rp.bytes)), what
    assert armed["dirt_pages"] == plain["dirt_pages"], what


def assert_triage(out: dict, env: dict, nbytes: int, stay: int, ret: int, what):
    """The report and pages of an armed dirty call equal the oracle's, from the call's own dirt page map."""
    t, entries = out["triage"], out["dirt_pages"]
    sp = spans(env, out["res"], nbytes)
    want = TR.report(entries, sp, stay, ret)
    assert t.triaged == 1 and t.hold_ms > 0 and t.ms_hold >= t.hold_ms and t.ms_triage >= t.ms_hold, what
    assert t.va_base == out["dirt"].va_base, what
    for k, v in want.items():
        assert getattr(t, k) == v, (what, k, getattr(t, k), v)
    rows = TR.classify(entries, stay, ret)
    got = [(p.page, p.chunk, p.cls, p.dirt_bytes, p.t2_bytes, p.t3_bytes) for p in out["triage_pages"]]
    assert got == rows, what
    assert t.stay_bytes + t.return_bytes + t.clear_bytes == out["dirt"].nonzero_bytes, what
    return len(TR.runs(entries, sp)), TR.drill_xors(entries, stay, ret)


@pytest.mark.parametrize("path", list(PATHS))
def test_triage_of_injected_dirt(lib, path):
    kind, env, nbytes, many = PATHS[path]
    drills = {"scrub_inject": PP.INJECT}
    plain = call(lib, kind, env, drills, nbytes, many)
    assert plain["rc"] == N.ERR_DIRTY and plain["dirt"].located and plain["triage"].triaged == 0, path
    assert plain["triage_pages"] == []
    # armed: the same call, and every dirt page clears
    armed = call(lib, kind, env, drills, nbytes, many, hold=HOLD_MS)
    assert_same_call(armed, plain, path)
    runs, xors = assert_triage(armed, env, nbytes, 0, 0, path)
    assert armed["triage"].clear_pages == len(armed["dirt_pages"]) and armed["triage"].t2_bytes == 0
    assert armed["launches"] == plain["launches"] + 3 * runs, (path, armed["launches"], plain["launches"], runs)
    # the drills: every class, exactly; pages of both drills stay (their byte is back to zero at T3)
    npages = len(armed["dirt_pages"])
    for stay, ret in ((1, 0), (0, 2), (2, 3), (npages, npages // 2), (0, npages + 5)):
        out = call(lib, kind, env, {**drills, "triage_stay": stay, "triage_return": ret}, nbytes, many, hold=HOLD_MS)
        assert_same_call(out, plain, (path, stay, ret))
        runs, xors = assert_triage(out, env, nbytes, stay, ret, (path, stay, ret))
        assert out["launches"] == plain["launches"] + 3 * runs + xors, (path, stay, ret)
    # a clean armed call launches what a clean unarmed one does, and empties the report
    clean = call(lib, kind, env, {}, nbytes, many)
    clean_armed = call(lib, kind, env, {}, nbytes, many, hold=HOLD_MS)
    assert clean["rc"] == clean_armed["rc"] == 0 and clean_armed["launches"] == clean["launches"], path
    assert clean_armed["triage"].triaged == 0 and clean_armed["triage_pages"] == [], path
    assert clean_armed["triage"].pages_examined == 0 and clean_armed["dirt_pages"] == [], path


@pytest.mark.parametrize("env", [{}, {"CCM_PIPELINE": "0"}], ids=["vmm", "fallback"])
def test_flood_examines_every_mapped_page(lib, env):
    nbytes = 0 if not env else 4 * GiB
    assert_flood(call(lib, "zero", env, {"scrub_flood": PP.FLOOD}, nbytes, hold=HOLD_MS), env, nbytes)


def assert_flood(out: dict, env: dict, nbytes: int):
    """An armed flooded call: every mapped page examined in one run per mapped range, and every page clears."""
    res, t = out["res"], out["triage"]
    assert out["rc"] == N.ERR_DIRTY and res.nonzero_bytes == res.bytes_scrubbed
    assert t.pages_examined == -(-res.bytes_scrubbed // PAGE) and t.bytes_examined == res.bytes_scrubbed
    assert t.runs == len(TR.runs(out["dirt_pages"], spans(env, res, nbytes)))
    assert t.clear_pages == t.pages_examined and t.clear_bytes == res.bytes_scrubbed and t.t2_bytes == t.t3_bytes == 0
    assert_triage(out, env, nbytes, 0, 0, env)


def test_hold_is_waited(lib):
    out = call(lib, "zero", {}, {"scrub_inject": 3}, GiB, hold=300)
    t = out["triage"]
    assert t.hold_ms == 300 and t.ms_hold >= 300 and out["res"].ms_total >= 300


def test_device_objects_arm_for_one_call_and_hand_the_hbm_back(lib):
    """scrub_and_verify(triage=True) arms the call, attaches `.triage` to the GpuError, and disarms: the next dirty
    call without it does not triage.  The HBM is handed back after every call."""
    gpu = next(g for g in D.find_gpus()[0] if g.is_gpu() and g.cuda_ordinal == 0)
    lib.ccm_sim_set(gpu.index, b"scrub_inject", 4)   # one range: its first, 17th, middle + 3 and last bytes
    try:
        with pytest.raises(D.GpuError) as ei:
            gpu.scrub_and_verify(GiB, triage=True, triage_hold_ms=HOLD_MS)
        tri = ei.value.triage
        assert tri is not None and tri.triaged and tri.hold_ms == HOLD_MS and tri.clear_pages == tri.pages_examined
        assert ei.value.dirt.pages.pages == tri.pages_examined and ei.value.dirt.nonzero_bytes == tri.clear_bytes == 4
        with pytest.raises(D.GpuError) as ei:
            gpu.scrub_and_verify(GiB)
        assert ei.value.triage is None and D.last_triage(0).triaged == 0
        reps, _ = D.scrub_and_verify_many([gpu], GiB, triage=True, triage_hold_ms=HOLD_MS)
        assert reps[0].triage is not None and reps[0].triage.pages_examined == reps[0].dirt.pages.pages
    finally:
        lib.ccm_sim_set(gpu.index, b"scrub_inject", 0)
    rep = gpu.scrub_and_verify(GiB, triage=True, triage_hold_ms=HOLD_MS)
    assert rep.clean and rep.triage is None
    ms_release, waited = gpu.wait_scrub_released()
    assert ms_release >= 0 and waited >= 0
    free, total = torch.cuda.mem_get_info()
    assert free > total // 2
