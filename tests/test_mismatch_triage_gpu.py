"""The mismatch triage on one H100, in every mapping mode, on the cudaMalloc fallback (also with 3 MiB segments),
through the fan-out and in a tagged census call.  For each, with "tag_inject" and a pinned seed:

- an armed call equals the unarmed call in status, error text, result, tag result, mismatch report (records included)
  and its page map, and dirt report, and every page of the mismatch page map clears;
- with the "triage_stay" / "triage_return" drills, every page's class and bytes equal tests/mismatch_triage_oracle.py;
- an armed call launches what the unarmed one launches, plus one re-tag, one check-and-zero and one read per run, plus
  the drills' XORs; an armed clean call launches exactly what an unarmed clean call launches.
"scrub_alias" makes both views of the aliased range stay, "tag_flood" makes the triage examine every mapped page, both
triages run on one call and each is armed on its own, the hold is waited, the device objects, the worker and the
manager carry the report, and the triage gives the same answers with programmatic dependent launch on and off.

Run as a script (`python tests/test_mismatch_triage_gpu.py`), this module makes the PDL cases in a fresh process and
prints one `RESULT <json>` line."""
from __future__ import annotations

import ctypes as C
import json
import logging
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
for p in (ROOT, ROOT / "tests", ROOT / "oracle"):
    if str(p) not in sys.path:
        sys.path.insert(0, str(p))
import product_gate_calls as PGC  # noqa: E402
import product_plan as PP  # noqa: E402
import scenarios as SC  # noqa: E402
import tag_oracle as TO  # noqa: E402
import mismatch_triage_oracle as MTR  # noqa: E402
import triage_oracle as TR  # noqa: E402
from k8s_cc_manager_b200 import _native as N  # noqa: E402
from k8s_cc_manager_b200 import devices as D  # noqa: E402

pytestmark = pytest.mark.gpu

GiB, MiB = 1 << 30, 1 << 20
PAGE = TR.PAGE_BYTES
HOLD_MS = 5
SEED = 0x5EED1234
N0 = GiB                               # scrub_alias: the first chunk (CCM_VMM_FIRST_CHUNK_MB default)
FLOOD = 0x5A
DRILL_KEYS = PP.DRILL_KEYS + ("tag_inject", "scrub_alias", "scrub_residue", "triage_stay", "triage_return",
                              "tag_flood")
RESULT_FIELDS = ("status", "bytes_requested", "bytes_scrubbed", "device_total_bytes", "nonzero_bytes", "segments",
                 "scrub_variant", "verify_variant", "release_deferred", "bytes_unreached")
DIRT_FIELDS = ("nonzero_bytes", "dirty_windows", "first_offset", "last_offset", "located", "nrecords", "truncated")
MISMATCH_FIELDS = ("mismatch_bytes", "mismatch_windows", "zero_windows", "first_offset", "last_offset", "seed",
                   "located", "nrecords", "truncated")
# the triage report's fields that do not depend on the virtual address or the clock
TRIAGE_FIELDS = tuple(f for f, _ in N.TriageReport._fields_ if f not in ("va_base", "ms_hold", "ms_triage"))

# gate path -> (call, env, bytes)
PATHS = {f"vmm-mf{mf}-il{il}": ("tagged", PP.mode_env(mf, il), 4 * GiB) for mf, il in PP.MODES}
PATHS.update({
    "fallback": ("tagged", {"CCM_PIPELINE": "0"}, 4 * GiB),
    "fallback-3MiB-segments": ("tagged", {"CCM_PIPELINE": "0", "CCM_ARENA_MAX_SEGMENT_MB": "3"}, 64 * MiB),
    "fan-out": ("many", {}, 4 * GiB),
    "census-tagged": ("census", {}, 4 * GiB),
})


def call(lib, kind: str, env: dict, drills: dict, nbytes: int, hold: int = 0, dirt_hold: int = 0) -> dict:
    """One tagged product call on device 0 with the seed SEED (armed for the mismatch triage with `hold` ms, for the
    dirt triage with `dirt_hold` ms, when > 0) and what it left behind."""
    with PGC.knobs(env):
        for k in DRILL_KEYS:
            assert lib.ccm_sim_set(0, k.encode(), int(drills.get(k, 0))) == 0
        assert lib.ccm_scrub_mismatch_triage(0, hold) == 0, N.last_error()
        assert lib.ccm_scrub_triage(0, dirt_hold) == 0, N.last_error()
        try:
            res, rr, wall = N.ScrubResult(), N.ResidueReport(), C.c_double()
            tag = N.TagResult(seed=SEED)
            devs = (C.c_int * 1)(0)
            l0 = lib.ccm_kernel_launches()
            if kind == "census":
                rc = lib.ccm_scrub_verify_residue(0, nbytes, C.byref(tag), C.byref(rr), C.byref(res))
            elif kind == "many":
                rc = lib.ccm_scrub_verify_many_tagged(1, devs, nbytes, C.byref(tag), C.byref(res), C.byref(wall))
            else:
                rc = lib.ccm_scrub_verify_tagged(0, nbytes, C.byref(tag), C.byref(res))
            launches = lib.ccm_kernel_launches() - l0
            err = N.last_error() if rc else ""
        finally:
            lib.ccm_scrub_mismatch_triage(0, 0)
            lib.ccm_scrub_triage(0, 0)
            for k in DRILL_KEYS:
                lib.ccm_sim_set(0, k.encode(), 0)
    d, m, t, mt = N.DirtReport(), N.MismatchReport(), N.TriageReport(), N.TriageReport()
    assert lib.ccm_scrub_last_dirt(0, C.byref(d)) == 0 and lib.ccm_scrub_last_mismatch(0, C.byref(m)) == 0
    assert lib.ccm_scrub_last_triage(0, C.byref(t)) == 0 and lib.ccm_scrub_last_mismatch_triage(0, C.byref(mt)) == 0
    out = {"rc": rc, "err": err, "res": res, "tag": tag, "dirt": d, "mm": m, "triage": t, "mtriage": mt,
           "launches": launches, "dirt_pages": D.last_page_map(0, N.BOOK_DIRT).entries,
           "mm_pages": D.last_page_map(0, N.BOOK_MISMATCH).entries, "triage_pages": D.last_triage_pages(0),
           "mtriage_pages": D.last_mismatch_triage_pages(0)}
    PGC.release_wait(lib)
    return out


def spans(env: dict, res, nbytes: int) -> list:
    """What the call mapped, as (offset, bytes) from the reports' va_base."""
    if env.get("CCM_PIPELINE") == "0":
        segs = PP.arena_segments(nbytes, res.device_free_before, env)
        assert sum(n for _, n in segs) == res.bytes_scrubbed and len(segs) == res.segments
        return segs
    return [(0, res.bytes_scrubbed)]


def assert_same_call(armed: dict, plain: dict, what):
    """Status, error text, result, tag result, mismatch report and page map, and dirt report as the unarmed call."""
    assert armed["rc"] == plain["rc"] and armed["err"] == plain["err"], what
    for f in RESULT_FIELDS:
        assert getattr(armed["res"], f) == getattr(plain["res"], f), (what, f)
    assert (armed["tag"].seed, armed["tag"].mismatch_bytes) == (plain["tag"].seed, plain["tag"].mismatch_bytes), what
    a, p = armed["mm"], plain["mm"]
    for f in MISMATCH_FIELDS:
        assert getattr(a, f) == getattr(p, f), (what, f)
    same_va = a.va_base == p.va_base   # the records' bytes hold tags of their virtual addresses
    for i in range(a.nrecords):
        ra, rp = a.records[i], p.records[i]
        assert (ra.offset, ra.chunk, ra.mask, ra.kind, ra.source_offset, ra.source_chunk) == \
            (rp.offset, rp.chunk, rp.mask, rp.kind, rp.source_offset, rp.source_chunk), what
        assert not same_va or bytes(ra.bytes) == bytes(rp.bytes), what
    assert armed["mm_pages"] == plain["mm_pages"], what
    for f in DIRT_FIELDS:
        assert getattr(armed["dirt"], f) == getattr(plain["dirt"], f), (what, f)
    assert armed["dirt_pages"] == plain["dirt_pages"], what


def assert_mtriage(out: dict, env: dict, nbytes: int, stay: int, ret: int, what):
    """The mismatch triage of an armed failed call equals the oracle's, from the call's own mismatch page map."""
    t, entries = out["mtriage"], out["mm_pages"]
    sp = spans(env, out["res"], nbytes)
    want = MTR.report(entries, sp, stay, ret)
    assert t.triaged == 1 and t.hold_ms > 0 and t.ms_hold >= t.hold_ms and t.ms_triage >= t.ms_hold, what
    assert t.va_base == out["mm"].va_base == out["tag"].va_base, what
    for k, v in want.items():
        assert getattr(t, k) == v, (what, k, getattr(t, k), v)
    rows = MTR.classify(entries, stay, ret)
    got = [(p.page, p.chunk, p.cls, p.dirt_bytes, p.t2_bytes, p.t3_bytes) for p in out["mtriage_pages"]]
    assert got == rows, what
    assert t.stay_bytes + t.return_bytes + t.clear_bytes == out["tag"].mismatch_bytes, what
    return len(TR.runs(entries, sp)), TR.drill_xors(entries, stay, ret)


def assert_dirt_triage(out: dict, env: dict, nbytes: int, what):
    t, entries = out["triage"], out["dirt_pages"]
    want = TR.report(entries, spans(env, out["res"], nbytes))
    assert t.triaged == 1, what
    for k, v in want.items():
        assert getattr(t, k) == v, (what, k, getattr(t, k), v)
    return len(TR.runs(entries, spans(env, out["res"], nbytes)))


# ------------------------------------------------------------------------------------------------------ on device 0
@pytest.fixture(scope="module")
def lib():
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return PGC.open_lib()


@pytest.mark.parametrize("path", list(PATHS))
def test_triage_of_injected_mismatches(lib, path):
    kind, env, nbytes = PATHS[path]
    drills = {"tag_inject": PP.INJECT}
    plain = call(lib, kind, env, drills, nbytes)
    assert plain["rc"] == N.ERR_MISMATCH and plain["mm"].located and plain["mtriage"].triaged == 0, path
    assert plain["res"].nonzero_bytes == 0 and plain["mtriage_pages"] == [], path
    armed = call(lib, kind, env, drills, nbytes, hold=HOLD_MS)
    assert_same_call(armed, plain, path)
    runs, _ = assert_mtriage(armed, env, nbytes, 0, 0, path)
    t = armed["mtriage"]
    assert t.clear_pages == len(armed["mm_pages"]) and t.t2_bytes == t.t3_bytes == 0, path
    assert armed["triage"].triaged == 0, path
    assert armed["launches"] == plain["launches"] + 3 * runs, (path, armed["launches"], plain["launches"], runs)
    npages = len(armed["mm_pages"])
    for stay, ret in ((1, 0), (0, 1), (2, 2), (0, 2), (npages, 1), (1, npages), (npages + 3, 0), (0, npages + 3),
                      (npages + 3, npages + 3)):
        out = call(lib, kind, env, {**drills, "triage_stay": stay, "triage_return": ret}, nbytes, hold=HOLD_MS)
        assert_same_call(out, plain, (path, stay, ret))
        runs, xors = assert_mtriage(out, env, nbytes, stay, ret, (path, stay, ret))
        assert out["launches"] == plain["launches"] + 3 * runs + xors, (path, stay, ret)
    clean = call(lib, kind, env, {}, nbytes)
    clean_armed = call(lib, kind, env, {}, nbytes, hold=HOLD_MS)
    assert clean["rc"] == clean_armed["rc"] == 0 and clean_armed["launches"] == clean["launches"], path
    assert clean_armed["mtriage"].triaged == 0 and clean_armed["mtriage_pages"] == [], path


def assert_alias(out: dict, env: dict, nbytes: int, what) -> tuple:
    """scrub_alias with CCM_MAP_FIRST=0: both views, [0, 2 N0), in one run; nothing returns; of every aliased pair of
    pages at least one stays.  Returns (pages that stay in the first view, in the second)."""
    t, pages = out["mtriage"], out["mtriage_pages"]
    assert out["rc"] == N.ERR_MISMATCH and out["res"].nonzero_bytes == 0, what
    assert t.runs == 1 and t.bytes_examined == 2 * N0 and t.pages_examined == 2 * N0 // PAGE, what
    assert [p.page for p in pages] == list(range(2 * N0 // PAGE)), what
    assert t.return_pages == 0 and t.t3_bytes == 0, what
    assert all((p.cls == "stays") == (p.t2_bytes > 0) and p.t3_bytes == 0 for p in pages), what
    assert t.stay_bytes + t.clear_bytes == out["tag"].mismatch_bytes == sum(p.dirt_bytes for p in pages), what
    assert t.t2_bytes == sum(p.t2_bytes for p in pages) and t.va_base == out["mm"].va_base, what
    stays = {p.page for p in pages if p.cls == "stays"}
    half = N0 // PAGE
    assert all(p in stays or p + half in stays for p in range(half)), what
    return sum(1 for p in stays if p < half), sum(1 for p in stays if p >= half)


@pytest.mark.parametrize("nbytes", [4 * GiB, 0], ids=["4GiB", "whole-HBM"])
def test_alias_stays(lib, nbytes):
    env = PP.mode_env(0, 1)
    out = call(lib, "tagged", env, {"scrub_alias": 1}, nbytes, hold=HOLD_MS)
    first, second = assert_alias(out, env, nbytes, nbytes)
    print(f"\nscrub_alias at {nbytes or 'whole HBM'}: {first} of {N0 // PAGE} first-view pages and {second} of "
          f"{N0 // PAGE} second-view pages stay")


def test_alias_map_first_adds_up(lib):
    env = PP.mode_env(1, 1)
    out = call(lib, "tagged", env, {"scrub_alias": 1}, 4 * GiB, hold=HOLD_MS)
    t = out["mtriage"]
    assert out["rc"] == N.ERR_MISMATCH and t.triaged and t.return_pages == 0
    assert t.stay_pages + t.clear_pages == t.pages_examined == len(out["mm_pages"])
    assert t.stay_bytes + t.clear_bytes == out["tag"].mismatch_bytes
    print(f"\nscrub_alias, CCM_MAP_FIRST=1: {t.stay_pages} of {t.pages_examined} pages stay")


def assert_flood(out: dict, env: dict, nbytes: int, what):
    """tag_flood: a clean read-back, every mapped page examined in one run per mapped span, and every page clears."""
    res, t = out["res"], out["mtriage"]
    assert out["rc"] == N.ERR_MISMATCH and res.nonzero_bytes == 0 and out["tag"].mismatch_bytes > 0, what
    assert t.pages_examined == -(-res.bytes_scrubbed // PAGE) and t.bytes_examined == res.bytes_scrubbed, what
    assert t.runs == len(spans(env, res, nbytes)), what
    assert t.clear_pages == t.pages_examined and t.clear_bytes == out["tag"].mismatch_bytes, what
    assert t.t2_bytes == t.t3_bytes == 0, what
    assert_mtriage(out, env, nbytes, 0, 0, what)


@pytest.mark.parametrize("env,nbytes", [({}, 0), ({"CCM_PIPELINE": "0"}, 4 * GiB)], ids=["vmm-whole-HBM", "fallback"])
def test_flood_examines_every_mapped_page(lib, env, nbytes):
    assert_flood(call(lib, "tagged", env, {"tag_flood": FLOOD}, nbytes, hold=HOLD_MS), env, nbytes, env)


def test_flood_counts_what_the_tag_oracle_counts(lib):
    env = {"CCM_PIPELINE": "0"}
    out = call(lib, "tagged", env, {"tag_flood": FLOOD}, 64 * MiB)
    res, tag = out["res"], out["tag"]
    assert res.segments == 1 and res.bytes_scrubbed == 64 * MiB and out["rc"] == N.ERR_MISMATCH
    want = int(np.count_nonzero(TO.tag_bytes(SEED, tag.va_base, 64 * MiB) != FLOOD))
    assert tag.mismatch_bytes == want and res.nonzero_bytes == 0


def test_zero_only_call_ignores_tag_flood(lib):
    assert lib.ccm_sim_set(0, b"tag_flood", FLOOD) == 0
    try:
        res = N.ScrubResult()
        assert lib.ccm_scrub_verify(0, 64 * MiB, C.byref(res)) == 0, N.last_error()
        assert res.nonzero_bytes == 0
    finally:
        lib.ccm_sim_set(0, b"tag_flood", 0)
        PGC.release_wait(lib)


@pytest.mark.parametrize("env", [{}, {"CCM_PIPELINE": "0"}], ids=["vmm", "fallback"])
def test_both_triages_on_one_call_and_each_armed_on_its_own(lib, env):
    drills = {"tag_inject": 4, "scrub_inject": 4}
    plain = call(lib, "tagged", env, drills, 4 * GiB)
    assert plain["rc"] == N.ERR_MISMATCH and plain["res"].nonzero_bytes > 0
    both = call(lib, "tagged", env, drills, 4 * GiB, hold=HOLD_MS, dirt_hold=HOLD_MS)
    assert_same_call(both, plain, "both")
    mruns, _ = assert_mtriage(both, env, 4 * GiB, 0, 0, "both")
    druns = assert_dirt_triage(both, env, 4 * GiB, "both")
    assert both["launches"] == plain["launches"] + 3 * mruns + 3 * druns
    only_m = call(lib, "tagged", env, drills, 4 * GiB, hold=HOLD_MS)
    assert_same_call(only_m, plain, "mismatch only")
    assert only_m["triage"].triaged == 0 and only_m["triage_pages"] == []
    assert only_m["launches"] == plain["launches"] + 3 * mruns
    only_d = call(lib, "tagged", env, drills, 4 * GiB, dirt_hold=HOLD_MS)
    assert_same_call(only_d, plain, "dirt only")
    assert only_d["mtriage"].triaged == 0 and only_d["mtriage_pages"] == []
    assert only_d["launches"] == plain["launches"] + 3 * druns
    assert (only_d["triage"].pages_examined, only_d["triage"].clear_pages) == \
        (both["triage"].pages_examined, both["triage"].clear_pages)


def test_hold_is_waited(lib):
    out = call(lib, "tagged", {}, {"tag_inject": 3}, GiB, hold=300)
    t = out["mtriage"]
    assert t.hold_ms == 300 and t.ms_hold >= 300 and out["res"].ms_total >= 300


def test_device_objects_and_the_worker_arm_for_one_call(lib):
    from k8s_cc_manager_b200 import scrub_worker
    gpu = next(g for g in D.find_gpus()[0] if g.is_gpu() and g.cuda_ordinal == 0)
    lib.ccm_sim_set(gpu.index, b"tag_inject", 4)   # one range: its first, 17th, middle + 3 and last bytes
    try:
        with pytest.raises(D.GpuError) as ei:
            gpu.scrub_and_verify(GiB, check="tagged", mismatch_triage=True, triage_hold_ms=HOLD_MS)
        mt = ei.value.mismatch_triage
        assert mt is not None and mt.triaged and mt.hold_ms == HOLD_MS and mt.clear_pages == mt.pages_examined
        assert ei.value.mismatch.pages.pages == mt.pages_examined and mt.clear_bytes == ei.value.mismatch.mismatch_bytes
        assert ei.value.triage is None
        PGC.release_wait(lib)
        with pytest.raises(D.GpuError) as ei:
            gpu.scrub_and_verify(GiB, check="tagged")
        assert ei.value.mismatch_triage is None and D.last_mismatch_triage(0).triaged == 0
        PGC.release_wait(lib)
        reps, _ = D.scrub_and_verify_many([gpu], GiB, check="tagged", mismatch_triage=True, triage_hold_ms=HOLD_MS)
        assert reps[0].mismatch_triage is not None
        assert reps[0].mismatch_triage.pages_examined == reps[0].mismatch.pages.pages
        PGC.release_wait(lib)
        js = scrub_worker.run([gpu.bdf], GiB, "tagged", mismatch_triage_hold_ms=HOLD_MS)["reports"][0]
        assert js["mismatch_triage"]["triaged"] == 1 and "triage" not in js
        PGC.release_wait(lib)
    finally:
        lib.ccm_sim_set(gpu.index, b"tag_inject", 0)
    rep = gpu.scrub_and_verify(GiB, check="tagged", mismatch_triage=True, triage_hold_ms=HOLD_MS)
    assert rep.clean and rep.mismatch_triage is None
    gpu.wait_scrub_released()
    # the worker in a child process: a clean tagged gate, armed, prints no report
    proc = subprocess.run([sys.executable, "-m", "k8s_cc_manager_b200.scrub_worker", "--backend", "cudasim", "--bdf",
                           gpu.bdf, "--bytes", str(GiB), "--check", "tagged", "--mismatch-triage"],
                          capture_output=True, text=True, timeout=300, cwd=str(ROOT),
                          env=dict(os.environ, PYTHONPATH=str(ROOT)))
    assert proc.returncode == 0, proc.stderr[-2000:]
    rep = json.loads(proc.stdout.strip().splitlines()[-1])["reports"][0]
    assert rep["status"] == 0 and rep["mismatch_bytes"] == 0 and "mismatch_triage" not in rep


def test_manager_transition_logs_the_alias_triage(lib, monkeypatch, caplog):
    import kubernetes
    from k8s_cc_manager_b200 import manager
    for k, v in dict(EVICT_OPERATOR_COMPONENTS="false", CC_RELEASE_CUDA_CONTEXT="false").items():
        monkeypatch.setenv(k, v)
    assert lib.ccm_init(N.BACKEND_CUDASIM) == 0
    lib.ccm_sim_set(-1, b"cc_mode", N.CC_MODES["off"])
    lib.ccm_sim_set(0, b"scrub_alias", 1)
    try:
        with PGC.knobs({}):
            c = kubernetes.reset_cluster()
            c.add_node(SC.NODE, {})
            mgr = manager.CCManager(SC.NODE, "on", True, device_source=D.find_gpus, scrub_bytes=4 * GiB,
                                    scrub_check="tagged", scrub_mismatch_triage="report")
            with caplog.at_level(logging.ERROR, logger="k8s-cc-manager"):
                assert mgr.set_cc_mode("on") is False
        bdf = next(d.bdf for d in D.find_gpus()[0] if d.cuda_ordinal == 0)
        assert mgr.last_transition["scrub_mismatch"][bdf].mismatch_windows == 2 * N0 // 16
        mt = mgr.last_transition["scrub_mismatch_triage"][bdf]
        assert mt.pages_examined == 2 * N0 // PAGE and mt.return_pages == 0 and mt.stay_pages >= N0 // PAGE
        msgs = [r.getMessage() for r in caplog.records]
        line = next(m for m in msgs if m.startswith(f"HBM mismatch triage on {bdf}: "))
        assert f"{2 * N0 // PAGE} pages in 1 runs" in line
        assert msgs.index(line) > msgs.index(next(m for m in msgs if m.startswith(f"HBM tag mismatch on {bdf}: ")))
    finally:
        lib.ccm_sim_set(0, b"scrub_alias", 0)
        for d in D.find_gpus()[0]:
            if d.is_gpu():
                d.wait_scrub_released()


# ------------------------------------------------------------------------------------------------------ PDL on and off
PDL_CASES = {
    "inject": (PATHS["vmm-mf0-il1"][1], {"tag_inject": PP.INJECT}, 0, 0),
    "inject-fallback": ({"CCM_PIPELINE": "0"}, {"tag_inject": PP.INJECT}, 0, 0),
    "stay-return": (PATHS["vmm-mf0-il1"][1], {"tag_inject": PP.INJECT}, 2, 3),
    "alias": (PP.mode_env(0, 1), {"scrub_alias": 1}, 0, 0),
    "flood": (PATHS["vmm-mf0-il1"][1], {"tag_flood": FLOOD}, 0, 0),
}


def pdl_record(out: dict) -> dict:
    """What a PDL case left, in JSON: the fields the two children must agree on, and what the oracle needs."""
    return {"rc": out["rc"], "launches": out["launches"], "bytes_scrubbed": out["res"].bytes_scrubbed,
            "segments": out["res"].segments, "device_free_before": out["res"].device_free_before,
            "mismatch_bytes": out["tag"].mismatch_bytes, "nonzero_bytes": out["res"].nonzero_bytes,
            "mm_pages": [list(e) for e in out["mm_pages"]],
            "mtriage": {f: getattr(out["mtriage"], f) for f, _ in N.TriageReport._fields_},
            "mtriage_pages": [[p.page, p.chunk, p.cls, p.dirt_bytes, p.t2_bytes, p.t3_bytes]
                              for p in out["mtriage_pages"]]}


def child() -> None:
    lib = PGC.open_lib()
    out = {}
    for name, (env, drills, stay, ret) in PDL_CASES.items():
        out[name] = pdl_record(call(lib, "tagged", env, {**drills, "triage_stay": stay, "triage_return": ret}, 4 * GiB,
                                    hold=HOLD_MS))
    print("RESULT " + json.dumps(out), flush=True)


def run_child(pdl: str) -> dict:
    proc = subprocess.run([sys.executable, str(Path(__file__).resolve())], capture_output=True, text=True, timeout=900,
                          cwd=str(ROOT), env=dict(os.environ, CCM_PDL=pdl))
    assert proc.returncode == 0, f"CCM_PDL={pdl}: exit {proc.returncode}\n{proc.stdout[-2000:]}\n{proc.stderr[-3000:]}"
    return json.loads(next(line for line in proc.stdout.splitlines() if line.startswith("RESULT "))[7:])


class _Res:
    def __init__(self, rec):
        self.bytes_scrubbed, self.segments = rec["bytes_scrubbed"], rec["segments"]
        self.device_free_before = rec["device_free_before"]


def test_pdl_on_and_off_agree_and_match_the_oracle(lib):
    got = {pdl: run_child(pdl) for pdl in ("1", "0")}
    for pdl, cases in got.items():
        for name, rec in cases.items():
            env, drills, stay, ret = PDL_CASES[name]
            entries = [tuple(e) for e in rec["mm_pages"]]
            what = (pdl, name)
            assert rec["rc"] == N.ERR_MISMATCH and rec["nonzero_bytes"] == 0, what
            t = rec["mtriage"]
            assert t["stay_bytes"] + t["return_bytes"] + t["clear_bytes"] == rec["mismatch_bytes"], what
            if name == "alias":   # memory that does not keep what is stored: the oracle does not apply
                assert t["return_pages"] == 0 and t["runs"] == 1 and t["bytes_examined"] == 2 * N0, what
                half = N0 // PAGE
                stays = {r[0] for r in rec["mtriage_pages"] if r[2] == "stays"}
                assert all(p in stays or p + half in stays for p in range(half)), what
                continue
            want = MTR.report(entries, spans(env, _Res(rec), 4 * GiB), stay, ret)
            for k, v in want.items():
                assert rec["mtriage"][k] == v, (what, k)
            assert [tuple(r) for r in rec["mtriage_pages"]] == MTR.classify(entries, stay, ret), what
            if name == "flood":
                assert t["clear_pages"] == t["pages_examined"] and t["t2_bytes"] == t["t3_bytes"] == 0, what
    on, off = got["1"], got["0"]
    assert set(on) == set(off) == set(PDL_CASES)
    for name in PDL_CASES:
        a, b = on[name], off[name]
        assert a["launches"] == b["launches"], name
        assert (a["rc"], a["bytes_scrubbed"], a["segments"]) == (b["rc"], b["bytes_scrubbed"], b["segments"]), name
        if name in ADDRESS_DEPENDENT:
            # which bytes differ from their tags depends on the addresses: compare the shape of the triage
            fields = ("runs", "pages_examined", "bytes_examined", "return_pages", "t3_bytes", "triaged", "hold_ms")
        else:
            assert {k: a[k] for k in ("mismatch_bytes", "mm_pages", "mtriage_pages")} == \
                {k: b[k] for k in ("mismatch_bytes", "mm_pages", "mtriage_pages")}, name
            fields = TRIAGE_FIELDS
        assert {f: a["mtriage"][f] for f in fields} == {f: b["mtriage"][f] for f in fields}, name


# cases whose mismatched bytes are tags compared with other addresses' tags or with a flood byte
ADDRESS_DEPENDENT = ("alias", "flood")


if __name__ == "__main__":
    child()
