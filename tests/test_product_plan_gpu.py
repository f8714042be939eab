"""The product scrub gate against its plan (-m gpu, run on an H100).

Every case runs four product calls — clean, poison (the previous tenant's data in every chunk before the
scrub), flood (every enqueued range refilled between its scrub and its read-back) and inject = 1000 — and
compares rc, nonzero_bytes, segments, bytes_scrubbed, bytes_unreached and device_free_before with
tests/product_plan.py.  Flood proves the read-back counts every byte the call reports as scrubbed; poison
proves the scrub zeroes everything the read-back reads; so every byte of [0, bytes_scrubbed) is scrubbed.

A. requested sizes around the granularity and the chunk sizes, under six chunk settings, all four
   CCM_MAP_FIRST x CCM_INTERLEAVE_VERIFY modes and both release modes (more than 32 chunks included);
B. whole HBM under the four modes and CCM_VMM_TAIL_MB 256, 2 and 0;
C. every CCM_SCRUB_VARIANT x CCM_VERIFY_VARIANT pin at whole HBM with map-first, in a fresh process, so the
   pinned kernels are first launched with all HBM mapped;
D. the arena fallback (CCM_PIPELINE=0);
E. ccm_scrub_verify_many's fan-out default (map first) on one GPU;
F. a 51-chunk and a whole-HBM call with and without programmatic dependent launch, in child processes.
"""
from __future__ import annotations

import json
import subprocess
import sys
import time
from pathlib import Path

import pytest

import product_gate_calls as G
import product_plan as PP
from k8s_cc_manager_b200 import _native as N

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parents[1]
MiB, GiB = PP.MiB, PP.GiB
FREE_SLACK = 64 * MiB        # free HBM must come back to where it was, within this
DRILLS = tuple(PP.DRILLS)


@pytest.fixture(scope="module")
def lib():
    if "torch" in sys.modules:           # memory cached by earlier tests in this process is not "free"
        sys.modules["torch"].cuda.empty_cache()
    return G.open_lib()


@pytest.fixture(scope="module")
def gran(lib):
    """The allocation granularity, as the product call reports it: a 1-byte call maps one granule."""
    rec = G.call(lib, 1, {})
    G.release_wait(lib)
    assert rec["rc"] == 0, rec
    g = rec["results"][0]["bytes_scrubbed"]
    assert g > 0 and g & (g - 1) == 0, g
    assert g == PP.H100_GRAN, f"granularity {g}, the header documents 2 MiB on H100"
    return g


@pytest.fixture(scope="module")
def free0(lib, gran):
    """Free HBM at the start, as the product call sees it."""
    rec = G.call(lib, 1, {})
    G.release_wait(lib)
    return rec["results"][0]["device_free_before"]


def check(rec: dict, gran: int, free0: int, fanout: bool = False) -> list:
    """Problems of one call record against the model ([] = exact)."""
    env, nbytes, drill = rec["env"], rec["bytes"], rec["drill"]
    bad = []

    def expect(what, got, want):
        if got != want:
            bad.append((what, got, want))

    for r in rec["results"]:
        mapped, free = r["bytes_scrubbed"], r["device_free_before"]
        if free < free0 - FREE_SLACK or free > r["device_total_bytes"]:
            bad.append(("device_free_before", free, free0))
        if PP.env_u64(env, "CCM_PIPELINE", 1) == 0:
            segs = PP.arena_segments(nbytes, free, env)
            if nbytes or r["segments"] == 1:
                expect("bytes_scrubbed", mapped, sum(n for _, n in segs))
                expect("segments", r["segments"], len(segs))
            ranges = segs if nbytes or r["segments"] == 1 else [(0, 64 * MiB)] * r["segments"]  # each >= 64 MiB
        else:
            p = PP.plan(nbytes, free, gran, env, node_fanout=fanout)
            if nbytes:
                run = PP.simulate(p, None)
                expect("bytes_scrubbed", mapped, p.va_bytes)
                expect("segments", r["segments"], len(run.chunks))
                ranges = run.ranges(p)
            else:
                if mapped % gran or mapped > p.va_bytes or mapped == 0:
                    bad.append(("bytes_scrubbed", mapped, p.va_bytes))
                    continue
                run = PP.simulate(p, mapped)
                if mapped >= p.main_end:
                    # the tail zone took the out-of-memory: main zone exact, tail granules bounded
                    expect("main zone", run.main, p.main)
                    tail = mapped - run.main_end
                    n_tail = r["segments"] - len(run.main)
                    if not len(run.tail) <= n_tail <= tail // gran:
                        bad.append(("tail segments", n_tail, (len(run.tail), tail // gran)))
                elif r["segments"] < 1:
                    bad.append(("segments", r["segments"], ">= 1"))
                # map first: one range whatever the split; otherwise the split is the driver's once
                # the main zone itself ran out of memory (small tail zone)
                ranges = run.ranges(p) if p.map_first or mapped >= p.main_end else None
        count = r["nonzero_bytes"]
        if ranges is None:
            want = PP.expected_count(drill, [(0, mapped)], mapped)
            if drill == "inject":
                if count % 4 or not 4 <= count <= 4 * r["segments"]:
                    bad.append(("inject count", count, f"4 x ranges, ranges <= {r['segments']}"))
                want = count
        else:
            want = PP.expected_count(drill, ranges, mapped)
        expect("nonzero_bytes", count, want)
        expect("status", r["status"], N.ERR_DIRTY if want else 0)
        expect("bytes_unreached", r["bytes_unreached"], max(free - mapped, 0) if nbytes == 0 else 0)
    want_rc = N.ERR_DIRTY if any(r["status"] for r in rec["results"]) else 0
    expect("rc", rec["rc"], want_rc)
    return bad


def run_cases(lib, cases, gran, free0, fanout=False, many=0):
    """Runs every (bytes, env) case under every drill; returns (failures, records)."""
    failures, recs = [], []
    for nbytes, env in cases:
        for drill in DRILLS:
            rec = G.call(lib, nbytes, env, drill, many)
            recs.append(rec)
            bad = check(rec, gran, free0, fanout)
            if bad:
                failures.append((nbytes, env, drill, rec["rc"], rec["error"][:200], bad))
    G.release_wait(lib)
    return failures, recs


def assert_free_back(lib, free0):
    G.release_wait(lib)
    rec = G.call(lib, 1, {})
    G.release_wait(lib)
    assert rec["results"][0]["device_free_before"] >= free0 - FREE_SLACK, "HBM was not handed back"


# --------------------------------------------------------------------------------- A. requested sizes
@pytest.mark.parametrize("setting", PP.CHUNK_SETTINGS, ids=lambda s: "default" if s is None else f"{s[0]}-{s[1]}MB")
def test_requested_sizes_match_the_plan(lib, gran, free0, setting):
    cases = PP.requested_cases(setting, gran)
    t0 = time.perf_counter()
    failures, recs = run_cases(lib, cases, gran, free0)
    assert not failures, f"{len(failures)} of {len(recs)} calls off the plan, first: {failures[:5]}"
    most = max(r["results"][0]["segments"] for r in recs)
    print(f"\nrequested sizes {setting}: {len(recs)} calls exact, up to {most} chunks, {time.perf_counter() - t0:.1f} s")
    assert_free_back(lib, free0)


# --------------------------------------------------------------------------------- B. whole HBM
@pytest.mark.parametrize("tail_mb", PP.TAIL_MBS)
def test_whole_hbm_gate_scrubs_and_counts_every_mapped_byte(lib, gran, free0, tail_mb):
    cases = [(0, env) for env in PP.whole_hbm_cases(tail_mb)]
    failures, recs = run_cases(lib, cases, gran, free0)
    assert not failures, f"{len(failures)} of {len(recs)} calls off the plan, first: {failures[:5]}"
    for rec in recs:
        r = rec["results"][0]
        assert r["bytes_scrubbed"] / r["device_total_bytes"] >= 0.99, rec
        if rec["drill"] == "flood":
            assert r["nonzero_bytes"] == r["bytes_scrubbed"] > 1 << 32
    assert_free_back(lib, free0)
    cov = min(r["results"][0]["bytes_scrubbed"] / r["results"][0]["device_total_bytes"] for r in recs)
    print(f"\nwhole HBM, tail {tail_mb} MiB: {len(recs)} calls exact, coverage >= {100 * cov:.2f} %")


# --------------------------------------------------------------------------------- children
def run_child(calls: list, env_extra: dict) -> tuple[list, int]:
    """Runs `calls` in a fresh process; returns the records and the free HBM the child's first call saw
    (this process keeps its own CUDA context, so the child sees less than free0)."""
    import os
    env = dict(os.environ, **env_extra)
    proc = subprocess.run([sys.executable, str(ROOT / "tests" / "product_gate_calls.py"), json.dumps(calls)],
                          capture_output=True, text=True, env=env, timeout=300, cwd=str(ROOT))
    assert proc.returncode == 0, f"{env_extra}: exit {proc.returncode}\n{proc.stdout[-2000:]}\n{proc.stderr[-3000:]}"
    recs = json.loads(next(l for l in proc.stdout.splitlines() if l.startswith("RESULT "))[7:])
    return recs, recs[0]["results"][0]["device_free_before"]


def reaches_all_free(r: dict) -> bool:
    return r["bytes_unreached"] <= 16 * MiB and r["bytes_scrubbed"] > 0


# --------------------------------------------------------------------------------- C. variant pins
def test_variant_pins_first_launched_with_all_hbm_mapped(lib, gran, free0):
    """Each pair in a fresh process, map first: its kernels' first launch finds every granule mapped."""
    failures, seen = [], []
    for sv, vv in PP.VARIANT_PINS:
        env = PP.variant_pin_env(sv, vv)
        recs, child_free = run_child([{"bytes": 0, "env": env, "drill": d} for d in ("clean", "flood")], {})
        for rec in recs:
            r = rec["results"][0]
            seen.append(f"{sv}/{vv} {rec['drill']}: rc {rec['rc']}, {r['bytes_scrubbed']} scrubbed, "
                        f"{r['nonzero_bytes']} counted")
            bad = check(rec, gran, child_free)
            if (r["scrub_variant"], r["verify_variant"]) != (N.SCRUB_VARIANTS[sv], N.VERIFY_VARIANTS[vv]):
                bad.append(("variants", (r["scrub_variant"], r["verify_variant"]), (sv, vv)))
            if not reaches_all_free(r):
                bad.append(("unreached", r["bytes_unreached"], r["device_free_before"]))
            if bad:
                failures.append((sv, vv, rec["drill"], rec["rc"], rec["error"][:200], bad))
    print("\n" + "\n".join(seen))
    assert not failures, failures
    assert_free_back(lib, free0)


# --------------------------------------------------------------------------------- D. arena fallback
def test_arena_fallback_honours_every_drill(lib, gran, free0):
    failures, recs = run_cases(lib, PP.arena_cases(gran), gran, free0)
    assert not failures, f"{len(failures)} of {len(recs)} calls off the plan, first: {failures[:5]}"
    segs = {(rec["bytes"], rec["env"].get("CCM_ARENA_MAX_SEGMENT_MB")): rec["results"][0]["segments"] for rec in recs}
    assert segs[(300 * MiB, "96")] == 4 and segs[(gran + 1, None)] == 1
    for rec in recs:
        if rec["drill"] == "inject":
            assert rec["results"][0]["nonzero_bytes"] == 4 * rec["results"][0]["segments"]
    whole = [rec["results"][0] for rec in recs if rec["bytes"] == 0 and rec["drill"] == "clean"]
    print("\narena fallback, whole HBM: " + ", ".join(
        f"{r['segments']} segment(s), coverage {100 * r['bytes_scrubbed'] / r['device_total_bytes']:.2f} %"
        for r in whole))
    assert_free_back(lib, free0)


# --------------------------------------------------------------------------------- E. fan-out default
def test_fanout_default_maps_first_on_one_gpu(lib, gran, free0):
    cases = [(b, {}) for b in PP.FANOUT_SIZES]
    failures, recs = run_cases(lib, cases, gran, free0, fanout=True, many=2)
    assert not failures, f"{len(failures)} of {len(recs)} calls off the plan, first: {failures[:5]}"
    for rec in recs:
        assert len(rec["results"]) == 2
        if rec["drill"] == "inject":                     # map first: one range per call
            assert [r["nonzero_bytes"] for r in rec["results"]] == [4, 4]
    assert_free_back(lib, free0)


# --------------------------------------------------------------------------------- F. PDL
def test_pdl_children_report_identical_exact_results(lib, gran, free0):
    calls = [{"bytes": b, "env": env, "drill": d} for b, env in PP.pdl_cases() for d in DRILLS]
    runs = {pdl: run_child(calls, {"CCM_PDL": pdl}) for pdl in PP.PDL_VALUES}
    outs = {pdl: recs for pdl, (recs, _) in runs.items()}
    failures = []
    for pdl, (recs, child_free) in runs.items():
        for rec in recs:
            bad = check(rec, gran, child_free)
            if rec["bytes"] == 0 and not reaches_all_free(rec["results"][0]):
                bad.append(("unreached", rec["results"][0]["bytes_unreached"], 16 * MiB))
            if bad:
                failures.append((pdl, rec["bytes"], rec["drill"], rec["rc"], rec["error"][:200], bad))
    assert not failures, failures

    def outcome(rec):
        r = rec["results"][0]
        key = (rec["rc"], r["status"], r["nonzero_bytes"] == r["bytes_scrubbed"] if rec["drill"] == "flood"
               else r["nonzero_bytes"])
        return key + ((r["bytes_scrubbed"], r["segments"]) if rec["bytes"] else ())

    a, b = ([outcome(r) for r in outs[p]] for p in PP.PDL_VALUES)
    assert a == b, (a, b)
    assert max(r["results"][0]["segments"] for r in outs["1"]) > 32
    assert_free_back(lib, free0)
