"""The coverage proof on one H100: clean armed calls are covered on every mapping path and leave what unarmed calls
leave; the proof never changes another verdict under the fault drills; the fail-open of a pass that skips chunks
(cover_skip) returns CCM_OK unarmed and CCM_ERR_UNCOVERED armed, with the oracle's missing bytes and pages; and the
proving kernels' rates against the same run's unarmed ones.  Each case list runs in a child process
(tests/cover_proof_calls.py), once with CCM_PDL=1 and once with CCM_PDL=0."""
from __future__ import annotations

import json
import os
import statistics
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "tests"))
import cover_oracle as CO  # noqa: E402
import product_plan as PP  # noqa: E402
from k8s_cc_manager_b200 import _native as N  # noqa: E402

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

MiB, GiB = 1 << 20, 1 << 30
SAME = ("status", "nonzero_bytes", "release_deferred", "scrub_variant", "verify_variant")
ONE_RANGE = {"CCM_MAP_FIRST": "1", "CCM_INTERLEAVE_VERIFY": "1"}


def clean_cases() -> list[dict]:
    """(name, call) pairs run unarmed, then armed."""
    cases = []
    for mf, il in PP.MODES:
        cases.append(("vmm", {"bytes": 1536 * MiB, "env": PP.mode_env(mf, il)}))
    for tail in PP.TAIL_MBS:
        cases.append(("whole", {"bytes": 0, "env": {"CCM_VMM_TAIL_MB": str(tail)}}))
    for n, seg in ((64 * MiB + 12345, 0), (10 * MiB + 777, 3), (5 * MiB + 16 * 9 + 5, 2)):
        env = {"CCM_PIPELINE": "0", **({"CCM_ARENA_MAX_SEGMENT_MB": str(seg)} if seg else {})}
        cases.append(("fallback", {"bytes": n, "env": env}))
    cases.append(("fanout", {"bytes": GiB, "many": 2}))
    cases.append(("pinned", {"bytes": 1536 * MiB, "env": {"CCM_SCRUB_VARIANT": "memset", "CCM_VERIFY_VARIANT": "ld256"}}))
    for kind in ("tagged", "census", "census_tagged"):
        cases.append((kind, {"bytes": 1536 * MiB, "kind": kind}))
        cases.append((kind, {"bytes": 10 * MiB + 777, "kind": kind, "env": {"CCM_PIPELINE": "0", "CCM_ARENA_MAX_SEGMENT_MB": "3"}}))
    return cases


def drill_cases() -> list[dict]:
    return [
        {"bytes": 1536 * MiB, "drill": {"scrub_inject": 1000}},
        {"bytes": 1536 * MiB, "drill": {"scrub_flood": PP.FLOOD}},
        {"bytes": 1536 * MiB, "drill": {"scrub_poison": PP.POISON}},
        {"bytes": 1536 * MiB, "kind": "tagged", "drill": {"tag_inject": 7}},
        {"bytes": 2 * GiB, "kind": "tagged", "drill": {"scrub_alias": 1}},
        {"bytes": 1536 * MiB, "kind": "census", "drill": {"scrub_residue": 9}},
        {"bytes": 10 * MiB + 777, "drill": {"scrub_inject": 1000}, "env": {"CCM_PIPELINE": "0", "CCM_ARENA_MAX_SEGMENT_MB": "3"}},
        {"bytes": 1536 * MiB, "drill": {"scrub_inject": 1000}, "triage": 5},
        {"bytes": 1536 * MiB, "kind": "tagged", "drill": {"tag_inject": 7}, "triage": 5, "mismatch_triage": 5},
        {"bytes": 1536 * MiB, "kind": "census", "drill": {"scrub_residue": 9, "scrub_inject": 3}, "triage": 5},
    ]


SKIP_BYTES = 256 * MiB
TWO_RANGES = {"CCM_MAP_FIRST": "0", "CCM_INTERLEAVE_VERIFY": "0"}    # a 1 GiB and a 512 MiB range, one read-back
FALLBACK = {"CCM_PIPELINE": "0", "CCM_ARENA_MAX_SEGMENT_MB": "3"}   # 3 MiB segments, the last one ragged
# (kind, cover_pass, k, bytes, env): the drilled pass of a call
SKIPS = [("zero", 3, SKIP_BYTES // CO.CHUNK, SKIP_BYTES, ONE_RANGE), ("zero", 3, 3, SKIP_BYTES, ONE_RANGE),
         ("zero", 0, 5, SKIP_BYTES, ONE_RANGE), ("zero", 1, 3, SKIP_BYTES, ONE_RANGE),
         ("tagged", 2, 3, SKIP_BYTES, ONE_RANGE), ("tagged", 1, 2, SKIP_BYTES, ONE_RANGE),
         ("census", 1, 4, SKIP_BYTES, ONE_RANGE),
         ("zero", 3, 3, 1536 * MiB, TWO_RANGES), ("zero", 1, 7, 1536 * MiB, TWO_RANGES),
         ("tagged", 1, 3, 1536 * MiB, ONE_RANGE), ("tagged", 2, 2, 1536 * MiB, TWO_RANGES),
         ("zero", 3, 5, 10 * MiB + 777, FALLBACK), ("zero", 1, 2, 10 * MiB + 777, FALLBACK),
         ("tagged", 2, 3, 10 * MiB + 777, FALLBACK)]


def skip_cases() -> list[dict]:
    out = []
    for kind, pass_, k, nbytes, env in SKIPS:
        drill = {"cover_skip": k, "cover_pass": pass_}
        if k == SKIP_BYTES // CO.CHUNK:
            drill["scrub_inject"] = 4   # all four candidates of the range lie in chunks the read-back skips
        out.append({"bytes": nbytes, "env": env, "kind": kind, "drill": drill})
    return out


def calls(rates: bool) -> list[dict]:
    out = []
    for _, c in clean_cases():
        out += [dict(c, prove=0), dict(c, prove=1)]
    for c in drill_cases():
        out += [dict(c, prove=0), dict(c, prove=1)]
    for c in skip_cases():
        # unarmed, armed, then a clean armed call: a grab word left non-zero would make it short
        out += [dict(c, prove=0), dict(c, prove=1), {"bytes": c["bytes"], "env": c["env"], "kind": c["kind"], "prove": 1}]
    if rates:
        for _ in range(3):
            for kind in ("zero", "tagged"):
                out += [{"bytes": 0, "kind": kind, "prove": 0, "rate": 1}, {"bytes": 0, "kind": kind, "prove": 1, "rate": 1}]
    return out


def run_child(pdl: str, rates: bool) -> list[dict]:
    env = dict(os.environ, CCM_PDL=pdl)
    proc = subprocess.run([sys.executable, str(ROOT / "tests" / "cover_proof_calls.py"), json.dumps(calls(rates))],
                          capture_output=True, text=True, env=env, cwd=ROOT, timeout=1800)
    assert proc.returncode == 0, proc.stdout[-4000:] + proc.stderr[-4000:]
    line = [x for x in proc.stdout.splitlines() if x.startswith("RESULT ")][-1]
    return json.loads(line[len("RESULT "):])


@pytest.fixture(scope="module", params=["1", "0"], ids=["pdl", "nopdl"])
def results(request):
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return request.param, run_child(request.param, rates=request.param == "0")


def assert_covered(r: dict, what):
    cov, res = r["cover"], r["results"]
    tagged = r["call"].get("kind", "zero") in ("tagged", "census_tagged")
    assert cov["proved"] == 1 and cov["covered"] == 1, (what, r["error"], cov)
    assert cov["bytes_mapped"] == res[-1]["bytes_scrubbed"] or r["call"].get("many"), what
    for name in CO.PASSES:
        p = cov["passes"][name]
        assert p["ran"] == (1 if name != "check" or tagged else 0), (what, name)
        if p["ran"]:
            assert p["bytes_counted"] == cov["bytes_mapped"], (what, name, p)
            assert p["bytes_missing"] == p["bytes_extra"] == p["bytes_outside"] == p["pages_short"] == 0, (what, p)
    assert r["pages"] == [], what
    assert all(x["scrub_variant"] == N.SCRUB_ST128 and x["verify_variant"] == N.VERIFY_LD128 for x in res), what


def settled(report, key: str):
    """A dirt or mismatch report without its records when more windows were booked than the 64 records hold: which
    windows win the record slots then depends on the order the CTAs reach them, in an armed and an unarmed call alike."""
    if key in ("dirt", "mismatch") and report[1] > 64:
        return report[:6]
    return report


def pairs(rs: list[dict], n: int, start: int = 0):
    return [(rs[start + 2 * i], rs[start + 2 * i + 1]) for i in range(n)]


def test_clean_armed_calls_are_covered_and_leave_what_unarmed_calls_leave(results):
    pdl, rs = results
    cases = clean_cases()
    for (name, _), (off, on) in zip(cases, pairs(rs, len(cases))):
        what = (pdl, name, on["call"])
        assert off["rc"] == on["rc"] == 0, (what, off["error"], on["error"])
        assert_covered(on, what)
        assert off["cover"]["proved"] == 0 and off["pages"] == [], what
        for a, b in zip(off["results"], on["results"]):
            same = SAME if name != "pinned" else ("status", "nonzero_bytes", "release_deferred")
            assert {k: a[k] for k in same} == {k: b[k] for k in same}, what
            if name != "whole":
                assert (a["bytes_scrubbed"], a["segments"]) == (b["bytes_scrubbed"], b["segments"]), what
        if name not in ("whole", "pinned"):   # whole HBM: the two calls map a granule apart; pinned: other kernels
            assert off["launches"] == on["launches"], what
        assert on["reports"] == off["reports"] or name == "whole", what
        for key in ("tags", "residue"):
            if key in off:
                strip = [{k: v for k, v in x.items() if not k.startswith("ms_")} for x in off[key]]
                assert strip == [{k: v for k, v in x.items() if not k.startswith("ms_")} for x in on[key]], what


def test_the_proof_never_changes_another_verdict(results):
    pdl, rs = results
    start = 2 * len(clean_cases())
    for off, on in pairs(rs, len(drill_cases()), start):
        what = (pdl, on["call"])
        assert off["rc"] == on["rc"] and off["rc"] in (0, N.ERR_DIRTY, N.ERR_MISMATCH), (what, off["error"], on["error"])
        assert on["cover"]["covered"] == 1 and on["pages"] == [], (what, on["cover"], on["pages"][:4])
        assert [x["nonzero_bytes"] for x in off["results"]] == [x["nonzero_bytes"] for x in on["results"]], what
        assert [x["bytes_scrubbed"] for x in off["results"]] == [x["bytes_scrubbed"] for x in on["results"]], what
        # the aliased view's mismatch count depends on the call's random tag seed; every other count is exact
        seeded = on["call"].get("drill", {}).get("scrub_alias")
        for key in ("tags", "residue"):
            if key in off and not seeded:
                strip = [{k: v for k, v in x.items() if not k.startswith("ms_")} for x in off[key]]
                assert strip == [{k: v for k, v in x.items() if not k.startswith("ms_")} for x in on[key]], what
        # every report, page map and triage the unarmed call left (the aliased call's mismatch records carry its tags)
        for key, value in off["reports"].items():
            if not (seeded and key in ("mismatch", "pages2")):
                assert settled(on["reports"][key], key) == settled(value, key), (what, key)
        assert off["launches"] == on["launches"], (what, off["launches"], on["launches"])


def test_a_skipped_pass_fails_closed_only_when_armed(results):
    pdl, rs = results
    start = 2 * len(clean_cases()) + 2 * len(drill_cases())
    for i, (kind, pass_, k, nbytes, env) in enumerate(SKIPS):
        off, on, after = rs[start + 3 * i: start + 3 * i + 3]
        what = (pdl, kind, pass_, k, nbytes, env)
        name = CO.DRILL_PASS[pass_]
        ranges, mappings, interleave, mapped = CO.call_launches(nbytes, env)
        assert on["results"][0]["bytes_scrubbed"] == mapped, what
        tagged = kind == "tagged"
        drilled = CO.first_launch(name, tagged, ranges, mappings, interleave, mapped)
        want = CO.report(mapped, tagged, (name, k, *drilled))
        if name == "readback" and k == SKIP_BYTES // CO.CHUNK:
            # the fail-open, pinned: every dirty byte lies in a chunk the read-back never reads
            assert off["rc"] == 0 and off["results"][0]["nonzero_bytes"] == 0, what
        if name == "check":
            assert off["rc"] == N.ERR_DIRTY, what   # the skipped chunks keep their tags
        assert on["rc"] == N.ERR_UNCOVERED, (what, on["error"])
        assert "coverage proof failed" in on["error"] and f"first short page {want['passes'][name]['first_short_page']}" \
            in on["error"], (what, on["error"])
        cov = on["cover"]
        assert cov["proved"] == 1 and cov["covered"] == 0, what
        for p in CO.PASSES:
            for f, v in want["passes"][p].items():
                assert cov["passes"][p][f] == v, (what, p, f, cov["passes"][p])
        got_pages = [{k2: v for k2, v in pg.items() if k2 != "chunk"} for pg in on["pages"]]
        assert got_pages == want["pages"], what
        # the result apart from the status: what the unarmed call left (after a skipped check: the tags of the
        # skipped chunks, whose non-zero bytes depend on each call's random seed)
        if name == "check":
            assert 0 < on["results"][0]["nonzero_bytes"] <= k * CO.CHUNK, what
        else:
            assert on["results"][0]["nonzero_bytes"] == off["results"][0]["nonzero_bytes"], what
        assert after["rc"] == 0 and after["cover"]["covered"] == 1, (what, after["error"])


def test_armed_kernels_keep_their_rates(results):
    pdl, rs = results
    if pdl != "0":
        pytest.skip("rates are measured in the child without PDL")
    rate = [r for r in rs if r["call"].get("rate")]
    for kind in ("zero", "tagged"):
        for field in ("ms_scrub", "ms_verify"):
            off = statistics.median(r["results"][0]["bytes_scrubbed"] / r["results"][0][field] for r in rate
                                    if r["call"]["kind"] == kind and not r["call"]["prove"])
            on = statistics.median(r["results"][0]["bytes_scrubbed"] / r["results"][0][field] for r in rate
                                   if r["call"]["kind"] == kind and r["call"]["prove"])
            assert on >= 0.85 * off, (kind, field, on, off)
        if kind == "tagged":
            off = statistics.median(r["results"][0]["bytes_scrubbed"] / r["tags"][0]["ms_tag"] for r in rate
                                    if r["call"]["kind"] == kind and not r["call"]["prove"])
            on = statistics.median(r["results"][0]["bytes_scrubbed"] / r["tags"][0]["ms_tag"] for r in rate
                                   if r["call"]["kind"] == kind and r["call"]["prove"])
            assert on >= 0.85 * off, ("ms_tag", on, off)
    for r in rate:
        if r["call"]["prove"]:
            assert r["rc"] == 0 and r["cover"]["covered"] == 1, r["error"]
