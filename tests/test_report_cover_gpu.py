"""The report proof on one H100: a proven call that fails runs the proving twins of its locate pass and triage steps,
launches and leaves exactly what the unproven call does, and counts every byte of every step; a clean proven call
proves nothing; the fail-open of a T3 that skips the run of a page that dirtied again (report_skip) classes it CLEARS
in both calls, and only the proven one names the missing bytes and pages the oracle predicts; every step can be drilled,
and the next call over the same kernels is exact again; and the locate twin's rate against the plain kernel's.  Each
case list runs in a child process (tests/report_cover_calls.py), once with CCM_PDL=1 and once with CCM_PDL=0."""
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
import product_plan as PP  # noqa: E402
import report_cover_oracle as RO  # noqa: E402
from k8s_cc_manager_b200 import _native as N  # noqa: E402

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

MiB, GiB = 1 << 20, 1 << 30
FALLBACK = {"CCM_PIPELINE": "0", "CCM_ARENA_MAX_SEGMENT_MB": "3"}   # 3 MiB segments, the last one ragged
TRIAGE_FIELDS = [f for f, _ in N.TriageReport._fields_ if not f.startswith("ms_") and f != "va_base"]
DIRT_STEPS = ("LOCATE", "DIRT_T1", "DIRT_T2", "DIRT_T3")
MISMATCH_STEPS = ("MISMATCH_T1", "MISMATCH_T2", "MISMATCH_T3")


def drill_cases() -> list[dict]:
    """Failed calls, run unproven then proven."""
    return [
        {"bytes": 1536 * MiB, "drill": {"scrub_inject": 1000}},
        {"bytes": 1536 * MiB, "drill": {"scrub_flood": PP.FLOOD}},
        {"bytes": 1536 * MiB, "drill": {"scrub_inject": 1000}, "triage": 5},
        {"bytes": 1536 * MiB, "drill": {"scrub_flood": PP.FLOOD}, "triage": 5},
        {"bytes": 1536 * MiB, "kind": "tagged", "drill": {"tag_inject": 7}, "triage": 5, "mismatch_triage": 5},
        {"bytes": 1536 * MiB, "kind": "census", "drill": {"scrub_residue": 9, "scrub_inject": 3}, "triage": 5},
        {"bytes": 10 * MiB + 777, "drill": {"scrub_inject": 1000}, "env": FALLBACK, "triage": 5},
        {"bytes": 10 * MiB + 777, "kind": "tagged", "drill": {"tag_inject": 7}, "env": FALLBACK, "mismatch_triage": 5},
        {"bytes": 2 * GiB, "kind": "tagged", "drill": {"scrub_alias": 1}, "mismatch_triage": 5},
        {"bytes": GiB, "many": 2, "drill": {"scrub_inject": 1000}, "triage": 5},
        {"bytes": 1536 * MiB, "probe": 1, "drill": {"probe_dirt": 3}, "triage": 5},
    ]


CLEAN = [{"bytes": 1536 * MiB}, {"bytes": 1536 * MiB, "kind": "tagged", "mismatch_triage": 5},
         {"bytes": 10 * MiB + 777, "env": FALLBACK, "triage": 5}]

# The fail-open, pinned: the first dirt page's first byte dirtied again between T2 and T3, and T3's first launch (the
# run holding it) skips its first chunk.
FAIL_OPEN = {"bytes": 1536 * MiB, "drill": {"scrub_inject": 4, "triage_return": 1, "report_skip": 1}, "triage": 5}

# (step, call) of every drilled step; report_skip = 2 chunks of its first launch
DIRT = {"bytes": 1536 * MiB, "drill": {"scrub_inject": 1000}, "triage": 5}
MISMATCH = {"bytes": 1536 * MiB, "kind": "tagged", "drill": {"tag_inject": 7}, "mismatch_triage": 5}
STEP_SKIPS = [(s, DIRT) for s in DIRT_STEPS] + [(s, MISMATCH) for s in MISMATCH_STEPS] + [
    ("LOCATE", {"bytes": 10 * MiB + 777, "drill": {"scrub_inject": 1000}, "env": FALLBACK, "triage": 5}),
    ("DIRT_T2", {"bytes": 10 * MiB + 777, "drill": {"scrub_inject": 1000}, "env": FALLBACK, "triage": 5})]
SKIP_K = 2


def with_drill(c: dict, **drill) -> dict:
    return dict(c, drill={**c.get("drill", {}), **drill})


def calls(rates: bool) -> list[dict]:
    out = []
    for c in drill_cases() + CLEAN:
        out += [dict(c, prove=0), dict(c, prove=1)]
    out += [dict(FAIL_OPEN, prove=0), dict(FAIL_OPEN, prove=1)]
    for step, c in STEP_SKIPS:
        drilled = with_drill(c, report_skip=SKIP_K, report_skip_step=RO.STEPS.index(step) + 1)
        # unproven, proven, then the same call proven without the drill: a grab word left non-zero would make it short
        out += [dict(drilled, prove=0), dict(drilled, prove=1), dict(c, prove=1)]
    if rates:
        for _ in range(3):
            for drill in ({"scrub_inject": 4}, {"scrub_flood": PP.FLOOD}):
                out += [{"bytes": 0, "drill": drill, "prove": p, "rate": 1} for p in (0, 1)]
    return out


def run_child(pdl: str, rates: bool) -> list[dict]:
    env = dict(os.environ, CCM_PDL=pdl)
    proc = subprocess.run([sys.executable, str(ROOT / "tests" / "report_cover_calls.py"), json.dumps(calls(rates))],
                          capture_output=True, text=True, env=env, cwd=ROOT, timeout=1800)
    assert proc.returncode == 0, proc.stdout[-4000:] + proc.stderr[-4000:]
    line = [x for x in proc.stdout.splitlines() if x.startswith("RESULT ")][-1]
    return json.loads(line[len("RESULT "):])


@pytest.fixture(scope="module", params=["1", "0"], ids=["pdl", "nopdl"])
def results(request):
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return request.param, run_child(request.param, rates=request.param == "0")


def triage(r: dict, fn: str) -> dict:
    return dict(zip(TRIAGE_FIELDS, r["reports"][fn]))


def spans(r: dict) -> list[tuple[int, int]]:
    """(offset, bytes) of what the call held: the mapping, or the fallback's segments."""
    c, mapped = r["call"], r["results"][-1]["bytes_scrubbed"]
    if c.get("env", {}).get("CCM_PIPELINE") == "0":
        seg = int(c["env"]["CCM_ARENA_MAX_SEGMENT_MB"]) * MiB
        return [(o, min(seg, mapped - o)) for o in range(0, mapped, seg)]
    return [(0, mapped)]


def ran_steps(r: dict) -> set:
    out = set()
    if r["reports"]["dirt"][5]:   # located
        out.add("LOCATE")
    if triage(r, "ccm_scrub_last_triage")["triaged"]:
        out |= {"DIRT_T1", "DIRT_T2", "DIRT_T3"}
    if triage(r, "ccm_scrub_last_mismatch_triage")["triaged"]:
        out |= set(MISMATCH_STEPS)
    return out


def assert_exact(r: dict, what) -> None:
    """Every step the call ran counted exactly what the oracle says it walks, and no other step ran."""
    rc_ = r["report_cover"]
    ran = ran_steps(r)
    assert rc_["proved"] == 1 and rc_["covered"] == 1 and rc_["pages"] == [], (what, rc_)
    dirt_pages = [tuple(p) for p in r["reports"]["pages1"]]
    mismatch_pages = [tuple(p) for p in r["reports"]["pages2"]]
    for name in RO.STEPS:
        s = rc_["steps"][name]
        assert s["ran"] == (name in ran), (what, name, s)
        if not s["ran"]:
            continue
        want = RO.step_report(RO.pieces(name, spans(r), dirt_pages, mismatch_pages))
        del want["pages"]
        assert {k: s[k] for k in want} == want, (what, name, s, want)
        if name == "LOCATE":
            assert s["bytes_expected"] == r["results"][-1]["bytes_scrubbed"], what
        else:
            t = triage(r, "ccm_scrub_last_triage" if name.startswith("DIRT") else "ccm_scrub_last_mismatch_triage")
            assert s["bytes_expected"] == t["bytes_examined"] and s["launches"] == t["runs"], (what, name, s, t)


def settled(report, key: str):
    """As test_cover_proof_gpu.settled: a dirt or mismatch report without its records past the 64 it holds."""
    if key in ("dirt", "mismatch") and report[1] > 64:
        return report[:6]
    return report


def assert_same(off: dict, on: dict, what, tags_seeded: bool = False) -> None:
    """The proven call returned, launched and left what the unproven one did.  Counts that depend on each call's random
    tag seed are left out: the aliased view's mismatch, and (tags_seeded: a mismatch triage whose T1 or T2 skipped
    chunks, so that T2 or T3 reads tags) the mismatch triage's bytes; the classes of its pages still match."""
    seeded = on["call"].get("drill", {}).get("scrub_alias")
    assert off["rc"] == on["rc"], (what, off["error"], on["error"])
    assert off["error"] == on["error"] or seeded, what
    assert off["launches"] == on["launches"], (what, off["launches"], on["launches"])
    assert [x["nonzero_bytes"] for x in off["results"]] == [x["nonzero_bytes"] for x in on["results"]], what
    assert off["report_cover"]["proved"] == 0 and off["report_cover"]["pages"] == [], what
    triage_keys = ("ccm_scrub_last_mismatch_triage", "ccm_last_mismatch_triage_pages")
    skip = (("mismatch", "pages2") + triage_keys if seeded else ()) + (triage_keys if tags_seeded else ())
    for key, value in off["reports"].items():
        if key not in skip:
            assert settled(on["reports"][key], key) == settled(value, key), (what, key)
    if skip:   # the classes of the pages still match
        cls = [[p[0], p[2]] for p in off["reports"]["ccm_last_mismatch_triage_pages"]]
        assert cls == [[p[0], p[2]] for p in on["reports"]["ccm_last_mismatch_triage_pages"]], what


def test_proven_failed_calls_leave_what_unproven_ones_leave_and_count_every_byte(results):
    pdl, rs = results
    for i, c in enumerate(drill_cases()):
        off, on = rs[2 * i], rs[2 * i + 1]
        what = (pdl, c)
        assert off["rc"] in (N.ERR_DIRTY, N.ERR_MISMATCH), (what, off["error"])
        assert on["cover"]["covered"] == 1, what
        assert_same(off, on, what)
        assert_exact(on, what)
        located = off["results"][-1]["nonzero_bytes"] != 0   # a tagged check zeroes what it finds off its tags
        assert ("LOCATE" in ran_steps(on)) == located, what
        if c.get("triage") and located:
            assert {"DIRT_T1", "DIRT_T2", "DIRT_T3"} <= ran_steps(on), what
        if c.get("mismatch_triage"):
            assert set(MISMATCH_STEPS) <= ran_steps(on), what


def test_clean_proven_calls_prove_nothing_and_launch_what_unproven_calls_do(results):
    pdl, rs = results
    start = 2 * len(drill_cases())
    for i, c in enumerate(CLEAN):
        off, on = rs[start + 2 * i], rs[start + 2 * i + 1]
        what = (pdl, c)
        assert off["rc"] == on["rc"] == 0, (what, off["error"], on["error"])
        assert on["report_cover"]["proved"] == 0 and on["report_cover"]["pages"] == [], what
        assert on["report_cover"]["ms_prove"] == 0.0, what   # nothing copied
        assert off["launches"] == on["launches"], what


def test_a_t3_that_skips_a_returned_page_fails_open_and_the_proof_names_it(results):
    pdl, rs = results
    start = 2 * (len(drill_cases()) + len(CLEAN))
    off, on = rs[start], rs[start + 1]
    what = (pdl, "fail-open")
    assert_same(off, on, what)
    first = off["reports"]["ccm_last_triage_pages"][0]
    assert first[0] == off["reports"]["pages1"][0][0], what
    assert N.TRIAGE_CLASSES[first[2]] == "clears", (what, first)   # the truth: RETURNS
    rc_ = on["report_cover"]
    assert rc_["proved"] == 1 and rc_["covered"] == 0, (what, rc_)
    dirt_pages = [tuple(p) for p in on["reports"]["pages1"]]
    want = RO.step_report(RO.pieces("DIRT_T3", spans(on), dirt_pages), k=1)
    got = rc_["steps"]["DIRT_T3"]
    assert {k: got[k] for k in want if k != "pages"} == {k: v for k, v in want.items() if k != "pages"}, (what, got, want)
    assert want["bytes_missing"] == RO.CO.CHUNK and first[0] in [p for p, _, _ in want["pages"]], want
    assert [(p["page"], p["expected"], p["counted"]) for p in rc_["pages"]] == want["pages"], (what, rc_["pages"])
    assert all(p["step"] == "DIRT_T3" for p in rc_["pages"]), what
    for name in ("LOCATE", "DIRT_T1", "DIRT_T2"):
        s = rc_["steps"][name]
        assert s["ran"] == 1 and s["bytes_missing"] == s["bytes_extra"] == 0, (what, name, s)


def test_every_step_can_be_drilled_and_the_next_call_is_exact(results):
    pdl, rs = results
    start = 2 * (len(drill_cases()) + len(CLEAN) + 1)
    for i, (step, c) in enumerate(STEP_SKIPS):
        off, on, after = rs[start + 3 * i: start + 3 * i + 3]
        what = (pdl, step, c)
        assert_same(off, on, what, tags_seeded=step in ("MISMATCH_T1", "MISMATCH_T2"))
        rc_ = on["report_cover"]
        assert rc_["proved"] == 1 and rc_["covered"] == 0, (what, rc_)
        dirt_pages = [tuple(p) for p in on["reports"]["pages1"]]
        mismatch_pages = [tuple(p) for p in on["reports"]["pages2"]]
        for name in RO.STEPS:
            s = rc_["steps"][name]
            if not s["ran"]:
                continue
            want = RO.step_report(RO.pieces(name, spans(on), dirt_pages, mismatch_pages), SKIP_K if name == step else 0)
            pages = want.pop("pages")
            assert {k: s[k] for k in want} == want, (what, name, s, want)
            assert [(p["page"], p["expected"], p["counted"]) for p in rc_["pages"] if p["step"] == name] == pages, what
        assert rc_["steps"][step]["ran"] and rc_["steps"][step]["bytes_missing"] > 0, (what, rc_["steps"][step])
        assert after["rc"] == off["rc"], (what, after["error"])
        assert_exact(after, what)


def test_the_locate_twin_keeps_its_rate(results):
    pdl, rs = results
    if pdl != "0":
        pytest.skip("rates are measured in the child without PDL")
    rate = [r for r in rs if r["call"].get("rate")]
    for key in ("scrub_inject", "scrub_flood"):
        sel = [r for r in rate if key in r["call"]["drill"]]
        for r in sel:
            assert r["rc"] == N.ERR_DIRTY, r["error"]
            if r["call"]["prove"]:
                assert r["report_cover"]["covered"] == 1, r["report_cover"]
        off = statistics.median(r["results"][0]["bytes_scrubbed"] / r["times"]["ms_locate"] for r in sel
                                if not r["call"]["prove"])
        on = statistics.median(r["results"][0]["bytes_scrubbed"] / r["times"]["ms_locate"] for r in sel
                               if r["call"]["prove"])
        assert on >= 0.85 * off, (key, on, off)
