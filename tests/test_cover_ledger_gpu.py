"""The coverage ledger on one H100: clean proven calls are exact for every kind, mapping mode and path, and leave what
unarmed calls leave; "cover_repeat" fails a call whose page report is covered, on exactly the oracle's slots;
"cover_lane_drop" leaves one slot short by exactly one thread's share; "cover_skip" gives a ledger that agrees with the
page report; the drills run clean under compute-sanitizer where it can instrument the device; and deliberately wrong
copies of the ledger code (MUTANTS) fail the driver.  Each case list runs in a child process
(tests/cover_ledger_calls.py), once with CCM_PDL=1 and once with CCM_PDL=0."""
from __future__ import annotations

import json
import os
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "tests"))
import cover_ledger_oracle as LO  # noqa: E402
import cover_oracle as CO  # noqa: E402
import kernel_mutants as KM  # noqa: E402
import product_plan as PP  # noqa: E402
from k8s_cc_manager_b200 import _native as N  # noqa: E402

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

MiB = 1 << 20
DRIVER = ROOT / "tests" / "cover_ledger_calls.py"
KINDS = ("zero", "tagged", "census", "census_tagged")
FALLBACK = {"CCM_PIPELINE": "0", "CCM_ARENA_MAX_SEGMENT_MB": "3"}   # 3 MiB segments, the last one ragged
SMALL = 256 * MiB


def clean_cases() -> list[dict]:
    cases = [{"bytes": SMALL, "kind": kind, "env": PP.mode_env(mf, il)} for kind in KINDS for mf, il in PP.MODES]
    cases += [{"bytes": 10 * MiB + 777, "kind": kind, "env": FALLBACK} for kind in KINDS]
    cases += [{"bytes": SMALL, "kind": "zero", "many": 1}, {"bytes": SMALL, "kind": "tagged", "many": 1},
              {"bytes": 0, "kind": "zero"}]
    return cases


# (kind, pass, value, bytes, env) of the drilled calls
REPEATS = [("zero", 1, 3, SMALL, {}), ("zero", 3, 5, SMALL, {}), ("tagged", 1, 1, SMALL, {}), ("tagged", 2, 15, SMALL, {}),
           ("census", 1, 2, SMALL, {}), ("zero", 3, 4, SMALL, {"CCM_INTERLEAVE_VERIFY": "0"}),
           ("zero", 1, 3, 10 * MiB + 777, FALLBACK), ("tagged", 2, 2, 10 * MiB + 777, FALLBACK)]
DROPS = [("zero", 1, 1, SMALL, {}), ("zero", 3, 0, SMALL, {}), ("tagged", 2, 511, SMALL, {}),
         ("census_tagged", 1, 7, SMALL, {}), ("zero", 1, 33, 10 * MiB + 777, FALLBACK)]
SKIPS = [("zero", 3, 3, SMALL, {}), ("tagged", 2, 2, SMALL, {}), ("zero", 1, 7, 10 * MiB + 777, FALLBACK)]


def drilled(kind, pass_, key, value, nbytes, env) -> dict:
    return {"bytes": nbytes, "kind": kind, "env": env, "prove": 1, "drill": {key: value, "cover_pass": pass_}}


def calls() -> list[dict]:
    out = []
    for c in clean_cases():
        out += [dict(c, prove=0), dict(c, prove=1)]
    out += [drilled(k, p, "cover_repeat", v, n, e) for k, p, v, n, e in REPEATS]
    out += [drilled(k, p, "cover_lane_drop", v + 1, n, e) for k, p, v, n, e in DROPS]   # the key takes t + 1
    out += [drilled(k, p, "cover_skip", v, n, e) for k, p, v, n, e in SKIPS]
    return out


def run_driver(case_calls: list, env: dict, prefix: list | None = None, timeout: int = 1800):
    return subprocess.run([*(prefix or []), sys.executable, str(DRIVER), json.dumps(case_calls)], capture_output=True,
                          text=True, env=dict(os.environ, **env), cwd=ROOT, timeout=timeout)


def result_of(proc) -> list | None:
    lines = [x for x in proc.stdout.splitlines() if x.startswith("RESULT ")]
    return json.loads(lines[-1][len("RESULT "):]) if lines else None


@pytest.fixture(scope="module", params=["1", "0"], ids=["pdl", "nopdl"])
def results(request):
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    proc = run_driver(calls(), {"CCM_PDL": request.param})
    rs = result_of(proc)
    assert proc.returncode == 0 and rs is not None, proc.stdout[-4000:] + proc.stderr[-4000:]
    return request.param, rs


def oracle_for(r: dict, name: str | None = None, value: int = 0) -> dict:
    """The oracle's ledger of a call's result r, drilled with `name` (skip, repeat, drop) on its cover_pass."""
    c = r["call"]
    kind = c.get("kind", "zero")
    tagged = kind in ("tagged", "census_tagged")
    mapped = r["results"][0]["bytes_scrubbed"]
    drill = None
    if name is not None:
        pass_ = CO.DRILL_PASS[c["drill"]["cover_pass"]]
        ranges, mappings, interleave, mapped2 = CO.call_launches(c["bytes"], c.get("env", {}))
        assert mapped2 == mapped
        launch = (LO.first_repeat_launch(pass_, tagged, ranges, mappings, interleave, mapped) if name == "repeat"
                  else CO.first_launch(pass_, tagged, ranges, mappings, interleave, mapped))
        drill = (name, pass_, value, *launch)
    return LO.ledger(mapped, tagged, drill)


def assert_ledger(r: dict, want: dict, what) -> None:
    led = r["ledger"]
    assert led["proved"] == 1 and led["exact"] == want["exact"], (what, r["error"], led)
    assert led["bytes_mapped"] == r["cover"]["bytes_mapped"] and led["slots_mapped"] == want["slots_mapped"], what
    assert led["va_base"] == r["cover"]["va_base"], what
    for p in LO.PASSES:
        for f, v in want["passes"][p].items():
            assert led["passes"][p][f] == v, (what, p, f, led["passes"][p])
    assert [{k: v for k, v in s.items() if k != "chunk"} for s in led["slots"]] == want["slots"], (what, led["slots"][:4])


def test_clean_proven_calls_are_exact_and_leave_what_unarmed_calls_leave(results):
    pdl, rs = results
    cases = clean_cases()
    for i, c in enumerate(cases):
        off, on = rs[2 * i], rs[2 * i + 1]
        what = (pdl, c)
        assert off["rc"] == on["rc"] == 0, (what, off["error"], on["error"])
        assert off["ledger"]["proved"] == 0 and off["ledger"]["slots"] == [], what
        assert on["cover"]["covered"] == 1, what
        if not c.get("many"):
            assert_ledger(on, oracle_for(on), what)
        else:
            assert on["ledger"]["exact"] == 1 and on["ledger"]["proved"] == 1, what
        for a, b in zip(off["results"], on["results"]):
            assert (a["status"], a["nonzero_bytes"]) == (b["status"], b["nonzero_bytes"]), what
            if c["bytes"]:
                assert (a["bytes_scrubbed"], a["segments"]) == (b["bytes_scrubbed"], b["segments"]), what
        if c["bytes"]:   # whole HBM: the armed call maps the ledgers' bytes less
            assert off["launches"] == on["launches"], what
            assert off["reports"] == on["reports"], what


def drill_results(rs: list, start: int, n: int) -> list:
    return rs[start: start + n]


def test_a_repeated_chunk_fails_the_ledger_while_its_page_is_covered(results):
    pdl, rs = results
    start = 2 * len(clean_cases())
    for (kind, pass_, k, nbytes, env), r in zip(REPEATS, drill_results(rs, start, len(REPEATS))):
        what = (pdl, kind, pass_, k, nbytes, env)
        assert r["rc"] == N.ERR_UNCOVERED, (what, r["error"])
        assert "coverage ledger failed" in r["error"], (what, r["error"])
        assert r["cover"]["proved"] == 1 and r["cover"]["covered"] == 1, (what, r["cover"])
        want = oracle_for(r, "repeat", k)
        assert want["exact"] == 0
        assert_ledger(r, want, what)


def test_a_dropped_lane_leaves_its_slot_short_by_its_share(results):
    pdl, rs = results
    start = 2 * len(clean_cases()) + len(REPEATS)
    for (kind, pass_, t, nbytes, env), r in zip(DROPS, drill_results(rs, start, len(DROPS))):
        what = (pdl, kind, pass_, t, nbytes, env)
        assert r["rc"] == N.ERR_UNCOVERED and r["cover"]["covered"] == 1, (what, r["error"])
        want = oracle_for(r, "drop", t)
        assert_ledger(r, want, what)
        name = CO.DRILL_PASS[pass_]
        assert r["ledger"]["passes"][name]["bytes_missing"] == LO.SHARE[name] and len(r["ledger"]["slots"]) == 1, what


def test_a_skipped_chunk_shows_in_the_ledger_as_in_the_page_report(results):
    pdl, rs = results
    start = 2 * len(clean_cases()) + len(REPEATS) + len(DROPS)
    for (kind, pass_, k, nbytes, env), r in zip(SKIPS, drill_results(rs, start, len(SKIPS))):
        what = (pdl, kind, pass_, k, nbytes, env)
        assert r["rc"] == N.ERR_UNCOVERED and r["cover"]["covered"] == 0, (what, r["error"])
        assert_ledger(r, oracle_for(r, "skip", k), what)
        name = CO.DRILL_PASS[pass_]
        assert r["ledger"]["passes"][name]["bytes_missing"] == r["cover"]["passes"][name]["bytes_missing"], what
        # the page report's pages are the pages of the ledger's slots
        assert {s["slot"] * LO.SLOT // LO.PAGE for s in r["ledger"]["slots"]} == {p["page"] for p in r["pages"]}, what


# ------------------------------------------------------------------------------------------------- sanitizer
from test_sanitizers_gpu import sanitizer  # noqa: E402,F401  (the fixture: skips where the tool cannot instrument the GPU)


def test_drills_run_clean_under_compute_sanitizer(sanitizer):
    tool = sanitizer
    one = [drilled("zero", 1, "cover_repeat", 3, 8 * MiB, {}), drilled("zero", 3, "cover_lane_drop", 6, 8 * MiB, {}),
           drilled("tagged", 2, "cover_skip", 2, 8 * MiB, {})]
    for check in ("memcheck", "racecheck"):
        proc = run_driver(one, {"CCM_PDL": "0"}, [tool, "--tool", check, "--error-exitcode", "1"], timeout=1800)
        assert proc.returncode == 0 and "ERROR SUMMARY: 0 errors" in proc.stdout + proc.stderr, \
            (check, proc.stdout[-3000:], proc.stderr[-3000:])
        rs = result_of(proc)
        assert rs is not None and all(r["rc"] == N.ERR_UNCOVERED for r in rs), check


# ------------------------------------------------------------------------------------------------- mutants
M = KM.Mutant
MUTANTS = [
    M("ledger_slot_plus_one", KM.KERNELS,
      "  const uint64_t slot = off >> kSlotShift;",
      "  const uint64_t slot = (off >> kSlotShift) + 1;",
      "ledger_word puts every byte on the next slot", KM.VALUE + " (the index stays clamped to the outside slot)",
      ("clean",)),
    M("ledger_chunk_unsplit", KM.KERNELS,
      "  const uint32_t lo = n < before ? n : before;",
      "  const uint32_t lo = n;",
      "ledger_chunk counts a chunk that crosses a slot boundary all on its first slot", KM.VALUE,
      ("clean",)),
    M("ledger_sum_alone", KM.KERNELS,
      "  const uint32_t total = __reduce_add_sync(same, bytes);",
      "  const uint32_t total = bytes;",
      "ledger_sum adds only the bytes of the lane that issues the atomic, not its peers'", KM.VALUE,
      ("clean",)),
    M("ledger_count_constant", KM.KERNELS,
      "    if (addr(p) != cover.drop) n = op.template chunk<THREADS, PER_THREAD>(p);",
      "    if (addr(p) != cover.drop) op.template chunk<THREADS, PER_THREAD>(p);\n    n = 256u;",
      "CoverOp::chunk counts 256 bytes per lane whatever its op addressed, and also for a dropped share", KM.VALUE,
      ("clean", "drop")),
]
# Calls that each mutant must fail: clean proven calls of every pass kind and a dropped lane on the read-back.
MUTANT_CALLS = [dict(c, label="clean") for c in (
    {"bytes": 64 * MiB, "kind": "zero", "prove": 1}, {"bytes": 64 * MiB, "kind": "tagged", "prove": 1},
    {"bytes": 64 * MiB, "kind": "census", "prove": 1}, {"bytes": 10 * MiB + 777, "kind": "zero", "prove": 1,
                                                        "env": FALLBACK})]
MUTANT_CALLS.append(dict(drilled("zero", 3, "cover_lane_drop", 6, 64 * MiB, {}), label="drop"))


def test_mutant_anchors_occur_once():
    for m in MUTANTS:
        assert KM.anchor_count(m) == 1, m.id


@pytest.fixture(scope="module")
def mutant_libs() -> dict:
    return {m.id: KM.build(m)[0] for m in MUTANTS}


def wrong(r: dict) -> bool:
    """True when a call's ledger is not what the oracle says."""
    name = "drop" if r["call"]["label"] == "drop" else None
    want = oracle_for(r, name, 5) if name else oracle_for(r)
    led = r["ledger"]
    if led["proved"] != 1 or led["exact"] != want["exact"]:
        return True
    if any(led["passes"][p].get(f) != v for p in LO.PASSES for f, v in want["passes"][p].items()):
        return True
    return [{k: v for k, v in s.items() if k != "chunk"} for s in led["slots"]] != want["slots"]


@pytest.mark.parametrize("mid", [m.id for m in MUTANTS])
def test_ledger_mutant_is_killed(mid, mutant_libs):
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    m = next(x for x in MUTANTS if x.id == mid)
    proc = run_driver(MUTANT_CALLS, {"CCM_PDL": "0", "CCM_LIB": str(mutant_libs[mid])}, timeout=600)
    rs = result_of(proc)
    assert rs is not None, (mid, proc.stdout[-3000:], proc.stderr[-3000:])
    assert all(r["rc"] in (0, N.ERR_UNCOVERED) for r in rs), (mid, [r["error"] for r in rs])
    killing = [r["call"]["label"] for r in rs if wrong(r)]
    print(f"\n{mid}: killed by {killing}")
    if mid == "ledger_chunk_unsplit":
        # no range of a product call starts off a slot boundary: VMM mappings are whole 2 MiB granules and every
        # fallback segment but the last is a whole number of MiB, so no chunk crosses one and this copy is equivalent
        assert not killing, (mid, killing)
        return
    assert any(k in m.killer for k in killing), (mid, killing)
