"""Seeded random product scrub gate calls on one H100 against the composed model (tests/gate_model.py), and paired
calls that must agree on everything but one named difference.

Every scenario of tests/gate_scenarios.py runs in a child process (tests/report_cover_calls.py), once with CCM_PDL=1
and once with CCM_PDL=0 (the library latches it per process), and every observable the child records must equal the
model's prediction.  A failure names the seed, the scenario and the first field that differs.  Replay seeds with
GATE_SCENARIO_SEEDS=17,402; GATE_SCENARIO_COUNT sets how many seeds run (default SEEDS).

Each batch starts and ends with a clean 1-byte call: the free HBM the last one sees must be what the first one saw.
"""
from __future__ import annotations

import collections
import copy
import json
import os
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "tests"))
import gate_model as GM  # noqa: E402
import gate_scenarios as GS  # noqa: E402

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

# 200 seeds per PDL value.  On one H100 80GB HBM3 at a 700 W power limit, a child made the 200 scenarios and their 336
# paired calls in 16 s (median call 4 ms to the verdict; the whole-HBM calls take longest), and the file took about two
# minutes in all with both PDL values, inside a bound of ten minutes.
SEEDS = 200
FREE_SLACK = 256 << 20
MARK = {"bytes": 1, "kind": "zero", "marker": 1}


def seeds() -> list[int]:
    env = os.environ.get("GATE_SCENARIO_SEEDS")
    if env:
        return [int(s) for s in env.split(",") if s.strip()]
    return list(range(int(os.environ.get("GATE_SCENARIO_COUNT", SEEDS))))


def run_child(pdl: str, calls: list[dict]) -> tuple[list[dict], float]:
    env = dict(os.environ, CCM_PDL=pdl)
    with tempfile.TemporaryDirectory() as tmp:   # too many calls for one argument
        path = Path(tmp) / "calls.json"
        path.write_text(json.dumps([MARK] + calls + [MARK]))
        t0 = time.perf_counter()
        proc = subprocess.run([sys.executable, str(ROOT / "tests" / "report_cover_calls.py"), f"@{path}"],
                              capture_output=True, text=True, env=env, cwd=ROOT, timeout=1800)
        wall = time.perf_counter() - t0
    assert proc.returncode == 0, proc.stdout[-4000:] + proc.stderr[-4000:]
    line = [x for x in proc.stdout.splitlines() if x.startswith("RESULT ")][-1]
    recs = json.loads(line[len("RESULT "):])
    first, last = recs[0], recs[-1]
    assert last["results"][0]["device_free_before"] >= first["results"][0]["device_free_before"] - FREE_SLACK, \
        ("HBM was not handed back", first["results"][0], last["results"][0])
    return recs[1:-1], wall


# ------------------------------------------------------------------------------------------------ pairs
def _plain(c: dict) -> bool:
    """A scenario whose observables do not depend on a random seed or on where the call's memory lies."""
    d = c.get("drill", {})
    return not (d.get("scrub_alias") or d.get("tag_flood") or d.get("probe_skip")
                or (d.get("cover_skip") and d.get("cover_pass") in (1, 2) and c["kind"] != "zero"))


def pairs(scs: list[dict]) -> list[tuple[str, dict, dict]]:
    """(name, a, b) of the paired calls made from the scenarios: each differs from its partner in one axis."""
    out = []
    for c in scs:
        if not _plain(c) or c["bytes"] == 0:
            continue
        d = c.get("drill", {})
        if not d.get("cover_skip") and not d.get("probe_skip") and not d.get("report_skip"):
            out.append(("prove", dict(c, prove=0), dict(c, prove=1)))
        if c.get("triage") or c.get("mismatch_triage"):
            out.append(("triage", dict(c, triage=0, mismatch_triage=0), dict(c)))
        if c["kind"] in ("tagged", "census_tagged"):
            out.append(("probe", dict(c, probe=0), dict(c, probe=1)))
        # a drilled read-back skips the chunks of its first launch, which the interleave moves
        if c.get("env", {}).get("CCM_PIPELINE") != "0" and not (d.get("cover_skip") and d.get("cover_pass") in (0, 3)):
            a, b = copy.deepcopy(c), copy.deepcopy(c)
            a["env"]["CCM_INTERLEAVE_VERIFY"], b["env"]["CCM_INTERLEAVE_VERIFY"] = "0", "1"
            out.append(("interleave", a, b))
    return out


def path_pairs() -> list[tuple[str, dict, dict]]:
    """Pipelined, map-first and fallback calls of the same bytes, with drills whose effect does not depend on the
    range split (poison, flood, tag flood on a small call)."""
    out = []
    for kind, nbytes, drill in (("zero", 100 << 20, {"scrub_flood": 0xC3}), ("zero", 100 << 20, {"scrub_poison": 0x5A}),
                                ("census", 10 << 20, {"scrub_poison": 0x5A}),
                                ("tagged", 4 << 20, {"tag_flood": 0x3C, "scrub_flood": 0xC3})):
        base = {"bytes": nbytes, "kind": kind, "drill": drill}
        calls = [dict(base, env={"CCM_VMM_FIRST_CHUNK_MB": "2", "CCM_VMM_CHUNK_MB": "8"}),
                 dict(base, env={"CCM_MAP_FIRST": "1"}), dict(base, env={"CCM_PIPELINE": "0"})]
        out += [("path", calls[0], calls[1]), ("path", calls[0], calls[2])]
    return out


def without(obs: dict, keys) -> dict:
    return {k: v for k, v in obs.items() if k not in keys}


# the report proof of a triage's steps is part of the triage's reports
ALLOWED = {"prove": ("cover", "report_cover", "probe_cover"), "triage": ("triage", "mismatch_triage", "report_cover"),
           "probe": (), "interleave": ()}


# ------------------------------------------------------------------------------------------------ the runs
@pytest.fixture(scope="module", params=["1", "0"], ids=["pdl", "nopdl"])
def batch(request):
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    scs = [GS.scenario(s) for s in seeds()]
    prs = pairs(scs) + path_pairs()
    calls = scs + [x for _, a, b in prs for x in (a, b)]
    recs, wall = run_child(request.param, calls)
    return request.param, scs, prs, recs[:len(scs)], recs[len(scs):], wall


def test_every_scenario_matches_the_model(batch):
    pdl, scs, prs, recs, _, wall = batch
    verdicts = collections.Counter()
    times = sorted(r["ms_verdict"] for r in recs)
    failures = []
    for c, r in zip(scs, recs):
        want = GM.predict(c, r)
        verdicts[want["fails"][0] if want["fails"] else "clean"] += 1
        diff = GM.compare(c, r)
        if diff:
            failures.append(f"seed {c['seed']} (CCM_PDL={pdl}): {json.dumps(c)}\n  first difference {diff[0]}: "
                            f"model {diff[1]!r}, call {diff[2]!r}")
    print("\n".join(failures))
    print(f"\nCCM_PDL={pdl}: {len(scs)} scenarios, {len(prs)} pairs, verdicts {dict(verdicts)}, median call "
          f"{times[len(times) // 2]:.1f} ms, child wall {wall:.1f} s")
    assert not failures, "\n".join(failures[:5]) + f"\n({len(failures)} of {len(scs)} scenarios differ)"


def test_paired_calls_differ_only_where_allowed(batch):
    pdl, _, prs, _, precs, _ = batch
    failures = []
    for i, (name, a, b) in enumerate(prs):
        ra, rb = precs[2 * i], precs[2 * i + 1]
        oa, ob = GM.observe(ra), GM.observe(rb)
        if name == "path":
            # rc and status match; the mapping fields differ; flood counts each call's own bytes
            assert ra["rc"] == rb["rc"], (pdl, name, a, b, ra["error"], rb["error"])
            for r in (ra, rb):
                if r["call"]["drill"].get("scrub_flood"):
                    x = r["results"][0]
                    assert x["nonzero_bytes"] == x["bytes_scrubbed"], (pdl, r["call"], x)
            continue
        diff = GM.first_difference(without(oa, ALLOWED[name]), without(ob, ALLOWED[name]))
        if diff:
            failures.append(f"{name} pair (CCM_PDL={pdl}) of seed {a.get('seed')}: {json.dumps(a)}\n  first difference "
                            f"{diff[0]}: {diff[1]!r} vs {diff[2]!r}")
    assert not failures, "\n".join(failures[:5]) + f"\n({len(failures)} of {len(prs)} pairs differ)"
