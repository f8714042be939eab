"""The HBM health report on one H100: a real snapshot (which queries answer on this card); armed calls on every path
and kind; armed and unarmed paired calls over seeded scenarios of tests/gate_scenarios.py, which must agree on every
field of the composed model (tests/gate_model.py) and on the kernels launched; every drill's exact status and reason
under require and report, and its precedence against the dirt, tag and coverage drills; and the report of a call that
fails after its first snapshot.

The calls run in one child process (tests/hbm_health_calls.py)."""
from __future__ import annotations

import ctypes as C
import json
import subprocess
import sys
import tempfile
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "tests"))
import gate_model as GM  # noqa: E402
import gate_scenarios as GS  # noqa: E402
from k8s_cc_manager_b200 import _native as N  # noqa: E402

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

MiB = 1 << 20
Q = {name: 1 << k for k, name in enumerate(N.HBM_QUERIES)}
R = {name: 1 << k for k, name in enumerate(N.HBM_REASONS)}
NEEDED = Q["ecc_mode"] | Q["dram_uncorrected"] | Q["sram_uncorrected"] | Q["remapped_rows"]
SEEDS = 60
REQUIRE, REPORT = 2, 1


def run_child(calls: list[dict]) -> list[dict]:
    with tempfile.TemporaryDirectory() as tmp:
        path = Path(tmp) / "calls.json"
        path.write_text(json.dumps(calls))
        proc = subprocess.run([sys.executable, str(ROOT / "tests" / "hbm_health_calls.py"), f"@{path}"],
                              capture_output=True, text=True, cwd=ROOT, timeout=1800)
    assert proc.returncode == 0, proc.stdout[-4000:] + proc.stderr[-4000:]
    line = [x for x in proc.stdout.splitlines() if x.startswith("RESULT ")][-1]
    return json.loads(line[len("RESULT "):])


@pytest.fixture(scope="module", autouse=True)
def need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def test_a_real_snapshot_answers_what_the_rule_needs():
    code = ("import ctypes as C, json; from k8s_cc_manager_b200 import _native as N; lib = N.lib(); "
            "assert lib.ccm_init(N.BACKEND_CUDASIM) == 0; s = N.HbmState(); rc = lib.ccm_hbm_snapshot(0, C.byref(s)); "
            "print(json.dumps({'rc': rc, 'available': s.available, 'nvml_rc': list(s.nvml_rc), 'ecc': s.ecc_current, "
            "'pending': s.remap_pending, 'failure': s.remap_failure, 'ms': s.ms_query}))")
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=ROOT, timeout=300)
    assert out.returncode == 0, out.stderr
    s = json.loads(out.stdout.splitlines()[-1])
    answered = [q for q in N.HBM_QUERIES if s["available"] & Q[q]]
    print(f"\nqueries that answered: {answered}; NVML codes {s['nvml_rc']}; {s['ms']:.3f} ms")
    assert s["rc"] == N.OK and s["available"] & NEEDED == NEEDED
    assert s["ecc"] == 1 and s["pending"] == 0 and s["failure"] == 0


def fit(h: dict, mode: int) -> None:
    assert h["mode"] == mode and h["verdict"] == N.HBM_FIT, h
    assert h["reasons"] == 0 and h["missing_queries"] == 0
    assert h["d_dram_uncorrected"] == 0 and h["d_sram_uncorrected"] == 0
    assert h["after"]["remap_pending"] == 0 and h["after"]["remap_failure"] == 0 and h["after"]["ecc_current"] == 1
    assert h["ms_health"] > 0


PATHS = {"pipelined": {"CCM_VMM_FIRST_CHUNK_MB": "2", "CCM_VMM_CHUNK_MB": "8"}, "map_first": {"CCM_MAP_FIRST": "1"},
         "fallback": {"CCM_PIPELINE": "0"}}


def test_armed_calls_pass_a_healthy_card_on_every_path():
    calls = [{"bytes": 64 * MiB + 3, "kind": kind, "env": env, "health": REQUIRE, "tag": f"{kind}/{path}"}
             for kind in ("zero", "tagged", "census") for path, env in PATHS.items()]
    calls += [{"bytes": 64 * MiB, "kind": "zero", "many": 2, "health": REQUIRE, "tag": "fan-out"},
              {"bytes": 0, "kind": "zero", "health": REQUIRE, "tag": "whole HBM"}]
    for c, r in zip(calls, run_child(calls)):
        assert r["rc"] == N.OK, (c["tag"], r["error"])
        assert all(x["status"] == N.OK for x in r["results"]), c["tag"]
        fit(r["health"], REQUIRE)


def _plain(c: dict) -> bool:
    """A scenario whose observables do not depend on a random seed or on where the call's memory lies (as the pairs of
    tests/test_gate_scenarios_gpu.py)."""
    d = c.get("drill", {})
    return c["bytes"] != 0 and not (d.get("scrub_alias") or d.get("tag_flood") or d.get("probe_skip")
                                    or (d.get("cover_skip") and d.get("cover_pass") in (1, 2) and c["kind"] != "zero"))


def test_armed_and_unarmed_calls_agree_on_everything_but_the_report():
    scs = [c for c in (GS.scenario(s) for s in range(SEEDS)) if _plain(c)]
    calls = [x for c in scs for x in (dict(c, health=0), dict(c, health=REQUIRE))]
    recs = run_child(calls)
    failures = []
    for c, a, b in zip(scs, recs[0::2], recs[1::2]):
        diff = GM.first_difference(GM.observe(a), GM.observe(b))
        if diff:
            failures.append(f"seed {c['seed']}: {json.dumps(c)}\n  first difference {diff[0]}: {diff[1]!r} vs {diff[2]!r}")
        if a["launches"] != b["launches"]:
            failures.append(f"seed {c['seed']}: {a['launches']} launches unarmed, {b['launches']} armed")
        assert a["health"]["mode"] == 0 and a["health"]["before"]["available"] == 0   # unarmed: nothing read
        fit(b["health"], REQUIRE)
        assert b["rc"] == a["rc"], (c, a["error"], b["error"])
    assert len(scs) >= SEEDS // 2
    assert not failures, "\n".join(failures[:5]) + f"\n({len(failures)} of {len(scs)} pairs differ)"


# (hbm drills, verdict, reasons, missing queries, extra checks on the report)
DRILLS = [
    ({"hbm_uncorrected": 1}, N.HBM_UNFIT, R["dram_uncorrected"], 0, {"d_dram_uncorrected": 1}),
    ({"hbm_uncorrected": 5}, N.HBM_UNFIT, R["dram_uncorrected"], 0, {"d_dram_uncorrected": 5}),
    ({"hbm_corrected": 5}, N.HBM_FIT, 0, 0, {"d_dram_corrected": 5}),
    ({"hbm_remap_pending": 1}, N.HBM_UNFIT, R["remap_pending"], 0, {}),
    ({"hbm_remap_failure": 1}, N.HBM_UNFIT, R["remap_failure"], 0, {}),
    ({"hbm_unavailable": Q["sram_uncorrected"]}, N.HBM_UNKNOWN, R["no_answer"], Q["sram_uncorrected"], {}),
    ({"hbm_unavailable": Q["ecc_mode"] | Q["remapped_rows"]}, N.HBM_UNKNOWN, R["no_answer"],
     Q["ecc_mode"] | Q["remapped_rows"], {}),
    ({"hbm_unavailable": Q["remap_histogram"] | Q["dram_corrected"]}, N.HBM_FIT, 0, 0, {}),
    ({"hbm_unavailable": Q["dram_uncorrected"], "hbm_uncorrected": 3}, N.HBM_UNKNOWN, R["no_answer"],
     Q["dram_uncorrected"], {"d_dram_uncorrected": 0}),
]
REASON_WORDS = {R["dram_uncorrected"]: "uncorrected DRAM errors +", R["remap_pending"]: "a row remap is pending",
                R["remap_failure"]: "a row remap failed", R["no_answer"]: "no answer from NVML for"}
# (kind, sim drills, prove, the status of the same call unarmed)
OTHERS = [("zero", {"scrub_inject": 4}, 0, N.ERR_DIRTY), ("tagged", {"tag_inject": 4}, 0, N.ERR_MISMATCH),
          ("zero", {"cover_skip": 2, "cover_pass": 3}, 1, N.ERR_UNCOVERED), ("zero", {}, 0, N.OK)]


def test_every_drill_gives_its_status_and_reason_and_ranks_first():
    calls, cases = [], []
    for hd, verdict, reasons, missing, extra in DRILLS:
        for kind, drill, prove, base in OTHERS:
            for mode in (REQUIRE, REPORT):
                calls.append({"bytes": 16 * MiB + 5, "kind": kind, "drill": drill, "prove": prove, "health": mode,
                              "hbm_drill": hd})
                cases.append((hd, verdict, reasons, missing, extra, kind, drill, base, mode))
    for (hd, verdict, reasons, missing, extra, kind, drill, base, mode), r in zip(cases, run_child(calls)):
        h, what = r["health"], (hd, kind, drill, mode)
        assert (h["mode"], h["verdict"], h["reasons"], h["missing_queries"]) == (mode, verdict, reasons, missing), what
        for k, v in extra.items():
            assert h[k] == v, (what, k)
        want = N.ERR_HBM_HEALTH if mode == REQUIRE and verdict != N.HBM_FIT else base
        assert r["rc"] == want == r["results"][0]["status"], (what, r["error"])
        if want == N.ERR_HBM_HEALTH:
            assert ("unfit" if verdict == N.HBM_UNFIT else "unknown") in r["error"], r["error"]
            for bit, words in REASON_WORDS.items():
                assert (words in r["error"]) == bool(reasons & bit), (what, r["error"])
        # the counts the other drills produce are reported whatever the status
        if drill.get("scrub_inject"):
            assert r["results"][0]["nonzero_bytes"] == 4, what
        if drill.get("tag_inject"):
            assert r["tags"][0]["mismatch_bytes"] == 4, what
        if drill.get("cover_skip"):
            assert r["cover"]["proved"] == 1 and r["cover"]["covered"] == 0, what


def test_a_call_that_fails_after_its_first_snapshot_keeps_its_status_and_the_report():
    """With an arena held, the product call stops with CCM_ERR_STATE after the first snapshot: no GPU fault is needed
    to reach an error path."""
    code = r"""
import ctypes as C, json
from k8s_cc_manager_b200 import _native as N
lib = N.lib()
assert lib.ccm_init(N.BACKEND_CUDASIM) == 0
info = N.ArenaInfo()
assert lib.ccm_arena_acquire(0, 64 << 20, C.byref(info)) == 0, N.last_error()
out = {}
try:
    for mode in (2, 1):
        assert lib.ccm_scrub_health(0, mode) == 0
        assert lib.ccm_sim_set(0, b"hbm_remap_pending", 1) == 0
        res = N.ScrubResult()
        rc = lib.ccm_scrub_verify(0, 1 << 20, C.byref(res))
        err = N.last_error()
        h = N.HbmHealth()
        assert lib.ccm_scrub_last_health(0, C.byref(h)) == 0
        out[mode] = dict(rc=rc, status=res.status, err=err, mode=h.mode, verdict=h.verdict, reasons=h.reasons,
                         before=h.before.available, after=h.after.available)
        lib.ccm_scrub_health(0, 0)
        lib.ccm_sim_set(0, b"hbm_remap_pending", 0)
finally:
    lib.ccm_arena_release(0)
print(json.dumps(out))
"""
    proc = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=ROOT, timeout=300)
    assert proc.returncode == 0, proc.stderr
    out = json.loads(proc.stdout.splitlines()[-1])
    for mode in ("2", "1"):
        o = out[mode]
        assert o["rc"] == o["status"] == N.ERR_STATE and "arena already held" in o["err"], o
        assert o["mode"] == int(mode) and o["verdict"] == N.HBM_UNFIT and o["reasons"] == R["remap_pending"], o
        assert o["before"] & NEEDED == NEEDED and o["after"] & NEEDED == NEEDED, o
