"""The probe proof on one H100: clean proven-and-probed calls count every probe window once on every mapping path and
leave what the same call probed but unproven leaves; the "probe_skip" drill on each step against the oracle, proven and
not; scrub_alias with P2's aliased windows skipped, the fail-open it closes; its precedence over the probe's mismatch;
no proof when only one of the two is armed; and the manager end to end.  The product calls run in a child process
(tests/probe_cover_calls.py)."""
from __future__ import annotations

import json
import logging
import os
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "tests"))
import probe_cover_oracle as PCO  # noqa: E402
import product_gate_calls as PGC  # noqa: E402
import product_plan as PP  # noqa: E402
import scenarios as SC  # noqa: E402
from k8s_cc_manager_b200 import _native as N  # noqa: E402
from k8s_cc_manager_b200 import devices as D  # noqa: E402

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

MiB, GiB = 1 << 20, 1 << 30
FALLBACK = {"CCM_PIPELINE": "0", "CCM_ARENA_MAX_SEGMENT_MB": "3"}
SMALL = {"CCM_VMM_FIRST_CHUNK_MB": "2", "CCM_VMM_CHUNK_MB": "8"}   # 2, 4, 8, 8 MiB: 512, 1024, 2048, 2048 windows
FIRST64 = {"CCM_VMM_FIRST_CHUNK_MB": "64"}
ALIAS_SKIP = 64 * MiB // 4096   # every window of the first (aliased) 64 MiB chunk


def needs_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def clean_cases() -> dict:
    cases = {f"vmm{mf}{il}": {"bytes": 1536 * MiB, "env": PP.mode_env(mf, il)} for mf, il in PP.MODES}
    cases["small"] = {"bytes": 22 * MiB, "env": SMALL}
    cases["whole"] = {"bytes": 0}
    cases["fallback"] = {"bytes": 10 * MiB + 777, "env": FALLBACK}
    cases["census"] = {"bytes": 1536 * MiB, "kind": "census"}
    return cases


def drill_cases() -> dict:
    cases = {f"skip{s}": {"bytes": 1536 * MiB, "drill": {"probe_skip": 5, "probe_skip_step": s}} for s in (1, 2, 3)}
    cases["skip_fallback"] = {"bytes": 10 * MiB + 777, "env": FALLBACK, "drill": {"probe_skip": 7}}
    cases["alias"] = {"bytes": 512 * MiB, "env": {**PP.mode_env(0, 1), **FIRST64},
                      "drill": {"scrub_alias": 1, "probe_skip": ALIAS_SKIP, "probe_skip_step": 2}}
    cases["precedence"] = {"bytes": 1536 * MiB, "drill": {"probe_mismatch": 3, "probe_skip": 2, "probe_skip_step": 3}}
    return cases


def calls() -> list:
    """Every case proven and probed, and probed but unproven; then the two single armings."""
    out = []
    for name, c in {**clean_cases(), **drill_cases()}.items():
        out += [(name, "both", dict(c, prove=1, probe=1)), (name, "probe", dict(c, prove=0, probe=1))]
    out += [("single", "prove", {"bytes": 1536 * MiB, "prove": 1, "probe": 0}),
            ("single", "none", {"bytes": 1536 * MiB, "prove": 0, "probe": 0}),
            ("single", "probe", {"bytes": 1536 * MiB, "prove": 0, "probe": 1})]
    return out


@pytest.fixture(scope="module")
def results():
    needs_gpu()
    todo = calls()
    proc = subprocess.run([sys.executable, str(ROOT / "tests" / "probe_cover_calls.py"), json.dumps([c for *_, c in todo])],
                          capture_output=True, text=True, cwd=ROOT, timeout=1800, env=dict(os.environ))
    assert proc.returncode == 0, proc.stdout[-4000:] + proc.stderr[-4000:]
    out = json.loads([x for x in proc.stdout.splitlines() if x.startswith("RESULT ")][-1][len("RESULT "):])
    res = {}
    for (name, arm, _), r in zip(todo, out):
        res.setdefault(name, {})[arm] = r
    return res


def chunks_of(r: dict) -> list:
    """The mapping loop's chunks of a VMM call with a requested size, as (address, bytes, offset)."""
    c, res = r["call"], r["results"][0]
    p = PP.plan(c["bytes"], res["device_free_before"], PP.H100_GRAN, c.get("env", {}), node_fanout=True)
    run = PP.simulate(p, None)
    assert run.mapped == res["bytes_scrubbed"]
    return PCO.vmm_chunks(r["probe"]["va_base"], run.chunks)


def same_as_unproven(both: dict, probe: dict) -> None:
    vary = ("device_free_before",) + (("bytes_scrubbed", "bytes_unreached", "segments") if not both["call"]["bytes"] else ())
    for a, b in zip(both["results"], probe["results"]):
        assert {k: v for k, v in a.items() if k not in vary and not k.startswith("ms_")} == \
               {k: v for k, v in b.items() if k not in vary and not k.startswith("ms_")}
    assert both["reports"] == probe["reports"] and both["mismatch_records"] == probe["mismatch_records"]
    skip = ("seed", "ms_probe", "va_base") + (("windows", "bytes_probed", "launches") if not both["call"]["bytes"] else ())
    assert {k: v for k, v in both["probe"].items() if k not in skip} == \
           {k: v for k, v in probe["probe"].items() if k not in skip}
    if both["call"]["bytes"]:
        assert both["launches"] == probe["launches"]
    assert probe["probe_cover"]["proved"] == 0 and probe["probe_cover_pages"] == []


@pytest.mark.parametrize("name", list(clean_cases()))
def test_clean_proven_probe_counts_every_window_once(results, name):
    both, probe = results[name]["both"], results[name]["probe"]
    assert both["rc"] == probe["rc"] == 0, both["error"]
    same_as_unproven(both, probe)
    pc, p = both["probe_cover"], both["probe"]
    assert pc["proved"] == 1 and pc["covered"] == 1 and both["probe_cover_pages"] == []
    assert pc["windows_expected"] == p["windows"] > 0 and pc["va_base"] == p["va_base"]
    for s in pc["steps"]:
        assert s["ran"] == 1 and s["windows_counted"] == p["windows"]
        assert s["windows_missing"] == s["windows_extra"] == s["windows_outside"] == s["pages_short"] == 0
    assert both["cover"]["proved"] == 1 and both["cover"]["covered"] == 1
    if name != "fallback" and both["call"]["bytes"]:
        chunks = chunks_of(both)
        assert PCO.windows(chunks) == p["windows"]
        if name == "small":
            assert [PCO.chunk_windows(a, n)[1] % 1024 for a, n, _ in chunks] == [512, 0, 0, 0]


# What the skipped windows do to an unproven call: untagged windows fail P2's check, unchecked windows keep their tags
# through P3, and unread windows go unseen.
UNPROVEN_RC = {1: N.ERR_MISMATCH, 2: N.ERR_DIRTY, 3: N.OK}


@pytest.mark.parametrize("step", [1, 2, 3])
def test_skip_drill_on_each_step_against_the_oracle(results, step):
    both, probe = results[f"skip{step}"]["both"], results[f"skip{step}"]["probe"]
    assert probe["rc"] == UNPROVEN_RC[step] and probe["probe_cover"]["proved"] == 0
    assert both["rc"] == N.ERR_UNCOVERED and "HBM alias probe proof failed" in both["error"]
    want = PCO.report(chunks_of(both), 5, step)
    pc = both["probe_cover"]
    assert pc["proved"] == 1 and pc["covered"] == 0 and pc["windows_expected"] == want["windows_expected"]
    for got, w in zip(pc["steps"], want["steps"]):
        assert {k: got[k] for k in w} == w
    assert {g["page"]: (g["expected"], g["count"]) for g in both["probe_cover_pages"]} == \
           {p: (e, c) for p, (e, c) in want["pages"].items()}
    assert all(g["chunk"] == 0 for g in both["probe_cover_pages"])
    assert both["launches"] == probe["launches"] and both["probe"]["windows"] == probe["probe"]["windows"]
    # the probe report is filled as unproven: the skipped windows' bytes that differ from their tags (a tag byte that
    # happens to be zero does not count, so the exact number depends on the call's seed)
    for k, s in (("mismatch_bytes", 1), ("reread_nonzero_bytes", 2)):
        for r in (both, probe):
            assert (0 < r["probe"][k] <= 5 * 32) if step == s else r["probe"][k] == 0


def test_skip_drill_on_the_fallback(results):
    both, probe = results["skip_fallback"]["both"], results["skip_fallback"]["probe"]
    assert probe["rc"] == N.ERR_DIRTY and both["rc"] == N.ERR_UNCOVERED
    pc = both["probe_cover"]
    s = pc["steps"][1]
    assert s["windows_missing"] == 7 and s["pages_short"] == 1 and s["first_short_page"] == 0
    assert pc["steps"][0]["windows_missing"] == pc["steps"][2]["windows_missing"] == 0
    assert s["windows_counted"] == pc["windows_expected"] - 7 == both["probe"]["windows"] - 7


def test_scrub_alias_with_its_windows_skipped_fails_only_proven(results):
    both, probe = results["alias"]["both"], results["alias"]["probe"]
    assert probe["rc"] == 0 and probe["probe"]["mismatch_bytes"] == 0   # the fail-open, reproduced
    assert both["rc"] == N.ERR_UNCOVERED
    want = PCO.report(chunks_of(both), ALIAS_SKIP, 2)
    s = both["probe_cover"]["steps"][1]
    assert s["windows_missing"] == ALIAS_SKIP == want["steps"][1]["windows_missing"]
    assert s["pages_short"] == want["steps"][1]["pages_short"] == 32 and s["first_short_page"] == 0
    assert [g["page"] for g in both["probe_cover_pages"]] == list(want["pages"])


def test_uncovered_takes_precedence_over_the_probes_mismatch(results):
    both, probe = results["precedence"]["both"], results["precedence"]["probe"]
    assert probe["rc"] == N.ERR_MISMATCH and both["rc"] == N.ERR_UNCOVERED
    assert both["probe"]["mismatch_bytes"] == probe["probe"]["mismatch_bytes"] == 3
    assert both["reports"]["mismatch"][0] == 3 and len(both["mismatch_records"]) == 3
    assert both["probe_cover"]["steps"][2]["windows_missing"] == 2


def test_no_proof_unless_both_are_armed(results):
    r = results["single"]
    for arm in ("prove", "probe", "none"):
        assert r[arm]["rc"] == 0 and r[arm]["probe_cover"]["proved"] == 0 and r[arm]["probe_cover_pages"] == []
    assert r["prove"]["launches"] == r["none"]["launches"]
    assert r["probe"]["launches"] == r["none"]["launches"] + 3 * r["probe"]["results"][0]["segments"]


# ---------------------------------------------------------------------------------- the manager end to end
def test_manager_fails_a_transition_whose_probe_skipped_windows(monkeypatch, caplog):
    needs_gpu()
    import kubernetes
    from k8s_cc_manager_b200 import manager
    lib = PGC.open_lib()
    for k, v in dict(EVICT_OPERATOR_COMPONENTS="false", CC_RELEASE_CUDA_CONTEXT="false").items():
        monkeypatch.setenv(k, v)
    assert lib.ccm_init(N.BACKEND_CUDASIM) == 0
    lib.ccm_sim_set(-1, b"cc_mode", N.CC_MODES["off"])
    lib.ccm_sim_set(0, b"probe_skip", 3)
    try:
        c = kubernetes.reset_cluster()
        c.add_node(SC.NODE, {})
        mgr = manager.CCManager(SC.NODE, "on", True, device_source=D.find_gpus, scrub_bytes=4 * GiB,
                                scrub_proof="require", scrub_alias_probe="require")
        with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
            assert mgr.set_cc_mode("on") is False
        bdf = next(d.bdf for d in D.find_gpus()[0] if d.cuda_ordinal == 0)
        pc = mgr.last_transition["scrub_probe_cover"][bdf]
        assert pc.proved == 1 and pc.covered == 0 and pc.short_step().name == "P2"
        assert pc.short_step().windows_missing == 3
        assert any(r.levelno == logging.ERROR and r.getMessage().startswith(f"HBM alias probe proof on {bdf}")
                   for r in caplog.records)
    finally:
        lib.ccm_sim_set(0, b"probe_skip", 0)
        PGC.release_wait(lib)
