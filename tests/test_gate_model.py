"""The composed model of a product gate call (tests/gate_model.py) and its scenario generator (tests/gate_scenarios.py),
on the CPU: the model reproduces fixed expectations the per-feature tests agree on, its sparse memory agrees with the
numpy oracles, the rules that the H100 corrected stay pinned, and the generator is reproducible and reaches every drill,
kind, path, arming and verdict, and every adjacent pair of the precedence order in one call."""
from __future__ import annotations

import collections
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
for p in (ROOT / "tests", ROOT / "oracle"):
    sys.path.insert(0, str(p))
import dirt_oracle as DO  # noqa: E402
import gate_model as GM  # noqa: E402
import gate_scenarios as GS  # noqa: E402
import page_oracle as PGO  # noqa: E402
import product_plan as PP  # noqa: E402
import triage_oracle as TO  # noqa: E402

MiB, GiB = 1 << 20, 1 << 30
N_SEEDS = 400
VA = 1 << 40


def rec(c: dict, mapped: int = 0, free: int = 79 * GiB, va: int = VA, seed: int = 0x12345678) -> dict:
    return {"results": [{"device_free_before": free, "bytes_scrubbed": mapped}], "va_base": va,
            "tags": [{"seed": seed}], "probe": {"seed": 0x9ABCDEF0}}


# ------------------------------------------------------------------------------------------ fixed expectations
def test_inject_counts_four_bytes_per_range_as_the_product_plan_says():
    c = {"bytes": 1536 * MiB, "drill": {"scrub_inject": 1000}}
    w = GM.predict(c, rec(c))
    plan = PP.plan(c["bytes"], 0, PP.H100_GRAN, {})
    want = len(PP.inject_offsets(PP.simulate(plan, None).ranges(plan), 1000))
    assert w["rc"] == GM.DIRTY and w["results"][0]["nonzero_bytes"] == want == 8
    assert w["dirt"][1] == want and len(w["dirt"][6]) == want


def test_flood_counts_every_mapped_byte_and_poison_stays_clean():
    for drill, rc, count in (({"scrub_flood": 0xC3}, GM.DIRTY, 1536 * MiB), ({"scrub_poison": 0x5A}, GM.OK, 0)):
        c = {"bytes": 1536 * MiB, "drill": drill}
        w = GM.predict(c, rec(c))
        assert w["rc"] == rc and w["results"][0]["nonzero_bytes"] == count


def test_tag_inject_mismatches_and_reads_back_clean():
    c = {"bytes": 1536 * MiB, "kind": "tagged", "drill": {"tag_inject": 7}, "mismatch_triage": 5}
    w = GM.predict(c, rec(c))
    assert w["rc"] == GM.MISMATCH and w["tags"] == [7] and w["results"][0]["nonzero_bytes"] == 0
    assert all(r[3] == GM.PARTIAL for r in w["mismatch"][6])
    assert w["mismatch_triage"]["report"][GM.TRIAGE_FIELDS.index("clear_pages")] == len(w["pages2"])


def test_census_counts_the_residue_drill_and_zero_fills_every_mapping():
    # csrc/ccm_scrub.cu GateRun::held: the zero fill acts on every mapping while the drill is set, even after its
    # budget is spent; a census then counts only the 0xA5 bytes, whatever poison was there before
    c = {"bytes": 1536 * MiB, "kind": "census_tagged", "drill": {"scrub_poison": 0x5A, "scrub_residue": 4}}
    w = GM.predict(c, rec(c))
    assert w["residue"] == [[4, 4]] and w["rc"] == GM.OK
    assert sum(p[1] for p in w["pages3"]) == 4


def test_dirt_triage_classes_match_the_triage_oracle():
    c = {"bytes": 1536 * MiB, "drill": {"scrub_inject": 1000, "triage_stay": 1, "triage_return": 2}, "triage": 5}
    w = GM.predict(c, rec(c))
    entries = [tuple(p) for p in w["pages1"]]
    want = TO.report(entries, [(0, 1536 * MiB)], 1, 2)
    got = dict(zip(GM.TRIAGE_FIELDS, w["triage"]["report"]))
    assert {k: got[k] for k in want} == want


def test_the_default_report_skip_step_is_dirt_t3():
    # include/ccm.h: "report_skip_step" 0 selects CCM_REPORT_DIRT_T3
    c = {"bytes": 1536 * MiB, "drill": {"scrub_inject": 4, "triage_return": 1, "report_skip": 1}, "triage": 5,
         "prove": 1}
    w = GM.predict(c, rec(c))
    steps = w["report_cover"]["steps"]
    assert steps["DIRT_T3"]["bytes_missing"] > 0 and steps["DIRT_T2"]["bytes_missing"] == 0
    first = w["triage"]["pages"][0]
    assert first[2] == 3      # the fail-open: the page that dirtied again is classed CLEARS


def test_the_residue_page_map_is_only_predicted_for_census_calls():
    c = {"bytes": 16 * MiB, "drill": {"scrub_residue": 4}}
    assert GM.predict(c, rec(c))["pages3"] is None


def test_probe_drills_and_precedence():
    c = {"bytes": 1536 * MiB, "probe": 1, "prove": 1, "drill": {"probe_mismatch": 3, "probe_dirt": 2}}
    w = GM.predict(c, rec(c))
    assert w["fails"] == ["probe_mismatch", "dirty"] and w["rc"] == GM.MISMATCH
    assert w["probe"]["mismatch_bytes"] == 3 and w["results"][0]["nonzero_bytes"] == 2
    c = dict(c, drill={"probe_skip": 2, "probe_skip_step": 2})
    w = GM.predict(c, rec(c))
    assert w["fails"][0] == "probe_uncovered" and w["rc"] == GM.UNCOVERED


def test_a_dirty_read_back_does_not_probe_and_tagged_calls_ignore_the_probe():
    c = {"bytes": 64 * MiB, "probe": 1, "drill": {"scrub_inject": 3, "probe_dirt": 5}}
    assert GM.predict(c, rec(c))["probe"] == {"probed": 0}
    c = {"bytes": 64 * MiB, "probe": 1, "kind": "tagged", "drill": {"probe_dirt": 5}}
    assert GM.predict(c, rec(c))["probe"] == {"probed": 0}


def test_cover_skip_of_the_first_pass_leaves_poison_for_the_read_back():
    c = {"bytes": 64 * MiB, "prove": 0, "drill": {"scrub_poison": 0x5A, "cover_skip": 1, "cover_pass": 1}}
    w = GM.predict(c, rec(c))
    assert w["rc"] == GM.DIRTY and w["results"][0]["nonzero_bytes"] == 128 << 10
    w = GM.predict(dict(c, prove=1), rec(c))
    assert w["fails"] == ["pass_uncovered", "dirty"]


def test_an_alias_inside_the_tagged_check_matches_the_tag_oracle():
    c = {"bytes": 6 * MiB, "kind": "tagged", "drill": {"scrub_alias": 1},
         "env": {"CCM_VMM_FIRST_CHUNK_MB": "2", "CCM_VMM_CHUNK_MB": "8"}}
    import tag_oracle as TAG
    w = GM.predict(c, rec(c, seed=77))
    assert w["tags"] == [TAG.alias_counts(77, VA, 2 * MiB)[0]]
    assert w["results"][0]["segments"] == 2     # the second chunk's first 2 MiB come from the first handle


# ------------------------------------------------------------------------------------------ sparse vs numpy
@pytest.mark.parametrize("seed", range(6))
def test_sparse_books_agree_with_the_numpy_oracles(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(1000, 40000))
    mem = GM.Mem(n, VA)
    mem.write(0, n, 0)
    mem.write(int(rng.integers(0, n // 2)), int(rng.integers(n // 2, n)), int(rng.integers(1, 256)))
    for o in rng.integers(0, n, 20).tolist():
        mem.xor(int(o))
    mem.tag(100, 700, 9)
    buf = mem.values(0, n)
    got = GM.book(mem, [(0, n)])
    want = DO.report(buf, VA)
    assert (got["bytes"], got["windows"], got["first"], got["last"]) == \
        (want["nonzero_bytes"], want["dirty_windows"], want["first_offset"], want["last_offset"])
    assert {p: k for p, k, _ in got["pages"]} == PGO.page_map(buf, VA)


# ------------------------------------------------------------------------------------------ the generator
def test_a_seed_always_yields_the_same_scenario():
    assert [GS.scenario(s) for s in range(30)] == [GS.scenario(s) for s in range(30)]


def test_the_generator_reaches_every_axis_and_verdict():
    keys, kinds, paths, arms, verdicts, pairs = (collections.Counter() for _ in range(6))
    knobs: dict = collections.defaultdict(set)
    for s in range(N_SEEDS):
        c = GS.scenario(s)
        w = GM.predict(c, GS.fake_record(c))
        keys.update(c["drill"].keys())
        kinds[c["kind"]] += 1
        env = c["env"]
        paths["whole" if c["bytes"] == 0 else "fallback" if env.get("CCM_PIPELINE") == "0" else
              "map_first" if env.get("CCM_MAP_FIRST") == "1" else "pipelined"] += 1
        for k, v in env.items():
            knobs[k].add(v)
        arms.update(a for a in ("prove", "probe", "triage", "mismatch_triage", "many") if c.get(a))
        verdicts[w["fails"][0] if w["fails"] else "clean"] += 1
        pairs.update(zip(w["fails"], w["fails"][1:]))
    print(f"\nover {N_SEEDS} seeds: drills {dict(keys)}\nkinds {dict(kinds)}\npaths {dict(paths)}\narmings {dict(arms)}"
          f"\nverdicts {dict(verdicts)}\nprecedence pairs {dict(pairs)}")
    assert set(keys) == set(GM.DRILL_KEYS), set(GM.DRILL_KEYS) - set(keys)
    assert set(kinds) == set(GM.KINDS) and set(paths) == set(GS.PATHS)
    assert set(arms) == {"prove", "probe", "triage", "mismatch_triage", "many"}
    for k in ("CCM_INTERLEAVE_VERIFY", "CCM_ASYNC_RELEASE", "CCM_MAP_FIRST", "CCM_PIPELINE"):
        assert len(knobs[k] | {"default"}) >= 2, k
    assert knobs["CCM_INTERLEAVE_VERIFY"] == {"0", "1"}
    assert all(verdicts[v] >= 5 for v in ("clean",) + GM.PRECEDENCE), verdicts
    # every adjacent pair of the precedence order that one call can hold happens with both outcomes in one call: a
    # tagged call never probes, so the probe's outcomes and the tag mismatch never meet, and the pairs that skip them
    # stand in for the ones across them
    for hi, lo in (("pass_uncovered", "probe_uncovered"), ("probe_uncovered", "probe_mismatch"),
                   ("probe_mismatch", "dirty"), ("pass_uncovered", "tag_mismatch"), ("tag_mismatch", "dirty")):
        assert pairs[(hi, lo)] >= 1, (hi, lo, pairs)
