"""Seeded random product scrub gate calls for the composed model (tests/gate_model.py).

scenario(seed) returns one call dict of tests/report_cover_calls.py, the same for the same seed: a gate kind, a path
(pipelined, map-first, whole HBM or the cudaMalloc fallback; interleaved read-back or not), the four armings and a
subset of the 17 drills.  Each is bounded to stay cheap on a shared H100: at most 8 GiB and mostly far less, whole HBM
for a few percent of seeds (zero gate, poison or flood only), triage holds of 1 to 5 ms.  The weights give every drill,
kind, path, arming and verdict a share (tests/test_gate_model.py counts them over the first seeds).  A draw the model
could not predict -- one that reads memory whose content only the driver knows, or that needs segment addresses the
call does not report -- is drawn again from the next sub-seed.
"""
from __future__ import annotations

import random

import gate_model as GM

MiB, GiB = 1 << 20, 1 << 30
GRAN = 2 * MiB
SIZES = [1, GRAN - 1, GRAN, GRAN + 1, 3 * GRAN + 5, 16 * MiB + 3, 100 * MiB + 1, 1536 * MiB, 3 * GiB + 2 * MiB + 1,
         8 * GiB]
SMALL = [1, GRAN - 1, GRAN, GRAN + 1, 4 * MiB]
FALLBACK_SIZES = [64 * 1024 + 7, GRAN + 1, 10 * MiB + 777, 100 * MiB + 1]
CHUNKS = [None, (2, 2), (2, 8), (64, 16)]
PATHS = ("pipelined", "map_first", "fallback", "whole")
PATH_WEIGHTS = (45, 25, 27, 3)
KIND_WEIGHTS = (40, 25, 15, 20)
FAKE_VA, FAKE_FREE = 1 << 40, 79 * GiB


def _draw(rng: random.Random) -> dict:
    path = rng.choices(PATHS, PATH_WEIGHTS)[0]
    kind = "zero" if path == "whole" else rng.choices(GM.KINDS, KIND_WEIGHTS)[0]
    tagged, census = kind in ("tagged", "census_tagged"), kind.startswith("census")
    env = {"CCM_INTERLEAVE_VERIFY": str(rng.randint(0, 1)), "CCM_ASYNC_RELEASE": str(rng.choice((1, 1, 1, 0)))}
    drill: dict = {}
    c: dict = {"kind": kind, "env": env, "drill": drill}
    if path == "whole":
        c["bytes"] = 0
        env["CCM_VMM_TAIL_MB"] = str(rng.choice((256, 2)))
        pick = rng.choice(("clean", "flood", "poison"))
        if pick == "flood":
            drill["scrub_flood"] = 0xC3
        elif pick == "poison":
            drill["scrub_poison"] = 0x5A
        c["prove"] = rng.randint(0, 1)
        return c
    if path == "fallback":
        env["CCM_PIPELINE"] = "0"
        seg = rng.choice((0, 0, 3, 96))
        if seg:
            env["CCM_ARENA_MAX_SEGMENT_MB"] = str(seg)
        c["bytes"] = rng.choice(FALLBACK_SIZES)
    else:
        if path == "map_first":
            env["CCM_MAP_FIRST"] = "1"
        ch = rng.choice(CHUNKS)
        if ch:
            env["CCM_VMM_FIRST_CHUNK_MB"], env["CCM_VMM_CHUNK_MB"] = str(ch[0]), str(ch[1])
        c["bytes"] = rng.choice(SIZES if not ch or ch[1] >= 16 else SIZES[:7])
    small = c["bytes"] <= 16 * MiB and env.get("CCM_ARENA_MAX_SEGMENT_MB") is None
    p = 0.3
    c["prove"] = int(rng.random() < 0.5)
    c["probe"] = int(not tagged and rng.random() < 0.4)
    c["triage"] = rng.randint(1, 5) if rng.random() < 0.4 else 0
    c["mismatch_triage"] = rng.randint(1, 5) if tagged and rng.random() < 0.5 else 0
    if rng.random() < p:
        drill["scrub_poison"] = 0x5A
    if rng.random() < p or (census and "scrub_poison" not in drill):
        drill["scrub_residue"] = rng.choice((1, 4, 9))
    if rng.random() < p:
        drill["scrub_flood"] = 0xC3
    if rng.random() < 0.4:
        drill["scrub_inject"] = rng.choice((1, 3, 4, 7, 1000))
    if tagged and rng.random() < 0.5:
        drill["tag_inject"] = rng.choice((1, 4, 7, 1000))
    if tagged and small and rng.random() < 0.25:
        drill["tag_flood"] = rng.choice((0x00, 0x3C))
        drill["tag_flood"] = drill["tag_flood"] or 0x3C
    # both views of an alias inside ONE launch race (oracle/tag_oracle.py alias_counts): only the per-mapping launches
    # of a pipelined call and the probe's per-chunk launches keep them apart
    if path == "pipelined" and (tagged or c["probe"]) and not c["mismatch_triage"] and rng.random() < 0.25:
        env["CCM_VMM_FIRST_CHUNK_MB"], env["CCM_VMM_CHUNK_MB"] = "2", "8"
        c["bytes"] = rng.choice((6 * MiB, 8 * MiB + 1, 100 * MiB + 1))
        drill["scrub_alias"] = 1
    if rng.random() < 0.25:
        drill["cover_skip"] = rng.choice((1, 2))
        drill["cover_pass"] = rng.choice((0, 1, 2, 3))
        if drill["cover_pass"] == 1 and not ("scrub_poison" in drill or "scrub_residue" in drill):
            drill["scrub_poison"] = 0x5A
    if c["triage"] or c["mismatch_triage"]:
        if rng.random() < 0.5:
            drill["triage_stay"] = rng.choice((1, 2, 5))
        if rng.random() < 0.5:
            drill["triage_return"] = rng.choice((1, 2, 5))
    if c["probe"]:
        if rng.random() < 0.4:
            drill["probe_mismatch"] = rng.choice((1, 3, 5))
        if rng.random() < 0.4:
            drill["probe_dirt"] = rng.choice((1, 3, 5))
        if rng.random() < 0.3:
            drill["probe_skip"] = rng.choice((1, 2))
            drill["probe_skip_step"] = rng.choice((0, 1, 2, 3))
            if c["prove"] and rng.random() < 0.5:   # both proofs short in one call: the read-back skips clean memory
                drill["cover_skip"], drill["cover_pass"] = 1, 3
    if rng.random() < 0.2:
        drill["report_skip"] = rng.choice((1, 2))
        drill["report_skip_step"] = rng.randint(0, 7)
    if kind == "zero" and not c["probe"] and not drill.get("scrub_alias") and path != "fallback" and rng.random() < 0.06:
        c["many"] = 2
    return c


def fake_record(c: dict) -> dict:
    """What the model takes from a call's record, made up: enough to tell whether the model can predict the call."""
    mapped = FAKE_FREE // GRAN * GRAN if c["bytes"] == 0 else 0
    return {"results": [{"device_free_before": FAKE_FREE, "bytes_scrubbed": mapped}], "va_base": FAKE_VA,
            "tags": [{"seed": 0x12345678}], "probe": {"seed": 0x9ABCDEF0}}


def scenario(seed: int) -> dict:
    """The call of `seed` (reproducible): drawn from random.Random(seed), then from sub-seeds while the model cannot
    predict the draw."""
    for sub in range(100):
        c = _draw(random.Random(seed * 1000 + sub))
        try:
            GM.predict(c, fake_record(c))
        except GM.Unpredictable:
            continue
        c["seed"] = seed
        return c
    raise RuntimeError(f"no predictable scenario for seed {seed}")
