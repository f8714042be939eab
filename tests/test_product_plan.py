"""CPU: the product gate's plan model (tests/product_plan.py) is self-consistent and agrees with the counts
the existing product tests pin; the GPU matrix sweeps every knob ccm_scrub.cu reads; the drill sim keys
round-trip on the sim backend and are no-ops on sysfs."""
from __future__ import annotations

import itertools
import re
from pathlib import Path

import pytest

import product_plan as PP
from helpers import sim_get, sim_set
from k8s_cc_manager_b200 import _native as N
from k8s_cc_manager_b200 import devices as D

ROOT = Path(__file__).resolve().parents[1]
MiB, GiB = PP.MiB, PP.GiB
GRAN = PP.H100_GRAN
FREE = 79 * GiB + 417 * MiB + 12345          # a whole-HBM call's free bytes on an 80 GB card
KNOB_RE = re.compile(r'(?:env_u64|getenv|env_variant)\(\s*"(CCM_[A-Z0-9_]+)"')


def knob_grid():
    for setting in PP.CHUNK_SETTINGS:
        for mf, il in PP.MODES:
            for tail in (None, 256, 2, 0, 100000):
                env = {**PP.chunk_env(setting), **PP.mode_env(mf, il)}
                if tail is not None:
                    env["CCM_VMM_TAIL_MB"] = str(tail)
                yield env


def check_run(p: PP.Plan, run: PP.Run):
    for off, n in run.chunks:
        assert n % p.gran == 0 and n > 0 and off % p.gran == 0
    assert [o for o, _ in run.chunks] == list(itertools.accumulate([0] + [n for _, n in run.chunks][:-1]))
    assert run.mapped == sum(n for _, n in run.chunks) <= p.va_bytes
    ranges = run.ranges(p)
    pos = 0
    for off, n in ranges:                    # in order, no gap, no overlap
        assert off == pos and n > 0
        pos += n
    assert pos == run.mapped
    if p.map_first:
        assert ranges == [(0, run.mapped)]
    elif run.tail:
        assert ranges[-1] == (run.main_end, run.mapped - run.main_end) and run.tail[0][0] == run.main_end
        assert len(ranges) == len(run.main) + 1
    for _, n in run.main[:-1]:
        assert n <= p.max_chunk
    for _, n in run.tail:
        assert n <= PP.TAIL_GRANULE


@pytest.mark.parametrize("nbytes", [1, GRAN - 1, GRAN, GRAN + 1, 100 * MiB + 1, (3 << 30) + (2 << 20) + 1,
                                    (7 << 30) + 3, 81 * GiB])
def test_requested_plan_invariants(nbytes):
    for env in knob_grid():
        p = PP.plan(nbytes, FREE, GRAN, env)
        assert p.va_bytes == -(-nbytes // GRAN) * GRAN and p.tail_zone == 0 and p.main_end == p.va_bytes
        assert p.gran <= p.first <= p.max_chunk and p.first % GRAN == 0 and p.max_chunk % GRAN == 0
        run = PP.simulate(p, None)
        check_run(p, run)
        assert run.mapped == p.va_bytes and run.main == run.chunks and not run.tail
        sizes = [n for _, n in run.chunks]
        assert sizes[0] == min(p.first, p.va_bytes)
        for a, b in zip(sizes, sizes[1:-1]):     # doubling up to the cap (the last chunk is the remainder)
            assert b == min(2 * a, p.max_chunk)


def test_whole_hbm_plan_invariants():
    for env in knob_grid():
        p = PP.plan(0, FREE, GRAN, env)
        assert p.va_bytes == FREE // GRAN * GRAN
        assert p.main_end + p.tail_zone == p.va_bytes and p.tail_zone % GRAN == 0
        for capacity in (p.va_bytes, p.main_end, p.va_bytes - GRAN, p.va_bytes - 300 * MiB, p.main_end - 5 * GRAN,
                         p.main_end + 7 * GRAN, 40 * GiB + 6 * MiB, 3 * GRAN):
            capacity = min(max(capacity, GRAN), p.va_bytes) // GRAN * GRAN
            run = PP.simulate(p, capacity)
            check_run(p, run)
            assert run.mapped == capacity                          # granules reach the driver's last byte
            if capacity >= p.main_end:                             # the tail zone absorbed the out-of-memory
                assert run.main == p.main and (run.main_end == p.main_end or not run.tail)
            else:
                assert run.main_end <= capacity


def test_plan_clamps_every_chunk_setting_to_the_granularity():
    cases = {None: (1024, 16384), (2, 2): (2, 2), (2, 8): (2, 8), (3, 5): (2, 4), (1, 1): (2, 2), (64, 16): (16, 16)}
    for setting, (first, cap) in cases.items():
        p = PP.plan(GiB, FREE, GRAN, PP.chunk_env(setting))
        assert (p.first, p.max_chunk) == (first * MiB, cap * MiB), setting
    p = PP.plan(GiB, FREE, 64 * MiB, {"CCM_VMM_FIRST_CHUNK_MB": "100", "CCM_VMM_CHUNK_MB": "1"})
    assert (p.first, p.max_chunk) == (64 * MiB, 64 * MiB)       # below the granularity: one granule


def test_plan_matches_the_counts_the_product_tests_pin():
    """tests/test_scrub_gpu.py and tests/test_scrub_exactness_gpu.py pin these numbers on the GPU."""
    def calls(nbytes, env):
        p = PP.plan(nbytes, FREE, GRAN, env)
        run = PP.simulate(p, None)
        return len(run.chunks), len(PP.inject_offsets(run.ranges(p), PP.INJECT))
    assert calls(2 << 30, {}) == (2, 8)
    assert calls((3 << 30) + (2 << 20), {}) == (3, 12)
    assert calls((3 << 30) + (2 << 20), {"CCM_INTERLEAVE_VERIFY": "0"}) == (3, 12)
    assert calls(1 << 30, {"CCM_MAP_FIRST": "1"}) == (1, 4)
    assert calls(100 * MiB + 1, PP.chunk_env((2, 2))) == (51, 204)           # more than kMaxPipeChunks
    assert PP.plan(GiB, FREE, GRAN, {}, node_fanout=True).map_first
    assert not PP.plan(GiB, FREE, GRAN, {"CCM_MAP_FIRST": "0"}, node_fanout=True).map_first
    # whole HBM with map first: four candidates, the last one the last mapped byte
    p = PP.plan(0, FREE, GRAN, {"CCM_MAP_FIRST": "1"})
    run = PP.simulate(p, p.va_bytes - 40 * MiB)
    assert PP.inject_offsets(run.ranges(p), 1000)[-1] == run.mapped - 1


def test_inject_candidates():
    assert PP.inject_offsets([(0, 1)], 1000) == [0]
    assert PP.inject_offsets([(0, 2)], 1000) == [0, 1]
    assert PP.inject_offsets([(0, 5)], 1000) == [0, 4]                         # 17 and 5 not inside: 0
    assert PP.inject_offsets([(0, 18)], 1000) == [0, 17, 12]
    assert PP.inject_offsets([(10, 100), (110, 100)], 1000) == [10, 27, 63, 109, 110, 127, 163, 209]
    assert PP.inject_offsets([(10, 100), (110, 100)], 5) == [10, 27, 63, 109, 110]
    assert PP.inject_offsets([(0, GRAN)], 3) == [0, 17, GRAN // 2 + 3]


def test_arena_segments():
    env = {"CCM_ARENA_MAX_SEGMENT_MB": "96"}
    assert PP.arena_segments(300 * MiB, FREE, env) == [(0, 96 * MiB), (96 * MiB, 96 * MiB), (192 * MiB, 96 * MiB),
                                                       (288 * MiB, 12 * MiB)]
    assert PP.arena_segments(GRAN + 1, FREE, {}) == [(0, GRAN + 1)]
    want = (FREE - 256 * MiB) & ~(2 * MiB - 1)
    assert PP.arena_segments(0, FREE, {}) == [(0, want)]
    assert PP.arena_segments(0, FREE, {"CCM_ARENA_RESERVE_MB": "1024"}) == [(0, (FREE - GiB) & ~(2 * MiB - 1))]


def test_gpu_matrix_shape():
    for setting in PP.CHUNK_SETTINGS:
        for nbytes, env in PP.requested_cases(setting, GRAN):
            p = PP.plan(nbytes, FREE, GRAN, env)
            assert len(PP.simulate(p, None).chunks) <= 512, (setting, nbytes)   # no call maps thousands
    most = max(len(PP.simulate(PP.plan(b, FREE, GRAN, env), None).chunks)
               for s in PP.CHUNK_SETTINGS for b, env in PP.requested_cases(s, GRAN))
    assert most > 32
    assert {tuple(sorted(PP.mode_env(mf, il).items())) for mf, il in PP.MODES} == {
        tuple(sorted(PP.mode_env(mf, il).items())) for mf in (0, 1) for il in (0, 1)}
    assert len(PP.VARIANT_PINS) == 8 and all(PP.variant_pin_env(*v)["CCM_MAP_FIRST"] == "1" for v in PP.VARIANT_PINS)


def test_gpu_matrix_sweeps_every_knob_the_scrub_stage_reads():
    src = (ROOT / "k8s_cc_manager_b200" / "csrc" / "ccm_scrub.cu").read_text()
    read = set(KNOB_RE.findall(src))
    assert {"CCM_VMM_TAIL_MB", "CCM_MAP_FIRST", "CCM_PIPELINE", "CCM_PDL"} <= read, sorted(read)
    swept = PP.swept_knobs()
    unswept = sorted(k for k in read - set(PP.EXEMPT_KNOBS) if len(swept.get(k, ())) < 2)
    assert not unswept, "knobs ccm_scrub.cu reads that the GPU matrix never changes: " + ", ".join(unswept)
    assert set(PP.EXEMPT_KNOBS) <= read, "exempt knobs the library no longer reads: " + \
        ", ".join(sorted(set(PP.EXEMPT_KNOBS) - read))
    assert set(PP.PLAN_KNOBS) <= read


@pytest.fixture()
def sim():
    lib = N.lib()
    assert lib.ccm_sim_topology(2, 0) == 0
    sim_set(-1, "cuda_ordinal", -1)
    return lib


def test_drill_keys_round_trip_on_the_sim_backend(sim):
    for key, value in (("scrub_poison", 0x5A), ("scrub_flood", 0xFF), ("scrub_inject", 1 << 40)):
        assert sim_get(0, key) == 0
        sim_set(0, key, value)
        assert sim_get(0, key) == value and sim_get(1, key) == 0
        sim_set(-1, key, 1)
        assert sim_get(0, key) == sim_get(1, key) == 1
        sim_set(-1, key, 0)
    for key in ("scrub_poison", "scrub_flood"):
        for bad in (-1, 256, 1 << 33):
            assert sim.ccm_sim_set(0, key.encode(), bad) == N.ERR_INVALID
            assert sim_get(0, key) == 0
    sim_set(0, "scrub_inject", -5)                       # negative budget: off
    assert sim_get(0, "scrub_inject") == 0


def test_drill_keys_are_no_ops_on_sysfs(tmp_path, monkeypatch):
    d = tmp_path / "devices" / "0000:1b:00.0"
    d.mkdir(parents=True)
    for name, value in (("vendor", "0x10de"), ("class", "0x030200"), ("device", "0x2330"), ("reset", "")):
        (d / name).write_text(value + "\n" if value else "")
    monkeypatch.setenv("CCM_SYSFS_ROOT", str(tmp_path / "devices"))
    try:
        D.select_backend("sysfs")
        for key in PP.DRILL_KEYS:
            assert N.lib().ccm_sim_set(0, key.encode(), 7) == 0
            assert sim_get(0, key) == 0
    finally:
        D.select_backend("sim")
