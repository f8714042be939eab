"""The coverage ledger on the CPU: fill_ledger (ccm_proof.h, compiled with g++) field by field against
tests/cover_ledger_oracle.py for clean calls and every drill on the product plan's launches, slots over and the
outside slot; the per-lane split of a chunk that crosses a slot boundary; the C ABI without a CUDA device (exports,
struct layouts from a C99 compile, refusals, drill keys); CoverLedger's JSON, summary, CLI and worker keys; and the
manager's policy in both isolation modes."""
from __future__ import annotations

import ctypes as C
import json
import logging
import re
import shutil
import subprocess
from pathlib import Path

import pytest

import cover_ledger_oracle as LO
import cover_oracle as CO
import product_plan as PP
import test_cover_proof as TC
import test_dirt_locate as TD
import test_tag_mismatch as TM
import scenarios as SC
from k8s_cc_manager_b200 import _native as N
from k8s_cc_manager_b200 import devices as D
from k8s_cc_manager_b200.devices import CoverLedger, GpuError, LedgerPass, LedgerSlot, ScrubReport

ROOT = Path(__file__).resolve().parents[1]
MiB = 1 << 20

HARNESS = r"""
#include <cstdio>
#include <vector>
#include "ccm_proof.h"
int main() {
  unsigned long long ns, mapped, base; int ran3[3]; size_t nchunks;
  if (scanf("%llu %llu %llu %d %d %d %zu", &ns, &mapped, &base, &ran3[0], &ran3[1], &ran3[2], &nchunks) != 7) return 2;
  ccm_proof::ChunkTable chunks(nchunks);
  for (auto& c : chunks) { unsigned long long o; unsigned k; if (scanf("%llu %u", &o, &k) != 2) return 2; c = {o, k}; }
  std::vector<uint32_t> words(3 * (ns + 1));
  for (auto& w : words) if (scanf("%u", &w) != 1) return 2;
  const bool ran[3] = {ran3[0] != 0, ran3[1] != 0, ran3[2] != 0};
  ccm_cover_ledger rep; std::vector<ccm_ledger_slot> slots;
  ccm_proof::fill_ledger(words.data(), ns, mapped, base, ran, chunks, &rep, &slots);
  printf("{\"bytes_mapped\": %llu, \"slots_mapped\": %llu, \"va_base\": %llu, \"proved\": %d, \"exact\": %d, \"passes\": [",
         (unsigned long long)rep.bytes_mapped, (unsigned long long)rep.slots_mapped, (unsigned long long)rep.va_base,
         rep.proved, rep.exact);
  for (int k = 0; k < 3; ++k) {
    const ccm_ledger_pass& p = rep.pass[k];
    printf("%s{\"ran\": %d, \"slots_short\": %llu, \"slots_over\": %llu, \"bytes_missing\": %llu, \"bytes_extra\": %llu, "
           "\"bytes_outside\": %llu, \"first_short_slot\": %llu, \"first_over_slot\": %llu}", k ? ", " : "", p.ran,
           (unsigned long long)p.slots_short, (unsigned long long)p.slots_over, (unsigned long long)p.bytes_missing,
           (unsigned long long)p.bytes_extra, (unsigned long long)p.bytes_outside, (unsigned long long)p.first_short_slot,
           (unsigned long long)p.first_over_slot);
  }
  printf("], \"slots\": [");
  for (size_t i = 0; i < slots.size(); ++i)
    printf("%s{\"slot\": %llu, \"chunk\": %u, \"expected\": %u, \"first\": %u, \"check\": %u, \"readback\": %u}",
           i ? ", " : "", (unsigned long long)slots[i].slot, slots[i].chunk, slots[i].expected, slots[i].count[0],
           slots[i].count[1], slots[i].count[2]);
  printf("]}\n");
  return 0;
}
"""


@pytest.fixture(scope="module")
def fill(tmp_path_factory):
    gxx = shutil.which("g++")
    if gxx is None:
        pytest.skip("no C++ compiler")
    d = tmp_path_factory.mktemp("ledger")
    (d / "h.cpp").write_text(HARNESS)
    subprocess.run([gxx, "-std=c++17", "-O1", "-Wall", "-Werror", "-I", str(ROOT / "include"), "-I",
                    str(ROOT / "k8s_cc_manager_b200" / "csrc"), str(d / "h.cpp"), "-o", str(d / "h")], check=True)

    def run(ledgers: list[list[int]], mapped: int, ran: tuple, chunks=((0, 0),), base: int = 1 << 40) -> dict:
        ns = len(ledgers[0]) - 1
        text = f"{ns} {mapped} {base} {ran[0]:d} {ran[1]:d} {ran[2]:d} {len(chunks)}\n"
        text += " ".join(f"{o} {k}" for o, k in chunks) + "\n" + " ".join(str(w) for led in ledgers for w in led)
        return json.loads(subprocess.run([str(d / "h")], input=text, capture_output=True, text=True,
                                         check=True).stdout)
    return run


def words_of(mapped: int, tagged: bool, drill, nslots: int) -> list[list[int]]:
    """The three ledgers (nslots words and the outside slot) the oracle says a call leaves."""
    want = LO.expected(mapped, nslots)
    out = []
    rep = LO.ledger(mapped, tagged, drill, nslots)
    for k, p in enumerate(LO.PASSES):
        if not rep["passes"][p]["ran"]:
            out.append([0] * (nslots + 1))
            continue
        got = {s["slot"]: s[p] for s in rep["slots"]}
        out.append([got.get(i, w) for i, w in enumerate(want)] + [0])
    return out


def compare(got: dict, want: dict, mapped: int) -> None:
    assert got["proved"] == 1 and got["exact"] == want["exact"] and got["bytes_mapped"] == mapped
    assert got["slots_mapped"] == want["slots_mapped"]
    for k, p in enumerate(LO.PASSES):
        for f, v in want["passes"][p].items():
            assert got["passes"][k][f] == v, (p, f, got["passes"][k])
    assert [{k: v for k, v in s.items() if k != "chunk"} for s in got["slots"]] == want["slots"]


PLANS = [(96 * MiB, {}), (96 * MiB, {"CCM_INTERLEAVE_VERIFY": "0"}), (64 * MiB + 12345, {}),
         (10 * MiB + 777, {"CCM_PIPELINE": "0", "CCM_ARENA_MAX_SEGMENT_MB": "3"})]
DRILLS = [None, ("repeat", "first", 3), ("repeat", "readback", 15), ("repeat", "check", 1), ("drop", "first", 0),
          ("drop", "readback", 0), ("drop", "check", 0), ("skip", "readback", 2), ("skip", "first", 5)]


@pytest.mark.parametrize("mapped_env", PLANS, ids=lambda x: f"{x[0]}-{'-'.join(x[1].values()) or 'vmm'}")
@pytest.mark.parametrize("tagged", [False, True])
@pytest.mark.parametrize("drill", DRILLS, ids=lambda d: "clean" if d is None else f"{d[0]}-{d[1]}-{d[2]}")
def test_fill_ledger_matches_the_oracle_on_the_plans_launches(fill, mapped_env, tagged, drill):
    nbytes, env = mapped_env
    ranges, mappings, interleave, mapped = CO.call_launches(nbytes, env)
    spec = None
    if drill is not None:
        name, pass_, value = drill
        launch = (LO.first_repeat_launch(pass_, tagged, ranges, mappings, interleave, mapped) if name == "repeat"
                  else CO.first_launch(pass_, tagged, ranges, mappings, interleave, mapped))
        if launch is None:
            pytest.skip("the pass does not run in this call")
        spec = (name, pass_, value, *launch)
    nslots = -(-mapped // LO.SLOT) + 3    # a few slots past the mapping, as on a device larger than the call
    want = LO.ledger(mapped, tagged, spec, nslots)
    got = fill(words_of(mapped, tagged, spec, nslots), mapped, (True, tagged, True))
    compare(got, want, mapped)
    if drill is not None and drill[0] == "repeat" and want["passes"][drill[1]].get("ran"):
        # page 0 of the drilled launch counts exactly: the page report cannot see it
        led = words_of(mapped, tagged, spec, nslots)[LO.PASSES.index(drill[1])]
        first = spec[3] // LO.SLOT
        assert sum(led[first:first + LO.PAGE // LO.SLOT]) == LO.PAGE and not want["exact"]


def test_slots_over_past_the_mapping_and_outside(fill):
    mapped = 5 * LO.SLOT + 100
    clean = [LO.expected(mapped, 8) + [0] for _ in range(3)]
    assert fill(clean, mapped, (True, False, True))["exact"] == 1
    led = [list(x) for x in clean]
    led[2][7] = 16          # a byte walked past the mapping, on a slot of the device
    led[2][8] = 3           # and three outside every slot
    led[0][1] += 256        # a slot walked one share too many
    led[0][5] -= 100        # the ragged last slot short
    led[1][0] = 99          # a pass that did not run is not compared
    got = fill(led, mapped, (True, False, True), chunks=((0, 0), (3 * LO.SLOT, 1)))
    assert got["exact"] == 0
    first, check, readback = got["passes"]
    assert (first["slots_short"], first["slots_over"], first["bytes_missing"], first["bytes_extra"]) == (1, 1, 100, 256)
    assert (first["first_short_slot"], first["first_over_slot"]) == (5, 1)
    assert check == {"ran": 0, "slots_short": 0, "slots_over": 0, "bytes_missing": 0, "bytes_extra": 0,
                     "bytes_outside": 0, "first_short_slot": 0, "first_over_slot": 0}
    assert (readback["slots_over"], readback["bytes_extra"], readback["bytes_outside"]) == (1, 19, 3)
    assert [(s["slot"], s["chunk"], s["expected"], s["first"], s["readback"]) for s in got["slots"]] == [
        (1, 0, LO.SLOT, LO.SLOT + 256, LO.SLOT), (5, 1, 100, 0, 100), (7, 1, 0, LO.SLOT * 0 + 0, 16)]


def lane_split(c0: int, lane_off: int, stride: int, n: int) -> tuple[int, int, int]:
    """ledger_chunk (scrub_kernels.cuh) restated: (slot of c0, bytes there, bytes on the next slot) of one lane's n
    bytes, its vectors at c0 + lane_off + u * stride."""
    room = LO.SLOT - c0 % LO.SLOT
    before = -(-(room - lane_off) // stride) * 16 if room > lane_off else 0
    lo = min(n, before)
    return c0 // LO.SLOT, lo, n - lo


@pytest.mark.parametrize("threads,per", [(512, 16), (1024, 8)])
@pytest.mark.parametrize("c0", [0, 16, 5000 * 16, LO.SLOT - 16, LO.SLOT // 2 + 48])
def test_a_chunk_that_crosses_a_slot_splits_lane_by_lane(threads, per, c0):
    """Concatenated segments could put a chunk across a slot boundary: every lane's split adds up to what it addressed,
    byte for byte on each slot."""
    counts = {}
    for t in range(threads):
        s, lo, hi = lane_split(c0, t * 16, threads * 16, per * 16)
        counts[s] = counts.get(s, 0) + lo
        counts[s + 1] = counts.get(s + 1, 0) + hi
    want = [0] * (c0 // LO.SLOT + 2)
    LO.add(want, c0, c0 + threads * per * 16, +1)
    assert [counts.get(i, 0) for i in range(len(want))] == want


def test_no_plan_puts_a_chunk_across_a_slot():
    """Why the split never runs in a product call: every mapping (VMM) and every fallback segment but the last starts on
    a slot boundary, and chunks are whole slots."""
    for nbytes in (96 * MiB, 64 * MiB + 12345, 10 * MiB + 777):
        for env in ({}, {"CCM_PIPELINE": "0", "CCM_ARENA_MAX_SEGMENT_MB": "3"}, PP.mode_env(0, 0)):
            ranges, mappings, _, _ = CO.call_launches(nbytes, env)
            assert all(o % LO.SLOT == 0 for o, _ in ranges + mappings), (nbytes, env)


# ---------------------------------------------------------------------------------- C ABI
ENTRY_POINTS = ("ccm_scrub_last_ledger", "ccm_last_ledger_slots")


def test_entry_points_are_exported_and_refuse_what_they_must(native):
    lib = native.lib()
    nm = subprocess.run(["nm", "-D", "--defined-only", str(native.LIB_PATH)], capture_output=True, text=True,
                        check=True).stdout
    for fn in ENTRY_POINTS:
        assert fn in native.EXPORTED_SYMBOLS and re.search(rf" T {fn}$", nm, re.M), fn
    for ordinal in (-1, 0, 1 << 12):
        rep = native.CoverLedger(proved=7)
        assert lib.ccm_scrub_last_ledger(ordinal, C.byref(rep)) == native.ERR_NO_CUDA and rep.proved == 0
        n = C.c_uint64(7)
        assert lib.ccm_last_ledger_slots(ordinal, None, 0, C.byref(n)) == native.ERR_NO_CUDA and n.value == 0
    assert lib.ccm_scrub_last_ledger(0, None) == native.ERR_INVALID
    assert lib.ccm_last_ledger_slots(0, None, 0, None) == native.ERR_INVALID
    n = C.c_uint64()
    assert lib.ccm_last_ledger_slots(0, None, 3, C.byref(n)) == native.ERR_INVALID
    assert "ccm_last_ledger_slots: cap 3" in native.last_error()
    assert D.last_ledger(-1) is None and D.last_ledger_slots(-1) is None
    header = (ROOT / "include" / "ccm.h").read_text()
    assert "#define CCM_ABI_VERSION 2 " in header and "#define CCM_LEDGER_SLOT_BYTES (128u << 10)" in header
    assert N.LEDGER_SLOT_BYTES == LO.SLOT
    for fn in ENTRY_POINTS:
        assert re.search(rf"^int {fn}\(", header, re.M), fn


LAYOUT_C = r"""
#include <stddef.h>
#include <stdio.h>
#include "ccm.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu\n", sizeof(ccm_ledger_pass), sizeof(ccm_cover_ledger),
         sizeof(ccm_ledger_slot), offsetof(ccm_cover_ledger, ms_ledger), offsetof(ccm_cover_ledger, exact),
         offsetof(ccm_cover_ledger, pass), offsetof(ccm_ledger_pass, ran), offsetof(ccm_ledger_slot, count),
         offsetof(ccm_ledger_pass, first_over_slot));
  return 0;
}
"""


def test_struct_layouts_match_a_c99_compile(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler")
    (tmp_path / "layout.c").write_text(LAYOUT_C)
    subprocess.run([cc, "-std=c99", "-Wall", "-Werror", "-I", str(ROOT / "include"), str(tmp_path / "layout.c"), "-o",
                    str(tmp_path / "layout")], check=True)
    got = [int(x) for x in subprocess.run([str(tmp_path / "layout")], capture_output=True, text=True,
                                          check=True).stdout.split()]
    want = [C.sizeof(N.LedgerPass), C.sizeof(N.CoverLedger), C.sizeof(N.LedgerSlot), N.CoverLedger.ms_ledger.offset,
            N.CoverLedger.exact.offset, N.CoverLedger.passes.offset, N.LedgerPass.ran.offset, N.LedgerSlot.count.offset,
            N.LedgerPass.first_over_slot.offset]
    assert got == want == [64, 232, 32, 24, 36, 40, 56, 16, 48]


def test_drill_keys_round_trip_and_refuse_what_they_must(native):
    lib = native.lib()
    assert lib.ccm_sim_topology(2, 0) == 0
    v = C.c_int64(-1)
    for key, top in (("cover_repeat", 15), ("cover_lane_drop", 512)):
        assert lib.ccm_sim_get(0, key.encode(), C.byref(v)) == 0 and v.value == 0
        for value in (1, top, 0):
            assert lib.ccm_sim_set(0, key.encode(), value) == 0
            assert lib.ccm_sim_get(0, key.encode(), C.byref(v)) == 0 and v.value == value
        for bad in (-1, top + 1, 1 << 40):
            assert lib.ccm_sim_set(0, key.encode(), bad) == native.ERR_INVALID
            assert f"sim key '{key}' takes 0..{top}" in native.last_error()
    header = (ROOT / "include" / "ccm.h").read_text()
    assert '"cover_repeat"' in header and '"cover_lane_drop"' in header


# ---------------------------------------------------------------------------------- JSON, summary, CLI, worker
def sample_ledger(exact=1) -> CoverLedger:
    passes = [LedgerPass("first", 1, 0, 0, 0, 0, 0, 0, 0), LedgerPass("check", 0, 0, 0, 0, 0, 0, 0, 0),
              LedgerPass("readback", 1, 0 if exact else 3, 0 if exact else 3, 0 if exact else 3 << 17,
                         0 if exact else 3 << 17, 0, 0 if exact else 13, 0)]
    slots = [] if exact else [LedgerSlot(s, 0, LO.SLOT, LO.SLOT, 0, 2 * LO.SLOT) for s in (0, 1, 2)] + \
        [LedgerSlot(s, 0, LO.SLOT, LO.SLOT, 0, 0) for s in (13, 14, 15)]
    return CoverLedger(6 * MiB, 48, 0x7F0000000000, 0.5, 1, exact, passes, slots)


def test_json_carries_the_ledger_only_when_set():
    rep = TM.report()
    base = set(json.loads(json.dumps(rep.as_json())))
    assert rep.ledger is None and "ledger" not in ScrubReport.__dataclass_fields__ and "cover_ledger" not in base
    rep.ledger = sample_ledger(0)
    js = json.loads(json.dumps(rep.as_json()))
    assert set(js) == base | {"cover_ledger"}
    assert ScrubReport.from_json(js).ledger == rep.ledger
    assert CoverLedger.from_json(sample_ledger(1).as_json()) == sample_ledger(1)
    assert GpuError("x").ledger is None


def test_summary_names_the_inexact_pass_and_its_slots():
    assert "every pass walked every slot once (first, readback)" in sample_ledger(1).summary()
    line = sample_ledger(0).summary()
    assert "the readback pass has 3 slots short and 3 over" in line and "slot 14 (chunk 0)" not in line
    assert "slot 0 (chunk 0): expected 131072, first 131072, check 0, read-back 262144" in line and "(+more)" in line
    assert sample_ledger(0).inexact_pass().name == "readback" and sample_ledger(1).inexact_pass() is None


def test_cli_prints_the_keys_the_worker_prints():
    src = (ROOT / "k8s_cc_manager_b200" / "csrc" / "ccm_scrub_cli.cpp").read_text()
    body = src[src.index("static void print_ledger"):src.index("static void print_rcover")]
    printed = set(re.findall(r'\\"(\w+)\\":', body))
    assert printed == ({"cover_ledger"} | set(CoverLedger.__dataclass_fields__) | set(LedgerPass.__dataclass_fields__)
                       | set(LedgerSlot.__dataclass_fields__))
    assert "ccm_last_ledger_slots(ordinal" in body and "keep = 64" in body and D.LEDGER_SLOTS == 64
    assert "proved && ccm_scrub_last_ledger(ordinals[i], &lg) == CCM_OK && lg.proved" in src


def test_worker_prints_the_key_only_for_a_proven_call(monkeypatch, capsys):
    from k8s_cc_manager_b200 import scrub_worker

    def fake_many(devs, n, check="zero", residue=False, triage=False, triage_hold_ms=D.TRIAGE_HOLD_MS,
                  mismatch_triage=False, prove=False):
        rep = TC.zero_report(devs[0].bdf, 0 if exact else N.ERR_UNCOVERED)
        rep.cover = TC.sample_cover(1) if prove else None
        rep.ledger = sample_ledger(int(exact)) if prove else None
        return [rep], 1.0
    monkeypatch.setattr(D, "find_gpus", lambda: ([TC._Dev("0000:01:00.0")], 1))
    monkeypatch.setattr(D, "scrub_and_verify_many", fake_many)
    for exact, argv, rc in ((True, ["--prove"], 0), (False, ["--prove"], 3), (True, [], 0)):
        assert scrub_worker.main(["--bdf", "0000:01:00.0", *argv]) == rc
        rep = json.loads(capsys.readouterr().out.strip().splitlines()[-1])["reports"][0]
        assert ("cover_ledger" in rep) == bool(argv)
        if argv:
            assert CoverLedger.from_json(rep["cover_ledger"]) == sample_ledger(int(exact))


def test_device_layer_fails_a_proven_call_without_its_ledger(monkeypatch):
    monkeypatch.setattr(D, "_arm_prove", lambda o, on: N.OK)
    monkeypatch.setattr(D, "last_cover", lambda o: TC.sample_cover(1))
    ledger = {"value": sample_ledger(1)}
    monkeypatch.setattr(D, "last_ledger", lambda o: ledger["value"])
    lib = type("Lib", (), {"ccm_scrub_verify_many": staticmethod(lambda n, idx, nbytes, res, wall: 0),
                           "ccm_scrub_last_ledger": staticmethod(lambda o, out: N.OK)})()
    monkeypatch.setattr(N, "lib", lambda: lib)
    devs = [type("Dev", (), {"index": 0, "cuda_ordinal": 0, "bdf": "0000:01:00.0"})()]
    reports, _ = D.scrub_and_verify_many(devs, prove=True)
    assert reports[0].status == 0 and reports[0].ledger == sample_ledger(1)
    reports, _ = D.scrub_and_verify_many(devs)
    assert reports[0].ledger is None and reports[0].status == 0
    for value in (CoverLedger(0, 0, 0, 0.0, 0, 0), None):   # did not run, or cannot be read
        ledger["value"] = value
        reports, _ = D.scrub_and_verify_many(devs, prove=True)
        assert reports[0].ledger is None and reports[0].status == N.ERR_UNCOVERED


# ---------------------------------------------------------------------------------- manager
class LedgerGpu(TC.ProofGpu):
    """A clean proving device whose reports carry a ledger: exact, or not (then its call fails as libccm's does)."""

    def __init__(self, bdf, exact=True):
        super().__init__(bdf)
        self.exact = exact

    def _scrub_prove(self, *a, **kw):
        rep = super()._scrub_prove(*a, **kw)
        if kw.get("prove"):
            rep.ledger = sample_ledger(int(self.exact))
            if not self.exact:
                err = GpuError(f"scrub_and_verify on {self.bdf}: HBM coverage ledger failed", N.ERR_UNCOVERED)
                err.cover, err.ledger = rep.cover, rep.ledger
                raise err
        return rep


def ledger_lines(caplog):
    return [(r.levelno, r.getMessage()) for r in caplog.records
            if r.getMessage().startswith("HBM coverage ledger on ")]


def test_per_gpu_gate_logs_and_keeps_the_ledger(monkeypatch, caplog):
    devs = [LedgerGpu(SC.GPU_BDFS[0]), LedgerGpu(SC.GPU_BDFS[1])]
    mgr, _ = TD.manager_for(devs, monkeypatch, scrub_proof="require")
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is True
    assert mgr.last_transition["scrub_cover_ledger"] == {d.bdf: sample_ledger(1) for d in devs}
    assert sorted(ledger_lines(caplog)) == sorted(
        (logging.INFO, f"HBM coverage ledger on {d.bdf}: {sample_ledger(1).summary()}") for d in devs)


def test_an_inexact_ledger_fails_the_gpu_and_is_logged(monkeypatch, caplog):
    devs = [LedgerGpu(SC.GPU_BDFS[0]), LedgerGpu(SC.GPU_BDFS[1], exact=False)]
    mgr, c = TD.manager_for(devs, monkeypatch, scrub_proof="require")
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is False
    assert TC.state(c) == "failed"
    bad = devs[1].bdf
    assert mgr.last_transition["scrub_cover_ledger"][bad] == sample_ledger(0)
    assert (logging.ERROR, f"HBM coverage ledger on {bad}: {sample_ledger(0).summary()}") in ledger_lines(caplog)


def test_an_inexact_ledger_on_an_ok_report_still_fails(monkeypatch, caplog):
    """Whatever status a report carries, the manager does not release a GPU whose ledger is inexact."""
    from k8s_cc_manager_b200 import manager
    TC._native_world(monkeypatch)

    def many(devices, nbytes=0, check="zero", residue=False, triage=False, triage_hold_ms=D.TRIAGE_HOLD_MS,
             mismatch_triage=False, prove=False):
        reps = []
        for i, d in enumerate(devices):
            r = TC.zero_report(d.bdf)
            r.cover, r.ledger = TC.sample_cover(1), sample_ledger(int(i == 0))
            reps.append(r)
        return reps, 1.0
    monkeypatch.setattr(manager._devices, "scrub_and_verify_many", many)
    mgr, c = TD.manager_for(None, monkeypatch, scrub_proof="require")
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is False
    assert TC.state(c) == "failed" and len(mgr.last_transition["scrub_cover_ledger"]) == 2
    assert any("HBM coverage ledger failed on" in r.getMessage() for r in caplog.records)
    assert {lvl for lvl, _ in ledger_lines(caplog)} == {logging.INFO, logging.ERROR}


@pytest.mark.parametrize("exact", [True, False])
def test_worker_process_isolation_keeps_and_enforces_it(monkeypatch, caplog, exact):
    TC._native_world(monkeypatch)
    monkeypatch.setenv("CC_SCRUB_ISOLATION", "process")
    monkeypatch.setenv("CC_SCRUB_PROOF", "require")

    def fake_run(cmd, **kw):
        reps = []
        for b in [cmd[i + 1] for i, a in enumerate(cmd) if a == "--bdf"]:
            r = TC.zero_report(b)
            r.cover, r.ledger = TC.sample_cover(1), sample_ledger(int(exact))
            reps.append(r.as_json())
        return subprocess.CompletedProcess(cmd, 0, json.dumps({"wall_ms": 1.0, "reports": reps}) + "\n", "")
    monkeypatch.setattr(subprocess, "run", fake_run)
    mgr, c = TD.manager_for(None, monkeypatch)
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is exact
    assert len(mgr.last_transition["scrub_cover_ledger"]) == 2
    assert {lvl for lvl, _ in ledger_lines(caplog)} == {logging.INFO if exact else logging.ERROR}
