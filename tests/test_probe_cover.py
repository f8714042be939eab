"""The probe proof on the CPU: the oracle against a brute-force walk of every probe window (unaligned fallback segments,
chunk boundaries inside a page, the drill on each step); the C ABI without a CUDA device (exports, layouts from a C99
compile, drill keys); the proving twins' resource usage; ProbeCoverReport in ScrubReport's and GpuError's JSON; the
worker and the CLI; and the manager's policy when CC_SCRUB_PROOF and CC_SCRUB_ALIAS_PROBE are both required."""
from __future__ import annotations

import ctypes as C
import json
import logging
import re
import shutil
import subprocess
from pathlib import Path

import pytest

import probe_cover_oracle as PCO
import scenarios as SC
import test_alias_probe as TA
import test_cover_proof as TC
import test_dirt_locate as TD
from k8s_cc_manager_b200 import _native as N
from k8s_cc_manager_b200 import devices as D
from k8s_cc_manager_b200.devices import GpuError, ProbeCoverPage, ProbeCoverReport, ProbeCoverStep, ScrubReport

ROOT = Path(__file__).resolve().parents[1]
MiB = 1 << 20
PAGE = PCO.PAGE
BASE = (3 << 34) + (5 << 21)


# ---------------------------------------------------------------------------------- oracle against a brute-force walk
def brute(chunks, skip=0):
    """{page: bytes}: every 4096-aligned 32-byte window inside a chunk, byte by byte onto the page of its offset; the
    first `skip` windows of the first chunk with any left out."""
    pages = {}
    pending = skip
    for a, n, off in chunks:
        ws = [w for w in range(-(-a // 4096) * 4096, a + n, 4096) if w + 32 <= a + n]
        if not ws:
            continue
        drop, pending = min(pending, len(ws)), 0
        for w in ws[drop:]:
            for b in range(32):
                p = (off + w - a + b) // PAGE
                pages[p] = pages.get(p, 0) + 1
    return pages


GEOMETRIES = {
    "vmm": PCO.vmm_chunks(BASE, [(0, 2 * MiB), (2 * MiB, 4 * MiB), (6 * MiB, 8 * MiB)]),
    "vmm_odd_chunks": PCO.vmm_chunks(BASE, [(0, 3 * MiB), (3 * MiB, MiB + 4096), (4 * MiB + 4096, 5 * MiB - 4096)]),
    "fallback_256": PCO.arena_chunks([(BASE + 256, 3 * MiB), (BASE - 40 * MiB + 512, 3 * MiB), (BASE + 9 * MiB, MiB + 777)]),
    "fallback_odd": PCO.arena_chunks([(BASE + 7, 3 * MiB + 5), (BASE + 20 * MiB + 4090, 2 * MiB + 16),
                                      (BASE + 90 * MiB + 17, 4096 * 3)]),
    "boundary_inside_a_page": PCO.arena_chunks([(BASE, PAGE + 100), (BASE + 8 * MiB + 4000, PAGE - 100)]),
    "window_across_a_page": [(BASE, 4096 * 3, PAGE - 4096 * 2 - 16)],
    "tiny": PCO.arena_chunks([(BASE + 1, 31), (BASE + 4096, 32), (BASE + 3 * 4096 - 1, 33)]),
}


@pytest.mark.parametrize("name", list(GEOMETRIES))
@pytest.mark.parametrize("skip", [0, 1, 5, 700, 1 << 20])
def test_oracle_matches_a_brute_force_walk(name, skip):
    chunks = GEOMETRIES[name]
    assert PCO.expected(chunks) == brute(chunks)
    assert PCO._count(chunks, skip) == {p: b for p, b in brute(chunks, skip).items() if b}
    assert sum(brute(chunks).values()) == 32 * PCO.windows(chunks)


@pytest.mark.parametrize("step", [0, 1, 2, 3])
def test_drill_misses_exactly_the_first_windows_of_its_step(step):
    chunks = PCO.arena_chunks([(BASE + 7, 100), (BASE + 256, 6 * MiB + 300), (BASE + 90 * MiB, 4 * MiB)])
    total = PCO.windows(chunks)
    first = PCO.chunk_windows(BASE + 256, 6 * MiB + 300)[1]   # the first chunk has no window: the drill skips it
    for k in (0, 3, 600, first + 50):
        rep = PCO.report(chunks, k, step)
        hit = (2 if step == 0 else step) - 1
        missing = min(k, first)
        assert rep["windows_expected"] == total
        assert rep["covered"] == int(missing == 0)
        for s in range(3):
            want = missing if s == hit else 0
            assert rep["steps"][s]["windows_missing"] == want
            assert rep["steps"][s]["windows_counted"] == total - want
        if missing:
            short = rep["steps"][hit]
            assert short["first_short_page"] == 0 and short["pages_short"] == -(-missing // 512)
            assert all(c[hit] < e for e, c in rep["pages"].values())


def test_a_clean_call_counts_every_window_of_every_page():
    chunks = PCO.vmm_chunks(BASE, [(0, 1024 * MiB), (1024 * MiB, 512 * MiB)])
    rep = PCO.report(chunks)
    assert rep["covered"] == 1 and rep["pages"] == {} and rep["windows_expected"] == 1536 * 256
    assert set(PCO.expected(chunks).values()) == {512 * 32}


# ---------------------------------------------------------------------------------- C ABI
ENTRY_POINTS = ("ccm_scrub_last_probe_cover", "ccm_last_probe_cover_pages")


def test_entry_points_are_exported_and_refuse_what_they_must(native):
    lib = N.lib()
    nm = subprocess.run(["nm", "-D", "--defined-only", str(N.LIB_PATH)], capture_output=True, text=True,
                        check=True).stdout
    for fn in ENTRY_POINTS:
        assert fn in N.EXPORTED_SYMBOLS and re.search(rf" T {fn}$", nm, re.M), fn
    for ordinal in (-1, 1 << 12):
        rep = N.ProbeCover(proved=7)
        assert lib.ccm_scrub_last_probe_cover(ordinal, C.byref(rep)) == N.ERR_NO_CUDA and rep.proved == 0
        n = C.c_uint64(7)
        assert lib.ccm_last_probe_cover_pages(ordinal, None, 0, C.byref(n)) == N.ERR_NO_CUDA and n.value == 0
    assert lib.ccm_scrub_last_probe_cover(0, None) == N.ERR_INVALID
    assert lib.ccm_last_probe_cover_pages(0, None, 0, None) == N.ERR_INVALID
    n = C.c_uint64()
    assert lib.ccm_last_probe_cover_pages(0, None, 3, C.byref(n)) == N.ERR_INVALID
    assert "ccm_last_probe_cover_pages: cap 3" in N.last_error()
    assert D.last_probe_cover(-1) is None and D.last_probe_cover_pages(-1) is None
    header = (ROOT / "include" / "ccm.h").read_text()
    for fn in ENTRY_POINTS:
        assert re.search(rf"^int {fn}\(", header, re.M), fn
    assert '"probe_skip"' in header and '"probe_skip_step"' in header


LAYOUT_C = r"""
#include <stddef.h>
#include <stdio.h>
#include "ccm.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu\n", sizeof(ccm_probe_cover_step), sizeof(ccm_probe_cover),
         sizeof(ccm_probe_cover_page), offsetof(ccm_probe_cover, ms_prove), offsetof(ccm_probe_cover, proved),
         offsetof(ccm_probe_cover, covered), offsetof(ccm_probe_cover, step), offsetof(ccm_probe_cover_step, ran),
         offsetof(ccm_probe_cover_step, first_short_page), offsetof(ccm_probe_cover_page, expected),
         offsetof(ccm_probe_cover_page, count));
  return 0;
}
"""


def test_struct_layouts_match_a_c99_compile(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "layout.c"
    src.write_text(LAYOUT_C)
    subprocess.run([cc, "-std=c99", "-Wall", "-Werror", "-I", str(ROOT / "include"), str(src), "-o",
                    str(tmp_path / "layout")], check=True)
    got = [int(x) for x in subprocess.run([str(tmp_path / "layout")], capture_output=True, text=True,
                                          check=True).stdout.split()]
    want = [C.sizeof(N.ProbeCoverStep), C.sizeof(N.ProbeCover), C.sizeof(N.ProbeCoverPage), N.ProbeCover.ms_prove.offset,
            N.ProbeCover.proved.offset, N.ProbeCover.covered.offset, N.ProbeCover.steps.offset,
            N.ProbeCoverStep.ran.offset, N.ProbeCoverStep.first_short_page.offset, N.ProbeCoverPage.expected.offset,
            N.ProbeCoverPage.count.offset]
    assert got == want == [64, 224, 32, 16, 24, 28, 32, 56, 48, 12, 16]


def test_drill_keys_round_trip_and_refuse_what_they_must(native):
    lib = N.lib()
    assert lib.ccm_sim_topology(2, 0) == 0
    assert lib.ccm_sim_set(-1, b"cuda_ordinal", -1) == 0
    v = C.c_int64(-1)
    assert lib.ccm_sim_get(0, b"probe_skip", C.byref(v)) == 0 and v.value == 0
    assert lib.ccm_sim_get(0, b"probe_skip_step", C.byref(v)) == 0 and v.value == 2
    assert lib.ccm_sim_set(0, b"probe_skip", 9) == 0 and lib.ccm_sim_get(0, b"probe_skip", C.byref(v)) == 0
    assert v.value == 9
    for value, stored in ((1, 1), (2, 2), (3, 3), (0, 2)):
        assert lib.ccm_sim_set(0, b"probe_skip_step", value) == 0
        assert lib.ccm_sim_get(0, b"probe_skip_step", C.byref(v)) == 0 and v.value == stored
    for bad in (-1, 4, 1 << 40):
        assert lib.ccm_sim_set(0, b"probe_skip_step", bad) == N.ERR_INVALID
        assert "sim key 'probe_skip_step' takes 0..3" in N.last_error()
    assert lib.ccm_sim_get(1, b"probe_skip", C.byref(v)) == 0 and v.value == 0
    assert lib.ccm_sim_set(0, b"probe_skip", 0) == 0


def test_proving_twins_have_no_spills_and_no_stack():
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not Path(cuobjdump).exists():
        pytest.skip("cuobjdump is not installed")
    out = subprocess.run([cuobjdump, "--dump-resource-usage", str(N.LIB_PATH)], capture_output=True, text=True,
                         check=True).stdout
    found = {}
    lines = out.splitlines()
    for i, line in enumerate(lines):
        m = re.search(r"Function (\S*cover_probe_(fill|check|reread)_pass\S*):", line)
        if m:
            found[m.group(2)] = lines[i + 1]
    assert set(found) == {"fill", "check", "reread"}
    for usage in found.values():
        assert re.search(r"STACK:0\b", usage) and re.search(r"LOCAL:0\b", usage), usage


# ---------------------------------------------------------------------------------- reports and JSON
def sample_probe_cover(covered=1) -> ProbeCoverReport:
    steps = [ProbeCoverStep(name, 1, 393216, 0, 0, 0, 0, 0, 0) for name in N.PROBE_STEPS]
    pages = []
    if not covered:
        steps[1] = ProbeCoverStep("P2", 1, 393211, 5, 0, 0, 1, 0, 0)
        pages = [ProbeCoverPage(0, 0, 16384, 16384, 16224, 16384)]
    return ProbeCoverReport(393216, 1 << 40, 0.2, 1, covered, steps, pages)


def test_json_carries_the_report_only_when_a_proof_ran():
    rep = TC.zero_report("0000:01:00.0")
    assert "probe_cover" not in rep.as_json()
    rep.probe = TA.sample_probe()
    rep.probe_cover = sample_probe_cover(0)
    d = rep.as_json()
    assert d["probe_cover"]["steps"][1]["windows_missing"] == 5
    back = ScrubReport.from_json(json.loads(json.dumps(d)))
    assert back.probe_cover == sample_probe_cover(0) and back.probe == TA.sample_probe()
    assert GpuError("x").probe_cover is None


def test_summary_names_the_short_step_and_its_pages():
    assert sample_probe_cover(1).summary() == "393216 probe windows: every step took every window once (P1, P2, P3)"
    s = sample_probe_cover(0).summary()
    assert "step P2 counted 393211 windows (5 missing, 0 extra) with 1 pages short, first short page 0" in s
    assert "page 0 (chunk 0): expected 16384, P1 16384, P2 16224, P3 16384" in s


def test_cli_prints_the_keys_the_worker_prints():
    src = (ROOT / "k8s_cc_manager_b200" / "csrc" / "ccm_scrub_cli.cpp").read_text()
    body = src[src.index("static void print_pcover(const ccm_probe_cover& c, int ordinal) {"):]
    printed = set(re.findall(r'\\"(\w+)\\":', body))
    assert printed == ({"probe_cover"} | set(ProbeCoverReport.__dataclass_fields__)
                       | set(ProbeCoverStep.__dataclass_fields__) | set(ProbeCoverPage.__dataclass_fields__))
    assert "prove && ran_probe && ccm_scrub_last_probe_cover(ordinals[i], &pc)" in src
    # a proving call that probed and has no proof prints ERR_UNCOVERED as its status, not only a failing exit code
    assert "r.status == CCM_OK && prove && ran_probe && !probe_proved ? (int)CCM_ERR_UNCOVERED : r.status" in src
    assert "r.ms_total, r.segments, status, r.release_deferred" in src


def test_worker_prints_the_key_only_when_a_proven_call_probed(monkeypatch, capsys):
    from k8s_cc_manager_b200 import scrub_worker

    def fake_many(devs, n, check="zero", residue=False, triage=False, triage_hold_ms=D.TRIAGE_HOLD_MS,
                  mismatch_triage=False, prove=False, probe=False):
        rep = TC.zero_report(devs[0].bdf, 0 if covered else N.ERR_UNCOVERED)
        rep.cover = TC.sample_cover(1) if prove else None
        rep.probe = TA.sample_probe() if probe else None
        rep.probe_cover = sample_probe_cover(int(covered)) if prove and probe else None
        return [rep], 1.0
    monkeypatch.setattr(D, "find_gpus", lambda: ([TC._Dev("0000:01:00.0")], 1))
    monkeypatch.setattr(D, "scrub_and_verify_many", fake_many)
    covered = True
    for argv, key in ((["--prove", "--probe"], True), (["--prove"], False), (["--probe"], False), ([], False)):
        assert scrub_worker.main(["--bdf", "0000:01:00.0", *argv]) == 0
        rep = json.loads(capsys.readouterr().out.strip().splitlines()[-1])["reports"][0]
        assert ("probe_cover" in rep) == key
    covered = False
    assert scrub_worker.main(["--bdf", "0000:01:00.0", "--prove", "--probe"]) == 3
    rep = json.loads(capsys.readouterr().out.strip().splitlines()[-1])["reports"][0]
    assert rep["status"] == N.ERR_UNCOVERED and ProbeCoverReport.from_json(rep["probe_cover"]) == sample_probe_cover(0)


def test_fan_out_attaches_the_proof_only_to_a_proven_call_that_probed(monkeypatch):
    monkeypatch.setattr(D, "_arm_prove", lambda o, on: N.OK)
    monkeypatch.setattr(D, "_arm_probe", lambda o, on: N.OK)
    monkeypatch.setattr(D, "last_probe", lambda o: TA.sample_probe())
    monkeypatch.setattr(D, "last_cover", lambda o: TC.sample_cover(1))
    proof = {"value": sample_probe_cover(1)}
    monkeypatch.setattr(D, "last_probe_cover", lambda o: proof["value"])
    lib = type("Lib", (), {"ccm_scrub_verify_many": staticmethod(lambda n, idx, nbytes, res, wall: 0),
                           "ccm_scrub_last_probe_cover": staticmethod(lambda o, out: N.OK)})()
    monkeypatch.setattr(N, "lib", lambda: lib)
    devs = [type("Dev", (), {"index": 0, "cuda_ordinal": 0, "bdf": "0000:01:00.0"})()]
    reports, _ = D.scrub_and_verify_many(devs, prove=True, probe=True)
    assert reports[0].status == 0 and reports[0].probe_cover == sample_probe_cover(1)
    reports, _ = D.scrub_and_verify_many(devs, probe=True)
    assert reports[0].probe_cover is None and reports[0].status == 0
    # a proof that did not run (proved == 0) and one that cannot be read (None) both fail the call
    for value in (ProbeCoverReport(0, 0, 0.0, 0, 0), None):
        proof["value"] = value
        reports, _ = D.scrub_and_verify_many(devs, prove=True, probe=True)
        assert reports[0].probe_cover is None and reports[0].status == N.ERR_UNCOVERED


def test_a_single_device_call_without_a_readable_proof_fails(native, monkeypatch):
    lib = native.lib()
    assert lib.ccm_sim_topology(1, 0) == 0
    gpu = [d for d in D.find_gpus()[0] if d.is_gpu()][0]
    monkeypatch.setattr(D, "_arm_prove", lambda o, on: N.OK)
    monkeypatch.setattr(D, "_arm_probe", lambda o, on: N.OK)
    monkeypatch.setattr(D, "last_probe", lambda o: TA.sample_probe())
    monkeypatch.setattr(D, "last_cover", lambda o: TC.sample_cover(1))
    monkeypatch.setattr(D, "last_probe_cover", lambda o: None)
    calls = []
    real = N.lib()
    fake = type("Lib", (), {"__getattr__": lambda self, name: getattr(real, name),
                            "ccm_scrub_verify": staticmethod(lambda *a: calls.append(a) or N.OK)})()
    monkeypatch.setattr(N, "lib", lambda: fake)
    with pytest.raises(GpuError) as err:
        gpu.scrub_and_verify(prove=True, probe=True)
    assert len(calls) == 1 and err.value.status == N.ERR_UNCOVERED and "the probe proof did not run" in str(err.value)
    assert err.value.probe == TA.sample_probe() and err.value.probe_cover is None


# ---------------------------------------------------------------------------------- manager
class BothGpu(TA.ProbeGpu):
    """A clean zero-gate device that takes `prove` and `probe`; proof: what its probe proof is (None: a library that
    does not attach one, 0: a short step)."""

    def __init__(self, bdf, proof=1):
        super().__init__(bdf)
        self.proof = proof

    def _scrub_probe(self, nbytes=0, check="zero", residue=False, triage=False, triage_hold_ms=100,
                     mismatch_triage=False, prove=False, probe=False):
        rep = super()._scrub_probe(nbytes, check, residue, triage, triage_hold_ms, mismatch_triage, prove, probe)
        if prove and probe and self.proof is not None:
            if not self.proof:
                err = GpuError(f"scrub_and_verify on {self.bdf}: HBM alias probe proof failed", N.ERR_UNCOVERED)
                err.cover, err.probe, err.probe_cover = rep.cover, rep.probe, sample_probe_cover(0)
                raise err
            rep.probe_cover = sample_probe_cover(1)
        return rep


def proof_lines(caplog):
    return [(r.levelno, r.getMessage()) for r in caplog.records
            if r.getMessage().startswith("HBM alias probe proof on ")]


BOTH = dict(scrub_proof="require", scrub_alias_probe="require")


def test_both_required_logs_and_keeps_the_proof(monkeypatch, caplog):
    devs = [BothGpu(SC.GPU_BDFS[0]), BothGpu(SC.GPU_BDFS[1])]
    mgr, _ = TD.manager_for(devs, monkeypatch, **BOTH)
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is True
    assert mgr.last_transition["scrub_probe_cover"] == {d.bdf: sample_probe_cover(1) for d in devs}
    assert sorted(proof_lines(caplog)) == sorted(
        (logging.INFO, f"HBM alias probe proof on {d.bdf}: {sample_probe_cover(1).summary()}") for d in devs)


@pytest.mark.parametrize("knobs", [dict(scrub_proof="require"), dict(scrub_alias_probe="require"), dict()])
def test_one_knob_alone_asks_for_no_probe_proof(monkeypatch, caplog, knobs):
    devs = [BothGpu(SC.GPU_BDFS[0], proof=None)]
    mgr, _ = TD.manager_for(devs, monkeypatch, **knobs)
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is True
    assert "scrub_probe_cover" not in mgr.last_transition and proof_lines(caplog) == []


def test_a_call_whose_probe_proof_did_not_run_fails_under_both(monkeypatch, caplog):
    """The device layer turns a proof that was asked for and did not run into ERR_UNCOVERED."""
    from k8s_cc_manager_b200 import manager
    TC._native_world(monkeypatch)
    monkeypatch.setattr(D, "_arm_prove", lambda o, on: N.OK)
    monkeypatch.setattr(D, "_arm_probe", lambda o, on: N.OK)
    monkeypatch.setattr(D, "last_probe", lambda o: TA.sample_probe())
    monkeypatch.setattr(D, "last_cover", lambda o: TC.sample_cover(1))
    monkeypatch.setattr(D, "last_probe_cover", lambda o: ProbeCoverReport(0, 0, 0.0, 0, 0))
    real_many = D.scrub_and_verify_many

    def many(devices, nbytes=0, check="zero", residue=False, triage=False, triage_hold_ms=D.TRIAGE_HOLD_MS,
             mismatch_triage=False, prove=False, probe=False):
        if not (prove and probe):   # the inner fan-out: every device clean
            return [TC.zero_report(d.bdf) for d in devices], 1.0
        return real_many(devices, nbytes, check, residue, triage, triage_hold_ms, mismatch_triage, prove, probe)
    monkeypatch.setattr(manager._devices, "scrub_and_verify_many", many)
    mgr, c = TD.manager_for(None, monkeypatch, **BOTH)
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is False
    assert TC.state(c) == "failed"
    assert any(f"status={N.ERR_UNCOVERED}" in r.getMessage() for r in caplog.records)


def test_a_report_whose_probe_proof_did_not_run_fails_under_both(monkeypatch, caplog):
    class NotProvedGpu(BothGpu):
        def _scrub_probe(self, *a, **kw):
            rep = super()._scrub_probe(*a, **kw)
            rep.probe_cover = ProbeCoverReport(0, 0, 0.0, 0, 0)
            return rep
    devs = [BothGpu(SC.GPU_BDFS[0]), NotProvedGpu(SC.GPU_BDFS[1])]
    mgr, c = TD.manager_for(devs, monkeypatch, **BOTH)
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is False
    assert TC.state(c) == "failed"
    assert any(f"HBM alias probe proof failed on {devs[1].bdf}" in r.getMessage() for r in caplog.records)


def test_an_uncovered_probe_fails_the_transition_and_logs_its_short_step(monkeypatch, caplog):
    devs = [BothGpu(SC.GPU_BDFS[0]), BothGpu(SC.GPU_BDFS[1], proof=0)]
    mgr, c = TD.manager_for(devs, monkeypatch, **BOTH)
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is False
    assert TC.state(c) == "failed"
    bad = devs[1].bdf
    assert mgr.last_transition["scrub_probe_cover"][bad] == sample_probe_cover(0)
    assert (logging.ERROR, f"HBM alias probe proof on {bad}: {sample_probe_cover(0).summary()}") in proof_lines(caplog)


@pytest.mark.parametrize("covered", [True, False])
def test_native_fan_out_and_a_status_ok_report_with_a_short_step(monkeypatch, caplog, covered):
    from k8s_cc_manager_b200 import manager
    TC._native_world(monkeypatch)

    def fake_many(devices, nbytes=0, check="zero", residue=False, triage=False, triage_hold_ms=D.TRIAGE_HOLD_MS,
                  mismatch_triage=False, prove=False, probe=False):
        reps = []
        for d in devices:
            r = TC.zero_report(d.bdf)   # status 0 either way: the manager reads the proof itself
            r.cover, r.probe = TC.sample_cover(1), TA.sample_probe()
            r.probe_cover = sample_probe_cover(int(covered)) if prove and probe else None
            reps.append(r)
        return reps, 1.0
    monkeypatch.setattr(manager._devices, "scrub_and_verify_many", fake_many)
    mgr, c = TD.manager_for(None, monkeypatch, **BOTH)
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is covered
    assert len(mgr.last_transition["scrub_probe_cover"]) == 2
    assert {lvl for lvl, _ in proof_lines(caplog)} == {logging.INFO if covered else logging.ERROR}
    if not covered:
        assert TC.state(c) == "failed"
        assert any("HBM alias probe proof failed on" in r.getMessage() for r in caplog.records)


def test_worker_process_passes_it(monkeypatch, caplog):
    TC._native_world(monkeypatch)
    monkeypatch.setenv("CC_SCRUB_ISOLATION", "process")
    monkeypatch.setenv("CC_SCRUB_PROOF", "require")
    monkeypatch.setenv("CC_SCRUB_ALIAS_PROBE", "require")
    cmds = []

    def fake_run(cmd, **kw):
        cmds.append(cmd)
        reps = []
        for b in [cmd[i + 1] for i, a in enumerate(cmd) if a == "--bdf"]:
            r = TC.zero_report(b)
            r.cover, r.probe, r.probe_cover = TC.sample_cover(1), TA.sample_probe(), sample_probe_cover(1)
            reps.append(r.as_json())
        return subprocess.CompletedProcess(cmd, 0, json.dumps({"wall_ms": 1.0, "reports": reps}) + "\n", "")
    monkeypatch.setattr(subprocess, "run", fake_run)
    mgr, _ = TD.manager_for(None, monkeypatch)
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is True
    assert "--prove" in cmds[0] and "--probe" in cmds[0]
    assert len(mgr.last_transition["scrub_probe_cover"]) == 2 and len(proof_lines(caplog)) == 2
