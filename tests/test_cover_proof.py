"""The coverage proof on the CPU: the oracle against a byte-by-byte walk of the kernels' grabs, with and without
cover_skip on each pass; the C ABI without a CUDA device (exports, struct layouts from a C99 compile, the status and
its text, the drill keys and their refusals); and CoverReport in ScrubReport's and GpuError's JSON."""
from __future__ import annotations

import ctypes as C
import inspect
import json
import re
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

import cover_oracle as CO
import test_tag_mismatch as TM
from k8s_cc_manager_b200 import _native as N
from k8s_cc_manager_b200 import devices as D
from k8s_cc_manager_b200.devices import CoverPage, CoverPass, CoverReport, GpuError, ScrubReport

ROOT = Path(__file__).resolve().parents[1]
MiB = 1 << 20


# ---------------------------------------------------------------------------------- oracle against a walk of the grabs
def walk(counts: np.ndarray, addr: int, off: int, n: int, skip: int, descending: bool) -> None:
    """One default-frame launch over [off, off + n) at address `addr`, byte by byte: the grab word starts at `skip`,
    each grabbed chunk is walked at its position (descending: from the top), then the leftover vectors and the ragged
    head and tail bytes.  Adds 1 to counts[o] for every byte it processes."""
    head = min((CO.ALIGN - addr % CO.ALIGN) % CO.ALIGN, n)
    vecs = (n - head) // 16
    nchunks = vecs * 16 // CO.CHUNK
    grab = skip
    while grab < nchunks:
        pos = nchunks - 1 - grab if descending else grab
        counts[off + head + pos * CO.CHUNK: off + head + (pos + 1) * CO.CHUNK] += 1
        grab += 1
    for v in range(nchunks * CO.CHUNK // 16, vecs):
        counts[off + head + 16 * v: off + head + 16 * v + 16] += 1
    counts[off: off + head] += 1
    counts[off + head + vecs * 16: off + n] += 1


def pages_of(counts: np.ndarray) -> list[int]:
    return [int(counts[p: p + CO.PAGE].sum()) for p in range(0, len(counts), CO.PAGE)]


GEOMETRIES = [(5 * MiB + 77, [(0, 5 * MiB + 77)]),                                       # one ragged range
              (6 * MiB + 16 * 9, [(0, 2 * MiB), (2 * MiB, 4 * MiB + 16 * 9)]),               # leftover vectors
              (7 * MiB + 5, [(0, 3 * MiB), (3 * MiB, 3 * MiB), (6 * MiB, MiB + 5)])]         # segments inside pages


@pytest.mark.parametrize("mapped,ranges", GEOMETRIES)
@pytest.mark.parametrize("tagged", [False, True])
@pytest.mark.parametrize("drill", [None, ("first", 1), ("first", 9), ("check", 2), ("readback", 1), ("readback", 3),
                                   ("readback", 10 ** 6)])
def test_oracle_matches_a_walk_of_the_grabs(mapped, ranges, tagged, drill):
    first_of = {p: CO.first_launch(p, tagged, ranges, ranges, True, mapped) for p in CO.PASSES}
    walked = {}
    for p in CO.PASSES:
        if p == "check" and not tagged:
            continue
        counts = np.zeros(mapped, np.uint32)
        for i, (off, n) in enumerate(ranges):
            k = drill[1] if drill and drill[0] == p and (off, n) == first_of[p] and i == 0 else 0
            walk(counts, off, off, n, k, p == "readback")
        walked[p] = pages_of(counts)
    rep = CO.report(mapped, tagged, (drill[0], drill[1], *first_of[drill[0]]) if drill and first_of[drill[0]] else None)
    want = CO.expected(mapped)
    for p, got in walked.items():
        row = rep["passes"][p]
        assert row["bytes_counted"] == sum(got) and row["bytes_missing"] == sum(want) - sum(got)
        short = [i for i, (g, w) in enumerate(zip(got, want)) if g < w]
        assert row["pages_short"] == len(short) and row["first_short_page"] == (short[0] if short else 0)
    assert [pg["page"] for pg in rep["pages"]] == sorted({i for got in walked.values()
                                                          for i, (g, w) in enumerate(zip(got, want)) if g != w})
    assert rep["covered"] == (drill is None or (drill[0] == "check" and not tagged))
    if not tagged:
        assert rep["passes"]["check"] == {"ran": 0}


def test_a_clean_call_counts_every_page_exactly():
    assert CO.expected(5 * MiB + 7) == [CO.PAGE, CO.PAGE, MiB + 7]
    assert CO.report(5 * MiB + 7, True)["pages"] == [] and CO.report(0, False)["covered"]


# ---------------------------------------------------------------------------------- C ABI
ENTRY_POINTS = ("ccm_scrub_prove", "ccm_scrub_last_cover", "ccm_last_cover_pages")


def test_entry_points_are_exported_and_refuse_what_they_must(native):
    lib = native.lib()
    nm = subprocess.run(["nm", "-D", "--defined-only", str(native.LIB_PATH)], capture_output=True, text=True,
                        check=True).stdout
    for fn in ENTRY_POINTS:
        assert fn in native.EXPORTED_SYMBOLS and re.search(rf" T {fn}$", nm, re.M), fn
    for ordinal in (-1, 0, 1 << 12):
        assert lib.ccm_scrub_prove(ordinal, 1) == native.ERR_NO_CUDA
        assert lib.ccm_scrub_prove(ordinal, 0) == native.ERR_NO_CUDA
        rep = native.CoverReport(proved=7)
        assert lib.ccm_scrub_last_cover(ordinal, C.byref(rep)) == native.ERR_NO_CUDA and rep.proved == 0
        n = C.c_uint64(7)
        assert lib.ccm_last_cover_pages(ordinal, None, 0, C.byref(n)) == native.ERR_NO_CUDA and n.value == 0
    assert lib.ccm_scrub_last_cover(0, None) == native.ERR_INVALID
    assert lib.ccm_last_cover_pages(0, None, 0, None) == native.ERR_INVALID
    n = C.c_uint64()
    assert lib.ccm_last_cover_pages(0, None, 3, C.byref(n)) == native.ERR_INVALID
    assert "ccm_last_cover_pages: cap 3" in native.last_error()
    assert D.last_cover(-1) is None and D.last_cover_pages(-1) is None


def test_status_and_its_text(native):
    assert native.ERR_UNCOVERED == -14
    assert native.strerror(-14) == "a scrub gate pass did not walk every mapped byte exactly once (coverage proof)"
    header = (ROOT / "include" / "ccm.h").read_text()
    assert re.search(r"CCM_ERR_UNCOVERED = -14 ", header)
    assert "#define CCM_ABI_VERSION 2 " in header
    for fn in ENTRY_POINTS:
        assert re.search(rf"^int {fn}\(", header, re.M), fn
    assert '"cover_skip"' in header and '"cover_pass"' in header


LAYOUT_C = r"""
#include <stddef.h>
#include <stdio.h>
#include "ccm.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu\n", sizeof(ccm_cover_pass), sizeof(ccm_cover_report),
         sizeof(ccm_cover_page), offsetof(ccm_cover_report, ms_prove), offsetof(ccm_cover_report, proved),
         offsetof(ccm_cover_report, pass), offsetof(ccm_cover_pass, ran), offsetof(ccm_cover_page, expected),
         offsetof(ccm_cover_page, count), offsetof(ccm_cover_pass, first_short_page));
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
    want = [C.sizeof(N.CoverPass), C.sizeof(N.CoverReport), C.sizeof(N.CoverPage), N.CoverReport.ms_prove.offset,
            N.CoverReport.proved.offset, N.CoverReport.passes.offset, N.CoverPass.ran.offset,
            N.CoverPage.expected.offset, N.CoverPage.count.offset, N.CoverPass.first_short_page.offset]
    assert got == want == [64, 232, 32, 24, 32, 40, 56, 12, 16, 48]


def test_drill_keys_round_trip_and_refuse_what_they_must(native):
    lib = native.lib()
    assert lib.ccm_sim_topology(2, 0) == 0
    assert lib.ccm_sim_set(-1, b"cuda_ordinal", -1) == 0
    v = C.c_int64(-1)
    assert lib.ccm_sim_get(0, b"cover_skip", C.byref(v)) == 0 and v.value == 0
    assert lib.ccm_sim_get(0, b"cover_pass", C.byref(v)) == 0 and v.value == N.COVER_PASSES.index("readback") + 1
    assert lib.ccm_sim_set(0, b"cover_skip", 12) == 0 and lib.ccm_sim_get(0, b"cover_skip", C.byref(v)) == 0
    assert v.value == 12
    for value, stored in ((1, 1), (2, 2), (3, 3), (0, 3)):
        assert lib.ccm_sim_set(0, b"cover_pass", value) == 0
        assert lib.ccm_sim_get(0, b"cover_pass", C.byref(v)) == 0 and v.value == stored
    for bad in (-1, 4, 1 << 40):
        assert lib.ccm_sim_set(0, b"cover_pass", bad) == native.ERR_INVALID
        assert "sim key 'cover_pass' takes 0..3" in native.last_error()
    assert lib.ccm_sim_get(1, b"cover_skip", C.byref(v)) == 0 and v.value == 0
    assert lib.ccm_sim_set(0, b"cover_skip", 0) == 0


# ---------------------------------------------------------------------------------- device API and JSON
def sample_cover(covered=0) -> CoverReport:
    passes = [CoverPass("first", 1, 6 * MiB, 0, 0, 0, 0, 0, 0), CoverPass("check", 0, 0, 0, 0, 0, 0, 0, 0),
              CoverPass("readback", 1, 6 * MiB - (0 if covered else 3 << 17), 0 if covered else 3 << 17, 0, 0,
                        0 if covered else 1, 0, 0 if covered else 2)]
    pages = [] if covered else [CoverPage(2, 0, CO.PAGE, CO.PAGE, 0, CO.PAGE - (3 << 17))]
    return CoverReport(6 * MiB, 3, 0x7F0000000000, 0.25, 1, covered, passes, pages)


def test_json_carries_the_report_only_when_a_proof_ran():
    rep = TM.report()
    base = set(json.loads(json.dumps(rep.as_json())))
    assert rep.cover is None and "cover" not in ScrubReport.__dataclass_fields__ and "cover" not in base
    rep.cover = sample_cover()
    js = json.loads(json.dumps(rep.as_json()))
    assert set(js) == base | {"cover"}
    back = ScrubReport.from_json(js)
    assert back.cover == rep.cover and back.dirt is None
    assert CoverReport.from_json(sample_cover(1).as_json()) == sample_cover(1)
    assert GpuError("x").cover is None


def test_summary_names_the_short_pass_and_its_pages():
    assert "every pass covered every byte once (first, readback)" in sample_cover(1).summary()
    line = sample_cover().summary()
    assert "the readback pass counted" in line and "393216 missing" in line and "page 2 (chunk 0)" in line
    assert sample_cover().short_pass().name == "readback" and sample_cover(1).short_pass() is None


def test_device_api_takes_prove():
    for fn in (D.NvidiaDevice.scrub_and_verify, D.ScrubbingProxy.scrub_and_verify, D.scrub_and_verify_many):
        assert inspect.signature(fn).parameters["prove"].default is False


class _Native:
    def __init__(self):
        self.calls = []

    def scrub_and_verify(self, nbytes=0, **kw):
        self.calls.append(kw)
        return "report"


def test_proxy_passes_prove_only_when_it_is_set():
    native = _Native()
    proxy = D.ScrubbingProxy(type("Foreign", (), {"bdf": "0000:01:00.0"})(), native)
    proxy.scrub_and_verify(0)
    proxy.scrub_and_verify(0, check="tagged", residue=True, prove=True)
    assert native.calls[0] == {} and native.calls[1]["prove"] is True and native.calls[1]["residue"] is True
    assert native.calls[1]["check"] == "tagged"


def test_a_device_without_cuda_fails_an_armed_call(native):
    lib = native.lib()
    assert lib.ccm_sim_topology(1, 0) == 0
    assert lib.ccm_sim_set(-1, b"cuda_ordinal", -1) == 0
    gpu = [d for d in D.find_gpus()[0] if d.is_gpu()][0]
    with pytest.raises(GpuError) as err:
        gpu.scrub_and_verify(prove=True)
    assert err.value.status == N.ERR_NO_CUDA and "coverage proof" in str(err.value)
    reports, _ = D.scrub_and_verify_many([gpu], prove=True)
    assert reports[0].status == N.ERR_NO_CUDA and reports[0].cover is None


# ---------------------------------------------------------------------------------- CLI and worker
def test_cli_prints_the_keys_the_worker_prints():
    src = (ROOT / "k8s_cc_manager_b200" / "csrc" / "ccm_scrub_cli.cpp").read_text()
    body = src[src.index("static void print_cover"):src.index('// The "mismatch_triage" object')]
    printed = set(re.findall(r'\\"(\w+)\\":', body))
    assert printed == ({"cover"} | set(CoverReport.__dataclass_fields__) | set(CoverPass.__dataclass_fields__)
                       | set(CoverPage.__dataclass_fields__))
    assert "ccm_last_cover_pages(ordinal" in body and "keep = 64" in body and D.COVER_PAGES == 64
    assert 'else if (a == "--prove") prove = true;' in src
    assert "ccm_scrub_prove(ordinals[i], 1)" in src and "ccm_scrub_prove(o, 0)" in src


def test_cli_never_scrubs_unproven_a_gpu_it_cannot_arm():
    cli = ROOT / "k8s_cc_manager_b200" / "ccm-scrub"
    if not cli.exists():
        pytest.skip("ccm-scrub is not built")
    proc = subprocess.run([str(cli), "--backend", "sim", "--prove", "--all"], capture_output=True, text=True, timeout=60)
    assert proc.returncode == 3 and "cannot arm the coverage proof" in proc.stderr and proc.stdout == ""


class _Dev:
    def __init__(self, bdf): self.bdf = bdf
    def is_gpu(self): return True


def zero_report(bdf, status=0):
    return ScrubReport(bdf, 0, 190 << 30, 191 << 30, 0, 1, 25, 25, 1, 52, 1, status)


def test_worker_takes_prove(monkeypatch, capsys):
    from k8s_cc_manager_b200 import scrub_worker
    seen = []

    def fake_many(devs, n, check="zero", residue=False, triage=False, triage_hold_ms=D.TRIAGE_HOLD_MS,
                  mismatch_triage=False, prove=False):
        seen.append(dict(check=check, residue=residue, triage=triage, mismatch_triage=mismatch_triage, prove=prove))
        rep = zero_report(devs[0].bdf, 0 if covered else N.ERR_UNCOVERED)
        rep.cover = sample_cover(int(covered)) if prove else None
        return [rep], 1.0
    monkeypatch.setattr(D, "find_gpus", lambda: ([_Dev("0000:01:00.0")], 1))
    monkeypatch.setattr(D, "scrub_and_verify_many", fake_many)
    covered = True
    assert scrub_worker.main(["--bdf", "0000:01:00.0", "--prove"]) == 0
    out = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    assert CoverReport.from_json(out["reports"][0]["cover"]) == sample_cover(1)
    covered = False
    assert scrub_worker.main(["--bdf", "0000:01:00.0", "--prove", "--residue", "--triage"]) == 3
    out = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    assert out["reports"][0]["status"] == N.ERR_UNCOVERED and out["reports"][0]["cover"]["covered"] == 0
    assert scrub_worker.main(["--bdf", "0000:01:00.0"]) == 3
    assert "cover" not in json.loads(capsys.readouterr().out.strip().splitlines()[-1])["reports"][0]
    assert [s["prove"] for s in seen] == [True, True, False] and seen[1]["residue"] and seen[1]["triage"]


# ---------------------------------------------------------------------------------- manager
import logging  # noqa: E402

import scenarios as SC  # noqa: E402
import test_dirt_locate as TD  # noqa: E402
import test_dirt_triage as TT  # noqa: E402
from helpers import build_native_world  # noqa: E402


class ProofGpu(TM.FakeGpu):
    """A clean device that takes `prove` (and every other gate argument) and records what it was called with;
    can_prove False: an older device library; uncovered: its proof finds a short pass."""

    def __init__(self, bdf, can_prove=True, uncovered=False):
        super().__init__(bdf)
        self.calls, self.uncovered = [], uncovered
        if can_prove:
            self.scrub_and_verify = self._scrub_prove

    def scrub_and_verify(self, nbytes=0, check="zero"):
        self.calls.append(("old", nbytes, {"check": check}))
        return zero_report(self.bdf) if check == "zero" else TM.report(self.bdf)

    def _scrub_prove(self, nbytes=0, check="zero", residue=False, triage=False, triage_hold_ms=100,
                     mismatch_triage=False, prove=False):
        kw = dict(check=check, residue=residue, triage=triage, mismatch_triage=mismatch_triage, prove=prove)
        self.calls.append(("new", nbytes, kw))
        if prove and self.uncovered:
            err = GpuError(f"scrub_and_verify on {self.bdf}: a scrub gate pass did not walk every mapped byte",
                           N.ERR_UNCOVERED)
            err.cover = sample_cover(0)
            raise err
        rep = zero_report(self.bdf) if check == "zero" else TM.report(self.bdf)
        rep.cover = sample_cover(1) if prove else None
        return rep


def cover_lines(caplog):
    return [(r.levelno, r.getMessage()) for r in caplog.records if r.getMessage().startswith("HBM coverage proof on ")]


def state(c):
    return c.labels(SC.NODE).get("nvidia.com/cc.mode.state")


@pytest.mark.parametrize("value,want", [(None, "off"), ("off", "off"), ("require", "require"), ("REQUIRE", "require")])
def test_setting_is_parsed(monkeypatch, value, want):
    if value is not None:
        monkeypatch.setenv("CC_SCRUB_PROOF", value)
    mgr, _ = TD.manager_for([ProofGpu(SC.GPU_BDFS[0])], monkeypatch)
    assert mgr.scrub_proof == want and mgr.prove == (want == "require")


def test_other_values_are_refused_at_start_up(monkeypatch):
    from k8s_cc_manager_b200 import manager
    for bad in ("on", "1", "report", "true"):
        monkeypatch.setenv("CC_SCRUB_PROOF", bad)
        with pytest.raises(ValueError, match="CC_SCRUB_PROOF must be 'off' or 'require'"):
            TD.manager_for([ProofGpu(SC.GPU_BDFS[0])], monkeypatch)
    monkeypatch.delenv("CC_SCRUB_PROOF")
    with pytest.raises(ValueError, match="CC_SCRUB_PROOF must be"):
        TD.manager_for([ProofGpu(SC.GPU_BDFS[0])], monkeypatch, scrub_proof="report")
    assert manager.build_arg_parser().parse_args(["--scrub-proof", "require"]).scrub_proof == "require"
    assert manager.build_arg_parser().parse_args([]).scrub_proof is None
    with pytest.raises(SystemExit):
        manager.build_arg_parser().parse_args(["--scrub-proof", "on"])


KNOB_SETS = [dict(), dict(scrub_check="tagged"), dict(scrub_residue="report"), dict(scrub_triage="report"),
             dict(scrub_check="tagged", scrub_mismatch_triage="report"),
             dict(scrub_check="tagged", scrub_residue="report", scrub_triage="report", scrub_mismatch_triage="report")]


@pytest.mark.parametrize("knobs", KNOB_SETS)
def test_per_gpu_gate_passes_prove_with_every_knob_and_logs(monkeypatch, caplog, knobs):
    devs = [ProofGpu(SC.GPU_BDFS[0]), ProofGpu(SC.GPU_BDFS[1])]
    mgr, c = TD.manager_for(devs, monkeypatch, scrub_proof="require", **knobs)
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is True
    check = knobs.get("scrub_check", "zero")
    for d in devs:
        assert len(d.calls) == 1 and d.calls[0][0] == "new" and d.calls[0][2]["prove"] is True
        kw = d.calls[0][2]
        assert kw["check"] == check and kw["residue"] == ("scrub_residue" in knobs)
        assert kw["triage"] == ("scrub_triage" in knobs) and kw["mismatch_triage"] == ("scrub_mismatch_triage" in knobs)
    assert mgr.last_transition["scrub_cover"] == {d.bdf: sample_cover(1) for d in devs}
    assert sorted(cover_lines(caplog)) == sorted(
        (logging.INFO, f"HBM coverage proof on {d.bdf}: {sample_cover(1).summary()}") for d in devs)


@pytest.mark.parametrize("knobs", KNOB_SETS)
def test_off_takes_the_calls_it_always_took(monkeypatch, caplog, knobs):
    devs = [ProofGpu(SC.GPU_BDFS[0])]
    mgr, _ = TD.manager_for(devs, monkeypatch, **knobs)
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is True
    assert devs[0].calls[0][2]["prove"] is False
    assert "scrub_cover" not in mgr.last_transition and cover_lines(caplog) == []


@pytest.mark.parametrize("knobs", [dict(), dict(scrub_check="tagged"), dict(scrub_residue="report")])
def test_a_device_without_prove_fails_the_gate(monkeypatch, caplog, knobs):
    devs = [ProofGpu(SC.GPU_BDFS[0]), ProofGpu(SC.GPU_BDFS[1], can_prove=False)]
    mgr, c = TD.manager_for(devs, monkeypatch, scrub_proof="require", **knobs)
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is False
    assert state(c) == "failed"
    assert devs[1].calls == []   # never scrubbed unproven in its place
    assert any(f"device {devs[1].bdf} cannot prove its HBM coverage (CC_SCRUB_PROOF=require)" in r.getMessage()
               for r in caplog.records)


def test_an_uncovered_gpu_fails_the_transition_and_logs_its_short_pass(monkeypatch, caplog):
    devs = [ProofGpu(SC.GPU_BDFS[0]), ProofGpu(SC.GPU_BDFS[1], uncovered=True)]
    mgr, c = TD.manager_for(devs, monkeypatch, scrub_proof="require")
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is False
    assert state(c) == "failed"
    bad = devs[1].bdf
    assert mgr.last_transition["scrub_cover"][bad] == sample_cover(0)
    lines = cover_lines(caplog)
    assert (logging.ERROR, f"HBM coverage proof on {bad}: {sample_cover(0).summary()}") in lines
    assert "the readback pass counted" in sample_cover(0).summary()


def _native_world(monkeypatch, n=2):
    build_native_world(SC.scenario("w", gpus_=SC.gpus(n), modes=[]))
    for k, v in dict(CCM_BACKEND="sim", CCM_SIM_GPUS=str(n), CCM_SIM_BIND_CUDA="0").items():
        monkeypatch.setenv(k, v)


@pytest.mark.parametrize("knobs", KNOB_SETS)
@pytest.mark.parametrize("covered", [True, False])
def test_native_fan_out_passes_it(monkeypatch, caplog, knobs, covered):
    from k8s_cc_manager_b200 import manager
    _native_world(monkeypatch)
    seen = {}

    def fake_many(devices, nbytes=0, check="zero", residue=False, triage=False, triage_hold_ms=D.TRIAGE_HOLD_MS,
                  mismatch_triage=False, prove=False):
        seen.update(check=check, residue=residue, triage=triage, mismatch_triage=mismatch_triage, prove=prove)
        reps = []
        for d in devices:
            r = zero_report(d.bdf, 0 if covered else N.ERR_UNCOVERED) if check == "zero" else TM.report(d.bdf)
            if check != "zero" and not covered:
                r.status = N.ERR_UNCOVERED
            r.cover = sample_cover(int(covered))
            reps.append(r)
        return reps, 1.0
    monkeypatch.setattr(manager._devices, "scrub_and_verify_many", fake_many)
    mgr, c = TD.manager_for(None, monkeypatch, scrub_proof="require", **knobs)
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is covered
    assert seen["prove"] is True and seen["check"] == knobs.get("scrub_check", "zero")
    assert seen["residue"] == ("scrub_residue" in knobs) and seen["mismatch_triage"] == ("scrub_mismatch_triage" in knobs)
    assert len(mgr.last_transition["scrub_cover"]) == 2
    assert {lvl for lvl, _ in cover_lines(caplog)} == {logging.INFO if covered else logging.ERROR}
    if not covered:
        assert state(c) == "failed"


def test_a_report_without_its_proof_fails_under_require(monkeypatch, caplog):
    from k8s_cc_manager_b200 import manager
    _native_world(monkeypatch)
    monkeypatch.setattr(manager._devices, "scrub_and_verify_many",
                        lambda devices, nbytes=0, prove=False, **kw: ([zero_report(d.bdf) for d in devices], 1.0))
    mgr, c = TD.manager_for(None, monkeypatch, scrub_proof="require")
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is False
    assert state(c) == "failed" and any("carries no coverage proof" in r.getMessage() for r in caplog.records)


@pytest.mark.parametrize("proof", ["off", "require"])
def test_worker_process_passes_it(monkeypatch, caplog, proof):
    _native_world(monkeypatch)
    monkeypatch.setenv("CC_SCRUB_ISOLATION", "process")
    monkeypatch.setenv("CC_SCRUB_PROOF", proof)
    monkeypatch.setenv("CC_SCRUB_CHECK", "tagged")
    monkeypatch.setenv("CC_SCRUB_TRIAGE", "report")
    cmds = []

    def fake_run(cmd, **kw):
        cmds.append(cmd)
        reps = []
        for b in [cmd[i + 1] for i, a in enumerate(cmd) if a == "--bdf"]:
            r = TM.report(b)
            r.cover = sample_cover(1) if "--prove" in cmd else None
            reps.append(r.as_json())
        return subprocess.CompletedProcess(cmd, 0, json.dumps({"wall_ms": 1.0, "reports": reps}) + "\n", "")
    monkeypatch.setattr(subprocess, "run", fake_run)
    mgr, c = TD.manager_for(None, monkeypatch)
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is True
    cmd = cmds[0]
    assert ("--prove" in cmd) == (proof == "require") and "--triage" in cmd and cmd[cmd.index("--check") + 1] == "tagged"
    if proof == "require":
        assert len(mgr.last_transition["scrub_cover"]) == 2 and len(cover_lines(caplog)) == 2
    else:
        assert "scrub_cover" not in mgr.last_transition
