"""The dirt triage on the CPU: the oracle's runs and classes against a brute-force walk, the C ABI without a CUDA device
(layouts, exports, refused arguments, the drill keys), TriageReport and its JSON, the CLI's and the worker's keys, and
the manager's knob, log line, last_transition key, every gate path that passes the setting on, and the warning for a
device that cannot triage."""
from __future__ import annotations

import ctypes as C
import inspect
import json
import logging
import re
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

import scenarios as SC
import test_dirt_locate as TD
from helpers import build_native_world
from k8s_cc_manager_b200 import _native as N
from k8s_cc_manager_b200 import devices as D
from k8s_cc_manager_b200.devices import GpuError, ScrubReport, TriagePage, TriageReport

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "oracle"))
import triage_oracle as TR  # noqa: E402

MiB = 1 << 20
PAGE = TR.PAGE_BYTES


# ---------------------------------------------------------------------------------- oracle
def random_layout(rng, npages: int, segment_mib=None):
    """(dirt page entries, spans): spans are the mapping (one span) or segments of `segment_mib` MiB, the last one
    shorter; a random set of pages is dirty."""
    total = npages * PAGE - (int(rng.integers(0, 2)) * MiB if segment_mib else 0)
    if segment_mib:
        spans = [(o, min(segment_mib * MiB, total - o)) for o in range(0, total, segment_mib * MiB)]
    else:
        spans = [(0, total)]
    dense = float(rng.choice([0.05, 0.5, 0.95]))
    pages = sorted(p for p in range(-(-total // PAGE)) if rng.random() < dense)
    return [(p, int(rng.integers(1, PAGE)), 0) for p in pages], spans


@pytest.mark.parametrize("seed", range(6))
def test_runs_match_a_brute_force_walk(seed):
    rng = np.random.default_rng(seed)
    for segment_mib in (None, 1, 2, 3, 5, 64):
        entries, spans = random_layout(rng, int(rng.integers(1, 40)), segment_mib)
        got = TR.runs(entries, spans)
        assert got == TR.brute_runs(entries, spans, MiB), (seed, segment_mib)
        assert sum(n for _, n, _ in got) == sum(min(PAGE, sum(s for _, s in spans) - p * PAGE) for p, _, _ in entries)
        # runs never cross a span, never touch inside one, and are ascending
        for (o1, n1, s1), (o2, _, s2) in zip(got, got[1:]):
            assert o1 + n1 <= o2 and (s1 != s2 or o1 + n1 < o2)


def test_runs_of_the_typical_layouts():
    spans = [(0, 80 * PAGE)]
    assert TR.runs([(p, 1, 0) for p in (0, 1, 2, 5, 7, 8)], spans) == [(0, 3 * PAGE, 0), (5 * PAGE, PAGE, 0),
                                                                         (7 * PAGE, 2 * PAGE, 0)]
    every_other = [(p, 1, 0) for p in range(0, 80, 2)]
    assert len(TR.runs(every_other, spans)) == 40                     # the most runs a contiguous mapping can have
    # 3 MiB segments: page 1 spans segments 0 and 1, so it is two pieces, and nothing merges across a segment
    segs = [(0, 3 * MiB), (3 * MiB, 3 * MiB), (6 * MiB, 3 * MiB)]
    assert TR.runs([(0, 1, 0), (1, 1, 0), (2, 1, 0)], segs) == [(0, 3 * MiB, 0), (3 * MiB, 3 * MiB, 1)]
    assert TR.runs([(0, 1, 0), (1, 1, 0)], segs) == [(0, 3 * MiB, 0), (3 * MiB, MiB, 1)]
    assert TR.runs([(1, 1, 0)], segs) == [(2 * MiB, MiB, 0), (3 * MiB, MiB, 1)]


@pytest.mark.parametrize("stay,ret", [(0, 0), (4, 0), (0, 4), (2, 5), (5, 2), (3, 3), (100, 0), (0, 100)])
def test_classes_follow_the_drills(stay, ret):
    entries = [(p, 10 + p, p // 4) for p in (0, 3, 4, 9, 10, 11, 40)]
    rows = TR.classify(entries, stay, ret)
    for i, (page, chunk, cls, dirt, t2, t3) in enumerate(rows):
        assert (page, dirt, chunk) == (entries[i][0], entries[i][1], entries[i][2])
        in_stay, in_ret = i < stay, i < ret
        want = "stays" if in_stay else "returns" if in_ret else "clears"
        assert cls == want and t2 == int(in_stay) and t3 == int(in_stay != in_ret)
    rep = TR.report(entries, [(0, 41 * PAGE)], stay, ret)
    assert rep["stay_pages"] + rep["return_pages"] + rep["clear_pages"] == len(entries) == rep["pages_examined"]
    assert rep["stay_bytes"] + rep["return_bytes"] + rep["clear_bytes"] == sum(b for _, b, _ in entries)
    assert rep["runs"] == 4 and rep["bytes_examined"] == len(entries) * PAGE
    assert TR.drill_xors(entries, stay, ret) == min(stay, 7) + min(ret, 7)
    if rep["t2_bytes"]:
        assert rep["t2_first_offset"] == 0 and rep["t2_last_offset"] == entries[min(stay, 7) - 1][0] * PAGE


# ---------------------------------------------------------------------------------- C ABI
def test_struct_layouts_match_the_header(tmp_path):
    src = tmp_path / "triage.c"
    fields = [("ccm_triage_report", f) for f, _ in N.TriageReport._fields_] + \
             [("ccm_triage_page", f) for f, _ in N.TriagePage._fields_]
    body = " ".join(f'printf("%zu\\n", offsetof({s}, {f}));' for s, f in fields)
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "ccm.h"\nint main(void){'
                   'printf("%zu\\n%zu\\n%u\\n%d\\n%d\\n%d\\n", sizeof(ccm_triage_report), sizeof(ccm_triage_page), '
                   'CCM_TRIAGE_MAX_HOLD_MS, CCM_TRIAGE_STAYS, CCM_TRIAGE_RETURNS, CCM_TRIAGE_CLEARS);'
                   + body + "return 0;}")
    exe = tmp_path / "triage"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-pedantic", "-I", str(ROOT / "include"), str(src), "-o",
                    str(exe)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    want = [C.sizeof(N.TriageReport), C.sizeof(N.TriagePage), N.TRIAGE_MAX_HOLD_MS, *sorted(N.TRIAGE_CLASSES)]
    want += [getattr(N.TriageReport if s == "ccm_triage_report" else N.TriagePage, f).offset for s, f in fields]
    assert got == want
    assert C.sizeof(N.TriagePage) == 32 and C.sizeof(N.TriageReport) == 152
    assert N.TRIAGE_CLASSES == {1: "stays", 2: "returns", 3: "clears"}


def test_entry_points_are_exported_and_refuse_what_they_must(native):
    lib = native.lib()
    nm = subprocess.run(["nm", "-D", "--defined-only", str(native.LIB_PATH)], capture_output=True, text=True,
                        check=True).stdout
    for fn in ("ccm_scrub_triage", "ccm_scrub_last_triage", "ccm_last_triage_pages"):
        assert fn in native.EXPORTED_SYMBOLS and re.search(rf" T {fn}$", nm, re.M), fn
    # a hold that is too long is refused whatever the device
    for ordinal in (0, -1, 1 << 12):
        assert lib.ccm_scrub_triage(ordinal, native.TRIAGE_MAX_HOLD_MS + 1) == native.ERR_INVALID
        assert "longer than 10000 ms" in native.last_error()
        assert lib.ccm_scrub_triage(ordinal, 0xFFFFFFFF) == native.ERR_INVALID
    # no such CUDA device (this suite runs without one)
    for ordinal in (-1, 1 << 12):
        for hold in (0, 1, native.TRIAGE_MAX_HOLD_MS):
            assert lib.ccm_scrub_triage(ordinal, hold) == native.ERR_NO_CUDA
        rep = native.TriageReport(triaged=7)
        assert lib.ccm_scrub_last_triage(ordinal, C.byref(rep)) == native.ERR_NO_CUDA and rep.triaged == 0
        n = C.c_uint64(7)
        assert lib.ccm_last_triage_pages(ordinal, None, 0, C.byref(n)) == native.ERR_NO_CUDA and n.value == 0
    assert lib.ccm_scrub_last_triage(0, None) == native.ERR_INVALID
    assert lib.ccm_last_triage_pages(0, None, 0, None) == native.ERR_INVALID
    n = C.c_uint64()
    assert lib.ccm_last_triage_pages(0, None, 3, C.byref(n)) == native.ERR_INVALID
    assert D.last_triage(-1) is None and D.last_triage_pages(-1) is None


def test_drill_keys_round_trip(native):
    lib = native.lib()
    assert lib.ccm_sim_topology(2, 0) == 0
    assert lib.ccm_sim_set(-1, b"cuda_ordinal", -1) == 0
    for key in (b"triage_stay", b"triage_return"):
        v = C.c_int64(-1)
        assert lib.ccm_sim_get(0, key, C.byref(v)) == 0 and v.value == 0
        assert lib.ccm_sim_set(0, key, 5) == 0 and lib.ccm_sim_get(0, key, C.byref(v)) == 0 and v.value == 5
        assert lib.ccm_sim_get(1, key, C.byref(v)) == 0 and v.value == 0
        assert lib.ccm_sim_set(0, key, -3) == 0 and lib.ccm_sim_get(0, key, C.byref(v)) == 0 and v.value == 0
    header = (ROOT / "include" / "ccm.h").read_text()
    assert '"triage_stay"' in header and '"triage_return"' in header


def test_a_triage_call_without_cuda_fails_as_the_plain_call_does(native):
    """No CUDA device: the call raises what it raises unarmed, and the hold is checked first."""
    lib = native.lib()
    assert lib.ccm_sim_topology(1, 0) == 0
    assert lib.ccm_sim_set(-1, b"cuda_ordinal", -1) == 0
    gpu = D.find_gpus()[0][0]
    with pytest.raises(GpuError) as plain:
        gpu.scrub_and_verify(MiB)
    with pytest.raises(GpuError) as armed:
        gpu.scrub_and_verify(MiB, triage=True)
    assert armed.value.status == plain.value.status == N.ERR_NO_CUDA and armed.value.triage is None
    for hold in (0, -1, N.TRIAGE_MAX_HOLD_MS + 1):
        with pytest.raises(ValueError):
            gpu.scrub_and_verify(MiB, triage=True, triage_hold_ms=hold)
        with pytest.raises(ValueError):
            D.scrub_and_verify_many([gpu], MiB, triage=True, triage_hold_ms=hold)
    reps, _ = D.scrub_and_verify_many([gpu], MiB, triage=True)
    assert reps[0].status == N.ERR_NO_CUDA and reps[0].triage is None


# ---------------------------------------------------------------------------------- TriageReport
def sample_triage(stay=1, ret=1, clear=2, truncated=0) -> TriageReport:
    pages = ([TriagePage(0, 0, "stays", 5, 1, 1)] * stay + [TriagePage(3, 1, "returns", 2, 0, 1)] * ret)
    return TriageReport(stay + ret + clear, (stay + ret + clear) * PAGE, stay, 5 * stay, ret, 2 * ret, clear, 7 * clear,
                        stay, stay + ret, 0, 0, 3 * PAGE if ret else 0, 3 * PAGE if ret else 0, 0x7F00_0000_0000,
                        100.2, 140.5, 100, stay + ret + clear, 1, pages, truncated)


def test_native_report_converts_and_keeps_the_pages_that_did_not_clear():
    t = N.TriageReport(pages_examined=70, runs=3, triaged=1, hold_ms=100, ms_hold=100.4, stay_pages=66, return_pages=2,
                       clear_pages=2, va_base=0x1000)
    pages = [TriagePage(p, 0, "stays" if p < 66 else "returns" if p < 68 else "clears", 1, 0, 0) for p in range(70)]
    rep = TriageReport.from_native(t, pages)
    assert len(rep.suspect_pages) == D.TRIAGE_PAGES == 64 and rep.suspect_truncated == 1
    assert all(p.cls == "stays" for p in rep.suspect_pages)
    rep = TriageReport.from_native(t, pages[60:])
    assert [p.page for p in rep.suspect_pages] == list(range(60, 68)) and rep.suspect_truncated == 0
    assert (rep.pages_examined, rep.runs, rep.hold_ms, rep.va_base, rep.triaged) == (70, 3, 100, 0x1000, 1)
    assert set(TriageReport.__dataclass_fields__) == \
        {f for f, _ in N.TriageReport._fields_ if f != "reserved"} | {"suspect_pages", "suspect_truncated"}
    assert TriageReport.from_native(N.TriageReport()).suspect_pages == []


def test_json_round_trip_and_unchanged_key_sets():
    rep = sample_triage()
    assert TriageReport.from_json(json.loads(json.dumps(rep.as_json()))) == rep
    sr = TD.report(nonzero=3)
    base = set(sr.as_json())
    assert sr.triage is None and "triage" not in ScrubReport.__dataclass_fields__
    sr.dirt = TD.sample_dirt()
    sr.triage = rep
    js = json.loads(json.dumps(sr.as_json()))
    assert set(js) == base | {"dirt", "triage"}
    back = ScrubReport.from_json(js)
    assert back.triage == rep and back.dirt == sr.dirt
    assert ScrubReport.from_json(TD.report().as_json()).triage is None
    assert GpuError("x").triage is None


def test_summary_line():
    rep = sample_triage(stay=0, ret=0, clear=4)
    assert rep.summary() == "4 pages in 4 runs: 0 stay, 0 return, 4 clear (hold 100 ms)"
    line = sample_triage(stay=2, ret=1, clear=1).summary()
    assert line.startswith("4 pages in 4 runs: 2 stay, 1 return, 1 clear (hold 100 ms); ")
    assert "+0x0 chunk 0 stays (5 B dirt, 1 B at once, 1 B after the hold)" in line
    assert "+0x600000 chunk 1 returns (2 B dirt, 0 B at once, 1 B after the hold)" in line


def test_device_api_takes_triage():
    for fn in (D.NvidiaDevice.scrub_and_verify, D.ScrubbingProxy.scrub_and_verify, D.scrub_and_verify_many):
        params = inspect.signature(fn).parameters
        assert params["triage"].default is False and params["triage_hold_ms"].default == D.TRIAGE_HOLD_MS == 100


# ---------------------------------------------------------------------------------- CLI and worker
def test_cli_prints_the_keys_the_worker_prints():
    src = (ROOT / "k8s_cc_manager_b200" / "csrc" / "ccm_scrub_cli.cpp").read_text()
    body = src[src.index("static void print_triage"):src.index("static void print_pages")]
    printed = set(re.findall(r'\\"(\w+)\\":', body))
    assert printed == {"triage"} | set(TriageReport.__dataclass_fields__) | set(TriagePage.__dataclass_fields__)
    assert "keep = 64" in body
    assert 'else if (a == "--triage") triage = true;' in src and '"--triage-hold-ms"' in src
    assert "ccm_scrub_triage(ordinals[i]" in src and "ccm_scrub_triage(o, 0)" in src
    assert "triage_hold_ms = 100;" in src


class _Dev:
    def __init__(self, bdf): self.bdf = bdf
    def is_gpu(self): return True


def test_worker_takes_triage(monkeypatch, capsys):
    from k8s_cc_manager_b200 import scrub_worker
    rep = TD.report("0000:01:00.0", nonzero=3)
    rep.dirt, rep.triage = TD.sample_dirt(), sample_triage()
    seen = []

    def fake_many(devs, n, check="zero", residue=False, triage=False, triage_hold_ms=D.TRIAGE_HOLD_MS):
        seen.append((check, residue, triage, triage_hold_ms))
        return [rep], 1.0
    monkeypatch.setattr(D, "find_gpus", lambda: ([_Dev(rep.bdf)], 1))
    monkeypatch.setattr(D, "scrub_and_verify_many", fake_many)
    assert scrub_worker.main(["--bdf", rep.bdf, "--triage"]) == 3
    out = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    assert TriageReport.from_json(out["reports"][0]["triage"]) == rep.triage
    assert scrub_worker.main(["--bdf", rep.bdf, "--triage", "--triage-hold-ms", "250", "--residue"]) == 3
    assert scrub_worker.main(["--bdf", rep.bdf]) == 3
    assert seen == [("zero", False, True, 100), ("zero", True, True, 250), ("zero", False, False, 100)]


# ---------------------------------------------------------------------------------- manager
class FakeGpu(TD.FakeGpu):
    """A device whose scrub finds dirt and takes `triage`; can_triage False: an older device library."""

    def __init__(self, bdf, dirt=None, triage=None, can_triage=True, cc="off"):
        super().__init__(bdf, cc=cc, dirt=dirt)
        self.triage, self.calls = triage, []
        if can_triage:
            self.scrub_and_verify = self._scrub_triage

    def scrub_and_verify(self, nbytes=0, check="zero"):
        self.calls.append((nbytes, check, None, None))
        return super().scrub_and_verify(nbytes, check)

    def _scrub_triage(self, nbytes=0, check="zero", residue=False, triage=False, triage_hold_ms=100):
        self.calls.append((nbytes, check, triage, triage_hold_ms))
        try:
            return TD.FakeGpu.scrub_and_verify(self, nbytes, check)
        except GpuError as err:
            err.triage = self.triage if triage else None
            raise


def triage_lines(caplog):
    return [r.getMessage() for r in caplog.records if r.getMessage().startswith("HBM dirt triage on ")]


@pytest.mark.parametrize("value,want", [(None, "off"), ("off", "off"), ("report", "report"), ("REPORT", "report")])
def test_setting_is_parsed(monkeypatch, value, want):
    if value is not None:
        monkeypatch.setenv("CC_SCRUB_TRIAGE", value)
    mgr, _ = TD.manager_for([FakeGpu(SC.GPU_BDFS[0])], monkeypatch)
    assert mgr.scrub_triage == want and mgr.triage == (want == "report")


def test_other_values_are_rejected(monkeypatch):
    from k8s_cc_manager_b200 import manager
    for bad in ("on", "1", "stay"):
        monkeypatch.setenv("CC_SCRUB_TRIAGE", bad)
        with pytest.raises(ValueError, match="CC_SCRUB_TRIAGE"):
            TD.manager_for([FakeGpu(SC.GPU_BDFS[0])], monkeypatch)
    monkeypatch.delenv("CC_SCRUB_TRIAGE")
    args = manager.build_arg_parser().parse_args(["--scrub-triage", "report"])
    assert args.scrub_triage == "report" and manager.build_arg_parser().parse_args([]).scrub_triage is None
    with pytest.raises(SystemExit):
        manager.build_arg_parser().parse_args(["--scrub-triage", "on"])
    assert manager.SCRUB_TRIAGE_HOLD_MS == 100


@pytest.mark.parametrize("check", ["zero", "tagged"])
def test_per_gpu_gate_passes_it_logs_and_keeps_the_report(monkeypatch, caplog, check):
    dirt, triage = TD.sample_dirt(), sample_triage(stay=0, ret=0, clear=4)
    devs = [FakeGpu(SC.GPU_BDFS[0]), FakeGpu(SC.GPU_BDFS[1], dirt=dirt, triage=triage)]
    mgr, c = TD.manager_for(devs, monkeypatch, scrub_triage="report", scrub_check=check)
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is False
    bdf = SC.GPU_BDFS[1]
    TD.assert_dirt_logged(mgr, c, caplog, bdf, dirt)
    assert all(d.calls == [(0, check, True, 100)] for d in devs)
    assert mgr.last_transition["scrub_triage"] == {bdf: triage}
    msgs = [r.getMessage() for r in caplog.records]
    lines = triage_lines(caplog)
    assert lines == [f"HBM dirt triage on {bdf}: 4 pages in 4 runs: 0 stay, 0 return, 4 clear (hold 100 ms)"]
    assert msgs.index(lines[0]) > msgs.index(next(m for m in msgs if m.startswith(f"HBM dirt on {bdf}: ")))


def test_off_takes_the_calls_it_always_took(monkeypatch, caplog):
    devs = [FakeGpu(SC.GPU_BDFS[0]), FakeGpu(SC.GPU_BDFS[1], dirt=TD.sample_dirt(), triage=sample_triage())]
    mgr, _ = TD.manager_for(devs, monkeypatch)
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is False
    assert all(d.calls == [(0, "zero", False, 100)] for d in devs)        # scrub_and_verify(0): no triage asked
    assert "scrub_triage" not in mgr.last_transition and triage_lines(caplog) == []


def test_a_device_without_triage_warns_and_runs_its_gate_unchanged(monkeypatch, caplog):
    dirt = TD.sample_dirt()
    devs = [FakeGpu(SC.GPU_BDFS[0], can_triage=False), FakeGpu(SC.GPU_BDFS[1], dirt=dirt, can_triage=False)]
    mgr, c = TD.manager_for(devs, monkeypatch, scrub_triage="report")
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is False
    warnings = [r.getMessage() for r in caplog.records if r.levelno == logging.WARNING and "cannot triage" in
                r.getMessage()]
    assert sorted(warnings) == sorted(f"Device {d.bdf} cannot triage HBM dirt (CC_SCRUB_TRIAGE=report): its gate runs "
                                      "without the triage" for d in devs)
    assert all(d.calls == [(0, "zero", None, None)] for d in devs)
    TD.assert_dirt_logged(mgr, c, caplog, SC.GPU_BDFS[1], dirt)
    assert "scrub_triage" not in mgr.last_transition and triage_lines(caplog) == []


def test_a_clean_gate_with_triage_passes(monkeypatch, caplog):
    devs = [FakeGpu(SC.GPU_BDFS[0], cc="off"), FakeGpu(SC.GPU_BDFS[1])]
    mgr, c = TD.manager_for(devs, monkeypatch, scrub_triage="report")
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is True
    assert "scrub_triage" not in mgr.last_transition and triage_lines(caplog) == []


def _native_world(monkeypatch, n=2):
    build_native_world(SC.scenario("w", gpus_=SC.gpus(n), modes=[]))
    for k, v in dict(CCM_BACKEND="sim", CCM_SIM_GPUS=str(n), CCM_SIM_BIND_CUDA="0").items():
        monkeypatch.setenv(k, v)


def dirty_report(bdf):
    r = TD.report(bdf, nonzero=3)
    r.dirt, r.triage = TD.sample_dirt(), sample_triage()
    return r


@pytest.mark.parametrize("residue", [False, True])
def test_native_fan_out_passes_it(monkeypatch, caplog, residue):
    from k8s_cc_manager_b200 import manager
    _native_world(monkeypatch)
    seen = {}

    def fake_many(devices, nbytes=0, check="zero", residue=False, triage=False, triage_hold_ms=D.TRIAGE_HOLD_MS):
        seen.update(check=check, residue=residue, triage=triage, hold=triage_hold_ms)
        return [dirty_report(d.bdf) for d in devices], 1.0
    monkeypatch.setattr(manager._devices, "scrub_and_verify_many", fake_many)
    mgr, c = TD.manager_for(None, monkeypatch, scrub_triage="report", scrub_residue="report" if residue else None)
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is False
    assert seen == {"check": "zero", "residue": residue, "triage": True, "hold": manager.SCRUB_TRIAGE_HOLD_MS}
    bdfs = [r.bdf for r in mgr.last_transition["scrub"]]
    assert set(mgr.last_transition["scrub_triage"]) == set(bdfs) and len(triage_lines(caplog)) == 2


def test_worker_process_passes_it(monkeypatch, caplog):
    _native_world(monkeypatch)
    monkeypatch.setenv("CC_SCRUB_ISOLATION", "process")
    monkeypatch.setenv("CC_SCRUB_TRIAGE", "report")
    cmds = []

    def fake_run(cmd, **kw):
        cmds.append(cmd)
        bdfs = [cmd[i + 1] for i, a in enumerate(cmd) if a == "--bdf"]
        reps = [dirty_report(b).as_json() for b in bdfs]
        return subprocess.CompletedProcess(cmd, 3, json.dumps({"wall_ms": 1.0, "reports": reps}) + "\n", "")
    monkeypatch.setattr(subprocess, "run", fake_run)
    mgr, c = TD.manager_for(None, monkeypatch)
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is False
    cmd = cmds[0]
    assert len(cmds) == 1 and "--triage" in cmd and cmd[cmd.index("--triage-hold-ms") + 1] == "100"
    assert all(r.triage == sample_triage() for r in mgr.last_transition["scrub"])
    assert len(mgr.last_transition["scrub_triage"]) == 2 and len(triage_lines(caplog)) == 2
