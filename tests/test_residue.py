"""The residue census on the CPU: the C structs against ctypes, the new entry points without a CUDA device, the JSON
of reports with and without a census, summary(), the scrub_residue drill's sim key and the offsets product_plan
predicts for it, CC_SCRUB_RESIDUE parsing and its pass-through on every gate path (including a device that cannot
take it), the manager's log line and last_transition["scrub_residue"], and --residue in both workers."""
from __future__ import annotations

import ctypes as C
import json
import logging
import subprocess
import sys
from pathlib import Path

import pytest

import product_plan as PP
import scenarios as SC
from helpers import build_native_world
from k8s_cc_manager_b200 import _native as N
from k8s_cc_manager_b200 import devices as D
from k8s_cc_manager_b200.devices import GpuError, ResidueReport, ResidueWindow, ScrubReport

ROOT = Path(__file__).resolve().parents[1]
GiB, MiB = 1 << 30, 1 << 20


# ---------------------------------------------------------------------------------- C ABI
def test_struct_layouts_match_the_header(tmp_path):
    src = tmp_path / "rr.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "ccm.h"\nint main(void){'
                   'printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu\\n",'
                   'sizeof(ccm_residue_record), offsetof(ccm_residue_record,chunk), offsetof(ccm_residue_record,mask),'
                   'offsetof(ccm_residue_record,reserved), sizeof(ccm_residue_report),'
                   'offsetof(ccm_residue_report,bytes_examined), offsetof(ccm_residue_report,va_base),'
                   'offsetof(ccm_residue_report,located), offsetof(ccm_residue_report,nrecords),'
                   'offsetof(ccm_residue_report,truncated), offsetof(ccm_residue_report,records),'
                   'sizeof(((ccm_residue_report*)0)->records) / sizeof(ccm_residue_record));return 0;}')
    exe = tmp_path / "rr"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", str(ROOT / "include"), str(src), "-o", str(exe)],
                   check=True)
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    R, P = N.ResidueRecord, N.ResidueReport
    assert got == [C.sizeof(R), R.chunk.offset, R.mask.offset, R.reserved.offset, C.sizeof(P), P.bytes_examined.offset,
                   P.va_base.offset, P.located.offset, P.nrecords.offset, P.truncated.offset, P.records.offset,
                   N.DIRT_RECORDS]
    assert C.sizeof(R) == 16 and C.sizeof(P) == 64 + 16 * N.DIRT_RECORDS


def test_new_entry_points_are_exported_and_need_a_cuda_device(native):
    lib = native.lib()
    assert {"ccm_scrub_verify_residue", "ccm_scrub_verify_many_residue", "ccm_region_census"} <= set(
        native.EXPORTED_SYMBOLS)
    assert lib.ccm_abi_version() == 2
    buf = (C.c_uint8 * 64)()
    for ordinal in (-1, 1 << 12):
        r = native.ResidueReport(located=7, nrecords=3)
        assert lib.ccm_region_census(ordinal, buf, 64, 0, 1, None, C.byref(r)) == native.ERR_NO_CUDA
        assert r.located == 0 and r.nrecords == 0
    assert lib.ccm_region_census(0, None, 0, 0, 1, None, None) == native.ERR_INVALID
    res = native.ScrubResult()
    assert lib.ccm_scrub_verify_residue(0, GiB, None, None, C.byref(res)) == native.ERR_INVALID
    devs = (C.c_int * 1)(0)
    assert lib.ccm_scrub_verify_many_residue(1, devs, GiB, None, None, C.byref(res), None) == native.ERR_INVALID


def test_census_call_without_cuda_reports_no_cuda(monkeypatch):
    build_native_world(SC.scenario("w", gpus_=SC.gpus(2), modes=[]))
    for k, v in dict(CCM_BACKEND="sim", CCM_SIM_GPUS="2", CCM_SIM_BIND_CUDA="0").items():
        monkeypatch.setenv(k, v)
    lib = N.lib()
    r, res = N.ResidueReport(located=5), N.ScrubResult()
    assert lib.ccm_scrub_verify_residue(0, GiB, None, C.byref(r), C.byref(res)) == N.ERR_NO_CUDA
    assert res.status == N.ERR_NO_CUDA and r.located == 0
    out, rr = (N.ScrubResult * 2)(), (N.ResidueReport * 2)()
    tags = (N.TagResult * 2)()
    devs = (C.c_int * 2)(0, 1)
    assert lib.ccm_scrub_verify_many_residue(2, devs, GiB, tags, rr, out, None) == N.ERR_NO_CUDA
    assert [o.status for o in out] == [N.ERR_NO_CUDA] * 2 and [x.located for x in rr] == [0, 0]
    with pytest.raises(GpuError) as ei:
        D.find_gpus()[0][0].scrub_and_verify(GiB, residue=True)
    assert ei.value.status == N.ERR_NO_CUDA


def test_scrub_residue_is_a_sim_key(monkeypatch):
    build_native_world(SC.scenario("w", gpus_=SC.gpus(1), modes=[]))
    for k, v in dict(CCM_BACKEND="sim", CCM_SIM_GPUS="1", CCM_SIM_BIND_CUDA="0").items():
        monkeypatch.setenv(k, v)
    lib = N.lib()
    v = C.c_int64()
    assert lib.ccm_sim_set(0, b"scrub_residue", 1000) == 0
    assert lib.ccm_sim_get(0, b"scrub_residue", C.byref(v)) == 0 and v.value == 1000
    assert lib.ccm_sim_set(0, b"scrub_residue", 0) == 0


def test_scrub_residue_offsets_follow_the_mappings():
    """The drill's bytes are inject_offsets over the mappings (Run.chunks), not over the enqueued ranges."""
    env = PP.mode_env(1, 1)
    p = PP.plan(4 * GiB, 70 * GiB, PP.H100_GRAN, env)
    run = PP.simulate(p, None)
    assert run.chunks == [(0, GiB), (GiB, 2 * GiB), (3 * GiB, GiB)] and run.ranges(p) == [(0, 4 * GiB)]
    offs = PP.inject_offsets(run.chunks, 1000)
    assert offs == [0, 17, GiB // 2 + 3, GiB - 1, GiB, GiB + 17, 2 * GiB + 3, 3 * GiB - 1,
                    3 * GiB, 3 * GiB + 17, 3 * GiB + GiB // 2 + 3, 4 * GiB - 1]
    assert PP.inject_offsets(run.chunks, 3) == [0, 17, GiB // 2 + 3]
    segs = PP.arena_segments(300 * MiB, 70 * GiB, {"CCM_PIPELINE": "0", "CCM_ARENA_MAX_SEGMENT_MB": "96"})
    assert len(PP.inject_offsets(segs, 1000)) == 16


def test_header_documents_the_drill_and_the_variant():
    h = (ROOT / "include" / "ccm.h").read_text()
    assert '"scrub_residue"' in h and "reports scrub_variant = CCM_SCRUB_ST128" in h


# ---------------------------------------------------------------------------------- JSON, summary
def sample_residue(n=3, truncated=0) -> ResidueReport:
    recs = [ResidueWindow(16 * i * 0x1000, i % 2, 1 << (i % 16)) for i in range(n)]
    return ResidueReport(residue_bytes=n, residue_windows=n + truncated * 100, first_offset=0,
                         last_offset=16 * (n - 1) * 0x1000 + (n - 1) % 16, bytes_examined=4 * GiB,
                         va_base=0x7F00_0000_0000, located=1, truncated=truncated, records=recs)


def report(bdf=SC.GPU_BDFS[0], **kw):
    return ScrubReport(bdf, 0, 190 << 30, 191 << 30, 0, 1, 25, 25, 1, 52, 1, 0, **kw)


def test_json_round_trip_and_unchanged_key_sets():
    plain = report()
    assert plain.residue is None and "residue" not in ScrubReport.__dataclass_fields__
    assert "residue" not in plain.as_json()
    keys = set(plain.as_json())
    rep = report()
    rep.residue = sample_residue()
    js = json.loads(json.dumps(rep.as_json()))
    assert set(js) - {"residue"} == keys and set(js["residue"]["records"][0]) == {"offset", "chunk", "mask"}
    back = ScrubReport.from_json(js)
    assert back == rep and back.residue == rep.residue and back.dirt is None and back.mismatch is None
    assert ResidueReport.from_json(sample_residue(70, 1).as_json()) == sample_residue(70, 1)
    assert GpuError("x").residue is None


def test_native_report_converts_with_signed_offsets():
    r = N.ResidueReport(residue_bytes=2, residue_windows=2, first_offset=0, last_offset=0x40, bytes_examined=100,
                        va_base=0x1003, located=1, nrecords=2, truncated=0)
    r.records[0].offset, r.records[0].mask = (1 << 64) - 3, 0x0008
    r.records[1].offset, r.records[1].mask, r.records[1].chunk = 0x40, 0x0001, 2
    rep = ResidueReport.from_native(r)
    assert [(w.offset, w.chunk, w.mask) for w in rep.records] == [(-3, 0, 8), (0x40, 2, 1)]
    assert rep.bytes_examined == 100 and rep.va_base == 0x1003


def test_summary_says_none_or_where():
    none = ResidueReport(0, 0, 0, 0, 4 * GiB, 0x7F00_0000_0000, 1, 0)
    assert none.summary().startswith("none: all 4294967296 bytes examined were zero")
    s = sample_residue().summary()
    assert s.startswith("3 of 4294967296 bytes were non-zero at first touch, in 3 16-byte windows") and "chunks [0, 1]" in s
    assert "+0x10000 chunk 1 mask 0002" in s
    assert "(records truncated)" in sample_residue(70, 1).summary()
    assert ResidueReport(0, 0, 0, 0, 0, 0, 0, 0).summary() == "no census ran"


# ---------------------------------------------------------------------------------- manager
class FakeGpu:
    """Duck-typed device; `census` False: a scrub_and_verify that takes no `residue` (an older device library)."""

    def __init__(self, bdf, cc="off", census=True, fail=False):
        self.bdf, self.name = bdf, "fake"
        self.is_cc_query_supported = self.is_ppcie_query_supported = True
        self.cc, self.staged, self.pp = cc, cc, "off"
        self.calls = []
        self.fail = fail
        if census:
            self.scrub_and_verify = self._scrub_census

    def is_gpu(self): return True
    def is_nvswitch(self): return False
    def query_cc_mode(self): return self.cc
    def set_cc_mode(self, m): self.staged = m
    def query_ppcie_mode(self): return self.pp
    def set_ppcie_mode(self, m): pass
    def reset_with_os(self): self.cc = self.staged
    def wait_for_boot(self): pass

    def scrub_and_verify(self, nbytes=0, check="zero"):
        self.calls.append((nbytes, check, None))
        return report(self.bdf, check=check)

    def _scrub_census(self, nbytes=0, check="zero", residue=False):
        self.calls.append((nbytes, check, residue))
        rep = report(self.bdf, check=check)
        if residue:
            rep.residue = sample_residue() if self.bdf == SC.GPU_BDFS[1] else ResidueReport(0, 0, 0, 0, 1 << 30, 0, 1, 0)
        if self.fail:
            err = GpuError(f"scrub_and_verify on {self.bdf}: verify found non-zero bytes", N.ERR_DIRTY)
            err.residue = rep.residue
            raise err
        return rep


def manager_for(devs, monkeypatch, labels=None, **kw):
    import kubernetes
    from k8s_cc_manager_b200 import manager
    c = kubernetes.reset_cluster()
    c.add_node(SC.NODE, labels or {})
    monkeypatch.setenv("EVICT_OPERATOR_COMPONENTS", "false")
    source = (lambda: (devs, len(devs))) if devs is not None else None
    return manager.CCManager(SC.NODE, "on", True, device_source=source, **kw), c


def residue_lines(caplog):
    return [r.getMessage() for r in caplog.records if r.getMessage().startswith("HBM residue on ")]


@pytest.mark.parametrize("value,want", [(None, "off"), ("off", "off"), ("report", "report"), ("REPORT", "report")])
def test_setting_is_parsed(monkeypatch, value, want):
    if value is None:
        monkeypatch.delenv("CC_SCRUB_RESIDUE", raising=False)
    else:
        monkeypatch.setenv("CC_SCRUB_RESIDUE", value)
    mgr, _ = manager_for([FakeGpu(SC.GPU_BDFS[0])], monkeypatch)
    assert mgr.scrub_residue == want


def test_other_values_are_rejected(monkeypatch):
    monkeypatch.setenv("CC_SCRUB_RESIDUE", "fail")
    with pytest.raises(ValueError, match="CC_SCRUB_RESIDUE must be 'off' or 'report'"):
        manager_for([FakeGpu(SC.GPU_BDFS[0])], monkeypatch)
    from k8s_cc_manager_b200 import manager
    assert manager.build_arg_parser().parse_args(["--scrub-residue", "report"]).scrub_residue == "report"
    with pytest.raises(SystemExit):
        manager.build_arg_parser().parse_args(["--scrub-residue", "on"])


@pytest.mark.parametrize("check", ["zero", "tagged"])
def test_per_gpu_fan_out_passes_it_logs_and_keeps_the_reports(monkeypatch, caplog, check):
    devs = [FakeGpu(SC.GPU_BDFS[0]), FakeGpu(SC.GPU_BDFS[1])]
    mgr, c = manager_for(devs, monkeypatch, scrub_residue="report", scrub_check=check)
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is True
    assert [d.calls for d in devs] == [[(0, check, True)]] * 2
    kept = mgr.last_transition["scrub_residue"]
    assert kept[SC.GPU_BDFS[1]] == sample_residue() and kept[SC.GPU_BDFS[0]].residue_bytes == 0
    lines = residue_lines(caplog)
    assert len(lines) == 2
    assert f"HBM residue on {SC.GPU_BDFS[0]}: none: " in lines[0] or f"HBM residue on {SC.GPU_BDFS[0]}: none: " in lines[1]
    assert any(f"HBM residue on {SC.GPU_BDFS[1]}: 3 of 4294967296 bytes" in ln for ln in lines)


def test_off_takes_the_calls_it_always_took(monkeypatch, caplog):
    devs = [FakeGpu(SC.GPU_BDFS[0]), FakeGpu(SC.GPU_BDFS[1], census=False)]
    monkeypatch.delenv("CC_SCRUB_RESIDUE", raising=False)
    mgr, c = manager_for(devs, monkeypatch)
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is True
    assert devs[0].calls == [(0, "zero", False)] and devs[1].calls == [(0, "zero", None)]
    assert "scrub_residue" not in mgr.last_transition and residue_lines(caplog) == []


@pytest.mark.parametrize("check", ["zero", "tagged"])
def test_a_device_without_the_census_warns_and_proceeds(monkeypatch, caplog, check):
    devs = [FakeGpu(SC.GPU_BDFS[0], census=False), FakeGpu(SC.GPU_BDFS[1])]
    mgr, c = manager_for(devs, monkeypatch, scrub_residue="report", scrub_check=check)
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is True
    assert devs[0].calls == [(0, check, None)] and devs[1].calls == [(0, check, True)]
    assert any(f"Device {SC.GPU_BDFS[0]} cannot report HBM residue" in r.getMessage() and r.levelno == logging.WARNING
               for r in caplog.records)
    assert set(mgr.last_transition["scrub_residue"]) == {SC.GPU_BDFS[1]}
    assert c.labels(SC.NODE).get("nvidia.com/cc.mode.state") == "on"


def test_a_failed_gate_keeps_the_residue_and_still_fails(monkeypatch, caplog):
    devs = [FakeGpu(SC.GPU_BDFS[1], fail=True)]
    mgr, c = manager_for(devs, monkeypatch, scrub_residue="report")
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is False
    assert c.labels(SC.NODE).get("nvidia.com/cc.mode.state") == "failed"
    assert mgr.last_transition["scrub_residue"] == {SC.GPU_BDFS[1]: sample_residue()}
    assert len(residue_lines(caplog)) == 1


def test_regate_passes_it(monkeypatch, caplog):
    dev = FakeGpu(SC.GPU_BDFS[1], cc="on")
    mgr, c = manager_for([dev], monkeypatch, labels={"nvidia.com/cc.mode.state": "failed"}, scrub_residue="report")
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is True
    assert mgr.last_transition["regate"] is True and dev.calls == [(0, "zero", True)]
    assert mgr.last_transition["scrub_residue"] == {SC.GPU_BDFS[1]: sample_residue()}
    assert len(residue_lines(caplog)) == 1


def _native_world(monkeypatch, n=2):
    build_native_world(SC.scenario("w", gpus_=SC.gpus(n), modes=[]))
    for k, v in dict(CCM_BACKEND="sim", CCM_SIM_GPUS=str(n), CCM_SIM_BIND_CUDA="0").items():
        monkeypatch.setenv(k, v)


@pytest.mark.parametrize("check", ["zero", "tagged"])
def test_native_fan_out_passes_it(monkeypatch, caplog, check):
    from k8s_cc_manager_b200 import manager
    _native_world(monkeypatch)
    seen = {}

    def fake_many(devices, nbytes=0, check="zero", residue=False):
        seen.update(check=check, residue=residue)
        reps = [report(d.bdf, check=check) for d in devices]
        for r in reps:
            r.residue = sample_residue()
        return reps, 1.0
    monkeypatch.setattr(manager._devices, "scrub_and_verify_many", fake_many)
    mgr, c = manager_for(None, monkeypatch, scrub_residue="report", scrub_check=check)
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is True
    assert seen == {"check": check, "residue": True}
    bdfs = [r.bdf for r in mgr.last_transition["scrub"]]
    assert set(mgr.last_transition["scrub_residue"]) == set(bdfs) and len(residue_lines(caplog)) == 2


def test_worker_process_passes_it(monkeypatch, caplog):
    _native_world(monkeypatch)
    monkeypatch.setenv("CC_SCRUB_ISOLATION", "process")
    monkeypatch.setenv("CC_SCRUB_RESIDUE", "report")
    cmds = []

    def fake_run(cmd, **kw):
        cmds.append(cmd)
        bdfs = [cmd[i + 1] for i, a in enumerate(cmd) if a == "--bdf"]
        reps = []
        for b in bdfs:
            r = report(b)
            r.residue = sample_residue()
            reps.append(r.as_json())
        return subprocess.CompletedProcess(cmd, 0, json.dumps({"wall_ms": 1.0, "reports": reps}) + "\n", "")
    monkeypatch.setattr(subprocess, "run", fake_run)
    mgr, c = manager_for(None, monkeypatch)
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is True
    assert len(cmds) == 1 and "--residue" in cmds[0]
    assert all(r.residue == sample_residue() for r in mgr.last_transition["scrub"])
    assert len(mgr.last_transition["scrub_residue"]) == 2 and len(residue_lines(caplog)) == 2


# ---------------------------------------------------------------------------------- CLI and worker
def test_worker_takes_residue(monkeypatch, capsys):
    from k8s_cc_manager_b200 import scrub_worker
    rep = report("0000:01:00.0")
    rep.residue = sample_residue()
    seen = {}

    class Dev:
        def __init__(self, bdf): self.bdf = bdf
        def is_gpu(self): return True

    def fake_many(devs, n, check="zero", residue=False):
        seen["residue"] = residue
        return [rep], 1.0
    monkeypatch.setattr(D, "find_gpus", lambda: ([Dev(rep.bdf)], 1))
    monkeypatch.setattr(D, "scrub_and_verify_many", fake_many)
    assert scrub_worker.main(["--bdf", rep.bdf, "--residue"]) == 0
    out = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    assert seen == {"residue": True} and ResidueReport.from_json(out["reports"][0]["residue"]) == rep.residue
    assert scrub_worker.main(["--bdf", rep.bdf]) == 0
    assert seen == {"residue": False}


def test_cli_takes_residue_and_prints_no_bytes():
    src = (ROOT / "k8s_cc_manager_b200" / "csrc" / "ccm_scrub_cli.cpp").read_text()
    assert 'else if (a == "--residue") residue = true;' in src and "ccm_scrub_verify_many_residue(" in src
    printed = src[src.index("static void print_residue"):src.index("static int usage")]
    keys = set(ResidueReport.__dataclass_fields__) | set(ResidueWindow.__dataclass_fields__)
    assert all(f'\\"{k}\\"' in printed for k in keys) and '\\"bytes\\"' not in printed
