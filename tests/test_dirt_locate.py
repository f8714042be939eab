"""The dirt report on the CPU: the numpy oracle against a byte-by-byte restatement and its own properties, the C
structs against ctypes, the JSON of reports with and without dirt, the manager's log line and
last_transition["scrub_dirt"] on every gate path, and the new entry points without a CUDA device."""
from __future__ import annotations

import ctypes as C
import json
import logging
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

import scenarios as SC
from helpers import build_native_world
from k8s_cc_manager_b200 import _native as N
from k8s_cc_manager_b200 import devices as D
from k8s_cc_manager_b200.devices import DirtReport, DirtWindow, GpuError, ScrubReport

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "oracle"))
import dirt_oracle as DO  # noqa: E402


# ---------------------------------------------------------------------------------- oracle
def brute_force(buf: np.ndarray, base: int) -> dict:
    """Byte by byte: every 16-aligned address window, its mask and bytes."""
    windows = {}
    for i, b in enumerate(buf.tolist()):
        if b:
            w = (base + i) // 16 * 16
            mask, data = windows.get(w, (0, bytearray(16)))
            data[(base + i) % 16] = b
            windows[w] = (mask | 1 << ((base + i) % 16), data)
    nz = [i for i, b in enumerate(buf.tolist()) if b]
    return {"nonzero_bytes": len(nz), "dirty_windows": len(windows),
            "first_offset": nz[0] if nz else None, "last_offset": nz[-1] if nz else None,
            "truncated": len(windows) > DO.RECORDS,
            "windows": [(w - base, m, bytes(d).hex()) for w, (m, d) in sorted(windows.items())]}


@pytest.mark.parametrize("seed", range(6))
def test_oracle_matches_a_byte_by_byte_restatement(seed):
    rng = np.random.default_rng(seed)
    for n in (0, 1, 15, 16, 17, 100, 1000, 5000):
        for base in (0x7F00_0000_0000, 0x7F00_0000_0001, 0x7F00_0000_000F, 0x7F00_0000_0011):
            buf = np.where(rng.random(n) < (0.02, 0.3, 1.0)[seed % 3], rng.integers(1, 256, n), 0).astype(np.uint8)
            assert DO.report(buf, base) == brute_force(buf, base), (n, base)


def test_oracle_properties():
    rng = np.random.default_rng(3)
    n, base = 70_001, 0x7F12_3456_7803
    buf = np.where(rng.random(n) < 0.01, rng.integers(1, 256, n), 0).astype(np.uint8)
    rep = DO.report(buf, base)
    assert sum(bin(m).count("1") for _, m, _ in rep["windows"]) == rep["nonzero_bytes"] == np.count_nonzero(buf)
    assert rep["dirty_windows"] == len(rep["windows"]) > DO.RECORDS and rep["truncated"]
    offs = [o for o, _, _ in rep["windows"]]
    assert offs == sorted(set(offs)) and all((base + o) % 16 == 0 for o in offs)
    for o, m, data in rep["windows"]:
        got = bytes.fromhex(data)
        assert all(((m >> i) & 1) == (got[i] != 0) for i in range(16))
        assert all(got[i] == (buf[o + i] if 0 <= o + i < n else 0) for i in range(16))
    # a window never leaks bytes outside the buffer, even when its neighbours are non-zero
    full = np.full(40, 7, dtype=np.uint8)
    inner = DO.report(full[3:37], 0x1003)
    assert inner["windows"][0] == (-3, 0xFFF8, "00" * 3 + "07" * 13)
    assert inner["windows"][-1][1] == (1 << ((0x1003 + 33) % 16 + 1)) - 1
    assert inner["dirty_windows"] == DO.window_count(0x1003, 34) == 3
    assert DO.window_count(0, 0) == 0 and DO.window_count(16, 16) == 1 and DO.window_count(15, 2) == 2


# ---------------------------------------------------------------------------------- C ABI
def test_struct_layouts_match_the_header(tmp_path):
    src = tmp_path / "dirt.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "ccm.h"\nint main(void){'
                   'printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %d\\n", sizeof(ccm_dirt_record),'
                   'offsetof(ccm_dirt_record,chunk), offsetof(ccm_dirt_record,mask), offsetof(ccm_dirt_record,bytes),'
                   'sizeof(ccm_dirt_report), offsetof(ccm_dirt_report,va_base), offsetof(ccm_dirt_report,ms_locate),'
                   'offsetof(ccm_dirt_report,located), offsetof(ccm_dirt_report,truncated),'
                   'offsetof(ccm_dirt_report,records), CCM_DIRT_RECORDS);return 0;}')
    exe = tmp_path / "dirt"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", str(ROOT / "include"), str(src), "-o", str(exe)],
                   check=True)
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    R, P = N.DirtRecord, N.DirtReport
    assert got == [C.sizeof(R), R.chunk.offset, R.mask.offset, R.bytes.offset, C.sizeof(P), P.va_base.offset,
                   P.ms_locate.offset, P.located.offset, P.truncated.offset, P.records.offset, N.DIRT_RECORDS]
    assert C.sizeof(R) == 32 and N.DIRT_RECORDS == DO.RECORDS == 64


def test_new_entry_points_are_exported_and_need_a_cuda_device(native):
    lib = native.lib()
    assert {"ccm_scrub_last_dirt", "ccm_region_locate"} <= set(native.EXPORTED_SYMBOLS)
    assert lib.ccm_abi_version() == 2
    for ordinal in (-1, 1 << 12):                    # no CUDA device has these ordinals, GPU or not
        d = native.DirtReport(located=7, nrecords=3)
        assert lib.ccm_scrub_last_dirt(ordinal, C.byref(d)) == native.ERR_NO_CUDA
        assert d.located == 0 and d.nrecords == 0
        buf = (C.c_uint8 * 64)()
        assert lib.ccm_region_locate(ordinal, buf, 64, None, C.byref(d)) == native.ERR_NO_CUDA
    assert lib.ccm_scrub_last_dirt(0, None) == native.ERR_INVALID
    assert lib.ccm_region_locate(0, None, 0, None, None) == native.ERR_INVALID
    assert D.last_dirt(-1) is None


def test_native_report_converts_with_signed_offsets():
    d = N.DirtReport(nonzero_bytes=3, dirty_windows=2, first_offset=1, last_offset=40, va_base=0x1003, ms_locate=0.5,
                     located=1, nrecords=2, truncated=0)
    d.records[0].offset, d.records[0].mask, d.records[0].bytes[13] = (1 << 64) - 3, 1 << 13, 0x11
    d.records[1].offset, d.records[1].chunk, d.records[1].mask = 29, 4, 0x0003
    d.records[1].bytes[0], d.records[1].bytes[1] = 0xAB, 0xCD
    rep = DirtReport.from_native(d)
    assert [(r.offset, r.chunk, r.mask) for r in rep.records] == [(-3, 0, 1 << 13), (29, 4, 3)]
    assert rep.records[0].bytes == "00" * 13 + "11" + "00" * 2 and rep.records[1].bytes.startswith("abcd")
    assert rep.chunks == [0, 4] and "chunks [0, 4]" in rep.summary()


# ---------------------------------------------------------------------------------- JSON
def sample_dirt(truncated=0) -> DirtReport:
    return DirtReport(nonzero_bytes=3, dirty_windows=2 + 100 * truncated, first_offset=0x10, last_offset=0x2011,
                      va_base=0x7F00_0000_0000, ms_locate=1.5, located=1, truncated=truncated,
                      records=[DirtWindow(0x10, 0, 1, "5a" + "00" * 15), DirtWindow(0x2010, 3, 3, "5a5a" + "00" * 14)])


def report(bdf=SC.GPU_BDFS[0], nonzero=0, **kw):
    return ScrubReport(bdf, 0, 190 << 30, 191 << 30, nonzero, 1, 25, 25, 1, 52, 1, N.ERR_DIRTY if nonzero else 0,
                       **kw)


def test_json_round_trip_and_clean_key_sets():
    clean = report()
    assert clean.dirt is None and "dirt" not in ScrubReport.__dataclass_fields__
    assert set(clean.as_json()) == set(ScrubReport.__dataclass_fields__) - set(D.TAG_FIELDS)
    tagged = report(check="tagged")
    assert set(tagged.as_json()) == set(ScrubReport.__dataclass_fields__)
    for rep in (report(nonzero=3), report(nonzero=3, check="tagged")):
        rep.dirt = sample_dirt()
        js = json.loads(json.dumps(rep.as_json()))
        assert set(js) - {"dirt"} == set(rep.as_json()) - {"dirt"} and js["dirt"]["records"][1]["chunk"] == 3
        back = ScrubReport.from_json(js)
        assert back == rep and back.dirt == rep.dirt
    assert ScrubReport.from_json(clean.as_json()) == clean and ScrubReport.from_json(clean.as_json()).dirt is None
    assert DirtReport.from_json(sample_dirt(1).as_json()) == sample_dirt(1)
    assert "(records truncated)" in sample_dirt(1).summary()


def test_gpu_error_carries_no_dirt_by_default():
    assert GpuError("x").dirt is None


# ---------------------------------------------------------------------------------- manager
class FakeGpu:
    """Duck-typed device whose scrub finds dirt: GpuError with .dirt, as NvidiaDevice.scrub_and_verify raises."""

    def __init__(self, bdf, cc="off", dirt=None):
        self.bdf, self.name = bdf, "fake"
        self.is_cc_query_supported = self.is_ppcie_query_supported = True
        self.cc, self.staged, self.pp = cc, cc, "off"
        self.dirt = dirt

    def is_gpu(self): return True
    def is_nvswitch(self): return False
    def query_cc_mode(self): return self.cc
    def set_cc_mode(self, m): self.staged = m
    def query_ppcie_mode(self): return self.pp
    def set_ppcie_mode(self, m): pass
    def reset_with_os(self): self.cc = self.staged
    def wait_for_boot(self): pass

    def scrub_and_verify(self, nbytes=0, check="zero"):
        if self.dirt is None:
            rep = report(self.bdf)
            rep.check = check
            return rep
        err = GpuError(f"scrub_and_verify on {self.bdf}: HBM verify found non-zero bytes after the scrub", N.ERR_DIRTY)
        err.dirt = self.dirt
        raise err


def manager_for(devs, monkeypatch, labels=None, **kw):
    import kubernetes
    from k8s_cc_manager_b200 import manager
    c = kubernetes.reset_cluster()
    c.add_node(SC.NODE, labels or {})
    monkeypatch.setenv("EVICT_OPERATOR_COMPONENTS", "false")
    source = (lambda: (devs, len(devs))) if devs is not None else None
    return manager.CCManager(SC.NODE, "on", True, device_source=source, **kw), c


def assert_dirt_logged(mgr, c, caplog, bdf, dirt):
    assert c.labels(SC.NODE).get("nvidia.com/cc.mode.state") == "failed"
    assert mgr.last_transition["scrub_dirt"] == {bdf: dirt}
    lines = [r.getMessage() for r in caplog.records if f"HBM dirt on {bdf}" in r.getMessage()]
    assert len(lines) == 1
    assert "0x10..0x2011" in lines[0] and "2 dirty 16-byte windows" in lines[0] and "chunks [0, 3]" in lines[0]
    assert "+0x2010 chunk 3 mask 0003" in lines[0]


@pytest.mark.parametrize("check", ["zero", "tagged"])
def test_per_gpu_fan_out_logs_and_keeps_the_report(check, monkeypatch, caplog):
    dirt = sample_dirt()
    devs = [FakeGpu(SC.GPU_BDFS[0]), FakeGpu(SC.GPU_BDFS[1], dirt=dirt)]
    mgr, c = manager_for(devs, monkeypatch, scrub_check=check)
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is False
    assert_dirt_logged(mgr, c, caplog, SC.GPU_BDFS[1], dirt)
    assert any("GPU error setting CC mode: scrub_and_verify on" in r.getMessage() for r in caplog.records)


def test_regate_logs_and_keeps_the_report(monkeypatch, caplog):
    dirt = sample_dirt()
    devs = [FakeGpu(SC.GPU_BDFS[0], cc="on", dirt=dirt)]
    mgr, c = manager_for(devs, monkeypatch, labels={"nvidia.com/cc.mode.state": "failed"})
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is False
    assert mgr.last_transition["regate"] is True
    assert_dirt_logged(mgr, c, caplog, SC.GPU_BDFS[0], dirt)


def _native_world(monkeypatch, n=2):
    build_native_world(SC.scenario("w", gpus_=SC.gpus(n), modes=[]))
    for k, v in dict(CCM_BACKEND="sim", CCM_SIM_GPUS=str(n), CCM_SIM_BIND_CUDA="0").items():
        monkeypatch.setenv(k, v)


def test_native_fan_out_logs_and_keeps_the_report(monkeypatch, caplog):
    from k8s_cc_manager_b200 import manager
    _native_world(monkeypatch)
    dirt = sample_dirt()

    def fake_many(devices, nbytes=0, **kw):
        reps = [report(d.bdf) for d in devices]
        reps[1] = report(devices[1].bdf, nonzero=3)
        reps[1].dirt = dirt
        return reps, 1.0
    monkeypatch.setattr(manager._devices, "scrub_and_verify_many", fake_many)
    mgr, c = manager_for(None, monkeypatch)
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is False
    bdf = mgr.last_transition["scrub"][1].bdf
    assert_dirt_logged(mgr, c, caplog, bdf, dirt)
    assert any(f"HBM scrub failed on {bdf}: status=-8 nonzero_bytes=3 of {190 << 30}" in r.getMessage()
               for r in caplog.records)


def test_worker_process_report_carries_the_dirt(monkeypatch, caplog):
    _native_world(monkeypatch)
    monkeypatch.setenv("CC_SCRUB_ISOLATION", "process")
    dirt = sample_dirt()
    captured = {}

    def fake_run(cmd, **kw):
        bdfs = [cmd[i + 1] for i, a in enumerate(cmd) if a == "--bdf"]
        reps = [report(b).as_json() for b in bdfs]
        bad = report(bdfs[0], nonzero=3)
        bad.dirt = dirt
        reps[0] = bad.as_json()
        captured["bdf"] = bdfs[0]
        return subprocess.CompletedProcess(cmd, 3, json.dumps({"wall_ms": 1.0, "reports": reps}) + "\n", "")
    monkeypatch.setattr(subprocess, "run", fake_run)
    mgr, c = manager_for(None, monkeypatch)
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is False
    assert_dirt_logged(mgr, c, caplog, captured["bdf"], dirt)
    assert mgr.last_transition["scrub"][0].dirt == dirt and mgr.last_transition["scrub"][1].dirt is None


def test_clean_gate_records_no_dirt(monkeypatch):
    mgr, c = manager_for([FakeGpu(b) for b in SC.GPU_BDFS[:2]], monkeypatch)
    assert mgr.set_cc_mode("on") is True
    assert "scrub_dirt" not in mgr.last_transition
