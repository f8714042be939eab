"""The mismatch triage on the CPU: the oracle's classes against a byte-level model of the triage's steps and drills,
the C ABI without a CUDA device (exports, refused arguments, the drill keys and their header text), the report in
ScrubReport's JSON, the device API's refusal of a zero-only call, the worker's and the CLI's flag and key, and the
manager's knob: its validation, every gate path that passes it on, its log line, its last_transition key and the
warning for a device that cannot triage mismatches."""
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
import test_dirt_triage as TT
import test_tag_mismatch as TM
from helpers import build_native_world
from k8s_cc_manager_b200 import _native as N
from k8s_cc_manager_b200 import devices as D
from k8s_cc_manager_b200.devices import GpuError, ScrubReport, TriagePage, TriageReport

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "oracle"))
import mismatch_triage_oracle as MTR  # noqa: E402
import triage_oracle as TR  # noqa: E402

MiB = 1 << 20
PAGE = TR.PAGE_BYTES


# ---------------------------------------------------------------------------------- oracle against a byte-level model
def tags_of(total: int, seed: int) -> np.ndarray:
    """Some address tags: one byte per offset of the mapping (what matters is that T1 writes what T2 checks)."""
    o = np.arange(total, dtype=np.uint64)
    return ((o * np.uint64(0x9E3779B1) + np.uint64(seed)) >> np.uint64(7)).astype(np.uint8)


def model(spans, total: int, bad: np.ndarray, seed: int, stay: int, ret: int):
    """The tagged gate and the mismatch triage, byte by byte, on memory that keeps what is stored: the gate checks the
    tags with the bytes at `bad` XORed, books their pages and zeroes everything; the triage re-tags every mapped byte of
    every booked page, XORs the stay bytes, checks and zeroes, XORs the return bytes and reads for non-zero bytes.
    Returns (mismatch page map entries, per-page (T2, T3) bytes, the memory the triage left)."""
    tag = tags_of(total, seed)
    mem = tag.copy()
    mem[bad] ^= 0xA5
    chunk_of = [next(k for k, (so, sn) in enumerate(spans) if so <= p * PAGE < so + sn) for p in range(-(-total // PAGE))]
    booked = np.bincount(np.flatnonzero(mem != tag) // PAGE, minlength=len(chunk_of))
    entries = [(p, int(n), chunk_of[p]) for p, n in enumerate(booked) if n]
    mem[:] = 0                                             # the gate's check zeroes all it checks
    examined = np.zeros(total, bool)
    for p, _, _ in entries:
        examined[p * PAGE:(p + 1) * PAGE] = True           # every span is mapped: each page's mapped bytes
    mem[examined] = tag[examined]                          # T1
    for p, _, _ in entries[:stay]:
        mem[p * PAGE] ^= 0xA5
    t2 = np.bincount(np.flatnonzero(examined & (mem != tag)) // PAGE, minlength=len(chunk_of))
    mem[examined] = 0                                      # T2 zeroes what it checks
    for p, _, _ in entries[:ret]:
        mem[p * PAGE] ^= 0xA5
    t3 = np.bincount(np.flatnonzero(examined & (mem != 0)) // PAGE, minlength=len(chunk_of))
    return entries, {p: (int(t2[p]), int(t3[p])) for p, _, _ in entries}, mem


def layouts():
    """(spans, total): one mapping, and cudaMalloc segments of 3, 1 and 5 MiB whose boundaries fall inside pages."""
    total = 7 * PAGE - MiB
    yield [(0, total)], total
    for seg in (3, 1, 5):
        yield [(o, min(seg * MiB, total - o)) for o in range(0, total, seg * MiB)], total


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("stay,ret", [(0, 0), (1, 0), (0, 1), (2, 3), (3, 2), (100, 0), (0, 100), (100, 100)])
def test_oracle_matches_a_byte_level_model(seed, stay, ret):
    rng = np.random.default_rng(seed)
    for spans, total in layouts():
        bad = np.unique(rng.integers(0, total, int(rng.integers(1, 12))))
        entries, per_page, mem = model(spans, total, bad, seed, stay, ret)
        rows = MTR.classify(entries, stay, ret)
        assert [(r[0], r[4], r[5]) for r in rows] == [(p, *per_page[p]) for p, _, _ in entries]
        for page, chunk, cls, nbytes, t2, t3 in rows:
            assert cls == ("stays" if t2 else "returns" if t3 else "clears")
        rep = MTR.report(entries, spans, stay, ret)
        assert rep["t2_bytes"] == sum(t2 for t2, _ in per_page.values())
        assert rep["t3_bytes"] == sum(t3 for _, t3 in per_page.values())
        assert rep["stay_bytes"] + rep["return_bytes"] + rep["clear_bytes"] == len(bad)   # == mismatch_bytes
        assert rep["bytes_examined"] == sum(min(PAGE, total - p * PAGE) for p, _, _ in entries)
        # what the triage leaves behind: zero, but for the return drill's bytes
        left = np.flatnonzero(mem)
        assert list(left) == [p * PAGE for p, _, _ in entries[:ret]]


def test_mismatch_classes_differ_from_the_dirt_triage_only_where_both_drills_hit():
    entries = [(p, 3, 0) for p in (0, 2, 3, 9)]
    for stay, ret in ((2, 3), (3, 1), (4, 4)):
        dirt, mm = TR.classify(entries, stay, ret), MTR.classify(entries, stay, ret)
        for i, (d, m) in enumerate(zip(dirt, mm)):
            assert d[:5] == m[:5]                          # the class and T2 are the same
            assert m[5] == int(i < ret) and d[5] == int((i < stay) != (i < ret))


# ---------------------------------------------------------------------------------- C ABI
ENTRY_POINTS = ("ccm_scrub_mismatch_triage", "ccm_scrub_last_mismatch_triage", "ccm_last_mismatch_triage_pages")


def test_entry_points_are_exported_and_refuse_what_they_must(native):
    lib = native.lib()
    nm = subprocess.run(["nm", "-D", "--defined-only", str(native.LIB_PATH)], capture_output=True, text=True,
                        check=True).stdout
    for fn in ENTRY_POINTS:
        assert fn in native.EXPORTED_SYMBOLS and re.search(rf" T {fn}$", nm, re.M), fn
    for ordinal in (0, -1, 1 << 12):
        assert lib.ccm_scrub_mismatch_triage(ordinal, native.TRIAGE_MAX_HOLD_MS + 1) == native.ERR_INVALID
        assert "ccm_scrub_mismatch_triage: hold of 10001 ms is longer than 10000 ms" in native.last_error()
        assert lib.ccm_scrub_mismatch_triage(ordinal, 0xFFFFFFFF) == native.ERR_INVALID
    for ordinal in (-1, 1 << 12):
        for hold in (0, 1, native.TRIAGE_MAX_HOLD_MS):
            assert lib.ccm_scrub_mismatch_triage(ordinal, hold) == native.ERR_NO_CUDA
        rep = native.TriageReport(triaged=7)
        assert lib.ccm_scrub_last_mismatch_triage(ordinal, C.byref(rep)) == native.ERR_NO_CUDA and rep.triaged == 0
        n = C.c_uint64(7)
        assert lib.ccm_last_mismatch_triage_pages(ordinal, None, 0, C.byref(n)) == native.ERR_NO_CUDA and n.value == 0
    assert lib.ccm_scrub_last_mismatch_triage(0, None) == native.ERR_INVALID
    assert lib.ccm_last_mismatch_triage_pages(0, None, 0, None) == native.ERR_INVALID
    n = C.c_uint64()
    assert lib.ccm_last_mismatch_triage_pages(0, None, 3, C.byref(n)) == native.ERR_INVALID
    assert "ccm_last_mismatch_triage_pages: cap 3" in native.last_error()
    assert D.last_mismatch_triage(-1) is None and D.last_mismatch_triage_pages(-1) is None


def test_tag_flood_key_round_trips_and_takes_a_byte(native):
    lib = native.lib()
    assert lib.ccm_sim_topology(2, 0) == 0
    assert lib.ccm_sim_set(-1, b"cuda_ordinal", -1) == 0
    v = C.c_int64(-1)
    assert lib.ccm_sim_get(0, b"tag_flood", C.byref(v)) == 0 and v.value == 0
    assert lib.ccm_sim_set(0, b"tag_flood", 0x5A) == 0 and lib.ccm_sim_get(0, b"tag_flood", C.byref(v)) == 0
    assert v.value == 0x5A
    assert lib.ccm_sim_get(1, b"tag_flood", C.byref(v)) == 0 and v.value == 0
    for bad in (-1, 256):
        assert lib.ccm_sim_set(0, b"tag_flood", bad) == native.ERR_INVALID
        assert "takes a byte value" in native.last_error()
    assert lib.ccm_sim_set(0, b"tag_flood", 0) == 0


def test_header_documents_the_entry_points_and_the_drills():
    header = (ROOT / "include" / "ccm.h").read_text()
    for fn in ENTRY_POINTS:
        assert re.search(rf"^int {fn}\(", header, re.M), fn
    assert '"tag_flood"' in header and "bytes of the MISMATCH page map" in header
    assert "page i has T2 bytes [i < stay] and\n * T3 bytes [i < ret]" in header
    assert "In a call that triages mismatches (ccm_scrub_mismatch_triage)" in header
    assert "#define CCM_ABI_VERSION 2 " in header


# ---------------------------------------------------------------------------------- device API and JSON
def test_json_carries_the_report_only_when_a_triage_ran():
    rep = TM.report(mismatch=5)
    rep.mismatch = TM.sample_mismatch()
    base = set(json.loads(json.dumps(rep.as_json())))
    assert rep.mismatch_triage is None and "mismatch_triage" not in ScrubReport.__dataclass_fields__
    rep.mismatch_triage = TT.sample_triage(stay=1, ret=0, clear=3)
    js = json.loads(json.dumps(rep.as_json()))
    assert set(js) == base | {"mismatch_triage"}
    back = ScrubReport.from_json(js)
    assert back.mismatch_triage == rep.mismatch_triage and back.triage is None and back.mismatch == rep.mismatch
    assert ScrubReport.from_json(TM.report().as_json()).mismatch_triage is None
    assert GpuError("x").mismatch_triage is None


def test_device_api_takes_mismatch_triage():
    for fn in (D.NvidiaDevice.scrub_and_verify, D.ScrubbingProxy.scrub_and_verify, D.scrub_and_verify_many):
        assert inspect.signature(fn).parameters["mismatch_triage"].default is False


def test_device_api_refuses_it_without_the_tagged_check(native):
    """check="zero" with mismatch_triage=True is a ValueError before anything runs; without CUDA the tagged call fails
    as it does unarmed."""
    lib = native.lib()
    assert lib.ccm_sim_topology(1, 0) == 0
    assert lib.ccm_sim_set(-1, b"cuda_ordinal", -1) == 0
    gpu = D.find_gpus()[0][0]
    with pytest.raises(ValueError, match="mismatch_triage needs check='tagged'"):
        gpu.scrub_and_verify(MiB, mismatch_triage=True)
    with pytest.raises(ValueError, match="mismatch_triage needs check='tagged'"):
        D.scrub_and_verify_many([gpu], MiB, mismatch_triage=True)
    with pytest.raises(ValueError, match="mismatch_triage needs check='tagged'"):
        D.ScrubbingProxy(object(), gpu).scrub_and_verify(MiB, mismatch_triage=True)
    with pytest.raises(ValueError):
        gpu.scrub_and_verify(MiB, check="tagged", mismatch_triage=True, triage_hold_ms=0)
    with pytest.raises(GpuError) as plain:
        gpu.scrub_and_verify(MiB, check="tagged")
    with pytest.raises(GpuError) as armed:
        gpu.scrub_and_verify(MiB, check="tagged", mismatch_triage=True)
    assert armed.value.status == plain.value.status == N.ERR_NO_CUDA and armed.value.mismatch_triage is None
    reps, _ = D.scrub_and_verify_many([gpu], MiB, check="tagged", mismatch_triage=True)
    assert reps[0].status == N.ERR_NO_CUDA and reps[0].mismatch_triage is None


class _Native:
    """Records the keyword arguments ScrubbingProxy passes on."""

    def __init__(self):
        self.calls = []

    def scrub_and_verify(self, nbytes, **kw):
        self.calls.append(kw)
        return "report"


def test_proxy_passes_mismatch_triage_only_when_it_is_set():
    native = _Native()
    proxy = D.ScrubbingProxy(SimpleForeign(), native)
    proxy.scrub_and_verify(0, check="tagged")
    proxy.scrub_and_verify(0, check="tagged", triage=True)
    proxy.scrub_and_verify(0, check="tagged", mismatch_triage=True, triage_hold_ms=7)
    assert "mismatch_triage" not in native.calls[0] and "mismatch_triage" not in native.calls[1]
    assert native.calls[2] == dict(check="tagged", residue=False, triage=False, triage_hold_ms=7, mismatch_triage=True)


class SimpleForeign:
    bdf = SC.GPU_BDFS[0]


# ---------------------------------------------------------------------------------- CLI and worker
def test_cli_prints_the_keys_the_worker_prints():
    src = (ROOT / "k8s_cc_manager_b200" / "csrc" / "ccm_scrub_cli.cpp").read_text()
    body = src[src.index("static void print_mismatch_triage"):src.index("static int usage")]
    printed = set(re.findall(r'\\"(\w+)\\":', body))
    assert printed == {"mismatch_triage"} | set(TriageReport.__dataclass_fields__) | set(TriagePage.__dataclass_fields__)
    assert "ccm_last_mismatch_triage_pages(ordinal" in body and "keep = 64" in body
    assert 'else if (a == "--mismatch-triage") mismatch_triage = true;' in src
    assert "ccm_scrub_mismatch_triage(ordinals[i]" in src and "ccm_scrub_mismatch_triage(o, 0)" in src


def test_cli_refuses_the_flag_without_the_tagged_check():
    cli = ROOT / "k8s_cc_manager_b200" / "ccm-scrub"
    if not cli.exists():
        pytest.skip("ccm-scrub is not built")
    proc = subprocess.run([str(cli), "--backend", "sim", "--mismatch-triage", "--all"], capture_output=True, text=True,
                          timeout=60)
    assert proc.returncode == 2 and "--mismatch-triage needs --check tagged" in proc.stderr and proc.stdout == ""


class _Dev:
    def __init__(self, bdf): self.bdf = bdf
    def is_gpu(self): return True


def test_worker_takes_mismatch_triage(monkeypatch, capsys):
    from k8s_cc_manager_b200 import scrub_worker
    rep = TM.report("0000:01:00.0", mismatch=5)
    rep.mismatch, rep.mismatch_triage = TM.sample_mismatch(), TT.sample_triage()
    seen = []

    def fake_many(devs, n, check="zero", residue=False, triage=False, triage_hold_ms=D.TRIAGE_HOLD_MS,
                  mismatch_triage=False):
        seen.append((check, residue, triage, triage_hold_ms, mismatch_triage))
        return [rep], 1.0
    monkeypatch.setattr(D, "find_gpus", lambda: ([_Dev(rep.bdf)], 1))
    monkeypatch.setattr(D, "scrub_and_verify_many", fake_many)
    assert scrub_worker.main(["--bdf", rep.bdf, "--check", "tagged", "--mismatch-triage"]) == 3
    out = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    assert TriageReport.from_json(out["reports"][0]["mismatch_triage"]) == rep.mismatch_triage
    assert scrub_worker.main(["--bdf", rep.bdf, "--check", "tagged", "--mismatch-triage", "--triage",
                              "--triage-hold-ms", "250", "--residue"]) == 3
    assert seen == [("tagged", False, False, 100, True), ("tagged", True, True, 250, True)]
    with pytest.raises(SystemExit) as ei:
        scrub_worker.main(["--bdf", rep.bdf, "--mismatch-triage"])
    assert ei.value.code == 2 and "--mismatch-triage needs --check tagged" in capsys.readouterr().err
    assert len(seen) == 2


# ---------------------------------------------------------------------------------- manager
class FakeGpu(TM.FakeGpu):
    """A device whose tagged check fails and that takes `mismatch_triage` (and `triage`); can_triage False: an older
    device library."""

    def __init__(self, bdf, mismatch=None, mtriage=None, can_triage=True, cc="off"):
        super().__init__(bdf, cc=cc, mismatch=mismatch)
        self.mtriage, self.calls = mtriage, []
        if can_triage:
            self.scrub_and_verify = self._scrub_triage

    def scrub_and_verify(self, nbytes=0, check="zero"):
        self.calls.append((nbytes, check, None))
        return super().scrub_and_verify(nbytes, check)

    def _scrub_triage(self, nbytes=0, check="zero", residue=False, triage=False, triage_hold_ms=100,
                      mismatch_triage=False):
        self.calls.append((nbytes, check, dict(residue=residue, triage=triage, hold=triage_hold_ms,
                                               mismatch_triage=mismatch_triage)))
        try:
            return TM.FakeGpu.scrub_and_verify(self, nbytes, check)
        except GpuError as err:
            err.mismatch_triage = self.mtriage if mismatch_triage else None
            err.triage = TT.sample_triage(stay=0, ret=0, clear=1) if triage else None
            raise


def mtriage_lines(caplog):
    return [r.getMessage() for r in caplog.records if r.getMessage().startswith("HBM mismatch triage on ")]


def manager_for(devs, monkeypatch, **kw):
    kw.setdefault("scrub_check", "tagged")
    return TD.manager_for(devs, monkeypatch, **kw)


@pytest.mark.parametrize("value,want", [(None, "off"), ("off", "off"), ("report", "report"), ("REPORT", "report")])
def test_setting_is_parsed(monkeypatch, value, want):
    if value is not None:
        monkeypatch.setenv("CC_SCRUB_MISMATCH_TRIAGE", value)
    mgr, _ = manager_for([FakeGpu(SC.GPU_BDFS[0])], monkeypatch)
    assert mgr.scrub_mismatch_triage == want and mgr.mismatch_triage == (want == "report")


def test_other_values_and_the_zero_check_are_rejected(monkeypatch):
    from k8s_cc_manager_b200 import manager
    for bad in ("on", "1", "stay"):
        monkeypatch.setenv("CC_SCRUB_MISMATCH_TRIAGE", bad)
        with pytest.raises(ValueError, match="CC_SCRUB_MISMATCH_TRIAGE must be"):
            manager_for([FakeGpu(SC.GPU_BDFS[0])], monkeypatch)
    monkeypatch.setenv("CC_SCRUB_MISMATCH_TRIAGE", "report")
    with pytest.raises(ValueError, match="needs CC_SCRUB_CHECK=tagged"):
        manager_for([FakeGpu(SC.GPU_BDFS[0])], monkeypatch, scrub_check="zero")
    monkeypatch.delenv("CC_SCRUB_MISMATCH_TRIAGE")
    with pytest.raises(ValueError, match="needs CC_SCRUB_CHECK=tagged"):
        manager_for([FakeGpu(SC.GPU_BDFS[0])], monkeypatch, scrub_check="zero", scrub_mismatch_triage="report")
    args = manager.build_arg_parser().parse_args(["--scrub-mismatch-triage", "report"])
    assert args.scrub_mismatch_triage == "report"
    assert manager.build_arg_parser().parse_args([]).scrub_mismatch_triage is None
    with pytest.raises(SystemExit):
        manager.build_arg_parser().parse_args(["--scrub-mismatch-triage", "on"])


@pytest.mark.parametrize("dirt_triage", [False, True])
def test_per_gpu_gate_passes_it_logs_and_keeps_the_report(monkeypatch, caplog, dirt_triage):
    mm, mt = TM.sample_mismatch(), TT.sample_triage(stay=2, ret=0, clear=2)
    devs = [FakeGpu(SC.GPU_BDFS[0]), FakeGpu(SC.GPU_BDFS[1], mismatch=mm, mtriage=mt)]
    extra = {"scrub_triage": "report"} if dirt_triage else {}
    mgr, c = manager_for(devs, monkeypatch, scrub_mismatch_triage="report", **extra)
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is False
    bdf = SC.GPU_BDFS[1]
    TM.assert_mismatch_logged(mgr, c, caplog, bdf, mm)
    want = dict(residue=False, triage=dirt_triage, hold=100, mismatch_triage=True)
    assert all(d.calls == [(0, "tagged", want)] for d in devs)
    assert mgr.last_transition["scrub_mismatch_triage"] == {bdf: mt}
    lines = mtriage_lines(caplog)
    assert lines == [f"HBM mismatch triage on {bdf}: {mt.summary()}"]
    assert lines[0].startswith(f"HBM mismatch triage on {bdf}: 4 pages in 4 runs: 2 stay, 0 return, 2 clear")
    msgs = [r.getMessage() for r in caplog.records]
    assert msgs.index(lines[0]) > msgs.index(next(m for m in msgs if m.startswith(f"HBM tag mismatch on {bdf}: ")))
    if dirt_triage:   # the dirt triage's line comes first
        dirt_line = next(m for m in msgs if m.startswith(f"HBM dirt triage on {bdf}: "))
        assert msgs.index(dirt_line) < msgs.index(lines[0])


def test_off_takes_the_calls_it_always_took(monkeypatch, caplog):
    devs = [FakeGpu(SC.GPU_BDFS[0]), FakeGpu(SC.GPU_BDFS[1], mismatch=TM.sample_mismatch(), mtriage=TT.sample_triage())]
    mgr, _ = manager_for(devs, monkeypatch)
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is False
    assert all(d.calls == [(0, "tagged", dict(residue=False, triage=False, hold=100, mismatch_triage=False))]
               for d in devs)   # scrub_and_verify(0, check="tagged"): no mismatch_triage passed
    assert "scrub_mismatch_triage" not in mgr.last_transition and mtriage_lines(caplog) == []


def test_a_device_without_it_warns_and_runs_its_gate_unchanged(monkeypatch, caplog):
    mm = TM.sample_mismatch()
    devs = [FakeGpu(SC.GPU_BDFS[0], can_triage=False), FakeGpu(SC.GPU_BDFS[1], mismatch=mm, can_triage=False)]
    mgr, c = manager_for(devs, monkeypatch, scrub_mismatch_triage="report")
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is False
    warnings = [r.getMessage() for r in caplog.records if r.levelno == logging.WARNING and "cannot triage" in
                r.getMessage()]
    assert sorted(warnings) == sorted(f"Device {d.bdf} cannot triage HBM tag mismatches (CC_SCRUB_MISMATCH_TRIAGE="
                                      "report): its gate runs without the mismatch triage" for d in devs)
    assert all(d.calls == [(0, "tagged", None)] for d in devs)
    TM.assert_mismatch_logged(mgr, c, caplog, SC.GPU_BDFS[1], mm)
    assert "scrub_mismatch_triage" not in mgr.last_transition and mtriage_lines(caplog) == []


def test_a_device_with_only_the_dirt_triage_keeps_it(monkeypatch, caplog):
    """CC_SCRUB_TRIAGE=report too: a device that takes `triage` but not `mismatch_triage` runs the dirt triage call."""
    dev = TT.FakeGpu(SC.GPU_BDFS[0])
    mgr, _ = manager_for([dev], monkeypatch, scrub_triage="report", scrub_mismatch_triage="report")
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is True
    assert dev.calls == [(0, "tagged", True, 100)]
    assert any("cannot triage HBM tag mismatches" in r.getMessage() for r in caplog.records)


def _native_world(monkeypatch, n=2):
    build_native_world(SC.scenario("w", gpus_=SC.gpus(n), modes=[]))
    for k, v in dict(CCM_BACKEND="sim", CCM_SIM_GPUS=str(n), CCM_SIM_BIND_CUDA="0").items():
        monkeypatch.setenv(k, v)


def failed_report(bdf):
    r = TM.report(bdf, mismatch=5)
    r.mismatch, r.mismatch_triage = TM.sample_mismatch(), TT.sample_triage()
    return r


@pytest.mark.parametrize("dirt_triage", [False, True])
def test_native_fan_out_passes_it(monkeypatch, caplog, dirt_triage):
    from k8s_cc_manager_b200 import manager
    _native_world(monkeypatch)
    seen = {}

    def fake_many(devices, nbytes=0, check="zero", residue=False, triage=False, triage_hold_ms=D.TRIAGE_HOLD_MS,
                  mismatch_triage=False):
        seen.update(check=check, residue=residue, triage=triage, hold=triage_hold_ms, mismatch_triage=mismatch_triage)
        return [failed_report(d.bdf) for d in devices], 1.0
    monkeypatch.setattr(manager._devices, "scrub_and_verify_many", fake_many)
    mgr, c = manager_for(None, monkeypatch, scrub_mismatch_triage="report",
                         scrub_triage="report" if dirt_triage else None)
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is False
    assert seen == {"check": "tagged", "residue": False, "triage": dirt_triage, "hold": manager.SCRUB_TRIAGE_HOLD_MS,
                    "mismatch_triage": True}
    bdfs = [r.bdf for r in mgr.last_transition["scrub"]]
    assert set(mgr.last_transition["scrub_mismatch_triage"]) == set(bdfs) and len(mtriage_lines(caplog)) == 2


@pytest.mark.parametrize("dirt_triage", [False, True])
def test_worker_process_passes_it(monkeypatch, caplog, dirt_triage):
    _native_world(monkeypatch)
    monkeypatch.setenv("CC_SCRUB_ISOLATION", "process")
    monkeypatch.setenv("CC_SCRUB_MISMATCH_TRIAGE", "report")
    if dirt_triage:
        monkeypatch.setenv("CC_SCRUB_TRIAGE", "report")
    cmds = []

    def fake_run(cmd, **kw):
        cmds.append(cmd)
        bdfs = [cmd[i + 1] for i, a in enumerate(cmd) if a == "--bdf"]
        reps = [failed_report(b).as_json() for b in bdfs]
        return subprocess.CompletedProcess(cmd, 3, json.dumps({"wall_ms": 1.0, "reports": reps}) + "\n", "")
    monkeypatch.setattr(subprocess, "run", fake_run)
    mgr, c = manager_for(None, monkeypatch)
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is False
    cmd = cmds[0]
    assert len(cmds) == 1 and "--mismatch-triage" in cmd and cmd[cmd.index("--check") + 1] == "tagged"
    assert cmd.count("--triage-hold-ms") == 1 and cmd[cmd.index("--triage-hold-ms") + 1] == "100"
    assert ("--triage" in cmd) == dirt_triage
    assert all(r.mismatch_triage == TT.sample_triage() for r in mgr.last_transition["scrub"])
    assert len(mgr.last_transition["scrub_mismatch_triage"]) == 2 and len(mtriage_lines(caplog)) == 2


def test_a_clean_gate_with_it_passes(monkeypatch, caplog):
    devs = [FakeGpu(SC.GPU_BDFS[0]), FakeGpu(SC.GPU_BDFS[1])]
    mgr, _ = manager_for(devs, monkeypatch, scrub_mismatch_triage="report")
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is True
    assert "scrub_mismatch_triage" not in mgr.last_transition and mtriage_lines(caplog) == []
