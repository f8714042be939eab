"""The mismatch report on the CPU: the numpy oracle against a brute-force search of every window of small mappings,
the host classification header against the oracle, the C structs against ctypes, the JSON of reports with and
without a mismatch report, summary(), the manager's log line and last_transition["scrub_mismatch"] on every gate
path, the CLI and worker output, and the new entry points without a CUDA device."""
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
from k8s_cc_manager_b200.devices import GpuError, MismatchReport, MismatchWindow, ScrubReport

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "oracle"))
import mismatch_oracle as MO  # noqa: E402
import tag_oracle as TO  # noqa: E402

GiB = 1 << 30
SEED = 0x1234_5678


# ---------------------------------------------------------------------------------- oracle vs brute force
def brute_force(buf: np.ndarray, addr: int, seed: int, ranges) -> list:
    """Byte by byte, and for an alias every 16-aligned window of `ranges` tried in turn."""
    n = buf.size
    tags = [TO.tag_word_py(seed, a & ~3) >> (8 * (a & 3)) & 0xFF for a in range(addr, addr + n)]
    wins = {}
    for i in range(n):
        if int(buf[i]) != tags[i]:
            w = (addr + i) & ~15
            wins[w] = wins.get(w, 0) | 1 << ((addr + i) & 15)
    candidates = [s for lo, hi in ranges for s in range((lo + 15) & ~15, hi, 16)]
    out = []
    for w, mask in sorted(wins.items()):
        present = [w + i for i in range(16) if addr <= w + i < addr + n]
        got = {a: int(buf[a - addr]) for a in present}
        if all(v == 0 for v in got.values()):
            kind, src = "zero", None
        else:
            hits = [s for s in candidates if s != w and all(
                any(lo <= s + (a - w) < hi for lo, hi in ranges) and got[a] == MO.tag_byte_py(seed, s + (a - w))
                for a in present)]
            # a match needs one whole word inside the buffer
            whole = any(all(w + 4 * k + j in got for j in range(4)) for k in range(4))
            if hits and whole:
                kind, src = "alias", hits[0]
            elif any(got[a] == MO.tag_byte_py(seed, a) for a in present):
                kind, src = "partial", None
            else:
                kind, src = "foreign", None
        out.append((w - addr, mask, kind, (src - addr) if src is not None else 0))
    return out


def oracle_windows(rep):
    return [(w["offset"], w["mask"], w["kind"], w["source_offset"]) for w in rep["windows"]]


def tagged(addr, n, seed=SEED):
    return TO.tag_bytes(seed, addr, n).copy()


@pytest.mark.parametrize("addr", [0x7F00_0000_0000, 0x7F00_0000_0003, 0x7F00_0000_000E, 0x3_FFFF_FF80 + 5])
def test_oracle_matches_brute_force(addr):
    rng = np.random.default_rng(addr & 0xFF)
    n = 16 * 24 + 9
    other = (addr & ~15) + 16 * 40                            # a second mapped range, not the buffer
    ranges = [(addr, addr + n), (other, other + 256)]
    buf = tagged(addr, n)
    a0 = (16 - addr % 16) % 16                               # first aligned byte offset
    buf[a0 + 16: a0 + 32] = 0                                # zero window
    buf[a0 + 35] ^= 0xA5                                     # partial
    buf[a0 + 64: a0 + 80] = rng.integers(0, 256, 16)         # foreign
    buf[a0 + 96: a0 + 112] = TO.tag_bytes(SEED, addr + a0 + 96 + 48, 16)        # alias in the buffer, delta +48
    buf[a0 + 128: a0 + 144] = TO.tag_bytes(SEED, other + 32, 16)                # alias into the other range
    buf[a0 + 160: a0 + 176] = TO.tag_bytes(SEED + 1, addr + a0 + 160, 16)       # another call's tags
    buf[: a0] = 0                                            # ragged head window: zero (if any)
    buf[n - 3:] ^= 0x11                                      # ragged tail bytes
    rep = MO.report(buf, addr, SEED, ranges)
    assert oracle_windows(rep) == brute_force(buf, addr, SEED, ranges)
    kinds = {w["kind"] for w in rep["windows"]}
    assert {"zero", "partial", "foreign", "alias"} <= kinds
    assert rep["mismatch_bytes"] == int(np.count_nonzero(buf != TO.tag_bytes(SEED, addr, n)))
    assert rep["zero_windows"] == sum(w["zero"] for w in rep["windows"])


@pytest.mark.parametrize("delta", [16, 48, 256, -256, 1 << 34, -(1 << 34) + 16])
def test_alias_at_several_deltas_and_across_16_gib(delta):
    """Ranges straddle a 16 GiB boundary (hi32 of the word index changes there)."""
    base = (5 << 34) - 512
    ranges = [(base, base + 1024), (base + (1 << 34), base + (1 << 34) + 1024), (base - (1 << 34), base - (1 << 34) + 1024)]
    addr = base + 256
    buf = tagged(addr, 512)
    buf[0:16] = TO.tag_bytes(SEED, addr + delta, 16)
    buf[496:512] = TO.tag_bytes(SEED, addr + 496 + delta, 16)          # this one sits above the boundary
    rep = MO.report(buf, addr, SEED, ranges)
    bf = brute_force(buf, addr, SEED, ranges)
    assert [(o, k, s) for o, _, k, s in oracle_windows(rep)] == [(0, "alias", delta), (496, "alias", 496 + delta)]
    assert [(o, k, s) for o, _, k, s in bf] == [(0, "alias", delta), (496, "alias", 496 + delta)]
    assert (addr + 496) >> 34 != addr >> 34


@pytest.mark.parametrize("whole_words", [0, 1, 2])
def test_ragged_windows_need_a_whole_word_for_alias(whole_words):
    """A head window with 0, 1 or 2 whole words inside the buffer, holding another window's tags."""
    base = 0x7F00_0000_1000
    lead = {0: 13, 1: 9, 2: 5}[whole_words]                  # bytes of the head window outside the buffer
    addr = base + lead
    n = 64 - lead
    buf = tagged(addr, n)
    buf[: 16 - lead] = TO.tag_bytes(SEED, base + 32 + lead, 16 - lead)
    ranges = [(addr, addr + n)]
    rep = MO.report(buf, addr, SEED, ranges)
    assert oracle_windows(rep) == brute_force(buf, addr, SEED, ranges)
    head = rep["windows"][0]
    assert head["offset"] == -lead and head["kind"] == ("alias" if whole_words else "foreign")
    if whole_words:
        assert head["source_offset"] == 32 - lead


def test_clean_buffer_has_no_windows():
    rep = MO.report(tagged(0x1003, 1000), 0x1003, SEED)
    assert rep["mismatch_bytes"] == rep["mismatch_windows"] == 0 and rep["windows"] == []


# ---------------------------------------------------------------------------------- host header vs oracle
PROBE = r'''
#include <cstdio>
#include <vector>
#include "ccm_mismatch.h"
int main() {
  unsigned seed; unsigned long long w; unsigned present; int nr;
  while (scanf("%u %llx %x %d", &seed, &w, &present, &nr) == 4) {
    uint8_t b[16];
    for (int i = 0; i < 16; ++i) { unsigned x = 0; if (scanf("%x", &x) != 1) return 1; b[i] = (uint8_t)x; }
    std::vector<ccm_mismatch::Range> r(nr);
    for (auto& x : r)
      if (scanf("%llx %llx", (unsigned long long*)&x.lo, (unsigned long long*)&x.hi) != 2) return 1;
    const ccm_mismatch::Verdict v = ccm_mismatch::classify(seed, w, b, present, r.data(), r.size());
    printf("%d %llx\n", v.kind, (unsigned long long)v.source);
  }
  return 0;
}
'''


@pytest.fixture(scope="module")
def probe(tmp_path_factory):
    d = tmp_path_factory.mktemp("probe")
    (d / "probe.cpp").write_text(PROBE)
    subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-Werror", "-I", str(ROOT / "k8s_cc_manager_b200" / "csrc"),
                    str(d / "probe.cpp"), "-o", str(d / "probe")], check=True)
    return d / "probe"


@pytest.mark.parametrize("seed", range(4))
def test_host_header_matches_the_oracle(probe, seed):
    rng = np.random.default_rng(seed)
    tseed = int(rng.integers(1, 1 << 32))
    lines, want = [], []
    for trial in range(40):
        addr = int(rng.integers(1 << 36, 1 << 37)) & ~3 | int(rng.integers(0, 4)) if trial % 3 else (5 << 34) - 256 + 7
        n = int(rng.integers(40, 400))
        ranges = [(addr, addr + n), (addr + (1 << 34) - 128, addr + (1 << 34) + 512)]
        buf = tagged(addr, n, tseed)
        for _ in range(4):
            o = int(rng.integers(0, max(1, n - 16)))
            what = rng.integers(0, 4)
            if what == 0:
                buf[o:o + 16] = 0
            elif what == 1:
                buf[o] ^= 1 << int(rng.integers(0, 8))
            elif what == 2:
                o = ((addr + o + 15) & ~15) - addr             # a whole window
                src = addr + o + 16 * int(rng.integers(1, 4)) if rng.random() < 0.5 else addr + (1 << 34) + 16 * int(rng.integers(0, 8)) + (addr + o) % 16
                buf[o:o + 16] = TO.tag_bytes(tseed, src, len(buf[o:o + 16]))
            else:
                buf[o:o + 16] = rng.integers(0, 256, len(buf[o:o + 16]))
        rep = MO.report(buf, addr, tseed, ranges)
        for win in rep["windows"]:
            w = addr + win["offset"]
            data = bytes.fromhex(win["bytes"])
            present = sum(1 << i for i in range(16) if addr <= w + i < addr + n)
            lines.append(f"{tseed} {w:x} {present:x} {len(ranges)} " + " ".join(f"{b:x}" for b in data) + " "
                         + " ".join(f"{lo:x} {hi:x}" for lo, hi in ranges))
            kind = {"zero": 1, "alias": 2, "partial": 3, "foreign": 4}[win["kind"]]
            want.append((kind, (addr + win["source_offset"]) if win["kind"] == "alias" else 0))
    out = subprocess.run([str(probe)], input="\n".join(lines) + "\n", capture_output=True, text=True, check=True).stdout
    got = [(int(k), int(s, 16)) for k, s in (ln.split() for ln in out.splitlines())]
    assert got == want
    assert {k for k, _ in want} == {1, 2, 3, 4}


# ---------------------------------------------------------------------------------- C ABI
def test_struct_layouts_match_the_header(tmp_path):
    src = tmp_path / "mm.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "ccm.h"\nint main(void){'
                   'printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %d %d %d %d\\n",'
                   'sizeof(ccm_mismatch_record), offsetof(ccm_mismatch_record,chunk), offsetof(ccm_mismatch_record,mask),'
                   'offsetof(ccm_mismatch_record,kind), offsetof(ccm_mismatch_record,source_offset),'
                   'offsetof(ccm_mismatch_record,source_chunk), offsetof(ccm_mismatch_record,bytes),'
                   'sizeof(ccm_mismatch_report), offsetof(ccm_mismatch_report,va_base), offsetof(ccm_mismatch_report,seed),'
                   'offsetof(ccm_mismatch_report,located), offsetof(ccm_mismatch_report,truncated),'
                   'offsetof(ccm_mismatch_report,records), CCM_MISMATCH_ZERO, CCM_MISMATCH_ALIAS, CCM_MISMATCH_PARTIAL,'
                   'CCM_MISMATCH_FOREIGN);return 0;}')
    exe = tmp_path / "mm"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", str(ROOT / "include"), str(src), "-o", str(exe)],
                   check=True)
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    R, P = N.MismatchRecord, N.MismatchReport
    assert got == [C.sizeof(R), R.chunk.offset, R.mask.offset, R.kind.offset, R.source_offset.offset,
                   R.source_chunk.offset, R.bytes.offset, C.sizeof(P), P.va_base.offset, P.seed.offset,
                   P.located.offset, P.truncated.offset, P.records.offset, 1, 2, 3, 4]
    assert C.sizeof(R) == 48 and C.sizeof(P) == 64 + 48 * N.DIRT_RECORDS
    assert N.MISMATCH_KINDS == {1: "zero", 2: "alias", 3: "partial", 4: "foreign"}


def test_new_entry_points_are_exported_and_need_a_cuda_device(native):
    lib = native.lib()
    assert {"ccm_scrub_last_mismatch", "ccm_region_tag_check_locate"} <= set(native.EXPORTED_SYMBOLS)
    assert lib.ccm_abi_version() == 2
    for ordinal in (-1, 1 << 12):
        m = native.MismatchReport(located=7, nrecords=3)
        assert lib.ccm_scrub_last_mismatch(ordinal, C.byref(m)) == native.ERR_NO_CUDA
        assert m.located == 0 and m.nrecords == 0
        buf = (C.c_uint8 * 64)()
        assert lib.ccm_region_tag_check_locate(ordinal, buf, 64, 1, None, C.byref(m)) == native.ERR_NO_CUDA
    assert lib.ccm_scrub_last_mismatch(0, None) == native.ERR_INVALID
    assert lib.ccm_region_tag_check_locate(0, None, 0, 1, None, None) == native.ERR_INVALID
    assert D.last_mismatch(-1) is None


def test_native_report_converts_with_kinds_and_signed_offsets():
    m = N.MismatchReport(mismatch_bytes=17, mismatch_windows=2, zero_windows=1, first_offset=0, last_offset=0x40000010,
                         va_base=0x7F00_0000_0000, seed=9, located=1, nrecords=2, truncated=0)
    m.records[0].offset, m.records[0].kind, m.records[0].mask = (1 << 64) - 3, 1, 0xFFF8
    m.records[1].offset, m.records[1].kind, m.records[1].mask = 0x10, 2, 0xFFFF
    m.records[1].source_offset, m.records[1].source_chunk, m.records[1].chunk = 0x40000010, 1, 0
    rep = MismatchReport.from_native(m)
    assert [(r.offset, r.kind, r.source_offset, r.source_chunk) for r in rep.records] == [
        (-3, "zero", 0, 0), (0x10, "alias", 0x40000010, 1)]
    assert rep.seed == 9 and rep.zero_windows == 1


# ---------------------------------------------------------------------------------- JSON, summary
def alias_rec(off, delta=0x40000000, chunk=0, src_chunk=0):
    return MismatchWindow(off, chunk, 0xFFFF, "alias", off + delta, src_chunk, "ab" * 16)


def sample_mismatch(truncated=0) -> MismatchReport:
    recs = [alias_rec(0x0), alias_rec(0x3ffffff0), MismatchWindow(0x40000000, 0, 0xFFFF, "zero", 0, 0, "00" * 16),
            MismatchWindow(0x50000011 & ~15, 1, 1 << 1, "partial", 0, 0, "00" + "5a" + "00" * 14)]
    return MismatchReport(mismatch_bytes=0x20000000, mismatch_windows=0x8000000 * (1 + truncated), zero_windows=0x4000000,
                          first_offset=0, last_offset=0x7fffffff, va_base=0x7F00_0000_0000, seed=0xC0FFEE, located=1,
                          truncated=truncated, records=recs)


def report(bdf=SC.GPU_BDFS[0], mismatch=0, **kw):
    return ScrubReport(bdf, 0, 190 << 30, 191 << 30, 0, 1, 25, 25, 1, 52, 1, N.ERR_MISMATCH if mismatch else 0,
                       check="tagged", mismatch_bytes=mismatch, **kw)


def test_json_round_trip_and_clean_key_sets():
    clean = report()
    assert clean.mismatch is None and "mismatch" not in ScrubReport.__dataclass_fields__
    assert set(clean.as_json()) == set(ScrubReport.__dataclass_fields__)
    zero_only = ScrubReport(SC.GPU_BDFS[0], 0, 1, 1, 0, 1, 1, 1, 1, 1, 1, 0)
    assert set(zero_only.as_json()) == set(ScrubReport.__dataclass_fields__) - set(D.TAG_FIELDS)
    rep = report(mismatch=5)
    rep.mismatch = sample_mismatch()
    js = json.loads(json.dumps(rep.as_json()))
    assert set(js) - {"mismatch"} == set(clean.as_json()) and js["mismatch"]["records"][0]["kind"] == "alias"
    back = ScrubReport.from_json(js)
    assert back == rep and back.mismatch == rep.mismatch and back.dirt is None
    assert ScrubReport.from_json(clean.as_json()).mismatch is None
    assert MismatchReport.from_json(sample_mismatch(1).as_json()) == sample_mismatch(1)
    assert GpuError("x").mismatch is None


def test_summary_names_deltas_chunk_pairs_and_kinds():
    s = sample_mismatch().summary()
    assert "alias: +0x0..+0x3ffffff0 hold the tags of +0x40000000.. (delta 0x40000000, chunk 0 ← chunk 0" in s
    assert "zero: 1 records, chunks [0]" in s and "partial: 1 records, chunks [1]" in s
    assert "+0x50000010 chunk 1 mask 0002" in s and "67108864 of them all zero" in s
    assert "(records truncated)" in sample_mismatch(1).summary()
    two = MismatchReport(32, 2, 0, 0, 31, 0, 1, 1, 0, [alias_rec(0, 0x40, 0, 0), alias_rec(16, -0x10, 2, 1)])
    s2 = two.summary()
    assert "delta 0x40, chunk 0 ← chunk 0" in s2 and "delta -0x10, chunk 2 ← chunk 1" in s2


# ---------------------------------------------------------------------------------- manager
class FakeGpu:
    """Duck-typed device whose tagged scrub fails its check: GpuError with .mismatch."""

    def __init__(self, bdf, cc="off", mismatch=None):
        self.bdf, self.name = bdf, "fake"
        self.is_cc_query_supported = self.is_ppcie_query_supported = True
        self.cc, self.staged, self.pp = cc, cc, "off"
        self.mismatch = mismatch

    def is_gpu(self): return True
    def is_nvswitch(self): return False
    def query_cc_mode(self): return self.cc
    def set_cc_mode(self, m): self.staged = m
    def query_ppcie_mode(self): return self.pp
    def set_ppcie_mode(self, m): pass
    def reset_with_os(self): self.cc = self.staged
    def wait_for_boot(self): pass

    def scrub_and_verify(self, nbytes=0, check="zero"):
        if self.mismatch is None:
            return report(self.bdf)
        err = GpuError(f"scrub_and_verify on {self.bdf}: tagged scrub found bytes that did not hold their tag",
                       N.ERR_MISMATCH)
        err.mismatch = self.mismatch
        raise err


def manager_for(devs, monkeypatch, labels=None, **kw):
    import kubernetes
    from k8s_cc_manager_b200 import manager
    c = kubernetes.reset_cluster()
    c.add_node(SC.NODE, labels or {})
    monkeypatch.setenv("EVICT_OPERATOR_COMPONENTS", "false")
    source = (lambda: (devs, len(devs))) if devs is not None else None
    return manager.CCManager(SC.NODE, "on", True, device_source=source, scrub_check="tagged", **kw), c


def assert_mismatch_logged(mgr, c, caplog, bdf, mm):
    assert c.labels(SC.NODE).get("nvidia.com/cc.mode.state") == "failed"
    assert mgr.last_transition["scrub_mismatch"] == {bdf: mm}
    lines = [r.getMessage() for r in caplog.records if f"HBM tag mismatch on {bdf}: " in r.getMessage()]
    assert len(lines) == 1 and "delta 0x40000000, chunk 0 ← chunk 0" in lines[0]
    assert "scrub_dirt" not in mgr.last_transition


def test_per_gpu_fan_out_logs_and_keeps_the_report(monkeypatch, caplog):
    mm = sample_mismatch()
    devs = [FakeGpu(SC.GPU_BDFS[0]), FakeGpu(SC.GPU_BDFS[1], mismatch=mm)]
    mgr, c = manager_for(devs, monkeypatch)
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is False
    assert_mismatch_logged(mgr, c, caplog, SC.GPU_BDFS[1], mm)


def test_regate_logs_and_keeps_the_report(monkeypatch, caplog):
    mm = sample_mismatch()
    mgr, c = manager_for([FakeGpu(SC.GPU_BDFS[0], cc="on", mismatch=mm)], monkeypatch,
                         labels={"nvidia.com/cc.mode.state": "failed"})
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is False
    assert mgr.last_transition["regate"] is True
    assert_mismatch_logged(mgr, c, caplog, SC.GPU_BDFS[0], mm)


def _native_world(monkeypatch, n=2):
    build_native_world(SC.scenario("w", gpus_=SC.gpus(n), modes=[]))
    for k, v in dict(CCM_BACKEND="sim", CCM_SIM_GPUS=str(n), CCM_SIM_BIND_CUDA="0").items():
        monkeypatch.setenv(k, v)


def test_native_fan_out_logs_and_keeps_the_report(monkeypatch, caplog):
    from k8s_cc_manager_b200 import manager
    _native_world(monkeypatch)
    mm = sample_mismatch()

    def fake_many(devices, nbytes=0, check="zero", **kw):
        reps = [report(d.bdf) for d in devices]
        reps[1] = report(devices[1].bdf, mismatch=5)
        reps[1].mismatch = mm
        return reps, 1.0
    monkeypatch.setattr(manager._devices, "scrub_and_verify_many", fake_many)
    mgr, c = manager_for(None, monkeypatch)
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is False
    bdf = mgr.last_transition["scrub"][1].bdf
    assert_mismatch_logged(mgr, c, caplog, bdf, mm)
    assert any(f"HBM scrub failed on {bdf}: status=-13" in r.getMessage() for r in caplog.records)


def test_worker_process_report_carries_the_mismatch(monkeypatch, caplog):
    _native_world(monkeypatch)
    monkeypatch.setenv("CC_SCRUB_ISOLATION", "process")
    mm = sample_mismatch()
    captured = {}

    def fake_run(cmd, **kw):
        bdfs = [cmd[i + 1] for i, a in enumerate(cmd) if a == "--bdf"]
        assert cmd[cmd.index("--check") + 1] == "tagged"
        reps = [report(b).as_json() for b in bdfs]
        bad = report(bdfs[0], mismatch=5)
        bad.mismatch = mm
        reps[0] = bad.as_json()
        captured["bdf"] = bdfs[0]
        return subprocess.CompletedProcess(cmd, 3, json.dumps({"wall_ms": 1.0, "reports": reps}) + "\n", "")
    monkeypatch.setattr(subprocess, "run", fake_run)
    mgr, c = manager_for(None, monkeypatch)
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is False
    assert_mismatch_logged(mgr, c, caplog, captured["bdf"], mm)
    assert mgr.last_transition["scrub"][0].mismatch == mm and mgr.last_transition["scrub"][1].mismatch is None


def test_clean_gate_records_no_mismatch(monkeypatch):
    mgr, c = manager_for([FakeGpu(b) for b in SC.GPU_BDFS[:2]], monkeypatch)
    assert mgr.set_cc_mode("on") is True
    assert "scrub_mismatch" not in mgr.last_transition


# ---------------------------------------------------------------------------------- CLI and worker
def test_worker_prints_mismatch_only_when_there_is_one(monkeypatch, capsys):
    from k8s_cc_manager_b200 import scrub_worker
    bad = report("0000:01:00.0", mismatch=5)
    bad.mismatch = sample_mismatch()
    good = report("0000:02:00.0")

    class Dev:
        def __init__(self, bdf): self.bdf = bdf
        def is_gpu(self): return True
    monkeypatch.setattr(D, "find_gpus", lambda: ([Dev(good.bdf), Dev(bad.bdf)], 2))
    monkeypatch.setattr(D, "scrub_and_verify_many", lambda devs, n, check="zero": ([good, bad], 1.0))
    assert scrub_worker.main(["--bdf", good.bdf, "--bdf", bad.bdf, "--check", "tagged"]) == 3
    out = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    assert "mismatch" not in out["reports"][0] and out["reports"][1]["mismatch"]["records"][2]["kind"] == "zero"
    assert MismatchReport.from_json(out["reports"][1]["mismatch"]) == bad.mismatch


def test_cli_prints_mismatch_only_for_a_failed_tagged_check():
    src = (ROOT / "k8s_cc_manager_b200" / "csrc" / "ccm_scrub_cli.cpp").read_text()
    assert 'tagged && tags[i].mismatch_bytes != 0 && ccm_scrub_last_mismatch(ordinals[i], &m) == CCM_OK' in src
    keys = set(MismatchReport.__dataclass_fields__)
    rec_keys = set(MismatchWindow.__dataclass_fields__)
    printed = src[src.index("static void print_mismatch"):src.index("static int usage")]
    assert all(f'\\"{k}\\"' in printed for k in keys | rec_keys)
