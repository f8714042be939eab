"""The alias probe on the CPU: the oracle against a byte-level model of physical pages and a page table (and a per-page
window offset that misses the alias); the C ABI without a CUDA device (exports, layouts from a C99 compile, constants,
drill keys); ProbeReport in ScrubReport's and GpuError's JSON; the proxy, the worker and the CLI; and the manager knob
CC_SCRUB_ALIAS_PROBE."""
from __future__ import annotations

import ctypes as C
import inspect
import json
import logging
import re
import shutil
import subprocess
from pathlib import Path

import pytest

import probe_oracle as PO
import scenarios as SC
import tag_oracle as TO
import test_cover_proof as TC
import test_dirt_locate as TD
import test_tag_mismatch as TM
from k8s_cc_manager_b200 import _native as N
from k8s_cc_manager_b200 import devices as D
from k8s_cc_manager_b200.devices import GpuError, ProbeReport, ScrubReport

ROOT = Path(__file__).resolve().parents[1]
KiB, MiB = 1 << 10, 1 << 20
PG = 4096
BASE = (3 << 34) + (5 << 21)     # 16 GiB window 3: the hi32 half of the tag is not zero


# ---------------------------------------------------------------------------------- oracle against a byte-level model
def model(chunks, seed, alias=None, place=lambda vpage: 0, probe_mismatch=0, probe_dirt=0):
    """Physical 4 KiB pages behind a page table, every chunk's pages mapped in order (`alias` = (view2, view1, n0):
    the pages of [view2, view2 + n0) map the physical pages of [view1, view1 + n0)).  The probe's windows lie at
    page address + place(virtual page index) inside each chunk; P1, the drills, P2 and P3 run byte by byte, chunk by
    chunk.  Returns (P2 bytes, {window offset from BASE: mask}, P3 bytes)."""
    table, mem = {}, {}
    for a, n in chunks:
        for vp in range(a // PG, (a + n) // PG):
            table[vp] = len(mem)
            mem[len(mem)] = bytearray(PG)
    if alias is not None:
        view2, view1, n0 = alias
        for k in range(n0 // PG):
            table[view2 // PG + k] = table[view1 // PG + k]

    def at(x):
        return mem[table[x // PG]], x % PG

    wins = [[vp * PG + place(vp) for vp in range(a // PG, (a + n) // PG) if vp * PG + place(vp) + 32 <= a + n]
            for a, n in chunks]
    flat = [w for ws in wins for w in ws]
    for ws in wins:                                                     # P1
        for w in ws:
            for i, b in enumerate(TO.tag_bytes(seed, w, 32)):
                page, o = at(w + i)
                page[o] = int(b)
    for w in flat[:probe_mismatch]:
        page, o = at(w)
        page[o] ^= 0xA5
    p2, masks = 0, {}
    for ws in wins:                                                     # P2
        for w in ws:
            tags = TO.tag_bytes(seed, w, 32)
            for i in range(32):
                page, o = at(w + i)
                if page[o] != tags[i]:
                    p2 += 1
                    off = w + i - BASE
                    masks[off & ~15] = masks.get(off & ~15, 0) | 1 << (off & 15)
                page[o] = 0
    for w in flat[:probe_dirt]:
        page, o = at(w)
        page[o] ^= 0xA5
    p3 = sum(1 for ws in wins for w in ws for i in range(32) if at(w + i)[0][at(w + i)[1]])   # P3
    return p2, masks, p3


# chunk 0, then chunk 1 whose first N0 bytes are a second view of chunk 0 (as "scrub_alias" maps them), then a granule
N0 = 64 * KiB
CHUNKS = [(BASE, N0), (BASE + N0, 2 * N0), (BASE + 3 * N0, 8 * KiB)]
ALIAS = (BASE + N0, BASE, N0)


@pytest.mark.parametrize("alias", [None, ALIAS])
@pytest.mark.parametrize("drills", [(0, 0), (3, 0), (0, 5), (40, 40)])
def test_oracle_matches_the_byte_level_model(alias, drills):
    seed = 0x5EED1234
    want = PO.expected(CHUNKS, seed, BASE, alias=alias, probe_mismatch=drills[0], probe_dirt=drills[1])
    p2, masks, p3 = model(CHUNKS, seed, alias, probe_mismatch=drills[0], probe_dirt=drills[1])
    assert want["windows"] == len(PO.windows(CHUNKS)) == (N0 + 2 * N0 + 8 * KiB) // PG
    assert want["mismatch_bytes"] == p2 and want["reread_nonzero_bytes"] == p3
    assert {r["offset"]: r["mask"] for r in want["records"]} == masks
    assert sum(want["pages"].values()) == p2
    if alias is not None and drills[0] == 0:
        kinds = {r["offset"]: (r["kind"], r["source_offset"]) for r in want["records"]}
        for off, (kind, src) in kinds.items():
            if off < N0:   # the first view reads the second view's tags
                assert kind == "alias" and src == off + N0
            else:          # the second view reads what the first view's check left: zero
                assert N0 <= off < 2 * N0 and kind == "zero"
    elif alias is None:
        assert p2 == min(drills[0], want["windows"]) and p3 == min(drills[1], want["windows"])
        assert all(r["kind"] == "partial" for r in want["records"])


def test_a_window_placed_by_page_index_misses_the_alias():
    seed = 77
    assert model(CHUNKS, seed, ALIAS)[0] > 0
    # a window whose place depends on the virtual page index lands on another sector in the second view of the page
    p2, masks, _ = model(CHUNKS, seed, ALIAS, place=lambda vp: (vp % 127) * 32)
    assert p2 == 0 and masks == {}


def test_window_geometry():
    assert PO.chunk_windows(0, 32) == (0, 1) and PO.chunk_windows(0, 31) == (0, 0)
    assert PO.chunk_windows(1, 4096 + 30) == (4096, 0) and PO.chunk_windows(1, 4096 + 31) == (4096, 1)
    assert PO.chunk_windows(4096, 3 * 4096) == (4096, 3) and PO.chunk_windows(4095, 2) == (4096, 0)
    for a in (0, 1, 17, 4095, 4096, 8191):
        for n in (0, 31, 32, 4127, 4128, 3 * 4096 + 40):
            brute = [x for x in range(a, a + n) if x % PG == 0 and x + 32 <= a + n]
            w0, k = PO.chunk_windows(a, n)
            assert k == len(brute) and (k == 0 or w0 == brute[0])


# ---------------------------------------------------------------------------------- C ABI
ENTRY_POINTS = ("ccm_scrub_probe", "ccm_scrub_last_probe", "ccm_region_probe")


def test_entry_points_are_exported_and_refuse_what_they_must(native):
    lib = native.lib()
    nm = subprocess.run(["nm", "-D", "--defined-only", str(native.LIB_PATH)], capture_output=True, text=True,
                        check=True).stdout
    for fn in ENTRY_POINTS:
        assert fn in native.EXPORTED_SYMBOLS and re.search(rf" T {fn}$", nm, re.M), fn
    for ordinal in (-1, 1 << 12):
        assert lib.ccm_scrub_probe(ordinal, 1) == native.ERR_NO_CUDA
        rep = native.ProbeReport(probed=7)
        assert lib.ccm_scrub_last_probe(ordinal, C.byref(rep)) == native.ERR_NO_CUDA and rep.probed == 0
        assert lib.ccm_region_probe(ordinal, None, 0, 0, None, C.byref(rep), None) == native.ERR_NO_CUDA
    assert lib.ccm_scrub_last_probe(0, None) == native.ERR_INVALID
    assert lib.ccm_region_probe(0, None, 0, 0, None, None, None) == native.ERR_INVALID
    assert D.last_probe(-1) is None


def test_header_constants_and_text():
    header = (ROOT / "include" / "ccm.h").read_text()
    assert "#define CCM_PROBE_STRIDE 4096u" in header and "#define CCM_PROBE_WINDOW 32u" in header
    assert N.PROBE_STRIDE == PO.STRIDE == 4096 and N.PROBE_WINDOW == PO.WINDOW == 32
    assert "#define CCM_ABI_VERSION 2 " in header
    for fn in ENTRY_POINTS:
        assert re.search(rf"^int {fn}\(", header, re.M), fn
    assert '"probe_mismatch"' in header and '"probe_dirt"' in header
    # the mismatch report is no longer the tagged check's alone
    assert "a failed tagged check or alias probe" in header and "probed zero-gate call" in header
    assert "address fault with a stride below 4 KiB" in header


LAYOUT_C = r"""
#include <stddef.h>
#include <stdio.h>
#include "ccm.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu %zu %zu\n", sizeof(ccm_probe_report), offsetof(ccm_probe_report, mismatch_windows),
         offsetof(ccm_probe_report, reread_nonzero_bytes), offsetof(ccm_probe_report, seed),
         offsetof(ccm_probe_report, launches), offsetof(ccm_probe_report, va_base), offsetof(ccm_probe_report, ms_probe),
         offsetof(ccm_probe_report, probed));
  return 0;
}
"""


def test_struct_layout_matches_a_c99_compile(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "layout.c"
    src.write_text(LAYOUT_C)
    subprocess.run([cc, "-std=c99", "-Wall", "-Werror", "-I", str(ROOT / "include"), str(src), "-o",
                    str(tmp_path / "layout")], check=True)
    got = [int(x) for x in subprocess.run([str(tmp_path / "layout")], capture_output=True, text=True,
                                          check=True).stdout.split()]
    R = N.ProbeReport
    want = [C.sizeof(R), R.mismatch_windows.offset, R.reread_nonzero_bytes.offset, R.seed.offset, R.launches.offset,
            R.va_base.offset, R.ms_probe.offset, R.probed.offset]
    assert got == want == [80, 24, 32, 40, 44, 48, 56, 64]


def test_drill_keys_round_trip(native):
    lib = native.lib()
    assert lib.ccm_sim_topology(2, 0) == 0
    v = C.c_int64(-1)
    for key in (b"probe_mismatch", b"probe_dirt"):
        assert lib.ccm_sim_get(0, key, C.byref(v)) == 0 and v.value == 0
        assert lib.ccm_sim_set(0, key, 9) == 0 and lib.ccm_sim_get(0, key, C.byref(v)) == 0 and v.value == 9
        assert lib.ccm_sim_get(1, key, C.byref(v)) == 0 and v.value == 0
        assert lib.ccm_sim_set(0, key, -3) == 0 and lib.ccm_sim_get(0, key, C.byref(v)) == 0 and v.value == 0


def test_probe_kernels_are_not_listed_as_scrub_or_verify_kernels():
    """As the proving twins, their names do not end in `kernel`: the kernel lists of the existing tests do not take
    them, and tests/test_alias_probe_gpu.py (the region probe) launches all three."""
    src = (ROOT / "k8s_cc_manager_b200" / "csrc" / "scrub_kernels.cuh").read_text()
    names = re.findall(r"^(alias_probe_\w+)\(", src, re.M)
    assert names == ["alias_probe_fill_pass", "alias_probe_check_pass", "alias_probe_reread_pass"]
    assert not any(re.search(r"(?:scrub|verify)_\w*kernel<", n + "<") or n.endswith("kernel") for n in names)


# ---------------------------------------------------------------------------------- device API and JSON
def sample_probe(mismatch=0) -> ProbeReport:
    return ProbeReport(windows=20_000_000, bytes_probed=640_000_000, mismatch_bytes=mismatch,
                       mismatch_windows=2 * (mismatch // 31), reread_nonzero_bytes=0, seed=0xC0FFEE, launches=42,
                       va_base=0x7F0000000000, ms_probe=12.5, probed=1)


def test_json_carries_the_report_only_when_the_probe_ran():
    rep = TC.zero_report("0000:01:00.0")
    base = set(json.loads(json.dumps(rep.as_json())))
    assert rep.probe is None and "probe" not in ScrubReport.__dataclass_fields__ and "probe" not in base
    rep.probe = sample_probe()
    js = json.loads(json.dumps(rep.as_json()))
    assert set(js) == base | {"probe"}
    back = ScrubReport.from_json(js)
    assert back.probe == rep.probe and back.mismatch is None and back.cover is None
    assert ProbeReport.from_json(sample_probe(62).as_json()) == sample_probe(62)
    assert GpuError("x").probe is None
    native = N.ProbeReport(windows=3, bytes_probed=96, mismatch_bytes=5, mismatch_windows=1, reread_nonzero_bytes=2,
                           seed=9, launches=6, va_base=1 << 40, ms_probe=0.5, probed=1)
    assert ProbeReport.from_native(native) == ProbeReport(3, 96, 5, 1, 2, 9, 6, 1 << 40, 0.5, 1)


def test_summary():
    assert "every window held its tags and read back zero" in sample_probe().summary()
    line = sample_probe(62).summary()
    assert "62 bytes off their tags in 4 16-byte windows" in line and sample_probe().held and not sample_probe(62).held


def test_device_api_takes_probe_and_refuses_it_with_the_tagged_check():
    for fn in (D.NvidiaDevice.scrub_and_verify, D.ScrubbingProxy.scrub_and_verify, D.scrub_and_verify_many):
        assert inspect.signature(fn).parameters["probe"].default is False
    proxy = D.ScrubbingProxy(type("Foreign", (), {"bdf": "0000:01:00.0"})(), TC._Native())
    with pytest.raises(ValueError, match="probe=True is for check='zero'"):
        proxy.scrub_and_verify(0, check="tagged", probe=True)
    with pytest.raises(ValueError, match="probe=True is for check='zero'"):
        D.scrub_and_verify_many([], check="tagged", probe=True)


def test_proxy_passes_probe_only_when_it_is_set():
    native = TC._Native()
    proxy = D.ScrubbingProxy(type("Foreign", (), {"bdf": "0000:01:00.0"})(), native)
    proxy.scrub_and_verify(0)
    proxy.scrub_and_verify(0, residue=True, probe=True)
    proxy.scrub_and_verify(0, prove=True)
    assert native.calls[0] == {} and "probe" not in native.calls[2]
    assert native.calls[1]["probe"] is True and native.calls[1]["residue"] is True and native.calls[1]["prove"] is False


def test_a_device_without_cuda_fails_an_armed_call(native):
    lib = native.lib()
    assert lib.ccm_sim_topology(1, 0) == 0
    assert lib.ccm_sim_set(-1, b"cuda_ordinal", -1) == 0
    gpu = [d for d in D.find_gpus()[0] if d.is_gpu()][0]
    with pytest.raises(GpuError) as err:
        gpu.scrub_and_verify(probe=True)
    assert err.value.status == N.ERR_NO_CUDA and "alias probe" in str(err.value)
    reports, _ = D.scrub_and_verify_many([gpu], probe=True)
    assert reports[0].status == N.ERR_NO_CUDA and reports[0].probe is None


# ---------------------------------------------------------------------------------- CLI and worker
def test_cli_prints_the_keys_the_worker_prints():
    src = (ROOT / "k8s_cc_manager_b200" / "csrc" / "ccm_scrub_cli.cpp").read_text()
    body = src[src.index("static void print_probe"):src.index("int main(")]
    assert set(re.findall(r'\\"(\w+)\\":', body)) == {"probe"} | set(ProbeReport.__dataclass_fields__)
    assert 'else if (a == "--probe") probe = true;' in src
    assert "ccm_scrub_probe(ordinals[i], 1)" in src and "ccm_scrub_probe(o, 0)" in src


def test_cli_refuses_the_tagged_check_and_never_scrubs_a_gpu_it_cannot_arm():
    cli = ROOT / "k8s_cc_manager_b200" / "ccm-scrub"
    if not cli.exists():
        pytest.skip("ccm-scrub is not built")
    proc = subprocess.run([str(cli), "--backend", "sim", "--probe", "--check", "tagged", "--all"], capture_output=True,
                          text=True, timeout=60)
    assert proc.returncode == 2 and "--probe is for --check zero" in proc.stderr and proc.stdout == ""
    proc = subprocess.run([str(cli), "--backend", "sim", "--probe", "--all"], capture_output=True, text=True, timeout=60)
    assert proc.returncode == 3 and "cannot arm the alias probe" in proc.stderr and proc.stdout == ""


def test_worker_takes_probe_and_refuses_the_tagged_check(monkeypatch, capsys):
    from k8s_cc_manager_b200 import scrub_worker
    seen = []

    def fake_many(devs, n, check="zero", residue=False, triage=False, triage_hold_ms=D.TRIAGE_HOLD_MS,
                  mismatch_triage=False, prove=False, probe=False):
        seen.append(dict(check=check, residue=residue, triage=triage, prove=prove, probe=probe))
        rep = TC.zero_report(devs[0].bdf, 0 if held else N.ERR_MISMATCH)
        rep.probe = sample_probe(0 if held else 62) if probe else None
        return [rep], 1.0
    monkeypatch.setattr(D, "find_gpus", lambda: ([TC._Dev("0000:01:00.0")], 1))
    monkeypatch.setattr(D, "scrub_and_verify_many", fake_many)
    held = True
    assert scrub_worker.main(["--bdf", "0000:01:00.0", "--probe"]) == 0
    out = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    assert ProbeReport.from_json(out["reports"][0]["probe"]) == sample_probe()
    held = False
    assert scrub_worker.main(["--bdf", "0000:01:00.0", "--probe", "--residue", "--prove"]) == 3
    out = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    assert out["reports"][0]["status"] == N.ERR_MISMATCH and out["reports"][0]["probe"]["mismatch_bytes"] == 62
    assert scrub_worker.main(["--bdf", "0000:01:00.0"]) == 3
    assert "probe" not in json.loads(capsys.readouterr().out.strip().splitlines()[-1])["reports"][0]
    assert [s["probe"] for s in seen] == [True, True, False] and seen[1]["residue"] and seen[1]["prove"]
    with pytest.raises(SystemExit) as exc:
        scrub_worker.main(["--bdf", "0000:01:00.0", "--probe", "--check", "tagged"])
    assert exc.value.code == 2 and len(seen) == 3


# ---------------------------------------------------------------------------------- manager
class ProbeGpu(TM.FakeGpu):
    """A clean zero-gate device that takes `probe` and records what it was called with; can_probe False: an older
    device library; aliased: its probe finds a page mapped twice."""

    def __init__(self, bdf, can_probe=True, aliased=False):
        super().__init__(bdf)
        self.calls, self.aliased = [], aliased
        if can_probe:
            self.scrub_and_verify = self._scrub_probe

    def scrub_and_verify(self, nbytes=0, check="zero"):
        self.calls.append(("old", nbytes, {"check": check}))
        return TC.zero_report(self.bdf)

    def _scrub_probe(self, nbytes=0, check="zero", residue=False, triage=False, triage_hold_ms=100,
                     mismatch_triage=False, prove=False, probe=False):
        self.calls.append(("new", nbytes, dict(check=check, residue=residue, triage=triage, prove=prove, probe=probe)))
        if probe and self.aliased:
            err = GpuError(f"scrub_and_verify on {self.bdf}: HBM alias probe found bytes that did not hold their tag",
                           N.ERR_MISMATCH)
            err.probe = sample_probe(62)
            err.mismatch = TM.sample_mismatch()
            raise err
        rep = TC.zero_report(self.bdf)
        rep.probe = sample_probe() if probe else None
        rep.cover = TC.sample_cover(1) if prove else None
        return rep


def probe_lines(caplog):
    return [(r.levelno, r.getMessage()) for r in caplog.records if r.getMessage().startswith("HBM alias probe on ")]


@pytest.mark.parametrize("value,want", [(None, "off"), ("off", "off"), ("require", "require"), ("REQUIRE", "require")])
def test_setting_is_parsed(monkeypatch, value, want):
    if value is not None:
        monkeypatch.setenv("CC_SCRUB_ALIAS_PROBE", value)
    mgr, _ = TD.manager_for([ProbeGpu(SC.GPU_BDFS[0])], monkeypatch)
    assert mgr.scrub_alias_probe == want and mgr.alias_probe == (want == "require")


def test_other_values_and_the_tagged_check_are_refused_at_start_up(monkeypatch):
    from k8s_cc_manager_b200 import manager
    for bad in ("on", "1", "report", "true"):
        monkeypatch.setenv("CC_SCRUB_ALIAS_PROBE", bad)
        with pytest.raises(ValueError, match="CC_SCRUB_ALIAS_PROBE must be 'off' or 'require'"):
            TD.manager_for([ProbeGpu(SC.GPU_BDFS[0])], monkeypatch)
    monkeypatch.setenv("CC_SCRUB_ALIAS_PROBE", "require")
    monkeypatch.setenv("CC_SCRUB_CHECK", "tagged")
    with pytest.raises(ValueError, match="CC_SCRUB_CHECK=tagged already checks every probe window"):
        TD.manager_for([ProbeGpu(SC.GPU_BDFS[0])], monkeypatch)
    monkeypatch.delenv("CC_SCRUB_CHECK")
    monkeypatch.delenv("CC_SCRUB_ALIAS_PROBE")
    with pytest.raises(ValueError, match="already checks every probe window"):
        TD.manager_for([ProbeGpu(SC.GPU_BDFS[0])], monkeypatch, scrub_alias_probe="require", scrub_check="tagged")
    parser = manager.build_arg_parser()
    assert parser.parse_args(["--scrub-alias-probe", "require"]).scrub_alias_probe == "require"
    assert parser.parse_args([]).scrub_alias_probe is None
    with pytest.raises(SystemExit):
        parser.parse_args(["--scrub-alias-probe", "on"])


KNOB_SETS = [dict(), dict(scrub_residue="report"), dict(scrub_triage="report"), dict(scrub_proof="require"),
             dict(scrub_residue="report", scrub_triage="report", scrub_proof="require")]


@pytest.mark.parametrize("knobs", KNOB_SETS)
def test_per_gpu_gate_passes_probe_and_logs(monkeypatch, caplog, knobs):
    devs = [ProbeGpu(SC.GPU_BDFS[0]), ProbeGpu(SC.GPU_BDFS[1])]
    mgr, _ = TD.manager_for(devs, monkeypatch, scrub_alias_probe="require", **knobs)
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is True
    for d in devs:
        assert len(d.calls) == 1 and d.calls[0][0] == "new"
        kw = d.calls[0][2]
        assert kw["probe"] is True and kw["check"] == "zero" and kw["residue"] == ("scrub_residue" in knobs)
        assert kw["triage"] == ("scrub_triage" in knobs) and kw["prove"] == ("scrub_proof" in knobs)
    assert mgr.last_transition["scrub_probe"] == {d.bdf: sample_probe() for d in devs}
    assert sorted(probe_lines(caplog)) == sorted(
        (logging.INFO, f"HBM alias probe on {d.bdf}: {sample_probe().summary()}") for d in devs)


def test_off_takes_the_calls_it_always_took(monkeypatch, caplog):
    devs = [ProbeGpu(SC.GPU_BDFS[0])]
    mgr, _ = TD.manager_for(devs, monkeypatch)
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is True
    assert devs[0].calls[0][2]["probe"] is False
    assert "scrub_probe" not in mgr.last_transition and probe_lines(caplog) == []


def test_a_device_without_probe_fails_the_gate(monkeypatch, caplog):
    devs = [ProbeGpu(SC.GPU_BDFS[0]), ProbeGpu(SC.GPU_BDFS[1], can_probe=False)]
    mgr, c = TD.manager_for(devs, monkeypatch, scrub_alias_probe="require")
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is False
    assert TC.state(c) == "failed" and devs[1].calls == []   # never scrubbed without the probe in its place
    assert any(f"device {devs[1].bdf} cannot probe its HBM for pages mapped twice" in r.getMessage()
               for r in caplog.records)


def test_an_aliased_gpu_fails_the_transition_and_logs_the_probe_and_the_mismatch(monkeypatch, caplog):
    devs = [ProbeGpu(SC.GPU_BDFS[0]), ProbeGpu(SC.GPU_BDFS[1], aliased=True)]
    mgr, c = TD.manager_for(devs, monkeypatch, scrub_alias_probe="require")
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is False
    assert TC.state(c) == "failed"
    bad = devs[1].bdf
    assert mgr.last_transition["scrub_probe"][bad] == sample_probe(62)
    assert (logging.ERROR, f"HBM alias probe on {bad}: {sample_probe(62).summary()}") in probe_lines(caplog)
    assert mgr.last_transition["scrub_mismatch"][bad] == TM.sample_mismatch()
    assert any(r.getMessage().startswith(f"HBM tag mismatch on {bad}") for r in caplog.records)


@pytest.mark.parametrize("knobs", KNOB_SETS)
@pytest.mark.parametrize("held", [True, False])
def test_native_fan_out_passes_it(monkeypatch, caplog, knobs, held):
    from k8s_cc_manager_b200 import manager
    TC._native_world(monkeypatch)
    seen = {}

    def fake_many(devices, nbytes=0, check="zero", residue=False, triage=False, triage_hold_ms=D.TRIAGE_HOLD_MS,
                  mismatch_triage=False, prove=False, probe=False):
        seen.update(check=check, residue=residue, triage=triage, prove=prove, probe=probe)
        reps = []
        for d in devices:
            r = TC.zero_report(d.bdf, 0 if held else N.ERR_MISMATCH)
            r.probe = sample_probe(0 if held else 62)
            r.cover = TC.sample_cover(1) if prove else None
            reps.append(r)
        return reps, 1.0
    monkeypatch.setattr(manager._devices, "scrub_and_verify_many", fake_many)
    mgr, c = TD.manager_for(None, monkeypatch, scrub_alias_probe="require", **knobs)
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is held
    assert seen["probe"] is True and seen["check"] == "zero" and seen["prove"] == ("scrub_proof" in knobs)
    assert seen["residue"] == ("scrub_residue" in knobs) and seen["triage"] == ("scrub_triage" in knobs)
    assert len(mgr.last_transition["scrub_probe"]) == 2
    assert {lvl for lvl, _ in probe_lines(caplog)} == {logging.INFO if held else logging.ERROR}
    if not held:
        assert TC.state(c) == "failed"
        assert any("see the alias probe" in r.getMessage() for r in caplog.records)


def test_a_report_without_its_probe_fails_under_require(monkeypatch, caplog):
    from k8s_cc_manager_b200 import manager
    TC._native_world(monkeypatch)
    monkeypatch.setattr(manager._devices, "scrub_and_verify_many",
                        lambda devices, nbytes=0, probe=False, **kw: ([TC.zero_report(d.bdf) for d in devices], 1.0))
    mgr, c = TD.manager_for(None, monkeypatch, scrub_alias_probe="require")
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is False
    assert TC.state(c) == "failed" and any("carries no alias probe" in r.getMessage() for r in caplog.records)


@pytest.mark.parametrize("probe", ["off", "require"])
def test_worker_process_passes_it(monkeypatch, caplog, probe):
    TC._native_world(monkeypatch)
    monkeypatch.setenv("CC_SCRUB_ISOLATION", "process")
    monkeypatch.setenv("CC_SCRUB_ALIAS_PROBE", probe)
    monkeypatch.setenv("CC_SCRUB_TRIAGE", "report")
    cmds = []

    def fake_run(cmd, **kw):
        cmds.append(cmd)
        reps = []
        for b in [cmd[i + 1] for i, a in enumerate(cmd) if a == "--bdf"]:
            r = TC.zero_report(b)
            r.probe = sample_probe() if "--probe" in cmd else None
            reps.append(r.as_json())
        return subprocess.CompletedProcess(cmd, 0, json.dumps({"wall_ms": 1.0, "reports": reps}) + "\n", "")
    monkeypatch.setattr(subprocess, "run", fake_run)
    mgr, _ = TD.manager_for(None, monkeypatch)
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is True
    cmd = cmds[0]
    assert ("--probe" in cmd) == (probe == "require") and "--triage" in cmd and "--check" not in cmd
    if probe == "require":
        assert len(mgr.last_transition["scrub_probe"]) == 2 and len(probe_lines(caplog)) == 2
    else:
        assert "scrub_probe" not in mgr.last_transition


@pytest.mark.parametrize("refuses", ["prove", "probe"])
def test_fan_out_attaches_no_report_to_a_device_it_did_not_scrub(monkeypatch, refuses):
    """A device that refuses one of the two armings is not scrubbed, so no report of an earlier call is attached to it,
    and whatever was armed on it is disarmed."""
    calls = []

    def arm(name):
        def fn(ordinal, on):
            calls.append((name, ordinal, on))
            return N.ERR_CUDA if on and name == refuses and ordinal == 1 else N.OK
        return fn
    monkeypatch.setattr(D, "_arm_prove", arm("prove"))
    monkeypatch.setattr(D, "_arm_probe", arm("probe"))
    monkeypatch.setattr(D, "last_probe", lambda ordinal: sample_probe())   # a stale report of an earlier call
    monkeypatch.setattr(D, "last_cover", lambda ordinal: TC.sample_cover(1))
    ran = []

    def fake_native_many(n, idx, nbytes, res, wall):
        ran.extend(idx[i] for i in range(n))
        return 0
    lib = type("Lib", (), {"ccm_scrub_verify_many": staticmethod(fake_native_many)})()
    monkeypatch.setattr(N, "lib", lambda: lib)
    devs = [type("Dev", (), {"index": i, "cuda_ordinal": i, "bdf": f"0000:0{i}:00.0"})() for i in (0, 1)]
    reports, _ = D.scrub_and_verify_many(devs, prove=True, probe=True)
    assert ran == [0]
    assert reports[0].status == 0 and reports[0].probe == sample_probe() and reports[0].cover == TC.sample_cover(1)
    assert reports[1].status == N.ERR_CUDA and reports[1].probe is None and reports[1].cover is None
    armed = {(name, o) for name, o, on in calls if on and not (name == refuses and o == 1)}
    disarmed = {(name, o) for name, o, on in calls if not on}
    assert armed == disarmed
