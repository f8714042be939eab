"""The HBM health report on the CPU: the rule (csrc/ccm_health.h, compiled with g++ -Wall -Werror) against a Python
restatement over every combination of its inputs; the NVML mapping of ccm_hbm_snapshot and the drills layered on an
armed call's second snapshot, through a fake libnvidia-ml.so.1 built here and loaded by a child process; the struct
layouts against the ctypes mirror and the exports; HbmHealth's JSON, summary and GpuError attachment; and the manager's
CC_SCRUB_HBM_HEALTH policy with fake devices in both isolation modes."""
from __future__ import annotations

import ctypes as C
import itertools
import json
import logging
import os
import re
import shutil
import subprocess
from pathlib import Path

import pytest

import scenarios as SC
import test_cover_proof as TC
import test_dirt_locate as TD
from k8s_cc_manager_b200 import _native as N
from k8s_cc_manager_b200 import devices as D
from k8s_cc_manager_b200.devices import GpuError, HbmHealth, HbmSnapshot, ScrubReport

ROOT = Path(__file__).resolve().parents[1]
CSRC = ROOT / "k8s_cc_manager_b200" / "csrc"
INCLUDE = ROOT / "include"

Q = {name: 1 << k for k, name in enumerate(N.HBM_QUERIES)}
R = {name: 1 << k for k, name in enumerate(N.HBM_REASONS)}
NEEDED = Q["ecc_mode"] | Q["dram_uncorrected"] | Q["sram_uncorrected"] | Q["remapped_rows"]
UNFIT = R["dram_uncorrected"] | R["sram_uncorrected"] | R["remap_pending"] | R["remap_failure"] | R["ecc_off"]
COUNTERS = ("dram_corrected", "dram_uncorrected", "sram_corrected", "sram_uncorrected")


def gxx():
    cc = shutil.which("g++")
    if cc is None:
        pytest.skip("no g++")
    return cc


# ---------------------------------------------------------------------------------- the rule
RULE_MAIN = r"""
#include <cstdio>
#include "ccm_health.h"
int main() {
  const long long after_of[3] = {5, 7, 3};   // delta 0, positive, negative against 5
  for (int d0 = 0; d0 < 3; ++d0) for (int d1 = 0; d1 < 3; ++d1) for (int d2 = 0; d2 < 3; ++d2) for (int d3 = 0; d3 < 3; ++d3)
  for (int pending = 0; pending < 2; ++pending) for (int failure = 0; failure < 2; ++failure)
  for (int ecc = 0; ecc < 2; ++ecc) for (unsigned am = 0; am < 128; ++am) for (int same = 0; same < 2; ++same) {
    ccm_hbm_state b{}, a{};
    b.dram_corrected = b.dram_uncorrected = b.sram_corrected = b.sram_uncorrected = 5;
    a.dram_corrected = after_of[d0]; a.dram_uncorrected = after_of[d1];
    a.sram_corrected = after_of[d2]; a.sram_uncorrected = after_of[d3];
    b.ecc_current = a.ecc_current = ecc;
    a.remap_pending = pending; a.remap_failure = failure;
    a.available = am;
    b.available = same ? am : 127u;
    ccm_hbm_health h{};
    ccm_health::judge(b, a, &h);
    printf("%d %u %u %lld %lld %lld %lld\n", h.verdict, h.reasons, h.missing_queries, (long long)h.d_dram_corrected,
           (long long)h.d_dram_uncorrected, (long long)h.d_sram_corrected, (long long)h.d_sram_uncorrected);
  }
  return 0;
}
"""


def rule(deltas, pending, failure, ecc, before_mask, after_mask):
    """The rule of include/ccm.h (ccm_scrub_health), restated: (verdict, reasons, missing, deltas)."""
    both = before_mask & after_mask
    d = [x if both & Q[name] else 0 for x, name in zip(deltas, COUNTERS)]
    r = 0
    if any(both & Q[name] and x < 0 for x, name in zip(deltas, COUNTERS)):
        r |= R["went_down"]
    if d[1] > 0:
        r |= R["dram_uncorrected"]
    if d[3] > 0:
        r |= R["sram_uncorrected"]
    if after_mask & Q["remapped_rows"] and pending:
        r |= R["remap_pending"]
    if after_mask & Q["remapped_rows"] and failure:
        r |= R["remap_failure"]
    if after_mask & Q["ecc_mode"] and not ecc:
        r |= R["ecc_off"]
    missing = NEEDED & ~both
    if missing:
        r |= R["no_answer"]
    verdict = N.HBM_UNFIT if r & UNFIT else N.HBM_UNKNOWN if r else N.HBM_FIT
    return verdict, r, missing, d


def test_rule_matches_its_restatement_over_every_input(tmp_path):
    src = tmp_path / "rule.cpp"
    src.write_text(RULE_MAIN)
    subprocess.run([gxx(), "-std=c++17", "-Wall", "-Werror", "-O1", "-I", str(INCLUDE), "-I", str(CSRC), str(src), "-o",
                    str(tmp_path / "rule")], check=True)
    lines = subprocess.run([str(tmp_path / "rule")], capture_output=True, text=True, check=True).stdout.splitlines()
    combos = itertools.product(range(3), range(3), range(3), range(3), range(2), range(2), range(2), range(128), range(2))
    n = 0
    seen = set()
    for line, (d0, d1, d2, d3, pending, failure, ecc, am, same) in zip(lines, combos):
        deltas = [(0, 2, -2)[x] for x in (d0, d1, d2, d3)]
        want = rule(deltas, pending, failure, ecc, am if same else 127, am)
        got = [int(x) for x in line.split()]
        assert got == [want[0], want[1], want[2], *want[3]], (line, deltas, pending, failure, ecc, am, same)
        seen.add(want[0])
        n += 1
    assert n == len(lines) == 81 * 2 * 2 * 2 * 128 * 2
    assert seen == {N.HBM_FIT, N.HBM_UNFIT, N.HBM_UNKNOWN}


# ---------------------------------------------------------------------------------- NVML mapping through a fake library
FAKE_NVML = r"""
#include <stdlib.h>
#include <string.h>
/* FAKE_NVML: ecc_cur ecc_pend dram_c dram_u sram_c sram_u rows_c rows_u pending failure hist*5, then the return code of
   each of the 7 queries (ccm_hbm_query order), then that of the handle lookup. */
static long v[32];
static int loaded;
static void load(void) {
  if (loaded) return;
  loaded = 1;
  const char* s = getenv("FAKE_NVML");
  char* end;
  for (int i = 0; s && *s && i < 32; ++i, s = end) { v[i] = strtol(s, &end, 10); if (end == s) break; }
}
#define H ((void*)0x5eed)
int nvmlInit_v2(void) { load(); return 0; }
int nvmlDeviceGetHandleByPciBusId_v2(const char* bus, void** h) {
  load();
  if (v[22]) return (int)v[22];
  const char* want = getenv("FAKE_NVML_BUS");
  if (!want || strcmp(bus, want)) return 6;   /* NVML_ERROR_NOT_FOUND */
  *h = H;
  return 0;
}
int nvmlDeviceGetEccMode(void* h, int* cur, int* pend) {
  if (h != H) return 999;
  if (v[15]) return (int)v[15];
  *cur = (int)v[0]; *pend = (int)v[1];
  return 0;
}
int nvmlDeviceGetMemoryErrorCounter(void* h, int type, int counter, int loc, unsigned long long* c) {
  if (h != H || counter != 0 || type < 0 || type > 1 || (loc != 2 && loc != 7)) return 999;   /* volatile, DRAM/SRAM */
  int k = (loc == 2 ? 0 : 2) + type;
  if (v[16 + k]) return (int)v[16 + k];
  *c = (unsigned long long)v[2 + k];
  return 0;
}
int nvmlDeviceGetRemappedRows(void* h, unsigned* c, unsigned* u, unsigned* p, unsigned* f) {
  if (h != H) return 999;
  if (v[20]) return (int)v[20];
  *c = (unsigned)v[6]; *u = (unsigned)v[7]; *p = (unsigned)v[8]; *f = (unsigned)v[9];
  return 0;
}
int nvmlDeviceGetRowRemapperHistogram(void* h, unsigned* hist) {
  if (h != H) return 999;
  if (v[21]) return (int)v[21];
  for (int i = 0; i < 5; ++i) hist[i] = (unsigned)v[10 + i];
  return 0;
}
"""

DRIVER = r"""
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include "ccm_internal.h"
static void print(const char* tag, int rc, const ccm_hbm_state& s) {
  printf("{\"tag\": \"%s\", \"rc\": %d, \"dram_corrected\": %llu, \"dram_uncorrected\": %llu, \"sram_corrected\": %llu, "
         "\"sram_uncorrected\": %llu, \"ecc_current\": %u, \"ecc_pending\": %u, \"rows_corrected\": %u, "
         "\"rows_uncorrected\": %u, \"remap_pending\": %u, \"remap_failure\": %u, \"hist\": [%u, %u, %u, %u, %u], "
         "\"available\": %u, \"nvml_rc\": [%d, %d, %d, %d, %d, %d, %d]}\n", tag, rc,
         (unsigned long long)s.dram_corrected, (unsigned long long)s.dram_uncorrected,
         (unsigned long long)s.sram_corrected, (unsigned long long)s.sram_uncorrected, s.ecc_current, s.ecc_pending,
         s.rows_corrected, s.rows_uncorrected, s.remap_pending, s.remap_failure, s.hist_max, s.hist_high, s.hist_partial,
         s.hist_low, s.hist_none, s.available, s.nvml_rc[0], s.nvml_rc[1], s.nvml_rc[2], s.nvml_rc[3], s.nvml_rc[4],
         s.nvml_rc[5], s.nvml_rc[6]);
}
int main(int argc, char** argv) {
  if (ccm_init(CCM_BACKEND_SIM) != CCM_OK) return 2;
  ccm_hbm_state s;
  print("public", ccm_hbm_snapshot(0, &s), s);
  for (int i = 1; i < argc; ++i) {   // key=value: the drills
    char key[64];
    long long val = 0;
    if (sscanf(argv[i], "%63[^=]=%lld", key, &val) != 2 || ccm_sim_set(0, key, val) != CCM_OK) return 3;
  }
  print("public_after_drills", ccm_hbm_snapshot(0, &s), s);
  ccm::ScrubDrill d;
  if (ccm::sim_scrub_hook(0, &d) != CCM_OK) return 4;
  ccm_dev_info info;
  int n = 1;
  ccm_enumerate(&info, 1, &n);
  const int rc = ccm::hbm_snapshot_bus(info.bdf, &s);
  ccm_health::layer(&s, d.hbm);
  print("drilled", rc, s);
  return 0;
}
"""

VALUES = [1, 0, 11, 12, 13, 14, 21, 22, 1, 0, 640, 3, 2, 1, 0]   # ecc on, pending off; every other field distinct
BUS = "0000:1b:00.0"   # the sim backend's first GPU


@pytest.fixture(scope="module")
def fake_world(tmp_path_factory):
    cc, gcc = gxx(), shutil.which("gcc") or shutil.which("cc")
    if gcc is None:
        pytest.skip("no C compiler")
    d = tmp_path_factory.mktemp("nvml")
    (d / "fake_nvml.c").write_text(FAKE_NVML)
    subprocess.run([gcc, "-shared", "-fPIC", "-O1", "-Wall", "-Werror", str(d / "fake_nvml.c"), "-o",
                    str(d / "libnvidia-ml.so.1")], check=True)
    (d / "driver.cpp").write_text(DRIVER)
    subprocess.run([cc, "-std=c++17", "-O1", "-Wall", "-Werror", "-I", str(INCLUDE), "-I", str(CSRC),
                    str(CSRC / "ccm_core.cpp"), str(ROOT / "tests" / "native" / "no_cuda_stub.cpp"), str(d / "driver.cpp"),
                    "-o", str(d / "driver"), "-ldl", "-lpthread"], check=True)
    return d


def snapshot_child(world, values=VALUES, rcs=(0,) * 7, handle_rc=0, bus=BUS, drills=()):
    env = {k: v for k, v in os.environ.items() if not k.startswith("CCM_")}
    env.update(LD_LIBRARY_PATH=str(world), FAKE_NVML=" ".join(map(str, [*values, *rcs, handle_rc])),
               FAKE_NVML_BUS=bus, CCM_BACKEND="sim", CCM_SIM_GPUS="1", CCM_SIM_BIND_CUDA="0")
    out = subprocess.run([str(world / "driver"), *[f"{k}={v}" for k, v in drills]], capture_output=True, text=True,
                         env=env, timeout=60)
    assert out.returncode == 0, out.stderr
    return {d["tag"]: d for d in map(json.loads, out.stdout.splitlines())}


def expect_fields(d, values=VALUES):
    return dict(ecc_current=values[0], ecc_pending=values[1], dram_corrected=values[2], dram_uncorrected=values[3],
                sram_corrected=values[4], sram_uncorrected=values[5], rows_corrected=values[6],
                rows_uncorrected=values[7], remap_pending=values[8], remap_failure=values[9], hist=values[10:15])


def test_every_field_comes_from_its_query(fake_world):
    got = snapshot_child(fake_world)["public"]
    assert got["rc"] == N.OK and got["available"] == 127 and got["nvml_rc"] == [0] * 7
    assert {k: got[k] for k in expect_fields(got)} == expect_fields(got)


# the fields each query fills (ccm_hbm_query order)
QUERY_FIELDS = {0: ("ecc_current", "ecc_pending"), 1: ("dram_corrected",), 2: ("dram_uncorrected",),
                3: ("sram_corrected",), 4: ("sram_uncorrected",),
                5: ("rows_corrected", "rows_uncorrected", "remap_pending", "remap_failure"), 6: ("hist",)}


@pytest.mark.parametrize("k", range(7))
@pytest.mark.parametrize("code", [3, 15])   # NVML_ERROR_NOT_SUPPORTED, and another error (GPU_IS_LOST)
def test_a_query_that_does_not_answer_leaves_its_bit_clear(fake_world, k, code):
    rcs = [0] * 7
    rcs[k] = code
    got = snapshot_child(fake_world, rcs=rcs)["public"]
    assert got["rc"] == (N.OK if code == 3 else N.ERR_IO)   # NOT_SUPPORTED is not an error of the call
    assert got["available"] == 127 & ~(1 << k) and got["nvml_rc"] == rcs
    want = expect_fields(got)
    for f in QUERY_FIELDS[k]:
        want[f] = [0] * 5 if f == "hist" else 0
    assert {f: got[f] for f in want} == want


def test_no_device_at_the_address_answers_nothing(fake_world):
    got = snapshot_child(fake_world, bus="0000:99:00.0")["public"]
    assert got["rc"] == N.ERR_UNSUPPORTED and got["available"] == 0 and got["nvml_rc"] == [3] * 7
    assert snapshot_child(fake_world, handle_rc=999)["public"]["available"] == 0


DRILL_CASES = [
    (dict(hbm_uncorrected=3), dict(dram_uncorrected=VALUES[3] + 3)),
    (dict(hbm_corrected=5), dict(dram_corrected=VALUES[2] + 5)),
    (dict(hbm_remap_pending=1), dict(remap_pending=1)),
    (dict(hbm_remap_failure=1), dict(remap_failure=1)),
    (dict(hbm_uncorrected=2, hbm_remap_pending=1, hbm_remap_failure=1),
     dict(dram_uncorrected=VALUES[3] + 2, remap_pending=1, remap_failure=1)),
]


@pytest.mark.parametrize("drills,changed", DRILL_CASES)
def test_drills_layer_on_the_armed_snapshot_only(fake_world, drills, changed):
    got = snapshot_child(fake_world, drills=drills.items())
    assert got["public"] == {**got["public_after_drills"], "tag": "public"}   # a plain snapshot is never drilled
    want = {**expect_fields(got["drilled"]), **changed}
    assert {f: got["drilled"][f] for f in want} == want and got["drilled"]["available"] == 127


@pytest.mark.parametrize("mask", [1 << k for k in range(7)] + [0x24, 0x7F])
def test_unavailable_drill_clears_what_it_names_and_wins_over_the_others(fake_world, mask):
    drills = dict(hbm_unavailable=mask, hbm_uncorrected=4, hbm_remap_pending=1)
    got = snapshot_child(fake_world, drills=drills.items())["drilled"]
    assert got["available"] == 127 & ~mask
    assert got["nvml_rc"] == [3 if mask >> k & 1 else 0 for k in range(7)]
    want = {**expect_fields(got), "dram_uncorrected": VALUES[3] + 4, "remap_pending": 1}
    for k in range(7):
        if mask >> k & 1:
            for f in QUERY_FIELDS[k]:
                want[f] = [0] * 5 if f == "hist" else 0
    assert {f: got[f] for f in want} == want


def test_only_read_only_nvml_entry_points_are_resolved():
    src = (CSRC / "ccm_core.cpp").read_text()
    names = set(re.findall(r'"(nvml\w+)"', src))
    assert names == {"nvmlInit_v2", "nvmlSystemGetConfComputeState", "nvmlDeviceGetHandleByPciBusId_v2",
                     "nvmlDeviceGetEccMode", "nvmlDeviceGetMemoryErrorCounter", "nvmlDeviceGetRemappedRows",
                     "nvmlDeviceGetRowRemapperHistogram"}
    assert src.count('dlopen("libnvidia-ml.so.1"') == 1   # one loader


# ---------------------------------------------------------------------------------- ABI
LAYOUT = r"""
#include <stddef.h>
#include <stdio.h>
#include "ccm.h"
#define S(f) printf("%zu ", offsetof(ccm_hbm_state, f))
#define H(f) printf("%zu ", offsetof(ccm_hbm_health, f))
int main(void) {
  printf("%zu %zu ", sizeof(ccm_hbm_state), sizeof(ccm_hbm_health));
  S(dram_corrected); S(dram_uncorrected); S(sram_corrected); S(sram_uncorrected); S(ecc_current); S(ecc_pending);
  S(rows_corrected); S(rows_uncorrected); S(remap_pending); S(remap_failure); S(hist_max); S(hist_high);
  S(hist_partial); S(hist_low); S(hist_none); S(available); S(nvml_rc); S(reserved); S(ms_query);
  H(before); H(after); H(d_dram_corrected); H(d_dram_uncorrected); H(d_sram_corrected); H(d_sram_uncorrected);
  H(ms_health); H(mode); H(verdict); H(reasons); H(missing_queries);
  printf("%d %d\n", (int)CCM_ERR_HBM_HEALTH, (int)CCM_HBM_QUERIES);
  return 0;
}
"""


def test_struct_layouts_match_a_c99_compile(tmp_path):
    cc = shutil.which("gcc") or shutil.which("cc")
    if cc is None:
        pytest.skip("no C compiler")
    (tmp_path / "layout.c").write_text(LAYOUT)
    subprocess.run([cc, "-std=c99", "-Wall", "-Werror", "-I", str(INCLUDE), str(tmp_path / "layout.c"), "-o",
                    str(tmp_path / "layout")], check=True)
    got = [int(x) for x in subprocess.run([str(tmp_path / "layout")], capture_output=True, text=True,
                                          check=True).stdout.split()]
    want = [C.sizeof(N.HbmState), C.sizeof(N.HbmHealth)]
    want += [getattr(N.HbmState, f).offset for f, _ in N.HbmState._fields_]
    want += [getattr(N.HbmHealth, f).offset for f, _ in N.HbmHealth._fields_]
    assert got == want + [N.ERR_HBM_HEALTH, len(N.HBM_QUERIES)]


def test_entry_points_are_exported_and_refuse_what_they_must(native):
    nm = subprocess.run(["nm", "-D", "--defined-only", str(N.LIB_PATH)], capture_output=True, text=True,
                        check=True).stdout
    for fn in ("ccm_hbm_snapshot", "ccm_scrub_health", "ccm_scrub_last_health"):
        assert re.search(rf" T {fn}$", nm, re.M), fn
    lib = N.lib()
    assert lib.ccm_hbm_snapshot(0, None) == N.ERR_INVALID
    assert lib.ccm_hbm_snapshot(1 << 20, C.byref(N.HbmState())) == N.ERR_NO_DEVICE
    assert lib.ccm_scrub_health(0, 3) == N.ERR_INVALID and lib.ccm_scrub_health(0, -1) == N.ERR_INVALID
    assert lib.ccm_scrub_health(1 << 20, 1) == N.ERR_NO_CUDA
    assert lib.ccm_scrub_last_health(1 << 20, C.byref(N.HbmHealth())) == N.ERR_NO_CUDA
    assert N.strerror(N.ERR_HBM_HEALTH).startswith("the GPU's HBM ECC or row-remapping state")


def test_drill_keys_round_trip_and_refuse_what_they_must(native, monkeypatch):
    lib = N.lib()
    for key, value in (("hbm_uncorrected", 7), ("hbm_corrected", 9), ("hbm_remap_pending", 1),
                       ("hbm_remap_failure", 1), ("hbm_unavailable", 0x7F)):
        assert lib.ccm_sim_set(0, key.encode(), value) == N.OK
        got = C.c_int64()
        assert lib.ccm_sim_get(0, key.encode(), C.byref(got)) == N.OK and got.value == value
        assert lib.ccm_sim_set(0, key.encode(), 0) == N.OK
    if N.lib().ccm_backend_in_use() != N.BACKENDS["sysfs"]:
        assert lib.ccm_sim_set(0, b"hbm_unavailable", 0x80) == N.ERR_INVALID


# ---------------------------------------------------------------------------------- Python
def snap(**kw):
    base = dict(dram_corrected=0, dram_uncorrected=0, sram_corrected=0, sram_uncorrected=0, ecc_current=1, ecc_pending=1,
                rows_corrected=0, rows_uncorrected=0, remap_pending=0, remap_failure=0, hist_max=640, hist_high=0,
                hist_partial=0, hist_low=0, hist_none=0, available=127, nvml_rc=[0] * 7, ms_query=0.05)
    return HbmSnapshot(**{**base, **kw})


def health(after=None, before=None, verdict=N.HBM_FIT, reasons=(), missing=(), mode=2, **deltas):
    d = dict(d_dram_corrected=0, d_dram_uncorrected=0, d_sram_corrected=0, d_sram_uncorrected=0)
    d.update(deltas)
    return HbmHealth(before or snap(), after or snap(), **d, ms_health=0.1, mode=mode, verdict=verdict,
                     reasons=list(reasons), missing_queries=list(missing))


FIT_LINE = "ECC on; DRAM corrected +0, uncorrected +0 during the gate; rows remapped 0/0, none pending, no failure"


def test_from_native_json_and_summary():
    h = N.HbmHealth()
    for s in (h.before, h.after):
        s.available, s.ecc_current, s.hist_max = 127, 1, 640
    h.after.dram_uncorrected, h.d_dram_uncorrected = 2, 2
    h.after.remap_pending = 1
    h.mode, h.verdict = 2, N.HBM_UNFIT
    h.reasons = R["dram_uncorrected"] | R["remap_pending"]
    rep = HbmHealth.from_native(h)
    assert rep.reasons == ["dram_uncorrected", "remap_pending"] and rep.missing_queries == [] and not rep.fit
    assert HbmHealth.from_json(json.loads(json.dumps(rep.as_json()))) == rep
    assert rep.summary() == ("ECC on; DRAM corrected +0, uncorrected +2 during the gate; rows remapped 0/0, remap "
                             "pending, no failure; UNFIT: uncorrected DRAM errors +2 during the gate; a row remap is "
                             "pending: the GPU must be reset before release")
    assert health().summary() == FIT_LINE


def test_summary_names_every_reason():
    h = health(after=snap(ecc_current=0, remap_failure=1, rows_uncorrected=3, hist_none=1,
                          available=127 & ~Q["sram_uncorrected"], nvml_rc=[0, 0, 0, 0, 3, 0, 0]),
               verdict=N.HBM_UNFIT, reasons=("remap_failure", "ecc_off", "no_answer", "went_down"),
               missing=("sram_uncorrected",), d_dram_corrected=-1)
    line = h.summary()
    assert line.startswith("ECC off; DRAM corrected -1, uncorrected +0 during the gate; rows remapped 0/3")
    for part in ("UNFIT: a row remap failed (3 rows remapped for uncorrected errors, 1 banks without spare rows): the GPU "
                 "should go to RMA", "ECC is off", "NVML did not answer sram_uncorrected (3)",
                 "an error counter went down between the snapshots"):
        assert part in line, part
    unknown = health(after=snap(available=0, nvml_rc=[3] * 7), verdict=N.HBM_UNKNOWN, reasons=("no_answer",),
                     missing=("ecc_mode", "dram_uncorrected", "sram_uncorrected", "remapped_rows"))
    assert unknown.summary().startswith("ECC unknown; DRAM corrected ?, uncorrected ? during the gate; row remapping "
                                        "unknown; UNKNOWN: NVML did not answer ecc_mode (3)")


def test_report_json_carries_hbm_health_only_when_attached():
    rep = TC.zero_report("0000:01:00.0")
    assert "hbm_health" not in rep.as_json() and "health" not in rep.as_json()
    rep.health = health()
    d = rep.as_json()
    assert d["hbm_health"] == health().as_json() and "health" not in d
    back = ScrubReport.from_json(json.loads(json.dumps(d)))
    assert back.health == health() and back.as_json() == d


def test_gpu_error_carries_the_report(native, monkeypatch):
    """A failed armed call raises GpuError with `.health` attached; the arming is undone whatever happened."""
    TC._native_world(monkeypatch, n=1)
    D.select_backend("sim")
    armed = []
    monkeypatch.setattr(D, "_arm_health", lambda o, mode: armed.append(mode) or N.OK)
    monkeypatch.setattr(D, "last_health", lambda o: health(verdict=N.HBM_UNFIT, reasons=("remap_pending",)))
    gpu = D.find_gpus()[0][0]
    monkeypatch.setattr(gpu, "cuda_ordinal", 0)
    with pytest.raises(GpuError) as err:
        gpu.scrub_and_verify(health="require")
    assert err.value.health == health(verdict=N.HBM_UNFIT, reasons=("remap_pending",)) and armed == [2, 0]
    assert GpuError("x").health is None
    with pytest.raises(ValueError):
        gpu.scrub_and_verify(health="maybe")


def test_missing_report_under_require_is_a_failed_call(native, monkeypatch):
    class Lib:
        def ccm_scrub_verify_many(self, n, idx, nbytes, res, wall):
            for i in range(n):
                res[i].status = N.OK
                res[i].bytes_scrubbed = 1 << 30
            return N.OK
    TC._native_world(monkeypatch, n=2)
    D.select_backend("sim")
    devs = D.find_gpus()[0]
    monkeypatch.setattr(D, "_arm_health", lambda o, mode: N.OK)
    monkeypatch.setattr(D, "last_health", lambda o: None)
    real = N.lib()
    monkeypatch.setattr(N, "lib", lambda: Lib())
    try:
        reps, _ = D.scrub_and_verify_many(devs, health="require")
        assert [r.status for r in reps] == [N.ERR_HBM_HEALTH] * 2 and all(r.health is None for r in reps)
        reps, _ = D.scrub_and_verify_many(devs, health="report")
        assert [r.status for r in reps] == [N.OK] * 2
    finally:
        monkeypatch.setattr(N, "lib", lambda: real)


def test_worker_and_cli_take_health(monkeypatch, capsys):
    from k8s_cc_manager_b200 import scrub_worker
    seen = []

    def fake_many(devs, n, check="zero", residue=False, triage=False, triage_hold_ms=D.TRIAGE_HOLD_MS,
                  mismatch_triage=False, prove=False, probe=False, health="off"):
        seen.append(health)
        rep = TC.zero_report(devs[0].bdf)
        rep.health = globals()["health"]() if health != "off" else None
        return [rep], 1.0
    monkeypatch.setattr(D, "find_gpus", lambda: ([TD.FakeGpu("0000:01:00.0")], 1))
    monkeypatch.setattr(D, "scrub_and_verify_many", fake_many)
    assert scrub_worker.main(["--bdf", "0000:01:00.0"]) == 0
    assert "hbm_health" not in json.loads(capsys.readouterr().out)["reports"][0]
    assert scrub_worker.main(["--bdf", "0000:01:00.0", "--health", "require"]) == 0
    assert json.loads(capsys.readouterr().out)["reports"][0]["hbm_health"] == health().as_json()
    assert seen == ["off", "require"]
    src = (CSRC / "ccm_scrub_cli.cpp").read_text()
    body = src[src.index("static void print_snapshot"):src.index("static void print_triage")]
    printed = set(re.findall(r'\\"(\w+)\\"', body))
    assert set(HbmHealth.__dataclass_fields__) | set(HbmSnapshot.__dataclass_fields__) | {"hbm_health", "%s"} >= printed
    assert set(HbmHealth.__dataclass_fields__) - {"before", "after", "reasons", "missing_queries"} <= printed
    assert set(HbmSnapshot.__dataclass_fields__) - {"nvml_rc"} <= printed | {"nvml_rc"}
    assert list(N.HBM_QUERIES) == re.findall(r'"(\w+)"', body[body.index("kQueries"):body.index("kReasons")])
    assert list(N.HBM_REASONS) == re.findall(r'"(\w+)"', body[body.index("kReasons"):body.index("printf(\", \\\"hbm")])


# ---------------------------------------------------------------------------------- manager
class HealthGpu(TD.FakeGpu):
    """A clean device that takes `health`; its report is `report` (None: a library that attaches none).  An unfit or
    unknown report under require fails the call with ERR_HBM_HEALTH, as NvidiaDevice.scrub_and_verify does."""

    def __init__(self, bdf, report="fit"):
        super().__init__(bdf)
        self.report, self.calls = report, []

    def scrub_and_verify(self, nbytes=0, check="zero", health="off"):
        self.calls.append(health)
        rep = TC.zero_report(self.bdf)
        rep.check = check
        rep.health = None if health == "off" or self.report is None else REPORTS[self.report](health)
        if health == "require" and rep.health is not None and not rep.health.fit:
            err = GpuError(f"scrub_and_verify on {self.bdf}: {N.strerror(N.ERR_HBM_HEALTH)}", N.ERR_HBM_HEALTH)
            err.health = rep.health
            raise err
        return rep


REPORTS = {
    "fit": lambda mode: health(mode=N.HBM_HEALTH_MODES[mode]),
    "uncorrected": lambda mode: health(after=snap(dram_uncorrected=1), verdict=N.HBM_UNFIT, reasons=("dram_uncorrected",),
                                       mode=N.HBM_HEALTH_MODES[mode], d_dram_uncorrected=1),
    "pending": lambda mode: health(after=snap(remap_pending=1), verdict=N.HBM_UNFIT, reasons=("remap_pending",),
                                   mode=N.HBM_HEALTH_MODES[mode]),
    "failure": lambda mode: health(after=snap(remap_failure=1), verdict=N.HBM_UNFIT, reasons=("remap_failure",),
                                   mode=N.HBM_HEALTH_MODES[mode]),
    "ecc_off": lambda mode: health(after=snap(ecc_current=0), verdict=N.HBM_UNFIT, reasons=("ecc_off",),
                                   mode=N.HBM_HEALTH_MODES[mode]),
    "no_answer": lambda mode: health(after=snap(available=127 & ~Q["remapped_rows"], nvml_rc=[0, 0, 0, 0, 0, 3, 0]),
                                     verdict=N.HBM_UNKNOWN, reasons=("no_answer",), missing=("remapped_rows",),
                                     mode=N.HBM_HEALTH_MODES[mode]),
}
REASON_TEXT = {"uncorrected": "uncorrected DRAM errors +1 during the gate",
               "pending": "the GPU must be reset before release", "failure": "the GPU should go to RMA",
               "ecc_off": "ECC is off", "no_answer": "NVML did not answer remapped_rows (3)"}


def health_lines(caplog):
    return [(r.levelno, r.getMessage()) for r in caplog.records if r.getMessage().startswith("HBM health on ")]


@pytest.mark.parametrize("value,want", [(None, "off"), ("off", "off"), ("report", "report"), ("REQUIRE", "require")])
def test_setting_is_parsed(monkeypatch, value, want):
    if value is not None:
        monkeypatch.setenv("CC_SCRUB_HBM_HEALTH", value)
    mgr, _ = TD.manager_for([HealthGpu(SC.GPU_BDFS[0])], monkeypatch)
    assert mgr.scrub_hbm_health == want and mgr.hbm_health_required == (want == "require")


def test_other_values_are_refused_at_start_up(monkeypatch):
    monkeypatch.setenv("CC_SCRUB_HBM_HEALTH", "on")
    with pytest.raises(ValueError, match="CC_SCRUB_HBM_HEALTH"):
        TD.manager_for([HealthGpu(SC.GPU_BDFS[0])], monkeypatch)
    from k8s_cc_manager_b200 import manager
    assert manager.build_arg_parser().parse_args(["--scrub-hbm-health", "require"]).scrub_hbm_health == "require"


def test_off_asks_for_nothing(monkeypatch, caplog):
    devs = [HealthGpu(b) for b in SC.GPU_BDFS[:2]]
    mgr, c = TD.manager_for(devs, monkeypatch)
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is True
    assert [d.calls for d in devs] == [["off"], ["off"]]   # called without `health`
    assert "scrub_hbm_health" not in mgr.last_transition and health_lines(caplog) == []


@pytest.mark.parametrize("kind", ["fit", "uncorrected", "pending"])
def test_report_logs_one_line_per_gpu_and_never_fails(monkeypatch, caplog, kind):
    devs = [HealthGpu(SC.GPU_BDFS[0]), HealthGpu(SC.GPU_BDFS[1], report=kind)]
    mgr, c = TD.manager_for(devs, monkeypatch, scrub_hbm_health="report")
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is True
    assert [d.calls for d in devs] == [["report"], ["report"]]
    assert mgr.last_transition["scrub_hbm_health"] == {devs[0].bdf: REPORTS["fit"]("report"),
                                                       devs[1].bdf: REPORTS[kind]("report")}
    lines = health_lines(caplog)
    assert (logging.INFO, f"HBM health on {devs[0].bdf}: {FIT_LINE}") in lines and len(lines) == 2
    assert (logging.INFO if kind == "fit" else logging.WARNING,
            f"HBM health on {devs[1].bdf}: {REPORTS[kind]('report').summary()}") in lines


@pytest.mark.parametrize("kind", sorted(REASON_TEXT))
def test_require_fails_an_unfit_or_unknown_gpu_and_says_why(monkeypatch, caplog, kind):
    devs = [HealthGpu(SC.GPU_BDFS[0]), HealthGpu(SC.GPU_BDFS[1], report=kind)]
    mgr, c = TD.manager_for(devs, monkeypatch, scrub_hbm_health="require")
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is False
    assert TC.state(c) == "failed"
    lines = health_lines(caplog)
    bad = [m for lvl, m in lines if lvl == logging.ERROR]
    assert len(bad) == 1 and bad[0].startswith(f"HBM health on {devs[1].bdf}: ") and REASON_TEXT[kind] in bad[0]


def test_require_passes_fit_gpus_and_fails_a_missing_report(monkeypatch, caplog):
    devs = [HealthGpu(b) for b in SC.GPU_BDFS[:2]]
    mgr, c = TD.manager_for(devs, monkeypatch, scrub_hbm_health="require")
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is True
    assert {lvl for lvl, _ in health_lines(caplog)} == {logging.INFO} and len(health_lines(caplog)) == 2
    devs = [HealthGpu(SC.GPU_BDFS[0]), HealthGpu(SC.GPU_BDFS[1], report=None)]
    mgr, c = TD.manager_for(devs, monkeypatch, scrub_hbm_health="require")
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is False
    assert TC.state(c) == "failed"
    assert any("carries no HBM health report" in r.getMessage() for r in caplog.records)


def test_a_device_without_health_fails_require_and_warns_under_report(monkeypatch, caplog):
    devs = [TD.FakeGpu(SC.GPU_BDFS[0])]
    mgr, c = TD.manager_for(devs, monkeypatch, scrub_hbm_health="require")
    assert mgr.set_cc_mode("on") is False and TC.state(c) == "failed"
    mgr, c = TD.manager_for([TD.FakeGpu(SC.GPU_BDFS[0])], monkeypatch, scrub_hbm_health="report")
    with caplog.at_level(logging.WARNING, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is True
    assert any("cannot report its HBM health" in r.getMessage() for r in caplog.records)


@pytest.mark.parametrize("mode,kind,ok", [("report", "fit", True), ("report", "failure", True),
                                          ("require", "fit", True), ("require", "failure", False),
                                          ("require", "no_answer", False), ("require", None, False)])
def test_worker_process_passes_it(monkeypatch, caplog, mode, kind, ok):
    TC._native_world(monkeypatch)
    monkeypatch.setenv("CC_SCRUB_ISOLATION", "process")
    monkeypatch.setenv("CC_SCRUB_HBM_HEALTH", mode)
    cmds = []

    def fake_run(cmd, **kw):
        cmds.append(cmd)
        reps = []
        for i, b in enumerate(cmd[j + 1] for j, a in enumerate(cmd) if a == "--bdf"):
            h = REPORTS["fit" if i == 0 else kind](mode) if (i == 0 or kind is not None) else None
            r = TC.zero_report(b, N.ERR_HBM_HEALTH if mode == "require" and (h is None or not h.fit) else 0)
            r.health = h
            reps.append(r.as_json())
        return subprocess.CompletedProcess(cmd, 0 if ok else 3, json.dumps({"wall_ms": 1.0, "reports": reps}) + "\n", "")
    monkeypatch.setattr(subprocess, "run", fake_run)
    mgr, c = TD.manager_for(None, monkeypatch)
    with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
        assert mgr.set_cc_mode("on") is ok
    assert cmds[0][cmds[0].index("--health") + 1] == mode
    assert len(mgr.last_transition["scrub_hbm_health"]) == (2 if kind is not None else 1)
    if not ok:
        assert TC.state(c) == "failed"
