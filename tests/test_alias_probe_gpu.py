"""The alias probe on one H100: the region probe against the oracle at its edges (guard bytes untouched, windows zero
afterwards); clean armed calls leave what unarmed calls leave and launch 3 kernels more per chunk, on every mapping
path; scrub_alias in all four modes fails armed with the oracle's exact counts, records and pages, and passes unarmed;
the probe's drills, the triage of probe_dirt, and the dirt drills that keep the probe from running; the rate bar
against a same-run tag check; and the manager end to end.  The product calls run in a child process
(tests/probe_calls.py), once with CCM_PDL=1 and once with CCM_PDL=0."""
from __future__ import annotations

import contextlib
import ctypes as C
import json
import logging
import os
import statistics
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "tests"))
sys.path.insert(0, str(ROOT / "oracle"))
import probe_oracle as PO  # noqa: E402
import product_gate_calls as PGC  # noqa: E402
import product_plan as PP  # noqa: E402
import region_cover_calls as RCC  # noqa: E402
import report_cover_oracle as RO  # noqa: E402
import scenarios as SC  # noqa: E402
from k8s_cc_manager_b200 import _native as N  # noqa: E402
from k8s_cc_manager_b200 import devices as D  # noqa: E402

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

MiB, GiB = 1 << 20, 1 << 30
KIND = {1: "zero", 2: "alias", 3: "partial", 4: "foreign"}
FIRST64 = {"CCM_VMM_FIRST_CHUNK_MB": "64"}   # scrub_alias: a 64 MiB first chunk, so the oracle follows 32768 windows
ALIAS_BYTES = 512 * MiB                      # chunks of 64, 128, 256 and 64 MiB; the second starts with the alias
FALLBACK = {"CCM_PIPELINE": "0", "CCM_ARENA_MAX_SEGMENT_MB": "3"}
TRIAGE_FIELDS = [f for f, _ in N.TriageReport._fields_ if not f.startswith("ms_") and f != "va_base"]


def needs_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


# ---------------------------------------------------------------------------------- product calls in a child
def pair(c: dict) -> list[dict]:
    return [dict(c, probe=0), dict(c, probe=1)]


def clean_cases() -> dict:
    cases = {}
    for mf, il in PP.MODES:
        cases[f"vmm{mf}{il}"] = {"bytes": 1536 * MiB, "env": PP.mode_env(mf, il)}
    cases["whole"] = {"bytes": 0}
    cases["fallback"] = {"bytes": 10 * MiB + 777, "env": FALLBACK}
    cases["fallback1"] = {"bytes": 64 * MiB + 12345, "env": {"CCM_PIPELINE": "0"}}
    cases["fanout"] = {"bytes": GiB, "many": 2}
    cases["census"] = {"bytes": 1536 * MiB, "kind": "census"}
    cases["census_fallback"] = {"bytes": 10 * MiB + 777, "kind": "census", "env": FALLBACK}
    cases["prove"] = {"bytes": 1536 * MiB, "prove": 1}
    cases["prove_fallback"] = {"bytes": 10 * MiB + 777, "prove": 1, "env": FALLBACK}
    cases["tagged"] = {"bytes": 1536 * MiB, "kind": "tagged"}
    return cases


def alias_cases() -> dict:
    return {f"alias{mf}{il}": {"bytes": ALIAS_BYTES, "env": {**PP.mode_env(mf, il), **FIRST64},
                               "drill": {"scrub_alias": 1}} for mf, il in PP.MODES}


def drill_cases() -> dict:
    return {
        "probe_mismatch": {"bytes": 1536 * MiB, "drill": {"probe_mismatch": 5}},
        "probe_dirt": {"bytes": 1536 * MiB, "drill": {"probe_dirt": 5}},
        "probe_dirt_triage": {"bytes": 1536 * MiB, "drill": {"probe_dirt": 5}, "triage": 5},
        "probe_mismatch_fallback": {"bytes": 10 * MiB + 777, "env": FALLBACK, "drill": {"probe_mismatch": 4}},
        "inject": {"bytes": 1536 * MiB, "drill": {"scrub_inject": 6}},
        "flood": {"bytes": 1536 * MiB, "drill": {"scrub_flood": PP.FLOOD}},
        "inject_fallback": {"bytes": 10 * MiB + 777, "env": FALLBACK, "drill": {"scrub_inject": 6}},
    }


def all_cases() -> dict:
    return {**clean_cases(), **alias_cases(), **drill_cases()}


def run_child(pdl: str) -> dict:
    names = list(all_cases())
    calls = [c for n in names for c in pair(all_cases()[n])]
    env = dict(os.environ, CCM_PDL=pdl)
    proc = subprocess.run([sys.executable, str(ROOT / "tests" / "probe_calls.py"), json.dumps(calls)],
                          capture_output=True, text=True, env=env, cwd=ROOT, timeout=1800)
    assert proc.returncode == 0, proc.stdout[-4000:] + proc.stderr[-4000:]
    out = json.loads([x for x in proc.stdout.splitlines() if x.startswith("RESULT ")][-1][len("RESULT "):])
    return {n: (out[2 * i], out[2 * i + 1]) for i, n in enumerate(names)}


@pytest.fixture(scope="module", params=["1", "0"], ids=["pdl", "nopdl"])
def results(request):
    needs_gpu()
    return run_child(request.param)


def chunks_of(r: dict) -> list[tuple[int, int]]:
    """The mapping loop's chunks of a VMM call with a requested size, as addresses."""
    c, res = r["call"], r["results"][0]
    p = PP.plan(c["bytes"], res["device_free_before"], PP.H100_GRAN, c.get("env", {}))
    run = PP.simulate(p, None)
    assert run.mapped == res["bytes_scrubbed"]
    return [(r["probe"]["va_base"] + off, n) for off, n in run.chunks]


def same_as_unarmed(off: dict, on: dict) -> None:
    # a whole-HBM call maps what is free at the time: its size and chunk count may differ by a few tail granules
    vary = ("device_free_before",) + (("bytes_scrubbed", "bytes_unreached", "segments") if not on["call"]["bytes"] else ())
    for a, b in zip(off["results"], on["results"]):
        assert {k: v for k, v in a.items() if k not in vary and not k.startswith("ms_")} == \
               {k: v for k, v in b.items() if k not in vary and not k.startswith("ms_")}
    assert off["rc"] == on["rc"] and off["reports"] == on["reports"]
    assert off.get("residue") == on.get("residue") and off.get("tags", [{}])[0].get("mismatch_bytes") == \
        on.get("tags", [{}])[0].get("mismatch_bytes")


@pytest.mark.parametrize("name", list(clean_cases()))
def test_clean_armed_call_leaves_what_an_unarmed_one_leaves(results, name):
    off, on = results[name]
    same_as_unarmed(off, on)
    assert off["probe"]["probed"] == 0
    p = on["probe"]
    res = on["results"][0]
    calls = max(1, on["call"].get("many", 0))
    if name == "tagged":   # a tagged call ignores the arming
        assert p["probed"] == 0 and on["launches"] == off["launches"]
        return
    assert on["rc"] == 0 and p["probed"] == 1 and p["mismatch_bytes"] == p["mismatch_windows"] == 0
    assert p["reread_nonzero_bytes"] == 0 and p["bytes_probed"] == 32 * p["windows"]
    assert p["launches"] == 3 * res["segments"]   # the last call's own probe: one launch per chunk and step
    if name == "prove" or name == "prove_fallback":
        assert on["cover"]["proved"] == 1 and on["cover"]["covered"] == 1
    if "fallback" in name:
        assert on["launches"] == off["launches"] + 3 * res["segments"]
        assert abs(p["windows"] - res["bytes_scrubbed"] // 4096) <= res["segments"]
        return
    # VMM: every chunk is a whole number of 2 MiB granules from a granule-aligned base
    assert p["windows"] == res["bytes_scrubbed"] // 4096 and p["va_base"] % (2 * MiB) == 0
    if on["call"]["bytes"]:
        assert on["launches"] == off["launches"] + 3 * calls * res["segments"]
        chunks = chunks_of(on)
        assert len(chunks) == res["segments"] and p["windows"] == len(PO.windows(chunks))


@pytest.mark.parametrize("name", list(alias_cases()))
def test_scrub_alias_fails_armed_with_the_oracles_report(results, name):
    off, on = results[name]
    assert off["rc"] == 0 and off["probe"]["probed"] == 0      # the zero gate alone passes it
    assert on["rc"] == N.ERR_MISMATCH and "HBM alias probe found" in on["error"]
    p, res = on["probe"], on["results"][0]
    assert p["probed"] == 1 and res["nonzero_bytes"] == 0 and p["reread_nonzero_bytes"] == 0
    va, n0 = p["va_base"], 64 * MiB
    chunks = chunks_of(on)
    assert chunks[0] == (va, n0) and len(chunks) == res["segments"] == 4
    want = PO.expected(chunks, p["seed"], va, alias=(va + n0, va, n0), classify_limit=0,
                       ranges=[(va, va + res["bytes_scrubbed"])])
    assert p["windows"] == want["windows"] and p["mismatch_bytes"] == want["mismatch_bytes"] > 0
    mm = on["reports"]["mismatch"]
    assert mm[0] == want["mismatch_bytes"] and mm[1] == p["mismatch_windows"] == want["mismatch_windows"]
    assert mm[2] == want["zero_windows"]
    recs = {r["offset"]: r for r in want["records"]}
    firsts = [r["offset"] + (r["mask"] & -r["mask"]).bit_length() - 1 for r in want["records"]]
    lasts = [r["offset"] + r["mask"].bit_length() - 1 for r in want["records"]]
    assert mm[3] == min(firsts) and mm[4] == max(lasts)
    got = on["mismatch_records"]
    assert len(got) == 64
    for g in got:
        w = recs[g["offset"]]
        assert g["mask"] == w["mask"] and g["bytes"] == w["bytes"] and g["chunk"] == 0
        kind, src = PO.classify(w, p["seed"], va, [(va, va + res["bytes_scrubbed"])])
        assert KIND[g["kind"]] == kind
        if g["offset"] < n0:   # view one reads view two's tags: ALIAS, source + n0
            assert kind == "alias" and g["source_offset"] == src == g["offset"] + n0 and g["source_chunk"] == 0
        else:                  # view two reads the zeros view one's check left
            assert kind == "zero" and n0 <= g["offset"] < 2 * n0
    assert [(pg, b) for pg, b, _ in on["reports"]["pages2"]] == sorted(want["pages"].items())


def test_probe_mismatch_drill(results):
    for name, k in (("probe_mismatch", 5), ("probe_mismatch_fallback", 4)):
        off, on = results[name]
        assert off["rc"] == 0
        p = on["probe"]
        assert on["rc"] == N.ERR_MISMATCH and p["mismatch_bytes"] == k and p["mismatch_windows"] == k
        assert p["launches"] == 3 * on["results"][0]["segments"] + k
        got = on["mismatch_records"]
        assert len(got) == k and all(KIND[g["kind"]] == "partial" and g["mask"] == 1 for g in got)
        if name == "probe_mismatch":
            assert [g["offset"] for g in got] == [4096 * i for i in range(k)]
            assert on["reports"]["pages2"] == [[0, k, 0]]


def test_probe_dirt_drill_and_its_triage(results):
    off, on = results["probe_dirt"]
    assert off["rc"] == 0
    assert on["rc"] == N.ERR_DIRTY and on["results"][0]["nonzero_bytes"] == 5 and on["probe"]["reread_nonzero_bytes"] == 5
    dirt = on["reports"]["dirt"]
    assert dirt[0] == 5 and dirt[1] == 5 and [r[0] for r in dirt[6]] == [4096 * i for i in range(5)]
    assert on["reports"]["pages1"] == [[0, 5, 0]] and on["probe"]["mismatch_bytes"] == 0
    _, tr = results["probe_dirt_triage"]
    t = dict(zip(TRIAGE_FIELDS, tr["reports"]["ccm_scrub_last_triage"]))
    assert tr["rc"] == N.ERR_DIRTY and t["triaged"] == 1 and t["pages_examined"] == 1 and t["clear_pages"] == 1
    assert t["clear_bytes"] == 5


@pytest.mark.parametrize("name", ["inject", "flood", "inject_fallback"])
def test_dirt_keeps_the_probe_from_running(results, name):
    off, on = results[name]
    assert on["probe"]["probed"] == 0 and on["rc"] == off["rc"] == N.ERR_DIRTY
    # a flood books more windows than the records hold, and which ones are kept is not fixed: counts and pages are
    a, b = dict(on["reports"]), dict(off["reports"])
    assert a.pop("dirt")[:6] == b.pop("dirt")[:6] and a == b
    assert on["results"][0]["nonzero_bytes"] == off["results"][0]["nonzero_bytes"]
    assert on["launches"] == off["launches"]


# ---------------------------------------------------------------------------------- the region probe
@pytest.fixture(scope="module")
def lib():
    needs_gpu()
    return PGC.open_lib()


def region_probe(lib, ptr: int, n: int, seed: int):
    rep, mm = N.ProbeReport(), N.MismatchReport()
    torch.cuda.synchronize()
    assert lib.ccm_region_probe(0, ptr, n, seed, None, C.byref(rep), C.byref(mm)) == 0, N.last_error()
    return rep, mm


def probe_map(lib, ptr: int, n: int) -> RCC.ArmedMap:
    """Three cover maps for an armed region probe over [ptr, ptr + n): one page, its base 7 bytes into the middle
    window, so that window splits between the outside slot and page 0, and the windows past the page (a 4 MiB region)
    count outside too."""
    w0, k = PO.chunk_windows(ptr, n)
    return RCC.ArmedMap(lib, ptr, n, 0, steps=3, at=(w0 + PO.STRIDE * (k // 2) + 7, 1))


@pytest.mark.parametrize("start,n", [(0, 4 * MiB), (100, 4 * MiB), (100, 3 * 4096 - 100 + 32), (100, 3 * 4096 - 100 + 31),
                                     (4095, 2), (7, 4096 * 5 + 1000), (0, 31)])
def test_region_probe_against_the_oracle(lib, start, n):
    """Plain, then armed (include/ccm.h: ccm_region_prove), where the proving twins run: the same report and bytes both
    times, and armed, three cover maps of the windows."""
    guard = 8192
    buf = torch.full((guard + start + n + guard,), 0xEE, dtype=torch.uint8, device="cuda")
    base = buf.data_ptr()
    ptr = base + guard + start
    for armed in (False, True):
        buf.fill_(0xEE)
        arm = probe_map(lib, ptr, n) if armed else None
        with arm or contextlib.nullcontext():
            rep, mm = region_probe(lib, ptr, n, 0xABCD)
        if arm:
            assert arm.take() == [arm.want(RO.probe_parts([(ptr, n)]))] * 3, (arm.base - ptr, arm.pages)
        w0, k = PO.chunk_windows(ptr, n)
        assert rep.probed == 1 and rep.windows == k and rep.bytes_probed == 32 * k and rep.seed == 0xABCD, armed
        assert rep.mismatch_bytes == 0 and rep.reread_nonzero_bytes == 0 and rep.va_base == ptr, armed
        assert rep.launches == (3 if k else 0) and mm.located == 1 and mm.mismatch_bytes == 0, armed
        host = buf.cpu().numpy()
        want = host.copy()
        want[:] = 0xEE
        for i in range(k):
            o = w0 + 4096 * i - base
            want[o:o + 32] = 0
        assert (host == want).all(), armed   # the windows zero, every other byte (guards included) untouched


class _Prop(C.Structure):      # CUmemAllocationProp
    _fields_ = [("type", C.c_int), ("handle_types", C.c_int), ("loc_type", C.c_int), ("loc_id", C.c_int),
                ("win32", C.c_void_p), ("compression", C.c_ubyte), ("rdma", C.c_ubyte), ("usage", C.c_ushort),
                ("reserved", C.c_ubyte * 4)]


class _Access(C.Structure):    # CUmemAccessDesc
    _fields_ = [("loc_type", C.c_int), ("loc_id", C.c_int), ("flags", C.c_int)]


class TwoViews:
    """One granule of device 0's memory mapped twice, end to end, through the driver's VMM calls: the region
    [va, va + 2 * gran) is two virtual views of the same physical memory, the alias the probe looks for."""

    def __enter__(self):
        torch.zeros(1, device="cuda")   # the primary context, current on this thread
        self.cu = cu = C.CDLL("libcuda.so.1")
        prop = _Prop(type=1, loc_type=1, loc_id=torch.cuda.current_device())   # pinned, on the device
        gran = C.c_size_t()
        self.ok(cu.cuMemGetAllocationGranularity(C.byref(gran), C.byref(prop), 0))
        self.gran = gran.value
        self.handle, self.va = C.c_ulonglong(), C.c_ulonglong()
        self.ok(cu.cuMemCreate(C.byref(self.handle), C.c_size_t(self.gran), C.byref(prop), C.c_ulonglong(0)))
        self.ok(cu.cuMemAddressReserve(C.byref(self.va), C.c_size_t(2 * self.gran), C.c_size_t(0), C.c_ulonglong(0),
                                       C.c_ulonglong(0)))
        self.mapped = []
        for k in range(2):
            a = C.c_ulonglong(self.va.value + k * self.gran)
            self.ok(cu.cuMemMap(a, C.c_size_t(self.gran), C.c_size_t(0), self.handle, C.c_ulonglong(0)))
            self.mapped.append(a)
        acc = _Access(loc_type=1, loc_id=prop.loc_id, flags=3)   # read and write
        self.ok(cu.cuMemSetAccess(self.va, C.c_size_t(2 * self.gran), C.byref(acc), C.c_size_t(1)))
        return self

    def ok(self, rc):
        assert rc == 0, f"CUDA driver error {rc}"

    def __exit__(self, *exc):
        torch.cuda.synchronize()
        for a in self.mapped:
            self.cu.cuMemUnmap(a, C.c_size_t(self.gran))
        self.cu.cuMemAddressFree(self.va, C.c_size_t(2 * self.gran))
        self.cu.cuMemRelease(self.handle)


def test_region_probe_books_the_windows_of_a_second_view(lib):
    """Off-tag bytes in the windows P2 checks: the second view's P1 overwrites the first view's tags (or the other way
    round: one launch takes both views).  Plain and armed, every window of the pair whose tags were lost books off-tag
    bytes, P2 zeroes both views, P3 reads zeros, and armed, each step counts every window on its page."""
    with TwoViews() as tv:
        ptr, n = tv.va.value, 2 * tv.gran
        k = n // PO.STRIDE
        for armed in (False, True):
            arm = probe_map(lib, ptr, n) if armed else None
            with arm or contextlib.nullcontext():
                rep, mm = region_probe(lib, ptr, n, 0x5EED)
            assert rep.probed == 1 and rep.windows == k and rep.reread_nonzero_bytes == 0, armed
            # each pair of windows shares one sector: at least the view whose tags were lost is off them
            assert rep.mismatch_bytes > 0 and mm.mismatch_bytes == rep.mismatch_bytes, (armed, rep.mismatch_bytes)
            assert k // 2 <= mm.mismatch_windows <= 2 * k and mm.truncated == 1, (armed, mm.mismatch_windows)
            if arm:
                assert arm.take() == [arm.want(RO.probe_parts([(ptr, n)]))] * 3, (arm.base - ptr, arm.pages)



def test_rate_bar_against_a_same_run_tag_check(lib):
    n = 16 * GiB
    buf = torch.empty(n, dtype=torch.uint8, device="cuda")
    ptr = buf.data_ptr()
    probe_ms, check_ms = [], []
    for i in range(5):
        rep, _ = region_probe(lib, ptr, n, 1 + i)
        # the check runs over its own tags, as in the tagged gate: the clean pass, not its booking branch
        assert lib.ccm_region_tag_fill(0, ptr, n, 1 + i, None, None) == 0, N.last_error()
        ms, mism = C.c_float(), C.c_uint64()
        assert lib.ccm_region_tag_check_zero(0, ptr, n, 1 + i, None, C.byref(mism), C.byref(ms)) == 0, N.last_error()
        assert mism.value == 0
        if i:   # the first round warms both up
            probe_ms.append(rep.ms_probe)
            check_ms.append(ms.value)
    name = torch.cuda.get_device_name(0)
    print(f"alias probe over 16 GiB on {name}: P1+P2+P3 {statistics.median(probe_ms):.2f} ms, "
          f"tag_check_zero {statistics.median(check_ms):.2f} ms")
    assert statistics.median(probe_ms) < statistics.median(check_ms)


# ---------------------------------------------------------------------------------- the manager end to end
def test_manager_fails_a_transition_with_a_page_mapped_twice(lib, monkeypatch, caplog):
    import kubernetes
    from k8s_cc_manager_b200 import manager
    for k, v in dict(EVICT_OPERATOR_COMPONENTS="false", CC_RELEASE_CUDA_CONTEXT="false").items():
        monkeypatch.setenv(k, v)
    assert lib.ccm_init(N.BACKEND_CUDASIM) == 0
    lib.ccm_sim_set(-1, b"cc_mode", N.CC_MODES["off"])
    lib.ccm_sim_set(0, b"scrub_alias", 1)
    try:
        c = kubernetes.reset_cluster()
        c.add_node(SC.NODE, {})
        mgr = manager.CCManager(SC.NODE, "on", True, device_source=D.find_gpus, scrub_bytes=4 * GiB,
                                scrub_alias_probe="require")
        with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
            assert mgr.set_cc_mode("on") is False
        bdf = next(d.bdf for d in D.find_gpus()[0] if d.cuda_ordinal == 0)
        probe = mgr.last_transition["scrub_probe"][bdf]
        assert probe.probed == 1 and probe.mismatch_bytes > 0
        assert mgr.last_transition["scrub_mismatch"][bdf].mismatch_bytes == probe.mismatch_bytes
        assert any(r.levelno == logging.ERROR and r.getMessage().startswith(f"HBM alias probe on {bdf}")
                   for r in caplog.records)
    finally:
        lib.ccm_sim_set(0, b"scrub_alias", 0)
        PGC.release_wait(lib)
