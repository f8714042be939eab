"""Drives failed product scrub gate calls on CUDA device 0, proven or not, and reports what each call returned and left:
the result, the tag and census counts, the dirt, mismatch and triage reports with their page maps and triage pages, the
coverage proof, the alias probe and its proof, the report proof and the inexact pages of each proof, the address the
reports' offsets are from, and the kernels launched.

Imported by tests/test_report_cover_gpu.py, tests/test_gate_scenarios_gpu.py and benchmarks/report_proof.py.  Run as a script it reads a JSON list of
calls from argv[1], or from the file argv[1] names after an "@" (`[{"bytes": ..., "env": {...}, "drill": {"scrub_inject": 4}, "kind": "zero", "prove": 1,
"triage": 5, "mismatch_triage": 5, "probe": 0, "many": 0}, ...]`; kind is zero, tagged, census or census_tagged), makes
them in this fresh process and prints one `RESULT <json>` line, so that CCM_PDL, which the library latches once per
process, takes this process's value.  Not collected by pytest.
"""
from __future__ import annotations

import ctypes as C
import json
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
for p in (ROOT, ROOT / "tests"):
    if str(p) not in sys.path:
        sys.path.insert(0, str(p))

import cover_proof_calls as CPC  # noqa: E402
import product_gate_calls as PGC  # noqa: E402
from k8s_cc_manager_b200 import _native as N  # noqa: E402

DRILL_KEYS = CPC.DRILL_KEYS + ("tag_flood", "triage_stay", "triage_return", "probe_mismatch", "probe_dirt", "probe_skip",
                               "probe_skip_step", "report_skip", "report_skip_step")
STEP_FIELDS = [f for f, _ in N.ReportCoverStep._fields_ if f != "reserved"]


def report_cover(lib) -> dict:
    r = N.ReportCover()
    assert lib.ccm_scrub_last_report_cover(0, C.byref(r)) == 0, N.last_error()
    d = {f: getattr(r, f) for f, _ in N.ReportCover._fields_ if f != "steps"}
    d["steps"] = {name: {f: getattr(r.steps[k], f) for f in STEP_FIELDS} for k, name in enumerate(N.REPORT_STEPS)}
    n = C.c_uint64(0)
    assert lib.ccm_last_report_cover_pages(0, None, 0, C.byref(n)) == 0, N.last_error()
    buf = (N.ReportCoverPage * max(1, n.value))()
    assert lib.ccm_last_report_cover_pages(0, buf, n.value, C.byref(n)) == 0, N.last_error()
    d["pages"] = [{"page": p.page, "chunk": p.chunk, "step": N.REPORT_STEPS[p.step - 1], "expected": p.expected,
                   "counted": p.counted} for p in buf[:n.value]]
    return d


def triage_pages(lib) -> dict:
    out = {}
    for fn in ("ccm_last_triage_pages", "ccm_last_mismatch_triage_pages"):
        n = C.c_uint64(0)
        assert getattr(lib, fn)(0, None, 0, C.byref(n)) == 0
        buf = (N.TriagePage * max(1, n.value))()
        assert getattr(lib, fn)(0, buf, n.value, C.byref(n)) == 0
        out[fn] = [[getattr(p, f) for f, _ in N.TriagePage._fields_ if f != "reserved"] for p in buf[:n.value]]
    return out


def timings(lib) -> dict:
    """The locate pass's and the triages' own times (for the benchmark)."""
    d = N.DirtReport()
    t, m = N.TriageReport(), N.TriageReport()
    assert lib.ccm_scrub_last_dirt(0, C.byref(d)) == 0
    assert lib.ccm_scrub_last_triage(0, C.byref(t)) == 0
    assert lib.ccm_scrub_last_mismatch_triage(0, C.byref(m)) == 0
    return {"ms_locate": d.ms_locate, "ms_triage": t.ms_triage, "ms_mismatch_triage": m.ms_triage}


def call(lib, c: dict) -> dict:
    kind, many = c.get("kind", "zero"), c.get("many", 0)
    count = max(1, many)
    res = (N.ScrubResult * count)()
    tags = (N.TagResult * count)() if kind in ("tagged", "census_tagged") else None
    census = (N.ResidueReport * count)() if kind.startswith("census") else None
    devs = (C.c_int * count)(*([0] * count))
    wall = C.c_double()
    with PGC.knobs(c.get("env", {})):
        for k in DRILL_KEYS:
            assert lib.ccm_sim_set(0, k.encode(), int(c.get("drill", {}).get(k, 0))) == 0, N.last_error()
        assert lib.ccm_scrub_prove(0, int(c.get("prove", 0))) == 0, N.last_error()
        assert lib.ccm_scrub_probe(0, int(c.get("probe", 0))) == 0, N.last_error()
        assert lib.ccm_scrub_triage(0, int(c.get("triage", 0))) == 0, N.last_error()
        assert lib.ccm_scrub_mismatch_triage(0, int(c.get("mismatch_triage", 0))) == 0, N.last_error()
        launches = lib.ccm_kernel_launches()
        t0 = time.perf_counter()
        try:
            if census is not None:
                rc = lib.ccm_scrub_verify_many_residue(count, devs, c["bytes"], tags, census, res, C.byref(wall))
            elif tags is not None:
                rc = lib.ccm_scrub_verify_many_tagged(count, devs, c["bytes"], tags, res, C.byref(wall))
            elif many:
                rc = lib.ccm_scrub_verify_many(count, devs, c["bytes"], res, C.byref(wall))
            else:
                rc = lib.ccm_scrub_verify(0, c["bytes"], res)
            ms_verdict = (time.perf_counter() - t0) * 1e3
            err = N.last_error() if rc else ""
            launches = lib.ccm_kernel_launches() - launches
        finally:
            lib.ccm_scrub_prove(0, 0)
            lib.ccm_scrub_probe(0, 0)
            lib.ccm_scrub_triage(0, 0)
            lib.ccm_scrub_mismatch_triage(0, 0)
            for k in DRILL_KEYS:
                lib.ccm_sim_set(0, k.encode(), 0)
    cover = N.CoverReport()
    assert lib.ccm_scrub_last_cover(0, C.byref(cover)) == 0, N.last_error()
    left = CPC.reports(lib)
    left.update(triage_pages(lib))
    probe, pcover = N.ProbeReport(), N.ProbeCover()
    assert lib.ccm_scrub_last_probe(0, C.byref(probe)) == 0, N.last_error()
    assert lib.ccm_scrub_last_probe_cover(0, C.byref(pcover)) == 0, N.last_error()
    dirt, mismatch = N.DirtReport(), N.MismatchReport()
    assert lib.ccm_scrub_last_dirt(0, C.byref(dirt)) == 0 and lib.ccm_scrub_last_mismatch(0, C.byref(mismatch)) == 0
    out = {"call": c, "rc": rc, "error": err, "launches": launches, "ms_verdict": ms_verdict,
           "results": [{f: getattr(r, f) for f in PGC.FIELDS} for r in res],
           "cover": CPC.cover_dict(cover), "cover_pages": CPC.cover_pages(lib), "report_cover": report_cover(lib),
           "reports": left, "times": timings(lib),
           "probe": {f: getattr(probe, f) for f, _ in N.ProbeReport._fields_ if f not in ("reserved", "ms_probe")},
           "probe_cover": {"proved": pcover.proved, "covered": pcover.covered, "windows_expected": pcover.windows_expected,
                           "steps": [{f: getattr(s, f) for f, _ in N.ProbeCoverStep._fields_ if f != "reserved"}
                                     for s in pcover.steps]}}
    PGC.release_wait(lib)
    if tags is not None:
        out["tags"] = [{"mismatch_bytes": t.mismatch_bytes, "seed": t.seed, "va_base": t.va_base} for t in tags]
    if census is not None:
        out["residue"] = [{"residue_bytes": r.residue_bytes, "residue_windows": r.residue_windows} for r in census]
    # the address every offset of the call is from: the tags', the probe's or a report's (0 when none was kept)
    out["va_base"] = next((v for v in ([t.va_base for t in tags] if tags is not None else []) +
                           [probe.va_base, dirt.va_base, mismatch.va_base] if v), 0)
    return out


def main() -> None:
    lib = PGC.open_lib()
    arg = sys.argv[1]
    calls = json.loads(Path(arg[1:]).read_text() if arg.startswith("@") else arg)
    print("RESULT " + json.dumps([call(lib, c) for c in calls]), flush=True)


if __name__ == "__main__":
    main()
