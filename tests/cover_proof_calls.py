"""Drives product scrub gate calls on CUDA device 0, armed for the coverage proof or not, and reports what each call
returned: the result, the tag and census counts, the coverage report and its inexact pages, and the kernels launched.

Imported by tests/test_cover_proof_gpu.py.  Run as a script it reads a JSON list of calls from argv[1]
(`[{"bytes": ..., "env": {...}, "drill": {"scrub_inject": 4}, "kind": "zero", "prove": 1, "many": 0}, ...]`; kind is
zero, tagged, census or census_tagged), makes them in this fresh process and prints one `RESULT <json>` line, so that
CCM_PDL, which the library latches once per process, takes this process's value.  Not collected by pytest.
"""
from __future__ import annotations

import ctypes as C
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
for p in (ROOT, ROOT / "tests"):
    if str(p) not in sys.path:
        sys.path.insert(0, str(p))

import product_gate_calls as PGC  # noqa: E402
from k8s_cc_manager_b200 import _native as N  # noqa: E402

DRILL_KEYS = ("scrub_inject", "scrub_poison", "scrub_flood", "tag_inject", "scrub_alias", "scrub_residue",
              "cover_skip", "cover_pass")
PASS_FIELDS = [f for f, _ in N.CoverPass._fields_ if f != "reserved"]


def cover_dict(r: N.CoverReport) -> dict:
    d = {f: getattr(r, f) for f, _ in N.CoverReport._fields_ if f != "passes"}
    d["passes"] = {name: {f: getattr(r.passes[k], f) for f in PASS_FIELDS} for k, name in enumerate(N.COVER_PASSES)}
    return d


def cover_pages(lib) -> list:
    n = C.c_uint64(0)
    assert lib.ccm_last_cover_pages(0, None, 0, C.byref(n)) == 0, N.last_error()
    buf = (N.CoverPage * max(1, n.value))()
    assert lib.ccm_last_cover_pages(0, buf, n.value, C.byref(n)) == 0, N.last_error()
    return [{"page": p.page, "chunk": p.chunk, "expected": p.expected, "first": p.count[0], "check": p.count[1],
             "readback": p.count[2]} for p in buf[:n.value]]


def reports(lib) -> dict:
    """What else the call left on device 0: the dirt and mismatch reports, the three page maps and both triages, without
    addresses (offsets are from va_base) and times."""
    out = {}
    d = N.DirtReport()
    assert lib.ccm_scrub_last_dirt(0, C.byref(d)) == 0
    out["dirt"] = [d.nonzero_bytes, d.dirty_windows, d.first_offset, d.last_offset, d.nrecords, d.located,
                   [(r.offset, r.chunk, r.mask, bytes(r.bytes).hex()) for r in d.records[:d.nrecords]]]
    m = N.MismatchReport()
    assert lib.ccm_scrub_last_mismatch(0, C.byref(m)) == 0
    out["mismatch"] = [m.mismatch_bytes, m.mismatch_windows, m.zero_windows, m.first_offset, m.last_offset, m.nrecords,
                       [(r.offset, r.chunk, r.mask, r.kind) for r in m.records[:m.nrecords]]]
    for book in (1, 2, 3):
        n = C.c_uint64(0)
        assert lib.ccm_last_page_map(0, book, None, 0, C.byref(n)) == 0
        buf = (N.PageEntry * max(1, n.value))()
        assert lib.ccm_last_page_map(0, book, buf, n.value, C.byref(n)) == 0
        out[f"pages{book}"] = [(e.page, e.bytes, e.chunk) for e in buf[:n.value]]
    for fn in ("ccm_scrub_last_triage", "ccm_scrub_last_mismatch_triage"):
        t = N.TriageReport()
        assert getattr(lib, fn)(0, C.byref(t)) == 0
        out[fn] = [getattr(t, f) for f, _ in N.TriageReport._fields_ if not f.startswith("ms_") and f != "va_base"]
    return out


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
        assert lib.ccm_scrub_triage(0, int(c.get("triage", 0))) == 0, N.last_error()
        assert lib.ccm_scrub_mismatch_triage(0, int(c.get("mismatch_triage", 0))) == 0, N.last_error()
        launches = lib.ccm_kernel_launches()
        try:
            if census is not None:
                rc = lib.ccm_scrub_verify_many_residue(count, devs, c["bytes"], tags, census, res, C.byref(wall))
            elif tags is not None:
                rc = lib.ccm_scrub_verify_many_tagged(count, devs, c["bytes"], tags, res, C.byref(wall))
            else:
                rc = lib.ccm_scrub_verify_many(count, devs, c["bytes"], res, C.byref(wall))
            err = N.last_error() if rc else ""
            launches = lib.ccm_kernel_launches() - launches
        finally:
            lib.ccm_scrub_prove(0, 0)
            lib.ccm_scrub_triage(0, 0)
            lib.ccm_scrub_mismatch_triage(0, 0)
            for k in DRILL_KEYS:
                lib.ccm_sim_set(0, k.encode(), 0)
    cover = N.CoverReport()
    assert lib.ccm_scrub_last_cover(0, C.byref(cover)) == 0, N.last_error()
    left = reports(lib)
    PGC.release_wait(lib)
    out = {"call": c, "rc": rc, "error": err, "launches": launches,
           "results": [{f: getattr(r, f) for f in PGC.FIELDS + ("ms_scrub", "ms_verify")} for r in res],
           "cover": cover_dict(cover), "pages": cover_pages(lib), "reports": left}
    if tags is not None:
        out["tags"] = [{"mismatch_bytes": t.mismatch_bytes, "ms_tag": t.ms_tag, "ms_check": t.ms_check} for t in tags]
    if census is not None:
        out["residue"] = [{"residue_bytes": r.residue_bytes, "residue_windows": r.residue_windows} for r in census]
    return out


def main() -> None:
    lib = PGC.open_lib()
    print("RESULT " + json.dumps([call(lib, c) for c in json.loads(sys.argv[1])]), flush=True)


if __name__ == "__main__":
    main()
