"""Drives product scrub gate calls on CUDA device 0, armed for the alias probe or not, and reports what each call
returned: what tests/cover_proof_calls.py reports (result, counts, coverage, the other reports and the kernels
launched), the probe report, and the mismatch report's records in full.

Imported by tests/test_alias_probe_gpu.py.  Run as a script it reads a JSON list of calls from argv[1] (those of
cover_proof_calls.py, plus "probe": 0/1 and the drills "probe_mismatch" / "probe_dirt"), makes them in this fresh
process and prints one `RESULT <json>` line, so that CCM_PDL, which the library latches once per process, takes this
process's value.  Not collected by pytest.
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

import cover_proof_calls as CPC  # noqa: E402
import product_gate_calls as PGC  # noqa: E402
from k8s_cc_manager_b200 import _native as N  # noqa: E402

PROBE_DRILLS = ("probe_mismatch", "probe_dirt")


def probe_dict(p: N.ProbeReport) -> dict:
    return {f: getattr(p, f) for f, _ in N.ProbeReport._fields_ if f != "reserved"}


def mismatch_records(lib) -> list:
    m = N.MismatchReport()
    assert lib.ccm_scrub_last_mismatch(0, C.byref(m)) == 0
    return [{"offset": r.offset, "chunk": r.chunk, "mask": r.mask, "kind": r.kind, "source_offset": r.source_offset,
             "source_chunk": r.source_chunk, "bytes": bytes(r.bytes).hex()} for r in m.records[:m.nrecords]]


def call(lib, c: dict) -> dict:
    for k in PROBE_DRILLS:
        assert lib.ccm_sim_set(0, k.encode(), int(c.get("drill", {}).get(k, 0))) == 0, N.last_error()
    assert lib.ccm_scrub_probe(0, int(c.get("probe", 0))) == 0, N.last_error()
    try:
        out = CPC.call(lib, c)
    finally:
        lib.ccm_scrub_probe(0, 0)
        for k in PROBE_DRILLS:
            lib.ccm_sim_set(0, k.encode(), 0)
    p = N.ProbeReport()
    assert lib.ccm_scrub_last_probe(0, C.byref(p)) == 0, N.last_error()
    out["probe"] = probe_dict(p)
    out["mismatch_records"] = mismatch_records(lib)
    return out


def main() -> None:
    lib = PGC.open_lib()
    print("RESULT " + json.dumps([call(lib, c) for c in json.loads(sys.argv[1])]), flush=True)


if __name__ == "__main__":
    main()
