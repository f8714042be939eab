"""Drives product scrub gate calls on CUDA device 0, proven and probed or not, and reports what each call returned:
what tests/probe_calls.py reports (which includes tests/cover_proof_calls.py's), the probe proof and its inexact pages.

Imported by tests/test_probe_cover_gpu.py.  Run as a script it reads a JSON list of calls from argv[1] (those of
probe_calls.py, plus the drills "probe_skip" / "probe_skip_step"), makes them in this fresh process and prints one
`RESULT <json>` line.  Not collected by pytest.
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

import probe_calls as PC  # noqa: E402
import product_gate_calls as PGC  # noqa: E402
from k8s_cc_manager_b200 import _native as N  # noqa: E402

SKIP_KEYS = ("probe_skip", "probe_skip_step")
STEP_FIELDS = [f for f, _ in N.ProbeCoverStep._fields_ if f != "reserved"]


def probe_cover_dict(r: N.ProbeCover) -> dict:
    d = {f: getattr(r, f) for f, _ in N.ProbeCover._fields_ if f != "steps"}
    d["steps"] = [{f: getattr(r.steps[k], f) for f in STEP_FIELDS} for k in range(3)]
    return d


def probe_cover_pages(lib) -> list:
    n = C.c_uint64(0)
    assert lib.ccm_last_probe_cover_pages(0, None, 0, C.byref(n)) == 0, N.last_error()
    buf = (N.ProbeCoverPage * max(1, n.value))()
    assert lib.ccm_last_probe_cover_pages(0, buf, n.value, C.byref(n)) == 0, N.last_error()
    return [{"page": p.page, "chunk": p.chunk, "expected": p.expected, "count": list(p.count)} for p in buf[:n.value]]


def call(lib, c: dict) -> dict:
    drill = c.get("drill", {})
    for k in SKIP_KEYS:
        assert lib.ccm_sim_set(0, k.encode(), int(drill.get(k, 0))) == 0, N.last_error()
    try:
        out = PC.call(lib, c)
    finally:
        for k in SKIP_KEYS:
            lib.ccm_sim_set(0, k.encode(), 0)
    pc = N.ProbeCover()
    assert lib.ccm_scrub_last_probe_cover(0, C.byref(pc)) == 0, N.last_error()
    out["probe_cover"] = probe_cover_dict(pc)
    out["probe_cover_pages"] = probe_cover_pages(lib)
    return out


def main() -> None:
    lib = PGC.open_lib()
    print("RESULT " + json.dumps([call(lib, c) for c in json.loads(sys.argv[1])]), flush=True)


if __name__ == "__main__":
    main()
