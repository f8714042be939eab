"""Drives product scrub gate calls on CUDA device 0, armed for the coverage proof or not, and reports what
tests/cover_proof_calls.py reports of each, plus its coverage ledger and inexact slots.  The ledger's drills
("cover_repeat", "cover_lane_drop") are set around each call like the others.

Imported by tests/test_cover_ledger_gpu.py.  Run as a script it reads a JSON list of calls from argv[1] (as
cover_proof_calls.py), makes them in this fresh process and prints one `RESULT <json>` line.  With CCM_LIB set it drives
that library (a mutant: tests/test_cover_ledger_gpu.py).  Not collected by pytest.
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

LEDGER_DRILLS = ("cover_repeat", "cover_lane_drop")
PASS_FIELDS = [f for f, _ in N.LedgerPass._fields_ if f != "reserved"]


def ledger_dict(lib) -> dict:
    r = N.CoverLedger()
    assert lib.ccm_scrub_last_ledger(0, C.byref(r)) == 0, N.last_error()
    d = {f: getattr(r, f) for f, _ in N.CoverLedger._fields_ if f != "passes"}
    d["passes"] = {name: {f: getattr(r.passes[k], f) for f in PASS_FIELDS} for k, name in enumerate(N.COVER_PASSES)}
    n = C.c_uint64(0)
    assert lib.ccm_last_ledger_slots(0, None, 0, C.byref(n)) == 0, N.last_error()
    buf = (N.LedgerSlot * max(1, n.value))()
    assert lib.ccm_last_ledger_slots(0, buf, n.value, C.byref(n)) == 0, N.last_error()
    d["slots"] = [{"slot": x.slot, "chunk": x.chunk, "expected": x.expected, "first": x.count[0], "check": x.count[1],
                   "readback": x.count[2]} for x in buf[:n.value]]
    return d


def call(lib, c: dict) -> dict:
    for k in LEDGER_DRILLS:
        assert lib.ccm_sim_set(0, k.encode(), int(c.get("drill", {}).get(k, 0))) == 0, N.last_error()
    try:
        out = CPC.call(lib, c)
    finally:
        for k in LEDGER_DRILLS:
            lib.ccm_sim_set(0, k.encode(), 0)
    out["ledger"] = ledger_dict(lib)
    return out


def main() -> None:
    lib = PGC.open_lib()
    print("RESULT " + json.dumps([call(lib, c) for c in json.loads(sys.argv[1])]), flush=True)


if __name__ == "__main__":
    main()
