"""Drives product scrub gate calls on CUDA device 0 as tests/report_cover_calls.py does, each optionally armed for the
HBM health report, and adds to each record the report the call left.

A call takes two more keys: "health" (ccm_scrub_health's mode, 0 = unarmed) and "hbm_drill" ({"hbm_uncorrected": 1,
...}, the drills of the health report).  Run as a script it reads the calls as report_cover_calls.py does and prints
one `RESULT <json>` line.  Imported by tests/test_hbm_health_gpu.py and benchmarks/hbm_health.py.  Not collected by
pytest.
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
import report_cover_calls as RCC  # noqa: E402
from k8s_cc_manager_b200 import _native as N  # noqa: E402

HBM_DRILL_KEYS = ("hbm_uncorrected", "hbm_corrected", "hbm_remap_pending", "hbm_remap_failure", "hbm_unavailable")


def snapshot_dict(s: N.HbmState) -> dict:
    return {f: (list(getattr(s, f)) if f == "nvml_rc" else getattr(s, f)) for f, _ in N.HbmState._fields_
            if f != "reserved"}


def health_dict(lib) -> dict:
    h = N.HbmHealth()
    assert lib.ccm_scrub_last_health(0, C.byref(h)) == 0, N.last_error()
    d = {f: getattr(h, f) for f, _ in N.HbmHealth._fields_ if f not in ("before", "after")}
    d["before"], d["after"] = snapshot_dict(h.before), snapshot_dict(h.after)
    return d


def call(lib, c: dict) -> dict:
    mode = int(c.get("health", 0))
    for k in HBM_DRILL_KEYS:
        assert lib.ccm_sim_set(0, k.encode(), int(c.get("hbm_drill", {}).get(k, 0))) == 0, N.last_error()
    assert lib.ccm_scrub_health(0, mode) == 0, N.last_error()
    try:
        out = RCC.call(lib, c)
    finally:
        lib.ccm_scrub_health(0, 0)
        for k in HBM_DRILL_KEYS:
            lib.ccm_sim_set(0, k.encode(), 0)
    out["health"] = health_dict(lib)
    return out


def main() -> None:
    lib = PGC.open_lib()
    arg = sys.argv[1]
    calls = json.loads(Path(arg[1:]).read_text() if arg.startswith("@") else arg)
    print("RESULT " + json.dumps([call(lib, c) for c in calls]), flush=True)


if __name__ == "__main__":
    main()
