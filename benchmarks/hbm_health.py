#!/usr/bin/env python3
"""Cost of the HBM health report on GPU 0: cold whole-HBM zero gates armed for it (ccm_scrub_health mode 2, require)
and unarmed, alternated call by call in one process after one warm-up round.  Prints ONE JSON line (and writes it to
--out when given).

  python benchmarks/hbm_health.py [--calls 15] [--out FILE]

Per arming: the call's own wall clock to the verdict and ms_total, and (armed) ms_health, the host time of the two
snapshots' NVML queries, each as median, p10, p90 and spread over --calls; which queries answered and the armed
calls' verdicts.  Then --snapshots standalone snapshots (ccm_hbm_snapshot, no CUDA work) for the cost of one snapshot
apart from any gate.  The card's name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parent))

from cover_proof import card, stats  # noqa: E402
from k8s_cc_manager_b200 import _native as N  # noqa: E402


def one_gate(lib, armed: bool) -> dict:
    assert lib.ccm_scrub_health(0, 2 if armed else 0) == 0, N.last_error()
    res = N.ScrubResult()
    try:
        t0 = time.perf_counter()
        rc = lib.ccm_scrub_verify(0, 0, C.byref(res))
        ms = (time.perf_counter() - t0) * 1e3
    finally:
        lib.ccm_scrub_health(0, 0)
    assert rc == 0, (armed, rc, N.last_error())
    h = N.HbmHealth()
    assert lib.ccm_scrub_last_health(0, C.byref(h)) == 0
    assert h.mode == (2 if armed else 0) and h.verdict == (N.HBM_FIT if armed else 0)
    lib.ccm_scrub_release_wait(0, None, None)
    return {"ms": ms, "ms_total": res.ms_total, "ms_health": h.ms_health, "ms_before": h.before.ms_query,
            "ms_after": h.after.ms_query, "available": h.after.available, "bytes_scrubbed": res.bytes_scrubbed,
            "d_dram_corrected": h.d_dram_corrected, "d_dram_uncorrected": h.d_dram_uncorrected}


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=15)
    ap.add_argument("--snapshots", type=int, default=200)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    lib = N.lib()
    assert lib.ccm_init(N.BACKEND_CUDASIM) == 0
    out = {"bench": "hbm_health", **card(), "calls": a.calls}
    runs = {"unarmed": [], "armed": []}
    for i in range(1 + a.calls):
        for name in ("unarmed", "armed"):
            r = one_gate(lib, name == "armed")
            if i:
                runs[name].append(r)
    for name, rs in runs.items():
        out[name] = {"verdict_ms": stats([r["ms"] for r in rs]), "ms_total": stats([r["ms_total"] for r in rs]),
                     "bytes_scrubbed": rs[-1]["bytes_scrubbed"]}
    arm = runs["armed"]
    out["armed"].update(ms_health=stats([r["ms_health"] for r in arm]), ms_before=stats([r["ms_before"] for r in arm]),
                        ms_after=stats([r["ms_after"] for r in arm]),
                        queries_answered=[q for k, q in enumerate(N.HBM_QUERIES) if arm[-1]["available"] >> k & 1],
                        d_dram_corrected=[r["d_dram_corrected"] for r in arm],
                        d_dram_uncorrected=[r["d_dram_uncorrected"] for r in arm])
    out["armed_minus_unarmed_verdict_ms"] = out["armed"]["verdict_ms"]["median"] - out["unarmed"]["verdict_ms"]["median"]
    snaps = []
    for _ in range(a.snapshots):
        s = N.HbmState()
        assert lib.ccm_hbm_snapshot(0, C.byref(s)) == 0, N.last_error()
        snaps.append(s.ms_query)
    out["snapshot_ms"] = stats(snaps)
    out["snapshots"] = a.snapshots
    line = json.dumps(out)
    print(line)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(line + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
