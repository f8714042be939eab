#!/usr/bin/env python3
"""Cost of the dirt triage on GPU 0: cold whole-HBM zero gates, armed (ccm_scrub_triage) and unarmed, alternated call by
call in one process.  Prints ONE JSON line (and writes it to --out when given).

  python benchmarks/dirt_triage.py [--calls 3] [--hold-ms 100] [--out FILE]

cases:   clean            no dirt: the armed call must cost nothing more;
         inject4          4 injected bytes (scrub_inject): 4 dirty pages;
         flood            every mapped byte dirty (scrub_flood): the triage covers all of HBM in one run;
         runs_worst       10 MiB chunks (CCM_VMM_FIRST_CHUNK_MB = CCM_VMM_CHUNK_MB = 10), each with its first, middle and
                          last byte dirty (scrub_inject): pages 0, 2 and 4 of every 5 are dirty, so the triage launches
                          three kernels for each of about 0.4 runs per page of HBM.
Per case: the call's own wall clock to the verdict (median of --calls after one warm-up round), the armed call's
ms_triage and ms_hold, its runs and pages, and armed minus unarmed with the hold taken out.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from k8s_cc_manager_b200 import _native as N  # noqa: E402

CASES = {"clean": ({}, {}), "inject4": ({"scrub_inject": 4}, {}), "flood": ({"scrub_flood": 0xC3}, {}),
         "runs_worst": ({"scrub_inject": 1 << 40}, {"CCM_VMM_FIRST_CHUNK_MB": "10", "CCM_VMM_CHUNK_MB": "10"})}
DRILLS = ("scrub_inject", "scrub_flood")


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True, check=True).stdout.strip().split(",")
    return {"gpu": q[0].strip(), "power_limit_w": float(q[1])}


def one_gate(lib, case: str, hold_ms: int) -> dict:
    drills, env = CASES[case]
    saved = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    for k in DRILLS:
        assert lib.ccm_sim_set(0, k.encode(), int(drills.get(k, 0))) == 0
    assert lib.ccm_scrub_triage(0, hold_ms) == 0
    res = N.ScrubResult()
    t0 = time.perf_counter()
    rc = lib.ccm_scrub_verify(0, 0, C.byref(res))
    ms = (time.perf_counter() - t0) * 1e3
    lib.ccm_scrub_triage(0, 0)
    for k in DRILLS:
        lib.ccm_sim_set(0, k.encode(), 0)
    for k, v in saved.items():
        if v is None:
            os.environ.pop(k, None)
        else:
            os.environ[k] = v
    assert rc == (N.ERR_DIRTY if drills else 0), (case, rc, N.last_error())
    t = N.TriageReport()
    assert lib.ccm_scrub_last_triage(0, C.byref(t)) == 0
    assert bool(t.triaged) == bool(drills and hold_ms), (case, hold_ms)
    lib.ccm_scrub_release_wait(0, None, None)
    return {"ms": ms, "ms_triage": t.ms_triage, "ms_hold": t.ms_hold, "runs": t.runs, "pages": t.pages_examined,
            "nonzero_bytes": res.nonzero_bytes, "bytes_scrubbed": res.bytes_scrubbed, "segments": res.segments,
            "clear_pages": t.clear_pages}


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=3)
    ap.add_argument("--hold-ms", type=int, default=100)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    lib = N.lib()
    assert lib.ccm_init(N.BACKEND_CUDASIM) == 0
    out = {"bench": "dirt_triage", **card(), "hold_ms": a.hold_ms, "calls": a.calls, "cases": {}}
    for case in CASES:
        runs = {"unarmed": [], "armed": []}
        for i in range(1 + a.calls):
            for name, hold in (("unarmed", 0), ("armed", a.hold_ms)):
                r = one_gate(lib, case, hold)
                if i:
                    runs[name].append(r)
        un, ar = ([r["ms"] for r in runs[k]] for k in ("unarmed", "armed"))
        last = runs["armed"][-1]
        med = statistics.median
        out["cases"][case] = {
            "unarmed_ms_median": med(un), "armed_ms_median": med(ar), "unarmed_ms": un, "armed_ms": ar,
            "spread_ms": max(max(un) - min(un), max(ar) - min(ar)),
            "ms_triage_median": med(r["ms_triage"] for r in runs["armed"]),
            "ms_hold_median": med(r["ms_hold"] for r in runs["armed"]),
            "armed_minus_unarmed_without_hold_ms": med(ar) - med(un) - med(r["ms_hold"] for r in runs["armed"]),
            "runs": last["runs"], "pages": last["pages"], "clear_pages": last["clear_pages"],
            "nonzero_bytes": last["nonzero_bytes"], "bytes_scrubbed": last["bytes_scrubbed"],
            "segments": last["segments"]}
    line = json.dumps(out)
    print(line)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(line + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
