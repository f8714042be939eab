#!/usr/bin/env python3
"""Cost of the mismatch triage on GPU 0: cold whole-HBM tagged gates, armed (ccm_scrub_mismatch_triage) and unarmed,
alternated call by call in one process.  Prints ONE JSON line (and writes it to --out when given).

  python benchmarks/mismatch_triage.py [--calls 3] [--hold-ms 100] [--out FILE]

cases:   clean            no mismatch: the armed call must cost nothing more;
         tag_inject4      4 injected mismatches (tag_inject): a few pages;
         alias            scrub_alias with CCM_MAP_FIRST=0: both 1 GiB views of the aliased range, in one run;
         tag_flood        every mapped byte off its tag (tag_flood): the triage re-tags, checks and re-reads all of HBM.
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

CASES = {"clean": ({}, {}), "tag_inject4": ({"tag_inject": 4}, {}),
         "alias": ({"scrub_alias": 1}, {"CCM_MAP_FIRST": "0"}), "tag_flood": ({"tag_flood": 0x5A}, {})}
DRILLS = ("tag_inject", "scrub_alias", "tag_flood")


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
    assert lib.ccm_scrub_mismatch_triage(0, hold_ms) == 0
    res, tag = N.ScrubResult(), N.TagResult()
    try:
        t0 = time.perf_counter()
        rc = lib.ccm_scrub_verify_tagged(0, 0, C.byref(tag), C.byref(res))
        ms = (time.perf_counter() - t0) * 1e3
    finally:
        lib.ccm_scrub_mismatch_triage(0, 0)
        for k in DRILLS:
            lib.ccm_sim_set(0, k.encode(), 0)
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    assert rc == (N.ERR_MISMATCH if drills else 0), (case, rc, N.last_error())
    t = N.TriageReport()
    assert lib.ccm_scrub_last_mismatch_triage(0, C.byref(t)) == 0
    assert bool(t.triaged) == bool(drills and hold_ms), (case, hold_ms)
    lib.ccm_scrub_release_wait(0, None, None)
    return {"ms": ms, "ms_triage": t.ms_triage, "ms_hold": t.ms_hold, "runs": t.runs, "pages": t.pages_examined,
            "mismatch_bytes": tag.mismatch_bytes, "bytes_scrubbed": res.bytes_scrubbed, "segments": res.segments,
            "stay_pages": t.stay_pages, "return_pages": t.return_pages, "clear_pages": t.clear_pages}


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=3)
    ap.add_argument("--hold-ms", type=int, default=100)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    lib = N.lib()
    assert lib.ccm_init(N.BACKEND_CUDASIM) == 0
    out = {"bench": "mismatch_triage", **card(), "hold_ms": a.hold_ms, "calls": a.calls, "cases": {}}
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
            "runs": last["runs"], "pages": last["pages"], "stay_pages": last["stay_pages"],
            "return_pages": last["return_pages"], "clear_pages": last["clear_pages"],
            "mismatch_bytes": last["mismatch_bytes"], "bytes_scrubbed": last["bytes_scrubbed"],
            "segments": last["segments"]}
    line = json.dumps(out)
    print(line)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(line + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
