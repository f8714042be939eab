#!/usr/bin/env python3
"""Cost of the coverage proof on GPU 0: cold whole-HBM zero and tagged gates, armed (ccm_scrub_prove) and unarmed,
alternated call by call in one process.  Prints ONE JSON line (and writes it to --out when given).

  python benchmarks/cover_proof.py [--calls 9] [--out FILE]

Per check (zero, tagged) and arming: the call's own wall clock to the verdict (median, p10, p90 and spread over --calls
after one warm-up round), and the medians of ms_scrub, ms_verify, ms_tag, ms_check and (armed) ms_prove.  The card's
name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from k8s_cc_manager_b200 import _native as N  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True, check=True).stdout.strip().split(",")
    return {"gpu": q[0].strip(), "power_limit_w": float(q[1])}


def one_gate(lib, tagged: bool, prove: bool) -> dict:
    assert lib.ccm_scrub_prove(0, int(prove)) == 0, N.last_error()
    res, tag = N.ScrubResult(), N.TagResult()
    try:
        t0 = time.perf_counter()
        rc = lib.ccm_scrub_verify_tagged(0, 0, C.byref(tag), C.byref(res)) if tagged else \
            lib.ccm_scrub_verify(0, 0, C.byref(res))
        ms = (time.perf_counter() - t0) * 1e3
    finally:
        lib.ccm_scrub_prove(0, 0)
    assert rc == 0, (tagged, prove, rc, N.last_error())
    cov = N.CoverReport()
    assert lib.ccm_scrub_last_cover(0, C.byref(cov)) == 0
    assert cov.proved == int(prove) and cov.covered == int(prove)
    lib.ccm_scrub_release_wait(0, None, None)
    return {"ms": ms, "ms_scrub": res.ms_scrub, "ms_verify": res.ms_verify, "ms_tag": tag.ms_tag if tagged else 0.0,
            "ms_check": tag.ms_check if tagged else 0.0, "ms_prove": cov.ms_prove, "bytes_scrubbed": res.bytes_scrubbed}


def stats(xs: list) -> dict:
    xs = sorted(xs)
    q = statistics.quantiles(xs, n=10) if len(xs) > 1 else [xs[0]] * 9
    return {"median": statistics.median(xs), "p10": q[0], "p90": q[-1], "spread": xs[-1] - xs[0], "n": len(xs)}


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=9)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    lib = N.lib()
    assert lib.ccm_init(N.BACKEND_CUDASIM) == 0
    out = {"bench": "cover_proof", **card(), "calls": a.calls, "checks": {}}
    for check in ("zero", "tagged"):
        runs = {"unarmed": [], "armed": []}
        for i in range(1 + a.calls):
            for name in ("unarmed", "armed"):
                r = one_gate(lib, check == "tagged", name == "armed")
                if i:
                    runs[name].append(r)
        med = statistics.median
        row = {}
        for name, rs in runs.items():
            row[name] = {"verdict_ms": stats([r["ms"] for r in rs]),
                         **{f"{k}_median": med(r[k] for r in rs) for k in ("ms_scrub", "ms_verify", "ms_tag",
                                                                           "ms_check", "ms_prove")},
                         "bytes_scrubbed": rs[-1]["bytes_scrubbed"]}
        row["armed_minus_unarmed_verdict_ms"] = row["armed"]["verdict_ms"]["median"] - row["unarmed"]["verdict_ms"]["median"]
        for k in ("ms_scrub", "ms_verify", "ms_tag", "ms_check"):
            if row["unarmed"][f"{k}_median"]:
                row[f"{k}_armed_over_unarmed"] = row["armed"][f"{k}_median"] / row["unarmed"][f"{k}_median"]
        out["checks"][check] = row
    line = json.dumps(out)
    print(line)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(line + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
