#!/usr/bin/env python3
"""Cost of the report proof on GPU 0: cold whole-HBM gates that fail, proven (ccm_scrub_prove) and unproven, alternated
call by call in one process after one warm-up round.  Prints ONE JSON line (and writes it to --out when given).

  python benchmarks/report_proof.py [--calls 9] [--out FILE]

Scenarios: "inject" (scrub_inject = 4, the dirt triage), "flood" (scrub_flood, every byte dirty, the dirt triage),
"tag_flood" (the tagged gate with tag_flood, the mismatch triage), and "clean" (a zero gate that passes, which proves
nothing).  Per scenario and arming: the call's wall clock to its verdict, the locate pass's time (ms_locate), the
triage's (ms_triage, or the mismatch triage's), and (proven) the report proof's copy and comparison time (ms_prove),
each as median, p10, p90 and spread over --calls.  Then, under torch.profiler, --profile-calls more "inject" and
"flood" gates of each arming, alternated: the GPU time of the locate kernels alone (the plain `locate_dirt_kernel`
against the proving `cover_locate_pass`), summed over the call's locate pass and triage re-reads.  The card's name and
power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import statistics
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
for p in (ROOT, ROOT / "tests", Path(__file__).resolve().parent):
    sys.path.insert(0, str(p))

import report_cover_calls as RCC  # noqa: E402
from cover_proof import card, stats  # noqa: E402
from k8s_cc_manager_b200 import _native as N  # noqa: E402

HOLD_MS = 1
SCENARIOS = {
    "inject": {"bytes": 0, "drill": {"scrub_inject": 4}, "triage": HOLD_MS},
    "flood": {"bytes": 0, "drill": {"scrub_flood": 0xC3}, "triage": HOLD_MS},
    "tag_flood": {"bytes": 0, "kind": "tagged", "drill": {"tag_flood": 0xC3}, "mismatch_triage": HOLD_MS},
    "clean": {"bytes": 0},
}
LOCATE_KERNELS = ("locate_dirt_kernel", "cover_locate_pass")


def one_gate(lib, name: str, prove: bool) -> dict:
    r = RCC.call(lib, dict(SCENARIOS[name], prove=int(prove)))
    want = 0 if name == "clean" else N.ERR_MISMATCH if name == "tag_flood" else N.ERR_DIRTY
    assert r["rc"] == want, (name, prove, r["rc"], r["error"])
    rc_ = r["report_cover"]
    assert rc_["proved"] == int(prove and name != "clean") and rc_["covered"] == rc_["proved"], (name, prove, rc_)
    t = r["times"]
    return {"ms": r["ms_verdict"], "ms_locate": t["ms_locate"],
            "ms_triage": t["ms_mismatch_triage"] if name == "tag_flood" else t["ms_triage"],
            "ms_prove": rc_["ms_prove"], "bytes_scrubbed": r["results"][0]["bytes_scrubbed"]}


def profile_locate(lib, calls: int) -> dict:
    """Per scenario and arming: the median over `calls` gates of the GPU time (ms) of the locate kernels in one call."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    out = {}
    for name in ("inject", "flood"):
        times = {"unproven": [], "proven": []}
        for _ in range(calls):
            for arm in times:
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    one_gate(lib, name, arm == "proven")
                kernel = LOCATE_KERNELS[arm == "proven"]
                times[arm].append(sum(e.device_time_total for e in prof.key_averages() if kernel in e.key) / 1e3)
        med = {arm: statistics.median(v) for arm, v in times.items()}
        out[name] = {**med, "proven_over_unproven": med["proven"] / med["unproven"] if med["unproven"] else None}
    out["calls"] = calls
    return out


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=9)
    ap.add_argument("--out", default=None)
    ap.add_argument("--profile-calls", type=int, default=3)
    a = ap.parse_args()
    lib = N.lib()
    assert lib.ccm_init(N.BACKEND_CUDASIM) == 0
    out = {"bench": "report_proof", **card(), "calls": a.calls, "triage_hold_ms": HOLD_MS}
    for name in SCENARIOS:
        runs = {"unproven": [], "proven": []}
        for i in range(1 + a.calls):
            for arm in runs:
                r = one_gate(lib, name, arm == "proven")
                if i:
                    runs[arm].append(r)
        out[name] = {arm: {"verdict_ms": stats([r["ms"] for r in rs]), "ms_locate": stats([r["ms_locate"] for r in rs]),
                           "ms_triage": stats([r["ms_triage"] for r in rs]), "ms_prove": stats([r["ms_prove"] for r in rs]),
                           "bytes_scrubbed": rs[-1]["bytes_scrubbed"]}
                     for arm, rs in runs.items()}
    if a.profile_calls:
        out["locate_kernels_ms"] = profile_locate(lib, a.profile_calls)
    line = json.dumps(out)
    print(line)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(line + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
