#!/usr/bin/env python3
"""Cost of the probe proof on GPU 0: cold whole-HBM zero gates with the alias probe, proven (ccm_scrub_prove) and
unproven, alternated call by call in one process after one warm-up round.  Prints ONE JSON line (and writes it to
--out when given).

  python benchmarks/probe_proof.py [--calls 9] [--out FILE]

Per arming: the call's own wall clock to the verdict, ms_probe and (proven) the probe proof's ms_prove, each as median,
p10, p90 and spread over --calls; the probe's windows and the warp atomics the twins issue per step (one per 32
windows).  Then, in a run of its own under torch.profiler, --profile-calls more gates of each arming, alternated:
the GPU time of each probe step's kernels alone (the plain `alias_probe_*_pass` against the proving
`cover_probe_*_pass`), summed over the call's launches, so the twins' cost is read apart from the passes before the
probe.  The card's name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import statistics
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parent))

from cover_proof import card, stats  # noqa: E402
from k8s_cc_manager_b200 import _native as N  # noqa: E402


def one_gate(lib, prove: bool) -> dict:
    assert lib.ccm_scrub_prove(0, int(prove)) == 0, N.last_error()
    assert lib.ccm_scrub_probe(0, 1) == 0, N.last_error()
    res = N.ScrubResult()
    try:
        t0 = time.perf_counter()
        rc = lib.ccm_scrub_verify(0, 0, C.byref(res))
        ms = (time.perf_counter() - t0) * 1e3
    finally:
        lib.ccm_scrub_prove(0, 0)
        lib.ccm_scrub_probe(0, 0)
    assert rc == 0, (prove, rc, N.last_error())
    probe, pc = N.ProbeReport(), N.ProbeCover()
    assert lib.ccm_scrub_last_probe(0, C.byref(probe)) == 0 and probe.probed == 1
    assert lib.ccm_scrub_last_probe_cover(0, C.byref(pc)) == 0
    assert pc.proved == int(prove) and pc.covered == int(prove)
    lib.ccm_scrub_release_wait(0, None, None)
    return {"ms": ms, "ms_probe": probe.ms_probe, "ms_prove": pc.ms_prove, "windows": probe.windows,
            "bytes_scrubbed": res.bytes_scrubbed}


STEP_KERNELS = {"P1": ("alias_probe_fill_pass", "cover_probe_fill_pass"),
                "P2": ("alias_probe_check_pass", "cover_probe_check_pass"),
                "P3": ("alias_probe_reread_pass", "cover_probe_reread_pass")}


def profile_steps(lib, calls: int) -> dict:
    """Per step and arming: the median over `calls` gates of the GPU time (ms) of that step's kernels in one call."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    times = {arm: {step: [] for step in STEP_KERNELS} for arm in ("unproven", "proven")}
    for _ in range(calls):
        for arm in ("unproven", "proven"):
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                one_gate(lib, arm == "proven")
            for step, names in STEP_KERNELS.items():
                name = names[arm == "proven"]
                us = sum(e.device_time_total for e in prof.key_averages() if name in e.key)
                times[arm][step].append(us / 1e3)
    out = {arm: {step: statistics.median(v) for step, v in steps.items()} for arm, steps in times.items()}
    out["proven_over_unproven"] = {step: out["proven"][step] / out["unproven"][step]
                                   for step in STEP_KERNELS if out["unproven"][step]}
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
    out = {"bench": "probe_proof", **card(), "calls": a.calls}
    runs = {"unproven": [], "proven": []}
    for i in range(1 + a.calls):
        for name in ("unproven", "proven"):
            r = one_gate(lib, name == "proven")
            if i:
                runs[name].append(r)
    for name, rs in runs.items():
        out[name] = {"verdict_ms": stats([r["ms"] for r in rs]), "ms_probe": stats([r["ms_probe"] for r in rs]),
                     "ms_prove": stats([r["ms_prove"] for r in rs]), "windows": rs[-1]["windows"],
                     "bytes_scrubbed": rs[-1]["bytes_scrubbed"]}
    out["warp_atomics_per_step"] = -(-out["proven"]["windows"] // 32)
    out["ms_probe_proven_over_unproven"] = out["proven"]["ms_probe"]["median"] / out["unproven"]["ms_probe"]["median"]
    out["proven_minus_unproven_verdict_ms"] = (out["proven"]["verdict_ms"]["median"]
                                               - out["unproven"]["verdict_ms"]["median"])
    if a.profile_calls:
        out["step_kernels_ms"] = profile_steps(lib, a.profile_calls)
    line = json.dumps(out)
    print(line)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(line + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
