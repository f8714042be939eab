#!/usr/bin/env python3
"""Cost of the alias probe on GPU 0, in one process.  Prints ONE JSON line (and writes it to --out when given).

  python benchmarks/alias_probe.py [--calls 9] [--region-gib 16] [--out FILE]

Region: P1+P2+P3 of ccm_region_probe over a resident region (its CUDA-event ms_probe), against a same-run
ccm_region_tag_check_zero over the region holding its tags (ccm_region_tag_fill with the same seed first, untimed; the
check must count 0) and ccm_region_verify (the zero read-back, which must count 0), alternated, median of five after one
warm-up round.
Cold gates: whole-HBM zero gates, zero gates with the probe armed, and tagged gates, alternated call by call after one
warm-up round, --calls each: the call's own wall clock to the verdict (median, p10, p90 and spread) and, armed, the
medians of ms_probe and of the probe's windows.  The card's name and power limit are read in the same run.
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


def stats(xs: list) -> dict:
    xs = sorted(xs)
    q = statistics.quantiles(xs, n=10) if len(xs) > 1 else [xs[0]] * 9
    return {"median": statistics.median(xs), "p10": q[0], "p90": q[-1], "spread": xs[-1] - xs[0], "n": len(xs)}


def region(lib, gib: int) -> dict:
    import torch
    n = gib << 30
    buf = torch.zeros(n, dtype=torch.uint8, device="cuda")
    ptr = buf.data_ptr()
    torch.cuda.synchronize()
    probe, check, verify = [], [], []
    for i in range(6):
        rep = N.ProbeReport()
        assert lib.ccm_region_probe(0, ptr, n, 7 + i, None, C.byref(rep), None) == 0, N.last_error()
        assert rep.mismatch_bytes == 0 and rep.reread_nonzero_bytes == 0
        # the check runs over memory that holds its tags, as in the tagged gate: its clean path, not its booking branch
        assert lib.ccm_region_tag_fill(0, ptr, n, 7 + i, None, None) == 0, N.last_error()
        ms, count = C.c_float(), C.c_uint64()
        assert lib.ccm_region_tag_check_zero(0, ptr, n, 7 + i, None, C.byref(count), C.byref(ms)) == 0, N.last_error()
        assert count.value == 0, count.value
        vms, nz = C.c_float(), C.c_uint64()
        assert lib.ccm_region_verify(0, ptr, n, N.VERIFY_AUTO, None, None, C.byref(nz), C.byref(vms)) == 0
        assert nz.value == 0, nz.value
        if i:
            probe.append(rep.ms_probe)
            check.append(ms.value)
            verify.append(vms.value)
    del buf
    torch.cuda.empty_cache()
    med = statistics.median
    return {"bytes": n, "windows": rep.windows, "probe_ms": stats(probe), "tag_check_zero_ms": stats(check),
            "readback_ms": stats(verify), "probe_over_tag_check": med(probe) / med(check),
            "probe_over_readback": med(probe) / med(verify),
            "probe_windows_per_s": rep.windows * 3 / (med(probe) / 1e3)}


def one_gate(lib, kind: str) -> dict:
    assert lib.ccm_scrub_probe(0, int(kind == "zero_probe")) == 0, N.last_error()
    res, tag = N.ScrubResult(), N.TagResult()
    try:
        t0 = time.perf_counter()
        rc = lib.ccm_scrub_verify_tagged(0, 0, C.byref(tag), C.byref(res)) if kind == "tagged" else \
            lib.ccm_scrub_verify(0, 0, C.byref(res))
        ms = (time.perf_counter() - t0) * 1e3
    finally:
        lib.ccm_scrub_probe(0, 0)
    assert rc == 0, (kind, rc, N.last_error())
    p = N.ProbeReport()
    assert lib.ccm_scrub_last_probe(0, C.byref(p)) == 0
    assert p.probed == int(kind == "zero_probe")
    lib.ccm_scrub_release_wait(0, None, None)
    return {"ms": ms, "ms_probe": p.ms_probe, "windows": p.windows, "bytes_scrubbed": res.bytes_scrubbed}


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=9)
    ap.add_argument("--region-gib", type=int, default=16)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    lib = N.lib()
    assert lib.ccm_init(N.BACKEND_CUDASIM) == 0
    out = {"bench": "alias_probe", **card(), "calls": a.calls}
    out["region"] = region(lib, a.region_gib)
    kinds = ("zero", "zero_probe", "tagged")
    runs = {k: [] for k in kinds}
    for i in range(1 + a.calls):
        for k in kinds:
            r = one_gate(lib, k)
            if i:
                runs[k].append(r)
    med = statistics.median
    out["gates"] = {k: {"verdict_ms": stats([r["ms"] for r in rs]), "bytes_scrubbed": rs[-1]["bytes_scrubbed"],
                        **({"ms_probe": stats([r["ms_probe"] for r in rs]), "windows": rs[-1]["windows"]}
                           if k == "zero_probe" else {})}
                    for k, rs in runs.items()}
    g = out["gates"]
    out["probe_minus_zero_verdict_ms"] = g["zero_probe"]["verdict_ms"]["median"] - g["zero"]["verdict_ms"]["median"]
    out["tagged_minus_zero_verdict_ms"] = g["tagged"]["verdict_ms"]["median"] - g["zero"]["verdict_ms"]["median"]
    line = json.dumps(out)
    print(line)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(line + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
