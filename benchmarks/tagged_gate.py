#!/usr/bin/env python3
"""Cost of the tagged scrub gate on GPU 0: its two kernels against same-run bars, and the cold whole-HBM
gate, zero against tagged.  Prints ONE JSON line (and writes it to --out when given).

  python benchmarks/tagged_gate.py [--calls 15] [--warmup 2] [--region-gib 32] [--out FILE]

kernels: tag_fill and tag_check_zero over a resident --region-gib region through the region entry points,
         against cudaMemsetAsync (ccm_region_scrub, variant memset) and a torch copy_ of half the region
         onto the other half, all timed with CUDA events in this run: best and median of --reps launches
         after one warm-up each.  Every check runs over freshly written tags (the fill before it is not timed).  Rates count the bytes each kernel must move: fill and memset write R,
         check and copy read and write (2R).
gate:    ccm_scrub_verify(0, 0) and ccm_scrub_verify_tagged(0, 0), alternating, --calls of each after
         --warmup of each.  `verdict_ms` is the call's own wall clock (time to verdict); `cycle_ms` adds the
         wait for its deferred HBM release, i.e. until the next call could start.  The gate runs before
         torch is imported, so no other allocation holds HBM in this process.
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


def pct(xs, q):
    xs = sorted(xs)
    return xs[min(len(xs) - 1, max(0, round(q * (len(xs) - 1))))]


def summary(xs):
    return {"median": statistics.median(xs), "p10": pct(xs, 0.1), "p90": pct(xs, 0.9)}


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True, check=True).stdout.strip().split(",")
    return {"gpu": q[0].strip(), "power_limit_w": float(q[1])}


def gate(lib, calls: int, warmup: int) -> dict:
    runs = {"zero": [], "tagged": []}
    for i in range(warmup + calls):
        for mode in ("zero", "tagged"):
            res, tag = N.ScrubResult(), N.TagResult()
            t0 = time.perf_counter()
            if mode == "zero":
                rc = lib.ccm_scrub_verify(0, 0, C.byref(res))
            else:
                rc = lib.ccm_scrub_verify_tagged(0, 0, C.byref(tag), C.byref(res))
            verdict = (time.perf_counter() - t0) * 1e3
            assert rc == 0, (mode, rc, N.last_error())
            assert lib.ccm_scrub_release_wait(0, None, None) == 0
            cycle = (time.perf_counter() - t0) * 1e3
            if i >= warmup:
                runs[mode].append({"verdict_ms": verdict, "cycle_ms": cycle, "ms_acquire": res.ms_acquire,
                                   "ms_gpu_span": res.ms_gpu_span, "ms_scrub": res.ms_scrub,
                                   "ms_verify": res.ms_verify, "ms_tag": tag.ms_tag, "ms_check": tag.ms_check,
                                   "bytes_scrubbed": res.bytes_scrubbed})
    out = {}
    for mode, rs in runs.items():
        out[mode] = {k: summary([r[k] for r in rs]) for k in rs[0] if k != "bytes_scrubbed"}
        out[mode]["bytes_scrubbed"] = summary([r["bytes_scrubbed"] for r in rs])["median"]
        out[mode]["calls"] = len(rs)
    out["added_verdict_ms"] = out["tagged"]["verdict_ms"]["median"] - out["zero"]["verdict_ms"]["median"]
    return out


def kernels(lib, region_gib: int, reps: int) -> dict:
    import torch
    n = region_gib << 30
    buf = torch.empty(n, dtype=torch.uint8, device="cuda")
    p = C.c_void_p(buf.data_ptr())
    # a stream of our own: the default stream's handle is NULL, which the library reads as "its own stream"
    # (not ordered with torch's events)
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    st = C.c_void_p(stream.cuda_stream)
    half = n // 2
    src, dst = buf[:half], buf[half:]

    def timed(fn, before=None):
        ts = []
        for _ in range(reps + 1):
            if before is not None:
                before()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            rc = fn()
            b.record()
            b.synchronize()
            assert not isinstance(rc, int) or rc == 0, N.last_error()
            ts.append(a.elapsed_time(b))
        return ts[1:]                                     # the first launch is the warm-up

    t = {
        "memset": timed(lambda: lib.ccm_region_scrub(0, p, n, N.SCRUB_MEMSET, None, st, None)),
        "tag_fill": timed(lambda: lib.ccm_region_tag_fill(0, p, n, 7, st, None)),
        # the region is tagged again (untimed) before every check: a check over matching tags is the gate's case
        "tag_check_zero": timed(lambda: lib.ccm_region_tag_check_zero(0, p, n, 7, st, None, None),
                                before=lambda: lib.ccm_region_tag_fill(0, p, n, 7, st, None)),
        "copy": timed(lambda: dst.copy_(src)),
    }
    moved = {"memset": n, "tag_fill": n, "tag_check_zero": 2 * n, "copy": 2 * half}
    out = {"region_bytes": n, "reps": reps}
    for k, ts in t.items():
        out[k] = {"ms_best": min(ts), "ms_median": statistics.median(ts),
                  "gbs_best": moved[k] / min(ts) / 1e6, "gbs_median": moved[k] / statistics.median(ts) / 1e6}
    out["fill_vs_memset"] = out["tag_fill"]["gbs_best"] / out["memset"]["gbs_best"]
    out["check_vs_copy"] = out["tag_check_zero"]["gbs_best"] / out["copy"]["gbs_best"]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=15)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--region-gib", type=int, default=32)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    lib = N.lib()
    assert lib.ccm_init(N.BACKEND_CUDASIM) == 0, N.last_error()
    result = {**card(), "gate": gate(lib, args.calls, args.warmup), "kernels": kernels(lib, args.region_gib, args.reps)}
    line = json.dumps(result)
    print(line, flush=True)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
