#!/usr/bin/env python3
"""Cost of the dirt report on GPU 0: the locate kernel against a same-run read-back, and what a failed whole-HBM
gate pays for it.  Prints ONE JSON line (and writes it to --out when given).

  python benchmarks/locate_dirt.py [--calls 5] [--region-gib 32] [--reps 10] [--out FILE]

kernel: ccm_region_locate against ccm_region_verify (verify_ld128_fast_kernel) over a resident --region-gib region,
        with sparse dirt (one byte every ~32 MiB) and with every byte non-zero, timed with CUDA events in this run:
        best and median of --reps launches after one warm-up.  Both read R.
gate:   ccm_scrub_verify(0, 0), clean against scrub_inject = 4 (a failed gate, which runs the locate pass before it
        hands the memory back), alternating, --calls of each after one warm-up of each.  `verdict_ms` is the call's
        own wall clock; `ms_locate` the locate kernel's CUDA-event time.  The gate runs before torch is imported.
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


def gate(lib, calls: int) -> dict:
    runs = {"clean": [], "dirty": []}
    for i in range(1 + calls):
        for mode in ("clean", "dirty"):
            assert lib.ccm_sim_set(0, b"scrub_inject", 4 if mode == "dirty" else 0) == 0
            res, dirt = N.ScrubResult(), N.DirtReport()
            t0 = time.perf_counter()
            rc = lib.ccm_scrub_verify(0, 0, C.byref(res))
            verdict = (time.perf_counter() - t0) * 1e3
            assert rc == (N.ERR_DIRTY if mode == "dirty" else 0), (mode, rc, N.last_error())
            assert lib.ccm_scrub_last_dirt(0, C.byref(dirt)) == 0
            assert dirt.located == (mode == "dirty") and dirt.dirty_windows == res.nonzero_bytes
            assert lib.ccm_scrub_release_wait(0, None, None) == 0
            if i:
                runs[mode].append({"verdict_ms": verdict, "ms_locate": dirt.ms_locate, "bytes": res.bytes_scrubbed})
    lib.ccm_sim_set(0, b"scrub_inject", 0)
    out = {}
    for mode, rs in runs.items():
        out[mode] = {"verdict_ms_median": statistics.median(r["verdict_ms"] for r in rs),
                     "verdict_ms_best": min(r["verdict_ms"] for r in rs),
                     "ms_locate_median": statistics.median(r["ms_locate"] for r in rs),
                     "bytes_scrubbed": rs[0]["bytes"], "calls": len(rs)}
    out["dirty"]["locate_gbs"] = out["dirty"]["bytes_scrubbed"] / out["dirty"]["ms_locate_median"] / 1e6
    out["added_verdict_ms"] = out["dirty"]["verdict_ms_median"] - out["clean"]["verdict_ms_median"]
    return out


def kernels(lib, region_gib: int, reps: int) -> dict:
    import torch
    n = region_gib << 30
    buf = torch.zeros(n, dtype=torch.uint8, device="cuda")
    p = C.c_void_p(buf.data_ptr())
    stream = torch.cuda.Stream()   # the default stream's handle is NULL, which the library reads as its own stream
    torch.cuda.set_stream(stream)
    st = C.c_void_p(stream.cuda_stream)
    d = N.DirtReport()

    def timed(fn):
        ts = []
        for _ in range(reps + 1):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            rc = fn()
            b.record()
            b.synchronize()
            assert rc == 0, N.last_error()
            ts.append(a.elapsed_time(b))
        return ts[1:]

    out = {"region_bytes": n, "reps": reps}
    for dirt in ("sparse", "every_byte"):
        if dirt == "sparse":
            buf[torch.arange(0, n, 32 << 20, device="cuda")] = 0x5A
        else:
            buf.fill_(0x5A)
        torch.cuda.synchronize()
        t = {"verify": timed(lambda: lib.ccm_region_verify(0, p, n, N.VERIFY_AUTO, None, st, None, None)),
             "locate": timed(lambda: lib.ccm_region_locate(0, p, n, st, C.byref(d)))}
        row = {k: {"ms_best": min(ts), "ms_median": statistics.median(ts), "gbs_best": n / min(ts) / 1e6}
               for k, ts in t.items()}
        row["locate_vs_verify"] = row["locate"]["gbs_best"] / row["verify"]["gbs_best"]
        row["dirty_windows"] = d.dirty_windows
        out[dirt] = row
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--region-gib", type=int, default=32)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    lib = N.lib()
    assert lib.ccm_init(N.BACKEND_CUDASIM) == 0, N.last_error()
    result = {**card(), "gate": gate(lib, args.calls), "kernels": kernels(lib, args.region_gib, args.reps)}
    line = json.dumps(result)
    print(line, flush=True)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
