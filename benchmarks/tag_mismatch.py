#!/usr/bin/env python3
"""Cost of the mismatch report on GPU 0.  Prints ONE JSON line (and writes it to --out when given).

  python benchmarks/tag_mismatch.py [--parent-lib OLD/libccm.so] [--calls 3] [--reps 10] [--out FILE]

gate:    cold whole-HBM tagged gates to the verdict (ccm_scrub_verify_tagged(0, 0)), clean and with scrub_alias = 1,
         alternating, --calls of each after one warm-up of each; medians of the call's own wall clock.  Runs before
         torch is imported.
kernel:  ccm_region_tag_check_locate over a resident 16 GiB region, clean, with one mismatched byte every 32 MiB
         (sparse) and with every byte mismatched (flood, another seed's tags), each against a same-run
         device-to-device copy of 8 GiB into 8 GiB (R = 16 GiB read + written by both); CUDA events, best of --reps.
parent:  with --parent-lib (a libccm.so built from the parent commit), ccm_region_tag_check_zero over a resident
         32 GiB region, this build and the parent's alternating launch by launch, best of --reps each, and the same
         for two rounds of the parent (the run-to-run spread).
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

GiB, MiB = 1 << 30, 1 << 20


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True, check=True).stdout.strip().split(",")
    return {"gpu": q[0].strip(), "power_limit_w": float(q[1])}


def gate(lib, calls: int) -> dict:
    runs = {"clean": [], "alias": []}
    for i in range(1 + calls):
        for mode in ("clean", "alias"):
            assert lib.ccm_sim_set(0, b"scrub_alias", 1 if mode == "alias" else 0) == 0
            tag, res = N.TagResult(), N.ScrubResult()
            t0 = time.perf_counter()
            rc = lib.ccm_scrub_verify_tagged(0, 0, C.byref(tag), C.byref(res))
            ms = (time.perf_counter() - t0) * 1e3
            assert rc == (N.ERR_MISMATCH if mode == "alias" else 0), (mode, rc, N.last_error())
            m = N.MismatchReport()
            lib.ccm_scrub_last_mismatch(0, C.byref(m))
            assert bool(m.located) == (mode == "alias")
            lib.ccm_scrub_release_wait(0, None, None)
            if i:
                runs[mode].append({"verdict_ms": ms, "ms_check": tag.ms_check, "bytes": res.bytes_scrubbed,
                                   "mismatch_windows": m.mismatch_windows})
    lib.ccm_sim_set(0, b"scrub_alias", 0)
    return {mode: {"verdict_ms_median": statistics.median(r["verdict_ms"] for r in rs),
                   "ms_check_median": statistics.median(r["ms_check"] for r in rs),
                   "bytes": rs[0]["bytes"], "mismatch_windows": rs[0]["mismatch_windows"], "calls": len(rs)}
            for mode, rs in runs.items()}


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent-lib", default=None)
    ap.add_argument("--calls", type=int, default=3)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    lib = N.lib()
    assert lib.ccm_init(N.BACKEND_CUDASIM) == 0
    out = {"bench": "tag_mismatch", **card(), "gate": gate(lib, a.calls)}

    import torch
    st = torch.cuda.Stream()

    def timed(fn, prep=None, reps=a.reps):
        ts = []
        for _ in range(max(reps, 0) + 1):
            if prep:
                prep()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            fn()
            e1.record(st)
            e1.synchronize()
            ts.append(e0.elapsed_time(e1))
        return min(ts[1:]) if reps > 0 else ts[0]

    with torch.cuda.stream(st):
        sp = C.c_void_p(st.cuda_stream)
        n = 16 * GiB
        buf = torch.empty(n, dtype=torch.uint8, device="cuda")
        p, seed = buf.data_ptr(), 0xA11CE
        half = n // 2
        t_copy = timed(lambda: buf[half:].copy_(buf[:half]))
        m = N.MismatchReport()

        def fill(s):
            assert lib.ccm_region_tag_fill(0, C.c_void_p(p), n, s, sp, None) == 0

        def sparse():
            fill(seed)
            buf[torch.arange(0, n, 32 * MiB, device="cuda")] ^= 0xA5

        run = lambda: lib.ccm_region_tag_check_locate(0, C.c_void_p(p), n, seed, sp, C.byref(m))  # noqa: E731
        kern = {"region_bytes": n, "copy_gbs_read_write": n / t_copy / 1e6}   # 8 GiB read + 8 GiB written
        for name, prep in (("clean", lambda: fill(seed)), ("sparse", sparse), ("flood", lambda: fill(seed ^ 0x5A5A5A5A))):
            t = timed(run, prep)
            kern[name] = {"ms": t, "gbs_read": n / t / 1e6, "gbs_read_write": 2 * n / t / 1e6,
                          "vs_copy": (2 * n / t / 1e6) / (n / t_copy / 1e6), "mismatch_bytes": m.mismatch_bytes,
                          "mismatch_windows": m.mismatch_windows}
        for name in ("sparse", "flood"):
            kern[name]["vs_clean"] = kern["clean"]["ms"] / kern[name]["ms"]
        out["kernel"] = kern
        del buf
        torch.cuda.empty_cache()

        if a.parent_lib:
            old = C.CDLL(a.parent_lib, mode=C.RTLD_LOCAL)
            for L in (old,):
                L.ccm_region_tag_check_zero.argtypes = [C.c_int, C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p,
                                                        C.POINTER(C.c_uint64), C.POINTER(C.c_float)]
                L.ccm_region_tag_fill.argtypes = [C.c_int, C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p,
                                                  C.POINTER(C.c_float)]
            n = 32 * GiB
            buf = torch.empty(n, dtype=torch.uint8, device="cuda")
            p = buf.data_ptr()
            mm = C.c_uint64()
            libs = {"change": lib, "parent": old}
            order = ("change", "parent", "parent_again")
            ts = {k: [] for k in order}
            for _ in range(a.reps + 1):
                for k in order:
                    L = libs["parent" if k.startswith("parent") else k]
                    ts[k].append(timed(lambda: L.ccm_region_tag_check_zero(0, C.c_void_p(p), n, seed, sp, C.byref(mm),
                                                                           None),
                                       lambda: lib.ccm_region_tag_fill(0, C.c_void_p(p), n, seed, sp, None), reps=0))
                    assert mm.value == 0
            best = {k: min(v[1:]) for k, v in ts.items()}   # the first round is a warm-up
            out["parent_vs_change_32gib"] = {
                "best_ms": best, "gbs_read": {k: n / v / 1e6 for k, v in best.items()},
                "change_over_parent": best["parent"] / best["change"],
                "parent_spread": best["parent"] / best["parent_again"]}
    line = json.dumps(out)
    print(line)
    if a.out:
        Path(a.out).write_text(line + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
