#!/usr/bin/env python3
"""Cost of the page maps on GPU 0: this tree's libccm.so against a build of the parent commit, in one process, the two
alternated call by call.  Prints ONE JSON line (and writes it to --out when given).

  python benchmarks/page_map.py --parent-lib PATH [--calls 5] [--reps 15] [--out FILE]

gate:    cold whole-HBM gates to the verdict (the call's own wall clock, median of --calls after one warm-up round):
         the zero gate clean, the zero gate with 4 injected bytes (its locate pass runs), and the census call over
         memory that is entirely residue (scrub_poison).  Runs before torch is imported.
kernel:  each book's pass over a resident --gib GiB region (locate; tag check; census storing zeros; census storing
         tags), clean, with one booked byte every 32 MiB (sparse) and with every byte booked (flood); CUDA events around
         each region call (ccm_region_locate / _tag_check_locate / _census: the launch and the host's read of the book),
         median of --reps; `ratio` is this tree's rate over the parent's (> 1: faster).  Every region call's counts are
         compared between the two builds.
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
GATES = {"zero_clean": ("zero", {}), "zero_inject4": ("zero", {"scrub_inject": 4}),
         "census_all_residue": ("census", {"scrub_poison": 0x5A})}
DRILLS = ("scrub_inject", "scrub_poison")


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True, check=True).stdout.strip().split(",")
    return {"gpu": q[0].strip(), "power_limit_w": float(q[1])}


def open_lib(path: str):
    lib = C.CDLL(path, mode=C.RTLD_LOCAL)
    for name, (restype, argtypes) in N._SIGNATURES.items():
        fn = getattr(lib, name, None)
        if fn is not None:
            fn.restype, fn.argtypes = restype, argtypes
    assert lib.ccm_init(N.BACKEND_CUDASIM) == 0
    return lib


def one_gate(lib, kind: str) -> tuple[float, int]:
    call, drills = GATES[kind]
    for k in DRILLS:
        assert lib.ccm_sim_set(0, k.encode(), int(drills.get(k, 0))) == 0
    res, rr = N.ScrubResult(), N.ResidueReport()
    t0 = time.perf_counter()
    if call == "census":
        rc = lib.ccm_scrub_verify_residue(0, 0, None, C.byref(rr), C.byref(res))
    else:
        rc = lib.ccm_scrub_verify(0, 0, C.byref(res))
    ms = (time.perf_counter() - t0) * 1e3
    for k in DRILLS:
        lib.ccm_sim_set(0, k.encode(), 0)
    assert rc == (N.ERR_DIRTY if drills.get("scrub_inject") else 0), (kind, rc)
    lib.ccm_scrub_release_wait(0, None, None)
    return ms, res.nonzero_bytes + rr.residue_bytes


def gates(libs: dict, calls: int) -> dict:
    runs = {(k, name): [] for k in GATES for name in libs}
    for i in range(1 + calls):
        for kind in GATES:
            for name, lib in libs.items():
                ms, _ = one_gate(lib, kind)
                if i:
                    runs[kind, name].append(ms)
    out = {}
    for kind in GATES:
        new, old = runs[kind, "new"], runs[kind, "parent"]
        out[kind] = {"new_ms_median": statistics.median(new), "parent_ms_median": statistics.median(old),
                     "new_ms": new, "parent_ms": old,
                     "spread_ms": max(max(new) - min(new), max(old) - min(old)),
                     "ratio_parent_over_new": statistics.median(old) / statistics.median(new)}
    return out


def kernels(libs: dict, gib: int, reps: int) -> dict:
    import torch
    st = torch.cuda.Stream()
    n = gib * GiB
    seed = 0xA11CE
    out = {"region_bytes": n}
    with torch.cuda.stream(st):
        sp = C.c_void_p(st.cuda_stream)
        buf = torch.empty(n, dtype=torch.uint8, device="cuda")
        p = C.c_void_p(buf.data_ptr())
        fill = libs["new"]

        def content(kind: str, what: str):
            """Puts the region in the state the pass `kind` books `what` from."""
            if kind == "check":
                assert fill.ccm_region_tag_fill(0, p, n, seed, sp, None) == 0
                if what == "sparse":
                    buf[torch.arange(0, n, 32 * MiB, device="cuda")] ^= 0xA5
                elif what == "flood":
                    buf.bitwise_not_()
            elif what == "clean":
                buf.zero_()
            elif what == "sparse":
                buf.zero_()
                buf[torch.arange(0, n, 32 * MiB, device="cuda")] = 0xA5
            else:
                buf.fill_(0x5A)

        def run(lib, kind: str) -> int:
            if kind == "locate":
                d = N.DirtReport()
                assert lib.ccm_region_locate(0, p, n, sp, C.byref(d)) == 0
                return d.nonzero_bytes
            if kind == "check":
                m = N.MismatchReport()
                assert lib.ccm_region_tag_check_locate(0, p, n, seed, sp, C.byref(m)) == 0
                return m.mismatch_bytes
            r = N.ResidueReport()
            assert lib.ccm_region_census(0, p, n, int(kind == "census_tags"), seed, sp, C.byref(r)) == 0
            return r.residue_bytes

        for kind in ("locate", "check", "census_zero", "census_tags"):
            for what in ("clean", "sparse", "flood"):
                times = {name: [] for name in libs}
                counts = {name: set() for name in libs}
                if kind == "locate":
                    content(kind, what)                # the locate pass writes nothing: one content for all
                for i in range(reps + 1):
                    for name, lib in libs.items():
                        if kind != "locate":
                            content(kind, what)
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record(st)
                        counts[name].add(run(lib, kind))
                        e1.record(st)
                        e1.synchronize()
                        if i:
                            times[name].append(e0.elapsed_time(e1))
                assert counts["new"] == counts["parent"] and len(counts["new"]) == 1, (kind, what, counts)
                rw = 1 if kind == "locate" else 2
                gbs = {name: rw * n / statistics.median(ts) / 1e6 for name, ts in times.items()}
                out[f"{kind}_{what}"] = {"booked_bytes": counts["new"].pop(), "new_gbs": gbs["new"],
                                         "parent_gbs": gbs["parent"], "ratio": gbs["new"] / gbs["parent"],
                                         "new_ms_median": statistics.median(times["new"]),
                                         "parent_ms_median": statistics.median(times["parent"]),
                                         "spread_ms": max(max(ts) - min(ts) for ts in times.values())}
        del buf
        torch.cuda.empty_cache()
    return out


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent-lib", required=True, help="libccm.so built from the parent commit")
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--gib", type=int, default=16)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    libs = {"new": open_lib(str(N.LIB_PATH)), "parent": open_lib(a.parent_lib)}
    out = {"bench": "page_map", **card(), "gate": gates(libs, a.calls), "kernel": kernels(libs, a.gib, a.reps)}
    line = json.dumps(out)
    print(line)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(line + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
