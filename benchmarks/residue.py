#!/usr/bin/env python3
"""Cost and first findings of the residue census on GPU 0.  Prints ONE JSON line (and writes it to --out when given).

  python benchmarks/residue.py [--calls 5] [--reps 10] [--out FILE]

handback: the FIRST call of this process is a whole-HBM zero gate with the census (ccm_scrub_verify_residue(0, 0)):
          what the driver handed back to a fresh process, before anything of this process wrote HBM.  Counts, extent
          and chunks only; the census reports no bytes.
gate:     cold whole-HBM gates of four kinds alternating (zero, zero + census, tagged, tagged + census), one warm-up
          round, then --calls of each; medians of the call's own wall clock (time to verdict), ms_scrub, ms_verify and
          ms_tag.  `census_cost_ms` is the zero + census median minus the zero median, against the zero gate's median
          ms_verify (one read of the mapping).  Runs before torch is imported.
kernel:   ccm_region_census over a resident 16 GiB region, storing zeros and storing tags, clean, with one non-zero
          byte every 32 MiB (sparse) and with every byte non-zero, against a same-run device-to-device copy of 8 GiB
          into 8 GiB and a same-run ccm_region_tag_check_zero of the 16 GiB (R = 16 GiB read + written by all);
          CUDA events, best of --reps.
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
from k8s_cc_manager_b200 import devices as D  # noqa: E402

GiB, MiB = 1 << 30, 1 << 20
KINDS = ("zero", "zero_census", "tagged", "tagged_census")


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True, check=True).stdout.strip().split(",")
    return {"gpu": q[0].strip(), "power_limit_w": float(q[1])}


def one_gate(lib, kind: str) -> dict:
    tagged, census = kind.startswith("tagged"), kind.endswith("census")
    tag, res, rr = N.TagResult(), N.ScrubResult(), N.ResidueReport()
    t0 = time.perf_counter()
    if census:
        rc = lib.ccm_scrub_verify_residue(0, 0, C.byref(tag) if tagged else None, C.byref(rr), C.byref(res))
    elif tagged:
        rc = lib.ccm_scrub_verify_tagged(0, 0, C.byref(tag), C.byref(res))
    else:
        rc = lib.ccm_scrub_verify(0, 0, C.byref(res))
    ms = (time.perf_counter() - t0) * 1e3
    assert rc == 0, (kind, rc, N.last_error())
    lib.ccm_scrub_release_wait(0, None, None)
    out = {"verdict_ms": ms, "ms_scrub": res.ms_scrub, "ms_verify": res.ms_verify, "ms_tag": tag.ms_tag if tagged else 0.0,
           "bytes": res.bytes_scrubbed}
    if census:
        out["residue"] = D.ResidueReport.from_native(rr)
    return out


def residue_json(r: D.ResidueReport) -> dict:
    return {"residue_bytes": r.residue_bytes, "residue_windows": r.residue_windows, "first_offset": r.first_offset,
            "last_offset": r.last_offset, "bytes_examined": r.bytes_examined, "truncated": r.truncated,
            "chunks": r.chunks, "summary": r.summary()}


def gate(lib, calls: int) -> dict:
    runs = {k: [] for k in KINDS}
    for i in range(1 + calls):
        for kind in KINDS:
            g = one_gate(lib, kind)
            if i:
                runs[kind].append(g)
    med = {k: {f: statistics.median(r[f] for r in rs) for f in ("verdict_ms", "ms_scrub", "ms_verify", "ms_tag")}
           for k, rs in runs.items()}
    for k, rs in runs.items():
        med[k]["bytes"] = rs[0]["bytes"]
        med[k]["calls"] = len(rs)
        if k.endswith("census"):
            med[k]["residue_bytes"] = [r["residue"].residue_bytes for r in rs]
    cost = med["zero_census"]["verdict_ms"] - med["zero"]["verdict_ms"]
    med["census_cost_ms"] = cost
    med["bound_ms_verify"] = med["zero"]["ms_verify"]
    med["within_bound"] = cost <= med["zero"]["ms_verify"]
    return med


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    lib = N.lib()
    assert lib.ccm_init(N.BACKEND_CUDASIM) == 0
    first = one_gate(lib, "zero_census")                     # nothing of this process has written HBM yet
    out = {"bench": "residue", **card(),
           "handback": {"first_call": True, "bytes_scrubbed": first["bytes"], **residue_json(first["residue"])},
           "gate": gate(lib, a.calls)}

    import torch
    st = torch.cuda.Stream()

    def timed(fn, prep=None, reps=a.reps):
        ts = []
        for _ in range(reps + 1):
            if prep:
                prep()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            fn()
            e1.record(st)
            e1.synchronize()
            ts.append(e0.elapsed_time(e1))
        return min(ts[1:])

    with torch.cuda.stream(st):
        sp = C.c_void_p(st.cuda_stream)
        n = 16 * GiB
        buf = torch.empty(n, dtype=torch.uint8, device="cuda")
        p, seed = buf.data_ptr(), 0xA11CE
        half = n // 2
        t_copy = timed(lambda: buf[half:].copy_(buf[:half]))
        mm = C.c_uint64()
        t_check = timed(lambda: lib.ccm_region_tag_check_zero(0, C.c_void_p(p), n, seed, sp, C.byref(mm), None),
                        lambda: lib.ccm_region_tag_fill(0, C.c_void_p(p), n, seed, sp, None))
        assert mm.value == 0
        kern = {"region_bytes": n, "copy_gbs_read_write": n / t_copy / 1e6,
                "tag_check_zero_gbs_read_write": 2 * n / t_check / 1e6}
        rr = N.ResidueReport()

        def sparse():
            buf.zero_()
            buf[torch.arange(0, n, 32 * MiB, device="cuda")] = 0xA5

        for tags in (0, 1):
            for name, prep in (("clean", buf.zero_), ("sparse", sparse), ("every_byte", lambda: buf.fill_(0x5A))):
                t = timed(lambda: lib.ccm_region_census(0, C.c_void_p(p), n, tags, seed, sp, C.byref(rr)), prep)
                gbs = 2 * n / t / 1e6
                kern[f"{'tags' if tags else 'zero'}_{name}"] = {
                    "ms": t, "gbs_read_write": gbs, "vs_copy": gbs / kern["copy_gbs_read_write"],
                    "vs_tag_check_zero": gbs / kern["tag_check_zero_gbs_read_write"],
                    "residue_bytes": rr.residue_bytes, "residue_windows": rr.residue_windows}
        out["kernel"] = kern
        del buf
        torch.cuda.empty_cache()
    line = json.dumps(out)
    print(line)
    if a.out:
        Path(a.out).write_text(line + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
