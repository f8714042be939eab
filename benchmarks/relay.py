#!/usr/bin/env python3
"""Cost and reach of the relayed whole-HBM gate on GPU 0: plain `ccm-scrub` whole-HBM runs alternated with
`ccm-scrub --relay` runs (DESIGN.md §5n), each a fresh process, after one warm-up round.  Prints ONE JSON line (and
writes it to --out when given).

  python benchmarks/relay.py [--runs 9] [--out FILE]

Per kind: the wall clock from starting the command to its JSON line and to its exit, the gate's own ms_total and
coverage (median, p10, p90, spread over --runs).  Per relay run: the relay's phase times (ms_first, ms_handover,
ms_settle, ms_second, settle_polls), footprint_a, freed, held and growth, both legs' unmappable bytes, the relay's
coverage and leg B's own.  The plain runs' total - device_free_before is the gate's own context footprint as its
process sees it.  This process creates no CUDA context.  The card's name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "benchmarks"))

from cover_proof import card, stats  # noqa: E402
from k8s_cc_manager_b200 import _native as N  # noqa: E402

CLI = ROOT / "k8s_cc_manager_b200" / "ccm-scrub"
RELAY_FIELDS = ("footprint_a", "freed", "held", "growth", "a_unreached", "b_unreached", "unreached", "coverage",
                "ms_first", "ms_handover", "ms_settle", "ms_second", "settle_polls", "settled")


def bdf0() -> str:
    lib = N.lib()
    assert lib.ccm_init(N.BACKEND_CUDASIM) == 0, N.last_error()
    n = C.c_int()
    lib.ccm_enumerate(None, 0, C.byref(n))
    infos = (N.DevInfo * max(n.value, 1))()
    lib.ccm_enumerate(infos, n.value, C.byref(n))
    return next(i.bdf.decode() for i in infos[:n.value] if i.cuda_ordinal == 0)


def one_run(bdf: str, relay: bool) -> dict:
    cmd = [str(CLI), *(["--relay"] if relay else []), "--bdf", bdf]
    t0 = time.perf_counter()
    proc = subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True,
                            env=dict(os.environ, CCM_BACKEND="cudasim"))
    line = ""
    for raw in proc.stdout:
        if raw.startswith("{"):
            line = raw
            t_line = time.perf_counter()
    err = proc.stderr.read()
    rc = proc.wait()
    t_exit = time.perf_counter()
    assert rc == 0 and line, (cmd, rc, err[-2000:])
    out = json.loads(line)
    rep = out["reports"][0]
    r = {"ms_to_line": (t_line - t0) * 1e3, "ms_to_exit": (t_exit - t0) * 1e3, "ms_total": rep["ms_total"],
         "coverage": rep["bytes_scrubbed"] / rep["device_total_bytes"],
         "footprint": rep["device_total_bytes"] - rep["device_free_before"], "bytes_unreached": rep["bytes_unreached"],
         "device_total_bytes": rep["device_total_bytes"]}
    if relay:
        r["relay"] = {k: rep["relay"][k] for k in RELAY_FIELDS}
        r["first_coverage"] = out["first"]["reports"][0]["bytes_scrubbed"] / rep["device_total_bytes"]
    return r


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=9)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    bdf = bdf0()
    out = {"bench": "relay", **card(), "bdf": bdf, "runs": a.runs}
    runs = {"plain": [], "relay": []}
    for i in range(1 + a.runs):
        for kind in ("plain", "relay"):
            r = one_run(bdf, kind == "relay")
            if i:
                runs[kind].append(r)
    for kind, rs in runs.items():
        out[kind] = {k: stats([r[k] for r in rs]) for k in ("ms_to_line", "ms_to_exit", "ms_total", "coverage",
                                                             "footprint", "bytes_unreached")}
        out[kind]["device_total_bytes"] = rs[-1]["device_total_bytes"]
    rel = runs["relay"]
    out["relay"]["fields"] = {k: stats([r["relay"][k] for r in rel]) for k in RELAY_FIELDS}
    out["relay"]["first_coverage"] = stats([r["first_coverage"] for r in rel])
    out["relay"]["each"] = [r["relay"] for r in rel]
    out["relay_minus_plain_ms_to_line"] = out["relay"]["ms_to_line"]["median"] - out["plain"]["ms_to_line"]["median"]
    line = json.dumps(out)
    print(line)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(line + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
