#!/usr/bin/env python3
"""Cost of the coverage ledger on GPU 0: this tree's libccm.so against a build of the parent commit, in one process,
both armed for the coverage proof (ccm_scrub_prove), the two alternated call by call.  Prints ONE JSON line (and writes
it to --out when given).

  python benchmarks/cover_ledger.py --parent-lib PATH [--calls 9] [--out FILE]

Cold whole-HBM gates, the zero gate and the tagged gate, one warm-up round, then --calls rounds.  Per build and gate:
the pass times the call reports (ms_scrub, ms_verify; tagged: ms_tag, ms_check), the host's proof time (ms_prove) and
this tree's ledger time (ms_ledger), the bytes mapped, and the time to verdict (the call's own wall clock) as median,
p10 and p90.  `ratio` is this tree's median over the parent's (> 1: slower).
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

from k8s_cc_manager_b200 import _native as N  # noqa: E402
from page_map import card, open_lib  # noqa: E402

PASS_FIELDS = {"zero": ("ms_scrub", "ms_verify"), "tagged": ("ms_scrub", "ms_verify", "ms_tag", "ms_check")}


def one_gate(lib, kind: str, ledger: bool) -> dict:
    res, tag, cover = N.ScrubResult(), N.TagResult(), N.CoverReport()
    t0 = time.perf_counter()
    rc = (lib.ccm_scrub_verify_tagged(0, 0, C.byref(tag), C.byref(res)) if kind == "tagged"
          else lib.ccm_scrub_verify(0, 0, C.byref(res)))
    ms = (time.perf_counter() - t0) * 1e3
    assert rc == 0, (kind, rc)
    assert lib.ccm_scrub_last_cover(0, C.byref(cover)) == 0 and cover.proved and cover.covered, kind
    out = {"ms_verdict": ms, "bytes_scrubbed": res.bytes_scrubbed, "ms_prove": cover.ms_prove,
           "ms_scrub": res.ms_scrub, "ms_verify": res.ms_verify, "ms_tag": tag.ms_tag, "ms_check": tag.ms_check}
    if ledger:
        led = N.CoverLedger()
        assert lib.ccm_scrub_last_ledger(0, C.byref(led)) == 0 and led.proved and led.exact, kind
        out["ms_ledger"] = led.ms_ledger
    lib.ccm_scrub_release_wait(0, None, None)
    return out


def pct(xs: list, q: float) -> float:
    xs = sorted(xs)
    return xs[min(len(xs) - 1, max(0, round(q * (len(xs) - 1))))]


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent-lib", required=True, help="libccm.so built from the parent commit")
    ap.add_argument("--calls", type=int, default=9)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    libs = {"new": open_lib(str(N.LIB_PATH)), "parent": open_lib(a.parent_lib)}
    for lib in libs.values():
        assert lib.ccm_scrub_prove(0, 1) == 0
    runs = {(kind, name): [] for kind in PASS_FIELDS for name in libs}
    for i in range(1 + a.calls):
        for kind in PASS_FIELDS:
            for name, lib in libs.items():
                r = one_gate(lib, kind, name == "new")
                if i:
                    runs[kind, name].append(r)
    out = {"bench": "cover_ledger", **card(), "calls": a.calls, "gate": {}}
    for kind, fields in PASS_FIELDS.items():
        row = {}
        for name in libs:
            rs = runs[kind, name]
            row[name] = {f: statistics.median(r[f] for r in rs) for f in fields + ("ms_prove", "bytes_scrubbed")}
            verdict = [r["ms_verdict"] for r in rs]
            row[name].update(ms_verdict_median=statistics.median(verdict), ms_verdict_p10=pct(verdict, 0.1),
                             ms_verdict_p90=pct(verdict, 0.9))
            if name == "new":
                row[name]["ms_ledger"] = statistics.median(r["ms_ledger"] for r in rs)
        row["ratio"] = {f: row["new"][f] / row["parent"][f] for f in fields + ("ms_verdict_median",)}
        row["bytes_mapped_less"] = row["parent"]["bytes_scrubbed"] - row["new"]["bytes_scrubbed"]
        out["gate"][kind] = row
    for lib in libs.values():
        lib.ccm_scrub_prove(0, 0)
    line = json.dumps(out)
    print(line)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(line + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
