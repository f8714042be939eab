"""Out-of-process HBM scrub: `python -m k8s_cc_manager_b200.scrub_worker --bdf <bdf> [...]`.

Why a worker process: the manager is a long-lived daemon and the GPUs it manages get RESET as
part of every transition.  CUDA state inside the daemon (device file descriptors, a poisoned
context after a fault) must not leak from one transition into the next, and a CUDA fault must not
take the control loop down.  With CC_SCRUB_ISOLATION=process the manager runs the whole
concurrent gate (ccm_scrub_verify_many: one host thread + context + stream per GPU) in this
short-lived process and reads ONE JSON line back; the process exit returns every CUDA resource.

Output (stdout, last line):  {"wall_ms": ..., "reports": [ {ScrubReport fields}, ... ]}
(the tagged-gate fields only with --check tagged; "residue" only with --residue; "triage" only with --triage, for a
GPU whose read-back found non-zero bytes; "mismatch_triage" only with --mismatch-triage, for a GPU whose tagged check
found bytes off their tags; "cover" and "cover_ledger" only with --prove, for every GPU whose passes finished; "probe"
only with --probe,
for every GPU whose alias probe ran; "probe_cover" only with --prove and --probe, for every GPU whose alias probe ran;
"report_cover" only with --prove, for every GPU that located dirt or triaged; "hbm_health" only with --health report
or --health require, for every GPU that was armed).
Exit code: 0 if every GPU is clean, 3 if the gate failed, 2 on usage errors.
"""
from __future__ import annotations

import argparse
import json
import sys
from typing import List, Optional

from . import _native as N
from . import devices as D


def run(bdfs: List[str], nbytes: int, check: str = "zero", residue: bool = False, triage_hold_ms: int = 0,
        mismatch_triage_hold_ms: int = 0, prove: bool = False, probe: bool = False, health: str = "off") -> dict:
    """triage_hold_ms > 0 arms the dirt triage with that hold, mismatch_triage_hold_ms > 0 the mismatch triage (with
    the same hold when both are armed); prove arms the coverage proof, probe the alias probe, health ('report' or
    'require') the HBM health report."""
    by_bdf = {d.bdf: d for d in D.find_gpus()[0] if d.is_gpu()}
    missing = [b for b in bdfs if b not in by_bdf]
    if missing:
        raise SystemExit(f"unknown GPU(s): {', '.join(missing)} (known: {', '.join(sorted(by_bdf))})")
    devs = [by_bdf[b] for b in bdfs]
    if health != "off":
        reports, wall_ms = D.scrub_and_verify_many(devs, nbytes, check=check, residue=residue,
                                                   triage=bool(triage_hold_ms),
                                                   triage_hold_ms=mismatch_triage_hold_ms or triage_hold_ms or
                                                   D.TRIAGE_HOLD_MS,
                                                   mismatch_triage=bool(mismatch_triage_hold_ms), prove=prove,
                                                   probe=probe, health=health)
    elif probe:
        reports, wall_ms = D.scrub_and_verify_many(devs, nbytes, check=check, residue=residue,
                                                   triage=bool(triage_hold_ms),
                                                   triage_hold_ms=mismatch_triage_hold_ms or triage_hold_ms or
                                                   D.TRIAGE_HOLD_MS,
                                                   mismatch_triage=bool(mismatch_triage_hold_ms), prove=prove,
                                                   probe=True)
    elif prove:
        reports, wall_ms = D.scrub_and_verify_many(devs, nbytes, check=check, residue=residue,
                                                   triage=bool(triage_hold_ms),
                                                   triage_hold_ms=mismatch_triage_hold_ms or triage_hold_ms or
                                                   D.TRIAGE_HOLD_MS,
                                                   mismatch_triage=bool(mismatch_triage_hold_ms), prove=True)
    elif mismatch_triage_hold_ms:
        reports, wall_ms = D.scrub_and_verify_many(devs, nbytes, check=check, residue=residue,
                                                   triage=bool(triage_hold_ms),
                                                   triage_hold_ms=mismatch_triage_hold_ms, mismatch_triage=True)
    elif triage_hold_ms:
        reports, wall_ms = D.scrub_and_verify_many(devs, nbytes, check=check, residue=residue, triage=True,
                                                   triage_hold_ms=triage_hold_ms)
    elif residue:
        reports, wall_ms = D.scrub_and_verify_many(devs, nbytes, check=check, residue=True)
    else:
        reports, wall_ms = D.scrub_and_verify_many(devs, nbytes, check=check)
    return {"wall_ms": wall_ms, "reports": [r.as_json() for r in reports]}


def main(argv: Optional[List[str]] = None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--bdf", action="append", default=[], help="PCI address of a GPU to scrub (repeatable)")
    ap.add_argument("--bytes", type=int, default=0, help="bytes per GPU (0 = all mappable HBM)")
    ap.add_argument("--backend", choices=sorted(N.BACKENDS), default=None)
    ap.add_argument("--check", choices=D.CHECKS, default="zero",
                    help="zero: zero-fill + read-back; tagged: an address-tagged known answer first")
    ap.add_argument("--residue", action="store_true",
                    help="report what the first pass found in the memory before it erased it (never fails the gate)")
    ap.add_argument("--triage", action="store_true",
                    help="after a failed read-back, re-zero and re-read the dirty pages: does the dirt stay, return or "
                         "clear (never fails the gate)")
    ap.add_argument("--mismatch-triage", action="store_true",
                    help="with --check tagged, after a failed check, re-tag, check and re-read the pages off their tags: "
                         "does the mismatch stay, return or clear (never fails the gate)")
    ap.add_argument("--prove", action="store_true",
                    help="prove that every pass walked every mapped byte exactly once (with --probe, that every probe "
                         "step took every window once); a GPU whose pass or step did not fails the gate")
    ap.add_argument("--probe", action="store_true",
                    help="with --check zero, after a clean read-back, tag, check and re-read one 32-byte window per 4 KiB "
                         "page; a GPU with a page mapped twice fails the gate")
    ap.add_argument("--health", choices=tuple(N.HBM_HEALTH_MODES), default="off",
                    help="read the GPU's ECC counters and row-remapping state before and after the gate; require: a GPU "
                         "whose memory failed during the gate, or whose state cannot be read, fails the gate")
    ap.add_argument("--triage-hold-ms", type=int, default=D.TRIAGE_HOLD_MS,
                    help="the triages' hold before their last re-read (default %(default)s)")
    args = ap.parse_args(argv)
    if not args.bdf:
        ap.error("at least one --bdf is required")
    if args.mismatch_triage and args.check != "tagged":
        ap.error("--mismatch-triage needs --check tagged")
    if args.probe and args.check == "tagged":
        ap.error("--probe is for --check zero: the tagged check already covers every probe window")
    if args.backend:
        D.select_backend(args.backend)
    out = run([b.lower() for b in args.bdf], args.bytes, args.check, args.residue,
              args.triage_hold_ms if args.triage else 0, args.triage_hold_ms if args.mismatch_triage else 0,
              args.prove, args.probe, args.health)
    print(json.dumps(out), flush=True)
    return 0 if all(r["status"] == 0 and r["nonzero_bytes"] == 0 and r.get("mismatch_bytes", 0) == 0
                    for r in out["reports"]) else 3


if __name__ == "__main__":
    sys.exit(main())
