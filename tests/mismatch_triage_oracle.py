"""The mismatch triage restated (include/ccm.h: ccm_scrub_mismatch_triage): the class of every page of a mismatch page
map under the two triage drills, and the exact fields of its ccm_triage_report.

The mismatch triage takes the runs of a mismatch page map as the dirt triage takes those of a dirt page map
(oracle/triage_oracle.py: runs()).  It writes the call's tags over every run again (T1), checks them and zeroes the run
(T2), holds, and reads the run for non-zero bytes (T3).  On memory that keeps what is stored, only the drills leave
bytes for T2 and T3: "triage_stay" = k XORs the first byte of each of the first k pages of the mismatch page map with
0xA5 between T1 and T2, "triage_return" = k the same bytes between T2 and T3.  T2 zeroes the stay byte, so page i has a
T2 byte when i < stay and a T3 byte when i < ret (unlike the dirt triage, whose T3 still sees the stay byte).

    classify(entries, stay, ret)            [(page, chunk, class, mismatch bytes, T2 bytes, T3 bytes)] per page
    report(entries, spans, stay, ret)       the exact fields of ccm_triage_report
"""
from __future__ import annotations

import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1] / "oracle"))
from triage_oracle import CLEARS, PAGE_BYTES, RETURNS, STAYS, runs  # noqa: E402


def classify(entries, stay: int = 0, ret: int = 0) -> list:
    """(page, chunk, class, mismatch bytes, T2 bytes, T3 bytes) of every (page, bytes, chunk) entry of a mismatch page
    map, ascending, on memory that keeps what is stored, with the drills "triage_stay" = stay and "triage_return" =
    ret."""
    out = []
    for i, (page, nbytes, chunk) in enumerate(sorted(entries)):
        t2, t3 = int(i < stay), int(i < ret)
        cls = STAYS if t2 else RETURNS if t3 else CLEARS
        out.append((page, chunk, cls, nbytes, t2, t3))
    return out


def report(entries, spans, stay: int = 0, ret: int = 0) -> dict:
    """The exact fields of ccm_triage_report (all but the offsets' base, the times and the hold)."""
    rows = classify(entries, stay, ret)
    rs = runs(entries, spans)
    out = {"pages_examined": len(rows), "bytes_examined": sum(n for _, n, _ in rs), "runs": len(rs),
           "t2_bytes": sum(r[4] for r in rows), "t3_bytes": sum(r[5] for r in rows)}
    for cls, key in ((STAYS, "stay"), (RETURNS, "return"), (CLEARS, "clear")):
        out[f"{key}_pages"] = sum(1 for r in rows if r[2] == cls)
        out[f"{key}_bytes"] = sum(r[3] for r in rows if r[2] == cls)
    for t, col in (("t2", 4), ("t3", 5)):
        hit = [r[0] * PAGE_BYTES for r in rows if r[col]]
        out[f"{t}_first_offset"] = min(hit) if hit else 0
        out[f"{t}_last_offset"] = max(hit) if hit else 0
    return out
