"""The window-book kernels, the tagged and census gates and the dirt triage under programmatic dependent launch, on one
H100.  tests/pdl_book_calls.py runs the same cases in one child with CCM_PDL=1 and one with CCM_PDL=0 (the library
latches the setting once per process).  Each child must equal the oracles case by case; the two must agree on
everything that does not depend on the virtual address or the clock, and launch exactly as many kernels."""
from __future__ import annotations

import json
import os
import subprocess
import sys
import time
from pathlib import Path
from types import SimpleNamespace

import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "oracle"))
import page_oracle as PO  # noqa: E402
import pdl_book_calls as PBC  # noqa: E402
import test_dirt_triage_gpu as TDT  # noqa: E402
import test_page_map_gpu as TPM  # noqa: E402
import test_window_books_gpu as WBG  # noqa: E402
from k8s_cc_manager_b200 import _native as N  # noqa: E402
from k8s_cc_manager_b200 import devices as D  # noqa: E402

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


def run_child(pdl: str) -> list:
    env = dict(os.environ, CCM_PDL=pdl)
    proc = subprocess.run([sys.executable, str(ROOT / "tests" / "pdl_book_calls.py")], capture_output=True, text=True,
                          env=env, timeout=1500, cwd=str(ROOT))
    assert proc.returncode == 0, f"CCM_PDL={pdl}: exit {proc.returncode}\n{proc.stdout[-2000:]}\n{proc.stderr[-3000:]}"
    return json.loads(next(line for line in proc.stdout.splitlines() if line.startswith("RESULT "))[7:])


@pytest.fixture(scope="module")
def children():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    t0 = time.monotonic()
    out = {pdl: run_child(pdl) for pdl in ("1", "0")}
    print(f"\ntwo children, {len(out['1'])} cases each: {time.monotonic() - t0:.1f} s")
    return out


# ------------------------------------------------------------------------------------ 1. each child against the oracles
def entries(rows) -> list:
    return [tuple(e) for e in rows]


def assert_region_case(rec: dict, what):
    chain, off, n, ptr, seed = rec["chain"], rec["offset"], rec["n"], rec["ptr"], rec["seed"]
    last = PBC.CHAINS[chain][-1]
    assert ptr % 128 == off, what
    region = PBC.booked_input(chain, off, n, ptr, seed)
    b = rec["book"]
    got = WBG.Book(b["count"], b["windows"], b["first"], b["last"], b["truncated"],
                   [tuple(r) for r in b["records"]], b["zero_windows"])
    WBG.assert_book(got, WBG.oracle(last, region, ptr, PBC.SEED), what)
    want_pages = PO.check_page_map(region, ptr, PBC.SEED) if last == "check" else PO.page_map(region, ptr)
    assert entries(rec["pages"]) == PO.entries(want_pages), what
    assert (rec["wrong"], rec["guards"]) == (0, 0), (what, "end state", rec["wrong"], "guard bytes", rec["guards"])
    # one launch per library step
    assert rec["launches"] == sum(s != "dirt" for s in PBC.CHAINS[chain]), what


def product_out(rec: dict):
    """(rc, result, tag, residue, dirt, mismatch, maps) as tests/test_page_map_gpu.py's product() returns them."""
    tag = SimpleNamespace(**rec["tag"]) if rec["tag"] is not None else None
    maps = {b: entries(e) for b, e in rec["maps"]}
    return (rec["rc"], SimpleNamespace(**rec["res"]), tag, D.ResidueReport.from_json(rec["residue"]),
            D.DirtReport.from_json(rec["dirt"]), D.MismatchReport.from_json(rec["mismatch"]), maps)


def triage_out(rec: dict) -> dict:
    """What tests/test_dirt_triage_gpu.py's call() returns."""
    return {"rc": rec["rc"], "res": SimpleNamespace(**rec["res"]), "dirt": D.DirtReport.from_json(rec["dirt"]),
            "triage": SimpleNamespace(**rec["triage"]), "dirt_pages": entries(rec["dirt_pages"]),
            "triage_pages": [D.TriagePage(**p) for p in rec["triage_pages"]]}


def assert_case(rec: dict, what):
    leg = rec["leg"]
    if leg == "region":
        assert_region_case(rec, what)
    elif leg == "product":
        TPM.assert_product(rec["drill"], rec["env"], rec["bytes"], False, product_out(rec))
    elif leg == "alias":
        TPM.assert_alias(rec["mf"], product_out(rec))
    elif leg == "triage":
        out = triage_out(rec)
        assert out["rc"] == N.ERR_DIRTY and out["dirt"].located, what
        TDT.assert_triage(out, rec["env"], rec["bytes"], rec["stay"], rec["ret"], what)
    else:
        TDT.assert_flood(triage_out(rec), rec["env"], rec["bytes"])


# ------------------------------------------------------------------------------------ 2. PDL against plain
def portable(rec: dict):
    """The case without what depends on the virtual address (va_base, the region pointer, the drawn tag seed, the
    tags themselves), the clock (ms_*) or the error text, and without the records of a truncated report (any 64 of its
    windows)."""
    def strip(x):
        if isinstance(x, dict):
            return {k: strip(v) for k, v in x.items()
                    if k not in ("va_base", "ptr", "seed", "err", "error") and not k.startswith("ms_")}
        if isinstance(x, list):
            return [strip(v) for v in x]
        return x

    out = strip(rec)
    if rec["leg"] == "region":
        out["seed"] = rec["seed"]
        if PBC.CHAINS[rec["chain"]][-1] == "census1":      # the residue of the tags: their non-zero bytes
            out.pop("book"), out.pop("pages")
        elif out["book"]["truncated"]:                     # any 64 of the windows: checked against the oracle
            out["book"].pop("records")
    if rec["leg"] == "alias":                              # which aliased bytes keep their tags depends on the tags
        out.pop("tag"), out.pop("mismatch"), out.pop("maps")
    elif rec["leg"] == "product" and not TPM.DRILL_CALLS[rec["drill"]][0].startswith("census"):
        # a call without a census leaves the residue page map of the last census, here a tagged region's
        out["maps"] = [m for m in out["maps"] if m[0] != N.BOOK_RESIDUE]
    for name in ("dirt", "mismatch", "residue"):
        if name in out and out[name]["truncated"]:
            out[name].pop("records")
    if "mismatch" in out:                                  # the bytes a mismatch record read are tag bytes
        for r in out["mismatch"].get("records", []):
            r.pop("bytes")
    if "res" in out:                                       # what the child found free, not what the call did
        out["res"].pop("device_free_before")
    return out


def test_each_child_equals_the_oracles(children):
    for pdl, recs in children.items():
        assert [(r["leg"], r.get("chain"), r.get("offset"), r.get("n")) for r in recs[:len(PBC.region_cases())]] == \
            [("region", c, o, n) for c, o, n in PBC.region_cases()]
        assert [{k: r[k] for k in c} for r, c in zip(recs[len(PBC.region_cases()):], PBC.product_cases())] == \
            PBC.product_cases()
        for i, rec in enumerate(recs):
            assert_case(rec, (f"CCM_PDL={pdl}", i, rec["leg"], rec.get("chain") or rec.get("drill"),
                              rec.get("path"), rec.get("offset"), rec.get("n")))


def same_mapping(x: dict, y: dict) -> bool:
    """A whole-HBM call maps until the driver runs out of memory, which may fall a granule apart in two processes; its
    report, page maps and launches depend on that mapping."""
    keys = ("device_free_before", "bytes_scrubbed", "segments")
    return x.get("bytes") != 0 or all(x["res"][k] == y["res"][k] for k in keys)


def test_pdl_and_plain_children_agree(children):
    a, b = children["1"], children["0"]
    assert len(a) == len(b)
    compared = 0
    for i, (x, y) in enumerate(zip(a, b)):
        if not same_mapping(x, y):                         # the verdict still may not differ
            assert (x["rc"], x["res"]["status"]) == (y["rc"], y["res"]["status"]), i
            continue
        assert portable(x) == portable(y), (i, x["leg"], x.get("chain") or x.get("drill"), x.get("path"))
        compared += 1
    print(f"\n{compared} of {len(a)} cases compared field by field")
    assert compared >= len(PBC.region_cases()) + sum(1 for r in a[len(PBC.region_cases()):] if r["bytes"] != 0)


def test_launch_counts_are_identical(children):
    a, b = children["1"], children["0"]
    assert [r["launches"] for r in a if r["leg"] == "region"] == [r["launches"] for r in b if r["leg"] == "region"]
    for i, (x, y) in enumerate(zip(a, b)):
        if same_mapping(x, y):
            assert x["launches"] == y["launches"], (i, x["leg"], x.get("drill"), x.get("path"))
    assert all(r["launches"] > 0 for r in a + b)
