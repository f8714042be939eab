"""The case list of tests/pdl_book_calls.py, checked on the CPU: every launch pair the programmatic-dependent-launch
test needs is in a region chain at every placement, every book is reached, and the placements reach the ragged head,
the tail, the leftover vectors and page boundaries inside a grab."""
from __future__ import annotations

import numpy as np

import pdl_book_calls as PBC
import product_plan as PP
import scrub_cases as CASES
import tag_oracle as TO
import test_window_book_cases as WBC
import window_book_cases as WB

# (predecessor, dependent) launches that must follow each other directly on one stream.  Every default-frame kernel
# that was never run under PDL before is a dependent here: the tag fill, the tag check, the locate pass and both
# censuses.
REQUIRED_PAIRS = {
    ("scrub_st128_fast_kernel", "census_zero_kernel"),
    ("scrub_st128_fast_kernel", "tag_fill_kernel"),
    ("tag_fill_kernel", "census_tag_fill_kernel"),
    ("tag_fill_kernel", "tag_check_zero_kernel"),
    (PBC.TORCH, "tag_fill_kernel"),
    ("scrub_st128_fast_kernel", PBC.TORCH),
    (PBC.TORCH, "locate_dirt_kernel"),
}


def test_every_pair_is_chained_at_every_placement():
    seen: dict = {}
    for chain, off, n in PBC.region_cases():
        for pair in PBC.pairs(chain):
            seen.setdefault(pair, set()).add((off, n))
    assert REQUIRED_PAIRS <= set(seen), sorted(REQUIRED_PAIRS - set(seen))
    for pair in REQUIRED_PAIRS:
        assert seen[pair] == set(PBC.PLACEMENTS), pair
    assert {d for _, d in seen} >= {"tag_fill_kernel", "tag_check_zero_kernel", "locate_dirt_kernel",
                                    "census_zero_kernel", "census_tag_fill_kernel"}
    assert {k for k in PBC.KERNELS.values() if k != PBC.TORCH} <= set(WBC.KERNEL_TESTS)


def test_every_book_is_reached():
    region_books = {PBC.BOOKS[steps[-1]] for steps in PBC.CHAINS.values()}
    assert region_books == {"dirt", "mismatch", "residue"}
    import test_page_map_gpu as TPM
    assert set(PBC.PRODUCT_DRILLS) == set(TPM.DRILL_CALLS)
    product_books = {TPM.DRILL_CALLS[d][2] for d in PBC.PRODUCT_DRILLS}
    assert product_books == {TPM.N.BOOK_DIRT, TPM.N.BOOK_MISMATCH, TPM.N.BOOK_RESIDUE}
    legs = [c["leg"] for c in PBC.product_cases()]
    assert {"product", "alias", "triage", "flood"} == set(legs)


def test_product_paths_and_triage_drills():
    envs = [env for env, _ in PBC.PRODUCT_PATHS.values()]
    for mf, il in PP.MODES:
        assert PP.mode_env(mf, il) in envs
    assert ({"CCM_PIPELINE": "0"}, 0) in PBC.PRODUCT_PATHS.values()
    assert ({"CCM_PIPELINE": "0", "CCM_ARENA_MAX_SEGMENT_MB": "3"}, 64 * PBC.MiB) in PBC.PRODUCT_PATHS.values()
    cases = PBC.product_cases()
    for path in PBC.PRODUCT_PATHS:
        assert {c["drill"] for c in cases if c["leg"] == "product" and c["path"] == path} == set(PBC.PRODUCT_DRILLS)
    assert {c["mf"] for c in cases if c["leg"] == "alias"} == {0, 1}
    assert set(PBC.TRIAGE_PATHS) == set(PBC.PRODUCT_PATHS)
    drills = {(c["stay"], c["ret"]) for c in cases if c["leg"] == "triage"}
    assert (0, 0) in drills and any(s and r for s, r in drills)   # every page clears; stays, returns and clears
    assert {env.get("CCM_PIPELINE") for env, _ in PBC.FLOOD_PATHS.values()} == {None, "0"}


def test_placements_reach_every_place_and_page_boundaries_inside_grabs():
    assert set(PBC.OFFSETS) == {0, 1, 17, 112, 127}
    short, long_ = PBC.LENGTHS
    assert long_ == 2 * PBC.PAGE + 3 * WB.CHUNK + 77
    assert set().union(*(WB.paths(o, short) for o in PBC.OFFSETS)) == set(WB.PATHS)
    for off in PBC.OFFSETS:
        head, body, tail = CASES.split(off, short, 16)
        assert body // 16 % (WB.CHUNK // 16) and tail, off               # leftover vectors and a tail window
        if off:
            assert head and (PBC.PAGE - head) % WB.CHUNK, off            # the first page boundary is inside a grab


def test_booked_input_and_planted_dirt():
    """The oracles' inputs: the dirt torch plants is non-zero, inside the region, on both sides of each page boundary
    and in every head and tail window; a fill's successor reads the tags."""
    for i, (chain, off, n) in enumerate(PBC.region_cases()):
        seed = PBC.case_seed(i)
        pos, vals = PBC.planted(off, n, seed)
        assert pos.min() >= 0 and pos.max() < n and np.all(vals != 0) and len(set(pos.tolist())) == pos.size
        if n > PBC.PAGE:
            assert {PBC.PAGE - 1, PBC.PAGE} <= set(pos.tolist())
        head, body, _ = CASES.split(off, n, 16)
        assert set(range(head)) | set(range(head + body, n)) <= set(pos.tolist())
        ptr = (1 << 40) + off
        got = PBC.booked_input(chain, off, n, ptr, seed)
        last = PBC.CHAINS[chain][-1]
        if last in ("census1", "check"):
            assert np.array_equal(got, TO.tag_bytes(PBC.SEED, ptr, n))
        elif last == "locate":
            assert np.count_nonzero(got) == pos.size and np.array_equal(got[pos], vals)
        else:
            assert not got.any()
        assert PBC.end_state(chain, off, n, ptr, seed).any() == (last in ("census1", "locate"))
