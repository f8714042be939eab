"""CPU: the window-book tests (tests/test_window_books_gpu.py) reach every head-window count and every place a book
kernel books from, their layouts put their windows where they say, and every kernel libccm.so defines is named in a
table of the GPU tests that launch it."""
from __future__ import annotations

import re
import shutil
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "oracle"))
import dirt_oracle as DO  # noqa: E402
import mismatch_oracle as MO  # noqa: E402
import scrub_cases as CASES  # noqa: E402
import tag_oracle as TO  # noqa: E402
import window_book_cases as WB  # noqa: E402
from k8s_cc_manager_b200 import _native as N  # noqa: E402

G = WB.geometry(CASES.H100_SMS)
BASE = 1 << 40                         # a 128-aligned address for the oracles


def test_placements_reach_every_head_window_count_and_every_place():
    seen = set()
    reach = set()
    for o, n in WB.placements(G):
        k, aligned = WB.head_windows(o, n)
        seen.add((k, aligned if k else None))
        reach |= WB.paths(o, n)
    assert {(k, True) for k in range(1, 8)} <= seen, sorted(seen)       # a whole first window: 1..7 head windows
    assert {(k, False) for k in range(1, 9)} <= seen, sorted(seen)      # a first window sticking out: 1..8
    assert (0, None) in seen
    assert reach == set(WB.PATHS)
    assert set(CASES.OFFSETS) <= set(WB.OFFSETS)
    for o in WB.OFFSETS:
        ls = WB.lengths(G, o)
        assert set(CASES.lengths(G)) <= set(ls) and 0 in ls
        inside = [n for n in ls if 0 < n and DO.window_count(BASE + o, n) == 1]
        straddle = [n for n in ls if DO.window_count(BASE + o, n) == 2]
        assert inside and straddle, o


def test_head_windows_match_the_oracle_window_count():
    for o in WB.OFFSETS:
        head, _, _ = CASES.split(o, 1000, 16)
        k, aligned = WB.head_windows(o, 1000)
        assert k == (DO.window_count(BASE + o, head) if head else 0)
        assert aligned == (o % 16 == 0)


def test_where_restates_the_chunk_rules():
    # offset 16: 112 head bytes in 7 whole windows; then 2 chunks, 3 leftover vectors and a 15-byte tail
    n = 112 + 2 * WB.CHUNK + 48 + 15
    assert WB.where(16, n, 0) == ("head", 0) and WB.where(16, n, 111) == ("head", 6)
    assert WB.where(1, n, 0) == ("head", 0) and WB.where(1, n, 15) == ("head", 1)
    assert WB.where(16, n, 112) == ("batch", 0, 0, 0)
    assert WB.where(16, n, 112 + WB.STRIDE - 1) == ("batch", 0, WB.THREADS - 1, 0)
    assert WB.where(16, n, 112 + WB.STRIDE) == ("batch", 0, 0, 1)
    assert WB.where(16, n, 112 + WB.CHUNK + 15 * WB.STRIDE + 16 * 5) == ("batch", 1, 5, 15)
    assert WB.where(16, n, 112 + 2 * WB.CHUNK) == ("leftover", 2 * WB.CHUNK // 16)
    assert WB.where(16, n, n - 15) == ("tail",) and WB.where(16, n, n - 1) == ("tail",)


@pytest.mark.parametrize("w", WB.LIMIT_COUNTS)
def test_layouts_put_their_windows_where_they_say(w):
    for lay in WB.limit_layouts(w):
        assert len(lay.windows) == len(set(lay.windows)) == w and list(lay.windows) == sorted(lay.windows), lay.name
        places = [WB.where(lay.offset, lay.n, wd) for wd in lay.windows]
        for wd in lay.windows:
            assert (BASE + lay.offset + wd) % 16 == 0 and WB.window_bytes(lay.offset, lay.n, wd), (lay.name, wd)
        if lay.path != "mixed":
            assert {p[0] for p in places} == {lay.path}, lay.name
        if lay.name.startswith("batch_u"):
            u = int(lay.name[len("batch_u"):])
            assert {p[3] for p in places} == {u} and len({p[1] for p in places}) == min(w, 4)
        if lay.name == "per_chunk":
            assert sorted(p[1] for p in places) == list(range(w)) and lay.n // WB.CHUNK > 65
        if lay.name == "one_chunk":
            assert {p[1] for p in places} == {0} and lay.n == WB.CHUNK
        if lay.name == "mixed":
            kinds = [p[0] for p in places]
            assert kinds.count("head") == min(w, 7) and kinds.count("tail") == (1 if w > 7 else 0)
            if w >= 64:
                assert {"batch", "leftover"} <= set(kinds)
        # under the oracles the layout books exactly its w windows
        masks = [0xFFFF & WB.in_region_mask(lay.n, wd) for wd in lay.windows]
        rng = np.random.default_rng(w)
        buf = WB.dirt_content(lay.offset, lay.n, lay.windows, masks, rng)
        rep = DO.report(buf, BASE + lay.offset)
        assert rep["dirty_windows"] == w and rep["truncated"] == (w > WB.RECORDS), lay.name
        assert [o for o, _, _ in rep["windows"]] == list(lay.windows)
        if lay.n <= 4 * WB.CHUNK:
            tags = TO.tag_bytes(3, BASE + lay.offset, lay.n)
            rep = MO.report(WB.flip_content(tags, lay.windows, masks, rng), BASE + lay.offset, 3, classify_limit=0)
            assert rep["mismatch_windows"] == w and [x["offset"] for x in rep["windows"]] == list(lay.windows)


def test_masks_and_content():
    assert len(WB.all_masks()) == 65535
    em = WB.edge_masks()
    assert len(em) == len(set(em)) > 273
    assert sum(1 for m in em if bin(m).count("1") <= 2 or bin(m).count("1") >= 14) == 16 + 120 + 120 + 16 + 1
    rng = np.random.default_rng(1)
    masks = list(range(1, 65))
    wins = [16 * 3 * i for i in range(64)]
    buf = WB.dirt_content(0, 4096, wins, masks, rng)
    rep = DO.report(buf, BASE)
    assert [(o, m) for o, m, _ in rep["windows"]] == list(zip(wins, masks))
    tags = TO.tag_bytes(9, BASE + 5, 4096)
    flipped = WB.flip_content(tags, [w - 5 for w in wins[1:]], masks[1:], rng)
    rep = MO.report(flipped, BASE + 5, 9, classify_limit=0)
    assert [(x["offset"], x["mask"]) for x in rep["windows"]] == list(zip([w - 5 for w in wins[1:]], masks[1:]))


# ------------------------------------------------------------------ every kernel libccm.so defines, and who runs it
# kernel -> the GPU test that launches it ("file::test")
KERNEL_TESTS = {
    "scrub_st_kernel": "test_scrub_exactness_gpu.py::test_scrub_matrix_writes_exactly_its_region",
    "scrub_tma_kernel": "test_scrub_exactness_gpu.py::test_scrub_matrix_writes_exactly_its_region",
    "scrub_st128_fast_kernel": "test_scrub_exactness_gpu.py::test_scrub_matrix_writes_exactly_its_region",
    "verify_ld_kernel": "test_scrub_exactness_gpu.py::test_verify_matrix_counts_exactly",
    "verify_ld128_fast_kernel": "test_scrub_exactness_gpu.py::test_verify_matrix_counts_exactly",
    "locate_dirt_kernel": "test_window_books_gpu.py::test_placement_matrix",
    "tag_check_zero_kernel": "test_window_books_gpu.py::test_placement_matrix",
    "census_zero_kernel": "test_window_books_gpu.py::test_placement_matrix",
    "census_tag_fill_kernel": "test_window_books_gpu.py::test_placement_matrix",
    "tag_fill_kernel": "test_window_books_gpu.py::test_placement_matrix",
    "xor_byte_kernel": "test_window_books_gpu.py::test_record_limit_in_product_calls",
    "fill_byte_kernel": "test_scrub_gpu.py::test_segmented_arena",
    "fill_pattern_kernel": "test_scrub_gpu.py::test_seeded_pattern_count_matches_oracle",
    # the proving twins, armed on caller-owned memory (include/ccm.h: ccm_region_prove)
    "cover_zero_pass": "test_scrub_exactness_gpu.py::test_scrub_matrix_writes_exactly_its_region",
    "cover_read_pass": "test_scrub_exactness_gpu.py::test_verify_matrix_counts_exactly",
    "cover_tag_fill_pass": "test_window_books_gpu.py::test_placement_matrix",
    "cover_tag_check_pass": "test_window_books_gpu.py::test_placement_matrix",
    "cover_census_zero_pass": "test_window_books_gpu.py::test_placement_matrix",
    "cover_census_tag_pass": "test_window_books_gpu.py::test_placement_matrix",
    "cover_locate_pass": "test_window_books_gpu.py::test_placement_matrix",
    "alias_probe_fill_pass": "test_alias_probe_gpu.py::test_region_probe_against_the_oracle",
    "alias_probe_check_pass": "test_alias_probe_gpu.py::test_region_probe_against_the_oracle",
    "alias_probe_reread_pass": "test_alias_probe_gpu.py::test_region_probe_against_the_oracle",
    "cover_probe_fill_pass": "test_alias_probe_gpu.py::test_region_probe_against_the_oracle",
    "cover_probe_check_pass": "test_alias_probe_gpu.py::test_region_probe_against_the_oracle",
    "cover_probe_reread_pass": "test_alias_probe_gpu.py::test_region_probe_against_the_oracle",
}
ENTRY_RE = re.compile(r"^STT_FUNC\s+STB_GLOBAL\s+\S+\s+(\S+)$", re.M)
KERNEL_RE = re.compile(r"^(?:void )?ccm::(\w+)(?:<[^>]*>)?\(")


def device_kernels() -> list[str]:
    """Every kernel entry of libccm.so's device code (its global functions), demangled."""
    from k8s_cc_manager_b200 import build
    cuobjdump = Path(build.find_nvcc()).parent / "cuobjdump"
    assert cuobjdump.exists(), f"{cuobjdump} lists the kernels libccm.so defines; it ships with nvcc"
    out = subprocess.run([str(cuobjdump), "-symbols", str(N.LIB_PATH)], check=True, capture_output=True,
                         text=True).stdout
    cxxfilt = shutil.which("c++filt")
    assert cxxfilt, "c++filt (binutils) is needed to demangle the kernel names"
    mangled = ENTRY_RE.findall(out)
    return subprocess.run([cxxfilt], input="\n".join(mangled), check=True, capture_output=True,
                          text=True).stdout.split("\n")[:len(mangled)]


def test_every_kernel_is_launched_by_a_named_gpu_test():
    entries = device_kernels()
    names = [KERNEL_RE.match(e) for e in entries]
    assert all(names), [e for e, m in zip(entries, names) if not m]
    defined = {m.group(1) for m in names}
    assert {"locate_dirt_kernel", "cover_locate_pass", "alias_probe_check_pass"} <= defined, sorted(defined)
    missing = sorted(defined - set(KERNEL_TESTS))
    assert not missing, "kernels no GPU test is named for (add them to KERNEL_TESTS):\n  " + "\n  ".join(missing)
    assert not set(KERNEL_TESTS) - defined, sorted(set(KERNEL_TESTS) - defined)
    for kernel, test in KERNEL_TESTS.items():
        fname, tname = test.split("::")
        src = (ROOT / "tests" / fname).read_text()
        assert re.search(rf"^def {tname}\(", src, re.M), (kernel, test)
    print(f"\n{len(entries)} kernel entries, {len(defined)} kernels, each launched by a named GPU test")
