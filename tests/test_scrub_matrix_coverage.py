"""CPU: the GPU exactness matrix (tests/test_scrub_exactness_gpu.py) reaches every scrub / verify kernel
instantiation libccm.so defines, and its pattern builders and expected counts agree with the C oracle."""
from __future__ import annotations

import re
import shutil
import subprocess

import numpy as np
import pytest

import scrub_cases as SC
import scrub_oracle as SO
from k8s_cc_manager_b200 import _native as N

KERNEL_RE = re.compile(r"ccm::((?:scrub|verify)_\w*kernel<[^>]*>)\(")


def defined_instantiations() -> set[str]:
    nm = shutil.which("nm")
    assert nm, "nm (binutils) is needed to list the kernels libccm.so defines"
    out = subprocess.run([nm, "-C", "--defined-only", str(N.LIB_PATH)], check=True, capture_output=True,
                         text=True).stdout
    return set(KERNEL_RE.findall(out))


def test_every_kernel_instantiation_is_reached_by_the_matrix():
    defined = defined_instantiations()
    families = {"scrub_st_kernel": 40, "verify_ld_kernel": 32, "scrub_tma_kernel": 3}
    for fam, n in families.items():
        assert sum(k.startswith(fam + "<") for k in defined) >= n, (fam, sorted(defined))
    assert any("_fast_kernel<" in k for k in defined)
    fast = N.default_kernels()
    reached = {SC.instantiation(c, fast) for c in SC.all_cases()} - {None}
    assert reached <= defined, f"the matrix maps cases to kernels libccm.so does not define: {sorted(reached - defined)}"
    missing = sorted(defined - reached)
    assert not missing, "kernel instantiations no GPU test launches:\n  " + "\n  ".join(missing)


def test_dispatch_rules_restated():
    fast = ("F", "V")
    cfg = lambda **kw: tuple(kw.get(k, 0) for k in ("ctas_per_sm", "threads", "tile_bytes", "unroll",  # noqa: E731
                                                     "cache_policy", "schedule"))
    inst = lambda kind, v, **kw: SC.instantiation(SC.Case(kind, v, cfg(**kw)), fast)  # noqa: E731
    assert SC.instantiation(SC.Case("scrub", SC.SCRUB_ST128, None), fast) == "F"
    assert SC.instantiation(SC.Case("verify", SC.VERIFY_LD128, None), fast) == "V"
    assert SC.instantiation(SC.Case("scrub", SC.SCRUB_ST256, None), fast) == "scrub_st_kernel<32, 4, 0>"
    assert SC.instantiation(SC.Case("verify", SC.VERIFY_LD256, None), fast) == "verify_ld_kernel<32, 4, 2>"
    assert inst("scrub", SC.SCRUB_ST128, unroll=3, cache_policy=2) == "scrub_st_kernel<16, 4, 1>"
    assert inst("scrub", SC.SCRUB_ST128, unroll=16) == "scrub_st_kernel<16, 16, 0>"
    assert inst("verify", SC.VERIFY_LD128, unroll=16, cache_policy=4) == "verify_ld_kernel<16, 4, 3>"
    assert inst("verify", SC.VERIFY_LD256, cache_policy=9) == "verify_ld_kernel<32, 4, 2>"
    assert inst("scrub", SC.SCRUB_TMA, cache_policy=3) == "scrub_tma_kernel<0>"
    assert inst("scrub", SC.SCRUB_TMA, cache_policy=4) == "scrub_tma_kernel<3>"
    assert SC.instantiation(SC.Case("scrub", SC.SCRUB_MEMSET, None), fast) is None


def test_geometry_rules():
    g = SC.geometry(SC.Case("scrub", SC.SCRUB_ST256, (1, 100, 12345, 4, 0, 3)), 132)
    assert (g.group, g.tile, g.chunk, g.grabbers) == (32, 32 * 4 * 32, 12345 // 4096 * 4096, 132 * 3)
    g = SC.geometry(SC.Case("verify", SC.VERIFY_LD128, (2, 100, 5000, 8, 0, 2)), 132)
    assert (g.tile, g.chunk, g.grabbers) == (96 * 8 * 16, 96 * 8 * 16, 264)
    g = SC.geometry(SC.Case("verify", SC.VERIFY_LD128, (0, 0, 0, 0, 0, 1)), 132)
    assert (g.tile, g.chunk, g.grabbers) == (1024 * 4 * 16, 1024 * 4 * 16, 132)
    g = SC.geometry(SC.Case("scrub", SC.SCRUB_TMA, (1, 64, SC.TMA_TILE_BYTES, 2, 1, 2)), 132)
    assert (g.tile, g.chunk, g.grabbers) == (12336, 2 * 12336, 264) and g.tile % 128
    g = SC.geometry(SC.FAST_VERIFY, 132)
    assert (g.tile, g.chunk, g.grabbers) == (SC.FAST_CHUNK, SC.FAST_CHUNK, 132)


def test_matrix_lengths_fit_and_cover_two_grabs_per_grabber():
    for case, full in SC.scrub_cases() + [(c, True) for grp in SC.verify_groups() for c in grp]:
        g = SC.geometry(case, SC.H100_SMS)
        ls = SC.lengths(g)
        assert max(ls) <= SC.MAX_LENGTH, case.label()
        assert SC.big_length(g) >= 2 * g.chunk * g.grabbers + 7
        assert SC.key_length(g) in ls
        assert g.chunk >= g.tile and g.chunk % g.tile == 0 or case.variant == SC.SCRUB_TMA
        # every placement at the largest length leaves a remainder vector after the last whole tile
        for o in SC.OFFSETS:
            head, body, _ = SC.split(o, SC.big_length(g), g.vb)
            assert body % g.tile >= g.vb, (case.label(), o)
    offsets_at_key = {}
    for case, full in SC.scrub_cases():
        g = SC.geometry(case, SC.H100_SMS)
        offsets_at_key[case] = {o for o, n in SC.placements(g, full) if n == SC.key_length(g)}
    assert all(v == set(SC.OFFSETS) for v in offsets_at_key.values())


@pytest.mark.parametrize("vb", [16, 32])
def test_split_matches_the_device_rule(vb):
    for o in SC.OFFSETS:
        for n in (0, 1, 5, 127, 128, 300, 4099):
            head, body, tail = SC.split(o, n, vb)
            assert head + body + tail == n and body % vb == 0 and tail < vb
            assert head == min((128 - o) % 128, n)
            if body:
                assert (o + head) % 128 == 0


def small_geometries():
    yield SC.Geometry(vb=16, unroll=2, group=32, tile=1024, chunk=2048, grabbers=3)
    yield SC.Geometry(vb=32, unroll=4, group=32, tile=4096, chunk=4096, grabbers=2)
    yield SC.Geometry(vb=16, unroll=1, group=1, tile=12336, chunk=24672, grabbers=2)


@pytest.mark.parametrize("gi", range(3))
def test_structural_dirt_counts_match_the_oracle(gi):
    g = list(small_geometries())[gi]
    for o in SC.OFFSETS:
        for n in SC.lengths(g):
            pos = SC.structural_positions(g, o, n)
            assert pos == sorted(set(pos)) and all(0 <= p < n for p in pos)
            buf = np.zeros(n, dtype=np.uint8)
            buf[pos] = SC.dirt_values(pos, seed=n * 131 + o)
            assert SO.count_nonzero_c(buf) == len(pos) == SO.count_nonzero_np(buf)
            head, body, tail = SC.split(o, n, g.vb)
            if head:
                assert 0 in pos and head - 1 in pos
            if tail:
                assert n - 1 in pos
            if body >= 2 * g.chunk:
                assert head + g.chunk in pos and head + 2 * g.chunk - 1 in pos


def test_bitplane_and_byte_value_patterns_match_the_oracle():
    for n in (1, 2, 3, 127, 128, 1000, 4099, 65536 + 77):
        for bit in SC.bitplane_bits(n):
            for comp, value in ((False, 0x80), (True, 0x01)):
                buf = np.full(n, 0x33, dtype=np.uint8)
                SC.fill_bitplane(buf, bit, value, comp)
                i = np.arange(n)
                want = np.where(((i >> bit) & 1) == (0 if comp else 1), value, 0).astype(np.uint8)
                assert np.array_equal(buf, want), (n, bit, comp)
                expect = n - SC.bitplane_count(n, bit) if comp else SC.bitplane_count(n, bit)
                assert SO.count_nonzero_c(buf) == expect
    for v in (0x01, 0x80, 0xFF):
        assert SO.count_nonzero_c(np.full(4099, v, dtype=np.uint8)) == 4099


def test_exhaustive_word_count_identity():
    """4 bytes x 255 non-zero values x 2^24 words each: the expected count of the 2^32-word test."""
    assert 4 * 255 * (1 << 24) == 17_112_760_320 > 1 << 32
    w = np.arange(1 << 16, dtype=np.uint32)
    lo = np.count_nonzero(w.view(np.uint8).reshape(-1, 4)[:, :2])     # low two bytes over 2^16 values
    assert lo == 2 * 255 * 256
