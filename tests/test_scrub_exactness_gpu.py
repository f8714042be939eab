"""Exactness of every scrub and verify kernel the library can launch (-m gpu, run on an H100).

* scrub matrix: every scrub_st_kernel / scrub_tma_kernel instantiation, memset and the default kernel
  on caller-owned memory at five start offsets and lengths taken from each launch's own tiling, inside
  guards at least one grab (and 256 KiB) wide; the WHOLE buffer must read back sentinel / zero / sentinel;
* verify matrix: every verify_ld_kernel instantiation under every schedule and the default verifier
  count a zero region, dirt at the edges of the decomposition, address bit-planes and byte-value edges
  exactly, with non-zero guards around the region;
* every 32-bit word once (16 GiB): the count is 4 x 255 x 2^24, above 2^32;
* the proving twins of the default kernels (include/ccm.h: ccm_region_prove) once more at every placement of the
  default scrub and verifier and over the 16 GiB: the same bytes and counts, and a cover map equal to the oracle's
  (tests/report_cover_oracle.py), with page boundaries inside the head, a chunk, a vector and the tail; every other
  variant armed at its first placement counts nothing;
* launch-to-launch state of the default kernels, with and without programmatic dependent launch;
* the product gate under every variant pair and to the last byte of a whole-HBM call.
Cases and patterns come from tests/scrub_cases.py (checked on the CPU by
tests/test_scrub_matrix_coverage.py).  Bar: bit-exact."""
from __future__ import annotations

import ctypes as C
import json
import os
import subprocess
import sys
from pathlib import Path

import pytest

import scrub_cases as SC
from region_cover_calls import ArmedMap
from k8s_cc_manager_b200 import _native as N

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parents[1]
SENTINEL = 0xEE
GiB = 1 << 30


def ok(rc, what=""):
    assert rc == 0, f"{what}: {N.strerror(rc)}: {N.last_error()}"


@pytest.fixture(scope="module")
def lib():
    L = N.lib()
    ok(L.ccm_init(N.BACKEND_CUDASIM), "init cudasim")
    n = C.c_int()
    ok(L.ccm_enumerate(None, 0, C.byref(n)))
    assert n.value >= 1, "no CUDA device visible: the gpu-marked tests need an H100"
    return L


@pytest.fixture(scope="module")
def dev():
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    stream = torch.cuda.Stream()
    yield torch, stream, C.c_void_p(stream.cuda_stream), sms
    stream.synchronize()
    torch.cuda.empty_cache()


def cfg_ref(case):
    kw = case.cfg_kwargs()
    if kw is None:
        return None
    return C.byref(N.launch_cfg(ctas_per_sm=kw["ctas_per_sm"], threads=kw["threads"], tile_bytes=kw["tile_bytes"],
                                unroll=kw["unroll"], cache_policy=kw["cache_policy"], schedule=kw["schedule"]))


def guarded_buffer(torch, max_len, guard):
    """[guard | 128 | region (<= max_len) | guard], base on a 128-byte boundary."""
    buf = torch.empty(2 * guard + 128 + max_len, dtype=torch.uint8, device="cuda")
    assert buf.data_ptr() % 128 == 0
    return buf


def test_scrub_matrix_writes_exactly_its_region(lib, dev):
    torch, stream, h, sms = dev
    plan = [(case, SC.geometry(case, sms), full) for case, full in SC.scrub_cases()]
    guard = max([256 * 1024] + [g.chunk for _, g, _ in plan])
    guard = -(-guard // 512) * 512
    max_len = max(n for case, g, full in plan for _, n in SC.placements(g, full))
    assert max_len <= SC.MAX_LENGTH
    buf = guarded_buffer(torch, max_len, guard)
    gen = torch.Generator(device="cuda").manual_seed(20261015)
    failures, runs, armed_runs = [], 0, 0
    with torch.cuda.stream(stream):
        src = torch.randint(1, 256, (max_len,), dtype=torch.uint8, device="cuda", generator=gen)
        for case, g, full in plan:
            cfg = cfg_ref(case)
            fast = SC.is_fast(case)
            for i, (o, n) in enumerate(SC.placements(g, full)):
                start, end = guard + o, guard + o + n
                ptr = buf.data_ptr() + start
                for armed in (False, True) if fast or i == 0 else (False,):
                    buf.fill_(SENTINEL)
                    buf[start:end].copy_(src[:n])
                    arm = ArmedMap(lib, ptr, n, armed_runs) if armed else None
                    if arm:
                        with arm:
                            ok(lib.ccm_region_scrub(0, C.c_void_p(ptr), n, case.variant, cfg, h, None), case.label())
                        got, want = arm.take()[0], arm.want([(ptr, n)] if fast else [])
                        armed_runs += 1
                        if got != want:
                            failures.append((case.label(), o, n, "cover map", arm.base - ptr, got, want))
                    else:
                        ok(lib.ccm_region_scrub(0, C.c_void_p(ptr), n, case.variant, cfg, h, None), case.label())
                    below = start - torch.count_nonzero(buf[:start] == SENTINEL)
                    inside = torch.count_nonzero(buf[start:end])
                    above = (buf.numel() - end) - torch.count_nonzero(buf[end:] == SENTINEL)
                    bad = torch.stack([below, inside, above]).tolist()
                    runs += 1
                    if any(bad):
                        failures.append((case.label(), o, n, armed, "below/inside/above", bad))
    stream.synchronize()
    assert not failures, f"{len(failures)} of {runs} scrubs inexact, first: {failures[:10]}"
    print(f"\nscrub matrix: {runs} scrubs over {len(plan)} launch shapes exact (guards {guard >> 10} KiB), "
          f"{armed_runs} of them armed")


def test_verify_matrix_counts_exactly(lib, dev):
    torch, stream, h, sms = dev
    groups = SC.verify_groups()
    geoms = [SC.geometry(g[0], sms) for g in groups]
    max_len = max(max(SC.lengths(g)) for g in geoms)
    guard = max([256 * 1024] + [g.chunk for g in geoms])
    guard = -(-guard // 512) * 512
    buf = guarded_buffer(torch, max_len, guard)
    failures, runs = [], [0, 0]

    def count_all(verifiers, o, n, expect, what):
        """Every verifier of the group, then the default one armed: the same count and a cover map of the region, or
        (the first count of each placement) a group verifier armed: its count and an empty map."""
        ptr = C.c_void_p(buf.data_ptr() + guard + o)
        armed = [SC.FAST_VERIFY] + ([verifiers[0]] if what == "zero" and verifiers[0] != SC.FAST_VERIFY else [])
        for case, arm in [(c, None) for c in verifiers] + [(c, ArmedMap(lib, ptr.value, n, runs[1])) for c in armed]:
            nz = C.c_uint64(1 << 63)
            if arm:
                with arm:
                    ok(lib.ccm_region_verify(0, ptr, n, case.variant, cfg_ref(case), h, C.byref(nz), None), case.label())
                got, want = arm.take()[0], arm.want([(ptr.value, n)] if case == SC.FAST_VERIFY else [])
                runs[1] += 1
                if got != want:
                    failures.append((case.label(), o, n, what, "cover map", arm.base - ptr.value, got, want))
            else:
                ok(lib.ccm_region_verify(0, ptr, n, case.variant, cfg_ref(case), h, C.byref(nz), None), case.label())
            runs[0] += 1
            if nz.value != expect:
                failures.append((case.label(), o, n, what, arm is not None, nz.value, expect))

    with torch.cuda.stream(stream):
        for group, g in zip(groups, geoms):
            verifiers = group if group[0] == SC.FAST_VERIFY else group + [SC.FAST_VERIFY]
            for o, n in SC.placements(g, full=True):
                region = buf[guard + o:guard + o + n]
                buf.fill_(SENTINEL)
                region.zero_()
                count_all(verifiers, o, n, 0, "zero")
                pos = SC.structural_positions(g, o, n)
                vals = SC.dirt_values(pos, seed=n * 131 + o)
                region[torch.tensor(pos, device="cuda")] = torch.tensor(vals, dtype=torch.uint8, device="cuda")
                count_all(verifiers, o, n, len(pos), "structural")
            o, n = 17, SC.big_length(g)
            region = buf[guard + o:guard + o + n]
            buf.fill_(SENTINEL)
            for bit in SC.bitplane_bits(n):
                for comp, value in ((False, 0x80), (True, 0x01)):
                    SC.fill_bitplane(region, bit, value, comp)
                    ones = SC.bitplane_count(n, bit)
                    count_all(verifiers, o, n, n - ones if comp else ones, f"bit {bit}{'~' if comp else ''}")
            for value in (0x01, 0x80, 0xFF):
                region.fill_(value)
                count_all(verifiers, o, n, n, f"all {value:#x}")
    stream.synchronize()
    assert not failures, f"{len(failures)} of {runs[0]} counts inexact, first: {failures[:10]}"
    print(f"\nverify matrix: {runs[0]} counts over {len(groups)} geometries exact, {runs[1]} of them armed")


def test_every_32bit_word_is_counted_exactly(lib, dev):
    """Every 32-bit pattern once: 4 x 255 x 2^24 = 17 112 760 320 non-zero bytes (above 2^32)."""
    torch, stream, h, sms = dev
    total = 1 << 34
    expect = 4 * 255 * (1 << 24)
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info(0)
    assert free >= total + 2 * GiB, f"needs 18 GiB of free HBM, {free / GiB:.1f} GiB free"
    failures = []
    with torch.cuda.stream(stream):
        words = torch.empty(1 << 32, dtype=torch.int32, device="cuda")
        step = 1 << 28
        ramp = torch.arange(step, dtype=torch.int32, device="cuda")
        for k in range(16):
            torch.add(ramp, -(1 << 31) + k * step, out=words[k * step:(k + 1) * step])
        del ramp
        raw = words.view(torch.uint8)
        assert raw.numel() == total
        by_torch = sum(int(torch.count_nonzero(raw[i:i + GiB])) for i in range(0, total, GiB))
        assert by_torch == expect
        skipped = int(torch.count_nonzero(raw[:3])) + int(torch.count_nonzero(raw[-5:]))
        for label, ptr, n, want in (("aligned", raw.data_ptr(), total, expect),
                                    ("+3/-5", raw.data_ptr() + 3, total - 8, expect - skipped)):
            for case in SC.exhaustive_verifiers():
                nz = C.c_uint64(0)
                ok(lib.ccm_region_verify(0, C.c_void_p(ptr), n, case.variant, cfg_ref(case), h, C.byref(nz), None),
                   case.label())
                if nz.value != want:
                    failures.append((case.label(), label, nz.value, want))
            # the read-back's proving twin: the same count, and every byte of the 16 GiB on its page of the map
            nz = C.c_uint64(0)
            with ArmedMap(lib, ptr, n, 0) as arm:
                ok(lib.ccm_region_verify(0, C.c_void_p(ptr), n, SC.FAST_VERIFY.variant, None, h, C.byref(nz), None),
                   "armed")
            got = arm.take()[0]
            if nz.value != want or sum(got) != n or got != arm.want([(ptr, n)]):
                failures.append(("armed", label, nz.value, want, sum(got), n, arm.pages, got[-1]))
    stream.synchronize()
    del words, raw
    torch.cuda.empty_cache()
    assert not failures, failures


def test_default_kernels_hand_back_clean_grab_state(lib, dev):
    """Dirt only in chunk 0 and the last whole chunk after each call: a grab word left non-zero by any
    earlier launch (nchunks == 0, 1 byte, multi-chunk, segmented-arena step, a proving twin, either stream)
    skips one."""
    from default_kernel_steps import launch_state_sequence
    rows = launch_state_sequence(lib)
    assert len(rows) == 13 and sum(str(r[0]).startswith("armed") for r in rows) == 4


def run_steps_child(pdl: str) -> dict:
    env = dict(os.environ, CCM_PDL=pdl)
    proc = subprocess.run([sys.executable, str(ROOT / "tests" / "default_kernel_steps.py")], capture_output=True,
                          text=True, env=env, timeout=600, cwd=str(ROOT))
    assert proc.returncode == 0, f"CCM_PDL={pdl}: exit {proc.returncode}\n{proc.stdout[-2000:]}\n{proc.stderr[-3000:]}"
    return json.loads(next(l for l in proc.stdout.splitlines() if l.startswith("RESULT "))[7:])


def test_pdl_chained_steps_match_the_plain_launches(lib):
    """CCM_PDL is latched once per process: one child with programmatic dependent launch, one without.
    Both must report the same exact results."""
    with_pdl, plain = run_steps_child("1"), run_steps_child("0")
    assert with_pdl == plain, (with_pdl, plain)
    assert all(step == [8, 0, 0] for step in with_pdl["arena_steps"]), with_pdl["arena_steps"]
    assert len(with_pdl["arena_steps"]) == 4
    assert all(r[1] == r[2] and r[3] == 0 and r[4] == 0 for r in with_pdl["sequence"])
    assert len(with_pdl["sequence"]) == 13 and sum(str(r[0]).startswith("armed") for r in with_pdl["sequence"]) == 4
    assert with_pdl["product_dirty"] == [N.ERR_DIRTY, 8, 2 << 30]


VARIANT_ENV = ("CCM_SCRUB_VARIANT", "CCM_VERIFY_VARIANT", "CCM_MAP_FIRST", "CCM_INTERLEAVE_VERIFY")


@pytest.fixture()
def restore_gate(lib):
    saved = {k: os.environ.get(k) for k in VARIANT_ENV}
    yield
    lib.ccm_sim_set(0, b"scrub_inject", 0)
    for k, v in saved.items():
        if v is None:
            os.environ.pop(k, None)
        else:
            os.environ[k] = v


@pytest.mark.parametrize("sv", ["st128", "st256", "tma", "memset"])
@pytest.mark.parametrize("vv", ["ld128", "ld256"])
def test_product_gate_under_every_variant(lib, restore_gate, sv, vv):
    os.environ["CCM_SCRUB_VARIANT"], os.environ["CCM_VERIFY_VARIANT"] = sv, vv
    res = N.ScrubResult()
    ok(lib.ccm_scrub_verify(0, 2 << 30, C.byref(res)), f"{sv}/{vv}")
    assert res.nonzero_bytes == 0 and res.bytes_scrubbed == 2 << 30
    assert (res.scrub_variant, res.verify_variant) == (N.SCRUB_VARIANTS[sv], N.VERIFY_VARIANTS[vv])
    lib.ccm_sim_set(0, b"scrub_inject", 1000)
    rc = lib.ccm_scrub_verify(0, 2 << 30, C.byref(res))
    assert rc == N.ERR_DIRTY and res.nonzero_bytes == 8, (rc, res.nonzero_bytes)   # 2 chunks x 4 candidates


def test_whole_hbm_gate_finds_dirt_in_its_last_byte(lib, dev, restore_gate):
    """One enqueue over the whole mapping: the four candidates are its first byte, byte 17, the middle
    and the last mapped byte (in the tail granules)."""
    torch = dev[0]
    torch.cuda.empty_cache()
    os.environ["CCM_MAP_FIRST"], os.environ["CCM_INTERLEAVE_VERIFY"] = "1", "0"
    lib.ccm_sim_set(0, b"scrub_inject", 4)
    res = N.ScrubResult()
    rc = lib.ccm_scrub_verify(0, 0, C.byref(res))
    assert rc == N.ERR_DIRTY and res.nonzero_bytes == 4, (rc, res.nonzero_bytes, N.last_error())
    assert res.bytes_scrubbed >= 0.95 * res.device_total_bytes
    lib.ccm_scrub_release_wait(0, None, None)
