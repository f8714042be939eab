"""The tagged scrub gate on one H100: exact writes and exact mismatch counts of the two kernels through the
region entry points, the tagged product call in every mapping mode and under every drill, the alias drill
that the zero gate passes and the tagged gate must not, the manager end to end, and the kernels' rates."""
from __future__ import annotations

import ctypes as C
import os
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "oracle"))
import product_gate_calls as PGC  # noqa: E402
import product_plan as PP  # noqa: E402
import scenarios as SC  # noqa: E402
import tag_oracle as TO  # noqa: E402
from k8s_cc_manager_b200 import _native as N  # noqa: E402

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

GiB, MiB, KiB = 1 << 30, 1 << 20, 1 << 10
GUARD = 256 * KiB
CHUNK = 128 * KiB                       # bytes per grab of both tag kernels
TAG_KEYS = ("tag_inject", "scrub_alias")


@pytest.fixture(scope="module")
def lib():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return PGC.open_lib()


@pytest.fixture(autouse=True)
def _own_stream():
    """Every test runs on a torch stream of its own and hands that stream to the library, so torch's copies
    and fills and the library's launches are ordered.  (The default stream's handle is NULL, which the
    library reads as "its own stream".)"""
    if not torch.cuda.is_available():
        yield
        return
    with torch.cuda.stream(torch.cuda.Stream()):
        yield
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def fill(lib, ptr, n, seed):
    assert lib.ccm_region_tag_fill(0, C.c_void_p(ptr), n, seed, stream(), None) == 0, N.last_error()


def check(lib, ptr, n, seed):
    mm = C.c_uint64()
    assert lib.ccm_region_tag_check_zero(0, C.c_void_p(ptr), n, seed, stream(), C.byref(mm), None) == 0, N.last_error()
    return mm.value


def verify(lib, ptr, n):
    nz = C.c_uint64()
    assert lib.ccm_region_verify(0, C.c_void_p(ptr), n, N.VERIFY_AUTO, None, stream(), C.byref(nz), None) == 0
    return nz.value


def lengths(sm_count):
    return [0, 1, 15, 16, 17, CHUNK - 1, CHUNK + 1, 2 * CHUNK * sm_count + 7]


OFFSETS = [0, 1, 3, 8, 15]


# ------------------------------------------------------------------------- kernel exactness
def test_fill_writes_exactly_the_tags_and_check_zeroes_exactly_the_region(lib):
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    top = max(lengths(sm)) + 16
    buf = torch.empty(GUARD + top + GUARD, dtype=torch.uint8, device="cuda")
    for n in lengths(sm):
        for off in OFFSETS:
            seed = (0x1000193 * (n + 1) + off) & 0xFFFFFFFF or 1
            buf.fill_(0xEE)
            ptr = buf.data_ptr() + GUARD + off
            fill(lib, ptr, n, seed)
            host = buf.cpu().numpy()
            lo, hi = GUARD + off, GUARD + off + n
            assert np.all(host[:lo] == 0xEE) and np.all(host[hi:] == 0xEE), (n, off)
            assert np.array_equal(host[lo:hi], TO.tag_bytes(seed, ptr, n)), (n, off)
            assert check(lib, ptr, n, seed) == 0, (n, off)
            assert verify(lib, ptr, n) == 0, (n, off)
            host = buf.cpu().numpy()
            assert np.all(host[:lo] == 0xEE) and np.all(host[hi:] == 0xEE), (n, off)
            assert not host[lo:hi].any()


def test_dirt_at_every_edge_is_counted_exactly(lib):
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    n_max = 2 * CHUNK * sm + 7
    buf = torch.zeros(GUARD + n_max + 16 + GUARD, dtype=torch.uint8, device="cuda")
    for n in (CHUNK + 1, n_max):
        for off in OFFSETS:
            ptr = buf.data_ptr() + GUARD + off
            head = (128 - ptr % 128) % 128
            body_end = head + (n - head) // 16 * 16
            marks = {0, n - 1, head - 1, head, body_end - 1, body_end}
            marks |= {head + k * CHUNK + d for k in (1, 2, (n - head) // CHUNK) for d in (-1, 0)}
            marks = sorted(m for m in marks if 0 <= m < n)
            seed = 0xC0FFEE + off
            fill(lib, ptr, n, seed)
            region = buf[GUARD + off: GUARD + off + n]
            idx = torch.tensor(marks, device="cuda")
            region[idx] = region[idx] ^ 0x5A
            got = region.cpu().numpy()
            assert TO.mismatch_count(got, seed, ptr) == len(marks)
            assert check(lib, ptr, n, seed) == len(marks), (n, off)
            assert verify(lib, ptr, n) == 0


def test_a_wrong_seed_counts_above_2_to_the_32(lib):
    n = 5 * GiB + 3
    buf = torch.empty(n + 16, dtype=torch.uint8, device="cuda")
    ptr = buf.data_ptr() + 5
    written, checked = 0x11111111, 0x22222222          # xor 0x33333333: every byte differs
    fill(lib, ptr, n, written)
    assert TO.wrong_seed_count(written, checked, ptr, 1 << 20) == 1 << 20
    got = check(lib, ptr, n, checked)
    assert got == n and got > 1 << 32
    assert verify(lib, ptr, n) == 0
    # two seeds that share two bytes: half the bytes differ, per the oracle
    m = 64 * MiB + 5
    fill(lib, ptr, m, 0x00FF00FF)
    assert check(lib, ptr, m, 0x00FFAAFF) == TO.wrong_seed_count(0x00FF00FF, 0x00FFAAFF, ptr, m)


# ------------------------------------------------------------------------------ product call
def tagged(lib, nbytes, env=None, drills=None, seed=0):
    drills = drills or {}
    with PGC.knobs(env or {}):
        for k in PP.DRILL_KEYS + TAG_KEYS:
            assert lib.ccm_sim_set(0, k.encode(), int(drills.get(k, 0))) == 0
        try:
            tag, res = N.TagResult(seed=seed), N.ScrubResult()
            rc = lib.ccm_scrub_verify_tagged(0, nbytes, C.byref(tag), C.byref(res))
        finally:
            for k in PP.DRILL_KEYS + TAG_KEYS:
                lib.ccm_sim_set(0, k.encode(), 0)
    PGC.release_wait(lib)
    return rc, tag, res


def zero(lib, nbytes, env=None, drills=None):
    drills = drills or {}
    with PGC.knobs(env or {}):
        for k in PP.DRILL_KEYS + TAG_KEYS:
            assert lib.ccm_sim_set(0, k.encode(), int(drills.get(k, 0))) == 0
        try:
            res = N.ScrubResult()
            rc = lib.ccm_scrub_verify(0, nbytes, C.byref(res))
        finally:
            for k in PP.DRILL_KEYS + TAG_KEYS:
                lib.ccm_sim_set(0, k.encode(), 0)
    PGC.release_wait(lib)
    return rc, res


def free_bytes():
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return torch.cuda.mem_get_info()[0]


MODES = {"pipelined": {"CCM_MAP_FIRST": "0"}, "map_first": {"CCM_MAP_FIRST": "1"}, "arena": {"CCM_PIPELINE": "0"}}


def ranges_of(nbytes, env, res):
    if env.get("CCM_PIPELINE") == "0":
        return PP.arena_segments(nbytes, res.device_free_before, env)
    p = PP.plan(nbytes, res.device_free_before, PP.H100_GRAN, env)
    return PP.simulate(p, None).ranges(p)


@pytest.mark.parametrize("mode", sorted(MODES))
@pytest.mark.parametrize("nbytes", [GiB + 3 * MiB, 4 * GiB, 0])
def test_clean_tagged_calls(lib, mode, nbytes):
    env = MODES[mode]
    before = free_bytes()
    rc, tag, res = tagged(lib, nbytes, env)
    assert rc == 0, N.last_error()
    assert tag.mismatch_bytes == 0 and res.nonzero_bytes == 0 and tag.seed != 0
    assert res.bytes_scrubbed >= nbytes and tag.ms_tag > 0 and tag.ms_check > 0
    if nbytes == 0:
        assert res.bytes_scrubbed / res.device_total_bytes > 0.98
    assert free_bytes() >= before - 64 * MiB


@pytest.mark.parametrize("mode", sorted(MODES))
@pytest.mark.parametrize("drill", ["poison", "flood", "inject"])
def test_zero_gate_drills_give_the_same_verdict_in_tagged_mode(lib, mode, drill):
    env, nbytes = MODES[mode], 4 * GiB
    rc, tag, res = tagged(lib, nbytes, env, PP.DRILLS[drill])
    want = PP.expected_count(drill, ranges_of(nbytes, env, res), res.bytes_scrubbed)
    assert tag.mismatch_bytes == 0
    assert res.nonzero_bytes == want
    assert rc == (N.ERR_DIRTY if want else 0)


@pytest.mark.parametrize("mode", sorted(MODES))
@pytest.mark.parametrize("k", [3, 1000])
def test_tag_inject_is_counted_exactly(lib, mode, k):
    env, nbytes = MODES[mode], 4 * GiB
    rc, tag, res = tagged(lib, nbytes, env, {"tag_inject": k})
    want = len(PP.inject_offsets(ranges_of(nbytes, env, res), k))
    assert want == min(k, 4 * len(ranges_of(nbytes, env, res)))
    assert rc == N.ERR_MISMATCH and tag.mismatch_bytes == want and res.nonzero_bytes == 0


def test_mismatch_takes_precedence_over_dirt(lib):
    rc, tag, res = tagged(lib, 4 * GiB, {}, {"tag_inject": 2, "scrub_inject": 5})
    assert rc == N.ERR_MISMATCH and tag.mismatch_bytes == 2 and res.nonzero_bytes == 5


# ---------------------------------------------------------------------------------- aliasing
@pytest.mark.parametrize("nbytes", [4 * GiB, 0])
def test_alias_passes_the_zero_gate(lib, nbytes):
    free_bytes()
    rc, res = zero(lib, nbytes, {}, {"scrub_alias": 1})
    assert rc == 0 and res.nonzero_bytes == 0, N.last_error()
    assert res.bytes_scrubbed / res.device_total_bytes > 0.99 if nbytes == 0 else res.bytes_scrubbed == nbytes


@pytest.mark.parametrize("mode", ["pipelined", "map_first"])
@pytest.mark.parametrize("nbytes", [4 * GiB, 0])
def test_alias_fails_the_tagged_gate(lib, mode, nbytes):
    before = free_bytes()
    rc, tag, res = tagged(lib, nbytes, MODES[mode], {"scrub_alias": 1})
    assert rc == N.ERR_MISMATCH and res.nonzero_bytes == 0
    n0 = GiB                                             # the first chunk: CCM_VMM_FIRST_CHUNK_MB default
    exact, low, high = TO.alias_counts(tag.seed, tag.va_base, n0)
    if mode == "pipelined":                              # the two views are checked by separate launches
        assert tag.mismatch_bytes == exact
    else:                                                # one launch covers both views
        assert low <= tag.mismatch_bytes <= high
    assert free_bytes() >= before - 64 * MiB


def test_alias_is_ignored_on_the_arena_fallback(lib):
    rc, tag, res = tagged(lib, 4 * GiB, MODES["arena"], {"scrub_alias": 1})
    assert rc == 0 and tag.mismatch_bytes == 0


# ------------------------------------------------------------------------------------- rates
def _best(fn, reps=5, before=None):
    ts = []
    for _ in range(reps + 1):
        if before is not None:
            before()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return min(ts[1:])


def test_kernel_rates_against_memset_and_copy(lib):
    n = 16 * GiB
    buf = torch.empty(n, dtype=torch.uint8, device="cuda")
    p = buf.data_ptr()
    st = stream()
    t_memset = _best(lambda: lib.ccm_region_scrub(0, C.c_void_p(p), n, N.SCRUB_MEMSET, None, st, None))
    t_fill = _best(lambda: lib.ccm_region_tag_fill(0, C.c_void_p(p), n, 7, st, None))
    t_check = _best(lambda: lib.ccm_region_tag_check_zero(0, C.c_void_p(p), n, 7, st, None, None),
                    before=lambda: lib.ccm_region_tag_fill(0, C.c_void_p(p), n, 7, st, None))
    half = n // 2
    src, dst = buf[:half], buf[half:]
    t_copy = _best(lambda: dst.copy_(src))
    fill_rate, memset_rate = n / t_fill, n / t_memset
    check_rate, copy_rate = 2 * n / t_check, 2 * half / t_copy
    print(f"fill {fill_rate / 1e6:.0f} GB/s memset {memset_rate / 1e6:.0f} GB/s "
          f"check {check_rate / 1e6:.0f} GB/s copy {copy_rate / 1e6:.0f} GB/s")
    assert fill_rate >= 0.85 * memset_rate
    assert check_rate >= 0.85 * copy_rate


# ------------------------------------------------------------------------------------ manager
@pytest.mark.parametrize("alias", [0, 1])
def test_manager_tagged_transition(lib, alias, monkeypatch):
    import kubernetes
    from k8s_cc_manager_b200 import devices as D
    from k8s_cc_manager_b200 import manager
    for k, v in dict(EVICT_OPERATOR_COMPONENTS="false", CC_SCRUB_CHECK="tagged",
                     CC_RELEASE_CUDA_CONTEXT="false").items():
        monkeypatch.setenv(k, v)
    assert lib.ccm_init(N.BACKEND_CUDASIM) == 0
    lib.ccm_sim_set(-1, b"cc_mode", N.CC_MODES["off"])
    lib.ccm_sim_set(0, b"scrub_alias", alias)
    try:
        c = kubernetes.reset_cluster()
        c.add_node(SC.NODE, {})
        mgr = manager.CCManager(SC.NODE, "on", True, device_source=D.find_gpus, scrub_bytes=4 * GiB)
        assert mgr.set_cc_mode("on") is (alias == 0)
        assert c.labels(SC.NODE).get("nvidia.com/cc.mode.state") == ("on" if alias == 0 else "failed")
    finally:
        lib.ccm_sim_set(0, b"scrub_alias", 0)
        for d in D.find_gpus()[0]:
            if d.is_gpu():
                d.wait_scrub_released()
