"""The residue census on one H100: both census kernels against the numpy dirt oracle at every tiling edge and above
2^32 bytes, the product call's report under scrub_poison and scrub_residue in every mapping mode, both checks, the
fallback and the fan-out, census calls against the same calls without it, the worker, the CLI and the manager, and
the kernels' rates against a same-run copy."""
from __future__ import annotations

import ctypes as C
import json
import logging
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "oracle"))
import dirt_oracle as DO  # noqa: E402
import product_gate_calls as PGC  # noqa: E402
import product_plan as PP  # noqa: E402
import scenarios as SC  # noqa: E402
import tag_oracle as TO  # noqa: E402
from k8s_cc_manager_b200 import _native as N  # noqa: E402
from k8s_cc_manager_b200 import devices as D  # noqa: E402

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

GiB, MiB, KiB = 1 << 30, 1 << 20, 1 << 10
CHUNK = 128 * KiB
GUARD = 256 * KiB
DRILL_KEYS = PP.DRILL_KEYS + ("tag_inject", "scrub_alias", "scrub_residue")
SEED = 0x5EED1234


@pytest.fixture(scope="module")
def lib():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return PGC.open_lib()


@pytest.fixture(autouse=True)
def _own_stream():
    if not torch.cuda.is_available():
        yield
        return
    with torch.cuda.stream(torch.cuda.Stream()):
        yield
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def census(lib, ptr, n, tags, seed=SEED) -> D.ResidueReport:
    r = N.ResidueReport()
    assert lib.ccm_region_census(0, C.c_void_p(ptr), n, int(tags), seed, stream(), C.byref(r)) == 0, N.last_error()
    assert r.located == 1 and r.va_base == ptr and r.bytes_examined == n
    return D.ResidueReport.from_native(r)


def assert_matches_oracle(rep: D.ResidueReport, want: dict, what):
    assert rep.residue_bytes == want["nonzero_bytes"], what
    assert rep.residue_windows == want["dirty_windows"], what
    if want["dirty_windows"]:
        assert (rep.first_offset, rep.last_offset) == (want["first_offset"], want["last_offset"]), what
    else:
        assert (rep.first_offset, rep.last_offset, rep.records) == (0, 0, []), what
    got = [(r.offset, r.mask) for r in rep.records]
    exp = [(o, m) for o, m, _ in want["windows"]]
    assert all(r.chunk == 0 for r in rep.records)
    if not want["truncated"]:
        assert not rep.truncated and got == exp, what
    else:
        assert rep.truncated and len(got) == DO.RECORDS == len(set(got)) and got == sorted(got), what
        assert set(got) <= set(exp), what


def lengths(sm_count):
    return [1, 15, 16, 17, CHUNK - 1, CHUNK + 1, 2 * CHUNK * sm_count + 7]


OFFSETS = [0, 1, 3, 8, 15]


# ------------------------------------------------------------------------- kernel exactness
def content(kind, n, rng):
    if kind == "sparse":
        x = np.zeros(n, dtype=np.uint8)
        picks = rng.choice(n, size=min(n, 5), replace=False)
        x[picks] = rng.integers(1, 256, picks.size)
        x[n - 1] = 0x80
        return x
    if kind == "patterned":
        x = rng.integers(0, 256, n, dtype=np.uint8)
        x[rng.random(n) < 0.9] = 0
        return x
    return rng.integers(1, 256, n, dtype=np.uint8)               # flooded: every byte non-zero


@pytest.mark.parametrize("tags", [0, 1])
def test_every_tiling_edge_matches_the_oracle(lib, tags):
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    top = max(lengths(sm)) + 32
    buf = torch.empty(GUARD + top + GUARD, dtype=torch.uint8, device="cuda")
    rng = np.random.default_rng(11 + tags)
    seen = set()
    for n in lengths(sm):
        for off in OFFSETS:
            for kind in ("sparse", "patterned", "flooded"):
                host = np.full(GUARD + top + GUARD, 0xEE, dtype=np.uint8)
                host[GUARD + off: GUARD + off + n] = content(kind, n, rng)
                buf.copy_(torch.from_numpy(host))
                ptr = buf.data_ptr() + GUARD + off
                want = DO.report(host[GUARD + off: GUARD + off + n], ptr)
                rep = census(lib, ptr, n, tags)
                assert_matches_oracle(rep, want, (n, off, kind, tags))
                after = buf.cpu().numpy()
                region = after[GUARD + off: GUARD + off + n]
                if tags:
                    assert np.array_equal(region, TO.tag_bytes(SEED, ptr, n)), (n, off, kind, "not the tags")
                else:
                    assert not region.any(), (n, off, kind, "region not zeroed")
                assert np.all(after[:GUARD + off] == 0xEE) and np.all(after[GUARD + off + n:] == 0xEE), (n, off)
                seen.add("truncated" if want["truncated"] else "exact")
            # a clean region books nothing (and the book was left empty by the calls above)
            buf.zero_()
            clean = census(lib, buf.data_ptr() + GUARD + off, n, tags)
            assert (clean.residue_bytes, clean.residue_windows, clean.records) == (0, 0, [])
    assert seen == {"exact", "truncated"}


def test_records_carry_no_bytes():
    assert C.sizeof(N.ResidueRecord) == 16 and [f for f, _ in N.ResidueRecord._fields_] == ["offset", "chunk", "mask",
                                                                                           "reserved"]
    assert set(D.ResidueWindow.__dataclass_fields__) == {"offset", "chunk", "mask"}


def test_count_above_2_to_the_32(lib):
    n = 17 * GiB + 5
    buf = torch.empty(n + 16, dtype=torch.uint8, device="cuda")
    buf.fill_(0x11)
    ptr = buf.data_ptr() + 3
    rep = census(lib, ptr, n, 0)
    assert rep.residue_bytes == n > 1 << 32
    assert rep.residue_windows == DO.window_count(ptr, n)
    assert (rep.first_offset, rep.last_offset) == (0, n - 1)
    assert rep.truncated and len(rep.records) == DO.RECORDS
    nz = C.c_uint64()
    assert lib.ccm_region_verify(0, C.c_void_p(ptr), n, 0, None, stream(), C.byref(nz), None) == 0
    assert nz.value == 0
    host = buf[:3].cpu().numpy().tolist() + buf[-13:].cpu().numpy().tolist()
    assert host == [0x11] * 16                                  # the bytes around the region
    del buf


# ------------------------------------------------------------------------------ product call
def product(lib, nbytes, env=None, drills=None, check="zero", residue=True, many=False):
    drills = drills or {}
    with PGC.knobs(env or {}):
        for k in DRILL_KEYS:
            assert lib.ccm_sim_set(0, k.encode(), int(drills.get(k, 0))) == 0
        try:
            tag = N.TagResult() if check == "tagged" else None
            res, rr = N.ScrubResult(), N.ResidueReport()
            tag_p = C.byref(tag) if tag is not None else None
            l0 = lib.ccm_kernel_launches()
            if many:
                devs, wall = (C.c_int * 1)(0), C.c_double()
                if residue:
                    rc = lib.ccm_scrub_verify_many_residue(1, devs, nbytes, tag_p, C.byref(rr), C.byref(res),
                                                           C.byref(wall))
                elif tag is not None:
                    rc = lib.ccm_scrub_verify_many_tagged(1, devs, nbytes, tag_p, C.byref(res), C.byref(wall))
                else:
                    rc = lib.ccm_scrub_verify_many(1, devs, nbytes, C.byref(res), C.byref(wall))
            elif residue:
                rc = lib.ccm_scrub_verify_residue(0, nbytes, tag_p, C.byref(rr), C.byref(res))
            elif tag is not None:
                rc = lib.ccm_scrub_verify_tagged(0, nbytes, tag_p, C.byref(res))
            else:
                rc = lib.ccm_scrub_verify(0, nbytes, C.byref(res))
            launches = lib.ccm_kernel_launches() - l0
        finally:
            for k in DRILL_KEYS:
                lib.ccm_sim_set(0, k.encode(), 0)
    PGC.release_wait(lib)
    return rc, res, tag, D.ResidueReport.from_native(rr), launches


CHECKS = ["zero", "tagged"]


@pytest.mark.parametrize("check", CHECKS)
@pytest.mark.parametrize("mf,il", PP.MODES)
def test_scrub_poison_is_counted_whole(lib, check, mf, il):
    rc, res, tag, rr, _ = product(lib, 4 * GiB, PP.mode_env(mf, il), {"scrub_poison": PP.POISON}, check)
    assert rc == 0 and res.nonzero_bytes == 0 and (tag is None or tag.mismatch_bytes == 0)
    assert rr.located and rr.residue_bytes == rr.bytes_examined == res.bytes_scrubbed
    assert rr.residue_windows == res.bytes_scrubbed // 16 and rr.truncated
    assert (rr.first_offset, rr.last_offset) == (0, res.bytes_scrubbed - 1)
    assert all(r.mask == 0xFFFF for r in rr.records)


@pytest.mark.parametrize("check", CHECKS)
@pytest.mark.parametrize("env", [{"CCM_PIPELINE": "0", "CCM_ARENA_MAX_SEGMENT_MB": "96"}, {}],
                         ids=["fallback", "whole_hbm"])
def test_scrub_poison_on_the_fallback_and_at_whole_hbm(lib, check, env):
    nbytes = 300 * MiB if env else 0
    rc, res, tag, rr, _ = product(lib, nbytes, env, {"scrub_poison": PP.POISON}, check)
    assert rc == 0 and rr.located and rr.residue_bytes == res.bytes_scrubbed > 0
    assert rr.bytes_examined == res.bytes_scrubbed


def check_residue_drill(rc, res, rr, mappings, k):
    offs = PP.inject_offsets(mappings, k)
    assert rc == 0 and res.nonzero_bytes == 0
    assert rr.located and rr.residue_bytes == rr.residue_windows == len(offs) > 0
    assert (rr.first_offset, rr.last_offset) == (min(offs), max(offs))
    assert not rr.truncated and len(rr.records) == len(offs)
    got = [r.offset + r.mask.bit_length() - 1 for r in rr.records]
    assert all(bin(r.mask).count("1") == 1 for r in rr.records)
    assert got == sorted(offs)
    for r, o in zip(rr.records, got):
        assert [i for i, (co, cn) in enumerate(mappings) if co <= o < co + cn] == [r.chunk], r


@pytest.mark.parametrize("check", CHECKS)
@pytest.mark.parametrize("mf,il", PP.MODES)
@pytest.mark.parametrize("k", [3, 1000])
def test_scrub_residue_offsets_and_chunks(lib, check, mf, il, k):
    env = PP.mode_env(mf, il)
    nbytes = 4 * GiB
    rc, res, tag, rr, _ = product(lib, nbytes, env, {"scrub_residue": k}, check)
    p = PP.plan(nbytes, res.device_free_before, PP.H100_GRAN, env)
    check_residue_drill(rc, res, rr, PP.simulate(p, None).chunks, k)


@pytest.mark.parametrize("check", CHECKS)
@pytest.mark.parametrize("k", [3, 1000])
def test_scrub_residue_on_the_fallback(lib, check, k):
    env = {"CCM_PIPELINE": "0", "CCM_ARENA_MAX_SEGMENT_MB": "96"}
    rc, res, tag, rr, _ = product(lib, 300 * MiB, env, {"scrub_residue": k}, check)
    segs = PP.arena_segments(300 * MiB, res.device_free_before, env)
    assert res.segments == len(segs) == 4
    check_residue_drill(rc, res, rr, segs, k)


@pytest.mark.parametrize("check", CHECKS)
@pytest.mark.parametrize("k", [3, 1000])
def test_scrub_residue_in_the_one_gpu_fan_out(lib, check, k):
    rc, res, tag, rr, _ = product(lib, 4 * GiB, {}, {"scrub_residue": k}, check, many=True)
    p = PP.plan(4 * GiB, res.device_free_before, PP.H100_GRAN, {}, node_fanout=False)
    check_residue_drill(rc, res, rr, PP.simulate(p, None).chunks, k)


RESULT_FIELDS = [f for f in PGC.FIELDS if f != "device_free_before"]


@pytest.mark.parametrize("check", CHECKS)
@pytest.mark.parametrize("env,drills", [
    ({"CCM_MAP_FIRST": "0"}, {}), ({"CCM_MAP_FIRST": "1"}, {"scrub_inject": 5}),
    ({"CCM_MAP_FIRST": "0", "CCM_INTERLEAVE_VERIFY": "0"}, {"scrub_flood": PP.FLOOD, "tag_inject": 2}),
    ({"CCM_PIPELINE": "0", "CCM_ARENA_MAX_SEGMENT_MB": "96"}, {"scrub_inject": 3}),
    ({"CCM_SCRUB_VARIANT": "st128"}, {"scrub_residue": 7}),
])
def test_census_calls_launch_and_return_what_plain_calls_do(lib, check, env, drills):
    nbytes = 300 * MiB if "CCM_PIPELINE" in env else 4 * GiB
    rc0, res0, tag0, _, l0 = product(lib, nbytes, env, drills, check, residue=False)
    rc1, res1, tag1, rr, l1 = product(lib, nbytes, env, drills, check, residue=True)
    assert rc1 == rc0 and l1 == l0
    assert {f: getattr(res1, f) for f in RESULT_FIELDS} == {f: getattr(res0, f) for f in RESULT_FIELDS}
    if tag0 is not None:
        assert tag1.mismatch_bytes == tag0.mismatch_bytes
    assert rr.located and rr.bytes_examined == res1.bytes_scrubbed


@pytest.mark.parametrize("check", CHECKS)
@pytest.mark.parametrize("nbytes", [4 * GiB, 0])
def test_clean_calls_are_self_consistent(lib, check, nbytes):
    rc, res, tag, rr, _ = product(lib, nbytes, {}, {}, check)
    assert rc == 0 and rr.located and rr.bytes_examined == res.bytes_scrubbed
    assert rr.residue_windows <= rr.residue_bytes <= 16 * rr.residue_windows
    assert len(rr.records) == min(rr.residue_windows, DO.RECORDS) and bool(rr.truncated) == (rr.residue_windows > 64)
    if rr.residue_bytes:
        assert rr.first_offset <= rr.last_offset < res.bytes_scrubbed
    print(f"{check} {nbytes}: {rr.summary()}")


def test_pinned_variants_do_not_apply_to_census_calls(lib):
    rc, res, _, rr, _ = product(lib, GiB, {"CCM_SCRUB_VARIANT": "memset"}, {"scrub_residue": 2})
    assert rc == 0 and res.scrub_variant == N.SCRUB_ST128 and rr.residue_bytes == 2
    rc, res, _, _, _ = product(lib, GiB, {"CCM_SCRUB_VARIANT": "memset"}, {}, residue=False)
    assert rc == 0 and res.scrub_variant == N.SCRUB_MEMSET


# ----------------------------------------------------------------------------------- end to end
def test_device_worker_and_cli_carry_the_report(lib):
    from k8s_cc_manager_b200 import scrub_worker
    gpu = next(d for d in D.find_gpus()[0] if d.cuda_ordinal == 0)
    lib.ccm_sim_set(gpu.index, b"scrub_residue", 3)
    try:
        rep = gpu.scrub_and_verify(GiB, residue=True)
        assert rep.clean and rep.residue.residue_bytes == 3 and rep.residue.located
        PGC.release_wait(lib)
        js = scrub_worker.run([gpu.bdf], GiB, "tagged", residue=True)["reports"][0]
        assert js["residue"]["residue_bytes"] == 3 and js["mismatch_bytes"] == 0
        assert D.ScrubReport.from_json(js).residue == D.ResidueReport.from_json(js["residue"])
        PGC.release_wait(lib)
        cli = ROOT / "k8s_cc_manager_b200" / "ccm-scrub"
        out = subprocess.run([str(cli), "--backend", "cudasim", "--bytes", str(GiB), "--residue", "--bdf", gpu.bdf],
                             capture_output=True, text=True, timeout=300)
        assert out.returncode == 0, out.stderr
        js = json.loads(out.stdout.strip().splitlines()[-1])["reports"][0]
        rr = D.ResidueReport.from_json(js["residue"])     # the CLI's own process: no drill, whatever the driver left
        assert rr.located and rr.bytes_examined == js["bytes_scrubbed"]
    finally:
        lib.ccm_sim_set(gpu.index, b"scrub_residue", 0)
        PGC.release_wait(lib)
    reps, _ = D.scrub_and_verify_many([gpu], GiB)
    assert reps[0].residue is None and "residue" not in reps[0].as_json()
    PGC.release_wait(lib)


def test_manager_transition_logs_the_residue(lib, monkeypatch, caplog):
    import kubernetes
    from k8s_cc_manager_b200 import manager
    for k, v in dict(EVICT_OPERATOR_COMPONENTS="false", CC_RELEASE_CUDA_CONTEXT="false",
                     CC_SCRUB_RESIDUE="report").items():
        monkeypatch.setenv(k, v)
    assert lib.ccm_init(N.BACKEND_CUDASIM) == 0
    lib.ccm_sim_set(-1, b"cc_mode", N.CC_MODES["off"])
    lib.ccm_sim_set(0, b"scrub_residue", 4)
    try:
        c = kubernetes.reset_cluster()
        c.add_node(SC.NODE, {})
        mgr = manager.CCManager(SC.NODE, "on", True, device_source=D.find_gpus, scrub_bytes=4 * GiB)
        with caplog.at_level(logging.INFO, logger="k8s-cc-manager"):
            assert mgr.set_cc_mode("on") is True
        bdf = next(d.bdf for d in D.find_gpus()[0] if d.cuda_ordinal == 0)
        rr = mgr.last_transition["scrub_residue"][bdf]
        assert rr.residue_bytes == 4
        assert sum(f"HBM residue on {bdf}: 4 of " in r.getMessage() for r in caplog.records) == 1
    finally:
        lib.ccm_sim_set(0, b"scrub_residue", 0)
        for d in D.find_gpus()[0]:
            if d.is_gpu():
                d.wait_scrub_released()


# ------------------------------------------------------------------------------------- rate
def _best(fn, prep, reps=5):
    ts = []
    for _ in range(reps + 1):
        prep()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return min(ts[1:])


@pytest.mark.parametrize("tags", [0, 1])
@pytest.mark.parametrize("residue", ["clean", "sparse", "every_byte"])
def test_census_keeps_up_with_a_copy(lib, tags, residue):
    """Rates in bytes moved (read + written) per second, against a same-run torch copy_ of half the size."""
    n = 16 * GiB
    buf = torch.empty(n, dtype=torch.uint8, device="cuda")
    src = torch.empty(n // 2, dtype=torch.uint8, device="cuda")
    dst = torch.empty(n // 2, dtype=torch.uint8, device="cuda")
    p, st = buf.data_ptr(), stream()
    rr = N.ResidueReport()
    step = 32 * MiB

    def prep():
        if residue == "every_byte":
            buf.fill_(0x5A)
        else:
            buf.zero_()
            if residue == "sparse":
                buf[torch.arange(0, n, step, device="cuda")] = 0xA5

    run = lambda: lib.ccm_region_census(0, C.c_void_p(p), n, tags, SEED, st, C.byref(rr))  # noqa: E731
    t_census = _best(run, prep)
    assert rr.residue_bytes == {"clean": 0, "sparse": n // step, "every_byte": n}[residue]
    t_copy = _best(lambda: dst.copy_(src), lambda: None)
    ratio = t_copy / t_census          # copy_ moves n bytes in t_copy; the census moves 2n in t_census
    ratio *= 2
    print(f"census tags={tags} {residue}: {2 * n / t_census / 1e6:.0f} GB/s moved, copy_ {n / t_copy / 1e6:.0f} GB/s "
          f"({ratio:.3f}x)")
    assert ratio >= (0.75 if residue == "every_byte" else 0.85)
