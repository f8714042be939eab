"""The tagged scrub gate on the CPU: the address-tag oracle against its goldens and its stated
properties, the kernel header's tag against the oracle, the C ABI surface, the drill keys, and
CC_SCRUB_CHECK through every gate path of the manager, the CLI and the worker."""
from __future__ import annotations

import ctypes as C
import json
import shutil
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

import scenarios as SC
from helpers import build_native_world, sim_get, sim_set
from k8s_cc_manager_b200 import _native as N
from k8s_cc_manager_b200 import devices as D
from k8s_cc_manager_b200.devices import ScrubReport

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "oracle"))
import tag_oracle as TO  # noqa: E402

GOLDEN = json.loads((ROOT / "tests" / "golden" / "tag_vectors.json").read_text())
G16 = 16 << 30


# ---------------------------------------------------------------- oracle and pattern
def test_oracle_matches_the_pinned_vectors():
    assert (GOLDEN["k1"], GOLDEN["k2"]) == (TO.K1, TO.K2)
    assert len(GOLDEN["vectors"]) >= 50
    for v in GOLDEN["vectors"]:
        assert TO.tag_bytes(v["seed"], v["addr"], v["n"]).tobytes().hex() == v["bytes"], v


def test_tags_are_unique_within_an_aligned_16_gib_window():
    # lo32(i) -> lo32(i) * K1 is a bijection mod 2**32 (K1 odd): the inverse recovers every word index
    k1_inv = pow(TO.K1, -1, 1 << 32)
    rng = np.random.default_rng(7)
    for seed in (1, 0xDEADBEEF):
        for window in (0x7F00_0000_0000 // G16, 5):
            idx = rng.integers(0, 1 << 32, size=4096, dtype=np.uint64)
            addrs = window * G16 + idx * 4
            words = np.array([TO.tag_word_py(seed, int(a)) for a in addrs], dtype=np.uint64)
            hi = np.uint64(window * (G16 >> 2) >> 32)
            lo = ((words ^ np.uint64(seed) ^ ((hi * np.uint64(TO.K2)) & np.uint64(0xFFFFFFFF)))
                  * np.uint64(k1_inv)) & np.uint64(0xFFFFFFFF)
            assert np.array_equal(lo, idx)
    # and a dense stretch of 2**22 consecutive words ending at a 16 GiB boundary
    words = TO.tag_bytes(0x5EED, 3 * G16 - (16 << 20), 16 << 20).view("<u4")
    assert np.unique(words).size == words.size


def test_an_alias_at_any_multiple_of_16_gib_differs_in_every_word():
    addrs = np.arange(0, 1 << 20, 4, dtype=np.uint64) + np.uint64(0x7F12_3456_7000)
    base = TO.tag_bytes(42, int(addrs[0]), 1 << 20).view("<u4")
    for k in (1, 2, 3, 5, 4095):
        other = TO.tag_bytes(42, int(addrs[0]) + k * G16, 1 << 20).view("<u4")
        assert np.all(base != other), k


def test_two_seeds_differ_in_every_word():
    a = 0x7F00_0000_0010
    for s1, s2 in ((1, 2), (0x12345678, 0x12345679), (0xFFFFFFFF, 1)):
        w1 = TO.tag_bytes(s1, a, 1 << 20).view("<u4")
        w2 = TO.tag_bytes(s2, a, 1 << 20).view("<u4")
        assert np.all((w1 ^ w2) == np.uint32(s1 ^ s2))


def test_alias_count_model_is_consistent():
    exact, low, high = TO.alias_counts(0xABCDEF01, 0x7F00_0000_0000, 1 << 20)
    assert low <= exact <= high
    assert exact > (1 << 20)           # almost every byte differs from both its own tag and from zero


def test_kernel_header_tag_matches_the_oracle(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not Path(nvcc).exists():
        pytest.skip("nvcc not available")
    src = tmp_path / "probe.cu"
    src.write_text('#include <cstdio>\n#include <cstdlib>\n#include "scrub_kernels.cuh"\n'
                   "int main(int c, char** v) { for (int i = 2; i < c; ++i) {\n"
                   "  unsigned long long a = strtoull(v[i], 0, 0);\n"
                   "  printf(\"%u %u\\n\", ccm::tag_word((uint32_t)strtoul(v[1], 0, 0), a),\n"
                   "         (unsigned)ccm::tag_byte((uint32_t)strtoul(v[1], 0, 0), a)); } }\n")
    exe = tmp_path / "probe"
    subprocess.run([nvcc, "-std=c++17", "-I", str(ROOT / "k8s_cc_manager_b200" / "csrc"), str(src), "-o", str(exe)],
                   check=True, capture_output=True)
    addrs = [0, 1, 3, 17, G16 - 1, G16 + 2, 0x7FFF_FFFF_FFFF]
    out = subprocess.run([str(exe), str(0x5EED1234), *map(str, addrs)], capture_output=True, text=True,
                         check=True).stdout.split("\n")
    for a, line in zip(addrs, out):
        word, byte = map(int, line.split())
        assert word == TO.tag_word_py(0x5EED1234, a & ~3)
        assert byte == int(TO.tag_bytes(0x5EED1234, a, 1)[0])


# ---------------------------------------------------------------------------- C ABI
def test_abi_surface_and_mismatch_status(native):
    lib = native.lib()
    assert native.ERR_MISMATCH == -13
    assert "tag" in native.strerror(native.ERR_MISMATCH)
    for name in ("ccm_scrub_verify_tagged", "ccm_scrub_verify_many_tagged", "ccm_region_tag_fill",
                 "ccm_region_tag_check_zero"):
        assert name in native.EXPORTED_SYMBOLS
    assert C.sizeof(native.TagResult) == 40 and native.TagResult.va_base.offset == 32
    assert lib.ccm_abi_version() == 2


def test_tagged_call_without_cuda_fails_loudly_and_reports_its_seed(native):
    lib = native.lib()
    assert lib.ccm_sim_topology(2, 0) == 0
    sim_set(-1, "cuda_ordinal", -1)
    tag, res = native.TagResult(), native.ScrubResult()
    assert lib.ccm_scrub_verify_tagged(0, 1 << 20, C.byref(tag), C.byref(res)) == native.ERR_NO_CUDA
    assert res.status == native.ERR_NO_CUDA and tag.seed != 0 and tag.mismatch_bytes == 0
    tag = native.TagResult(seed=1234)
    assert lib.ccm_scrub_verify_tagged(0, 1 << 20, C.byref(tag), C.byref(res)) == native.ERR_NO_CUDA
    assert tag.seed == 1234
    assert lib.ccm_scrub_verify_tagged(0, 1 << 20, None, C.byref(res)) == native.ERR_INVALID
    idx = (C.c_int * 2)(0, 1)
    tags, out = (native.TagResult * 2)(), (native.ScrubResult * 2)()
    assert lib.ccm_scrub_verify_many_tagged(2, idx, 0, tags, out, None) == native.ERR_NO_CUDA
    assert tags[0].seed != 0 and tags[1].seed != 0
    assert lib.ccm_scrub_verify_many_tagged(2, idx, 0, None, out, None) == native.ERR_INVALID


def test_drill_keys_round_trip_on_sim(native):
    lib = native.lib()
    assert lib.ccm_sim_topology(2, 0) == 0
    for key, value in (("tag_inject", 1 << 40), ("scrub_alias", 1)):
        assert sim_get(0, key) == 0
        sim_set(0, key, value)
        assert sim_get(0, key) == value and sim_get(1, key) == 0
        sim_set(-1, key, 0)
        assert sim_get(0, key) == sim_get(1, key) == 0
    sim_set(0, "tag_inject", -3)
    assert sim_get(0, "tag_inject") == 0
    sim_set(0, "scrub_alias", 9)
    assert sim_get(0, "scrub_alias") == 1
    sim_set(0, "scrub_alias", 0)


def test_drill_keys_are_no_ops_on_sysfs(tmp_path, monkeypatch):
    d = tmp_path / "devices" / "0000:1b:00.0"
    d.mkdir(parents=True)
    for name, value in (("vendor", "0x10de"), ("class", "0x030200"), ("device", "0x2330"), ("reset", "")):
        (d / name).write_text(value + "\n" if value else "")
    monkeypatch.setenv("CCM_SYSFS_ROOT", str(tmp_path / "devices"))
    try:
        D.select_backend("sysfs")
        for key in ("tag_inject", "scrub_alias"):
            assert N.lib().ccm_sim_set(0, key.encode(), 7) == 0
            assert sim_get(0, key) == 0
    finally:
        D.select_backend("sim")


# ------------------------------------------------------------------- Python devices
def test_reports_default_to_zero_mode_and_serialise_as_before():
    rep = ScrubReport("0000:1b:00.0", 0, 1, 2, 0, 1.0, 1.0, 1.0, 0.0, 3.0, 1, 0)
    assert rep.check == "zero" and rep.mismatch_bytes == 0 and rep.tag_seed == 0
    assert set(rep.as_json()) == set(ScrubReport.__dataclass_fields__) - set(D.TAG_FIELDS)
    rep.check, rep.mismatch_bytes = "tagged", 5
    assert set(D.TAG_FIELDS) <= set(rep.as_json()) and not rep.clean


def test_unknown_check_is_rejected():
    with pytest.raises(ValueError):
        D.scrub_and_verify_many([], 0, check="march")


# ------------------------------------------------------------------------- manager
class FakeGpu:
    """Duck-typed device; `tagged` decides whether its scrub takes the check argument."""

    def __init__(self, bdf, tagged=True, cc="off", report_check=None):
        self.bdf, self.name = bdf, "fake"
        self.is_cc_query_supported = self.is_ppcie_query_supported = True
        self.cc, self.staged, self.pp = cc, cc, "off"
        self.calls = []
        self._report_check = report_check
        self.scrub_and_verify = self._scrub_checked if tagged else self._scrub_zero

    def is_gpu(self): return True
    def is_nvswitch(self): return False
    def query_cc_mode(self): return self.cc
    def set_cc_mode(self, m): self.staged = m
    def query_ppcie_mode(self): return self.pp
    def set_ppcie_mode(self, m): pass
    def reset_with_os(self): self.cc = self.staged
    def wait_for_boot(self): pass

    def _report(self, nbytes, check):
        rep = ScrubReport(self.bdf, nbytes, 190 << 30, 191 << 30, 0, 1, 25, 25, 1, 52, 1, 0)
        rep.check = self._report_check or check
        return rep

    def _scrub_zero(self, nbytes=0):
        self.calls.append(("zero-only", nbytes))
        return self._report(nbytes, "zero")

    def _scrub_checked(self, nbytes=0, check="zero"):
        self.calls.append((check, nbytes))
        return self._report(nbytes, check)


def make_manager(devs, monkeypatch, labels=None, **kw):
    import kubernetes
    from k8s_cc_manager_b200 import manager
    c = kubernetes.reset_cluster()
    c.add_node(SC.NODE, labels or {})
    monkeypatch.setenv("EVICT_OPERATOR_COMPONENTS", "false")
    return manager.CCManager(SC.NODE, "on", True, device_source=lambda: (devs, len(devs)), **kw), c


def state(c):
    return c.labels(SC.NODE).get("nvidia.com/cc.mode.state")


def test_scrub_check_parsing(monkeypatch):
    devs = [FakeGpu(SC.GPU_BDFS[0])]
    assert make_manager(devs, monkeypatch)[0].scrub_check == "zero"
    monkeypatch.setenv("CC_SCRUB_CHECK", "TAGGED")
    assert make_manager(devs, monkeypatch)[0].scrub_check == "tagged"
    assert make_manager(devs, monkeypatch, scrub_check="zero")[0].scrub_check == "zero"
    monkeypatch.setenv("CC_SCRUB_CHECK", "march")
    with pytest.raises(ValueError, match="CC_SCRUB_CHECK"):
        make_manager(devs, monkeypatch)
    from k8s_cc_manager_b200 import manager
    assert manager.build_arg_parser().parse_args(["--scrub-check", "tagged"]).scrub_check == "tagged"
    assert manager.build_arg_parser().parse_args([]).scrub_check is None
    with pytest.raises(SystemExit):
        manager.build_arg_parser().parse_args(["--scrub-check", "march"])


def test_per_gpu_fan_out_passes_the_check(monkeypatch):
    devs = [FakeGpu(b) for b in SC.GPU_BDFS[:3]]
    mgr, c = make_manager(devs, monkeypatch, scrub_check="tagged")
    assert mgr.set_cc_mode("on") is True and state(c) == "on"
    assert all(d.calls == [("tagged", 0)] for d in devs)
    assert all(r.check == "tagged" for r in mgr.last_transition["scrub"])


def test_zero_mode_calls_devices_exactly_as_before(monkeypatch):
    devs = [FakeGpu(b, tagged=False) for b in SC.GPU_BDFS[:2]]
    mgr, c = make_manager(devs, monkeypatch)
    assert mgr.set_cc_mode("on") is True and state(c) == "on"
    assert all(d.calls == [("zero-only", 0)] for d in devs)


@pytest.mark.parametrize("case", ["no_check_argument", "zero_report"])
def test_a_device_that_cannot_run_the_tagged_check_fails_closed(case, monkeypatch):
    devs = [FakeGpu(SC.GPU_BDFS[0]),
            FakeGpu(SC.GPU_BDFS[1], tagged=case != "no_check_argument",
                    report_check="zero" if case == "zero_report" else None)]
    mgr, c = make_manager(devs, monkeypatch, scrub_check="tagged")
    assert mgr.set_cc_mode("on") is False and state(c) == "failed"
    assert ("zero-only", 0) not in devs[1].calls


def test_regate_of_an_already_set_node_passes_the_check(monkeypatch):
    devs = [FakeGpu(b, cc="on") for b in SC.GPU_BDFS[:2]]
    mgr, c = make_manager(devs, monkeypatch, labels={"nvidia.com/cc.mode.state": "failed"}, scrub_check="tagged")
    assert mgr.set_cc_mode("on") is True and state(c) == "on"
    assert mgr.last_transition.get("regate") is True
    assert all(d.calls == [("tagged", 0)] for d in devs)


def test_mismatch_report_fails_the_gate_and_names_the_count(monkeypatch):
    dev = FakeGpu(SC.GPU_BDFS[0])
    real = dev._scrub_checked

    def mismatching(nbytes=0, check="zero"):
        rep = real(nbytes, check)
        rep.status, rep.mismatch_bytes = N.ERR_MISMATCH, 123
        return rep
    dev.scrub_and_verify = mismatching
    mgr, c = make_manager([dev], monkeypatch, scrub_check="tagged")
    from k8s_cc_manager_b200 import manager
    with pytest.raises(manager.ScrubFailure, match="mismatch_bytes=123"):
        mgr._run_scrub([dev])


def _native_world(monkeypatch, n=2):
    build_native_world(SC.scenario("w", gpus_=SC.gpus(n), modes=[]))
    for k, v in dict(CCM_BACKEND="sim", CCM_SIM_GPUS=str(n), CCM_SIM_BIND_CUDA="0").items():
        monkeypatch.setenv(k, v)


@pytest.mark.parametrize("check", ["zero", "tagged"])
def test_native_fan_out_passes_the_check(check, monkeypatch):
    import kubernetes
    from k8s_cc_manager_b200 import manager
    _native_world(monkeypatch)
    seen = []

    def fake_many(devices, nbytes=0, **kw):
        seen.append(kw)
        return [ScrubReport(d.bdf, nbytes, 190 << 30, 191 << 30, 0, 1, 25, 25, 1, 52, 1, 0,
                            check=kw.get("check", "zero")) for d in devices], 1.0
    monkeypatch.setattr(manager._devices, "scrub_and_verify_many", fake_many)
    c = kubernetes.reset_cluster()
    c.add_node(SC.NODE, {})
    monkeypatch.setenv("EVICT_OPERATOR_COMPONENTS", "false")
    mgr = manager.CCManager(SC.NODE, "on", True, scrub_check=check)
    assert mgr.set_cc_mode("on") is True
    assert seen == ([{}] if check == "zero" else [{"check": "tagged"}])


@pytest.mark.parametrize("flavour", ["native", "python"])
@pytest.mark.parametrize("check", ["zero", "tagged"])
def test_process_isolation_passes_the_check(flavour, check, monkeypatch):
    import kubernetes
    from k8s_cc_manager_b200 import manager
    _native_world(monkeypatch)
    for k, v in dict(CC_SCRUB_ISOLATION="process", CC_SCRUB_WORKER=flavour, EVICT_OPERATOR_COMPONENTS="false").items():
        monkeypatch.setenv(k, v)
    cmds = []
    real_run = subprocess.run

    def run(cmd, **kw):
        cmds.append(cmd)
        return real_run(cmd, **kw)
    monkeypatch.setattr(subprocess, "run", run)
    c = kubernetes.reset_cluster()
    c.add_node(SC.NODE, {})
    mgr = manager.CCManager(SC.NODE, "on", True, scrub_check=check)
    assert mgr.set_cc_mode("on") is False                 # no CUDA behind the sim GPUs: fails closed
    assert len(cmds) == 1
    assert ("--check" in cmds[0]) == (check == "tagged")
    if check == "tagged":
        assert cmds[0][cmds[0].index("--check") + 1] == "tagged"
    reps = mgr.last_transition["scrub"]
    assert [r.status for r in reps] == [N.ERR_NO_CUDA] * 2 and all(r.check == check for r in reps)


# --------------------------------------------------------------------- CLI / worker
def _worker(args):
    env = dict(CCM_BACKEND="sim", CCM_SIM_BIND_CUDA="0", PYTHONPATH=str(ROOT), PATH="/usr/bin:/bin")
    return subprocess.run([sys.executable, "-m", "k8s_cc_manager_b200.scrub_worker", *args], capture_output=True,
                          text=True, env=env, timeout=300)


def _cli(args):
    env = dict(CCM_BACKEND="sim", CCM_SIM_BIND_CUDA="0", PATH="/usr/bin:/bin")
    return subprocess.run([str(ROOT / "k8s_cc_manager_b200" / "ccm-scrub"), *args], capture_output=True, text=True,
                          env=env, timeout=60)


def test_cli_and_worker_take_the_check_and_print_the_same_keys():
    base = ["--bdf", SC.GPU_BDFS[1], "--bytes", "4096"]
    outs = {}
    for name, fn in (("cli", _cli), ("worker", _worker)):
        for check in ("zero", "tagged"):
            p = fn(base + (["--check", check] if check == "tagged" else []))
            assert p.returncode == 3, p.stderr[-1000:]
            outs[name, check] = json.loads(p.stdout.splitlines()[-1])["reports"][0]
        assert fn(base + ["--check", "march"]).returncode == 2
    assert set(outs["cli", "zero"]) == set(outs["worker", "zero"])
    assert set(outs["cli", "tagged"]) == set(outs["worker", "tagged"])
    assert set(outs["cli", "tagged"]) - set(outs["cli", "zero"]) == set(D.TAG_FIELDS)
    assert not set(D.TAG_FIELDS) & set(outs["cli", "zero"])
    for name in ("cli", "worker"):
        r = outs[name, "tagged"]
        assert r["check"] == "tagged" and r["tag_seed"] != 0 and r["status"] == N.ERR_NO_CUDA
