"""The relayed whole-HBM gate (ccm-scrub --relay, DESIGN.md §5n) on one H100: both legs clean, the relay's fields
recomputed from the raw ones, the first context's footprint given back and reached by the second leg (a 0xA5 marker the
first leg holds until it exits comes back and is mapped by the second leg), every gate option relayed with the plain call's
report shape, and no process left behind.

Every gate runs in a ccm-scrub child, so no context of this process takes part in the relay."""
from __future__ import annotations

import ctypes as C
import json
import os
import subprocess
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
from k8s_cc_manager_b200 import _native as N  # noqa: E402

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

CLI = ROOT / "k8s_cc_manager_b200" / "ccm-scrub"
MiB = 1 << 20
SLACK = 2 * MiB
# What the driver keeps of the first context on a device while another context lives on it: the first context's
# footprint exceeds a later one's by 3 473 408 B on an H100 80GB HBM3, and the first leg's exit gives back only the
# later one's (profiles/h100_relay.json, DESIGN.md §5n).
KEPT = 4 * MiB


@pytest.fixture(scope="module", autouse=True)
def need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


@pytest.fixture(scope="module")
def bdf():
    """The PCI address of CUDA device 0, as libccm names it."""
    lib = N.lib()
    assert lib.ccm_init(N.BACKEND_CUDASIM) == 0
    n = C.c_int()
    lib.ccm_enumerate(None, 0, C.byref(n))
    infos = (N.DevInfo * max(n.value, 1))()
    lib.ccm_enumerate(infos, n.value, C.byref(n))
    return next(i.bdf.decode() for i in infos[:n.value] if i.cuda_ordinal == 0)


def others_used() -> int:
    """The bytes CUDA device 0 holds for every context on it right now (nvidia-smi's device-wide memory.used, which it
    also reports inside a container that cannot list the processes or the bus id), this test process's own included: a
    test that ran earlier in the same process may have left its context and allocations.  The device is found by UUID."""
    uuid = str(torch.cuda.get_device_properties(0).uuid).lower()
    out = subprocess.run(["nvidia-smi", "--query-gpu=uuid,memory.used", "--format=csv,noheader,nounits"],
                         capture_output=True, text=True, timeout=60, check=True).stdout
    rows = [[x.strip() for x in line.rpartition(",")[::2]] for line in out.splitlines() if line.strip()]
    match = [int(mib) for u, mib in rows if u.lower().endswith(uuid)] or [int(mib) for _, mib in rows if len(rows) == 1]
    assert match, (uuid, out)
    return match[0] * MiB


def alive(pid: int) -> bool:
    try:
        state = Path(f"/proc/{pid}/stat").read_text().rsplit(")", 1)[1].split()[0]
    except (FileNotFoundError, ProcessLookupError):
        return False
    return state != "Z"


def run(bdf: str, *args: str) -> tuple[int, dict]:
    env = dict(os.environ, CCM_BACKEND="cudasim")
    proc = subprocess.run([str(CLI), *args, "--bdf", bdf], capture_output=True, text=True, timeout=600, env=env)
    lines = [x for x in proc.stdout.splitlines() if x.startswith("{")]
    assert lines, proc.stderr[-2000:]
    return proc.returncode, json.loads(lines[-1])


def check_relay(rep: dict, first: dict) -> dict:
    """The relay's fields, recomputed in plain Python from the two reports and the raw reads, must be the printed ones."""
    r = rep["relay"]
    assert r["total"] == rep["device_total_bytes"]
    assert r["a_free_before"] == first["device_free_before"] and r["a_unreached"] == first["bytes_unreached"]
    assert r["b_free_before"] == rep["device_free_before"] and r["b_unreached"] == rep["bytes_unreached"]
    footprint = max(0, r["total"] - r["a_free_before"])
    freed = max(0, r["b_free_settled"] - r["b_free_held"])
    held = max(0, footprint - freed)
    growth = max(0, r["b_free_settled"] - r["b_free_before"])
    unreached = held + growth + r["a_unreached"] + r["b_unreached"]
    assert (r["footprint_a"], r["freed"], r["held"], r["growth"], r["unreached"]) == (footprint, freed, held, growth,
                                                                                       unreached)
    assert r["coverage"] == pytest.approx(1 - unreached / r["total"], abs=1e-8)
    assert r["settled"] == 1 and r["settle_polls"] >= 1
    return r


def test_a_whole_hbm_relay_reaches_the_first_context_footprint(bdf):
    others = others_used()
    rc, out = run(bdf, "--relay")
    assert rc == 0, out
    rep, first = out["reports"][0], out["first"]["reports"][0]
    assert rep["status"] == 0 and rep["nonzero_bytes"] == 0 and first["status"] == 0 and first["nonzero_bytes"] == 0
    r = check_relay(rep, first)
    assert r["freed"] > 0 and r["growth"] <= SLACK and r["marked"] == 0
    assert r["held"] <= others + KEPT, (r, others)
    assert r["coverage"] > rep["bytes_scrubbed"] / rep["device_total_bytes"]
    assert not alive(out["first_pid"])


def test_the_second_leg_erases_and_counts_what_the_first_context_held(bdf):
    others = others_used()
    rc, out = run(bdf, "--relay", "--residue", "--relay-mark-mib", "256")
    assert rc == 0, out
    rep, first = out["reports"][0], out["first"]["reports"][0]
    assert rep["status"] == 0 and rep["nonzero_bytes"] == 0
    r = check_relay(rep, first)
    assert r["marked"] == 256 * MiB
    # the marker came back with the first leg's exit (all of the first leg's footprint but what other contexts hold and
    # what the driver keeps), and leg B mapped, erased and read back what came back
    assert r["freed"] >= r["footprint_a"] + r["marked"] - others - KEPT, (r, others)
    assert rep["bytes_scrubbed"] >= r["b_free_settled"] - r["b_unreached"] - r["growth"] - SLACK
    # the census counts what leg B found there: on the H100 the driver hands a departed process's memory back zeroed,
    # so it finds none of the marker (DESIGN.md §5n); it must never find more than the marker and what was there before
    assert "residue" in rep and rep["residue"]["residue_bytes"] <= first["bytes_scrubbed"] + r["marked"]
    assert not alive(out["first_pid"])


@pytest.mark.parametrize("option", [["--check", "tagged"], ["--prove"], ["--probe"], ["--health", "report"]],
                         ids=["tagged", "prove", "probe", "health"])
def test_every_gate_option_is_relayed_with_the_plain_report(bdf, option):
    rc, plain = run(bdf, *option)
    assert rc == 0, plain
    rc, out = run(bdf, "--relay", *option)
    assert rc == 0, out
    rep, first = out["reports"][0], out["first"]["reports"][0]
    check_relay(rep, first)
    assert set(rep) == set(plain["reports"][0]) | {"relay"}
    assert set(out["first"]) == set(plain) and set(first) == set(plain["reports"][0])
    assert not alive(out["first_pid"])
