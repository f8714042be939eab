"""Mutation tests of the device code: copies of libccm.so with one small, deliberate bug each (tests/kernel_mutants.py),
and the exactness driver (tests/sanitize_calls.py) run against each copy in a child process (CCM_LIB).  A suite that
passes on a kernel that misses a 0x80 byte, stops a loop one byte early or books 63 records where 64 are due would
pass on the same bug in the product: these tests show that the checks fail when a kernel is subtly wrong.

On the CPU: every anchor occurs once in the sources (a refactor that moves the code names the stale mutant), every
mutant compiles for sm_90a with the product's flags, the pristine rebuild has the product library's SASS in every
function, every mutant changes the SASS of at least one function (one the compiler folded away is a no-op, not an
equivalent), and every kernel entry of the registry has its SASS changed by at least one KILL mutant.

On the GPU, one case per mutant: a KILL mutant must make the driver report mismatches, at least one of them in a call
its `killer` names; an EQUIVALENT one must leave every result exact; no run may end in a CUDA error (`fault`): a mutant
that does had a wrong safety argument and is to be corrected or removed, not run again.  With CCM_MUTANT_RECORD=<path>
the run adds each mutant's verdict, killing calls and wall time there, with the card's name and power limit read in
the same run (profiles/h100_kernel_mutants.json).
"""
from __future__ import annotations

import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "tests"))
sys.path.insert(0, str(ROOT / "oracle"))
import kernel_mutants as KM  # noqa: E402
from test_window_book_cases import device_kernels  # noqa: E402

DRIVER = ROOT / "tests" / "sanitize_calls.py"
TIMEOUT = 300                  # seconds per driver run


def entry_key(name: str):
    from test_sanitizers_gpu import entry_key as key
    return key(name)


@pytest.fixture(scope="module")
def built() -> dict:
    libs, cpu, wall = KM.build_all()
    print(f"\n{len(KM.MUTANTS)} mutants and the pristine rebuild: {cpu:.0f} s of nvcc (0 for a cached library), "
          f"{wall:.0f} s wall")
    return libs


@pytest.fixture(scope="module")
def sass(built) -> dict:
    """{mutant id, None for the pristine rebuild, "product" for libccm.so: sass()}."""
    from k8s_cc_manager_b200 import _native as N
    libs = dict(built, product=N.LIB_PATH)
    with ThreadPoolExecutor(max_workers=os.cpu_count() or 1) as pool:
        return dict(zip(libs, pool.map(KM.sass, libs.values())))


# ------------------------------------------------------------------------------------ CPU
def test_every_anchor_occurs_once():
    stale = {m.id: KM.anchor_count(m) for m in KM.MUTANTS if KM.anchor_count(m) != 1}
    assert not stale, f"mutants whose anchor does not occur exactly once (id: occurrences): {stale}"


def test_the_table_is_well_formed():
    for m in KM.MUTANTS:
        assert m.kind in (KM.KILL, KM.EQUIVALENT) and m.phase in ("region", "all"), m.id
        assert m.breaks and m.safe and m.anchor != m.replacement, m.id
        assert m.file in (KM.KERNELS, KM.SCRUB), m.id
        assert bool(m.killer) == (m.kind == KM.KILL), m.id
    assert sum(m.kind == KM.EQUIVALENT for m in KM.MUTANTS) == 2


def test_pristine_rebuild_is_the_product(sass):
    diff = sorted(KM.changed(sass[None], sass["product"]))
    assert not diff, f"a rebuild of the unchanged sources differs from libccm.so in: {diff[:10]}"
    print(f"\npristine rebuild: {len(sass[None])} functions, SASS identical to libccm.so")


def test_every_mutant_changes_the_sass(sass):
    folded = [m.id for m in KM.MUTANTS if not KM.changed(sass[m.id], sass[None])]
    assert not folded, f"mutants the compiler folded away (no function changed): {folded}"
    for m in KM.MUTANTS:
        print(f"\n{m.id}: {len(KM.changed(sass[m.id], sass[None]))} functions changed", end="")


def test_kill_mutants_reach_every_kernel_entry(sass):
    import shutil
    cxxfilt = shutil.which("c++filt")
    assert cxxfilt, "c++filt (binutils) is needed to demangle the kernel names"
    touched = set()
    for m in KM.MUTANTS:
        if m.kind == KM.KILL:
            touched |= KM.changed(sass[m.id], sass[None])
    names = sorted(touched)
    demangled = subprocess.run([cxxfilt], input="\n".join(names), check=True, capture_output=True,
                               text=True).stdout.split("\n")[:len(names)]
    reached = {entry_key(d) for d in demangled} - {None}
    registry = {entry_key(e) for e in device_kernels()}
    assert len(registry) >= 98, len(registry)
    missing = sorted(registry - reached)
    assert not missing, "kernel entries no KILL mutant changes:\n  " + "\n  ".join(missing)
    print(f"\n{len(registry)} of {len(registry)} registry entries changed by a KILL mutant")


# ------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def record():
    """Adds one mutant's verdict to $CCM_MUTANT_RECORD (when set), with the card it ran on: after every case, so a run
    cut short keeps what it measured, and a run of a few cases updates theirs."""
    path = os.environ.get("CCM_MUTANT_RECORD")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    name, power = (q.stdout.splitlines()[0].split(", ") + [""])[:2] if q.returncode == 0 and q.stdout else ("", "")

    def add(mid: str, row: dict) -> None:
        if not path:
            return
        p = Path(path)
        out = json.loads(p.read_text()) if p.exists() else {"driver": str(DRIVER.relative_to(ROOT)),
                                                            "timeout_s": TIMEOUT, "mutants": {}}
        out["mutants"][mid] = dict(row, gpu=name, power_limit=power)
        p.parent.mkdir(parents=True, exist_ok=True)
        p.write_text(json.dumps(out, indent=1) + "\n")
    return add


@pytest.mark.gpu
@pytest.mark.parametrize("mid", [m.id for m in KM.MUTANTS])
def test_mutant(mid, built, record):
    pytest.importorskip("torch")
    m = KM.BY_ID[mid]
    env = dict(os.environ, CCM_LIB=str(built[mid]))
    t0 = time.perf_counter()
    try:
        proc = subprocess.run([sys.executable, str(DRIVER), "--phase", m.phase], capture_output=True, text=True,
                              env=env, cwd=ROOT, timeout=TIMEOUT)
    except subprocess.TimeoutExpired:
        record(mid, {"kind": m.kind, "verdict": "timeout", "wall_s": TIMEOUT})
        pytest.fail(f"{mid}: the driver ran past {TIMEOUT} s")
    wall = time.perf_counter() - t0
    lines = [x for x in proc.stdout.splitlines() if x.startswith("RESULT ")]
    res = json.loads(lines[-1][len("RESULT "):]) if lines else None
    if res is None:
        record(mid, {"kind": m.kind, "verdict": "no result", "wall_s": round(wall, 1)})
        pytest.fail(f"{mid}: no RESULT (exit {proc.returncode})\n{proc.stdout[-3000:]}{proc.stderr[-3000:]}")
    killing = [f for f in res["failed"] if KM.killed_by(f, m.killer)]
    verdict = "fault" if res["fault"] else ("killed" if res["mismatches"] else "survived")
    record(mid, {"kind": m.kind, "verdict": verdict, "phase": m.phase, "wall_s": round(wall, 1),
                 "mismatches": res["mismatches"], "calls": res["calls"], "killing": killing[:8]})
    print(f"\n{mid} ({m.kind}, {m.phase} phase, {wall:.0f} s): {verdict}, {res['mismatches']} of {res['calls']} "
          f"results wrong; killed by {killing[:3]}")
    assert not res["fault"], f"{mid} ended in a CUDA error: its safety argument ({m.safe}) is wrong: {res}"
    if m.kind == KM.EQUIVALENT:
        assert res["mismatches"] == 0 and proc.returncode == 0, f"{mid} is not equivalent: {res['first_mismatch']}"
    else:
        assert res["mismatches"], f"{mid} survived: no check fails when {m.breaks}"
        assert killing, f"{mid} was not killed by {m.killer}, only by {res['failed'][:10]}"
