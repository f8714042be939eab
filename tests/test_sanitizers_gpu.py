"""Every device kernel of libccm.so under compute-sanitizer: memcheck, racecheck, synccheck and initcheck, at its tiling
edges, with every result checked exactly while it runs (tests/sanitize_calls.py, a child process per run).

A kernel can return the right count and still read past its region into memory that happens to hold zeros, race on
shared memory, or call a warp intrinsic with a mask that names lanes which are not there; such a kernel passes every
exactness test and fails later, on another driver, SM count or neighbouring allocation.  These runs see that:

  memcheck   --padding 256 --leak-check full, the whole run, once with programmatic dependent launch (CCM_PDL=1) and
             once without: every region ends flush against its own allocation (and, in a second call, starts at it)
  racecheck  the whole run: the shared-memory block reductions and the double-buffered grab slots, with every grabber
             taking two grabs
  synccheck  the whole run: the warp reductions on __activemask() inside data-dependent branches
  initcheck  the region phase only: the product calls read, by design, what the previous tenant left

Each run must exit 0, report `ERROR SUMMARY: 0 errors` and an exact RESULT.  A plain run under torch.profiler must
launch every kernel entry of the registry (tests/test_window_book_cases.py: device_kernels), and on the CPU the
driver's case table must name every entry, so a new kernel has to join these runs.

compute-sanitizer is tried first on one tiny torch kernel: where it cannot instrument the device at all (it reports
"Device not supported", as compute-sanitizer 12.9 did on an H100 80GB HBM3 at a 700 W power limit), the tool runs skip
and say so, and any other failure of that probe fails them.

Open: no tool run has been measured yet, on any device.  The plain profiled run, which checks every result exactly,
took 30 s on that H100.  The wall time of each tool's run is printed with its result and belongs here, beside the GPU
and power limit it was measured at, once a device the tool instruments has run them.  That the driver's exact checks
fail when a kernel is subtly wrong is shown without a sanitizer: tests/test_kernel_mutants.py runs the driver against
copies of libccm.so with one value or loop-narrowing bug each, and requires it to fail on every one.  The two mutation
checks each tool run exists for stay open (racecheck must fail with the barrier between the writes and reads of `part`
in WindowBook::flush dropped; memcheck must fail with ragged_bytes walking one byte past the tail): both mutants race or
access out of bounds on purpose, which a shared GPU must not be asked to run, and the tools do not instrument the H100
that runs this suite (see above).  TIMEOUT is a bound, not a measurement:
a run that reaches it fails, names itself and asks for smaller regions.  The regions stay at the sizes their tiling
edges need (at most 34 MiB: every grabber of the default-frame kernels takes two grabs) and the product calls at a few
2 MiB chunks, to keep the instrumented runs to minutes.
"""
from __future__ import annotations

import json
import os
import re
import subprocess
import sys
import time
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "tests"))
sys.path.insert(0, str(ROOT / "oracle"))
ALLOCATOR_KNOB = "PYTORCH_NO_CUDA_MEMORY_CACHING"
ALLOCATOR_BEFORE = os.environ.get(ALLOCATOR_KNOB)   # as the session had it, before this module imports the driver
import gate_model as GM  # noqa: E402
import gate_scenarios as GS  # noqa: E402
import sanitize_calls as SCL  # noqa: E402
from test_window_book_cases import device_kernels  # noqa: E402

SANITIZER = Path("/usr/local/cuda/bin/compute-sanitizer")
DRIVER = ROOT / "tests" / "sanitize_calls.py"
TIMEOUT = 1500                 # seconds per child: a bound on a run not yet measured under any tool (see above)

# kernel entry -> why the profiled run need not launch it (none: every entry launches)
EXEMPT: dict = {}

# run -> (tool arguments, phase, environment)
RUNS = {
    "memcheck-pdl": (["--tool", "memcheck", "--padding", "256", "--leak-check", "full"], "all", {"CCM_PDL": "1"}),
    "memcheck-nopdl": (["--tool", "memcheck", "--padding", "256", "--leak-check", "full"], "all", {"CCM_PDL": "0"}),
    "racecheck": (["--tool", "racecheck"], "all", {}),
    "synccheck": (["--tool", "synccheck"], "all", {}),
    "initcheck": (["--tool", "initcheck"], "region", {}),
}
PROBE = "import torch; torch.ones(1, device='cuda').add_(1); torch.cuda.synchronize()"

_ENTRY_RE = re.compile(r"ccm::(\w+)(?:<([^>]*)>)?")


def entry_key(name: str) -> str | None:
    """`name<args>` of a demangled kernel name (cuobjdump + c++filt, or the profiler's): casts and integer suffixes off
    the template arguments.  None for a name outside namespace ccm (a torch kernel, a copy)."""
    m = _ENTRY_RE.search(name)
    if not m:
        return None
    if m.group(2) is None:
        return m.group(1)
    args = [re.sub(r"[uUlL]+$", "", re.sub(r"^\(\w[\w ]*\)", "", a.strip())) for a in m.group(2).split(",")]
    return f"{m.group(1)}<{', '.join(args)}>"


def registry() -> set:
    keys = {entry_key(e) for e in device_kernels()}
    assert None not in keys and len(keys) >= 98, sorted(map(str, keys))
    return keys


# ------------------------------------------------------------------------------------ CPU: the case table
def test_case_table_names_every_registry_entry():
    reg = registry()
    missing = sorted(reg - set(SCL.ENTRIES))
    assert not missing, ("kernel entries tests/sanitize_calls.py does not launch (add them to its ENTRIES and its run):"
                         "\n  " + "\n  ".join(missing))
    unknown = sorted(set(SCL.ENTRIES) - reg)
    assert not unknown, f"ENTRIES names kernels libccm.so does not define: {unknown}"
    assert not set(EXEMPT) - reg, sorted(set(EXEMPT) - reg)
    print(f"\ncase table: {len(reg)} of {len(reg)} registry entries")


def test_importing_the_driver_changes_no_environment():
    """Only the driver's own process turns torch's caching allocator off: pytest imports the driver to read its case
    table, and the GPU tests of the same session, and the children they start, must keep the allocator they had."""
    code = ("import os, sys; before = dict(os.environ); sys.path[:0] = [sys.argv[1], sys.argv[2]]; "
            "import sanitize_calls; assert dict(os.environ) == before, set(os.environ.items()) ^ set(before.items())")
    env = {k: v for k, v in os.environ.items() if k != ALLOCATOR_KNOB}
    proc = subprocess.run([sys.executable, "-c", code, str(ROOT / "tests"), str(ROOT / "oracle")], capture_output=True,
                          text=True, cwd=ROOT, env=env, timeout=120)
    assert proc.returncode == 0, proc.stderr[-2000:]
    assert os.environ.get(ALLOCATOR_KNOB) == ALLOCATOR_BEFORE, "importing the driver changed this session's allocator"


def test_product_calls_are_predicted_by_the_model():
    """Every product call of the driver is one the composed model predicts, and together they reach every verdict the
    driver means to reach."""
    fails = set()
    for c in SCL.PRODUCT_CALLS:
        want = GM.predict(c, GS.fake_record(c))
        fails |= set(want["fails"]) or {"clean"}
        assert 0 < c["bytes"] <= 16 << 20, c
    assert {"clean", "dirty", "tag_mismatch"} <= fails, fails
    kinds = {c["kind"] for c in SCL.PRODUCT_CALLS}
    assert kinds == set(GM.KINDS), kinds
    assert any(c.get("probe") and c.get("prove") for c in SCL.PRODUCT_CALLS)
    assert any(c.get("triage") and c.get("mismatch_triage") and c.get("prove") for c in SCL.PRODUCT_CALLS)
    assert {c["env"].get("CCM_PIPELINE", "1") for c in SCL.PRODUCT_CALLS} == {"0", "1"}
    assert any(c["env"].get("CCM_MAP_FIRST") == "1" for c in SCL.PRODUCT_CALLS)


def test_regions_stay_small_and_reach_two_grabs():
    import scrub_cases as SC
    import window_book_cases as WB
    g = WB.geometry(SC.H100_SMS)
    names = [p[0] for p in SCL.placements(g)]
    assert "two grabs each" in names
    _, _, n = SCL.placements(g)[names.index("two grabs each")]
    assert n >= 2 * g.chunk * g.grabbers
    sizes = [n for _, _, n in SCL.placements(g)]
    for case in SCL.generic_cases().values():
        gg = SC.geometry(case, SC.H100_SMS)
        ls = SCL.generic_lengths(gg, 111)
        assert ls[:2] == [0, 1] and ls[3] - ls[2] == 1 and ls[-1] > gg.chunk * gg.grabbers
        sizes += ls
    assert max(sizes) <= 48 << 20, max(sizes)


# ------------------------------------------------------------------------------------ GPU
def run_driver(args: list, phase: str, env: dict, kernels: bool = False) -> tuple:
    cmd = args + [sys.executable, str(DRIVER), "--phase", phase] + (["--kernels"] if kernels else [])
    t0 = time.perf_counter()
    try:
        proc = subprocess.run(cmd, capture_output=True, text=True, env=dict(os.environ, **env), cwd=ROOT,
                              timeout=TIMEOUT)
    except subprocess.TimeoutExpired as exc:
        tail = (exc.stdout or b"")[-2000:]
        pytest.fail(f"{' '.join(cmd[:4])} ... --phase {phase} ran past {TIMEOUT} s: cut the driver's region sizes, not "
                    f"its kernels\n{tail.decode(errors='replace') if isinstance(tail, bytes) else tail}")
    return proc, time.perf_counter() - t0


def result_of(proc) -> dict | None:
    lines = [x for x in proc.stdout.splitlines() if x.startswith("RESULT ")]
    return json.loads(lines[-1][len("RESULT "):]) if lines else None


def first_reports(proc, k: int = 80) -> str:
    lines = [x for x in (proc.stdout + proc.stderr).splitlines() if x.startswith("=========")]
    return "\n".join(lines[:k]) or (proc.stdout[-3000:] + proc.stderr[-3000:])


@pytest.mark.gpu
def test_driver_launches_every_kernel():
    pytest.importorskip("torch")
    proc, wall = run_driver([], "all", {}, kernels=True)
    assert proc.returncode == 0, proc.stdout[-3000:] + proc.stderr[-3000:]
    res = result_of(proc)
    assert res and res["first_mismatch"] is None, res
    line = [x for x in proc.stdout.splitlines() if x.startswith("KERNELS ")][-1]
    launched = {k for k in map(entry_key, json.loads(line[len("KERNELS "):])) if k}
    reg = registry()
    missing = sorted(reg - launched - set(EXEMPT))
    assert not missing, "kernel entries the driver never launched:\n  " + "\n  ".join(missing)
    assert launched <= reg, sorted(launched - reg)
    print(f"\n{len(reg & launched)} of {len(reg)} entries launched ({len(EXEMPT)} exempt), {res['calls']} exact "
          f"results, {wall:.0f} s")


@pytest.fixture(scope="module")
def sanitizer() -> str:
    """compute-sanitizer, once it has instrumented one tiny torch kernel without error."""
    if not SANITIZER.exists():
        pytest.skip(f"{SANITIZER} is not installed: the kernels ran under no sanitizer")
    pytest.importorskip("torch")
    proc = subprocess.run([str(SANITIZER), "--error-exitcode", "1", sys.executable, "-c", PROBE], capture_output=True,
                          text=True, cwd=ROOT, timeout=600)
    out = proc.stdout + proc.stderr
    if "Device not supported" in out:
        line = next(x for x in out.splitlines() if "Device not supported" in x)
        pytest.skip(f"compute-sanitizer cannot instrument this GPU ({line.strip('= ')}): the kernels ran under no "
                    "sanitizer")
    assert proc.returncode == 0 and "ERROR SUMMARY: 0 errors" in out, f"compute-sanitizer probe failed:\n{out[-3000:]}"
    return str(SANITIZER)


@pytest.mark.gpu
@pytest.mark.parametrize("run", list(RUNS))
def test_sanitizer(sanitizer, run):
    args, phase, env = RUNS[run]
    cmd = [sanitizer, "--error-exitcode", "1", "--target-processes", "application-only"] + args
    proc, wall = run_driver(cmd, phase, env)
    out = proc.stdout + proc.stderr
    res = result_of(proc)
    what = f"{run} on the {phase} phase ({wall:.0f} s)"
    assert proc.returncode == 0 and "ERROR SUMMARY: 0 errors" in out, \
        f"{what}: exit {proc.returncode}\n{first_reports(proc)}"
    assert res is not None and res["first_mismatch"] is None, f"{what}: {res}"
    print(f"\n{what}: ERROR SUMMARY: 0 errors, {res['calls']} exact results")
