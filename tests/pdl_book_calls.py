"""The window-book kernels, the tagged and census gates and the dirt triage with and without programmatic dependent
launch: a child process for tests/test_pdl_books_gpu.py, which runs it once with CCM_PDL=1 and once with CCM_PDL=0
(the library latches CCM_PDL once per process).

With CCM_PDL=1 every default-frame kernel (default_kernel in k8s_cc_manager_b200/csrc/scrub_kernels.cuh) is launched
with the programmatic-stream-serialization attribute and triggers its dependents as soon as its grab loop ends, before
it resets its GrabCtl pair, takes the leftover vectors and ragged windows and flushes its book.  Only the dependent's
griddepcontrol.wait keeps the two apart.  Two legs exercise that:

  region chains   library calls and torch kernels on one torch stream over a guarded region (tests/
                  test_window_books_gpu.py's Rig), each launch directly behind the one before it: CHAINS names the
                  steps.  Every chain runs at every placement of PLACEMENTS.
  product calls   the page-map drills of tests/test_page_map_gpu.py in every mapping mode and on the fallback, the
                  aliased tagged call, and armed triage calls (tests/test_dirt_triage_gpu.py), whose re-reads launch
                  the locate kernel once per run back to back.

Run as a script it makes every call on CUDA device 0 and prints one `RESULT <json>` line.  The case lists and the
content builders are plain Python, so tests/test_pdl_cases.py checks them on the CPU.  Not collected by pytest.
"""
from __future__ import annotations

import dataclasses
import json
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
for p in (ROOT, ROOT / "tests", ROOT / "oracle"):
    if str(p) not in sys.path:
        sys.path.insert(0, str(p))

import product_plan as PP  # noqa: E402
import tag_oracle as TO  # noqa: E402
import window_book_cases as WB  # noqa: E402

MiB, GiB = 1 << 20, 1 << 30
PAGE = 2 * MiB
SEED = 0x7A61B00C                        # tests/test_window_books_gpu.py: SEED
TORCH = "torch scatter_"                 # a torch kernel on the same stream

# ------------------------------------------------------------------------------------ A. region chains
# step -> the kernel it launches ("dirt": torch scatters bytes into the region).  "check" is
# ccm_region_tag_check_locate, which zeroes its mismatch counter with a memset in front of the check kernel.
KERNELS = {"scrub": "scrub_st128_fast_kernel", "fill": "tag_fill_kernel", "census0": "census_zero_kernel",
           "census1": "census_tag_fill_kernel", "check": "tag_check_zero_kernel", "locate": "locate_dirt_kernel",
           "dirt": TORCH}
# chain -> steps on the stream, in order; the last one books (census0 / census1: residue, check: mismatch,
# locate: dirt).  The region holds INITIAL content before the first step.
CHAINS = {
    "scrub>census0": ("scrub", "census0"),
    "scrub>fill>census1": ("scrub", "fill", "census1"),
    "scrub>fill>check": ("scrub", "fill", "check"),
    "dirt>fill>check": ("dirt", "fill", "check"),
    "scrub>dirt>locate": ("scrub", "dirt", "locate"),
}
BOOKS = {"census0": "residue", "census1": "residue", "check": "mismatch", "locate": "dirt"}
OFFSETS = (0, 1, 17, 112, 127)           # region start mod 128
LENGTHS = (3 * WB.CHUNK + 40 * 16 + 9,   # whole chunks, 40 leftover vectors, ragged head and tail windows
           2 * PAGE + 3 * WB.CHUNK + 77)  # page boundaries inside a grab (whenever the start is not 128-aligned)
PLACEMENTS = [(o, n) for o in OFFSETS for n in LENGTHS]


def pairs(chain: str) -> list[tuple[str, str]]:
    """(predecessor kernel, dependent kernel) of every step of a chain."""
    steps = CHAINS[chain]
    return [(KERNELS[a], KERNELS[b]) for a, b in zip(steps, steps[1:])]


def region_cases() -> list[tuple[str, int, int]]:
    return [(chain, off, n) for chain in CHAINS for off, n in PLACEMENTS]


def case_seed(i: int) -> int:
    return 0xB00C + 7919 * i


def initial(n: int, seed: int) -> np.ndarray:
    """Dense random bytes: any step that reads the region before its predecessor wrote it books them."""
    return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8)


def planted(off: int, n: int, seed: int) -> tuple[np.ndarray, np.ndarray]:
    """(positions, non-zero values) torch scatters into the region: its first and last bytes, both sides of every page
    boundary, one byte in every head and tail window, and 300 more."""
    rng = np.random.default_rng(seed ^ 0x5EED)
    head, body, _ = WB.CASES.split(off, n, 16)
    pos = {0, n - 1} | set(rng.integers(0, n, size=300).tolist())
    for k in range(1, n // PAGE + 1):
        pos |= {k * PAGE + d for d in (-17, -1, 0, 1, 16) if 0 <= k * PAGE + d < n}
    pos |= {r for r in range(head)} | {r for r in range(head + body, n)}
    pos = np.array(sorted(pos), dtype=np.int64)
    return pos, rng.integers(1, 256, pos.size, dtype=np.uint8)


def booked_input(chain: str, off: int, n: int, ptr: int, seed: int) -> np.ndarray:
    """What the chain's last step reads, when every step sees everything its predecessors wrote (and what the region
    then holds, except after a check or a zero census, which leave zeros)."""
    last = CHAINS[chain][-1]
    if last == "census0":
        return np.zeros(n, dtype=np.uint8)
    if last in ("census1", "check"):
        return TO.tag_bytes(SEED, ptr, n)
    region = np.zeros(n, dtype=np.uint8)
    pos, vals = planted(off, n, seed)
    region[pos] = vals
    return region


def end_state(chain: str, off: int, n: int, ptr: int, seed: int) -> np.ndarray:
    last = CHAINS[chain][-1]
    return np.zeros(n, dtype=np.uint8) if last in ("census0", "check") else booked_input(chain, off, n, ptr, seed)


# ------------------------------------------------------------------------------------ B. product calls
# The drills of tests/test_page_map_gpu.py's DRILL_CALLS, on these paths: path -> (env, bytes; 0 = whole HBM).
PRODUCT_DRILLS = ("scrub_inject", "scrub_flood", "tag_inject", "scrub_residue", "scrub_poison")
PRODUCT_PATHS = {f"vmm-mf{mf}-il{il}": (PP.mode_env(mf, il), 0) for mf, il in PP.MODES}
PRODUCT_PATHS.update({"fallback": ({"CCM_PIPELINE": "0"}, 0),
                      "fallback-3MiB-segments": ({"CCM_PIPELINE": "0", "CCM_ARENA_MAX_SEGMENT_MB": "3"}, 64 * MiB)})
ALIAS_MAP_FIRST = (0, 1)
# The armed triage: path -> (env, bytes) of tests/test_dirt_triage_gpu.py, with "scrub_inject" and these
# (triage_stay, triage_return) drills; then "scrub_flood" armed, which triages every mapped page.
TRIAGE_PATHS = {f"vmm-mf{mf}-il{il}": (PP.mode_env(mf, il), 4 * GiB) for mf, il in PP.MODES}
TRIAGE_PATHS.update({"fallback": ({"CCM_PIPELINE": "0"}, 4 * GiB),
                     "fallback-3MiB-segments": ({"CCM_PIPELINE": "0", "CCM_ARENA_MAX_SEGMENT_MB": "3"}, 64 * MiB)})
TRIAGE_DRILLS = ((0, 0), (2, 3))
FLOOD_PATHS = {"vmm": ({}, 0), "fallback": ({"CCM_PIPELINE": "0"}, 4 * GiB)}
HOLD_MS = 5


def product_cases() -> list[dict]:
    out = [{"leg": "product", "drill": d, "path": p} for p in PRODUCT_PATHS for d in PRODUCT_DRILLS]
    out += [{"leg": "alias", "mf": mf} for mf in ALIAS_MAP_FIRST]
    out += [{"leg": "triage", "path": p, "stay": s, "ret": r} for p in TRIAGE_PATHS for s, r in TRIAGE_DRILLS]
    out += [{"leg": "flood", "path": p} for p in FLOOD_PATHS]
    return out


# ------------------------------------------------------------------------------------ running them
def run_region_cases(lib) -> list[dict]:
    import ctypes as C

    import torch

    import test_window_books_gpu as WBG
    from k8s_cc_manager_b200 import _native as N
    from k8s_cc_manager_b200 import devices as D

    book_of = {"census0": N.BOOK_RESIDUE, "census1": N.BOOK_RESIDUE, "check": N.BOOK_MISMATCH,
               "locate": N.BOOK_DIRT}
    out = []
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        rig = WBG.Rig(max(LENGTHS))
        h = WBG.stream()
        for i, (chain, off, n) in enumerate(region_cases()):
            seed = case_seed(i)
            ptr, _, (a, b) = rig.place(off, initial(n, seed))
            region = rig.buf[a + WBG.GUARD:b - WBG.GUARD]
            want = torch.from_numpy(end_state(chain, off, n, ptr, seed)).cuda()
            pos, vals = planted(off, n, seed)
            pos_t, vals_t = torch.from_numpy(pos).cuda(), torch.from_numpy(vals).cuda()
            stream.synchronize()             # the uploads are done: nothing but the chain is left on the stream
            l0 = lib.ccm_kernel_launches()
            rep = None
            for step in CHAINS[chain]:
                if step == "scrub":
                    assert lib.ccm_region_scrub(0, C.c_void_p(ptr), n, N.SCRUB_AUTO, None, h, None) == 0, N.last_error()
                elif step == "fill":
                    assert lib.ccm_region_tag_fill(0, C.c_void_p(ptr), n, SEED, h, None) == 0, N.last_error()
                elif step == "dirt":
                    region.scatter_(0, pos_t, vals_t)
                elif step == "locate":
                    rep = WBG.locate(lib, ptr, n)
                elif step == "check":
                    rep = WBG.check_locate(lib, ptr, n, SEED)
                else:
                    rep = WBG.census(lib, ptr, n, step == "census1", SEED)
            launches = lib.ccm_kernel_launches() - l0
            last = CHAINS[chain][-1]
            pages = D.last_page_map(0, book_of[last]).entries
            wrong = int((region != want).sum())                      # counted on the same stream
            guards = int((rig.buf[a:a + WBG.GUARD] != WBG.GUARD_BYTE).sum()
                         + (rig.buf[b - WBG.GUARD:b] != WBG.GUARD_BYTE).sum())
            out.append({"leg": "region", "chain": chain, "offset": off, "n": n, "ptr": ptr, "seed": seed,
                        "book": dataclasses.asdict(WBG.book_of("locate" if last == "locate" else
                                                               "check" if last == "check" else "census", rep)),
                        "pages": pages, "wrong": wrong, "guards": guards, "launches": launches})
    torch.cuda.synchronize()
    return out


def run_product_cases(lib) -> list[dict]:
    import test_dirt_triage_gpu as TDT
    import test_page_map_gpu as TPM
    from k8s_cc_manager_b200 import _native as N
    from k8s_cc_manager_b200 import devices as D

    out = []
    for case in product_cases():
        l0 = lib.ccm_kernel_launches()
        rec = dict(case)
        if case["leg"] in ("product", "alias"):
            if case["leg"] == "product":
                env, nbytes = PRODUCT_PATHS[case["path"]]
                call, drills, _ = TPM.DRILL_CALLS[case["drill"]]
            else:
                env, nbytes, call, drills = {"CCM_MAP_FIRST": str(case["mf"])}, 4 * GiB, "tagged", {"scrub_alias": 1}
            rc, res, tag, rr, dirt, mm, maps = TPM.product(lib, call, env, drills, nbytes)
            rec.update(rc=rc, res=res.as_dict(), residue=rr.as_json(), dirt=dirt.as_json(), mismatch=mm.as_json(),
                       tag=None if tag is None else {f: getattr(tag, f) for f, _ in N.TagResult._fields_},
                       maps=[[b, e] for b, e in sorted(maps.items())])
        else:
            if case["leg"] == "triage":
                env, nbytes = TRIAGE_PATHS[case["path"]]
                drills = {"scrub_inject": PP.INJECT, "triage_stay": case["stay"], "triage_return": case["ret"]}
            else:
                env, nbytes = FLOOD_PATHS[case["path"]]
                drills = {"scrub_flood": PP.FLOOD}
            got = TDT.call(lib, "zero", env, drills, nbytes, hold=HOLD_MS)
            rec.update(rc=got["rc"], res=got["res"].as_dict(), dirt=D.DirtReport.from_native(got["dirt"]).as_json(),
                       triage={f: getattr(got["triage"], f) for f, _ in N.TriageReport._fields_ if f != "reserved"},
                       triage_pages=[dataclasses.asdict(p) for p in got["triage_pages"]],
                       dirt_pages=got["dirt_pages"])
        rec.update(env=env, bytes=nbytes, launches=lib.ccm_kernel_launches() - l0)
        out.append(rec)
    return out


def main() -> None:
    import product_gate_calls as PGC
    import torch
    lib = PGC.open_lib()
    out = run_region_cases(lib)
    torch.cuda.empty_cache()                 # the product calls map all free HBM
    out += run_product_cases(lib)
    PGC.release_wait(lib)
    print("RESULT " + json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
