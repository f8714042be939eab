"""Drives the product scrub gate (`ccm_scrub_verify` / `ccm_scrub_verify_many` on CUDA device 0) with the
plan knobs and fault drills of tests/product_plan.py, and reports what each call returned.

Imported by tests/test_product_plan_gpu.py.  Run as a script it reads a JSON list of calls from argv[1]
(`[{"bytes": ..., "env": {...}, "drill": "flood", "many": 0}, ...]`), makes them in this fresh process and
prints one `RESULT <json>` line: the first launch of every kernel then happens in the state the call leaves
(for instance with all HBM mapped), and CCM_PDL, which the library latches once per process, takes the value
of this process's environment.  Not collected by pytest.
"""
from __future__ import annotations

import contextlib
import ctypes as C
import json
import os
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
for p in (ROOT, ROOT / "tests"):
    if str(p) not in sys.path:
        sys.path.insert(0, str(p))

import product_plan as PP  # noqa: E402
from k8s_cc_manager_b200 import _native as N  # noqa: E402

FIELDS = ("status", "bytes_scrubbed", "bytes_unreached", "nonzero_bytes", "segments", "device_free_before",
          "device_total_bytes", "release_deferred", "scrub_variant", "verify_variant")


@contextlib.contextmanager
def knobs(env: dict):
    """Sets every plan knob to its value in `env` (absent = unset) and restores the caller's values."""
    names = set(PP.PLAN_KNOBS) | set(env)
    saved = {k: os.environ.get(k) for k in names}
    try:
        for k in names:
            if k in env:
                os.environ[k] = str(env[k])
            else:
                os.environ.pop(k, None)
        yield
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def set_drill(lib, drill: str) -> None:
    vals = PP.DRILLS[drill]
    for k in PP.DRILL_KEYS:
        rc = lib.ccm_sim_set(0, k.encode(), int(vals.get(k, 0)))
        assert rc == 0, N.last_error()


def call(lib, nbytes: int, env: dict, drill: str = "clean", many: int = 0) -> dict:
    """One product call; `many` > 0 runs ccm_scrub_verify_many over `many` copies of device 0."""
    with knobs(env):
        set_drill(lib, drill)
        try:
            if many:
                out = (N.ScrubResult * many)()
                devs = (C.c_int * many)(*([0] * many))
                wall = C.c_double()
                rc = lib.ccm_scrub_verify_many(many, devs, nbytes, out, C.byref(wall))
                results = list(out)
            else:
                res = N.ScrubResult()
                rc = lib.ccm_scrub_verify(0, nbytes, C.byref(res))
                results = [res]
            err = N.last_error() if rc else ""
        finally:
            set_drill(lib, "clean")
    return {"bytes": nbytes, "env": env, "drill": drill, "rc": rc, "error": err,
            "results": [{f: getattr(r, f) for f in FIELDS} for r in results]}


def release_wait(lib) -> None:
    rc = lib.ccm_scrub_release_wait(0, None, None)
    assert rc == 0, N.last_error()


def open_lib():
    lib = N.lib()
    rc = lib.ccm_init(N.BACKEND_CUDASIM)
    assert rc == 0, N.last_error()
    return lib


def main() -> None:
    lib = open_lib()
    out = []
    for c in json.loads(sys.argv[1]):
        out.append(call(lib, c["bytes"], c.get("env", {}), c.get("drill", "clean"), c.get("many", 0)))
        release_wait(lib)
    print("RESULT " + json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
