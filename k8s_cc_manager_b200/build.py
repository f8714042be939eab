"""Builds libccm.so (sm_90a, H100) in-tree with nvcc.

The shared library lands next to this file (k8s_cc_manager_b200/libccm.so) so it
travels with the repo snapshot to the GPU box; it is git-ignored.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from pathlib import Path

PKG_DIR = Path(__file__).resolve().parent
REPO_ROOT = PKG_DIR.parent
CSRC = PKG_DIR / "csrc"
LIB_PATH = PKG_DIR / "libccm.so"
CLI_PATH = PKG_DIR / "ccm-scrub"
CLI_SOURCE = CSRC / "ccm_scrub_cli.cpp"

SOURCES = [CSRC / "ccm_scrub.cu", CSRC / "ccm_core.cpp"]
HEADERS = [CSRC / "scrub_kernels.cuh", CSRC / "ccm_internal.h", CSRC / "ccm_mismatch.h", CSRC / "ccm_proof.h", CSRC / "ccm_health.h",
           CSRC / "ccm_relay.h", REPO_ROOT / "include" / "ccm.h"]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC,-fvisibility=hidden,-Wall",
    "--shared",
    "-cudart", "static",
]


def find_nvcc() -> str:
    nvcc = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not Path(nvcc).exists():
        raise RuntimeError("nvcc not found: libccm.so cannot be built (set NVCC=/path/to/nvcc)")
    return nvcc


def needs_build() -> bool:
    if not LIB_PATH.exists() or not CLI_PATH.exists():
        return True
    built = min(LIB_PATH.stat().st_mtime, CLI_PATH.stat().st_mtime)
    return any(p.stat().st_mtime > built for p in SOURCES + HEADERS + [CLI_SOURCE, Path(__file__)])


def compile_lib(src_dir: Path, include_dir: Path, out: Path, verbose: bool = False) -> Path:
    """libccm.so from the sources under src_dir (laid out as csrc/) and include_dir, with the product's flags."""
    cmd = [find_nvcc(), *NVCC_FLAGS, "-I", str(include_dir), "-I", str(src_dir)]
    if verbose:
        cmd += ["-Xptxas", "-v"]
    cmd += [str(src_dir / s.name) for s in SOURCES]
    cmd += ["-o", str(out), "-ldl", "-lpthread"]
    proc = subprocess.run(cmd, capture_output=True, text=True)
    if proc.returncode != 0:
        sys.stderr.write(proc.stdout + proc.stderr)
        raise RuntimeError(f"nvcc failed ({proc.returncode}) building {out}")
    if verbose:
        sys.stderr.write(proc.stderr)
    return out


def build(force: bool = False, verbose: bool = False) -> Path:
    if not force and not needs_build():
        return LIB_PATH
    compile_lib(CSRC, REPO_ROOT / "include", LIB_PATH, verbose)
    # native CLI front end (ccm-scrub): plain host C++, finds libccm.so next to itself
    gxx = shutil.which("g++") or "g++"
    cli = subprocess.run([gxx, "-O2", "-std=c++17", "-Wall", "-I", str(REPO_ROOT / "include"), str(CLI_SOURCE),
                          "-o", str(CLI_PATH), "-L", str(PKG_DIR), "-lccm", "-Wl,-rpath,$ORIGIN"],
                         capture_output=True, text=True)
    if cli.returncode != 0:
        sys.stderr.write(cli.stdout + cli.stderr)
        raise RuntimeError(f"g++ failed ({cli.returncode}) building {CLI_PATH}")
    return LIB_PATH


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
