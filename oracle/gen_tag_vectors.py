#!/usr/bin/env python3
"""Writes tests/golden/tag_vectors.json: the address tags of the tagged scrub gate, pinned.

ORACLE / TEST INFRASTRUCTURE.  A few seeds x addresses (16-aligned, odd, just below and across a
16 GiB boundary, high in the 48-bit space) x lengths, each with its tag bytes in hex.  The bytes come
from the pure-Python statement (tag_word_py), not from numpy or the kernels, so a change of the
pattern in any of them fails tests/test_tagged_gate.py.
"""
from __future__ import annotations

import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "oracle"))
import tag_oracle as TO  # noqa: E402

SEEDS = [1, 0x5EED1234, 0xFFFFFFFF]
G16 = 16 << 30
ADDRS = [0x7F0000000000, 0x7F0000000001, 0x7F0000000003, G16 * 5 - 5, G16 * 7 - 16, 0x7FFFFFFFFFF0 - 32]
LENGTHS = [1, 7, 16, 37]


def tag_hex(seed: int, addr: int, n: int) -> str:
    return bytes((TO.tag_word_py(seed, x & ~3) >> (8 * (x & 3))) & 0xFF for x in range(addr, addr + n)).hex()


def main() -> None:
    vectors = [{"seed": s, "addr": a, "n": n, "bytes": tag_hex(s, a, n)} for s in SEEDS for a in ADDRS for n in LENGTHS]
    out = ROOT / "tests" / "golden" / "tag_vectors.json"
    out.write_text(json.dumps({"k1": TO.K1, "k2": TO.K2, "vectors": vectors}, indent=1) + "\n")
    print(f"wrote {len(vectors)} vectors to {out}")


if __name__ == "__main__":
    main()
