"""A caller-owned cover map armed around region calls (include/ccm.h: ccm_region_prove): the proving twins then run in
place of the default kernels and count, per 2 MiB page from a base tests/report_cover_oracle.py (map_base) chooses,
every byte they walk.  Used by the GPU tests that run the plain kernels at their tiling edges."""
from __future__ import annotations

import ctypes as C

import numpy as np

import report_cover_oracle as RO
from k8s_cc_manager_b200 import _native as N


class ArmedMap:
    """`steps` maps of `pages` words and an outside slot, end to end, on the current stream, armed on CUDA device 0
    inside the `with` block for region passes over [addr, addr + n).  take() reads them back and zeroes them."""

    def __init__(self, lib, addr: int, n: int, run: int, steps: int = 1, at: tuple[int, int] | None = None):
        """at: (base, pages) in place of RO.map_base's."""
        import torch
        self.lib, self.steps = lib, steps
        self.base, self.pages = at or RO.map_base(addr, n, run)
        self.words = torch.zeros(steps * (self.pages + 1), dtype=torch.int32, device="cuda")

    def __enter__(self) -> "ArmedMap":
        rc = self.lib.ccm_region_prove(0, C.c_void_p(self.words.data_ptr()), self.base, self.pages)
        assert rc == 0, N.last_error()
        return self

    def __exit__(self, *exc) -> None:
        assert self.lib.ccm_region_prove(0, None, 0, 0) == 0, N.last_error()

    def take(self) -> list[list[int]]:
        """Every map (its pages, then its outside slot), read back and zeroed for the next pass."""
        w = self.words.cpu().numpy().view(np.uint32).astype(np.int64)
        self.words.zero_()
        k = self.pages + 1
        return [w[i * k:(i + 1) * k].tolist() for i in range(self.steps)]

    def want(self, parts: list[tuple[int, int]]) -> list[int]:
        """The map of a pass that walked `parts` ((address, bytes)) exactly once."""
        return RO.cover_map(parts, self.base, self.pages)
