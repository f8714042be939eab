"""Numpy page maps of the three window books (include/ccm.h: ccm_last_page_map).

A book counts its booked bytes per 2 MiB page: the non-zero bytes (locate, census) or the bytes that differ from their
tags (the tagged check).  Every booked byte counts on the page of its 16-byte, 16-aligned address WINDOW, and a window
belongs to the page of its offset from the pass's base: (window address - base) >> 21, page 0 when that is negative
(the head window of a region that does not start 16-aligned).

    page_map(region, ptr, base=None)        content `region` at device address ptr, offsets from base (default ptr)
    check_page_map(region, ptr, seed, base) the same for region XOR the tags of `seed` at ptr
    brute_page_map(...)                     the same, one window at a time (the definition, for small inputs)
"""
from __future__ import annotations

import numpy as np

import tag_oracle as TO

PAGE_SHIFT = 21
PAGE_BYTES = 1 << PAGE_SHIFT


def _pages(booked: np.ndarray, ptr: int, base: int) -> dict:
    idx = np.flatnonzero(booked).astype(np.int64)
    if idx.size == 0:
        return {}
    win = ((ptr + idx) & ~np.int64(15)) - base          # window offsets from base (a head window may be negative)
    page = np.where(win < 0, 0, win >> PAGE_SHIFT)
    pages, counts = np.unique(page, return_counts=True)
    return {int(p): int(c) for p, c in zip(pages, counts)}


def page_map(region: np.ndarray, ptr: int, base: int | None = None) -> dict:
    """{page: non-zero bytes} of `region` (uint8) at address ptr, pages counted from base (default ptr)."""
    return _pages(np.asarray(region) != 0, ptr, ptr if base is None else base)


def check_page_map(region: np.ndarray, ptr: int, seed: int, base: int | None = None) -> dict:
    """{page: bytes that differ from their tags} of `region` at address ptr."""
    region = np.asarray(region, dtype=np.uint8)
    return _pages(region != TO.tag_bytes(seed, ptr, region.size), ptr, ptr if base is None else base)


def brute_page_map(region, ptr: int, base: int | None = None, seed: int | None = None) -> dict:
    """The definition, window by window: every 16-aligned address window that overlaps the region adds its booked
    bytes (non-zero, or with `seed` off their tags) to the page of its offset from base."""
    base = ptr if base is None else base
    region = np.asarray(region, dtype=np.uint8)
    n = region.size
    want = TO.tag_bytes(seed, ptr, n) if seed is not None else np.zeros(n, dtype=np.uint8)
    out: dict = {}
    w = ptr & ~15
    while w < ptr + n:
        booked = sum(1 for a in range(max(w, ptr), min(w + 16, ptr + n)) if region[a - ptr] != want[a - ptr])
        if booked:
            off = w - base
            page = 0 if off < 0 else off // PAGE_BYTES
            out[page] = out.get(page, 0) + booked
        w += 16
    return out


def entries(pages: dict, chunk_of=lambda offset: 0) -> list:
    """(page, bytes, chunk) rows of a page map, ascending, each with the chunk of its first byte."""
    return [(p, b, chunk_of(p * PAGE_BYTES)) for p, b in sorted(pages.items())]
