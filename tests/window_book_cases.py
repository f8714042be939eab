"""Placements, window layouts and content builders of the window-book tests (tests/test_window_books_gpu.py).

The locate pass, the tag check and both censuses keep one book (WindowBook in
k8s_cc_manager_b200/csrc/scrub_kernels.cuh): a window count, the first and last booked byte, and up to 64 records
claimed one slot at a time.  Each kernel reaches the book from four places, and each place computes masks and
offsets its own way:
  batch     a thread's PER_THREAD vectors of one grabbed chunk, vector u at p + u * STRIDE;
  leftover  a vector after the last whole chunk (finish_region);
  head      one of the up to 8 windows of the ragged head (ragged_window; the first may stick out of the region);
  tail      the one window of the ragged tail (less than 16 bytes of it lie in the region).

Plain Python + numpy, so that tests/test_window_book_cases.py can check on the CPU that the placements reach every
place and that each layout puts its windows where it says.  All four book kernels run at the same shape
(kLocateThreads / kTagThreads / kCensusThreads = 512 threads, 16 vectors per thread: one 128 KiB chunk per grab, one
CTA per SM), which is the geometry of the default verifier in tests/scrub_cases.py.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

import scrub_cases as CASES

THREADS, PER_THREAD = 512, 16
STRIDE = THREADS * 16                   # bytes between vectors u and u + 1 of one thread in a chunk
CHUNK = THREADS * PER_THREAD * 16       # bytes per grab
RECORDS = 64                            # include/ccm.h: CCM_DIRT_RECORDS
assert CHUNK == CASES.FAST_CHUNK

# Region start mod 128.  With CASES.OFFSETS these give every head-window count: 0 (offset 0), 1..7 windows that
# start 16-aligned (offsets 112, 96, ..., 16) and 1..8 windows whose first sticks out of the region (127, 113, 97,
# ..., 17, and 1, 3, 8, 15).
EXTRA_OFFSETS = (3, 8, 15, 32, 33, 48, 49, 64, 65, 80, 81, 96, 97, 112, 113)
OFFSETS = tuple(sorted(set(CASES.OFFSETS) | set(EXTRA_OFFSETS)))
LIMIT_COUNTS = (1, 63, 64, 65, 128)     # booked windows around the record limit
PATHS = ("batch", "leftover", "head", "tail")


def geometry(sm: int) -> CASES.Geometry:
    return CASES.geometry(CASES.FAST_VERIFY, sm)


def lengths(g: CASES.Geometry, offset: int) -> list[int]:
    """CASES.lengths plus an empty region, one that ends where its first window ends and one a byte longer
    (straddling two windows)."""
    inside = 16 - offset % 16
    return sorted(set(CASES.lengths(g)) | {0, inside, inside + 1})


def placements(g: CASES.Geometry) -> list[tuple[int, int]]:
    return [(o, n) for o in OFFSETS for n in lengths(g, o)]


# ------------------------------------------------------------------ split_region and the chunk rules, restated
def head_windows(offset: int, n: int) -> tuple[int, bool]:
    """(number of head windows, does the first start 16-aligned) of a region starting `offset` past a 128-byte
    boundary (ragged_window)."""
    head, _, _ = CASES.split(offset, n, 16)
    if head == 0:
        return 0, True
    first = offset // 16 * 16
    return (offset + head - first + 15) // 16, offset % 16 == 0


def where(offset: int, n: int, rel: int) -> tuple:
    """Where the book kernels take the window that holds region byte `rel`: ("head", k), ("tail",),
    ("leftover", vector) or ("batch", chunk, thread, u)."""
    head, body, _ = CASES.split(offset, n, 16)
    if rel < head:
        return ("head", (offset + rel) // 16 - offset // 16)
    if rel >= head + body:
        return ("tail",)
    v = (rel - head) // 16
    nchunks = body // CHUNK
    if v < nchunks * CHUNK // 16:
        c, within = divmod(v, CHUNK // 16)
        u, t = divmod(within, THREADS)
        return ("batch", c, t, u)
    return ("leftover", v)


def paths(offset: int, n: int) -> set[str]:
    """The places a region whose every byte is booked reaches (where() at the first and last byte of each part)."""
    head, body, _ = CASES.split(offset, n, 16)
    whole = head + body // CHUNK * CHUNK
    return {where(offset, n, rel)[0] for rel in {0, head, whole - 1, whole, head + body - 1, n - 1} if 0 <= rel < n}


def window_bytes(offset: int, n: int, w: int) -> list[int]:
    """Region offsets of the bytes of the window that starts at region offset w (address-aligned) that lie in the
    region."""
    return [w + i for i in range(16) if 0 <= w + i < n]


def window_of(offset: int, rel: int) -> int:
    """Region offset of the (address-aligned) window holding region byte rel."""
    return (offset + rel) // 16 * 16 - offset


# ------------------------------------------------------------------ layouts
@dataclass(frozen=True)
class Layout:
    name: str
    path: str                 # where every window is taken ("mixed": spread over all four places)
    offset: int               # region start mod 128
    n: int                    # region bytes
    windows: tuple            # region offsets of the windows, ascending


def _batch(c: int, t: int, u: int, head: int = 0) -> int:
    return head + c * CHUNK + u * STRIDE + t * 16


def batch_layout(w: int, u: int) -> Layout:
    """w <= 4 * THREADS windows at vector u of threads spread over four chunks (four CTAs)."""
    wins = sorted(_batch(i % 4, (i * 7) % THREADS, u) for i in range(w))
    return Layout(f"batch_u{u}", "batch", 0, 4 * CHUNK + 5 * 16, tuple(wins))


def leftover_layout(w: int) -> Layout:
    """w windows on every other vector after the last whole chunk."""
    return Layout("leftover", "leftover", 0, CHUNK + 2 * w * 16 + 16, tuple(CHUNK + 32 * i for i in range(w)))


def mixed_layout(w: int) -> Layout:
    """A region that starts 16 bytes past a 128-byte boundary (7 whole head windows) and ends 15 bytes into a tail
    window: the head windows, the tail window, then leftover and chunk vectors in turn, up to w."""
    n = 112 + 2 * CHUNK + 256 * 16 + 15
    order = [16 * k for k in range(7)] + [n - 15]
    for i in range(256):
        order += [112 + 2 * CHUNK + 16 * i, _batch(i % 2, (i * 11) % THREADS, (i * 5) % PER_THREAD, 112)]
    return Layout("mixed", "mixed", 16, n, tuple(sorted(order[:w])))


def per_chunk_layout(w: int) -> Layout:
    """One window in each of the first w chunks of a 130-chunk region, at a different thread and u in each: one CTA
    per window, all claiming at once."""
    nchunks = max(130, w)
    wins = [_batch(c, (c * 37) % THREADS, c % PER_THREAD) for c in range(w)]
    return Layout("per_chunk", "batch", 0, nchunks * CHUNK, tuple(wins))


def one_chunk_layout(w: int) -> Layout:
    """All w windows in the one chunk of a one-chunk region: one CTA books them all."""
    wins = sorted(_batch(0, i % THREADS, (i * 5) % PER_THREAD) for i in range(w))
    return Layout("one_chunk", "batch", 0, CHUNK, tuple(wins))


def limit_layouts(w: int) -> list[Layout]:
    return [batch_layout(w, 0), batch_layout(w, PER_THREAD - 1), leftover_layout(w), mixed_layout(w),
            per_chunk_layout(w), one_chunk_layout(w)]


# ------------------------------------------------------------------ masks
def all_masks() -> list[int]:
    return list(range(1, 1 << 16))


def edge_masks(seed: int = 7, sample: int = 200) -> list[int]:
    """Every mask of popcount <= 2 or >= 14, then a seeded sample of the others."""
    edge = [m for m in range(1, 1 << 16) if bin(m).count("1") <= 2 or bin(m).count("1") >= 14]
    rng = np.random.default_rng(seed)
    rest = [m for m in dict.fromkeys(rng.integers(1, 1 << 16, size=4 * sample).tolist()) if 2 < bin(m).count("1") < 14]
    return edge + rest[:sample]


# ------------------------------------------------------------------ content
def dirt_content(offset: int, n: int, windows, masks, rng) -> np.ndarray:
    """Zero region of n bytes with the bytes `masks[i]` of window `windows[i]` set to random non-zero values (bits
    of bytes outside the region are ignored)."""
    buf = np.zeros(n, dtype=np.uint8)
    for w, m in zip(windows, masks):
        idx = [w + i for i in range(16) if m >> i & 1 and 0 <= w + i < n]
        buf[idx] = rng.integers(1, 256, len(idx))
    return buf


def flip_content(tags: np.ndarray, windows, masks, rng) -> np.ndarray:
    """The tags with the bytes `masks[i]` of window `windows[i]` XORed with random non-zero values: exactly those
    bytes differ from their tags."""
    buf = tags.copy()
    n = buf.size
    for w, m in zip(windows, masks):
        idx = [w + i for i in range(16) if m >> i & 1 and 0 <= w + i < n]
        buf[idx] ^= rng.integers(1, 256, len(idx)).astype(np.uint8)
    return buf


def in_region_mask(n: int, w: int) -> int:
    return sum(1 << i for i in range(16) if 0 <= w + i < n)
