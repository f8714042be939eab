"""Case generators and pattern builders of the scrub / verify exactness matrix.

Plain Python + numpy so that the CPU suite can import and check them
(tests/test_scrub_matrix_coverage.py) and the GPU suite can drive the device with them
(tests/test_scrub_exactness_gpu.py).

The launch rules restated here are those of k8s_cc_manager_b200/csrc/ccm_scrub.cu:
scrub_shape / verify_shape (per-variant defaults, cache_policy - 1 = template policy),
clamp_threads, the unroll normalisation in scrub_range / verify_range, make_sched (tile,
chunk and per-warp rules) and the TMA tile clamp.  A launch with cfg == None takes the
compile-time-shape default kernels (one 128 KiB chunk per grab, one CTA per SM).
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

# include/ccm.h variant numbers (also in k8s_cc_manager_b200/_native.py)
SCRUB_ST128, SCRUB_ST256, SCRUB_TMA, SCRUB_MEMSET = 1, 2, 3, 4
VERIFY_LD128, VERIFY_LD256 = 1, 2

# ccm_launch_cfg.cache_policy (1..4) -> template POL of the kernels (kPolDefault .. kPolEvictLast)
CACHE_POLICIES = (1, 2, 3, 4)
SCHEDULES = (1, 2, 3)                  # static grid-stride, per-CTA chunk grabs, per-warp chunk grabs
SCRUB_UNROLLS = (1, 2, 4, 8, 16)
VERIFY_UNROLLS = (1, 2, 4, 8)
OFFSETS = (0, 1, 16, 17, 127)          # region start mod 128 -> head = 0, 127, 112, 111, 1
FAST_CHUNK = 128 * 1024                # bytes per grab of the compile-time-shape default kernels
MAX_LENGTH = 1 << 30
H100_SMS = 132                         # H100 SXM; the GPU tests read the SM count from the device
H100_SMEM_OPTIN = 232448

TMA_TILE_BYTES = 12345                 # not a multiple of 128: the kernel's tile is 12336 bytes


@dataclass(frozen=True)
class Case:
    kind: str                 # "scrub" | "verify"
    variant: int
    cfg: tuple | None         # (ctas_per_sm, threads, tile_bytes, unroll, cache_policy, schedule) or None

    def cfg_kwargs(self) -> dict | None:
        if self.cfg is None:
            return None
        keys = ("ctas_per_sm", "threads", "tile_bytes", "unroll", "cache_policy", "schedule")
        return dict(zip(keys, self.cfg))

    def label(self) -> str:
        name = {("scrub", SCRUB_ST128): "st128", ("scrub", SCRUB_ST256): "st256", ("scrub", SCRUB_TMA): "tma",
                ("scrub", SCRUB_MEMSET): "memset", ("verify", VERIFY_LD128): "ld128",
                ("verify", VERIFY_LD256): "ld256"}[(self.kind, self.variant)]
        if self.cfg is None:
            return name + ("" if self.variant == SCRUB_MEMSET and self.kind == "scrub" else "-fast")
        c, t, tb, u, p, s = self.cfg
        return f"{name}-u{u}-p{p}-s{s}-t{t}x{c}-tb{tb}"


@dataclass(frozen=True)
class Geometry:
    """How one launch cuts a region: VB-byte vectors, T bytes per tile, C bytes per grab,
    N independent grabbers, `group` threads sharing one tile (lane-contiguous halves for VB 32)."""
    vb: int
    unroll: int
    group: int
    tile: int      # T
    chunk: int     # C
    grabbers: int  # N


# ------------------------------------------------------------------ launch rules
def clamp_threads(t: int) -> int:
    t = max(32, min(1024, t))
    return t // 32 * 32


def _shape(case: Case) -> dict:
    """scrub_shape / verify_shape with the cfg applied (cfg == None: the defaults)."""
    if case.kind == "scrub":
        sh = (dict(ctas_per_sm=1, threads=32, unroll=1, policy=0, tile_bytes=65536, schedule=2)
              if case.variant == SCRUB_TMA else
              dict(ctas_per_sm=1, threads=512, unroll=4, policy=0, tile_bytes=131072, schedule=2))
    else:
        sh = dict(ctas_per_sm=1, threads=1024, unroll=4, policy=2, tile_bytes=131072, schedule=2)
    kw = case.cfg_kwargs()
    if kw:
        for key in ("ctas_per_sm", "threads", "unroll", "tile_bytes"):
            if kw[key] > 0:
                sh[key] = kw[key]
        if 1 <= kw["cache_policy"] <= 4:
            sh["policy"] = kw["cache_policy"] - 1
        if 1 <= kw["schedule"] <= 3:
            sh["schedule"] = kw["schedule"]
    sh["threads"] = clamp_threads(sh["threads"])
    if case.kind == "scrub" and case.variant != SCRUB_TMA and sh["unroll"] not in (1, 2, 8, 16):
        sh["unroll"] = 4
    if case.kind == "verify" and sh["unroll"] not in (1, 2, 8):
        sh["unroll"] = 4
    return sh


def is_fast(case: Case) -> bool:
    return case.cfg is None and case.variant in ((SCRUB_ST128,) if case.kind == "scrub" else (VERIFY_LD128,))


def tma_tile(tile_bytes: int, smem_optin: int = H100_SMEM_OPTIN) -> int:
    tile = tile_bytes & ~15
    tile = max(tile, 1024)
    if tile > smem_optin - 1024:
        tile = (smem_optin - 1024) & ~127
    return tile


def instantiation(case: Case, fast_names: tuple[str, str]) -> str | None:
    """The kernel template instantiation the case launches (None: cudaMemsetAsync, no kernel of ours).
    fast_names = (scrub, verify) names of the compile-time-shape kernels, as ccm_default_kernels() gives them."""
    if is_fast(case):
        return fast_names[0] if case.kind == "scrub" else fast_names[1]
    if case.kind == "scrub" and case.variant == SCRUB_MEMSET:
        return None
    sh = _shape(case)
    pol = sh["policy"]
    if case.kind == "scrub" and case.variant == SCRUB_TMA:
        return f"scrub_tma_kernel<{pol if pol in (1, 3) else 0}>"   # no streaming TMA instantiation
    if case.kind == "scrub":
        vb = 32 if case.variant == SCRUB_ST256 else 16
        return f"scrub_st_kernel<{vb}, {sh['unroll']}, {pol}>"
    vb = 32 if case.variant == VERIFY_LD256 else 16
    return f"verify_ld_kernel<{vb}, {sh['unroll']}, {pol}>"


def geometry(case: Case, sms: int, smem_optin: int = H100_SMEM_OPTIN) -> Geometry:
    """T, C and N of one launch (clamp_threads, make_sched, the TMA tile clamp)."""
    if is_fast(case) or (case.kind == "scrub" and case.variant == SCRUB_MEMSET):
        # memset has no tiling of ours: it borrows the default kernel's placements
        return Geometry(vb=16, unroll=1, group=FAST_CHUNK // 16, tile=FAST_CHUNK, chunk=FAST_CHUNK, grabbers=sms)
    sh = _shape(case)
    grid = sms * sh["ctas_per_sm"]
    if case.kind == "scrub" and case.variant == SCRUB_TMA:
        tile = tma_tile(sh["tile_bytes"], smem_optin)
        warps = min(sh["threads"], 256) // 32
        dynamic = sh["schedule"] in (2, 3)
        chunk = (sh["unroll"] if sh["unroll"] > 0 else 4) * tile if dynamic else tile
        return Geometry(vb=16, unroll=1, group=1, tile=tile, chunk=chunk, grabbers=grid * warps)
    vb = 32 if case.variant == (SCRUB_ST256 if case.kind == "scrub" else VERIFY_LD256) else 16
    u, threads = sh["unroll"], sh["threads"]
    per_warp = sh["schedule"] == 3
    group = 32 if per_warp else threads
    tile = group * u * vb
    if sh["schedule"] == 1:
        return Geometry(vb=vb, unroll=u, group=group, tile=tile, chunk=tile, grabbers=grid)
    chunk = max(1, sh["tile_bytes"] // tile) * tile
    return Geometry(vb=vb, unroll=u, group=group, tile=tile, chunk=chunk,
                    grabbers=grid * (threads // 32) if per_warp else grid)


def big_length(g: Geometry) -> int:
    """Every grabber takes at least two chunks; a remainder (< one tile) and a tail follow."""
    return 2 * g.chunk * g.grabbers + 3 * g.vb + 135


def lengths(g: Geometry) -> list[int]:
    cn = g.chunk * g.grabbers
    out = [1, 127, 128 + g.vb - 1, g.tile - 1, g.tile, g.tile + g.vb + 3, cn - g.vb, cn + g.tile + 29, big_length(g)]
    return sorted(set(x for x in out if x > 0))


def key_length(g: Geometry) -> int:
    """The length at which every instantiation sees all offsets."""
    return g.chunk * g.grabbers + g.tile + 29


# ------------------------------------------------------------------ the matrix
def _generic_cfg(kind: str, variant: int, u: int, pol: int, sched: int) -> tuple:
    """Launch shapes of the matrix: small CTAs so N*C stays small, a different thread count per
    schedule (96 is not a power of two), and two tiles per grab plus 5 bytes of slack."""
    threads = {1: 96, 2: 128, 3: 160}[sched]
    ctas = 2 if sched == 1 else 1
    vb = 32 if variant in ((SCRUB_ST256,) if kind == "scrub" else (VERIFY_LD256,)) else 16
    tile = (32 if sched == 3 else threads) * u * vb
    return (ctas, threads, 2 * tile + 5, u, pol, sched)


def scrub_cases() -> list[tuple[Case, bool]]:
    """(case, full offset x length grid?) — every scrub instantiation under every schedule; the full
    grid for one configuration per (variant, schedule), for TMA, memset and the default kernel."""
    out = []
    for variant in (SCRUB_ST128, SCRUB_ST256):
        for sched in SCHEDULES:
            for u in SCRUB_UNROLLS:
                for pol in CACHE_POLICIES:
                    full = (u, pol) == (4, 2)
                    out.append((Case("scrub", variant, _generic_cfg("scrub", variant, u, pol, sched)), full))
    for pol in (1, 2, 4):
        for sched in (1, 2):
            out.append((Case("scrub", SCRUB_TMA, (1, 64, TMA_TILE_BYTES, 2, pol, sched)), True))
    out.append((Case("scrub", SCRUB_MEMSET, None), True))
    out.append((Case("scrub", SCRUB_ST128, None), True))
    return out


def verify_groups() -> list[list[Case]]:
    """Verifiers that share one geometry (they differ in cache policy only): each pattern is built once
    per placement and every verifier of the group, plus the default fast verifier, counts it."""
    groups = []
    for variant in (VERIFY_LD128, VERIFY_LD256):
        for sched in SCHEDULES:
            for u in VERIFY_UNROLLS:
                groups.append([Case("verify", variant, _generic_cfg("verify", variant, u, pol, sched))
                               for pol in CACHE_POLICIES])
    groups.append([Case("verify", VERIFY_LD128, None)])
    return groups


FAST_VERIFY = Case("verify", VERIFY_LD128, None)


def exhaustive_verifiers() -> list[Case]:
    """The 2^32-word count: fast, and ld128 / ld256 over every unroll and policy, default schedule."""
    out = [FAST_VERIFY]
    for variant in (VERIFY_LD128, VERIFY_LD256):
        for u in VERIFY_UNROLLS:
            for pol in CACHE_POLICIES:
                out.append(Case("verify", variant, (0, 0, 0, u, pol, 0)))
    return out


def all_cases() -> list[Case]:
    cases = [c for c, _ in scrub_cases()]
    cases += [c for g in verify_groups() for c in g]
    cases += exhaustive_verifiers()
    return cases


def placements(g: Geometry, full: bool) -> list[tuple[int, int]]:
    """(offset, length) pairs: the full grid, or every offset at the key length."""
    if full:
        return [(o, n) for n in lengths(g) for o in OFFSETS]
    return [(o, key_length(g)) for o in OFFSETS]


# ------------------------------------------------------------------ patterns
def split(offset: int, n: int, vb: int) -> tuple[int, int, int]:
    """split_region: (head, body bytes, tail) of a region whose start is `offset` mod 128."""
    head = min((128 - offset) % 128, n)
    body = (n - head) // vb * vb
    return head, body, n - head - body


def structural_positions(g: Geometry, offset: int, n: int) -> list[int]:
    """Byte indices (relative to the region) at the edges of the decomposition: head, body, chunks
    0 / 1 / last whole, the first remainder vector, the last lane x last unroll slot of the first tile,
    the second 16-byte half of the first 32-byte step, and the tail."""
    head, body, tail = split(offset, n, g.vb)
    pos = set()
    if head:
        pos.update((0, head - 1))
    if body:
        pos.update((head, head + body - 1))
        whole = body // g.chunk
        for k in {0, 1, whole - 1}:
            if 0 <= k < whole:
                pos.update((head + k * g.chunk, head + (k + 1) * g.chunk - 1))
        rem = body // g.tile * g.tile
        if rem < body:
            pos.add(head + rem)
        if body >= g.tile:
            pos.add(head + g.tile - 16 + 12)          # word 3 of the tile's last 16-byte access
        half = g.group * 16 if g.vb == 32 else 16
        if body > half + 3:
            pos.add(head + half + 3)
    if tail:
        pos.update((head + body, n - 1))
    return sorted(p for p in pos if 0 <= p < n)


def dirt_values(positions: list[int], seed: int) -> list[int]:
    rng = np.random.default_rng(seed)
    return [int(v) for v in rng.integers(1, 256, size=len(positions))]


def bitplane_count(n: int, bit: int) -> int:
    """Number of i in [0, n) whose bit `bit` is 1."""
    period, half = 2 << bit, 1 << bit
    return n // period * half + max(0, n % period - half)


def fill_bitplane(a, bit: int, value: int, complement: bool) -> None:
    """a[i] = value iff bit `bit` of i is 1 (0 otherwise); complement=True swaps the two.  `a` is a
    contiguous 1-D uint8 numpy array or torch tensor (works through reshape views, no index array)."""
    n = len(a)
    period, half = 2 << bit, 1 << bit
    lo, hi = (value, 0) if complement else (0, value)
    whole = n // period * period
    if whole:
        v = a[:whole].reshape(-1, period)
        v[:, :half] = lo
        v[:, half:] = hi
    rest = a[whole:]
    rest[:half] = lo
    rest[half:] = hi


def bitplane_bits(n: int) -> range:
    return range(max(1, (n - 1).bit_length()))
