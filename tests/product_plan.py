"""The product scrub gate's plan, restated in plain Python: which bytes `ccm_scrub_verify` maps, how it cuts
them into chunks, which ranges it enqueues for scrub and read-back, and what each fault drill must then
count.  It plays the role for the product call that tests/scrub_cases.py plays for single launches.

Restated from k8s_cc_manager_b200/csrc/ccm_scrub.cu:
* pipelined VMM path (`scrub_verify_pipelined`): the virtual range is `bytes` rounded up to the allocation
  granularity (bytes == 0: all free HBM rounded down).  With bytes == 0 the last CCM_VMM_TAIL_MB of it are the
  "tail zone".  Main-zone chunks start at CCM_VMM_FIRST_CHUNK_MB and double up to CCM_VMM_CHUNK_MB, every size
  rounded down to the granularity and never below it; tail granules start at 32 MiB.  On out-of-memory a chunk
  halves (main zone: down to 64 MiB, then the tail starts there; tail: down to one granule, then the region
  ends).  Without CCM_MAP_FIRST every main chunk is one enqueued range and the tail granules share one range;
  with it the whole mapping is one range.  CCM_INTERLEAVE_VERIFY moves the read-back, not the ranges.
* arena fallback (CCM_PIPELINE=0 or no VMM): one cudaMalloc of `bytes` (bytes == 0: free minus
  CCM_ARENA_RESERVE_MB, rounded down to 2 MiB), or CCM_ARENA_MAX_SEGMENT_MB segments; each segment is a range.
* drills (sim keys): poison fills every mapped chunk before the scrub (gate must stay clean), flood fills every
  enqueued range between scrub and read-back (count == bytes_scrubbed), inject dirties the first, +17,
  middle + 3 and last byte of each range until its budget runs out.

With bytes == 0 the out-of-memory point is the driver's, so `simulate` takes a capacity (the observed
bytes_scrubbed): it predicts the main zone exactly when the tail zone absorbed the out-of-memory, and the tail
granule count only from below.  The GPU matrix that checks all of this (tests/test_product_plan_gpu.py) is
defined here too, so that tests/test_product_plan.py can check on the CPU which knobs it sweeps.
"""
from __future__ import annotations

from dataclasses import dataclass, field

MiB = 1 << 20
GiB = 1 << 30
H100_GRAN = 2 * MiB          # include/ccm.h: the VMM allocation granularity on H100
TAIL_GRANULE = 32 * MiB      # first tail-zone granule
MAIN_FLOOR = 64 * MiB        # smallest main-zone chunk before the tail takes over
ARENA_ALIGN = 2 * MiB


def env_u64(env: dict, name: str, dflt: int) -> int:
    v = env.get(name)
    return dflt if v is None or v == "" else int(v)


def gran_floor(x: int, gran: int) -> int:
    return x // gran * gran


@dataclass
class Plan:
    bytes: int
    gran: int
    va_bytes: int
    tail_zone: int
    main_end: int                 # nominal start of the tail zone (va_bytes when there is none)
    first: int                    # first main chunk after clamping
    max_chunk: int
    map_first: bool
    interleave: bool

    @property
    def main(self) -> list[tuple[int, int]]:
        """(offset, bytes) of the main-zone chunks when no Create runs out of memory."""
        return simulate(self, None).main


@dataclass
class Run:
    """One walk of the mapping loop: chunks in map order, and where the main zone really ended."""
    chunks: list[tuple[int, int]] = field(default_factory=list)
    main: list[tuple[int, int]] = field(default_factory=list)
    tail: list[tuple[int, int]] = field(default_factory=list)
    main_end: int = 0
    mapped: int = 0

    def ranges(self, plan: Plan) -> list[tuple[int, int]]:
        """The enqueued ranges, in enqueue order."""
        if plan.map_first:
            return [(0, self.mapped)] if self.mapped else []
        out = list(self.main)
        if self.tail:
            out.append((self.main_end, self.mapped - self.main_end))
        return out


def plan(nbytes: int, free: int, gran: int, env: dict, node_fanout: bool = False) -> Plan:
    want_max = nbytes == 0
    va = gran_floor(free, gran) if want_max else -(-nbytes // gran) * gran
    tail = min(gran_floor(env_u64(env, "CCM_VMM_TAIL_MB", 256) * MiB, gran), va) if want_max else 0
    max_chunk = max(gran_floor(env_u64(env, "CCM_VMM_CHUNK_MB", 16384) * MiB, gran), gran)
    first = min(max(gran_floor(env_u64(env, "CCM_VMM_FIRST_CHUNK_MB", 1024) * MiB, gran), gran), max_chunk)
    return Plan(bytes=nbytes, gran=gran, va_bytes=va, tail_zone=tail, main_end=va - tail, first=first,
                max_chunk=max_chunk, map_first=env_u64(env, "CCM_MAP_FIRST", 1 if node_fanout else 0) != 0,
                interleave=env_u64(env, "CCM_INTERLEAVE_VERIFY", 1) != 0)


def simulate(p: Plan, capacity: int | None) -> Run:
    """The mapping loop of scrub_verify_pipelined against a driver that can create `capacity` bytes in all
    (None: unlimited) and never fails a map."""
    gran, va = p.gran, p.va_bytes
    want_max = p.bytes == 0
    chunk, tail_chunk = p.first, max(gran_floor(TAIL_GRANULE, gran), gran)
    main_end = p.main_end
    run = Run()
    off, in_tail, tail_start = 0, False, 0
    while off < va:
        if not in_tail and off >= main_end:
            in_tail, tail_start = True, off
        limit = va if in_tail else main_end
        ck = tail_chunk if in_tail else chunk
        n = min(limit - off, ck)
        if capacity is not None and off + n > capacity:            # cuMemCreate: out of memory
            floor_bytes = gran if in_tail else max(MAIN_FLOOR, gran)
            if ck > floor_bytes:
                ck = max(gran_floor(ck // 2, gran), gran)
                if in_tail:
                    tail_chunk = ck
                else:
                    chunk = ck
                continue
            if want_max and not in_tail:
                main_end = off
                continue
            if want_max and off > 0:
                break
            raise MemoryError(f"no room for {n} bytes at {off}")
        run.chunks.append((off, n))
        (run.tail if in_tail else run.main).append((off, n))
        off += n
        if not in_tail and chunk < p.max_chunk:
            chunk = min(chunk * 2, p.max_chunk)
    run.mapped = off
    run.main_end = tail_start if in_tail else off
    return run


def inject_offsets(ranges: list[tuple[int, int]], budget: int) -> list[int]:
    """Bytes the `scrub_inject` drill dirties: first, +17, middle + 3 and last byte of each range, each
    once, in enqueue order until the budget runs out."""
    out = []
    for off, n in ranges:
        seen: list[int] = []
        for c in (0, 17 if 17 < n else 0, n // 2 + 3 if n // 2 + 3 < n else 0, n - 1):
            if budget == 0:
                return out
            if c in seen:
                continue
            seen.append(c)
            out.append(off + c)
            budget -= 1
    return out


def arena_segments(nbytes: int, free: int, env: dict) -> list[tuple[int, int]]:
    """(offset, bytes) of the fallback's arena segments when every cudaMalloc succeeds."""
    reserve = env_u64(env, "CCM_ARENA_RESERVE_MB", 256) * MiB
    want = nbytes if nbytes else ((free - reserve) & ~(ARENA_ALIGN - 1) if free > reserve else 0)
    seg = env_u64(env, "CCM_ARENA_MAX_SEGMENT_MB", 0) * MiB or want
    return [(o, min(seg, want - o)) for o in range(0, want, seg)] if want else []


# ------------------------------------------------------------------------------------------- drills
POISON, FLOOD, INJECT = 0x5A, 0xC3, 1000
DRILLS = {"clean": {}, "poison": {"scrub_poison": POISON}, "flood": {"scrub_flood": FLOOD},
          "inject": {"scrub_inject": INJECT}}
DRILL_KEYS = ("scrub_inject", "scrub_poison", "scrub_flood")


def expected_count(drill: str, ranges: list[tuple[int, int]], bytes_scrubbed: int) -> int:
    if drill == "flood":
        return bytes_scrubbed
    if drill == "inject":
        return len(inject_offsets(ranges, INJECT))
    return 0


# ------------------------------------------------------------------------------------------- GPU matrix
# Knobs the plan depends on; every call sets all of them (absent = the library's default).
PLAN_KNOBS = ("CCM_VMM_FIRST_CHUNK_MB", "CCM_VMM_CHUNK_MB", "CCM_VMM_TAIL_MB", "CCM_MAP_FIRST",
              "CCM_INTERLEAVE_VERIFY", "CCM_ASYNC_RELEASE", "CCM_PIPELINE", "CCM_ARENA_MAX_SEGMENT_MB",
              "CCM_ARENA_RESERVE_MB", "CCM_SCRUB_VARIANT", "CCM_VERIFY_VARIANT")
# Knobs ccm_scrub.cu reads that the matrix deliberately leaves alone.
EXEMPT_KNOBS = {
    "CCM_CUDA_MAX_CONNECTIONS": "context set-up (hardware work queues), read once when CUDA initialises; "
                                "it does not change which bytes are mapped, scrubbed or counted",
}

CHUNK_SETTINGS = [None, (2, 2), (2, 8), (3, 5), (1, 1), (64, 16)]   # (first, max) MiB; None = defaults
SMALL_CHUNK_LIMIT = 512 * MiB    # chunk settings below 16 MiB only pair with sizes up to this
MODES = [(mf, il) for mf in (0, 1) for il in (0, 1)]                 # CCM_MAP_FIRST x CCM_INTERLEAVE_VERIFY
TAIL_MBS = (256, 2, 0)
VARIANT_PINS = [(sv, vv) for sv in ("st128", "st256", "tma", "memset") for vv in ("ld128", "ld256")]
FANOUT_SIZES = (GiB, 0)


def requested_sizes(gran: int) -> list[int]:
    return [1, gran - 1, gran, gran + 1, 100 * MiB + 1, 3 * GiB + 2 * MiB + 1, 7 * GiB + 3]


def chunk_env(setting) -> dict:
    if setting is None:
        return {}
    return {"CCM_VMM_FIRST_CHUNK_MB": str(setting[0]), "CCM_VMM_CHUNK_MB": str(setting[1])}


def mode_env(mf: int, il: int, async_release: int = 1) -> dict:
    return {"CCM_MAP_FIRST": str(mf), "CCM_INTERLEAVE_VERIFY": str(il), "CCM_ASYNC_RELEASE": str(async_release)}


def requested_cases(setting, gran: int) -> list[tuple[int, dict]]:
    small = setting is not None and setting[1] < 16
    sizes = [s for s in requested_sizes(gran) if not small or s <= SMALL_CHUNK_LIMIT]
    return [(s, {**chunk_env(setting), **mode_env(mf, il, ar)})
            for s in sizes for mf, il in MODES for ar in (1, 0)]


def whole_hbm_cases(tail_mb: int) -> list[dict]:
    return [{"CCM_VMM_TAIL_MB": str(tail_mb), **mode_env(mf, il)} for mf, il in MODES]


def variant_pin_env(sv: str, vv: str) -> dict:
    return {"CCM_SCRUB_VARIANT": sv, "CCM_VERIFY_VARIANT": vv, "CCM_MAP_FIRST": "1"}


def arena_cases(gran: int) -> list[tuple[int, dict]]:
    return [(gran + 1, {"CCM_PIPELINE": "0"}),
            (300 * MiB, {"CCM_PIPELINE": "0", "CCM_ARENA_MAX_SEGMENT_MB": "96"}),
            (0, {"CCM_PIPELINE": "0"}),
            (0, {"CCM_PIPELINE": "0", "CCM_ARENA_RESERVE_MB": "1024"})]


def pdl_cases() -> list[tuple[int, dict]]:
    """Run in one child per CCM_PDL value (the library latches it once per process)."""
    return [(100 * MiB + 1, {**chunk_env((2, 2)), **mode_env(0, 1)}), (0, {})]


PDL_VALUES = ("1", "0")


def swept_knobs(gran: int = H100_GRAN) -> dict[str, set[str]]:
    """Every CCM_* value the GPU matrix sets ("" = left at the library default)."""
    envs = [env for setting in CHUNK_SETTINGS for _, env in requested_cases(setting, gran)]
    envs += [env for t in TAIL_MBS for env in whole_hbm_cases(t)]
    envs += [variant_pin_env(sv, vv) for sv, vv in VARIANT_PINS]
    envs += [env for _, env in arena_cases(gran)]
    envs += [{**env, "CCM_PDL": pdl} for _, env in pdl_cases() for pdl in PDL_VALUES]
    out: dict[str, set[str]] = {}
    for env in envs:
        for k in set(PLAN_KNOBS) | {"CCM_PDL"} | set(env):
            out.setdefault(k, set()).add(env.get(k, ""))
    return out
