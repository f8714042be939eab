"""Deliberately wrong copies of libccm.so's device code, one small bug each, for tests/test_kernel_mutants.py: the
exactness driver (tests/sanitize_calls.py) must fail on every KILL mutant, for the reason its `killer` names, and pass
on every EQUIVALENT one.  A check that passes on a broken kernel is a check whose inputs never reach the broken case,
or whose expected value comes from the same code.  Not collected by pytest.

Each mutant replaces one `anchor` (exact source text that occurs once in `file`, under k8s_cc_manager_b200/) by
`replacement`.  `breaks` says what is now wrong; `safe` says why the mutant touches no address the original does not
and always terminates: it changes a value (what is written, counted, booked or compared, at the same addresses) or
narrows a loop (`i + 1 < bound`, never an unsigned bound minus one, which walks out of the region at 0).  No mutant
raises a bound, enlarges an offset, or touches a barrier, fence, griddepcontrol or warp mask.  `killer`: labels of the
driver's calls, each a string or a tuple of strings that must all occur in one failing call's label, one of which must
fail.  `phase`: the driver phase that holds the killer ("all" where the product calls do).  An EQUIVALENT mutant
carries, in `breaks`, the argument from the code that no result can change.

build(mutant) compiles a copy of csrc/ and include/ with the product's nvcc flags (build.compile_lib) into
tests/_mutants/<key>/libccm.so, keyed by a hash of the pristine sources, the flags and the mutant; build_all() builds
them in a process pool.  sass(lib) gives every function's instructions (cuobjdump -sass, addresses and encodings
stripped), so a SASS diff shows which kernel entries a mutant changed.
"""
from __future__ import annotations

import hashlib
import multiprocessing
import os
import re
import shutil
import subprocess
import tempfile
import time
from concurrent.futures import ProcessPoolExecutor
from dataclasses import dataclass
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
PKG = ROOT / "k8s_cc_manager_b200"
CACHE = ROOT / "tests" / "_mutants"
KERNELS = "csrc/scrub_kernels.cuh"
SCRUB = "csrc/ccm_scrub.cu"

KILL, EQUIVALENT = "KILL", "EQUIVALENT"
NARROW = "narrows a loop: it visits a subset of the original's indices and its exit test is reached sooner"
VALUE = "changes a value only: the same loads and stores at the same addresses, and the same loop bounds"


@dataclass(frozen=True)
class Mutant:
    id: str
    file: str
    anchor: str
    replacement: str
    breaks: str
    safe: str
    killer: tuple = ()
    kind: str = KILL
    phase: str = "region"


M = Mutant
MUTANTS = [
    # ---------------------------------------------------------------- counting
    M("nonzero_bytes_0x80", KERNELS,
      "  uint32_t m = (((w & 0x7f7f7f7fu) + 0x7f7f7f7fu) | w) & 0x80808080u;\n  return __popc(m);",
      "  uint32_t m = ((w & 0x7f7f7f7fu) + 0x7f7f7f7fu) & 0x80808080u;\n  return __popc(m);",
      "nonzero_bytes_in_word counts a byte of 0x80 as zero", VALUE,
      (("verify", "all bytes"), ("verify_ld_kernel", "all bytes"))),
    M("verify_tile_last_word", KERNELS,
      "      for (int k = 0; k < W; ++k) c += nonzero_bytes_in_word(w[u][k]);",
      "      for (int k = 0; k + 1 < W; ++k) c += nonzero_bytes_in_word(w[u][k]);",
      "verify_tile's exact count skips the last word of every vector", VALUE + " (the OR still reads every word)",
      ("verify_ld_kernel",)),
    M("count_chunk_last_vector", KERNELS,
      "      for (int u = 0; u < PER_THREAD; ++u)\n#pragma unroll\n"
      "        for (int k = 0; k < 4; ++k) n += nonzero_bytes_in_word(v[u].w[k]);",
      "      for (int u = 0; u + 1 < PER_THREAD; ++u)\n#pragma unroll\n"
      "        for (int k = 0; k < 4; ++k) n += nonzero_bytes_in_word(v[u].w[k]);",
      "CountNonzeroOp::chunk does not count the last vector of its batch", VALUE + " (all loads stay)",
      (("verify", "two grabs each"), ("verify", "all bytes"))),
    M("count_vec_last_word", KERNELS,
      "      for (int k = 0; k < 4; ++k) cnt += nonzero_bytes_in_word(v.w[k]);",
      "      for (int k = 0; k + 1 < 4; ++k) cnt += nonzero_bytes_in_word(v.w[k]);",
      "CountNonzeroOp::vec (16-byte vectors) does not count the vector's last word", VALUE,
      (("verify", "leftover vectors"), ("verify", "all bytes"))),
    M("count_vec32_last_word", KERNELS,
      "      for (int k = 0; k < 8; ++k) cnt += nonzero_bytes_in_word(v.w[k]);",
      "      for (int k = 0; k + 1 < 8; ++k) cnt += nonzero_bytes_in_word(v.w[k]);",
      "CountNonzeroOp::vec (32-byte vectors) does not count the vector's last word", VALUE,
      ("verify_ld_kernel<32",)),
    M("count_byte_gt1", KERNELS,
      "cnt += (*p != 0); }",
      "cnt += (*p > 1); }",
      "CountNonzeroOp::byte counts a ragged byte of 0x01 as zero", VALUE,
      (("verify", "all bytes"), ("verify_ld_kernel", "all bytes"))),
    M("block_accumulate_one", KERNELS,
      "    if (lane == 0 && v != 0) atomicAdd(counter, (unsigned long long)v);",
      "    if (lane == 0 && v > 1) atomicAdd(counter, (unsigned long long)v);",
      "block_accumulate drops the sum of a CTA that counted exactly one byte", VALUE + " (one atomic fewer)",
      ("verify_ld_kernel", "verify")),
    M("warp_sum_half", KERNELS,
      "  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);",
      "  for (int o = 16; o > 1; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);",
      "warp_sum_u64 skips its last butterfly step: lane 0 holds the sum of the even lanes only",
      NARROW + "; every lane of the warp still runs every shuffle it runs, with the full mask",
      ("verify_ld_kernel", "verify", "check")),
    # ---------------------------------------------------------------- writes
    M("zero_byte_7f", KERNELS,
      "  __device__ __forceinline__ void byte(uint8_t* p) { *p = 0; }",
      "  __device__ __forceinline__ void byte(uint8_t* p) { *p &= 0x7f; }",
      "ZeroOp::byte leaves bit 7 of each ragged byte", VALUE + " (a read and a write of the byte it wrote)",
      ("scrub_st_kernel", "scrub_tma_kernel", "scrub")),
    M("scrub_tile_unroll", KERNELS,
      "    for (int u = 0; u < UNROLL; ++u) st_zero16<POL>(p + u * stride_bytes, l2pol);",
      "    for (int u = 0; u + 1 < UNROLL; ++u) st_zero16<POL>(p + u * stride_bytes, l2pol);",
      "scrub_tile (16-byte vectors) skips the last unroll step of every tile", NARROW,
      ("scrub_st_kernel<16",)),
    M("scrub_tile32_half", KERNELS,
      "      st_zero16<POL>(p + u * stride_bytes + half, l2pol);\n",
      "",
      "scrub_tile (32-byte vectors) never stores the second half of a step", "drops a store: touches fewer addresses",
      ("scrub_st_kernel<32",)),
    M("tma_zero_tile", KERNELS,
      "    reinterpret_cast<uint4*>(zero_tile)[i] = make_uint4(0, 0, 0, 0);",
      "    reinterpret_cast<uint4*>(zero_tile)[i] = make_uint4(0, 0, 0, i == 0);",
      "scrub_tma_kernel's source tile holds a 1 in its first vector, so every bulk store writes it",
      VALUE + " (no bulk-copy size changes: a narrower legal size would leave whole tiles, not a subtle bug)",
      ("scrub_tma_kernel",)),
    M("tag_vec_word3", KERNELS,
      "(b + 2 * kTagK1) ^ h, (b + 3 * kTagK1) ^ h);",
      "(b + 2 * kTagK1) ^ h, (b + 2 * kTagK1) ^ h);",
      "tag_vec's fourth word is the third word's tag", VALUE,
      (("fill",), ("census1",), ("probe",))),
    M("tag_byte_x1", KERNELS,
      "  return (uint8_t)(tag_word(seed, x & ~3ull) >> (8 * (x & 3)));",
      "  return (uint8_t)(tag_word(seed, x & ~3ull) >> (8 * (x & 1)));",
      "tag_byte takes byte x & 1 of the word: bytes 2 and 3 get the tags of bytes 0 and 1", VALUE,
      (("fill",), ("census1",), ("check",))),
    M("tag_fill_vec_seed", KERNELS,
      "  __device__ __forceinline__ void vec(uint8_t* q) { st16(q, tag_vec(seed, addr(q))); }",
      "  __device__ __forceinline__ void vec(uint8_t* q) { st16(q, tag_vec(seed ^ 1u, addr(q))); }",
      "TagFillOp::vec writes a leftover vector with the tags of seed ^ 1", VALUE,
      (("fill", "leftover vectors"),)),
    M("xor_byte_zero", KERNELS,
      "__global__ void xor_byte_kernel(uint8_t* p) { *p ^= 0xA5; }",
      "__global__ void xor_byte_kernel(uint8_t* p) { *p ^= 0x00; }",
      "xor_byte_kernel (the inject drills) changes nothing", VALUE,
      ("product",), phase="all"),
    M("fill_byte_word0", SCRUB,
      "  const uint4 v = make_uint4(word, word, word, word);",
      "  const uint4 v = make_uint4(word + 1, word, word, word);",
      "fill_byte_kernel writes byte value + 1 into the first byte of every vector", VALUE,
      ("arena fill",)),
    M("fill_pattern_shift", KERNELS,
      "    words[i] = pattern_word(seed, word_index0 + i);",
      "    words[i] = pattern_word(seed, word_index0 + i + 1);",
      "fill_pattern_kernel writes word j + 1 of the pattern at word j", VALUE,
      ("arena pattern",)),
    # ---------------------------------------------------------------- frame
    M("ragged_head_short", KERNELS,
      "    for (uint64_t i = threadIdx.x; i < s.head; i += nthreads) op.byte(s.base + i);",
      "    for (uint64_t i = threadIdx.x; i + 1 < s.head; i += nthreads) op.byte(s.base + i);",
      "ragged_bytes skips the last head byte", NARROW,
      ("scrub", "verify", "fill")),
    M("ragged_tail_short", KERNELS,
      "    for (uint64_t i = threadIdx.x; i < s.tail; i += nthreads) op.byte(t + i);",
      "    for (uint64_t i = threadIdx.x; i + 1 < s.tail; i += nthreads) op.byte(t + i);",
      "ragged_bytes skips the last tail byte", NARROW,
      ("scrub", "verify", "fill")),
    M("finish_last_vector", KERNELS,
      "  for (uint64_t i = first_vec + (uint64_t)blockIdx.x * nthreads + threadIdx.x; i < s.body_vecs;",
      "  for (uint64_t i = first_vec + (uint64_t)blockIdx.x * nthreads + threadIdx.x; i + 1 < s.body_vecs;",
      "finish_region skips the last leftover vector", NARROW,
      ("leftover vectors", "scrub_st_kernel", "verify_ld_kernel")),
    M("grab_last_chunk", KERNELS,
      "    if (c >= nchunks) break;",
      "    if (c + 1 >= nchunks) break;",
      "grab_chunks stops before the last chunk", NARROW + "; the exit test stays uniform over the CTA (c is read from "
      "shared memory after the barrier)",
      ("two grabs each", "page-cut grab")),
    M("static_last_tile", KERNELS,
      "    for (uint64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) tile_fn(tile);",
      "    for (uint64_t tile = blockIdx.x; tile + 1 < ntiles; tile += gridDim.x) tile_fn(tile);",
      "for_each_tile's static schedule skips the last tile", NARROW,
      ("-s1-",)),
    M("per_warp_last_chunk", KERNELS,
      "    while (c < sched.nchunks) {",
      "    while (c + 1 < sched.nchunks) {",
      "for_each_tile's per-warp schedule stops before the last chunk", NARROW + "; c is the same in every lane (shuffled)",
      ("-s3-",)),
    M("chunk_tiles_last", KERNELS,
      "    for (uint64_t tile = t0; tile < t1; ++tile) tile_fn(tile);",
      "    for (uint64_t tile = t0; tile + 1 < t1; ++tile) tile_fn(tile);",
      "for_each_tile's chunk_tiles skips the last tile of every grabbed chunk", NARROW,
      ("-s2-", "-s3-", "-s0-")),
    M("grab_release_done", KERNELS,
      "    *g.grab = 0;\n    *g.done = 0;\n",
      "    *g.grab = 0;\n",
      "grab_release leaves `done` set: the launch after next on the same words starts from a stale grab and does nothing",
      "drops a store; every later grab loop still ends (a stale grab is >= nchunks)",
      ("scrub", "verify", "fill", "check")),
    M("release_keeps_counter", KERNELS,
      "  if (threadIdx.x == 0) grab_release(ctl, zero_on_exit);",
      "  if (threadIdx.x == 0) grab_release(ctl, nullptr);",
      "default_kernel never clears zero_on_exit: an arena scrub-and-verify step adds to the previous read-back's count",
      "drops a store",
      ("arena step",)),
    M("descending_ascending", KERNELS,
      "  default_kernel<THREADS, PER_THREAD, true>(s, nchunks, ctl, nullptr, op);\n  block_accumulate(op.cnt, counter);",
      "  default_kernel<THREADS, PER_THREAD, false>(s, nchunks, ctl, nullptr, op);\n"
      "  block_accumulate(op.cnt, counter);",
      "verify_ld128_fast_kernel reads its chunks in ascending order.  Equivalent: c -> nchunks - 1 - c is a bijection "
      "of [0, nchunks), so the same chunks are read, each once; the count is a sum of per-chunk counts, which does not "
      "depend on their order; the kernel writes nothing into the region.  Order is an L2 and speed property only",
      "reads the same chunks in another order", kind=EQUIVALENT),
    M("block_accumulate_whole_warps", KERNELS,
      "    uint64_t v = lane < ((blockDim.x + 31) >> 5) ? warp_part[lane] : 0;",
      "    uint64_t v = lane < (blockDim.x >> 5) ? warp_part[lane] : 0;",
      "block_accumulate rounds the warp count down.  Equivalent: every launch of a kernel that calls it has a block size "
      "that is a multiple of 32: the generic verifier through clamp_threads ((t / 32) * 32), the default-frame kernels "
      "at kFastVerifyThreads / kFastTagThreads, the probe at kProbeThreads (ccm_scrub.cu), so (b + 31) >> 5 == b >> 5",
      "reads fewer shared words (never more)", kind=EQUIVALENT),
    # ---------------------------------------------------------------- tag check
    M("check_count_byte3", KERNELS,
      "      n += nonzero_bytes_in_word(v[u].x ^ t.x) + nonzero_bytes_in_word(v[u].y ^ t.y) +\n"
      "           nonzero_bytes_in_word(v[u].z ^ t.z) + nonzero_bytes_in_word(v[u].w ^ t.w);",
      "      n += nonzero_bytes_in_word((v[u].x ^ t.x) & 0xffffffu) + nonzero_bytes_in_word((v[u].y ^ t.y) & 0xffffffu) +\n"
      "           nonzero_bytes_in_word((v[u].z ^ t.z) & 0xffffffu) + nonzero_bytes_in_word((v[u].w ^ t.w) & 0xffffffu);",
      "TagCheckZeroOp::chunk never counts byte 3 of a word as a mismatch", VALUE,
      (("check", "all bytes"), ("check", "two grabs each"))),
    M("check_zero_window_word3", KERNELS,
      "    book.count += (v.w[0] | v.w[1] | v.w[2] | v.w[3]) == 0;",
      "    book.count += (v.w[0] | v.w[1] | v.w[2]) == 0;",
      "TagCheckZeroOp::window counts a mismatched window as all-zero when only its last word is non-zero", VALUE,
      (("check", "all bytes"),)),
    M("check_vec_byte15", KERNELS,
      "    st16(q, make_uint4(0, 0, 0, 0));\n    cnt += __popc(mask);",
      "    st16(q, make_uint4(0, 0, 0, 0));\n    cnt += __popc(mask & 0x7fffu);",
      "TagCheckZeroOp::vec does not count byte 15 of a leftover vector", VALUE,
      (("check", "leftover vectors"), ("check", "all bytes"))),
    M("check_chunk_store", KERNELS,
      "    for (int u = 0; u < PER_THREAD; ++u) st16(p + (uint32_t)u * THREADS * 16u, make_uint4(0, 0, 0, 0));",
      "    for (int u = 0; u < PER_THREAD; ++u) st16(p + (uint32_t)u * THREADS * 16u, make_uint4(0, 0, 0, u == 0));",
      "TagCheckZeroOp::chunk leaves a 1 in the first vector of every batch", VALUE,
      ("check",)),
    M("check_ragged_store", KERNELS,
      "        *b = 0;\n",
      "        *b = (uint8_t)(w0 + i + 1 == hi);\n",
      "TagCheckZeroOp::ragged_windows leaves a 1 in the last byte of every head and tail window", VALUE,
      ("check",)),
    # ---------------------------------------------------------------- books
    M("claim_63", KERNELS,
      "    if (slot + 1 >= (uint64_t)kDirtRecords) {",
      "    if (slot + 2 >= (uint64_t)kDirtRecords) {",
      "WindowBook::claim sets the full flag one slot early: 63 records, not 64", VALUE + " (records go to slots < 64 "
      "only, as before)",
      ("64 windows in warp rounds",)),
    M("tally_last_low", KERNELS,
      "    last = max(last, hi);\n  }",
      "    last = max(last, hi - (hi != lo));\n  }",
      "WindowBook::tally books the last byte of a window with more than one byte one low", VALUE,
      ("locate", "check")),
    M("tally_span_windows", KERNELS,
      "    windows += n;\n    first_inv",
      "    windows += n > 1 ? n - 1 : n;\n    first_inv",
      "WindowBook::tally_span books one window fewer for a batch with several", VALUE,
      ("census0", "census1")),
    M("flush_one_window", KERNELS,
      "      if (lane == 0 && b != 0) {",
      "      if (lane == 0 && b > 1) {",
      "WindowBook::flush drops the words of a CTA that booked exactly one window", VALUE + " (fewer atomics)",
      ("locate", "check", "census0", "census1", "probe", "product")),
    M("pages_batch_crosses", KERNELS,
      "      if (crosses && hi) atomicAdd(out.pages + page + 1, hi);\n",
      "",
      "WindowBook::pages_batch drops the bytes of a batch that lie on the next page", "drops an atomic",
      ("page-cut grab",)),
    M("pages_window_low", KERNELS,
      "    bytes = __reduce_add_sync(peers, bytes);",
      "    bytes = __reduce_add_sync(peers, bytes - (bytes > 1));",
      "WindowBook::pages_window books a window with several bytes one byte low on its page", VALUE,
      ("locate", "check", "census0", "census1")),
    M("record_bytes_word3", KERNELS,
      "    r.bytes = make_uint4(v.w[0], v.w[1], v.w[2], v.w[3]);",
      "    r.bytes = make_uint4(v.w[0], v.w[1], v.w[2], v.w[3] & 0xffffffu);",
      "WindowBook::record keeps byte 15 of a window as 0", VALUE,
      ("locate", "check")),
    M("record_mask_bit0", KERNELS,
      "recs[slot] = MaskRecord{off, 0u, (uint16_t)mask, (uint16_t)0};",
      "recs[slot] = MaskRecord{off, 0u, (uint16_t)(mask | 1u), (uint16_t)0};",
      "WindowBook::record_mask records byte 0 of every census window as non-zero", VALUE,
      ("census0", "census1")),
    M("mask16_byte15", KERNELS,
      "    m |= (((f >> 7) & 1u) | ((f >> 14) & 2u) | ((f >> 21) & 4u) | ((f >> 28) & 8u)) << (4 * k);\n  }\n  return m;",
      "    m |= (((f >> 7) & 1u) | ((f >> 14) & 2u) | ((f >> 21) & 4u) | ((f >> 28) & 8u)) << (4 * k);\n  }\n"
      "  return m & 0x7fffu;",
      "nonzero_mask16 never books byte 15 of a window", VALUE,
      ("locate", "check", "census0", "census1")),
    M("locate_chunk_byte15", KERNELS,
      "        const uint32_t mask = nonzero_mask16(v[u]);",
      "        const uint32_t mask = nonzero_mask16(v[u]) & 0x7fffu;",
      "LocateOp::chunk never books byte 15 of a window of a batch", VALUE,
      ("locate",)),
    M("locate_vec_byte0", KERNELS,
      "    single(addr(p) - base, nonzero_mask16(v), v);",
      "    single(addr(p) - base, nonzero_mask16(v) & 0xfffeu, v);",
      "LocateOp::vec never books byte 0 of a leftover vector", VALUE,
      (("locate", "leftover vectors"), ("locate", "all bytes"))),
    M("locate_ragged_short", KERNELS,
      "      if (w0 + i >= lo && w0 + i < hi) v.w[i >> 2] |=",
      "      if (w0 + i >= lo && w0 + i + 1 < hi) v.w[i >> 2] |=",
      "LocateOp::ragged_windows does not read the last byte of a head or tail window", NARROW,
      ("locate",)),
    M("ragged_window_head", KERNELS,
      "  if (t < nhead) { w0 = first_win + 16 * t; lo = max(w0, a0); hi = min(w0 + 16, head_end); return true; }",
      "  if (t < nhead) { w0 = first_win + 16 * t; lo = max(w0, a0); hi = min(w0 + 15, head_end); return true; }",
      "ragged_window leaves out the last byte of every whole head window", NARROW + " (hi only shrinks)",
      ("head windows", "all bytes", "probe")),
    # ---------------------------------------------------------------- census
    M("census_zero_store", KERNELS,
      "    else st16(q, make_uint4(0, 0, 0, 0));",
      "    else st16(q, make_uint4(0, 0, 0, 1));",
      "CensusOp<false>::store leaves a 1 in byte 12 of every vector", VALUE,
      ("census0",)),
    M("census_tag_store", KERNELS,
      "    if constexpr (TAGS) st16(q, tag_vec(seed, addr(q)));",
      "    if constexpr (TAGS) st16(q, tag_vec(seed ^ 1u, addr(q)));",
      "CensusOp<true>::store writes the tags of seed ^ 1", VALUE,
      ("census1",)),
    M("census_ragged_zero", KERNELS,
      "        *b = TAGS ? tag_byte(seed, w0 + i) : (uint8_t)0;",
      "        *b = TAGS ? tag_byte(seed, w0 + i) : (uint8_t)(w0 + i + 1 == hi);",
      "CensusOp<false>::ragged_windows leaves a 1 in the last byte of every head and tail window", VALUE,
      ("census0",)),
    M("census_record_last", KERNELS,
      "      for (int u = 0; u < PER_THREAD; ++u)\n        if (mask[u] != 0) book.record_mask(",
      "      for (int u = 0; u + 1 < PER_THREAD; ++u)\n        if (mask[u] != 0) book.record_mask(",
      "CensusOp::chunk never records the last vector of a batch", NARROW,
      ("census0", "census1")),
    # ---------------------------------------------------------------- cover maps
    M("cover_add_short", KERNELS,
      "  atomicAdd(c.map + cover_word(c, a), lo);",
      "  atomicAdd(c.map + cover_word(c, a), lo - 1);",
      "cover_add counts one byte fewer per chunk", VALUE + " (lo >= 1: n > 0 and room >= 1)",
      ("armed",)),
    M("cover_lanes_short", KERNELS,
      "  const uint32_t sum = __reduce_add_sync(peers, lo);",
      "  const uint32_t sum = __reduce_add_sync(peers, lo - 1);",
      "cover_lanes counts one byte fewer per lane", VALUE,
      ("armed",)),
    M("cover_op_byte", KERNELS,
      "    if constexpr (BYTES) cover_lanes(cover, addr(p), 1u);",
      "    if constexpr (BYTES) if (addr(p) & 1) cover_lanes(cover, addr(p), 1u);",
      "CoverOp::byte does not count a ragged byte at an even address", VALUE + " (cover_lanes reduces over the "
      "active lanes, as it does in every other divergent caller)",
      (("armed", "scrub"), ("armed", "fill"), ("armed", "verify"))),
    M("cover_ragged_short", KERNELS,
      "  if (ragged_window(s, w0, lo, hi) && hi > lo) cover_lanes(c, lo, (uint32_t)(hi - lo));",
      "  if (ragged_window(s, w0, lo, hi) && hi > lo) cover_lanes(c, lo, (uint32_t)(hi - lo - 1));",
      "cover_ragged_windows counts one byte fewer per ragged window", VALUE,
      ("armed",)),
    # ---------------------------------------------------------------- probe
    M("probe_fill_second_half", KERNELS,
      "      st16((void*)(uintptr_t)(q + 16), tag_vec(seed, q + 16));",
      "      st16((void*)(uintptr_t)(q + 16), tag_vec(seed, q));",
      "ProbeFillOp writes the first half's tags into the second half of a window", VALUE,
      ("probe",)),
    M("probe_check_word0", KERNELS,
      "        n += nonzero_bytes_in_word(v[u][h].x ^ t.x) + nonzero_bytes_in_word(v[u][h].y ^ t.y) +",
      "        n += nonzero_bytes_in_word(0u) + nonzero_bytes_in_word(v[u][h].y ^ t.y) +",
      "ProbeCheckOp ignores the first word of each 16-byte half", VALUE + " (the load stays)",
      ("product",), phase="all"),
    M("probe_reread_word0", KERNELS,
      "        for (int k = 0; k < 4; ++k) n += nonzero_bytes_in_word(v[u][0].w[k]) + nonzero_bytes_in_word(v[u][1].w[k]);",
      "        for (int k = 1; k < 4; ++k) n += nonzero_bytes_in_word(v[u][0].w[k]) + nonzero_bytes_in_word(v[u][1].w[k]);",
      "ProbeRereadOp ignores the first word of each 16-byte half", VALUE + " (registers only: the OR still reads every "
      "word)",
      ("product",), phase="all"),
    M("probe_tail_window", KERNELS,
      "       i += (uint64_t)gridDim.x * THREADS)\n    op.template batch<1>(w0 + i * kProbeStride, 0);",
      "       i += (uint64_t)gridDim.x * THREADS)\n    if (i + 1 < nwin) op.template batch<1>(w0 + i * kProbeStride, 0);",
      "probe_windows skips the last window after the whole batches", NARROW,
      ("probe",)),
    M("cover_probe_short", KERNELS,
      "    for (int u = 0; u < K; ++u) cover_lanes(cover, a + u * step, kProbeWindow);",
      "    for (int u = 0; u < K; ++u) cover_lanes(cover, a + u * step, kProbeWindow - 1);",
      "CoverProbeOp counts 31 bytes per window", VALUE,
      (("probe", "armed"),)),
]

BY_ID = {m.id: m for m in MUTANTS}
assert len(BY_ID) == len(MUTANTS), "mutant ids must be unique"


def source(m: Mutant) -> str:
    return (PKG / m.file).read_text()


def anchor_count(m: Mutant) -> int:
    return source(m).count(m.anchor)


def _digest() -> hashlib._Hash:
    """A hash of the pristine sources and the product's compile flags."""
    from k8s_cc_manager_b200 import build as B
    h = hashlib.sha256(" ".join(B.NVCC_FLAGS).encode())
    for p in sorted(list((PKG / "csrc").iterdir()) + list((ROOT / "include").iterdir())):
        if p.is_file():
            h.update(p.name.encode() + b"\0" + p.read_bytes())
    return h


def lib_path(m: Mutant | None) -> Path:
    h = _digest()
    if m is not None:
        h.update(repr((m.file, m.anchor, m.replacement)).encode())
    return CACHE / f"{m.id if m else 'pristine'}-{h.hexdigest()[:16]}" / "libccm.so"


def build(m: Mutant | None) -> tuple:
    """(library, seconds spent compiling: 0 when cached) of mutant m; None: the pristine sources, rebuilt."""
    from k8s_cc_manager_b200 import build as B
    out = lib_path(m)
    if out.exists():
        return out, 0.0
    t0 = time.perf_counter()
    with tempfile.TemporaryDirectory(prefix="ccm-mutant-") as tmp:
        src = Path(tmp) / "csrc"
        inc = Path(tmp) / "include"
        shutil.copytree(PKG / "csrc", src)
        shutil.copytree(ROOT / "include", inc)
        if m is not None:
            f = Path(tmp) / m.file
            text = f.read_text()
            assert text.count(m.anchor) == 1, f"{m.id}: its anchor occurs {text.count(m.anchor)} times in {m.file}"
            f.write_text(text.replace(m.anchor, m.replacement))
        B.compile_lib(src, inc, Path(tmp) / "libccm.so")
        out.parent.mkdir(parents=True, exist_ok=True)
        part = out.with_suffix(".part")
        shutil.copyfile(Path(tmp) / "libccm.so", part)
        os.replace(part, out)
    return out, time.perf_counter() - t0


def _build_id(mid: str | None) -> tuple:
    return build(BY_ID[mid] if mid else None)


def build_all(workers: int | None = None) -> tuple:
    """({mutant id or None for the pristine rebuild: library}, compile seconds summed, wall seconds)."""
    ids = [None] + [m.id for m in MUTANTS]
    t0 = time.perf_counter()
    # spawn, not fork: the caller (pytest, torch) may have threads running
    with ProcessPoolExecutor(max_workers=workers or os.cpu_count() or 1,
                             mp_context=multiprocessing.get_context("spawn")) as pool:
        res = dict(zip(ids, pool.map(_build_id, ids)))
    return {k: v[0] for k, v in res.items()}, sum(v[1] for v in res.values()), time.perf_counter() - t0


_COMMENT = re.compile(r"/\*.*?\*/")


def sass(lib: Path) -> dict:
    """{mangled function name: [instructions]} of every function in lib, addresses and encodings stripped."""
    from k8s_cc_manager_b200 import build as B
    cuobjdump = Path(B.find_nvcc()).parent / "cuobjdump"
    out = subprocess.run([str(cuobjdump), "-sass", str(lib)], check=True, capture_output=True, text=True).stdout
    funcs, cur = {}, None
    for line in out.splitlines():
        s = line.strip()
        if s.startswith("Function : "):
            cur = funcs.setdefault(s[len("Function : "):], [])
            continue
        s = _COMMENT.sub("", s).strip()
        if cur is not None and s and not s.startswith(".") and s not in ("{", "}"):
            cur.append(s)
    return funcs


def changed(a: dict, b: dict) -> set:
    """Functions whose instructions differ between two sass() results (or that only one has)."""
    return {f for f in set(a) | set(b) if a.get(f) != b.get(f)}


def killed_by(label: list, killer) -> bool:
    """True when one failing call's label matches one killer: a string, or a tuple of strings that must all occur."""
    text = " | ".join(label)
    return any(all(k in text for k in ((pat,) if isinstance(pat, str) else pat)) for pat in killer)
