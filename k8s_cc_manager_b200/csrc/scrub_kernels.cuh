// scrub_kernels.cuh — sm_90a (Hopper) kernels of the HBM scrub-and-verify stage.
//
// SURVEY.md §8a row S: the reference has NO scrub (reference main.py:502-529 goes
// stage -> reset -> wait -> verify-mode only); these kernels are the new stage
// inserted after main.py:529.  Contract: after scrub every byte of the region is
// 0x00; verify returns the EXACT number of bytes != 0 (u64).
//
// Bound: HBM bandwidth.  Integer / byte work only — no FP, no tensor cores (there
// is no contraction).  Algorithmic bytes: scrub = R written, verify = R read.
//
// Region decomposition (any pointer, any length):
//   [ head bytes | body: whole VB-byte vectors, VB-aligned | tail bytes ]
// head/tail are < 128+VB bytes and are handled with byte accesses by CTA 0; the
// body is cut into tiles (tile = threads * UNROLL vectors; every warp instruction
// covers whole 128-byte lines -> only full-sector writes) that are handed to
// PERSISTENT CTAs (grid = ctas_per_sm * #SMs) either statically (grid-stride) or —
// the default — dynamically: a CTA grabs the next chunk of tiles off an atomic
// counter, so SMs that drain faster take more work (see "work distribution").
//
// The widest global access Hopper has is 128 bits (STG.128 / LDG.128).  VB = 16 is
// the native vector; VB = 32 (the "256" variants) gives every thread 32 bytes per
// unroll step as two 128-bit accesses: inside a tile, step u of a group of G threads
// covers G*32 contiguous bytes as two lane-contiguous halves of G*16 bytes (thread i
// at i*16 and at G*16 + i*16), so each warp instruction still writes whole lines.
//
// Kernels in this file:
//   scrub_st128_fast_kernel / verify_ld128_fast_kernel   what AUTO launches (compile-time shape)
//   scrub_st_kernel / verify_ld_kernel                   any shape / width / policy / schedule
//   scrub_tma_kernel                                     cp.async.bulk stores from one zero tile
//   tag_fill_kernel / tag_check_zero_kernel              the tagged gate's known-answer pass
//   locate_dirt_kernel                                   where the dirt is, after a failed read-back
//   census_zero_kernel / census_tag_fill_kernel          what the first pass found before it erased it
//   cover_*_pass                                         proving twins of the six above that run a product call's
//                                                        passes: they count the bytes they walk per 2 MiB page;
//                                                        cover_locate_pass also runs a failed call's reports
//   alias_probe_*_pass                                  the alias probe's three steps (one 32-byte window per 4 KiB)
//   cover_probe_*_pass                                   their proving twins: they count the windows they take per page
//   fill_pattern_kernel                                  seeded test pattern (tests only)
// The grab loop (grab_chunks) and the epilogue after the last whole chunk or tile (finish_region,
// ragged_bytes) are written once.  The five compile-time-shape kernels are one frame (default_kernel)
// around an op struct that says what happens to each chunk, leftover vector and ragged byte.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace ccm {

enum CachePolicy : int { kPolDefault = 0, kPolEvictFirst = 1, kPolStreaming = 2, kPolEvictLast = 3 };

// ---------------------------------------------------------------- PTX wrappers
// 128-bit stores/loads take an L2 eviction priority only through a createpolicy
// cache hint (an .L2::cache_hint operand).
template <int POL>
__device__ __forceinline__ uint64_t make_l2_policy() {
  uint64_t pol = 0;
  if constexpr (POL == kPolEvictFirst)
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  if constexpr (POL == kPolEvictLast)
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}

template <int POL>
__device__ __forceinline__ void st_zero16(void* p, uint64_t l2pol) {
  if constexpr (POL == kPolEvictFirst || POL == kPolEvictLast)
    asm volatile("st.global.L2::cache_hint.v4.b32 [%0], {%1,%1,%1,%1}, %2;" ::"l"(p), "r"(0), "l"(l2pol) : "memory");
  else if constexpr (POL == kPolStreaming)
    asm volatile("st.global.cs.v4.b32 [%0], {%1,%1,%1,%1};" ::"l"(p), "r"(0) : "memory");
  else
    asm volatile("st.global.v4.b32 [%0], {%1,%1,%1,%1};" ::"l"(p), "r"(0) : "memory");
}

// 32 bytes at one address as two 128-bit stores (Hopper has no 256-bit store).  Used for the
// few vectors after the last whole tile; tiles use the lane-contiguous halves (scrub_tile).
template <int POL>
__device__ __forceinline__ void st_zero32(void* p, uint64_t l2pol) {
  st_zero16<POL>(p, l2pol);
  st_zero16<POL>((uint8_t*)p + 16, l2pol);
}

template <int VB, int POL>
__device__ __forceinline__ void st_zero(void* p, uint64_t l2pol) {
  if constexpr (VB == 32) st_zero32<POL>(p, l2pol); else st_zero16<POL>(p, l2pol);
}

struct Vec16 { uint32_t w[4]; };
struct Vec32 { uint32_t w[8]; };

template <int POL>
__device__ __forceinline__ Vec16 ld16(const void* p, uint64_t l2pol) {
  Vec16 v;
  if constexpr (POL == kPolEvictFirst || POL == kPolEvictLast)
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.b32 {%0,%1,%2,%3}, [%4], %5;"
                 : "=r"(v.w[0]), "=r"(v.w[1]), "=r"(v.w[2]), "=r"(v.w[3]) : "l"(p), "l"(l2pol));
  else if constexpr (POL == kPolStreaming)
    asm volatile("ld.global.nc.L1::no_allocate.v4.b32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.w[0]), "=r"(v.w[1]), "=r"(v.w[2]), "=r"(v.w[3]) : "l"(p));
  else
    asm volatile("ld.global.nc.v4.b32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.w[0]), "=r"(v.w[1]), "=r"(v.w[2]), "=r"(v.w[3]) : "l"(p));
  return v;
}

// 32 bytes at one address as two 128-bit loads (vectors after the last whole tile, see above).
template <int POL>
__device__ __forceinline__ Vec32 ld32(const void* p, uint64_t l2pol) {
  const Vec16 a = ld16<POL>(p, l2pol), b = ld16<POL>((const uint8_t*)p + 16, l2pol);
  Vec32 v;
#pragma unroll
  for (int k = 0; k < 4; ++k) { v.w[k] = a.w[k]; v.w[4 + k] = b.w[k]; }
  return v;
}

// Exact number of non-zero BYTES in a 32-bit word, branch-free:
// bit 7 of each byte of m is set iff that byte != 0.
__device__ __forceinline__ uint32_t nonzero_bytes_in_word(uint32_t w) {
  uint32_t m = (((w & 0x7f7f7f7fu) + 0x7f7f7f7fu) | w) & 0x80808080u;
  return __popc(m);
}

// ------------------------------------------------------------------- layout
struct RegionSplit {
  uint8_t* base;       // region start
  uint64_t head;       // bytes before the aligned body
  uint64_t body_vecs;  // number of VB-byte vectors in the body
  uint64_t tail;       // bytes after the body
};

__host__ __device__ inline RegionSplit split_region(const void* p, uint64_t n, int vb, int align) {
  RegionSplit s;
  s.base = (uint8_t*)p;
  uint64_t mis = (uint64_t)(uintptr_t)p & (uint64_t)(align - 1);
  uint64_t head = mis ? (uint64_t)align - mis : 0;
  if (head > n) head = n;
  s.head = head;
  s.body_vecs = (n - head) / (uint64_t)vb;
  s.tail = (n - head) - s.body_vecs * (uint64_t)vb;
  return s;
}

// ------------------------------------------------------------ work distribution
// Tiles are handed to the persistent CTAs either statically (grid-stride) or
// DYNAMICALLY: a CTA grabs the next chunk of `chunk_tiles` consecutive tiles with
// one atomicAdd on a device counter (zeroed by the host before the launch).  The
// grab for chunk k+1 is issued before the stores of chunk k, so its latency is
// hidden.  Why: SMs do not all drain their stores into the memory system at the
// same rate; with a static split the slowest SM sets the kernel time.
struct Sched {
  unsigned long long* counter;  // nullptr = static grid-stride
  uint32_t chunk_tiles;         // tiles per grab (dynamic only)
  uint64_t ntiles;              // whole tiles in the body   } computed on the host: no 64-bit
  uint64_t nchunks;             // ceil(ntiles / chunk_tiles) } divides in the kernel prologue
  uint32_t per_warp;            // 1: every WARP grabs its own chunks (tile = 32 lanes x UNROLL vectors);
                                //    no block barrier, no shared memory in the hot loop
};

// One CTA grabs chunks [0, nchunks) off *counter and calls body(c) for each, with every thread of the
// CTA.  Double-buffered: thread 0 has the grab for the next chunk in flight while the CTA works on this one,
// and one block barrier per chunk publishes it.
template <typename Body>
__device__ __forceinline__ void grab_chunks(unsigned long long* counter, uint64_t nchunks, Body&& body) {
  __shared__ unsigned long long s_chunk[2];
  if (threadIdx.x == 0) s_chunk[0] = atomicAdd(counter, 1ull);
  __syncthreads();
  int buf = 0;
  for (;;) {
    const uint64_t c = s_chunk[buf];
    if (c >= nchunks) break;
    unsigned long long nxt = 0;
    // next grab in flight while we work.  The raw result goes straight to shared memory at the end of
    // the iteration: any arithmetic on it here would make warp 0 wait out the atomic's round trip
    // before its stores.
    if (threadIdx.x == 0) nxt = atomicAdd(counter, 1ull);
    body(c);
    if (threadIdx.x == 0) s_chunk[buf ^ 1] = nxt;
    __syncthreads();
    buf ^= 1;  // two slots: a slow warp may still be reading slot k when thread 0 already writes slot k+1
  }
}

// Calls tile_fn(tile) for every tile this thread's group covers under `sched`: grid-stride (static), chunks
// grabbed by each warp, or chunks grabbed by each CTA.  idx: the thread's index in its group (the lane, when
// every warp grabs); the kernel has it live anyway, and testing it rather than threadIdx.x & 31 keeps the
// generic kernels' register counts and spills where they were.
template <typename TileFn>
__device__ __forceinline__ void for_each_tile(const Sched& sched, uint32_t idx, TileFn&& tile_fn) {
  const uint64_t ntiles = sched.ntiles;
  auto chunk_tiles = [&](uint64_t c) {
    const uint64_t t0 = c * sched.chunk_tiles;
    const uint64_t t1 = t0 + sched.chunk_tiles < ntiles ? t0 + sched.chunk_tiles : ntiles;
    for (uint64_t tile = t0; tile < t1; ++tile) tile_fn(tile);
  };
  if (sched.counter == nullptr) {
    for (uint64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) tile_fn(tile);
  } else if (sched.per_warp) {
    unsigned long long c = 0;
    if (idx == 0) c = atomicAdd(sched.counter, 1ull);
    c = __shfl_sync(0xffffffffu, c, 0);
    while (c < sched.nchunks) {
      unsigned long long nxt = 0;
      if (idx == 0) nxt = atomicAdd(sched.counter, 1ull);  // prefetch the next grab
      chunk_tiles(c);
      c = __shfl_sync(0xffffffffu, nxt, 0);
    }
  } else {
    grab_chunks(sched.counter, sched.nchunks, chunk_tiles);
  }
}

// ------------------------------------------------------------------ epilogue
// CTA 0 takes the ragged head and tail bytes, op.byte(p) for each.
template <int VB, typename Op>
__device__ __forceinline__ void ragged_bytes(const RegionSplit& s, uint32_t nthreads, Op& op) {
  if (blockIdx.x == 0) {
    for (uint64_t i = threadIdx.x; i < s.head; i += nthreads) op.byte(s.base + i);
    uint8_t* t = s.base + s.head + s.body_vecs * VB;
    for (uint64_t i = threadIdx.x; i < s.tail; i += nthreads) op.byte(t + i);
  }
}

// The vectors from first_vec on (what is left after the last whole chunk or tile: less than one of them),
// op.vec(p) spread over the grid, then the ragged head / tail bytes.
template <int VB, typename Op>
__device__ __forceinline__ void finish_region(const RegionSplit& s, uint64_t first_vec, uint32_t nthreads, Op& op) {
  uint8_t* body = s.base + s.head;
  for (uint64_t i = first_vec + (uint64_t)blockIdx.x * nthreads + threadIdx.x; i < s.body_vecs;
       i += (uint64_t)gridDim.x * nthreads)
    op.vec(body + i * VB);
  ragged_bytes<VB>(s, nthreads, op);
}

// ----------------------------------------------------- default shapes, tight loops
// The four kernels built on default_kernel below are what AUTO and the tagged gate launch.  Same
// algorithm as scrub_st_kernel / verify_ld_kernel with a per-CTA dynamic schedule, but block size and
// vectors per thread are compile-time constants, so one chunk = THREADS * PER_THREAD * 16 bytes is
// addressed from ONE 64-bit base with immediate offsets: PER_THREAD STG.128 / LDG.128 per thread per
// chunk (consecutive lanes touch consecutive 16-byte vectors, so every warp instruction covers
// four whole 128-byte lines) and a few instructions of bookkeeping, instead of a 64-bit add pair
// per access in the generic kernel (runtime stride).
//
// Launch bookkeeping lives IN the kernel: the grab counter is handed back zeroed by the last
// CTA to finish (GrabCtl below), so a step is two kernel nodes and nothing else — no
// cudaMemsetAsync nodes in front of each launch, which would cost a few microseconds apiece
// on small regions.  griddepcontrol.wait / launch_dependents let the host chain the
// two kernels with programmatic dependent launch (no-ops when launched the ordinary way).
struct GrabCtl {
  unsigned long long* grab;  // next chunk index; 0 before and after every launch
  unsigned long long* done;  // CTAs that have stopped grabbing; 0 before and after every launch
};

// One thread per CTA calls this after the CTA's last grab returned: the CTA that arrives last
// knows nobody will touch `grab` again and resets both words for the next launch on the stream.
__device__ __forceinline__ void grab_release(const GrabCtl& g, unsigned long long* also_zero) {
  __threadfence();
  if (atomicAdd(g.done, 1ull) == (unsigned long long)gridDim.x - 1) {
    *g.grab = 0;
    *g.done = 0;
    if (also_zero) *also_zero = 0;
    __threadfence();
  }
}

__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// The frame of the four default kernels: persistent CTAs grab whole chunks (from the top of the region
// down when DESCENDING) and hand each to op.chunk<THREADS, PER_THREAD>(p), where p is this thread's first
// vector and its PER_THREAD vectors are at p + u * THREADS * 16; then the self-resetting GrabCtl, then the
// vectors after the last whole chunk and the ragged bytes (finish_region).
// zero_on_exit (may be null): a word the last CTA clears as well.
template <int THREADS, int PER_THREAD, bool DESCENDING, typename Op>
__device__ __forceinline__ void default_kernel(const RegionSplit& s, uint64_t nchunks, const GrabCtl& ctl,
                                               unsigned long long* zero_on_exit, Op& op) {
  constexpr uint64_t kChunk = (uint64_t)THREADS * PER_THREAD * 16;
  uint8_t* body = s.base + s.head;
  pdl_wait();
  grab_chunks(ctl.grab, nchunks, [&](uint64_t c) {
    op.template chunk<THREADS, PER_THREAD>(body + (DESCENDING ? nchunks - 1 - c : c) * kChunk + threadIdx.x * 16u);
  });
  pdl_launch_dependents();
  if (threadIdx.x == 0) grab_release(ctl, zero_on_exit);
  finish_region<16>(s, nchunks * (kChunk / 16), THREADS, op);
}

// ------------------------------------------------------------- scrub (stores)
template <int VB, int POL>
struct ZeroOp {
  uint64_t l2pol;
  template <int THREADS, int PER_THREAD>
  __device__ __forceinline__ uint32_t chunk(uint8_t* p) {
#pragma unroll
    for (int u = 0; u < PER_THREAD; ++u) st_zero16<POL>(p + (uint32_t)u * THREADS * 16u, l2pol);
    return (uint32_t)PER_THREAD * 16u;
  }
  __device__ __forceinline__ void vec(uint8_t* p) { st_zero<VB, POL>(p, l2pol); }
  __device__ __forceinline__ void byte(uint8_t* p) { *p = 0; }
};

template <int VB, int UNROLL, int POL>
__device__ __forceinline__ void scrub_tile(uint8_t* body, uint64_t tile, uint64_t tile_vecs, uint32_t idx,
                                           uint64_t stride_bytes, uint64_t l2pol) {
  if constexpr (VB == 32) {
    // lane-contiguous halves: stride_bytes = group * 32, each half is group * 16 bytes
    uint8_t* p = body + tile * tile_vecs * 32 + (uint64_t)idx * 16;
    const uint64_t half = stride_bytes / 2;
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      st_zero16<POL>(p + u * stride_bytes, l2pol);
      st_zero16<POL>(p + u * stride_bytes + half, l2pol);
    }
  } else {
    uint8_t* p = body + (tile * tile_vecs + idx) * VB;
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) st_zero16<POL>(p + u * stride_bytes, l2pol);
  }
}

template <int VB, int UNROLL, int POL>
__global__ void __launch_bounds__(1024)
scrub_st_kernel(RegionSplit s, Sched sched) {
  uint8_t* body = s.base + s.head;
  const uint32_t group = sched.per_warp ? 32u : blockDim.x;   // threads that share one tile
  const uint32_t idx = sched.per_warp ? (threadIdx.x & 31u) : threadIdx.x;
  const uint64_t tile_vecs = (uint64_t)group * UNROLL;
  const uint64_t stride_bytes = (uint64_t)group * VB;
  ZeroOp<VB, POL> op{make_l2_policy<POL>()};
  for_each_tile(sched, idx, [&](uint64_t tile) {
    scrub_tile<VB, UNROLL, POL>(body, tile, tile_vecs, idx, stride_bytes, op.l2pol);
  });
  finish_region<VB>(s, sched.ntiles * tile_vecs, blockDim.x, op);
}

// zero_on_exit (may be null): the arena step passes the verify counter, so "scrub" also resets the
// verdict of the previous read-back.
template <int THREADS, int PER_THREAD, int POL>
__global__ void __launch_bounds__(THREADS)
scrub_st128_fast_kernel(RegionSplit s, uint64_t nchunks, GrabCtl ctl, unsigned long long* zero_on_exit) {
  ZeroOp<16, POL> op{0};
  default_kernel<THREADS, PER_THREAD, false>(s, nchunks, ctl, zero_on_exit, op);
}

// ------------------------------------------------------ scrub (TMA bulk store)
// One zeroed shared-memory tile per CTA is the source of EVERY bulk store: it
// never changes, so there is no WAR hazard and no per-op wait — the issuing lane
// streams cp.async.bulk.global.shared::cta ops (SASS: UBLKCP.G.S) grid-strided
// over the body and drains them once at exit.
template <int POL>
__device__ __forceinline__ void bulk_store(uint8_t* dst, uint32_t src_smem, uint32_t bytes, uint64_t policy) {
  if constexpr (POL == kPolEvictFirst || POL == kPolEvictLast)
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group.L2::cache_hint [%0], [%1], %2, %3;"
                 ::"l"(dst), "r"(src_smem), "r"(bytes), "l"(policy) : "memory");
  else
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                 ::"l"(dst), "r"(src_smem), "r"(bytes) : "memory");
}

template <int POL>
__global__ void __launch_bounds__(256)
scrub_tma_kernel(RegionSplit s /* VB = 16 */, uint32_t tile_bytes, uint32_t ops_per_group, Sched sched) {
  extern __shared__ __align__(128) uint8_t zero_tile[];
  for (uint32_t i = threadIdx.x; i < tile_bytes / 16; i += blockDim.x)
    reinterpret_cast<uint4*>(zero_tile)[i] = make_uint4(0, 0, 0, 0);
  // make the generic-proxy smem writes visible to the async proxy
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();

  uint8_t* body = s.base + s.head;
  const uint64_t body_bytes = s.body_vecs * 16;
  const uint64_t ntiles = sched.ntiles;  // = body_bytes / tile_bytes
  const uint32_t last_bytes = (uint32_t)(body_bytes - ntiles * (uint64_t)tile_bytes);  // multiple of 16

  // each WARP's lane 0 issues; warps take interleaved tiles / their own chunks.
  const uint32_t warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  if ((threadIdx.x & 31) == 0) {
    const uint32_t src = (uint32_t)__cvta_generic_to_shared(zero_tile);
    const uint64_t policy = make_l2_policy<POL>();
    if (sched.counter == nullptr) {
      uint32_t in_group = 0;
      const uint64_t first = (uint64_t)blockIdx.x * nwarps + warp;
      const uint64_t step = (uint64_t)gridDim.x * nwarps;
      for (uint64_t tile = first; tile < ntiles; tile += step) {
        bulk_store<POL>(body + tile * (uint64_t)tile_bytes, src, tile_bytes, policy);
        if (++in_group == ops_per_group) {
          in_group = 0;
          asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        }
      }
    } else {
      const uint64_t nchunks = sched.nchunks;
      unsigned long long c = atomicAdd(sched.counter, 1ull);
      while (c < nchunks) {
        const unsigned long long nxt = atomicAdd(sched.counter, 1ull);
        const uint64_t t0 = c * sched.chunk_tiles;
        const uint64_t t1 = t0 + sched.chunk_tiles < ntiles ? t0 + sched.chunk_tiles : ntiles;
        for (uint64_t tile = t0; tile < t1; ++tile)
          bulk_store<POL>(body + tile * (uint64_t)tile_bytes, src, tile_bytes, policy);
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        c = nxt;
      }
    }
    if (last_bytes && blockIdx.x == 0 && warp == 0)
      bulk_store<kPolDefault>(body + ntiles * (uint64_t)tile_bytes, src, last_bytes, 0);
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
  }
  ZeroOp<16, POL> zero{0};
  ragged_bytes<16>(s, blockDim.x, zero);
}

// ----------------------------------------------------------------- reductions
__device__ __forceinline__ uint64_t warp_sum_u64(uint64_t v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// One atomicAdd(u64) per CTA into the single device counter.
__device__ __forceinline__ void block_accumulate(uint64_t cnt, unsigned long long* counter) {
  __shared__ uint64_t warp_part[32];
  cnt = warp_sum_u64(cnt);
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) warp_part[warp] = cnt;
  __syncthreads();
  if (warp == 0) {
    uint64_t v = lane < ((blockDim.x + 31) >> 5) ? warp_part[lane] : 0;
    v = warp_sum_u64(v);
    if (lane == 0 && v != 0) atomicAdd(counter, (unsigned long long)v);
  }
}

// --------------------------------------------------------------- verify (loads)
// All UNROLL loads are issued before any use (UNROLL*VB bytes in flight per
// thread).  The expected answer is "all zero", so the hot loop only ORs the words
// together; the exact per-byte count runs on the (rare) batches whose OR != 0.
template <int VB, int UNROLL, int POL>
__device__ __forceinline__ uint32_t verify_tile(const uint8_t* body, uint64_t tile, uint64_t tile_vecs, uint32_t idx,
                                                uint64_t stride_bytes, uint64_t l2pol) {
  constexpr int W = VB / 4;
  uint32_t w[UNROLL][W];
#pragma unroll
  for (int u = 0; u < UNROLL; ++u) {
    if constexpr (VB == 32) {  // lane-contiguous halves, as in scrub_tile
      const uint8_t* p = body + tile * tile_vecs * 32 + (uint64_t)idx * 16 + u * stride_bytes;
      const Vec16 a = ld16<POL>(p, l2pol), b = ld16<POL>(p + stride_bytes / 2, l2pol);
#pragma unroll
      for (int k = 0; k < 4; ++k) { w[u][k] = a.w[k]; w[u][4 + k] = b.w[k]; }
    } else {
      const uint8_t* p = body + (tile * tile_vecs + idx) * VB;
      Vec16 v = ld16<POL>(p + u * stride_bytes, l2pol);
#pragma unroll
      for (int k = 0; k < W; ++k) w[u][k] = v.w[k];
    }
  }
  uint32_t any = 0;
#pragma unroll
  for (int u = 0; u < UNROLL; ++u)
#pragma unroll
    for (int k = 0; k < W; ++k) any |= w[u][k];
  uint32_t c = 0;
  if (any != 0) {
#pragma unroll
    for (int u = 0; u < UNROLL; ++u)
#pragma unroll
      for (int k = 0; k < W; ++k) c += nonzero_bytes_in_word(w[u][k]);
  }
  return c;
}

// Counts the non-zero bytes it reads into cnt.  chunk() batches like verify_tile.  The chunk() of every op returns the
// bytes it addressed (the coverage ledger counts them; the plain kernels ignore the value).
template <int VB, int POL>
struct CountNonzeroOp {
  uint64_t l2pol;
  uint64_t cnt = 0;
  template <int THREADS, int PER_THREAD>
  __device__ __forceinline__ uint32_t chunk(const uint8_t* p) {
    Vec16 v[PER_THREAD];
#pragma unroll
    for (int u = 0; u < PER_THREAD; ++u) v[u] = ld16<POL>(p + (uint32_t)u * THREADS * 16u, l2pol);  // all loads first
    uint32_t any = 0;
#pragma unroll
    for (int u = 0; u < PER_THREAD; ++u)
#pragma unroll
      for (int k = 0; k < 4; ++k) any |= v[u].w[k];
    if (any != 0) {  // rare: exact per-byte count of this batch
      uint32_t n = 0;
#pragma unroll
      for (int u = 0; u < PER_THREAD; ++u)
#pragma unroll
        for (int k = 0; k < 4; ++k) n += nonzero_bytes_in_word(v[u].w[k]);
      cnt += n;
    }
    return (uint32_t)PER_THREAD * 16u;
  }
  __device__ __forceinline__ void vec(const uint8_t* p) {
    if constexpr (VB == 32) {
      Vec32 v = ld32<POL>(p, l2pol);
#pragma unroll
      for (int k = 0; k < 8; ++k) cnt += nonzero_bytes_in_word(v.w[k]);
    } else {
      Vec16 v = ld16<POL>(p, l2pol);
#pragma unroll
      for (int k = 0; k < 4; ++k) cnt += nonzero_bytes_in_word(v.w[k]);
    }
  }
  __device__ __forceinline__ void byte(const uint8_t* p) { cnt += (*p != 0); }
};

template <int VB, int UNROLL, int POL>
__global__ void __launch_bounds__(1024)
verify_ld_kernel(RegionSplit s, unsigned long long* counter, Sched sched) {
  const uint8_t* body = s.base + s.head;
  const uint32_t group = sched.per_warp ? 32u : blockDim.x;
  const uint32_t idx = sched.per_warp ? (threadIdx.x & 31u) : threadIdx.x;
  const uint64_t tile_vecs = (uint64_t)group * UNROLL;
  const uint64_t stride_bytes = (uint64_t)group * VB;
  CountNonzeroOp<VB, POL> op{make_l2_policy<POL>()};
  for_each_tile(sched, idx, [&](uint64_t tile) {
    op.cnt += verify_tile<VB, UNROLL, POL>(body, tile, tile_vecs, idx, stride_bytes, op.l2pol);
  });
  finish_region<VB>(s, sched.ntiles * tile_vecs, blockDim.x, op);
  block_accumulate(op.cnt, counter);
}

// DESCENDING chunk order.  The scrub ran in ascending order and left the last L2-sized stretch it
// wrote (up to 50 MB on H100) dirty in L2.  Reading upwards would stream the whole region from DRAM
// and, on top of that, evict those dirty lines (extra write-back traffic); reading downwards takes
// them out of L2 first, so the DRAM traffic of a read-back is R again, not R + L2.
template <int THREADS, int PER_THREAD, int POL>
__global__ void __launch_bounds__(THREADS)
verify_ld128_fast_kernel(RegionSplit s, uint64_t nchunks, GrabCtl ctl, unsigned long long* counter) {
  CountNonzeroOp<16, POL> op{0};
  default_kernel<THREADS, PER_THREAD, true>(s, nchunks, ctl, nullptr, op);
  block_accumulate(op.cnt, counter);
}

// ------------------------------------------------- address-tagged known answer
// A zero read-back cannot tell a byte the scrub zeroed from one that was already zero, or from a
// second virtual view of a byte zeroed elsewhere.  The tagged gate first writes a pattern that only
// this call, at this virtual address, could have produced, and checks it before zeroing.
//
// tag(seed, a) of the 4-byte word at device address a (i = a >> 2):
//     lo32(i) * kTagK1  ^  hi32(i) * kTagK2  ^  seed
// A byte at address x is byte (x & 3) (little-endian) of tag(seed, x & ~3).  Both constants are odd,
// so multiplying by them is a bijection mod 2^32:
//   * within one 16 GiB-aligned window (hi32 fixed) distinct words get distinct tags;
//   * a word and its alias at any non-zero multiple of 16 GiB (lo32 fixed) get distinct tags;
//   * two seeds differ in every word by seed1 ^ seed2.
// oracle/scrub_oracle.py (tag_bytes) restates this formula.
constexpr uint32_t kTagK1 = 0x9E3779B1u;
constexpr uint32_t kTagK2 = 0x85EBCA77u;

__host__ __device__ __forceinline__ uint32_t tag_word(uint32_t seed, uint64_t a) {
  const uint64_t i = a >> 2;
  return ((uint32_t)i * kTagK1) ^ ((uint32_t)(i >> 32) * kTagK2) ^ seed;
}

__host__ __device__ __forceinline__ uint8_t tag_byte(uint32_t seed, uint64_t x) {
  return (uint8_t)(tag_word(seed, x & ~3ull) >> (8 * (x & 3)));
}

// The four words of the 16-byte vector at the 16-aligned address a: one 32-bit multiply per pair of
// constants per vector, then one add and one xor per word (hi32 is the same for all four words).
__device__ __forceinline__ uint4 tag_vec(uint32_t seed, uint64_t a) {
  const uint64_t i = a >> 2;
  const uint32_t b = (uint32_t)i * kTagK1;
  const uint32_t h = ((uint32_t)(i >> 32) * kTagK2) ^ seed;
  return make_uint4(b ^ h, (b + kTagK1) ^ h, (b + 2 * kTagK1) ^ h, (b + 3 * kTagK1) ^ h);
}

__device__ __forceinline__ void st16(void* p, uint4 v) {
  asm volatile("st.global.v4.b32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

// Coherent streaming load: the check kernel writes every address it reads, so the read-only (.nc)
// path of the verifier is not used here.
__device__ __forceinline__ uint4 ld16_cs(const void* p) {
  uint4 v;
  asm volatile("ld.global.cs.v4.b32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
  return v;
}

__device__ __forceinline__ uint64_t addr(const void* p) { return (uint64_t)(uintptr_t)p; }

struct TagFillOp {
  uint32_t seed;
  template <int THREADS, int PER_THREAD>
  __device__ __forceinline__ uint32_t chunk(uint8_t* p) {
#pragma unroll
    for (int u = 0; u < PER_THREAD; ++u) vec(p + (uint32_t)u * THREADS * 16u);
    return (uint32_t)PER_THREAD * 16u;
  }
  __device__ __forceinline__ void vec(uint8_t* q) { st16(q, tag_vec(seed, addr(q))); }
  __device__ __forceinline__ void byte(uint8_t* x) { *x = tag_byte(seed, addr(x)); }
};

// Writes the tags over a region.  Shape and bookkeeping of scrub_st128_fast_kernel: persistent CTAs,
// one THREADS * PER_THREAD * 16-byte chunk per grab, self-resetting GrabCtl, CTA 0 takes the ragged bytes.
template <int THREADS, int PER_THREAD>
__global__ void __launch_bounds__(THREADS)
tag_fill_kernel(RegionSplit s, uint64_t nchunks, GrabCtl ctl, uint32_t seed) {
  TagFillOp op{seed};
  default_kernel<THREADS, PER_THREAD, false>(s, nchunks, ctl, nullptr, op);
}

// Fault drill "tag_inject": flips bits of single bytes (XOR, so the byte can never keep its tag).
__global__ void xor_byte_kernel(uint8_t* p) { *p ^= 0xA5; }

// ---------------------------------------------------------------- window books
// The locate pass, the tag check and the census say WHERE they found what they count, in 16-byte, 16-aligned address
// windows (in the body a window is one vector).  All keep the same book: exact window count and first / last byte in
// registers, one atomic per result word per CTA, and up to kDirtRecords records of (window offset, mask, 16 bytes);
// the census records no bytes (MaskRecord).  Each also counts its booked bytes per 2 MiB page (LocateOut::pages): a
// batch's bytes add up over the active lanes of the warp, one atomic per page per warp per batch, and only in the
// branch that books.
constexpr int kDirtRecords = 64;

struct DirtRecord {       // layout of ccm_dirt_record (include/ccm.h); `chunk` is filled in by the host
  uint64_t offset;        // window address - region base (negative, two's complement, for the head window of a
                          // region that does not start 16-aligned)
  uint32_t chunk;
  uint16_t mask;          // bit i: byte i of the window is booked (locate: non-zero; check: differs from its tag)
  uint16_t reserved;
  uint4 bytes;
};

struct MaskRecord {       // layout of ccm_residue_record (include/ccm.h): a window without its bytes
  uint64_t offset;        // as DirtRecord::offset
  uint32_t chunk;         // filled in by the host
  uint16_t mask;          // bit i: byte i of the window is non-zero
  uint16_t reserved;
};

// The page map: booked bytes per 2 MiB page (the VMM granule: every chunk the product call maps is a whole number of
// pages).  A window belongs to the page of its offset, offset >> kPageShift; the head window of a region that does
// not start 16-aligned, whose offset is negative, belongs to page 0.
constexpr int kPageShift = 21;
constexpr uint32_t kPageBytes = 1u << kPageShift;

// Result words of one pass, each on its own line of the engine's control block; zero before the launch.
struct LocateOut {
  unsigned long long* count;      // += the op's own count: non-zero bytes (locate), all-zero windows (tag check)
  unsigned long long* windows;    // += windows booked
  unsigned long long* first_inv;  // max of ~offset of the first booked byte (0: none)
  unsigned long long* last;       // max of the offset of the last booked byte
  unsigned long long* slots;      // record slots claimed (may run past kDirtRecords)
  unsigned long long* full;       // set once kDirtRecords slots are taken
  DirtRecord* records;
  uint32_t* pages;                // += booked bytes of each page (zero before the launch, like the words)
};

// Bit 7 of each byte of the result is set iff that byte of w is non-zero (as in nonzero_bytes_in_word).
__device__ __forceinline__ uint32_t nonzero_byte_flags(uint32_t w) {
  return (((w & 0x7f7f7f7fu) + 0x7f7f7f7fu) | w) & 0x80808080u;
}

// 16-bit mask of the non-zero bytes of one vector.
__device__ __forceinline__ uint32_t nonzero_mask16(const Vec16& v) {
  uint32_t m = 0;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const uint32_t f = nonzero_byte_flags(v.w[k]);
    m |= (((f >> 7) & 1u) | ((f >> 14) & 2u) | ((f >> 21) & 4u) | ((f >> 28) & 8u)) << (4 * k);
  }
  return m;
}

// Counts, first / last offset and window count stay in registers; only records go through memory.  A record slot
// is claimed with an atomicAdd only while the "records full" word is clear, and a thread that has seen it set (or
// drew the last slot or a later one) never reads it again: a region that is booked everywhere would otherwise
// serialise one atomic per vector on a single address, about 5e9 of them at whole HBM.
struct WindowBook {
  LocateOut out;
  uint64_t count = 0, windows = 0, first_inv = 0, last = 0;   // count: the op's own (out.count)
  bool full_seen = false;

  // A record slot (>= kDirtRecords: none left).
  __device__ __forceinline__ uint64_t claim() {
    if (*(volatile unsigned long long*)out.full) { full_seen = true; return kDirtRecords; }
    const uint64_t slot = atomicAdd(out.slots, 1ull);
    if (slot + 1 >= (uint64_t)kDirtRecords) { *(volatile unsigned long long*)out.full = 1; full_seen = true; }
    return slot;
  }

  // Counts one window at offset `off` whose booked bytes are `mask` (!= 0).
  __device__ __forceinline__ void tally(uint64_t off, uint32_t mask) {
    windows += 1;
    const uint64_t lo = off + (uint64_t)(__ffs(mask) - 1), hi = off + (uint64_t)(31 - __clz(mask));
    first_inv = max(first_inv, (uint64_t)~lo);
    last = max(last, hi);
  }

  // Counts n windows (n may be 0: then nothing changes) whose booked bytes run from off + lo to off + hi, without a
  // branch.
  __device__ __forceinline__ void tally_span(uint64_t off, uint32_t lo, uint32_t hi, uint32_t n) {
    windows += n;
    first_inv = max(first_inv, n ? (uint64_t)~(off + lo) : (uint64_t)0);
    last = max(last, n ? off + hi : (uint64_t)0);
  }

  // Records a window (mask != 0) by offset and mask only, into `recs`, while slots last: for a pass whose bytes must
  // not leave the device.  The window is tallied by the caller.
  __device__ __forceinline__ void record_mask(MaskRecord* recs, uint64_t off, uint32_t mask) {
    if (full_seen) return;
    const uint64_t slot = claim();
    if (slot < (uint64_t)kDirtRecords) recs[slot] = MaskRecord{off, 0u, (uint16_t)mask, (uint16_t)0};
  }

  __device__ __forceinline__ void record(uint64_t slot, uint64_t off, uint32_t mask, const Vec16& v) {
    DirtRecord r;
    r.offset = off;
    r.chunk = 0;
    r.mask = (uint16_t)mask;
    r.reserved = 0;
    r.bytes = make_uint4(v.w[0], v.w[1], v.w[2], v.w[3]);
    out.records[slot] = r;
  }

  // Counts one window (mask != 0) and records it while slots last.
  __device__ __forceinline__ void book(uint64_t off, uint32_t mask, const Vec16& v) {
    tally(off, mask);
    if (full_seen) return;
    const uint64_t slot = claim();
    if (slot < (uint64_t)kDirtRecords) record(slot, off, mask, v);
  }

  __device__ __forceinline__ static uint32_t page_of(uint64_t off) {
    return (int64_t)off < 0 ? 0u : (uint32_t)(off >> kPageShift);
  }

  // Bytes from a chunk's first byte (offset c0, never negative: every caller's base lies at or before its body) to
  // the next page boundary.  A chunk (128 KiB) is shorter than a page, so its vectors lie on c0's page (chunk-relative
  // offset < the room) or the next one.
  __device__ __forceinline__ static uint32_t page_room(uint64_t c0) {
    return kPageBytes - ((uint32_t)c0 & (kPageBytes - 1));
  }

  // Pages of one batch: lo booked bytes on the page of the chunk offset c0, hi on the next (only when the chunk
  // `crosses` a page boundary, which a 2 MiB-aligned body never does; the same for every lane of the chunk).  Every
  // active lane is in the same chunk, so they add up over the active lanes and one lane issues one atomic per non-zero
  // page.
  // (Before sm_80 there is no __reduce_add_sync: every lane adds its own bytes.  The library builds for sm_90a only;
  // the fallback keeps this header compiling for any architecture.)
  __device__ __forceinline__ void pages_batch(uint64_t c0, uint32_t lo, uint32_t hi, bool crosses) {
#if defined(__CUDA_ARCH__) && __CUDA_ARCH__ < 800
    if (lo) atomicAdd(out.pages + page_of(c0), lo);
    if (crosses && hi) atomicAdd(out.pages + page_of(c0) + 1, hi);
#else
    const uint32_t active = __activemask();
    lo = __reduce_add_sync(active, lo);
    if (crosses) hi = __reduce_add_sync(active, hi);
    if ((threadIdx.x & 31u) == (uint32_t)(__ffs(active) - 1)) {
      const uint32_t page = page_of(c0);
      if (lo) atomicAdd(out.pages + page, lo);
      if (crosses && hi) atomicAdd(out.pages + page + 1, hi);
    }
#endif
  }

  // Pages of one window outside the batches (a leftover vector, a ragged window) with `bytes` != 0 booked: the active
  // lanes that book into one page add up, and one of them issues the atomic.
  __device__ __forceinline__ void pages_window(uint64_t off, uint32_t bytes) {
#if defined(__CUDA_ARCH__) && __CUDA_ARCH__ < 800
    atomicAdd(out.pages + page_of(off), bytes);
#else
    const uint32_t active = __activemask();
    const uint32_t page = page_of(off);
    const uint32_t peers = __match_any_sync(active, page);
    bytes = __reduce_add_sync(peers, bytes);
    if ((threadIdx.x & 31u) == (uint32_t)(__ffs(peers) - 1)) atomicAdd(out.pages + page, bytes);
#endif
  }

  // One atomic per result word per CTA (skipped when the CTA booked nothing), after a block reduction.
  __device__ __forceinline__ void flush() {
    __shared__ uint64_t part[4][32];
    uint64_t a = count, b = windows, c = first_inv, d = last;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      a += __shfl_xor_sync(0xffffffffu, a, o);
      b += __shfl_xor_sync(0xffffffffu, b, o);
      c = max(c, __shfl_xor_sync(0xffffffffu, c, o));
      d = max(d, __shfl_xor_sync(0xffffffffu, d, o));
    }
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) { part[0][warp] = a; part[1][warp] = b; part[2][warp] = c; part[3][warp] = d; }
    __syncthreads();
    if (warp == 0) {
      const bool in = lane < ((blockDim.x + 31) >> 5);
      a = in ? part[0][lane] : 0;
      b = in ? part[1][lane] : 0;
      c = in ? part[2][lane] : 0;
      d = in ? part[3][lane] : 0;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        a += __shfl_xor_sync(0xffffffffu, a, o);
        b += __shfl_xor_sync(0xffffffffu, b, o);
        c = max(c, __shfl_xor_sync(0xffffffffu, c, o));
        d = max(d, __shfl_xor_sync(0xffffffffu, d, o));
      }
      if (lane == 0 && b != 0) {
        atomicAdd(out.count, (unsigned long long)a);
        atomicAdd(out.windows, (unsigned long long)b);
        atomicMax(out.first_inv, (unsigned long long)c);
        atomicMax(out.last, (unsigned long long)d);
      }
    }
  }
};

// CTA 0, one thread per window of the ragged head and tail: false for every other thread, otherwise true with the
// window's address w0 and the part [lo, hi) of it that lies inside the region.
__device__ __forceinline__ bool ragged_window(const RegionSplit& s, uint64_t& w0, uint64_t& lo, uint64_t& hi) {
  if (blockIdx.x != 0) return false;
  const uint64_t a0 = addr(s.base);
  const uint64_t head_end = a0 + s.head, tail_start = head_end + s.body_vecs * 16, end = tail_start + s.tail;
  const uint64_t first_win = a0 & ~15ull;
  const uint64_t nhead = s.head ? (head_end - first_win + 15) / 16 : 0;   // at most 8
  const uint64_t t = threadIdx.x;
  if (t < nhead) { w0 = first_win + 16 * t; lo = max(w0, a0); hi = min(w0 + 16, head_end); return true; }
  if (t == nhead && s.tail) { w0 = tail_start; lo = tail_start; hi = end; return true; }
  return false;
}

// Counts the bytes that differ from the tags into cnt and stores zero over them.
// The exact per-byte count is computed for every batch, branch-free, and the loaded words die before the
// stores: on H100 this runs at 0.97x of a same-run device-to-device copy, where counting only batches whose
// XOR is non-zero (verify_ld128_fast_kernel's trick) keeps the loaded words live across the stores and
// runs at 0.75x (one H100 80GB HBM3, 700 W, 32 GiB region).
//
// Where the mismatches are: only a batch whose exact count is non-zero takes the rare branch, and it sits BEFORE
// the stores, so the loaded words still die there.  It books every window of the batch that differs from its
// tags (WindowBook: mask = the bytes that differ, the 16 bytes as read) and counts the booked windows whose bytes
// inside the region all read 0 into book.count.  Offsets are addresses - `base`, so every launch of one call
// books into the same words.  The ragged head and tail are not taken byte by byte (byte() does nothing):
// tag_check_zero_kernel takes them window by window, so no window is counted or recorded twice.
struct TagCheckZeroOp {
  uint32_t seed;
  WindowBook book;
  uint64_t base;
  uint64_t cnt = 0;

  // One window given as what was read (bytes outside the region as 0) and its mask of bytes that differ.
  __device__ __forceinline__ void window(uint64_t off, uint32_t mask, const Vec16& v) {
    if (mask == 0) return;
    book.count += (v.w[0] | v.w[1] | v.w[2] | v.w[3]) == 0;
    book.book(off, mask, v);
  }

  // A window outside the batches: booked, and its bytes added to its page.
  __device__ __forceinline__ void single(uint64_t off, uint32_t mask, const Vec16& v) {
    if (mask == 0) return;
    window(off, mask, v);
    book.pages_window(off, __popc(mask));
  }

  __device__ __forceinline__ static uint32_t diff_mask(const uint4& v, const uint4& t) {
    const Vec16 x = {{v.x ^ t.x, v.y ^ t.y, v.z ^ t.z, v.w ^ t.w}};
    return nonzero_mask16(x);
  }

  template <int THREADS, int PER_THREAD>
  __device__ __forceinline__ uint32_t chunk(uint8_t* p) {
    uint4 v[PER_THREAD];
#pragma unroll
    for (int u = 0; u < PER_THREAD; ++u) v[u] = ld16_cs(p + (uint32_t)u * THREADS * 16u);  // all loads first
    uint32_t n = 0;
#pragma unroll
    for (int u = 0; u < PER_THREAD; ++u) {
      const uint4 t = tag_vec(seed, addr(p + (uint32_t)u * THREADS * 16u));
      n += nonzero_bytes_in_word(v[u].x ^ t.x) + nonzero_bytes_in_word(v[u].y ^ t.y) +
           nonzero_bytes_in_word(v[u].z ^ t.z) + nonzero_bytes_in_word(v[u].w ^ t.w);
    }
    if (n != 0) {  // rare except in a flood: book the batch's windows, before the stores
      // The branch reads the batch's vectors again, four at a time: they come from L2 (this thread loaded them a
      // moment ago) and nothing has stored over them yet.  Keeping the loaded words live into the branch instead
      // would need more registers than a 512-thread CTA leaves a thread (128: ptxas spills).  Unless something
      // else writes the range during the check (two views of one range checked in one launch), the branch reads
      // exactly the bytes counted above.
      const uint64_t off0 = addr(p) - base;
      const uint32_t room = WindowBook::page_room(off0 - threadIdx.x * 16u);
      const bool crosses = room < (uint32_t)THREADS * PER_THREAD * 16u;
      uint32_t hi = 0;   // bytes on the page after the chunk's first (n - hi on its own)
#pragma unroll 4
      for (uint32_t u = 0; u < (uint32_t)PER_THREAD; ++u) {
        uint8_t* q = p + u * THREADS * 16u;
        const uint4 x = ld16_cs(q);
        const uint32_t mask = diff_mask(x, tag_vec(seed, addr(q)));
        window(off0 + u * THREADS * 16u, mask, Vec16{{x.x, x.y, x.z, x.w}});
        if (crosses) hi += threadIdx.x * 16u + u * THREADS * 16u >= room ? __popc(mask) : 0u;
      }
      // The pages add up to n, the count the verdict takes, also when a second view changed the batch in between.
      hi = min(hi, n);
      book.pages_batch(off0 - threadIdx.x * 16u, n - hi, hi, crosses);
    }
#pragma unroll
    for (int u = 0; u < PER_THREAD; ++u) st16(p + (uint32_t)u * THREADS * 16u, make_uint4(0, 0, 0, 0));
    cnt += n;
    return (uint32_t)PER_THREAD * 16u;
  }
  __device__ __forceinline__ void vec(uint8_t* q) {
    uint4 v = ld16_cs(q);
    const uint32_t mask = diff_mask(v, tag_vec(seed, addr(q)));
    single(addr(q) - base, mask, Vec16{{v.x, v.y, v.z, v.w}});
    st16(q, make_uint4(0, 0, 0, 0));
    cnt += __popc(mask);
  }
  __device__ __forceinline__ void byte(uint8_t*) {}

  // CTA 0: the windows of the ragged head and tail, one thread per window.  Only bytes inside the region are
  // compared and zeroed; the others count as 0 that holds its tag.
  __device__ __forceinline__ void ragged_windows(const RegionSplit& s) {
    uint64_t w0 = 0, lo = 0, hi = 0;
    if (!ragged_window(s, w0, lo, hi)) return;
    Vec16 v = {{0, 0, 0, 0}}, x = {{0, 0, 0, 0}};
#pragma unroll
    for (int i = 0; i < 16; ++i)
      if (w0 + i >= lo && w0 + i < hi) {
        uint8_t* b = (uint8_t*)(uintptr_t)(w0 + i);
        const uint32_t got = *b;
        v.w[i >> 2] |= got << (8 * (i & 3));
        x.w[i >> 2] |= (uint32_t)(uint8_t)(got ^ tag_byte(seed, w0 + i)) << (8 * (i & 3));
        *b = 0;
      }
    const uint32_t mask = nonzero_mask16(x);
    single(w0 - base, mask, v);
    cnt += __popc(mask);
  }
};

// Reads the tags back, counts every byte that differs from them (exact, u64, one atomic per CTA into
// *mismatch) and stores zero over the same addresses.  All PER_THREAD loads are in flight before any use.
// Chunks are taken in ascending order, so the last stretch this kernel writes is the first one the
// descending zero read-back reads.  The windows that differ are booked into `out` with offsets from `base`
// (TagCheckZeroOp); a check that finds nothing writes none of those words.
template <int THREADS, int PER_THREAD>
__global__ void __launch_bounds__(THREADS)
tag_check_zero_kernel(RegionSplit s, uint64_t nchunks, GrabCtl ctl, uint32_t seed, unsigned long long* mismatch,
                      LocateOut out, uint64_t base) {
  TagCheckZeroOp op{seed, {out}, base};
  default_kernel<THREADS, PER_THREAD, false>(s, nchunks, ctl, nullptr, op);
  op.ragged_windows(s);
  op.book.flush();
  block_accumulate(op.cnt, mismatch);
}

// ------------------------------------------------------------ locate the dirt
// When the zero read-back counted dirt, this pass says where it is.  A dirty WINDOW holds at least one non-zero
// byte of the region.  Results: the exact number of non-zero bytes (book.count) and of dirty windows, the offsets
// (from the region base) of the first and the last non-zero byte, and up to kDirtRecords records of (window offset,
// mask of its non-zero bytes, its 16 bytes).  The ragged head and tail are not taken byte by byte (byte() does
// nothing): locate_dirt_kernel takes them window by window, so no window is counted or recorded twice.
struct LocateOp {
  WindowBook book;
  uint64_t base;

  template <int THREADS, int PER_THREAD>
  __device__ __forceinline__ uint32_t chunk(const uint8_t* p) {
    Vec16 v[PER_THREAD];
#pragma unroll
    for (int u = 0; u < PER_THREAD; ++u) v[u] = ld16<kPolStreaming>(p + (uint32_t)u * THREADS * 16u, 0);  // all loads first
    uint32_t any = 0;
#pragma unroll
    for (int u = 0; u < PER_THREAD; ++u)
#pragma unroll
      for (int k = 0; k < 4; ++k) any |= v[u].w[k];
    if (any != 0) {  // rare except in a flood
      const uint64_t off0 = addr(p) - base;
      uint32_t n = 0;
#pragma unroll
      for (int u = 0; u < PER_THREAD; ++u) {
        const uint32_t mask = nonzero_mask16(v[u]);
        window(off0 + (uint32_t)u * THREADS * 16u, mask, v[u]);
        n += __popc(mask);
      }
      // the pages: the bytes past the page boundary inside the chunk, if there is one, go on the next page
      const uint32_t room = WindowBook::page_room(off0 - threadIdx.x * 16u);
      const bool crosses = room < (uint32_t)THREADS * PER_THREAD * 16u;
      uint32_t hi = 0;
      if (crosses) {
#pragma unroll
        for (int u = 0; u < PER_THREAD; ++u)
          hi += threadIdx.x * 16u + (uint32_t)u * THREADS * 16u >= room ? __popc(nonzero_mask16(v[u])) : 0u;
      }
      book.pages_batch(off0 - threadIdx.x * 16u, n - hi, hi, crosses);
    }
    return (uint32_t)PER_THREAD * 16u;
  }

  // One window given as its aligned vector (a body vector, or a head / tail window from ragged_windows).
  __device__ __forceinline__ void window(uint64_t off, uint32_t mask, const Vec16& v) {
    if (mask == 0) return;
    book.count += __popc(mask);
    book.book(off, mask, v);
  }

  // A window outside the batches: booked, and its bytes added to its page.
  __device__ __forceinline__ void single(uint64_t off, uint32_t mask, const Vec16& v) {
    if (mask == 0) return;
    window(off, mask, v);
    book.pages_window(off, __popc(mask));
  }

  __device__ __forceinline__ void vec(const uint8_t* p) {
    const Vec16 v = ld16<kPolStreaming>(p, 0);
    single(addr(p) - base, nonzero_mask16(v), v);
  }

  __device__ __forceinline__ void byte(const uint8_t*) {}

  // CTA 0: the windows of the ragged head and tail, one thread per window, bytes outside the region as 0.
  __device__ __forceinline__ void ragged_windows(const RegionSplit& s) {
    uint64_t w0 = 0, lo = 0, hi = 0;
    if (!ragged_window(s, w0, lo, hi)) return;
    Vec16 v = {{0, 0, 0, 0}};
#pragma unroll
    for (int i = 0; i < 16; ++i)
      if (w0 + i >= lo && w0 + i < hi) v.w[i >> 2] |= (uint32_t)*(const uint8_t*)(uintptr_t)(w0 + i) << (8 * (i & 3));
    single(w0 - base, nonzero_mask16(v), v);
  }
};

// Reads the region (writes nothing into it) and reports where its non-zero bytes are.  Frame, loads and batching of
// verify_ld128_fast_kernel: persistent CTAs, one THREADS * PER_THREAD * 16-byte chunk per grab in ascending order, all
// PER_THREAD loads in flight, then OR; only batches whose OR is non-zero do more work.  Minimum one CTA per SM in the
// launch bounds: the compiler may then use the registers the flood path needs instead of spilling it.  Offsets are
// addresses - `base` (as the tag check's), so every launch of one call books into the same words and page map.
template <int THREADS, int PER_THREAD>
__global__ void __launch_bounds__(THREADS, 1)
locate_dirt_kernel(RegionSplit s, uint64_t nchunks, GrabCtl ctl, LocateOut out, uint64_t base) {
  LocateOp op{{out}, base};
  default_kernel<THREADS, PER_THREAD, false>(s, nchunks, ctl, nullptr, op);
  op.ragged_windows(s);
  op.book.flush();
}

// ------------------------------------------------------- census of what the gate erases
// The first pass of a census call reads every vector before it writes it, and books what was there: the exact
// number of non-zero bytes (book.count) and of non-zero windows, the first and last non-zero byte, and up to
// kDirtRecords records of (window offset, mask of its non-zero bytes).  What it reads is the previous tenant's data,
// so no byte of it is recorded: only counts, offsets and masks leave the registers.
//
// Residue may be everywhere (memory nobody cleared), so the dense case must stay cheap: each vector's mask is
// computed while its words are live, the window is tallied branch-free, and the only branch claims a record slot
// while the book is not full.  The loaded words die before the stores.  Then it stores zero, or (TAGS) the tags of
// `seed`, over the same addresses.  Offsets are addresses - `base`, so every launch of one call books into the
// same words.  The ragged head and tail are taken window by window by CTA 0 (byte() does nothing).
template <bool TAGS>
struct CensusOp {
  uint32_t seed;
  WindowBook book;
  MaskRecord* records;
  uint64_t base;

  __device__ __forceinline__ void store(uint8_t* q) {
    if constexpr (TAGS) st16(q, tag_vec(seed, addr(q)));
    else st16(q, make_uint4(0, 0, 0, 0));
  }

  // One window outside the batches (a leftover vector, a ragged window).
  __device__ __forceinline__ void window(uint64_t off, uint32_t mask) {
    if (mask == 0) return;
    book.count += __popc(mask);
    book.tally(off, mask);
    book.record_mask(records, off, mask);
    book.pages_window(off, __popc(mask));
  }

  // The batch's tally runs on offsets relative to its first vector (< 2^32), and the branch that claims record slots
  // depends on every mask: all PER_THREAD loads are in flight before the first branch.
  template <int THREADS, int PER_THREAD>
  __device__ __forceinline__ uint32_t chunk(uint8_t* p) {
    constexpr uint32_t kStride = THREADS * 16u;
    uint32_t mask[PER_THREAD];
    {
      uint4 v[PER_THREAD];
#pragma unroll
      for (int u = 0; u < PER_THREAD; ++u) v[u] = ld16_cs(p + (uint32_t)u * kStride);  // all loads first
#pragma unroll
      for (int u = 0; u < PER_THREAD; ++u) mask[u] = nonzero_mask16(Vec16{{v[u].x, v[u].y, v[u].z, v[u].w}});
    }
    uint32_t any = 0, n = 0, nwin = 0, lo = 0xFFFFFFFFu, hi = 0;
#pragma unroll
    for (int u = 0; u < PER_THREAD; ++u) {
      const uint32_t m = mask[u], at = (uint32_t)u * kStride;
      any |= m;
      n += __popc(m);
      nwin += m != 0;
      lo = min(lo, m ? at + (uint32_t)(__ffs(m) - 1) : 0xFFFFFFFFu);
      hi = max(hi, m ? at + (uint32_t)(31 - __clz(m)) : 0u);
    }
    const uint64_t off0 = addr(p) - base;
    book.count += n;
    book.tally_span(off0, lo, hi, nwin);
    if (n != 0) {   // the pages: bytes on the chunk's first page and (past a boundary inside the chunk) on the next
      const uint32_t room = WindowBook::page_room(off0 - threadIdx.x * 16u);
      const bool crosses = room < (uint32_t)PER_THREAD * kStride;
      uint32_t up = 0;
      if (crosses) {
#pragma unroll
        for (int u = 0; u < PER_THREAD; ++u) up += threadIdx.x * 16u + (uint32_t)u * kStride >= room ? __popc(mask[u]) : 0u;
      }
      book.pages_batch(off0 - threadIdx.x * 16u, n - up, up, crosses);
    }
    if (any != 0 && !book.full_seen) {  // only until the book is full, however dense the residue
#pragma unroll
      for (int u = 0; u < PER_THREAD; ++u)
        if (mask[u] != 0) book.record_mask(records, off0 + (uint32_t)u * kStride, mask[u]);
    }
#pragma unroll
    for (int u = 0; u < PER_THREAD; ++u) store(p + (uint32_t)u * kStride);
    return (uint32_t)PER_THREAD * 16u;
  }

  __device__ __forceinline__ void vec(uint8_t* q) {
    const uint4 v = ld16_cs(q);
    window(addr(q) - base, nonzero_mask16(Vec16{{v.x, v.y, v.z, v.w}}));
    store(q);
  }

  __device__ __forceinline__ void byte(uint8_t*) {}

  // CTA 0: the windows of the ragged head and tail, one thread per window.  Only bytes inside the region are read
  // and written; the others count as 0.
  __device__ __forceinline__ void ragged_windows(const RegionSplit& s) {
    uint64_t w0 = 0, lo = 0, hi = 0;
    if (!ragged_window(s, w0, lo, hi)) return;
    uint32_t mask = 0;
#pragma unroll
    for (int i = 0; i < 16; ++i)
      if (w0 + i >= lo && w0 + i < hi) {
        uint8_t* b = (uint8_t*)(uintptr_t)(w0 + i);
        mask |= (uint32_t)(*b != 0) << i;
        *b = TAGS ? tag_byte(seed, w0 + i) : (uint8_t)0;
      }
    window(w0 - base, mask);
  }
};

// The zero gate's first pass with a census: books what each vector held (CensusOp), then zeroes it.  Frame of
// scrub_st128_fast_kernel: persistent CTAs, one THREADS * PER_THREAD * 16-byte chunk per grab in ascending order,
// self-resetting GrabCtl.  A census that finds nothing writes none of `out`'s words.  Minimum one CTA per SM in the
// launch bounds, as locate_dirt_kernel: ptxas then keeps more of the batch's loads in flight before the first mask.
template <int THREADS, int PER_THREAD>
__global__ void __launch_bounds__(THREADS, 1)
census_zero_kernel(RegionSplit s, uint64_t nchunks, GrabCtl ctl, LocateOut out, MaskRecord* records, uint64_t base) {
  CensusOp<false> op{0, {out}, records, base};
  default_kernel<THREADS, PER_THREAD, false>(s, nchunks, ctl, nullptr, op);
  op.ragged_windows(s);
  op.book.flush();
}

// The tagged gate's fill with a census: books what each vector held, then writes the tags of `seed` (tag_fill_kernel).
template <int THREADS, int PER_THREAD>
__global__ void __launch_bounds__(THREADS, 1)
census_tag_fill_kernel(RegionSplit s, uint64_t nchunks, GrabCtl ctl, uint32_t seed, LocateOut out, MaskRecord* records,
                       uint64_t base) {
  CensusOp<true> op{seed, {out}, records, base};
  default_kernel<THREADS, PER_THREAD, false>(s, nchunks, ctl, nullptr, op);
  op.ragged_windows(s);
  op.book.flush();
}

// ------------------------------------------------------------ coverage proof
// A read-back that reads nothing returns what a read-back of clean memory returns, so a pass that skipped part of its
// range cannot be told from one that walked it by its result.  The proving twins below run the same op on the same
// frame (default_kernel: shape, grab words, PDL, loads and stores) and count, on the device, the bytes each of them
// processed on every 2 MiB page of the mapping: the host compares the counts against the mapping itself.
//
// The cover map of one pass: u32 words, one per page of offset (address - base) >> kPageShift, and a last word, the
// "outside" slot, for any byte whose page would lie past it (or before base).  Zero before and after every call.
//
// The ledger of a product call's pass (nullptr: none) counts the same bytes per 128 KiB slot, (address - base) >> 17,
// lane by lane: every thread adds the bytes its own op call addressed.  A page map adds a whole chunk for thread 0, so
// it cannot see a chunk walked twice and another on the same page skipped, or a thread that dropped its share; the
// ledger can.  128 KiB is the chunk of every default-frame pass.
constexpr int kSlotShift = 17;
constexpr uint32_t kSlotBytes = 1u << kSlotShift;

struct CoverOut {
  uint32_t* map;
  uint64_t base;     // address of the map's page 0
  uint32_t outside;  // index of the outside slot (the map's last word)
  uint32_t ledger_outside;   // index of the ledger's outside slot (its last word)
  uint32_t* ledger;          // nullptr: no ledger
  uint64_t drop;     // drill "cover_lane_drop": the first vector of the one thread share chunk() skips (0: none)
};

__device__ __forceinline__ uint32_t cover_word(const CoverOut& c, uint64_t a) {
  const uint64_t off = a - c.base;
  if ((int64_t)off < 0) return c.outside;
  const uint64_t page = off >> kPageShift;
  return page < c.outside ? (uint32_t)page : c.outside;
}

// n bytes (n <= kPageBytes) from address a, by one thread: split at a page boundary, as the page maps split a chunk.
__device__ __forceinline__ void cover_add(const CoverOut& c, uint64_t a, uint32_t n) {
  const uint32_t room = kPageBytes - (uint32_t)((a - c.base) & (kPageBytes - 1));
  const uint32_t lo = n < room ? n : room;
  atomicAdd(c.map + cover_word(c, a), lo);
  if (n > lo) atomicAdd(c.map + cover_word(c, a + lo), n - lo);
}

// n bytes (n <= 32) from address a, by every active lane: the lanes whose bytes start on one page add up and one of
// them issues the atomic; the rare bytes past a page boundary go one atomic per lane.
__device__ __forceinline__ void cover_lanes(const CoverOut& c, uint64_t a, uint32_t n) {
  const uint32_t room = kPageBytes - (uint32_t)((a - c.base) & (kPageBytes - 1));
  const uint32_t lo = n < room ? n : room;
  const uint32_t w = cover_word(c, a);
#if defined(__CUDA_ARCH__) && __CUDA_ARCH__ < 800
  atomicAdd(c.map + w, lo);
#else
  const uint32_t peers = __match_any_sync(__activemask(), w);
  const uint32_t sum = __reduce_add_sync(peers, lo);
  if ((threadIdx.x & 31u) == (uint32_t)(__ffs(peers) - 1)) atomicAdd(c.map + w, sum);
#endif
  if (n > lo) atomicAdd(c.map + cover_word(c, a + lo), n - lo);
}

__device__ __forceinline__ uint32_t ledger_word(const CoverOut& c, uint64_t a) {
  const uint64_t off = a - c.base;
  if ((int64_t)off < 0) return c.ledger_outside;
  const uint64_t slot = off >> kSlotShift;
  return slot < c.ledger_outside ? (uint32_t)slot : c.ledger_outside;
}

// `bytes` of every active lane into ledger word w: the lanes with the same word add up, and one of them issues the atomic.
__device__ __forceinline__ void ledger_sum(const CoverOut& c, uint32_t w, uint32_t bytes) {
#if defined(__CUDA_ARCH__) && __CUDA_ARCH__ < 800
  if (bytes) atomicAdd(c.ledger + w, bytes);
#else
  const uint32_t same = __match_any_sync(__activemask(), w);
  const uint32_t total = __reduce_add_sync(same, bytes);
  if ((threadIdx.x & 31u) == (uint32_t)(__ffs(same) - 1) && total) atomicAdd(c.ledger + w, total);
#endif
}

// n bytes (n <= 32) from address a, by every active lane, split at a slot boundary (as cover_lanes splits at a page).
__device__ __forceinline__ void ledger_lanes(const CoverOut& c, uint64_t a, uint32_t n) {
  const uint32_t room = kSlotBytes - (uint32_t)((a - c.base) & (kSlotBytes - 1));
  const uint32_t near = n < room ? n : room;
  ledger_sum(c, ledger_word(c, a), near);
  if (n > near) atomicAdd(c.ledger + ledger_word(c, a + near), n - near);
}

// The n bytes one lane's chunk() addressed: its vectors at a + u * STRIDE, where a lies lane_off bytes into the chunk.
// The vectors before the chunk's first slot boundary count on the chunk's slot, the others on the next one (a chunk
// crosses a boundary only where a range does not start on one).
template <uint32_t STRIDE>
__device__ __forceinline__ void ledger_chunk(const CoverOut& c, uint64_t a, uint32_t lane_off, uint32_t n) {
  const uint64_t c0 = a - lane_off;
  const uint32_t room = kSlotBytes - (uint32_t)((c0 - c.base) & (kSlotBytes - 1));
  const uint32_t before = room > lane_off ? (room - lane_off + STRIDE - 1) / STRIDE * 16u : 0u;
  const uint32_t lo = n < before ? n : before;
  ledger_sum(c, ledger_word(c, c0), lo);
  if (n > lo) atomicAdd(c.ledger + ledger_word(c, c0 + room), n - lo);
}

// The op of a proving kernel: `op` does the work, and what it did is counted into `cover` after it, in program order.
// A chunk by thread 0 (its p is the chunk's first byte) once the CTA's chunk body is issued; leftover vectors and ragged
// bytes by every lane that takes one.  BYTES = false for the window ops, whose byte() does nothing: their kernels take
// the ragged head and tail window by window, and count them there (cover_ragged_windows).  With a ledger, every thread
// also adds what its own op call addressed: chunk() returns that count, and the "cover_lane_drop" drill makes the
// thread whose share starts at cover.drop skip its call (and count 0).
template <typename Op, bool BYTES = true>
struct CoverOp {
  Op& op;
  CoverOut cover;
  template <int THREADS, int PER_THREAD, typename P>
  __device__ __forceinline__ void chunk(P p) {
    uint32_t n = 0;
    if (addr(p) != cover.drop) n = op.template chunk<THREADS, PER_THREAD>(p);
    if (threadIdx.x == 0) cover_add(cover, addr(p), (uint32_t)THREADS * PER_THREAD * 16u);
    if (cover.ledger) ledger_chunk<(uint32_t)THREADS * 16u>(cover, addr(p), threadIdx.x * 16u, n);
  }
  template <typename P>
  __device__ __forceinline__ void vec(P p) {
    op.vec(p);
    cover_lanes(cover, addr(p), 16u);
    if (cover.ledger) ledger_lanes(cover, addr(p), 16u);
  }
  template <typename P>
  __device__ __forceinline__ void byte(P p) {
    op.byte(p);
    if constexpr (BYTES) cover_lanes(cover, addr(p), 1u);
    if constexpr (BYTES) if (cover.ledger) ledger_lanes(cover, addr(p), 1u);
  }
};

// The ragged head and tail windows the window ops (tag check, census) take after the frame: the part inside the region.
__device__ __forceinline__ void cover_ragged_windows(const RegionSplit& s, const CoverOut& c) {
  uint64_t w0 = 0, lo = 0, hi = 0;
  if (ragged_window(s, w0, lo, hi) && hi > lo) cover_lanes(c, lo, (uint32_t)(hi - lo));
  if (c.ledger && ragged_window(s, w0, lo, hi) && hi > lo) ledger_lanes(c, lo, (uint32_t)(hi - lo));
}

// Proving twin of scrub_st128_fast_kernel.
template <int THREADS, int PER_THREAD, int POL>
__global__ void __launch_bounds__(THREADS)
cover_zero_pass(RegionSplit s, uint64_t nchunks, GrabCtl ctl, unsigned long long* zero_on_exit, CoverOut cover) {
  ZeroOp<16, POL> op{0};
  CoverOp<ZeroOp<16, POL>> cop{op, cover};
  default_kernel<THREADS, PER_THREAD, false>(s, nchunks, ctl, zero_on_exit, cop);
}

// Proving twin of verify_ld128_fast_kernel (descending).
template <int THREADS, int PER_THREAD, int POL>
__global__ void __launch_bounds__(THREADS)
cover_read_pass(RegionSplit s, uint64_t nchunks, GrabCtl ctl, unsigned long long* counter, CoverOut cover) {
  CountNonzeroOp<16, POL> op{0};
  CoverOp<CountNonzeroOp<16, POL>> cop{op, cover};
  default_kernel<THREADS, PER_THREAD, true>(s, nchunks, ctl, nullptr, cop);
  block_accumulate(op.cnt, counter);
}

// Proving twin of tag_fill_kernel.
template <int THREADS, int PER_THREAD>
__global__ void __launch_bounds__(THREADS)
cover_tag_fill_pass(RegionSplit s, uint64_t nchunks, GrabCtl ctl, uint32_t seed, CoverOut cover) {
  TagFillOp op{seed};
  CoverOp<TagFillOp> cop{op, cover};
  default_kernel<THREADS, PER_THREAD, false>(s, nchunks, ctl, nullptr, cop);
}

// Proving twin of tag_check_zero_kernel.
template <int THREADS, int PER_THREAD>
__global__ void __launch_bounds__(THREADS)
cover_tag_check_pass(RegionSplit s, uint64_t nchunks, GrabCtl ctl, uint32_t seed, unsigned long long* mismatch,
                       LocateOut out, uint64_t base, CoverOut cover) {
  TagCheckZeroOp op{seed, {out}, base};
  CoverOp<TagCheckZeroOp, false> cop{op, cover};
  default_kernel<THREADS, PER_THREAD, false>(s, nchunks, ctl, nullptr, cop);
  op.ragged_windows(s);
  cover_ragged_windows(s, cover);
  op.book.flush();
  block_accumulate(op.cnt, mismatch);
}

// Proving twins of census_zero_kernel and census_tag_fill_kernel.
template <int THREADS, int PER_THREAD>
__global__ void __launch_bounds__(THREADS, 1)
cover_census_zero_pass(RegionSplit s, uint64_t nchunks, GrabCtl ctl, LocateOut out, MaskRecord* records,
                         uint64_t base, CoverOut cover) {
  CensusOp<false> op{0, {out}, records, base};
  CoverOp<CensusOp<false>, false> cop{op, cover};
  default_kernel<THREADS, PER_THREAD, false>(s, nchunks, ctl, nullptr, cop);
  op.ragged_windows(s);
  cover_ragged_windows(s, cover);
  op.book.flush();
}

template <int THREADS, int PER_THREAD>
__global__ void __launch_bounds__(THREADS, 1)
cover_census_tag_pass(RegionSplit s, uint64_t nchunks, GrabCtl ctl, uint32_t seed, LocateOut out,
                        MaskRecord* records, uint64_t base, CoverOut cover) {
  CensusOp<true> op{seed, {out}, records, base};
  CoverOp<CensusOp<true>, false> cop{op, cover};
  default_kernel<THREADS, PER_THREAD, false>(s, nchunks, ctl, nullptr, cop);
  op.ragged_windows(s);
  cover_ragged_windows(s, cover);
  op.book.flush();
}

// Proving twin of locate_dirt_kernel: the locate pass and the triages' re-reads of a proven call that failed.
template <int THREADS, int PER_THREAD>
__global__ void __launch_bounds__(THREADS, 1)
cover_locate_pass(RegionSplit s, uint64_t nchunks, GrabCtl ctl, LocateOut out, uint64_t base, CoverOut cover) {
  LocateOp op{{out}, base};
  CoverOp<LocateOp, false> cop{op, cover};
  default_kernel<THREADS, PER_THREAD, false>(s, nchunks, ctl, nullptr, cop);
  op.ragged_windows(s);
  cover_ragged_windows(s, cover);
  op.book.flush();
}

// ------------------------------------------------------------ alias probe
// Two virtual views of one physical page both read back zero, so the zero gate cannot see them.  An alias is a
// page-table event, so one known-answer window per 4 KiB page (the smallest page the MMU maps) is enough to catch it:
// the later view's tags overwrite the earlier view's tags in the shared page.  A probe WINDOW is the 32-byte sector at
// a 4096-aligned address; its position depends only on the address modulo 4096, so two views of one physical page
// probe the same sector.  One launch covers the windows w0 + i * kProbeStride, i < nwin, of one mapped chunk (the host
// computes w0, the chunk's first window, and nwin).
constexpr uint64_t kProbeStride = 4096;
constexpr uint32_t kProbeWindow = 32;

// Batches of THREADS * PER windows, window i of a batch on lane i % THREADS, PER windows in flight per thread; the
// windows after the last whole batch one per thread.  op.batch<K>(a, step) takes the K windows a, a + step, ...
template <int THREADS, int PER, typename Op>
__device__ __forceinline__ void probe_windows(uint64_t w0, uint64_t nwin, Op& op) {
  constexpr uint64_t kBatch = (uint64_t)THREADS * PER;
  const uint64_t nbatch = nwin / kBatch;
  for (uint64_t b = blockIdx.x; b < nbatch; b += gridDim.x)
    op.template batch<PER>(w0 + (b * kBatch + threadIdx.x) * kProbeStride, (uint64_t)THREADS * kProbeStride);
  for (uint64_t i = nbatch * kBatch + (uint64_t)blockIdx.x * THREADS + threadIdx.x; i < nwin;
       i += (uint64_t)gridDim.x * THREADS)
    op.template batch<1>(w0 + i * kProbeStride, 0);
}

// P1: the tags of `seed` into every window (two 16-byte stores).
struct ProbeFillOp {
  uint32_t seed;
  template <int K>
  __device__ __forceinline__ void batch(uint64_t a, uint64_t step) {
#pragma unroll
    for (int u = 0; u < K; ++u) {
      const uint64_t q = a + u * step;
      st16((void*)(uintptr_t)q, tag_vec(seed, q));
      st16((void*)(uintptr_t)(q + 16), tag_vec(seed, q + 16));
    }
  }
};

// P2: every window checked against its tags, then zeroed.  All loads are issued first and the exact count of bytes
// off their tags is branch-free; only a batch whose count is non-zero takes the branch, which books each 16-byte half
// with the tag check's rules (TagCheckZeroOp::single: mask, record while slots last, page map by warp reduction).
struct ProbeCheckOp {
  TagCheckZeroOp op;   // seed, book, base, cnt
  template <int K>
  __device__ __forceinline__ void batch(uint64_t a, uint64_t step) {
    uint4 v[K][2];
#pragma unroll
    for (int u = 0; u < K; ++u) {
      v[u][0] = ld16_cs((const void*)(uintptr_t)(a + u * step));
      v[u][1] = ld16_cs((const void*)(uintptr_t)(a + u * step + 16));
    }
    uint32_t n = 0;
#pragma unroll
    for (int u = 0; u < K; ++u)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const uint4 t = tag_vec(op.seed, a + u * step + 16 * h);
        n += nonzero_bytes_in_word(v[u][h].x ^ t.x) + nonzero_bytes_in_word(v[u][h].y ^ t.y) +
             nonzero_bytes_in_word(v[u][h].z ^ t.z) + nonzero_bytes_in_word(v[u][h].w ^ t.w);
      }
    if (n != 0) {
      // The branch reads the batch's windows again, one at a time: they come from L2 (this thread loaded them a moment
      // ago) and nothing has stored over them yet, so the loaded words die before it, as in TagCheckZeroOp::chunk.
      // Keeping them live through the eight bookings would take the registers of two more CTAs per SM.
#pragma unroll 1
      for (int u = 0; u < K; ++u)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const uint64_t q = a + u * step + 16 * h;
          const uint4 x = ld16_cs((const void*)(uintptr_t)q);
          op.single(q - op.base, TagCheckZeroOp::diff_mask(x, tag_vec(op.seed, q)), Vec16{{x.x, x.y, x.z, x.w}});
        }
    }
#pragma unroll
    for (int u = 0; u < K; ++u) {
      st16((void*)(uintptr_t)(a + u * step), make_uint4(0, 0, 0, 0));
      st16((void*)(uintptr_t)(a + u * step + 16), make_uint4(0, 0, 0, 0));
    }
    op.cnt += n;
  }
};

// P3: the non-zero bytes of every window (OR first; the exact count only for a batch that is not all zero).
struct ProbeRereadOp {
  uint64_t cnt = 0;
  template <int K>
  __device__ __forceinline__ void batch(uint64_t a, uint64_t step) {
    Vec16 v[K][2];
#pragma unroll
    for (int u = 0; u < K; ++u) {
      v[u][0] = ld16<kPolStreaming>((const void*)(uintptr_t)(a + u * step), 0);
      v[u][1] = ld16<kPolStreaming>((const void*)(uintptr_t)(a + u * step + 16), 0);
    }
    uint32_t any = 0;
#pragma unroll
    for (int u = 0; u < K; ++u)
#pragma unroll
      for (int k = 0; k < 4; ++k) any |= v[u][0].w[k] | v[u][1].w[k];
    if (any != 0) {
      uint32_t n = 0;
#pragma unroll
      for (int u = 0; u < K; ++u)
#pragma unroll
        for (int k = 0; k < 4; ++k) n += nonzero_bytes_in_word(v[u][0].w[k]) + nonzero_bytes_in_word(v[u][1].w[k]);
      cnt += n;
    }
  }
};

template <int THREADS, int PER>
__global__ void __launch_bounds__(THREADS)
alias_probe_fill_pass(uint64_t w0, uint64_t nwin, uint32_t seed) {
  ProbeFillOp op{seed};
  probe_windows<THREADS, PER>(w0, nwin, op);
}

// Bytes off their tags into *mismatch (one atomic per CTA), the windows that differ into `out` with offsets from `base`.
template <int THREADS, int PER>
__global__ void __launch_bounds__(THREADS)
alias_probe_check_pass(uint64_t w0, uint64_t nwin, uint32_t seed, unsigned long long* mismatch, LocateOut out,
                         uint64_t base) {
  ProbeCheckOp op{{seed, {out}, base}};
  probe_windows<THREADS, PER>(w0, nwin, op);
  op.op.book.flush();
  block_accumulate(op.op.cnt, mismatch);
}

template <int THREADS, int PER>
__global__ void __launch_bounds__(THREADS)
alias_probe_reread_pass(uint64_t w0, uint64_t nwin, unsigned long long* nonzero) {
  ProbeRereadOp op;
  probe_windows<THREADS, PER>(w0, nwin, op);
  block_accumulate(op.cnt, nonzero);
}

// The proving twins of the probe kernels: the same op through the same loop, and after each batch kProbeWindow bytes of
// every window it took counted into `cover`, one window slot u at a time across the lanes.  The 32 lanes of a warp take
// 32 consecutive windows (128 KiB), so a slot is normally one atomic per warp.
template <typename Op>
struct CoverProbeOp {
  Op& op;
  CoverOut cover;
  template <int K>
  __device__ __forceinline__ void batch(uint64_t a, uint64_t step) {
    op.template batch<K>(a, step);
#pragma unroll
    for (int u = 0; u < K; ++u) cover_lanes(cover, a + u * step, kProbeWindow);
  }
};

template <int THREADS, int PER>
__global__ void __launch_bounds__(THREADS)
cover_probe_fill_pass(uint64_t w0, uint64_t nwin, uint32_t seed, CoverOut cover) {
  ProbeFillOp op{seed};
  CoverProbeOp<ProbeFillOp> cop{op, cover};
  probe_windows<THREADS, PER>(w0, nwin, cop);
}

template <int THREADS, int PER>
__global__ void __launch_bounds__(THREADS)
cover_probe_check_pass(uint64_t w0, uint64_t nwin, uint32_t seed, unsigned long long* mismatch, LocateOut out,
                       uint64_t base, CoverOut cover) {
  ProbeCheckOp op{{seed, {out}, base}};
  CoverProbeOp<ProbeCheckOp> cop{op, cover};
  probe_windows<THREADS, PER>(w0, nwin, cop);
  op.op.book.flush();
  block_accumulate(op.op.cnt, mismatch);
}

template <int THREADS, int PER>
__global__ void __launch_bounds__(THREADS)
cover_probe_reread_pass(uint64_t w0, uint64_t nwin, unsigned long long* nonzero, CoverOut cover) {
  ProbeRereadOp op;
  CoverProbeOp<ProbeRereadOp> cop{op, cover};
  probe_windows<THREADS, PER>(w0, nwin, cop);
  block_accumulate(op.cnt, nonzero);
}

// ------------------------------------------------------------ test scaffolding
__device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}

// Deterministic sparse pattern: 8-byte word j (arena-global index) is
//   r = splitmix64(seed + j);  word = (r & 7) == 0 ? r & mask(r) : 0
// where mask keeps a pseudo-random subset of the bytes.  The C oracle
// (oracle/scrub_oracle.c: ccm_oracle_fill_random) restates the same formula.
__host__ __device__ inline uint64_t pattern_word(uint64_t seed, uint64_t j) {
  uint64_t x = seed + j;
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  x = x ^ (x >> 31);
  if ((x & 7) != 0) return 0;
  uint64_t keep = 0;
  for (int b = 0; b < 8; ++b)
    if ((x >> (8 + b)) & 1) keep |= 0xFFull << (8 * b);
  return (x >> 3 | 0x0101010101010101ull) & keep;  // kept bytes are guaranteed non-zero
}

__global__ void fill_pattern_kernel(uint64_t* words, uint64_t nwords, uint64_t word_index0, uint64_t seed) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nwords;
       i += (uint64_t)gridDim.x * blockDim.x)
    words[i] = pattern_word(seed, word_index0 + i);
}

}  // namespace ccm
