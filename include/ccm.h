/*
 * ccm.h — C ABI of libccm.so, the device shim of the H100-native CC-mode manager.
 *
 * This is the drop-in boundary for the ONE hot path (SURVEY.md §8): the per-GPU
 * stage -> reset -> wait-for-boot -> verify-mode sequence of the reference
 * (reference main.py:502-529), plus the NEW full-HBM scrub-and-verify stage that
 * gates a GPU's release after every CC transition (insertion point: after
 * reference main.py:529, before the state label is written at main.py:541).
 *
 * The reference has no C ABI at this boundary: it calls a duck-typed Python device
 * object from the external NVIDIA/gpu-admin-tools library (pinned v2025.11.21,
 * reference versions.mk:22; not vendored under /root/reference). Each entry point
 * below names the reference call site it replaces. k8s_cc_manager_b200/devices.py
 * rebuilds the duck-typed object on top of this ABI, so a reference-shaped manager
 * runs against it unchanged (see INTEGRATION.md for the ctypes stub).
 *
 * Conventions
 *  - plain C types only: ints, pointers, sizes.  No torch / C++ types cross the ABI.
 *  - every function returns CCM_OK (0) or a negative ccm_status; nothing throws.
 *  - the caller owns every out-struct / buffer; the library owns nothing the caller
 *    must free, except the scrub arena, which is released with ccm_arena_release().
 *  - thread safety: all per-device entry points may be called concurrently for
 *    DIFFERENT device indices (no global lock is held across reset / wait / scrub).
 *    Calls for the SAME device index are serialised by a per-device mutex.
 *  - `dev` is an index into the table returned by ccm_enumerate().
 *  - `stream` arguments are CUDA stream handles (cudaStream_t / CUstream) passed as
 *    void*; NULL means the library's own per-device stream.  Launches on ONE device
 *    must be ordered with respect to each other (same stream, or event-ordered
 *    streams): they share that device's result counter and tile-grab counter.
 */
#ifndef CCM_H_
#define CCM_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif
#if defined(__GNUC__)
#pragma GCC visibility push(default) /* the library is built -fvisibility=hidden */
#endif

#define CCM_ABI_VERSION 2 /* v2: deferred release, coverage fields; ccm_transition_many and the
                             TMA verify variant removed (one phase engine, one verify family).
                             Additions that change no existing entry point or struct (the tagged
                             gate, the dirt report, the residue census) keep the version. */

/* ---- status codes ------------------------------------------------------- */
typedef enum ccm_status {
  CCM_OK = 0,
  CCM_ERR_INVALID = -1,     /* bad argument                                    */
  CCM_ERR_NO_DEVICE = -2,   /* device index out of range                       */
  CCM_ERR_UNSUPPORTED = -3, /* op not supported by this device / backend       */
  CCM_ERR_IO = -4,          /* register / sysfs access failed                  */
  CCM_ERR_TIMEOUT = -5,     /* wait_for_boot timed out                         */
  CCM_ERR_CUDA = -6,        /* a CUDA runtime call failed (see ccm_last_error) */
  CCM_ERR_NOMEM = -7,       /* could not obtain the requested scrub arena      */
  CCM_ERR_DIRTY = -8,       /* verify found non-zero bytes after the scrub     */
  CCM_ERR_NO_CUDA = -9,     /* no usable CUDA device behind this entry         */
  CCM_ERR_STATE = -10,      /* call out of order (e.g. no arena held)          */
  CCM_ERR_FAULT = -11,      /* fault injected by the sim backend               */
  CCM_ERR_NOT_BOOTED = -12, /* device was reset and has not been waited for    */
  CCM_ERR_MISMATCH = -13,   /* tagged gate: bytes did not hold their tag       */
  CCM_ERR_UNCOVERED = -14 , /* coverage proof: a pass missed or repeated bytes */
  CCM_ERR_HBM_HEALTH = -15  /* HBM health: the GPU's ECC / row-remap state is
                               unfit or unknown (ccm_scrub_health mode 2)      */
} ccm_status;

/* ---- modes (string values of the reference: 'off' 'on' 'devtools') ------ */
typedef enum ccm_cc_mode { CCM_CC_OFF = 0, CCM_CC_ON = 1, CCM_CC_DEVTOOLS = 2 } ccm_cc_mode;
typedef enum ccm_ppcie_mode { CCM_PPCIE_OFF = 0, CCM_PPCIE_ON = 1 } ccm_ppcie_mode;

typedef enum ccm_dev_kind { CCM_KIND_GPU = 0, CCM_KIND_NVSWITCH = 1 } ccm_dev_kind;

/* Register backends.  A node whose GPUs stay bound to the driver cannot reset them, so the
 * CC-mode register file is simulated there; see DESIGN.md "what is simulated". */
typedef enum ccm_backend {
  CCM_BACKEND_SIM = 0,     /* synthetic topology, simulated registers           */
  CCM_BACKEND_CUDASIM = 1, /* real CUDA devices (BDF/name/HBM), sim registers   */
  CCM_BACKEND_SYSFS = 2    /* real PCI enumeration via sysfs, NVML CC query;
                              set/stage are UNSUPPORTED (register map lives in
                              gpu-admin-tools, not in the reference tree)       */
} ccm_backend;

/* One row per NVIDIA PCI function.
 * Replaces: pci.devices.find_gpus() -> (devices, count), reference main.py:155;
 * fields mirror what the reference reads from each device object:
 *   .bdf / .name                      main.py:187,191,210,239,280
 *   .is_gpu() / .is_nvswitch()        main.py:165,175
 *   .is_cc_query_supported            main.py:186
 *   .is_ppcie_query_supported         main.py:205,477                         */
typedef struct ccm_dev_info {
  int32_t index;               /* index to pass as `dev`                        */
  int32_t kind;                /* ccm_dev_kind                                  */
  int32_t cc_query_supported;  /* bool                                          */
  int32_t ppcie_query_supported; /* bool                                        */
  int32_t cuda_ordinal;        /* CUDA device ordinal backing the scrub, or -1  */
  int32_t reserved0;
  uint64_t hbm_total_bytes;    /* cudaMemGetInfo total, 0 when no CUDA device   */
  char bdf[32];                /* "0000:1b:00.0"                                */
  char name[96];               /* "NVIDIA H100 80GB HBM3"                       */
} ccm_dev_info;

/* ---- library / backend -------------------------------------------------- */
int ccm_abi_version(void);
const char* ccm_strerror(int status);
/* Copies this thread's last detailed error message; returns its length. */
int ccm_last_error(char* buf, size_t cap);

/* Selects the backend and (re)builds the device table.  Called implicitly with
 * the environment's choice (CCM_BACKEND = sim | cudasim | sysfs; default cudasim
 * when a CUDA device is visible, else sim) on first use. */
int ccm_init(int backend);
int ccm_backend_in_use(void);

/* find_gpus(): fills up to `cap` rows, writes the total count to *n.
 * Re-enumeration is cheap and keeps register state (reference calls find_gpus()
 * repeatedly: main.py:164,174,203,275,473). */
int ccm_enumerate(ccm_dev_info* out, int cap, int* n);

/* ---- register-level device ops (reference boundary, SURVEY §8b) --------- */
/* dev.query_cc_mode()      reference main.py:441,505,524 */
int ccm_query_cc_mode(int dev, int* mode);
/* dev.set_cc_mode(mode)    reference main.py:511 — STAGES only; applied by reset */
int ccm_set_cc_mode(int dev, int mode);
/* dev.query_ppcie_mode()   reference main.py:310,340,353,373,479,495 */
int ccm_query_ppcie_mode(int dev, int* mode);
/* dev.set_ppcie_mode(m)    reference main.py:345,359,482 — stages only */
int ccm_set_ppcie_mode(int dev, int mode);
/* dev.reset_with_os()      reference main.py:346,368,490,519 */
int ccm_reset(int dev);
/* dev.wait_for_boot()      reference main.py:347,372,494,523; timeout_ms<=0 = default */
int ccm_wait_for_boot(int dev, int timeout_ms);

/* ---- HBM scrub-and-verify (NEW stage; SURVEY §8a row S) ------------------ */
typedef enum ccm_scrub_variant {
  CCM_SCRUB_AUTO = 0,
  CCM_SCRUB_ST128 = 1,   /* st.global.v4.b32, persistent CTAs (AUTO)            */
  CCM_SCRUB_ST256 = 2,   /* 32 B per thread as two st.global.v4.b32             */
  CCM_SCRUB_TMA = 3,     /* cp.async.bulk.global.shared::cta from a zero tile   */
  CCM_SCRUB_MEMSET = 4   /* cudaMemsetAsync — library bar, baseline only        */
} ccm_scrub_variant;

typedef enum ccm_verify_variant {
  CCM_VERIFY_AUTO = 0,
  CCM_VERIFY_LD128 = 1,  /* ld.global.nc.v4.b32 (AUTO)                          */
  CCM_VERIFY_LD256 = 2   /* 32 B per thread as two ld.global.nc.v4.b32          */
} ccm_verify_variant;

/* Launch shape override; zeros mean "library default for this variant". */
typedef struct ccm_launch_cfg {
  int32_t ctas_per_sm;
  int32_t threads_per_cta;
  int32_t tile_bytes;   /* TMA variants: bytes per bulk op (multiple of 16);
                           ST/LD variants with a dynamic schedule: bytes per grab */
  int32_t unroll;       /* ST/LD variants: vectors in flight per thread (2,4,8) */
  int32_t cache_policy; /* 0 library default, 1 plain, 2 L2::evict_first,
                           3 streaming (.cs / L1::no_allocate), 4 L2::evict_last */
  int32_t schedule;     /* 0 library default, 1 static grid-stride, 2 dynamic
                           (persistent CTAs grab chunks off an atomic counter),
                           3 dynamic per WARP (ST/LD variants; no block barrier) */
} ccm_launch_cfg;

typedef struct ccm_scrub_result {
  uint64_t bytes_requested;    /* as passed (0 = max)                           */
  uint64_t bytes_scrubbed;     /* bytes actually zeroed and read back           */
  uint64_t device_total_bytes; /* cudaMemGetInfo total — coverage denominator   */
  uint64_t nonzero_bytes;      /* EXACT count of bytes != 0 found by verify     */
  double ms_acquire;           /* host time inside create/map/set-access; it
                                  overlaps the GPU work (chunk i is scrubbed
                                  while chunk i+1 is being mapped)              */
  double ms_scrub;             /* sum of the scrub kernels' CUDA-event times    */
  double ms_verify;            /* sum of the verify kernels' CUDA-event times   */
  double ms_release;           /* unmap + release when done inside the call; 0
                                  when release_deferred (ask
                                  ccm_scrub_release_wait for the real figure)   */
  double ms_total;             /* host wall-clock of the call = time to verdict */
  int32_t segments;            /* physical chunks mapped                        */
  int32_t scrub_variant;       /* variant that actually ran                     */
  int32_t verify_variant;
  int32_t sm_count;
  int32_t status;              /* ccm_status of this device (batched calls)     */
  int32_t release_deferred;    /* 1: the HBM is being handed back by the
                                  engine's background reaper (see below)        */
  /* ---- ABI v2 ---- */
  uint64_t device_free_before; /* cudaMemGetInfo free when the call started     */
  uint64_t bytes_unreached;    /* free HBM that could NOT be mapped and was
                                  therefore not scrubbed (0 on a clean device)  */
  double ms_release_wait;      /* time this call waited for the PREVIOUS call's
                                  deferred release before it could start        */
  double ms_gpu_span;          /* first scrub launch .. last verify done on the
                                  stream (includes waiting for mappings)        */
} ccm_scrub_result;

/* The product call.  Obtains `bytes` of HBM on device `dev` (0 = everything the
 * context can map, down to the last 2 MiB granule), zero-fills it, reads it back
 * and counts non-zero bytes.  The verdict is returned as soon as the count is on the
 * host; handing the HBM back to the driver (cuMemUnmap / cuMemRelease — the most
 * expensive part of the call, 0.33 ms/GiB, serialised node-wide by the driver)
 * runs on a per-device background thread.  That "reaper" is joined by the next
 * scrub / arena call on the device, by ccm_scrub_release_wait() and by
 * ccm_device_release(); CCM_ASYNC_RELEASE=0 keeps the release inside the call.
 * Returns CCM_ERR_DIRTY if nonzero_bytes != 0, CCM_ERR_NO_CUDA when the device has
 * no CUDA ordinal.  Never falls back to a host path. */
int ccm_scrub_verify(int dev, uint64_t bytes, ccm_scrub_result* out);

/* Blocks until the HBM of the last ccm_scrub_verify() on `dev` is back with the
 * driver.  *ms_release (optional) = duration of that background release,
 * *ms_waited (optional) = how long THIS call blocked.  CCM_OK when nothing is pending. */
int ccm_scrub_release_wait(int dev, double* ms_release, double* ms_waited);

/* Concurrent multi-context launcher: one host thread + primary context + stream
 * per device, no peer access, no collective.  With n > 1 each device maps its whole
 * range before its first launch: driver VMM calls interleaved with kernel launches on
 * several devices of ONE process contend in the driver, whereas a single device per
 * process is fastest pipelined (ccm_scrub_verify).  out[i].status is per device;
 * *wall_ms is the host wall-clock of the whole fan-out (max over devices).
 * Returns CCM_OK iff every device returned CCM_OK. */
int ccm_scrub_verify_many(int n, const int* devs, uint64_t bytes,
                          ccm_scrub_result* out, double* wall_ms);

/* ---- tagged gate: an address-tagged known answer before the zeroing -------
 * A zero read-back cannot tell a byte the scrub zeroed from a byte that was already zero, or
 * from a second virtual view of a physical byte zeroed elsewhere.  The tagged calls first write
 * every mapped byte with a tag that depends on its virtual address and on a per-call seed (the
 * word at address a holds lo32(a>>2)*0x9E3779B1 ^ hi32(a>>2)*0x85EBCA77 ^ seed; byte x is byte
 * x&3 of the word at x&~3), each range as soon as it is mapped.  After the last mapping every
 * range, in mapping order, is read back against its tags and zeroed in the same pass, and then
 * read back for zeros as in ccm_scrub_verify.  A view that aliases another one, a store that
 * does not land, or memory that was never written cannot hold the tag.  HBM traffic is about 4R
 * instead of 2R (R = bytes mapped). */
typedef struct ccm_tag_result {
  uint32_t seed;               /* in: 0 = draw one (std::random_device); out: the seed used */
  uint32_t reserved;
  uint64_t mismatch_bytes;     /* EXACT count of bytes that did not hold their tag */
  double ms_tag;               /* sum of the tag-fill kernels' CUDA-event times    */
  double ms_check;             /* sum of the check-and-zero kernels' times          */
  uint64_t va_base;            /* virtual address of the first byte scrubbed (the tags
                                  are a function of it; 0 when nothing was mapped) */
} ccm_tag_result;

/* ccm_scrub_verify with the tagged check.  Returns CCM_ERR_MISMATCH when
 * tag->mismatch_bytes != 0 (it takes precedence over CCM_ERR_DIRTY; both counts are
 * reported), otherwise what ccm_scrub_verify returns. */
int ccm_scrub_verify_tagged(int dev, uint64_t bytes, ccm_tag_result* tag, ccm_scrub_result* out);
/* ccm_scrub_verify_many with the tagged check; tag[i] belongs to devs[i]. */
int ccm_scrub_verify_many_tagged(int n, const int* devs, uint64_t bytes, ccm_tag_result* tag,
                                 ccm_scrub_result* out, double* wall_ms);

/* ---- where the dirt is: the report of a failed read-back ----------------------------------
 * When the zero read-back of a product call (zero or tagged) counts nonzero_bytes != 0, the call runs one
 * more kernel over what it mapped (one launch per segment on the cudaMalloc fallback) before the memory goes
 * back to the driver, and keeps the result as the engine's dirt report; a clean call launches nothing more.
 * Every product call on the device replaces the report.  The verdict and the status do not change.
 *
 * A dirty WINDOW is a 16-byte, 16-aligned address window that holds at least one non-zero byte.  Everything
 * but the choice of records is exact: when there are more than CCM_DIRT_RECORDS dirty windows, the records
 * are some CCM_DIRT_RECORDS of them, not necessarily the lowest. */
#define CCM_DIRT_RECORDS 64
typedef struct ccm_dirt_record {
  uint64_t offset;     /* first byte of the window - va_base (product call: offset into the mapping, or into the
                          concatenated segments on the fallback; a raw region that does not start 16-aligned
                          has its head window begin before it: negative, two's complement) */
  uint32_t chunk;      /* physical allocation behind the window, in creation order: the cuMemCreate handle
                          (main-zone chunks and tail granules alike; the aliased view of "scrub_alias" reports
                          handle 0), or the segment index on the fallback; 0 for a raw region */
  uint16_t mask;       /* bit i: byte i of the window is non-zero (bytes outside the region count as 0) */
  uint16_t reserved;
  uint8_t bytes[16];   /* the window as the pass read it */
} ccm_dirt_record;     /* 32 B */

typedef struct ccm_dirt_report {
  uint64_t nonzero_bytes;  /* non-zero bytes the locate pass counted: it recounts the read-back, and both
                              are reported when something wrote the memory in between */
  uint64_t dirty_windows;
  uint64_t first_offset;   /* offset of the first / last non-zero byte from va_base */
  uint64_t last_offset;
  uint64_t va_base;        /* address of the first byte the pass read (fallback: of the first segment) */
  double ms_locate;        /* CUDA-event time of the locate kernel(s) */
  int32_t located;         /* 1: a locate pass ran; 0: the last call read back clean (or never ran) */
  int32_t nrecords;        /* min(dirty_windows, CCM_DIRT_RECORDS), distinct windows sorted by offset */
  int32_t truncated;       /* dirty_windows > CCM_DIRT_RECORDS */
  int32_t reserved;
  ccm_dirt_record records[CCM_DIRT_RECORDS];
} ccm_dirt_report;

/* The dirt report of the last product call on the CUDA device `cuda_ordinal` (located == 0 when it read
 * back clean).  CCM_ERR_NO_CUDA when there is no such CUDA device. */
int ccm_scrub_last_dirt(int cuda_ordinal, ccm_dirt_report* out);
/* The locate pass on caller-owned memory (any alignment, any length; synchronises).  Reads the region and
 * writes nothing into it; located == 1 and every record's chunk is 0. */
int ccm_region_locate(int cuda_ordinal, const void* dptr, uint64_t bytes, void* stream, ccm_dirt_report* out);

/* ---- where the tags were wrong: the report of a failed tagged check or alias probe ---------------
 * The tagged check-and-zero kernel books, in the same pass that counts mismatch_bytes, every 16-byte, 16-aligned
 * window that differs from its tags; a check that finds nothing costs nothing more (no launch, memset or copy).
 * When a tagged product call counts tag->mismatch_bytes != 0, it copies that book once after its last kernel and
 * keeps it, classified, as the engine's mismatch report; so does a probed zero-gate call whose alias probe (below)
 * found bytes off their tags, with the probe's seed and mismatch count.  Every product call on the device replaces the
 * report.
 * The verdict, its precedence and the dirt report do not change.
 *
 * EXACT: mismatch_bytes, mismatch_windows, zero_windows, first_offset, last_offset.  The split of the other
 * windows between ALIAS, PARTIAL and FOREIGN is known for the records only (telling them apart needs the
 * decode below, which is not in the kernel's loop); with more than CCM_DIRT_RECORDS mismatched windows the records
 * are some CCM_DIRT_RECORDS of them, not necessarily the lowest.
 *
 * Each record gets the first kind that fits, in this order:
 *   CCM_MISMATCH_ZERO     every byte of the window inside the region reads 0 (the fill never reached it, or
 *                         something zeroed it afterwards: e.g. the check of a second view got there first);
 *   CCM_MISMATCH_ALIAS    the bytes are exactly this call's tags of a DIFFERENT 16-aligned window inside what the
 *                         call mapped (the region, for ccm_region_tag_check_locate): two virtual views of one
 *                         physical range.  source_offset / source_chunk name that window.  The decode: the tag is
 *                         a bijection of the address within each 16 GiB window, so one whole 4-byte word of the
 *                         window is inverted for every 16 GiB window the mapping spans, and a candidate is kept
 *                         only if every byte of the window equals its tag.  A window with no whole word inside
 *                         the region is never ALIAS;
 *   CCM_MISMATCH_PARTIAL  some byte still holds its own tag: flipped or overwritten bytes in a tagged window;
 *   CCM_MISMATCH_FOREIGN  anything else: data this call did not write (another writer, a stale mapping). */
typedef enum ccm_mismatch_kind {
  CCM_MISMATCH_ZERO = 1,
  CCM_MISMATCH_ALIAS = 2,
  CCM_MISMATCH_PARTIAL = 3,
  CCM_MISMATCH_FOREIGN = 4
} ccm_mismatch_kind;

typedef struct ccm_mismatch_record {
  uint64_t offset;         /* first byte of the window - va_base (as ccm_dirt_record.offset) */
  uint32_t chunk;          /* physical allocation behind the window (as ccm_dirt_record.chunk) */
  uint16_t mask;           /* bit i: byte i of the window differs from its tag (bytes outside the region: 0) */
  uint16_t kind;           /* ccm_mismatch_kind */
  uint64_t source_offset;  /* ALIAS: the window whose tags these are, - va_base; otherwise 0 */
  uint32_t source_chunk;   /* ALIAS: the physical allocation behind it; otherwise 0 */
  uint32_t reserved;
  uint8_t bytes[16];       /* the window as the check read it, before it zeroed it */
} ccm_mismatch_record;     /* 48 B */

typedef struct ccm_mismatch_report {
  uint64_t mismatch_bytes;    /* bytes that did not hold their tag (== ccm_tag_result.mismatch_bytes) */
  uint64_t mismatch_windows;  /* windows with at least one such byte */
  uint64_t zero_windows;      /* of those, windows whose bytes inside the region all read 0 */
  uint64_t first_offset;      /* first / last mismatched byte, from va_base */
  uint64_t last_offset;
  uint64_t va_base;           /* as ccm_dirt_report.va_base */
  uint32_t seed;              /* the tags' seed */
  int32_t located;            /* 1: the report describes a failed check; 0: the last call's check was clean */
  int32_t nrecords;           /* min(mismatch_windows, CCM_DIRT_RECORDS), distinct windows sorted by signed offset */
  int32_t truncated;          /* mismatch_windows > CCM_DIRT_RECORDS */
  ccm_mismatch_record records[CCM_DIRT_RECORDS];
} ccm_mismatch_report;

/* The mismatch report of the last product call on the CUDA device `cuda_ordinal` (located == 0 when its tagged
 * check was clean, or it was not tagged).  CCM_ERR_NO_CUDA when there is no such CUDA device. */
int ccm_scrub_last_mismatch(int cuda_ordinal, ccm_mismatch_report* out);
/* ccm_region_tag_check_zero on caller-owned memory that also fills `out` (synchronises; any alignment, any
 * length).  located == 1, every record's chunk is 0 and the ALIAS search is limited to the region. */
int ccm_region_tag_check_locate(int cuda_ordinal, void* dptr, uint64_t bytes, uint32_t seed, void* stream,
                                ccm_mismatch_report* out);

/* ---- what the gate found before it erased it: the residue census ------------------------------
 * Opt-in, per call.  A census call replaces the first pass of the gate, the one that first writes every mapped byte
 * (the zero gate's scrub, the tagged gate's tag fill), by a kernel that reads each 16-byte vector, books it, and
 * then stores zeros (or the tags) to the same addresses: the same ranges, the same number of launches, timed as
 * ms_scrub (zero gate) or tag->ms_tag (tagged gate).  It answers "did the gate have anything to erase?": how many
 * bytes of what it mapped were non-zero at first touch, and where.  It is a report, never a check: the verdict, the
 * status, the error text and the dirt and mismatch reports are those of the same call without it.
 *
 * What the census reads is the previous tenant's data, so no byte of it is reported: only counts, offsets, masks and
 * chunks.  EXACT: residue_bytes, residue_windows, first_offset, last_offset.  With more than CCM_DIRT_RECORDS
 * non-zero windows the records are some CCM_DIRT_RECORDS of them, not necessarily the lowest.
 *
 * CCM_SCRUB_VARIANT pins only calls without the census; a census call always runs the census kernel, which has the
 * shape and stores of the default 128-bit scrub, and reports scrub_variant = CCM_SCRUB_ST128. */
typedef struct ccm_residue_record {
  uint64_t offset;     /* first byte of the window - va_base (as ccm_dirt_record.offset) */
  uint32_t chunk;      /* physical allocation behind the window (as ccm_dirt_record.chunk) */
  uint16_t mask;       /* bit i: byte i of the window was non-zero (bytes outside the region count as 0) */
  uint16_t reserved;
} ccm_residue_record;  /* 16 B; no bytes */

typedef struct ccm_residue_report {
  uint64_t residue_bytes;    /* bytes that were non-zero when the census read them */
  uint64_t residue_windows;  /* 16-byte windows with at least one such byte */
  uint64_t first_offset;     /* first / last non-zero byte, from va_base (0 when there is none) */
  uint64_t last_offset;
  uint64_t bytes_examined;   /* bytes the census read (== ccm_scrub_result.bytes_scrubbed) */
  uint64_t va_base;          /* as ccm_dirt_report.va_base */
  int32_t located;           /* 1: a census ran over everything the call mapped */
  int32_t nrecords;          /* min(residue_windows, CCM_DIRT_RECORDS), distinct windows sorted by signed offset */
  int32_t truncated;         /* residue_windows > CCM_DIRT_RECORDS */
  int32_t reserved;
  ccm_residue_record records[CCM_DIRT_RECORDS];
} ccm_residue_report;

/* ccm_scrub_verify (tag == NULL) or ccm_scrub_verify_tagged (tag != NULL) with the census; `residue` is required. */
int ccm_scrub_verify_residue(int dev, uint64_t bytes, ccm_tag_result* tag, ccm_residue_report* residue,
                             ccm_scrub_result* out);
/* The fan-out form: tag is NULL (zero gate) or n blocks; residue[i] belongs to devs[i]. */
int ccm_scrub_verify_many_residue(int n, const int* devs, uint64_t bytes, ccm_tag_result* tag,
                                  ccm_residue_report* residue, ccm_scrub_result* out, double* wall_ms);
/* The census on caller-owned memory (any alignment, any length; synchronises).  Afterwards the region holds
 * exactly zero (store_tags == 0) or exactly the tags of `seed`; no byte outside it is touched.  located == 1 and
 * every record's chunk is 0. */
int ccm_region_census(int cuda_ordinal, void* dptr, uint64_t bytes, int store_tags, uint32_t seed, void* stream,
                      ccm_residue_report* out);

/* ---- which pages the three reports' bytes lie on: the page maps --------------------------------
 * Beyond its records, each book (the dirt, mismatch and residue reports) counts its bytes per 2 MiB page, in the same
 * pass: the non-zero bytes (dirt), the bytes off their tags (mismatch) and the bytes non-zero at first touch
 * (residue).  The entries of a map add up to the report's exact count (nonzero_bytes, mismatch_bytes,
 * residue_bytes).  A window belongs to the page of its offset from va_base, offset / CCM_PAGE_BYTES; the head window
 * of a raw region that does not start 16-aligned (negative offset) belongs to page 0.  2 MiB is the VMM granule: every
 * chunk and tail granule the product call maps is a whole number of pages, so each page lies in exactly one
 * cuMemCreate allocation.
 *
 * `chunk` follows the rule of the record chunks: the handle index (VMM), the segment index (cudaMalloc fallback), 0
 * for a raw region.  On the fallback a page can span two segments; it then has the chunk of its first byte.
 *
 * A clean report has an empty map, and costs nothing more (no launch, memset or copy). */
#define CCM_PAGE_BYTES (2u << 20)
typedef enum ccm_book { CCM_BOOK_DIRT = 1, CCM_BOOK_MISMATCH = 2, CCM_BOOK_RESIDUE = 3 } ccm_book;
typedef struct ccm_page_entry {
  uint64_t page;    /* offset of the page from the report's va_base = page * CCM_PAGE_BYTES */
  uint32_t bytes;   /* booked bytes of the windows on this page (>= 1, <= CCM_PAGE_BYTES) */
  uint32_t chunk;   /* physical allocation behind the page's first byte (as ccm_dirt_record.chunk) */
} ccm_page_entry;   /* 16 B */
/* The pages behind the last report of `book` (ccm_book) on this CUDA device: one entry per 2 MiB page (offset =
 * page * CCM_PAGE_BYTES from the report's va_base) holding at least one booked byte, ascending.  Writes min(*n, cap)
 * entries, *n = all of them.  The last report of a book is the one the last call on the device that reports it
 * returned or kept: dirt and mismatch, a product call or ccm_region_locate / ccm_region_tag_check_locate; residue, a
 * census product call or ccm_region_census.  CCM_ERR_NO_CUDA when there is no such CUDA device, CCM_ERR_INVALID for
 * an unknown book, n == NULL, or out == NULL with cap > 0. */
int ccm_last_page_map(int cuda_ordinal, int book, ccm_page_entry* out, uint64_t cap, uint64_t* n);

/* ---- what kind of dirt: the triage of a failed read-back ----------------------------------------
 * Opt-in, per device.  An armed product call whose zero read-back counted nonzero_bytes != 0, and whose locate pass
 * produced the dirt report, looks at the dirty memory once more before the mapping goes back to the driver.  It takes
 * every page of the dirt page map, intersects it with what the call mapped (on the cudaMalloc fallback, with each
 * segment) and merges adjacent pieces into maximal contiguous runs.  Then, over every run:
 *   T1  stores zero with the default scrub (scrub_st128_fast_kernel): one launch per run;
 *   T2  reads it back with the locate kernel: one launch per run;
 *   hold: waits hold_ms on the host, the mapping still held;
 *   T3  reads it back with the locate kernel again: one launch per run.
 * Each page of the dirt page map gets one class:
 *   CCM_TRIAGE_STAYS    T2 found non-zero bytes on the page: zero stored over it does not read back as zero (stores
 *                       that do not land, or something writing it continuously);
 *   CCM_TRIAGE_RETURNS  T2 read the page back clean, T3 did not: something wrote it again during the hold;
 *   CCM_TRIAGE_CLEARS   T2 and T3 both read it back clean: the dirt was written once, and the memory holds zero.
 * The counts per page come from the page maps of T2 and T3, so they are exact.  The triage is a report: the verdict,
 * the status, the error text, ccm_scrub_result, the dirt, mismatch and residue reports and the dirt page map are
 * those of the same call unarmed.  A clean armed call launches, copies and waits for nothing more than a clean
 * unarmed one.  Two drills (ccm_sim_set) give every class an exact answer: "triage_stay" = k XORs the first byte of
 * each of the first k dirt pages (in page order) with 0xA5 between T1 and T2, "triage_return" = k the same bytes
 * between T2 and T3. */
#define CCM_TRIAGE_MAX_HOLD_MS 10000u
typedef enum ccm_triage_class {
  CCM_TRIAGE_STAYS = 1,
  CCM_TRIAGE_RETURNS = 2,
  CCM_TRIAGE_CLEARS = 3
} ccm_triage_class;

typedef struct ccm_triage_report {
  uint64_t pages_examined;   /* pages of the dirt page map (each is one ccm_triage_page) */
  uint64_t bytes_examined;   /* mapped bytes of those pages: what T1, T2 and T3 each covered */
  uint64_t stay_pages, stay_bytes;        /* pages of each class, and the dirt page map's bytes on them (the three */
  uint64_t return_pages, return_bytes;    /* byte counts add up to ccm_dirt_report.nonzero_bytes) */
  uint64_t clear_pages, clear_bytes;
  uint64_t t2_bytes;         /* non-zero bytes T2 / T3 found (exact) */
  uint64_t t3_bytes;
  uint64_t t2_first_offset;  /* first / last non-zero byte T2 / T3 found, from va_base (0 when it found none) */
  uint64_t t2_last_offset;
  uint64_t t3_first_offset;
  uint64_t t3_last_offset;
  uint64_t va_base;          /* as ccm_dirt_report.va_base */
  double ms_hold;            /* the hold actually waited (>= hold_ms) */
  double ms_triage;          /* host wall-clock of the whole triage, hold included */
  uint32_t hold_ms;          /* the hold the device was armed with */
  int32_t runs;              /* maximal contiguous runs the dirt pages make */
  int32_t triaged;           /* 1: the last product call ran the triage; 0: it did not (the report is empty) */
  int32_t reserved;
} ccm_triage_report;

typedef struct ccm_triage_page {
  uint64_t page;        /* as ccm_page_entry.page: offset page * CCM_PAGE_BYTES from va_base */
  uint32_t chunk;       /* as ccm_page_entry.chunk */
  uint32_t cls;         /* ccm_triage_class */
  uint32_t dirt_bytes;  /* the dirt page map's bytes on the page */
  uint32_t t2_bytes;    /* non-zero bytes T2 / T3 found on it */
  uint32_t t3_bytes;
  uint32_t reserved;
} ccm_triage_page;      /* 32 B */

/* Arms (hold_ms > 0) or disarms (hold_ms == 0) the triage for every later product call on the CUDA device
 * `cuda_ordinal`.  CCM_ERR_INVALID for hold_ms > CCM_TRIAGE_MAX_HOLD_MS, CCM_ERR_NO_CUDA when there is no such CUDA
 * device. */
int ccm_scrub_triage(int cuda_ordinal, uint32_t hold_ms);
/* The triage report of the last product call on the CUDA device `cuda_ordinal` (triaged == 0 when it did not triage).
 * CCM_ERR_NO_CUDA when there is no such CUDA device. */
int ccm_scrub_last_triage(int cuda_ordinal, ccm_triage_report* out);
/* The pages of that report, one per page of the dirt page map, ascending.  Writes min(*n, cap) entries, *n = all of
 * them.  CCM_ERR_NO_CUDA as above, CCM_ERR_INVALID for n == NULL, or out == NULL with cap > 0. */
int ccm_last_triage_pages(int cuda_ordinal, ccm_triage_page* out, uint64_t cap, uint64_t* n);

/* ---- what kind of mismatch: the triage of a failed tagged check ---------------------------------
 * The tagged twin of the dirt triage, armed separately (arming one never arms the other).  A failed tagged check
 * zeroes what it counts in the same pass, so its read-back is clean and the dirt triage never sees it.  An armed
 * product call whose tagged check counted mismatch_bytes != 0, and which produced the mismatch report and its page map,
 * takes every page of the mismatch page map, intersects it with what the call mapped (on the cudaMalloc fallback, with
 * each segment) and merges adjacent pieces into maximal contiguous runs, as the dirt triage does.  It runs after the
 * dirt triage when the call runs both, and over every run:
 *   T1  writes the call's tags again (tag_fill_kernel, the call's seed): one launch per run;
 *   T2  checks the tags and zeroes the run (tag_check_zero_kernel, offsets from the mismatch report's va_base, so its
 *       pages are those of the mismatch page map): one launch per run;
 *   hold: waits hold_ms on the host, the mapping still held;
 *   T3  reads the run for non-zero bytes (the locate kernel): one launch per run.
 * T2 leaves the runs zero, so the triage leaves no tag behind in memory that goes back to the driver.  Each page of the
 * mismatch page map gets one class:
 *   CCM_TRIAGE_STAYS    T2 found bytes off their tags on the page: a fresh tag does not read back (a store that does
 *                       not land, a stuck cell, or a second view of the same memory);
 *   CCM_TRIAGE_RETURNS  T2 was clean and T3 found non-zero bytes: something wrote the memory during the hold;
 *   CCM_TRIAGE_CLEARS   otherwise: a one-time write.
 * T3 tests whether zero holds, not whether the tags hold: with the check-and-zero at T2, at least one view of every
 * aliased pair stays whatever order the stores land in.  The reports are ccm_triage_report and ccm_triage_page, where
 * dirt_bytes, stay_bytes, return_bytes and clear_bytes are bytes of the MISMATCH page map (stay + return + clear ==
 * ccm_tag_result.mismatch_bytes), t2_bytes are bytes T2 found off their tags, t3_bytes non-zero bytes T3 found, and
 * va_base is the mismatch report's va_base.  The invariants of the dirt triage hold: the verdict, the status, the error
 * text, ccm_scrub_result, ccm_tag_result, the dirt, mismatch, residue and dirt-triage reports and every page map are
 * those of the same call unarmed, and a clean armed call launches, copies and waits for nothing more.  The drills
 * "triage_stay" and "triage_return" act on the first pages of the mismatch page map: page i has T2 bytes [i < stay] and
 * T3 bytes [i < ret] (T2 zeroes the stay byte); "tag_flood" makes every mapped page a mismatch page. */
/* Arms (hold_ms > 0) or disarms (hold_ms == 0) the mismatch triage, as ccm_scrub_triage. */
int ccm_scrub_mismatch_triage(int cuda_ordinal, uint32_t hold_ms);
/* The mismatch triage report of the last product call, as ccm_scrub_last_triage. */
int ccm_scrub_last_mismatch_triage(int cuda_ordinal, ccm_triage_report* out);
/* Its pages, one per page of the mismatch page map, ascending, as ccm_last_triage_pages. */
int ccm_last_mismatch_triage_pages(int cuda_ordinal, ccm_triage_page* out, uint64_t cap, uint64_t* n);

/* ---- coverage proof: did every pass walk every byte it mapped? ----------------------------------
 * Opt-in, per device.  A read-back that reads nothing returns what a read-back of clean memory returns, so a clean
 * verdict says nothing about how much memory the kernels walked.  An armed product call runs the proving twin of
 * every kernel of its passes (the default scrub and read-back, tag fill, tag check and both census kernels: same
 * shape, grab words, loads and stores, whatever CCM_SCRUB_VARIANT / CCM_VERIFY_VARIANT pin; the call reports
 * CCM_SCRUB_ST128 / CCM_VERIFY_LD128).  Each counts on the device, per pass, the bytes it processed on every 2 MiB
 * page from va_base.  Its passes:
 *   CCM_PASS_FIRST     the scrub, the census, or the tag fill;
 *   CCM_PASS_CHECK     the tagged check-and-zero (tagged calls only);
 *   CCM_PASS_READBACK  the zero read-back.
 * After the call's final synchronise, before the locate pass and the triages (proven apart: ccm_report_cover), the host copies the
 * maps once and requires of every pass that ran: page p of [0, bytes_mapped) counted exactly
 * min(CCM_PAGE_BYTES, bytes_mapped - p * CCM_PAGE_BYTES) bytes, every other page and the outside slot 0.  When a pass
 * missed a byte, or counted one twice or outside the mapping, the call returns CCM_ERR_UNCOVERED: it takes precedence
 * over CCM_ERR_MISMATCH and CCM_ERR_DIRTY (their counts come from an incomplete pass; both are still reported).  Apart
 * from the status and the timings, an armed call leaves what an unarmed one leaves, and launches no more kernels.
 * The proof says the kernels issued a store or load for every mapped byte once per pass; not that the stores landed
 * (the read-back's job) or that no second view of the memory exists (the tagged gate's job).  The region calls and
 * the arena entry points are never proven.  On the cudaMalloc fallback, page p is counted from va_base = the first
 * segment's address, in the concatenated segments. */
typedef enum ccm_cover_pass_id {
  CCM_PASS_FIRST = 1,
  CCM_PASS_CHECK = 2,
  CCM_PASS_READBACK = 3
} ccm_cover_pass_id;

typedef struct ccm_cover_pass {
  uint64_t bytes_counted;     /* every byte the pass's kernels counted, the outside slot included */
  uint64_t bytes_missing;     /* sum over pages of (expected - counted) where short */
  uint64_t bytes_extra;       /* sum over pages of (counted - expected) where over, plus the outside slot */
  uint64_t bytes_outside;     /* the outside slot: bytes counted before va_base or past the last page */
  uint64_t pages_short;       /* pages that counted fewer bytes than expected */
  uint64_t pages_over;        /* pages that counted more (the outside slot is not a page) */
  uint64_t first_short_page;  /* the first short page (0 when none) */
  int32_t ran;                /* 1: the call ran this pass (the rest of the row is then meaningful) */
  int32_t reserved;
} ccm_cover_pass;             /* 64 B */

typedef struct ccm_cover_report {
  uint64_t bytes_mapped;      /* what the call mapped (ccm_scrub_result.bytes_scrubbed) */
  uint64_t pages_mapped;      /* ceil(bytes_mapped / CCM_PAGE_BYTES) */
  uint64_t va_base;           /* address of page 0 */
  double ms_prove;            /* host wall-clock of the copy and the comparison */
  int32_t proved;             /* 1: the last product call was armed and its passes finished */
  int32_t covered;            /* 1: every pass that ran counted every page exactly */
  ccm_cover_pass pass[3];     /* indexed by ccm_cover_pass_id - 1 */
} ccm_cover_report;           /* 232 B */

typedef struct ccm_cover_page {
  uint64_t page;              /* offset page * CCM_PAGE_BYTES from va_base */
  uint32_t chunk;             /* as ccm_page_entry.chunk (pages past the mapping: the last chunk) */
  uint32_t expected;          /* bytes every pass that ran had to count on the page */
  uint32_t count[3];          /* bytes each pass counted (indexed as ccm_cover_report.pass; 0 for a pass not run) */
  uint32_t reserved;
} ccm_cover_page;             /* 32 B */

/* Arms (on != 0) or disarms (on == 0) the coverage proof for every later product call on the CUDA device
 * `cuda_ordinal`.  The first arming sets aside the cover maps (three maps of one u32 per 2 MiB page of the device and
 * an outside slot, and a pinned host copy) and the coverage ledgers (ccm_cover_ledger, below), and makes the proving
 * kernels resident.  CCM_ERR_NO_CUDA when there is no
 * such CUDA device. */
int ccm_scrub_prove(int cuda_ordinal, int on);
/* The coverage report of the last product call on the CUDA device (proved == 0 when it was not armed, or its passes
 * did not finish).  CCM_ERR_NO_CUDA when there is no such CUDA device. */
int ccm_scrub_last_cover(int cuda_ordinal, ccm_cover_report* out);
/* One entry per page that some pass that ran did not count exactly, ascending.  Writes min(*n, cap) entries, *n = all
 * of them.  CCM_ERR_NO_CUDA as above, CCM_ERR_INVALID for n == NULL, or out == NULL with cap > 0. */
int ccm_last_cover_pages(int cuda_ordinal, ccm_cover_page* out, uint64_t cap, uint64_t* n);

/* ---- coverage ledger: did every thread of every pass walk its share of every chunk once? ----------
 * Part of the coverage proof, armed with it (ccm_scrub_prove).  A cover map adds a whole chunk per grab, for the CTA's
 * thread 0, per 2 MiB page: a pass that walked one chunk twice and skipped another on the same page counts that page
 * exactly, and so does a CTA some of whose threads dropped their stores or loads.  The ledger counts, per pass, per
 * CCM_LEDGER_SLOT_BYTES slot (address - va_base) / CCM_LEDGER_SLOT_BYTES, the bytes EVERY thread's own store or load
 * step addressed, lane by lane, and an outside slot.  128 KiB is the chunk of every default-frame pass, so on the VMM
 * path one chunk is one slot.  Where the cover maps are copied, the host copies the ledgers once and requires of every
 * pass that ran: slot s of [0, bytes_mapped) counted exactly min(CCM_LEDGER_SLOT_BYTES, bytes_mapped - s *
 * CCM_LEDGER_SLOT_BYTES) bytes, every other slot and the outside slot 0.  An inexact ledger returns CCM_ERR_UNCOVERED
 * at the cover maps' rank (ahead of the probe proof, CCM_ERR_MISMATCH and CCM_ERR_DIRTY).  A call can then return
 * CCM_ERR_UNCOVERED with ccm_cover_report.covered == 1: its pages counted exactly, its slots did not (the
 * "cover_repeat" drill does this on purpose).  The first arming sets aside the three ledgers (ceil(device total /
 * CCM_LEDGER_SLOT_BYTES) + 1 words each, about 2.6 MB each at 85 GB) and their pinned host copy, with the cover maps,
 * before anything is mapped: an armed whole-HBM call maps that much less.  The report proof, ccm_region_prove and the
 * probe keep no ledger. */
#define CCM_LEDGER_SLOT_BYTES (128u << 10)

typedef struct ccm_ledger_pass {
  uint64_t slots_short;       /* slots that counted fewer bytes than expected */
  uint64_t slots_over;        /* slots that counted more (the outside slot is not a slot) */
  uint64_t bytes_missing;     /* sum over slots of (expected - counted) where short */
  uint64_t bytes_extra;       /* sum over slots of (counted - expected) where over, plus the outside slot */
  uint64_t bytes_outside;     /* the outside slot: bytes counted before va_base or past the last slot */
  uint64_t first_short_slot;  /* the first short slot (0 when none) */
  uint64_t first_over_slot;   /* the first over slot (0 when none) */
  int32_t ran;                /* 1: the call ran this pass (the rest of the row is then meaningful) */
  int32_t reserved;
} ccm_ledger_pass;            /* 64 B */

typedef struct ccm_cover_ledger {
  uint64_t bytes_mapped;      /* as ccm_cover_report.bytes_mapped */
  uint64_t slots_mapped;      /* ceil(bytes_mapped / CCM_LEDGER_SLOT_BYTES) */
  uint64_t va_base;           /* address of slot 0 (the cover report's page 0) */
  double ms_ledger;           /* host wall-clock of the ledgers' copy and comparison */
  int32_t proved;             /* 1: the last product call was armed and its passes finished */
  int32_t exact;              /* 1: every pass that ran counted every slot exactly */
  ccm_ledger_pass pass[3];    /* indexed by ccm_cover_pass_id - 1 */
} ccm_cover_ledger;           /* 232 B */

typedef struct ccm_ledger_slot {
  uint64_t slot;              /* offset slot * CCM_LEDGER_SLOT_BYTES from va_base */
  uint32_t chunk;             /* as ccm_cover_page.chunk, of the slot's first byte */
  uint32_t expected;          /* bytes every pass that ran had to count on the slot */
  uint32_t count[3];          /* bytes each pass counted (indexed as ccm_cover_ledger.pass; 0 for a pass not run) */
  uint32_t reserved;
} ccm_ledger_slot;            /* 32 B */

/* The coverage ledger of the last product call on the CUDA device (proved == 0 when it was not armed, or its passes
 * did not finish).  CCM_ERR_NO_CUDA when there is no such CUDA device, CCM_ERR_INVALID for out == NULL. */
int ccm_scrub_last_ledger(int cuda_ordinal, ccm_cover_ledger* out);
/* One entry per slot that some pass that ran did not count exactly, ascending, with the conventions of
 * ccm_last_cover_pages. */
int ccm_last_ledger_slots(int cuda_ordinal, ccm_ledger_slot* out, uint64_t cap, uint64_t* n);

/* ---- alias probe: is any page of the zero gate mapped twice? -------------------------------------
 * Opt-in, per device, for the zero gate.  Two virtual views of one physical page both read back zero, both count in
 * bytes_scrubbed and in the coverage proof, and the memory that should have backed the second view keeps whatever it
 * held.  A probe WINDOW is every 32-byte sector whose address is a multiple of CCM_PROBE_STRIDE (4 KiB, the smallest
 * page the MMU maps) and that lies entirely inside one mapped chunk: one iteration of the VMM mapping loop (a main-zone
 * chunk or a tail granule), or one segment on the cudaMalloc fallback.  The window's place depends only on the address
 * modulo 4096, so two views of one physical page probe the same sector.
 *
 * An armed zero-gate product call whose passes finished and whose read-back counted nonzero_bytes == 0 probes after its
 * last read-back, before the coverage proof is compared, the locate pass, the triages and the release.  Each step is
 * one launch per chunk (segment) in mapping order, and each step ends before the next starts:
 *   P1  writes the tags (the tagged gate's tag function, a seed drawn per call) into every window;
 *   P2  checks every window against its tags, books the bytes that differ into the mismatch report and its page map
 *       (CCM_BOOK_MISMATCH), and stores zeros to the window;
 *   P3  reads every window for non-zero bytes.
 * A P2 count above zero returns CCM_ERR_MISMATCH; a P3 count above zero returns CCM_ERR_DIRTY with nonzero_bytes = that
 * count, and the locate pass finds it.  CCM_ERR_UNCOVERED still takes precedence over both.  Afterwards every window
 * holds zero again.  A call whose read-back found dirt does not probe (probed == 0): the dirt stays as the read-back saw
 * it.  With mapping order, the later view's tags win P1; P2 of the earlier view reads them (ALIAS records) and zeroes
 * them, and P2 of the later view reads zeros (ZERO records).
 *
 * The probe sees view-level aliases only: an address fault with a stride below 4 KiB, or stores that fail over memory
 * that already holds zero, stay the tagged gate's job.  Tagged calls ignore the arming (their check covers every
 * window); region and arena calls never probe.  A call that is both proven (ccm_scrub_prove) and probed proves the
 * probe too (ccm_probe_cover, below).  A probed call launches the unarmed call's kernels plus 3 per chunk (segment),
 * plus the drills' launches. */
#define CCM_PROBE_STRIDE 4096u
#define CCM_PROBE_WINDOW 32u
typedef struct ccm_probe_report {
  uint64_t windows;               /* probe windows of the call (of every step) */
  uint64_t bytes_probed;          /* windows * CCM_PROBE_WINDOW */
  uint64_t mismatch_bytes;        /* bytes P2 found off their tags (== the mismatch report's mismatch_bytes) */
  uint64_t mismatch_windows;      /* 16-byte windows of the mismatch report with such bytes */
  uint64_t reread_nonzero_bytes;  /* non-zero bytes P3 found */
  uint32_t seed;                  /* the tags' seed */
  uint32_t launches;              /* kernels the probe launched (its drills included) */
  uint64_t va_base;               /* as ccm_mismatch_report.va_base: what the offsets are from */
  double ms_probe;                /* CUDA-event time from the first P1 launch to the end of the last P3 launch */
  int32_t probed;                 /* 1: the last product call ran the probe */
  int32_t reserved[3];
} ccm_probe_report;               /* 80 B */

/* Arms (on != 0) or disarms (on == 0) the alias probe for every later zero-gate product call on the CUDA device
 * `cuda_ordinal`; arming makes the probe kernels resident.  CCM_ERR_NO_CUDA when there is no such CUDA device. */
int ccm_scrub_probe(int cuda_ordinal, int on);
/* The probe report of the last product call on the CUDA device (probed == 0 when it did not probe).  CCM_ERR_NO_CUDA
 * when there is no such CUDA device. */
int ccm_scrub_last_probe(int cuda_ordinal, ccm_probe_report* out);
/* P1, P2 and P3 on caller-owned memory (any alignment, any length; synchronises), with the tags of `seed`: the windows
 * are those of [dptr, dptr + bytes), no byte outside them is touched, and they hold zero afterwards.  `out` is required;
 * `mismatch` (optional) gets the mismatch report of P2 (located == 1, offsets from dptr, every record's chunk 0), and the
 * mismatch page map is replaced. */
int ccm_region_probe(int cuda_ordinal, void* dptr, uint64_t bytes, uint32_t seed, void* stream, ccm_probe_report* out,
                     ccm_mismatch_report* mismatch);

/* ---- probe proof: did every step of the alias probe take every window? ---------------------------
 * A P2 launch that skips windows reports 0 mismatches, exactly as a clean one does, so an alias in the skipped windows
 * goes unseen.  A product call that is both proven (ccm_scrub_prove) and probes (ccm_scrub_probe) runs the proving
 * twin of each probe kernel: same grids, order and number of launches, same loads and stores.  Each counts on the
 * device, per step, CCM_PROBE_WINDOW bytes for every window it took, on the 2 MiB page of va_base (the coverage
 * proof's) the window starts on.  After the probe, where the coverage proof is compared, the host copies the three
 * maps once and requires of every step: page p counted exactly CCM_PROBE_WINDOW times the probe windows of the call's
 * chunks that start on it, and the outside slot 0.  A step that missed a window, or took one twice or outside the
 * mapping, returns CCM_ERR_UNCOVERED, which takes precedence over the probe's CCM_ERR_MISMATCH and CCM_ERR_DIRTY (the
 * probe report, the mismatch report and its page map are still filled).  A call that does not probe (unproven,
 * unprobed, tagged, or whose read-back found dirt) has proved == 0 and no pages. */
typedef struct ccm_probe_cover_step {
  uint64_t windows_counted;   /* windows the step's kernels counted, the outside slot included */
  uint64_t windows_missing;   /* sum over pages of (expected - counted) where short, in windows */
  uint64_t windows_extra;     /* sum over pages of (counted - expected) where over, plus the outside slot */
  uint64_t windows_outside;   /* the outside slot: windows counted before va_base or past the last page */
  uint64_t pages_short;       /* pages that counted fewer windows than expected */
  uint64_t pages_over;        /* pages that counted more (the outside slot is not a page) */
  uint64_t first_short_page;  /* the first short page (0 when none) */
  int32_t ran;                /* 1: the call ran this step */
  int32_t reserved;
} ccm_probe_cover_step;       /* 64 B */

typedef struct ccm_probe_cover {
  uint64_t windows_expected;  /* probe windows of the call (ccm_probe_report.windows) */
  uint64_t va_base;           /* address of page 0 (the coverage proof's) */
  double ms_prove;            /* host wall-clock of the copy and the comparison */
  int32_t proved;             /* 1: the last product call was proven and probed, and its probe finished */
  int32_t covered;            /* 1: every step counted every page exactly */
  ccm_probe_cover_step step[3];   /* P1, P2, P3 */
} ccm_probe_cover;            /* 224 B */

typedef struct ccm_probe_cover_page {
  uint64_t page;              /* offset page * CCM_PAGE_BYTES from va_base */
  uint32_t chunk;             /* as ccm_cover_page.chunk */
  uint32_t expected;          /* bytes (CCM_PROBE_WINDOW per window) every step had to count on the page */
  uint32_t count[3];          /* bytes each step counted (P1, P2, P3) */
  uint32_t reserved;
} ccm_probe_cover_page;       /* 32 B */

/* The probe proof of the last product call on the CUDA device (proved == 0 when it did not run).  CCM_ERR_NO_CUDA when
 * there is no such CUDA device. */
int ccm_scrub_last_probe_cover(int cuda_ordinal, ccm_probe_cover* out);
/* One entry per page that some step did not count exactly, ascending.  Writes min(*n, cap) entries, *n = all of them.
 * CCM_ERR_NO_CUDA as above, CCM_ERR_INVALID for n == NULL, or out == NULL with cap > 0. */
int ccm_last_probe_cover_pages(int cuda_ordinal, ccm_probe_cover_page* out, uint64_t cap, uint64_t* n);

/* ---- report proof: did the locate pass and the triages of a failed call walk every byte they report on? -----------
 * The reports of a failed call run after its verdict: a T3 launch that skips a run classes its pages CLEARS where the
 * truth may be RETURNS, a T2 launch that skips one classes STAYS pages CLEARS, and a locate pass that skips part of the
 * mapping leaves pages out of the dirt page map, which the triage then never looks at.  A proven product call
 * (ccm_scrub_prove) whose read-back counted dirt (zero, tagged or census, a dirty probe P3 included), or whose tagged
 * check counted a mismatch, runs the proving twin of every kernel of its locate pass and of each triage step it runs:
 * same grids, order and number of launches.  Each counts on the device, per step, the bytes it walked on every 2 MiB
 * page from va_base (the dirt and mismatch reports').  Its steps:
 *   CCM_REPORT_LOCATE        the locate pass, over every span of what the call holds;
 *   CCM_REPORT_DIRT_T1..T3   the dirt triage's re-zero and its two re-reads, over the runs of the dirt page map;
 *   CCM_REPORT_MISMATCH_T1..T3  the mismatch triage's re-tag, check-and-zero and read for zeros, over the runs of
 *                            the mismatch page map.
 * After the locate pass, after the dirt triage and after the mismatch triage, the host copies that report's maps once
 * and requires of every step that ran: page p counted exactly the bytes of what the step walks that lie on it (the
 * locate pass: min(CCM_PAGE_BYTES, bytes - p * CCM_PAGE_BYTES); a triage step: the bytes of its runs on the page, in all
 * ccm_triage_report.bytes_examined), and the outside slot 0.  The call has already failed: a short step changes no
 * status, verdict, error text or report, and says only which pages of those reports rest on a step that missed or
 * repeated bytes.  An unproven call, and a proven one that locates and triages nothing, has proved == 0 and copies
 * nothing.  The maps (seven of one u32 per 2 MiB page and an outside slot, and a pinned host copy) are set aside with
 * the coverage proof's, when a device is first armed: a whole-HBM call has mapped everything by the time it locates. */
typedef enum ccm_report_step_id {
  CCM_REPORT_LOCATE = 1,
  CCM_REPORT_DIRT_T1 = 2,
  CCM_REPORT_DIRT_T2 = 3,
  CCM_REPORT_DIRT_T3 = 4,
  CCM_REPORT_MISMATCH_T1 = 5,
  CCM_REPORT_MISMATCH_T2 = 6,
  CCM_REPORT_MISMATCH_T3 = 7
} ccm_report_step_id;
#define CCM_REPORT_STEPS 7u

typedef struct ccm_report_cover_step {
  uint64_t launches;          /* kernels the step launched */
  uint64_t bytes_expected;    /* bytes it had to walk (the locate pass: the call's bytes; a triage step: bytes_examined) */
  uint64_t bytes_counted;     /* every byte its kernels counted, the outside slot included */
  uint64_t bytes_missing;     /* sum over pages of (expected - counted) where short */
  uint64_t bytes_extra;       /* sum over pages of (counted - expected) where over, plus the outside slot */
  uint64_t bytes_outside;     /* the outside slot: bytes counted before va_base or past the last page */
  uint64_t pages_short;       /* pages that counted fewer bytes than expected */
  uint64_t pages_over;        /* pages that counted more (the outside slot is not a page) */
  uint64_t first_short_page;  /* the first short page (0 when none) */
  int32_t ran;                /* 1: the call ran this step to its end (the rest of the row is then meaningful) */
  int32_t reserved;
} ccm_report_cover_step;      /* 80 B */

typedef struct ccm_report_cover {
  uint64_t va_base;           /* address of page 0 (the dirt and mismatch reports') */
  double ms_prove;            /* host wall-clock of the copies and the comparisons */
  int32_t proved;             /* 1: the last product call was proven and ran a locate pass or a triage */
  int32_t covered;            /* 1: every step that ran counted every page exactly */
  ccm_report_cover_step step[CCM_REPORT_STEPS];   /* indexed by ccm_report_step_id - 1 */
} ccm_report_cover;           /* 584 B */

typedef struct ccm_report_cover_page {
  uint64_t page;              /* offset page * CCM_PAGE_BYTES from va_base */
  uint32_t chunk;             /* as ccm_page_entry.chunk */
  int32_t step;               /* ccm_report_step_id */
  uint32_t expected;          /* bytes the step had to count on the page */
  uint32_t counted;           /* bytes it counted */
} ccm_report_cover_page;      /* 24 B */

/* The report proof of the last product call on the CUDA device (proved == 0 when it did not run).  CCM_ERR_NO_CUDA
 * when there is no such CUDA device. */
int ccm_scrub_last_report_cover(int cuda_ordinal, ccm_report_cover* out);
/* One entry per (step, page) that the step did not count exactly, by step, then ascending pages.  Writes min(*n, cap)
 * entries, *n = all of them.  CCM_ERR_NO_CUDA as above, CCM_ERR_INVALID for n == NULL, or out == NULL with cap > 0. */
int ccm_last_report_cover_pages(int cuda_ordinal, ccm_report_cover_page* out, uint64_t cap, uint64_t* n);

/* ---- HBM health: the GPU's own record of memory faults around the gate ------------------------------------------
 * HBM3 is ECC-protected, so the kernels never see a flipped cell: it is corrected on its way to the SM, and the gate
 * passes.  An uncorrectable error kills the call's context (CCM_ERR_CUDA) without saying it was the memory, and a row
 * that raised one is marked for remapping, which the GPU applies only at its next reset.  Only the GPU's counters record
 * such faults.  A snapshot reads them through NVML (libnvidia-ml.so.1, loaded at run time; read-only queries only),
 * with the device handle of the PCI address: the device table's bdf (ccm_hbm_snapshot), or the CUDA device's PCI bus
 * id (an armed product call).  No CUDA context is needed.  Each query that answers sets its bit in `available`; one
 * that does not leaves its fields 0 and its NVML return code in nvml_rc (NVML_ERROR_NOT_SUPPORTED = 3). */
typedef enum ccm_hbm_query {
  CCM_HBM_Q_ECC_MODE = 1,          /* nvmlDeviceGetEccMode                                              */
  CCM_HBM_Q_DRAM_CORRECTED = 2,    /* nvmlDeviceGetMemoryErrorCounter, volatile, NVML_MEMORY_LOCATION_DRAM */
  CCM_HBM_Q_DRAM_UNCORRECTED = 4,
  CCM_HBM_Q_SRAM_CORRECTED = 8,    /* likewise, NVML_MEMORY_LOCATION_SRAM                               */
  CCM_HBM_Q_SRAM_UNCORRECTED = 16,
  CCM_HBM_Q_REMAPPED_ROWS = 32,    /* nvmlDeviceGetRemappedRows                                         */
  CCM_HBM_Q_REMAP_HISTOGRAM = 64   /* nvmlDeviceGetRowRemapperHistogram                                 */
} ccm_hbm_query;
#define CCM_HBM_QUERIES 7u          /* nvml_rc[k] belongs to the query 1 << k */

typedef struct ccm_hbm_state {
  uint64_t dram_corrected;         /* volatile ECC error counts (since the driver loaded) */
  uint64_t dram_uncorrected;
  uint64_t sram_corrected;
  uint64_t sram_uncorrected;
  uint32_t ecc_current;            /* 1: ECC on; ecc_pending: what the next reset applies */
  uint32_t ecc_pending;
  uint32_t rows_corrected;         /* rows remapped for corrected / uncorrected errors */
  uint32_t rows_uncorrected;
  uint32_t remap_pending;          /* 1: a remap waits for the next reset */
  uint32_t remap_failure;          /* 1: a remap failed: the banks are out of spare rows */
  uint32_t hist_max, hist_high, hist_partial, hist_low, hist_none;   /* remapper banks by spare rows left */
  uint32_t available;              /* ccm_hbm_query bits of the queries that answered */
  int32_t nvml_rc[CCM_HBM_QUERIES]; /* NVML return code of each query (0 when it answered) */
  int32_t reserved;
  double ms_query;                 /* host time of the snapshot's NVML calls */
} ccm_hbm_state;                /* 120 B */

/* One snapshot of the GPU at device-table index `dev`.  CCM_OK when every query answered or was NOT_SUPPORTED;
 * CCM_ERR_IO when one failed otherwise (the snapshot is still filled); CCM_ERR_UNSUPPORTED when NVML cannot be loaded
 * or has no device with that bdf (available == 0).  Never changes device state. */
int ccm_hbm_snapshot(int dev, ccm_hbm_state* out);

/* Opt-in, per CUDA device: ccm_scrub_health(ordinal, mode), mode 0 off, 1 report, 2 require.  An armed product call
 * (zero, tagged or census, alone or in a fan-out, on the VMM path or the cudaMalloc fallback) takes a snapshot before
 * it maps or allocates anything, and another once its passes, reports and triages are done, before the memory goes
 * back; on every error path too, CCM_ERR_CUDA included.  It launches nothing more.  The report compares the two:
 *   UNFIT    an uncorrected DRAM or SRAM count rose during the call, a remap is pending after it, a remap failed, or
 *            ECC is off;
 *   UNKNOWN  otherwise, when a query the rule needs (ECC mode, both uncorrected counts, remapped rows) did not answer
 *            in either snapshot, or a counter went down between them (a reset in between);
 *   FIT      otherwise.  Corrected errors are reported and never make a GPU unfit.
 * Mode 2 returns CCM_ERR_HBM_HEALTH for an UNFIT or UNKNOWN report when the call would otherwise return CCM_OK,
 * CCM_ERR_UNCOVERED, CCM_ERR_MISMATCH or CCM_ERR_DIRTY (the hardware's record explains those counts); the result
 * fields and every other report are those the call left.  Any other error keeps its status.  Mode 1 never changes
 * the status.  An unarmed call reads nothing from NVML.  The "hbm_*" drills of ccm_sim_set act on the second
 * snapshot of an armed call. */
typedef enum ccm_hbm_verdict { CCM_HBM_FIT = 1, CCM_HBM_UNFIT = 2, CCM_HBM_UNKNOWN = 3 } ccm_hbm_verdict;
typedef enum ccm_hbm_reason {
  CCM_HBM_R_DRAM_UNCORRECTED = 1,  /* the uncorrected DRAM count rose during the call */
  CCM_HBM_R_SRAM_UNCORRECTED = 2,  /* the uncorrected SRAM count rose */
  CCM_HBM_R_REMAP_PENDING = 4,     /* a remap is pending: the GPU must be reset before it holds a tenant's data */
  CCM_HBM_R_REMAP_FAILURE = 8,     /* a remap failed: no spare rows left */
  CCM_HBM_R_ECC_OFF = 16,          /* ECC is off */
  CCM_HBM_R_NO_ANSWER = 32,        /* a query the rule needs did not answer (missing_queries says which) */
  CCM_HBM_R_WENT_DOWN = 64         /* a counter went down between the snapshots */
} ccm_hbm_reason;

typedef struct ccm_hbm_health {
  ccm_hbm_state before;
  ccm_hbm_state after;
  int64_t d_dram_corrected;        /* after - before */
  int64_t d_dram_uncorrected;
  int64_t d_sram_corrected;
  int64_t d_sram_uncorrected;
  double ms_health;                /* host time of both snapshots */
  int32_t mode;                    /* the arming of the call: 1 report, 2 require (0: the last call was not armed) */
  int32_t verdict;                 /* ccm_hbm_verdict (0 when not armed) */
  uint32_t reasons;                /* ccm_hbm_reason bits */
  uint32_t missing_queries;        /* ccm_hbm_query bits the rule needs that did not answer */
} ccm_hbm_health;                  /* 296 B */

/* Arms (mode 1 or 2) or disarms (0) the HBM health report for every later product call on the CUDA device.
 * CCM_ERR_INVALID for another mode, CCM_ERR_NO_CUDA when there is no such CUDA device. */
int ccm_scrub_health(int cuda_ordinal, int mode);
/* The health report of the last product call on the CUDA device (mode == 0 when it was not armed).  CCM_ERR_NO_CUDA
 * when there is no such CUDA device. */
int ccm_scrub_last_health(int cuda_ordinal, ccm_hbm_health* out);

/* -- arena: the device-resident region, held across calls (bench / tests) -- */
typedef struct ccm_arena_info {
  uint64_t bytes;              /* total bytes held                              */
  uint64_t device_total_bytes;
  uint64_t device_free_before; /* cudaMemGetInfo free before acquiring          */
  int32_t segments;
  int32_t reserved;
  double ms_acquire;
} ccm_arena_info;

int ccm_arena_acquire(int dev, uint64_t bytes, ccm_arena_info* out);
int ccm_arena_release(int dev);
/* Zero the whole arena.  *ms (optional) = CUDA-event duration on `stream`. */
int ccm_arena_scrub(int dev, int variant, const ccm_launch_cfg* cfg, void* stream, float* ms);
/* Count non-zero bytes in the whole arena (synchronises to return the count). */
int ccm_arena_verify(int dev, int variant, const ccm_launch_cfg* cfg, void* stream,
                     uint64_t* nonzero, float* ms);
/* Enqueue only (no sync): scrub then verify into the arena's device counter;
 * used inside timed regions.  Fetch the count with ccm_arena_fetch_count(). */
int ccm_arena_scrub_verify_async(int dev, int scrub_variant, int verify_variant,
                                 const ccm_launch_cfg* scrub_cfg,
                                 const ccm_launch_cfg* verify_cfg, void* stream);
int ccm_arena_fetch_count(int dev, void* stream, uint64_t* nonzero);
/* Per-step kernel durations (CUDA events recorded on the launching stream by
 * ccm_arena_scrub_verify_async, up to 64 steps since the last call); waits for
 * the recorded steps to finish, then clears the ring. */
int ccm_arena_step_times(int dev, int cap, float* scrub_ms, float* verify_ms, int* n);
/* Test scaffolding at full size: fill with a byte / a seeded xorshift pattern,
 * poke and peek host bytes at an arena offset. */
int ccm_arena_fill(int dev, int byte_value, void* stream);
int ccm_arena_fill_random(int dev, uint64_t seed, void* stream);
int ccm_arena_write(int dev, uint64_t offset, const void* host_src, uint64_t bytes);
int ccm_arena_read(int dev, uint64_t offset, void* host_dst, uint64_t bytes);

/* -- raw regions: caller-owned device memory (any alignment, any length) --- */
int ccm_region_scrub(int cuda_ordinal, void* dptr, uint64_t bytes, int variant,
                     const ccm_launch_cfg* cfg, void* stream, float* ms);
int ccm_region_verify(int cuda_ordinal, const void* dptr, uint64_t bytes, int variant,
                      const ccm_launch_cfg* cfg, void* stream, uint64_t* nonzero, float* ms);
/* The tagged gate's two kernels on caller-owned memory: write the tags of `seed`, or count the
 * bytes that differ from them (exact, synchronises) and zero the region in the same pass. */
int ccm_region_tag_fill(int cuda_ordinal, void* dptr, uint64_t bytes, uint32_t seed, void* stream, float* ms);
int ccm_region_tag_check_zero(int cuda_ordinal, void* dptr, uint64_t bytes, uint32_t seed, void* stream,
                              uint64_t* mismatch, float* ms);
/* Test entry of the proving kernels (the coverage, probe and report proofs') on caller-owned memory.  While a map is
 * armed on the CUDA device, every launch of a default-frame kernel that is not a product call's runs its proving twin
 * into `map`: ccm_region_scrub and ccm_region_verify when they resolve to the default kernel (no cfg),
 * ccm_region_tag_fill, ccm_region_tag_check_zero, ccm_region_tag_check_locate, ccm_region_census and
 * ccm_region_locate, and the arena and round-trip entries' default launches.  Results, books and written bytes are the
 * unarmed call's.  Each launch adds, for every byte it processed, one to the u32 word of the 2 MiB page
 * (address - base) / CCM_PAGE_BYTES (any base, aligned or not), or to word `pages`, the outside slot, for a byte before
 * base or on a page >= pages.  ccm_region_probe runs its three proving twins into three such maps laid end to end
 * (P1 at map, P2 at map + pages + 1, P3 at map + 2 * (pages + 1)), CCM_PROBE_WINDOW bytes per window.  The other scrub
 * and verify variants run their own kernels and count nothing; product calls keep their own maps.  The caller zeroes
 * the map and reads it back on its streams; map == NULL disarms, and so does ccm_device_release.  CCM_ERR_NO_CUDA when
 * there is no such CUDA device. */
int ccm_region_prove(int cuda_ordinal, uint32_t* map, uint64_t base, uint32_t pages);
/* Host-buffer round trip through the public path (tests, e2e): copies `bytes`
 * from host_buf to the device, counts non-zero bytes BEFORE (pre_nonzero, may be
 * NULL), scrubs, verifies, copies the region back into host_buf. */
int ccm_host_roundtrip(int cuda_ordinal, void* host_buf, uint64_t bytes, uint64_t dev_offset,
                       int scrub_variant, int verify_variant,
                       uint64_t* pre_nonzero, uint64_t* post_nonzero);

/* Drops everything the library holds on the CUDA device behind `dev` — arena, stream, events,
 * counters — and resets that device's primary context (cudaDeviceReset).  A daemon must not sit
 * on a CUDA context between transitions: the context pins ~0.5 GB of HBM, keeps the GPU "in use"
 * (it cannot be unbound for vfio) and does not survive the device reset of the next transition
 * (reference main.py:519).  Joins the background release of the last scrub first.  The next scrub
 * call re-creates what it needs.  The sysfs backend
 * calls this implicitly before it resets a device.  No-op (CCM_OK) when nothing is held. */
int ccm_device_release(int dev);
/* Concurrent form for `n` devices (one host thread each); *wall_ms = host wall-clock. */
int ccm_device_release_many(int n, const int* devs, double* wall_ms);

/* NEW: cudaMemGetInfo on a CUDA device, from the context a product call runs on.  Creates the device's engine (its
 * context, stream, books and resident kernels) exactly as a product call would when it does not exist yet, and sets
 * aside what an armed product call would set aside at its start (the probe proof's maps, when the device is armed for
 * the alias probe and the coverage proof), so that the free memory it returns is what the next product call starts
 * from.  The relayed gate (ccm-scrub --relay) reads it before and after the first leg's process ends.  CCM_ERR_NO_CUDA
 * when there is no such CUDA device. */
int ccm_device_memory(int cuda_ordinal, uint64_t* free_bytes, uint64_t* total_bytes);

/* Names of the two kernels AUTO launches, as ncu prints them, separated by ';' —
 * "scrub_st128_fast_kernel<512, 16, 0>;verify_ld128_fast_kernel<1024, 8, 2>".  Built from the
 * same compile-time constants as the launches, so tools that key measurements by kernel name
 * notice when the default changes. */
const char* ccm_default_kernels(void);

/* Number of kernels this library has launched since load (all threads). */
uint64_t ccm_kernel_launches(void);

/* ---- sim backend controls (tests, bench; no-ops on sysfs) ---------------- */
/* Rebuild a synthetic topology: n_gpus GPUs then n_switches NVSwitches. */
int ccm_sim_topology(int n_gpus, int n_switches);
/* key: "cc_mode" "ppcie_mode" "cc_supported" "ppcie_supported" "reset_ms"
 *      "boot_ms" "fail_op" (bitmask of ccm_sim_op) "stuck" (reset ignores staged)
 *      "cuda_ordinal", and three fault drills of ccm_scrub_verify (0 = off; they only ever add
 *      dirt, and only inside memory the call has mapped or allocated):
 *      "scrub_inject"  dirties that many bytes between the scrub and the read-back: the first,
 *                      byte 17, the middle + 3 and the last byte of each enqueued range (each once,
 *                      in enqueue order).  The VMM path enqueues one range per main-zone chunk and
 *                      one for all tail granules, or ONE range for the whole mapping when it maps
 *                      first; the arena path one range per segment.  So the call comes back
 *                      CCM_ERR_DIRTY with nonzero_bytes == min(value, 4 x ranges), fewer when a
 *                      range is too short for four distinct bytes;
 *      "scrub_poison"  (byte value) fills every physical chunk (arena: segment) right after it is
 *                      mapped, before any scrub — the previous tenant: the call must stay clean;
 *      "scrub_flood"   (byte value) fills every enqueued range between its scrub and its
 *                      read-back: CCM_ERR_DIRTY with nonzero_bytes == bytes_scrubbed.
 *      Three drills of the tagged calls (ccm_scrub_verify_tagged; the zero-only call ignores them):
 *      "tag_inject"    XORs that many bytes between the tag fill and the check, the same four
 *                      candidates per enqueued range as "scrub_inject": CCM_ERR_MISMATCH with
 *                      mismatch_bytes == min(value, 4 x ranges) and a clean zero read-back;
 *      "scrub_alias"   (1 = on) maps the first n0 bytes of the second main-zone chunk from the
 *                      first chunk's handle (n0 = the first chunk's size; when the second chunk
 *                      is at least that large) instead of from fresh
 *                      memory: two virtual views of one physical range, legal VMM use, no extra
 *                      memory.  The zero gate passes it; the tagged gate must not.  VMM path only
 *                      (the cudaMalloc fallback accepts the key and ignores it);
 *      "tag_flood"     (byte value) fills every range "tag_inject" acts on with that byte between the tag fill and
 *                      the check (before "tag_inject"): CCM_ERR_MISMATCH with mismatch_bytes == the mapped bytes
 *                      whose tag byte differs from the value, and a clean zero read-back.
 *      A drill for the residue census (ccm_scrub_verify_residue; it acts on every product call):
 *      "scrub_residue" zero-fills every mapping (a main-zone chunk or a tail granule, in mapping order;
 *                      arena: every segment) right after it is mapped, after "scrub_poison" and before the
 *                      gate's first write to it, then sets that many bytes to 0xA5: the first, byte 17, the
 *                      middle + 3 and the last byte of each mapping (each once, in mapping order).  The gate
 *                      erases them and stays clean; a census counts exactly those bytes, whatever the driver
 *                      handed back.
 *      Two drills of the dirt triage (ccm_scrub_triage; they act only in a call that triages):
 *      "triage_stay"   XORs the first byte of each of the first that many pages of the dirt page map with 0xA5
 *                      between the triage's re-zero (T1) and its first re-read (T2);
 *      "triage_return" XORs the same bytes between its first and second re-read (T2 and T3).
 *      In a call that triages mismatches (ccm_scrub_mismatch_triage) they act on the first pages of the mismatch
 *      page map: "triage_stay" between its re-tag (T1) and its check-and-zero (T2), "triage_return" between T2 and
 *      its read for zeros (T3).
 *      Two drills of the coverage proof (ccm_scrub_prove; they act on armed and unarmed calls alike):
 *      "cover_skip"    writes that many into the grab word of the first launch of the chosen pass, in stream order
 *                      just before it: the kernel skips the chunks it would grab first (the lowest; the read-back,
 *                      which walks down, the highest) and its last CTA still hands the word back zeroed.  It acts
 *                      only on launches of the default-frame kernels (an armed call, or the default variants);
 *      "cover_pass"    chooses the pass: 0 or 3 the read-back, 1 the first pass, 2 the tagged check.  Any other value
 *                      is CCM_ERR_INVALID.
 *      Two drills of the coverage ledger (they act on the pass "cover_pass" chooses, armed or not, and only narrow or
 *      repeat launch ranges inside what the call mapped, or drop one thread's stores or loads):
 *      "cover_repeat"  k (1..15; 0 = off): the pass's first launch whose range [a, end) starts on a page boundary of
 *                      the map ((a - va_base) % CCM_PAGE_BYTES == 0) and holds at least CCM_PAGE_BYTES is enqueued as
 *                      [a, a + CCM_PAGE_BYTES - k x 128 KiB), [a + CCM_PAGE_BYTES, end), then [a, a + k x 128 KiB)
 *                      again: page 0 counts exactly, ledger slots 0..k-1 twice and 16-k..15 not at all, so a proven
 *                      call returns CCM_ERR_UNCOVERED with ccm_cover_report.covered == 1.  Any other value is
 *                      CCM_ERR_INVALID;
 *      "cover_lane_drop" t + 1 (t = 0..511; 0 = off): in a proven call, thread t skips its share of chunk 0 (the chunk
 *                      at the range's first whole vector) of the pass's first launch, whichever CTA grabs it.  The
 *                      page map is unchanged; the ledger is PER_THREAD x 16 bytes short on that slot (256 for the
 *                      scrub, census and tag kernels, 128 for the read-back).  Any other value is CCM_ERR_INVALID.
 *      Two drills of the alias probe (ccm_scrub_probe; they act only in a call that probes):
 *      "probe_mismatch" XORs the first byte of each of the first that many probe windows (in launch order) with 0xA5
 *                      between P1 and P2: CCM_ERR_MISMATCH with mismatch_bytes == min(value, windows), PARTIAL records;
 *      "probe_dirt"    XORs the same bytes between P2 and P3: CCM_ERR_DIRTY with nonzero_bytes == min(value, windows).
 *      A drill of the probe proof (it acts in every call that probes, proven or not):
 *      "probe_skip"    the first launch of the chosen step (the first chunk with windows) starts that many windows
 *                      later and takes that many fewer (at most all of them): a proven call returns CCM_ERR_UNCOVERED
 *                      with exactly min(value, the chunk's windows) windows missing;
 *      "probe_skip_step" chooses the step: 1 (P1), 2 (P2, the default; 0 also selects it) or 3 (P3).  Any other value
 *                      is CCM_ERR_INVALID.
 *      A drill of the report proof (it acts in every call that runs the chosen step, proven or not):
 *      "report_skip"   writes that many into the grab word of the first launch of the chosen report step, in stream
 *                      order just before it, as "cover_skip" does: the kernel skips the lowest chunks of its range
 *                      (the first locate span, or the first triage run) and its last CTA hands the word back zeroed;
 *      "report_skip_step" chooses the step (ccm_report_step_id): 1..7, 0 selects CCM_REPORT_DIRT_T3 (the default).
 *                      Any other value is CCM_ERR_INVALID.
 *      Five drills of the HBM health report (ccm_scrub_health; they act only in an armed call, on its second snapshot,
 *      on top of what NVML returned):
 *      "hbm_uncorrected" adds that many to the uncorrected DRAM count;
 *      "hbm_corrected" adds that many to the corrected DRAM count;
 *      "hbm_remap_pending" (1 = on) sets remap_pending;
 *      "hbm_remap_failure" (1 = on) sets remap_failure;
 *      "hbm_unavailable" (ccm_hbm_query bits) reports those queries as not supported: fields 0, bit cleared,
 *                      nvml_rc 3.
 *      dev = -1 applies to every device. */
int ccm_sim_set(int dev, const char* key, int64_t value);
int ccm_sim_get(int dev, const char* key, int64_t* value);
typedef enum ccm_sim_op {
  CCM_OP_QUERY_CC = 1, CCM_OP_SET_CC = 2, CCM_OP_QUERY_PPCIE = 4, CCM_OP_SET_PPCIE = 8,
  CCM_OP_RESET = 16, CCM_OP_WAIT_BOOT = 32, CCM_OP_SCRUB = 64
} ccm_sim_op;
/* Ordered trace of register-level ops since the last clear: lines
 * "<seq> <bdf> <op> <arg>\n".  Returns bytes needed (excluding NUL). */
int ccm_sim_trace(char* buf, size_t cap);
int ccm_sim_trace_clear(void);

#if defined(__GNUC__)
#pragma GCC visibility pop
#endif
#ifdef __cplusplus
}
#endif
#endif /* CCM_H_ */
