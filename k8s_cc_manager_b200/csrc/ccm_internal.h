// ccm_internal.h — glue between the register backends (ccm_core.cpp) and the CUDA
// scrub engine (ccm_scrub.cu).  Nothing here crosses the public ABI (include/ccm.h).
#pragma once
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <string>

#include "ccm.h"
#include "ccm_health.h"

namespace ccm {

// thread-local detailed error text behind ccm_last_error()
void set_error(const char* fmt, ...);
const std::string& last_error();

// ---- implemented in ccm_scrub.cu ------------------------------------------
int cuda_device_count();  // 0 when no driver / no device (never throws)
int cuda_describe(int ordinal, char* bdf, size_t bdf_cap, char* name, size_t name_cap,
                  uint64_t* total_bytes);

struct ScrubEngine;  // one per CUDA ordinal, created lazily
ScrubEngine* engine_for(int ordinal);  // nullptr + error text if unusable
ScrubEngine* engine_lookup(int ordinal);  // the engine if it exists; never creates a context

int engine_arena_acquire(ScrubEngine*, uint64_t bytes, ccm_arena_info* out);
int engine_arena_release(ScrubEngine*, double* ms);
int engine_arena_scrub(ScrubEngine*, int variant, const ccm_launch_cfg*, void* stream, float* ms);
int engine_arena_verify(ScrubEngine*, int variant, const ccm_launch_cfg*, void* stream,
                        uint64_t* nonzero, float* ms);
int engine_arena_scrub_verify_async(ScrubEngine*, int sv, int vv, const ccm_launch_cfg*,
                                    const ccm_launch_cfg*, void* stream);
int engine_arena_fetch_count(ScrubEngine*, void* stream, uint64_t* nonzero);
int engine_arena_step_times(ScrubEngine*, int cap, float* scrub_ms, float* verify_ms, int* n);
int engine_arena_fill(ScrubEngine*, int byte_value, void* stream);
int engine_arena_fill_random(ScrubEngine*, uint64_t seed, void* stream);
int engine_arena_rw(ScrubEngine*, uint64_t offset, void* host, uint64_t bytes, bool write);
// Fault drills of the product call (sim keys "scrub_inject", "scrub_poison", "scrub_flood"; 0 = off).
// They only ever ADD dirt, and only inside memory the call has already mapped (or allocated):
//   inject: that many bytes are dirtied AFTER the scrub and BEFORE the read-back — first, +17,
//           middle + 3 and last byte of each enqueued range (arena path: of each segment);
//   poison: every physical chunk (arena path: segment) is filled with this byte right after it is
//           mapped, before any scrub of it — the previous tenant; the verdict must be CLEAN;
//   flood:  every enqueued range (arena path: segment) is filled with this byte between its scrub
//           and its read-back; the verdict must be DIRTY with nonzero_bytes == bytes_scrubbed.
// Drills of the tagged call (sim keys "tag_inject", "scrub_alias"; ccm.h):
//   tag_inject: that many bytes are XORed between the tag fill and the check, same candidates as inject;
//   alias:      the second main-zone chunk starts with a second view of the first chunk (VMM path only);
//   tag_flood:  every range tag_inject acts on is filled with this byte between the tag fill and the check.
// Drill of the residue census (sim key "scrub_residue"; ccm.h):
//   residue:    every mapping (arena path: segment) is zero-filled right after it is mapped (after poison), then
//               that many bytes are set to 0xA5, same candidates as inject but per mapping.
// Drills of the dirt and mismatch triages (sim keys "triage_stay", "triage_return"; ccm.h), only in a call that
// triages; each triage acts on the pages of its own page map:
//   triage_stay:   the first byte of each of the first that many pages is XORed between the triage's first step (the
//                  re-zero, or the re-tag) and its second (the first re-read, or the check-and-zero);
//   triage_return: the same bytes, between its second and third step.
// Drill of the coverage proof (sim keys "cover_skip", "cover_pass"; ccm.h), armed or not:
//   cover_skip:    that many is written into the grab word of the first default-frame launch of pass cover_pass
//                  (CCM_PASS_*; the sim key's 0 is stored as CCM_PASS_READBACK), just before it on the stream.
// Drills of the coverage ledger (sim keys "cover_repeat", "cover_lane_drop"; ccm.h), on pass cover_pass:
//   cover_repeat:    k: the first page-aligned launch of at least a page is enqueued as three, repeating k chunks;
//   cover_lane_drop: t + 1: in a proven call, thread t skips its share of chunk 0 of the first launch.
// Drills of the alias probe (sim keys "probe_mismatch", "probe_dirt"; ccm.h), only in a call that probes:
//   probe_mismatch: the first byte of each of the first that many probe windows is XORed between P1 and P2;
//   probe_dirt:     the same bytes, between P2 and P3.
// Drill of the probe proof (sim keys "probe_skip", "probe_skip_step"; ccm.h), in every call that probes:
//   probe_skip:     the first launch of step probe_skip_step (1..3 = P1..P3; the sim key's 0 is stored as 2) starts
//                   that many windows later and takes that many fewer (at most all of its windows).
// Drill of the report proof (sim keys "report_skip", "report_skip_step"; ccm.h), armed or not:
//   report_skip:    that many is written into the grab word of the first launch of report step report_skip_step
//                   (CCM_REPORT_*; the sim key's 0 is stored as CCM_REPORT_DIRT_T3), just before it on the stream.
// Drills of the HBM health report (sim keys "hbm_uncorrected", "hbm_corrected", "hbm_remap_pending",
// "hbm_remap_failure", "hbm_unavailable"; ccm.h), only in an armed call: layered on its second snapshot
// (ccm_health::layer).
struct ScrubDrill {
  uint64_t inject = 0;
  int poison = 0;
  int flood = 0;
  uint64_t tag_inject = 0;
  int alias = 0;
  uint64_t residue = 0;
  uint64_t triage_stay = 0;
  uint64_t triage_return = 0;
  int tag_flood = 0;
  uint64_t cover_skip = 0;
  int cover_pass = CCM_PASS_READBACK;
  uint32_t cover_repeat = 0;
  uint32_t cover_lane_drop = 0;
  uint64_t probe_mismatch = 0;
  uint64_t probe_dirt = 0;
  uint64_t probe_skip = 0;
  int probe_skip_step = 2;
  uint64_t report_skip = 0;
  int report_skip_step = CCM_REPORT_DIRT_T3;
  ccm_health::Drills hbm;
};
// inject: the call's "scrub_inject" budget.  Its poison and flood drills are those current_scrub_drill()
// returns on the calling thread.  (The engine entry points keep the signatures that host-only builds of
// ccm_core.cpp stub, tests/native/no_cuda_stub.cpp.)
// node_fanout: the call is one of several running concurrently in THIS process (ccm_scrub_verify_many).
int engine_scrub_verify(ScrubEngine*, uint64_t bytes, uint64_t inject, bool node_fanout, ccm_scrub_result* out);
// Joins the background release of the last product call (no-op when none is pending).
int engine_release_wait(ScrubEngine*, double* ms_release, double* ms_waited);
int engine_region_scrub(ScrubEngine*, void* dptr, uint64_t bytes, int variant,
                        const ccm_launch_cfg*, void* stream, float* ms);
int engine_region_verify(ScrubEngine*, const void* dptr, uint64_t bytes, int variant,
                         const ccm_launch_cfg*, void* stream, uint64_t* nonzero, float* ms);
int engine_host_roundtrip(ScrubEngine*, void* host_buf, uint64_t bytes, uint64_t dev_offset,
                          int sv, int vv, uint64_t* pre, uint64_t* post);
uint64_t kernel_launches();
const char* default_kernel_names();
// Tears down the engine of a CUDA ordinal (if any) and resets its primary context.
int engine_teardown(int ordinal);

// ---- implemented in ccm_core.cpp -------------------------------------------
// One HBM health snapshot of the GPU at PCI address `bus_id` through NVML (include/ccm.h: ccm_hbm_state).
int hbm_snapshot_bus(const char* bus_id, ccm_hbm_state* out);
// Maps a device-table index to its CUDA ordinal (or a negative ccm_status).
int cuda_ordinal_of(int dev);
// sim fault hook for the scrub op (returns CCM_OK or CCM_ERR_FAULT) + trace line; *drill = the
// device's scrub drills (all off on the sysfs backend).
int sim_scrub_hook(int dev, ScrubDrill* drill);
// The drills of the product call running on this thread (all off outside such a call): the product
// call is synchronous, one host thread per device call, so the thread identifies the call.
const ScrubDrill& current_scrub_drill();
// The tag block of the tagged product call running on this thread (its seed already drawn), or nullptr
// for the zero-only call.  The engine writes the call's mismatch count and kernel times into it.
ccm_tag_result* current_tag_call();
// The residue report of the census call running on this thread, or nullptr for a call without the census.  The
// engine fills it.
ccm_residue_report* current_residue_call();

}  // namespace ccm
