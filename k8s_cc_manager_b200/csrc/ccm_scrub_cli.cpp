// ccm-scrub — native command-line front end of the HBM scrub gate (links libccm.so).
//
//   ccm-scrub [--bytes N] [--backend sim|cudasim|sysfs] [--check zero|tagged] [--residue] [--triage]
//             [--mismatch-triage] [--triage-hold-ms MS] [--prove] [--probe] [--health report|require]
//             (--all | --bdf <pci address> ...)
//
// Runs the concurrent gate (ccm_scrub_verify_many, or ccm_scrub_verify_many_tagged with --check tagged)
// and prints ONE JSON line with the same fields as k8s_cc_manager_b200.devices.ScrubReport (the
// tagged-gate fields only with --check tagged, "dirt" only for a GPU whose read-back found non-zero bytes: where
// they are, as ccm_scrub_last_dirt reports it; "mismatch" only for a GPU whose tagged check found bytes off their
// tags, as ccm_scrub_last_mismatch reports it; "residue" for every GPU with --residue, which runs the census
// calls, ccm_scrub_verify_many_residue; each of the three with a "pages" member, the digest of its page map from
// ccm_last_page_map; "triage" with --triage, which arms every GPU for the dirt triage (ccm_scrub_triage), for a GPU whose
// read-back found non-zero bytes: what kind of dirt, as ccm_scrub_last_triage and ccm_last_triage_pages report it;
// "mismatch_triage" with --mismatch-triage, which needs --check tagged and arms every GPU for the mismatch triage
// (ccm_scrub_mismatch_triage), for a GPU whose tagged check found bytes off their tags: what kind of mismatch, as
// ccm_scrub_last_mismatch_triage and ccm_last_mismatch_triage_pages report it; "cover" with --prove, which arms every
// GPU for the coverage proof (ccm_scrub_prove), for every GPU whose passes finished, as ccm_scrub_last_cover and
// ccm_last_cover_pages report it; "probe" with --probe, which refuses --check tagged and arms every GPU for the alias
// probe (ccm_scrub_probe), for every GPU whose probe ran, as ccm_scrub_last_probe reports it, with "mismatch" when it
// found bytes off their tags); "probe_cover" with --prove and --probe, for every GPU whose probe ran, as
// ccm_scrub_last_probe_cover and ccm_last_probe_cover_pages report it; "cover_ledger" with --prove, for every GPU whose
// passes finished, as ccm_scrub_last_ledger and ccm_last_ledger_slots report it; "report_cover" with --prove, for every GPU that
// located dirt or triaged, as ccm_scrub_last_report_cover and ccm_last_report_cover_pages report it; "hbm_health" with
// --health report or --health require, which arms every GPU for the HBM health report (ccm_scrub_health), as
// ccm_scrub_last_health reports it (under require, a GPU armed and without one gets CCM_ERR_HBM_HEALTH).  With --prove,
// --probe or --health, a GPU that cannot be armed is never scrubbed without: nothing is scrubbed and the exit code is 3.
//
// --relay (whole-HBM only: it refuses --bytes other than 0) runs the gate twice, so that it also reaches the memory the
// first gate's own CUDA context held (DESIGN.md §5n).  Before this process creates any context it starts leg A, its own
// binary with --relay-first and the same options, fork + exec, stdin and stdout pipes to this process, killed when this
// process dies and ending when its stdin closes.  A runs the gate exactly as a plain call does, prints the same line,
// gives its HBM back (ccm_scrub_release_wait; its contexts stay), prints one "released" line and waits.  This process
// then creates its engine on every GPU and arms it as A was armed, reads each GPU's free memory (ccm_device_memory),
// closes A's stdin, reaps A, waits for the free memory to settle (ccm_relay.h), and runs leg B, the same gate: one JSON
// line whose reports are leg B's, each with a "relay" object (ccm_relay::account), then "first", A's line verbatim, and
// "first_pid".  When A fails or dies there is no leg B: A's line is printed as this call's, each report with
// "relay": null, and the exit code is 3.  --relay-mark-mib N (a drill) has A hold N MiB of 0xA5 from its release until it
// exits, a stand-in for a context footprint with a known content.
// Exit 0: every GPU clean (with --relay: both legs, and every GPU's relay computed); 3: gate failed;
// 2: usage.  Used by the manager for CC_SCRUB_ISOLATION=process (no Python start-up in the
// child) and usable from the legacy shell engine (reference scripts/cc-manager.sh) as a
// post-reset step.
#include <fcntl.h>
#include <sys/prctl.h>
#include <sys/wait.h>
#include <unistd.h>

#include <cerrno>
#include <chrono>
#include <csignal>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <map>
#include <string>
#include <thread>
#include <vector>

#include "ccm.h"
#include "ccm_relay.h"

// The "hbm_health" object: the fields of k8s_cc_manager_b200.devices.HbmHealth.
static void print_snapshot(const char* key, const ccm_hbm_state& s) {
  printf("\"%s\": {\"dram_corrected\": %llu, \"dram_uncorrected\": %llu, \"sram_corrected\": %llu, "
         "\"sram_uncorrected\": %llu, \"ecc_current\": %u, \"ecc_pending\": %u, \"rows_corrected\": %u, "
         "\"rows_uncorrected\": %u, \"remap_pending\": %u, \"remap_failure\": %u, \"hist_max\": %u, \"hist_high\": %u, "
         "\"hist_partial\": %u, \"hist_low\": %u, \"hist_none\": %u, \"available\": %u, \"nvml_rc\": [",
         key, (unsigned long long)s.dram_corrected, (unsigned long long)s.dram_uncorrected,
         (unsigned long long)s.sram_corrected, (unsigned long long)s.sram_uncorrected, s.ecc_current, s.ecc_pending,
         s.rows_corrected, s.rows_uncorrected, s.remap_pending, s.remap_failure, s.hist_max, s.hist_high, s.hist_partial,
         s.hist_low, s.hist_none, s.available);
  for (unsigned k = 0; k < CCM_HBM_QUERIES; ++k) printf("%s%d", k ? ", " : "", s.nvml_rc[k]);
  printf("], \"ms_query\": %.3f}", s.ms_query);
}

static void print_names(uint32_t bits, const char* const* names, unsigned n) {
  printf("[");
  for (unsigned k = 0, first = 1; k < n; ++k)
    if (bits >> k & 1) { printf("%s\"%s\"", first ? "" : ", ", names[k]); first = 0; }
  printf("]");
}

static void print_health(const ccm_hbm_health& h) {
  static const char* const kQueries[CCM_HBM_QUERIES] = {"ecc_mode", "dram_corrected", "dram_uncorrected", "sram_corrected",
                                                        "sram_uncorrected", "remapped_rows", "remap_histogram"};
  static const char* const kReasons[7] = {"dram_uncorrected", "sram_uncorrected", "remap_pending", "remap_failure",
                                          "ecc_off", "no_answer", "went_down"};
  printf(", \"hbm_health\": {");
  print_snapshot("before", h.before);
  printf(", ");
  print_snapshot("after", h.after);
  printf(", \"d_dram_corrected\": %lld, \"d_dram_uncorrected\": %lld, \"d_sram_corrected\": %lld, "
         "\"d_sram_uncorrected\": %lld, \"ms_health\": %.3f, \"mode\": %d, \"verdict\": %d, \"reasons\": ",
         (long long)h.d_dram_corrected, (long long)h.d_dram_uncorrected, (long long)h.d_sram_corrected,
         (long long)h.d_sram_uncorrected, h.ms_health, h.mode, h.verdict);
  print_names(h.reasons, kReasons, 7);
  printf(", \"missing_queries\": ");
  print_names(h.missing_queries, kQueries, CCM_HBM_QUERIES);
  printf("}");
}

// The "triage" object: the fields of k8s_cc_manager_b200.devices.TriageReport, with the first 64 pages that did not clear
// (devices.TRIAGE_PAGES).
static void print_triage(const ccm_triage_report& t, int ordinal) {
  static const char* const classes[] = {"?", "stays", "returns", "clears"};
  printf(", \"triage\": {\"pages_examined\": %llu, \"bytes_examined\": %llu, \"stay_pages\": %llu, \"stay_bytes\": %llu, "
         "\"return_pages\": %llu, \"return_bytes\": %llu, \"clear_pages\": %llu, \"clear_bytes\": %llu, \"t2_bytes\": %llu, "
         "\"t3_bytes\": %llu, \"t2_first_offset\": %llu, \"t2_last_offset\": %llu, \"t3_first_offset\": %llu, "
         "\"t3_last_offset\": %llu, \"va_base\": %llu, \"ms_hold\": %.3f, \"ms_triage\": %.3f, \"hold_ms\": %u, \"runs\": %d, "
         "\"triaged\": %d, \"suspect_pages\": [",
         (unsigned long long)t.pages_examined, (unsigned long long)t.bytes_examined, (unsigned long long)t.stay_pages,
         (unsigned long long)t.stay_bytes, (unsigned long long)t.return_pages, (unsigned long long)t.return_bytes,
         (unsigned long long)t.clear_pages, (unsigned long long)t.clear_bytes, (unsigned long long)t.t2_bytes,
         (unsigned long long)t.t3_bytes, (unsigned long long)t.t2_first_offset, (unsigned long long)t.t2_last_offset,
         (unsigned long long)t.t3_first_offset, (unsigned long long)t.t3_last_offset, (unsigned long long)t.va_base,
         t.ms_hold, t.ms_triage, t.hold_ms, t.runs, t.triaged);
  uint64_t n = 0;
  std::vector<ccm_triage_page> v;
  if (ccm_last_triage_pages(ordinal, nullptr, 0, &n) == CCM_OK) {
    v.resize(n);
    if (n && ccm_last_triage_pages(ordinal, v.data(), n, &n) != CCM_OK) v.clear();
  }
  const size_t keep = 64;   // k8s_cc_manager_b200.devices.TRIAGE_PAGES
  size_t shown = 0, suspect = 0;
  for (const ccm_triage_page& p : v) {
    if (p.cls == CCM_TRIAGE_CLEARS) continue;
    if (suspect++ >= keep) continue;
    printf("%s{\"page\": %llu, \"chunk\": %u, \"cls\": \"%s\", \"dirt_bytes\": %u, \"t2_bytes\": %u, \"t3_bytes\": %u}",
           shown++ ? ", " : "", (unsigned long long)p.page, p.chunk, classes[p.cls <= 3 ? p.cls : 0], p.dirt_bytes,
           p.t2_bytes, p.t3_bytes);
  }
  printf("], \"suspect_truncated\": %d}", suspect > keep);
}

// The value of a report's "pages" member: null when it booked no window, else the fields of
// k8s_cc_manager_b200.devices.PageDigest, from ccm_last_page_map: page count, exact bytes and pages per chunk, and the
// first 64 runs of consecutive pages in one chunk.
static void print_pages(int ordinal, int book, uint64_t windows) {
  uint64_t n = 0;
  std::vector<ccm_page_entry> v;
  if (windows == 0 || ccm_last_page_map(ordinal, book, nullptr, 0, &n) != CCM_OK) { printf("null"); return; }
  v.resize(n);
  if (n && ccm_last_page_map(ordinal, book, v.data(), n, &n) != CCM_OK) { printf("null"); return; }
  struct Run { uint64_t first, pages, bytes; uint32_t chunk; };
  std::vector<Run> runs;
  std::map<uint32_t, std::pair<uint64_t, uint64_t>> chunks;   // chunk -> (pages, bytes)
  uint64_t bytes = 0;
  for (const ccm_page_entry& p : v) {
    bytes += p.bytes;
    chunks[p.chunk].first += 1;
    chunks[p.chunk].second += p.bytes;
    if (!runs.empty() && runs.back().chunk == p.chunk && runs.back().first + runs.back().pages == p.page) {
      runs.back().pages += 1;
      runs.back().bytes += p.bytes;
    } else {
      runs.push_back({p.page, 1, p.bytes, p.chunk});
    }
  }
  const size_t keep = 64;   // k8s_cc_manager_b200.devices.PAGE_RUNS
  printf("{\"pages\": %llu, \"bytes\": %llu, \"nruns\": %llu, \"runs_truncated\": %d, \"by_chunk\": [",
         (unsigned long long)v.size(), (unsigned long long)bytes, (unsigned long long)runs.size(), runs.size() > keep);
  bool sep = false;
  for (const auto& c : chunks) {
    printf("%s{\"chunk\": %u, \"pages\": %llu, \"bytes\": %llu}", sep ? ", " : "", c.first,
           (unsigned long long)c.second.first, (unsigned long long)c.second.second);
    sep = true;
  }
  printf("], \"runs\": [");
  for (size_t k = 0; k < runs.size() && k < keep; ++k)
    printf("%s{\"first_page\": %llu, \"pages\": %llu, \"chunk\": %u, \"bytes\": %llu}", k ? ", " : "",
           (unsigned long long)runs[k].first, (unsigned long long)runs[k].pages, runs[k].chunk,
           (unsigned long long)runs[k].bytes);
  printf("]}");
}

// The "dirt" object: the fields of k8s_cc_manager_b200.devices.DirtReport, records with their bytes in hex.
static void print_dirt(const ccm_dirt_report& d, int ordinal) {
  printf(", \"dirt\": {\"nonzero_bytes\": %llu, \"dirty_windows\": %llu, \"first_offset\": %llu, \"last_offset\": %llu, "
         "\"va_base\": %llu, \"ms_locate\": %.3f, \"located\": %d, \"truncated\": %d, \"records\": [",
         (unsigned long long)d.nonzero_bytes, (unsigned long long)d.dirty_windows, (unsigned long long)d.first_offset,
         (unsigned long long)d.last_offset, (unsigned long long)d.va_base, d.ms_locate, d.located, d.truncated);
  for (int k = 0; k < d.nrecords; ++k) {
    const ccm_dirt_record& w = d.records[k];
    printf("%s{\"offset\": %lld, \"chunk\": %u, \"mask\": %u, \"bytes\": \"", k ? ", " : "", (long long)w.offset,
           w.chunk, (unsigned)w.mask);
    for (int b = 0; b < 16; ++b) printf("%02x", w.bytes[b]);
    printf("\"}");
  }
  printf("], \"pages\": ");
  print_pages(ordinal, CCM_BOOK_DIRT, d.dirty_windows);
  printf("}");
}

// The "mismatch" object: the fields of k8s_cc_manager_b200.devices.MismatchReport, kinds by name.
static void print_mismatch(const ccm_mismatch_report& m, int ordinal) {
  static const char* const kinds[] = {"?", "zero", "alias", "partial", "foreign"};
  printf(", \"mismatch\": {\"mismatch_bytes\": %llu, \"mismatch_windows\": %llu, \"zero_windows\": %llu, "
         "\"first_offset\": %llu, \"last_offset\": %llu, \"va_base\": %llu, \"seed\": %u, \"located\": %d, "
         "\"truncated\": %d, \"records\": [",
         (unsigned long long)m.mismatch_bytes, (unsigned long long)m.mismatch_windows, (unsigned long long)m.zero_windows,
         (unsigned long long)m.first_offset, (unsigned long long)m.last_offset, (unsigned long long)m.va_base, m.seed,
         m.located, m.truncated);
  for (int k = 0; k < m.nrecords; ++k) {
    const ccm_mismatch_record& w = m.records[k];
    printf("%s{\"offset\": %lld, \"chunk\": %u, \"mask\": %u, \"kind\": \"%s\", \"source_offset\": %lld, "
           "\"source_chunk\": %u, \"bytes\": \"", k ? ", " : "", (long long)w.offset, w.chunk, (unsigned)w.mask,
           kinds[w.kind <= 4 ? w.kind : 0], (long long)w.source_offset, w.source_chunk);
    for (int b = 0; b < 16; ++b) printf("%02x", w.bytes[b]);
    printf("\"}");
  }
  printf("], \"pages\": ");
  print_pages(ordinal, CCM_BOOK_MISMATCH, m.mismatch_windows);
  printf("}");
}

// The "residue" object: the fields of k8s_cc_manager_b200.devices.ResidueReport (no bytes: there are none).
static void print_residue(const ccm_residue_report& r, int ordinal) {
  printf(", \"residue\": {\"residue_bytes\": %llu, \"residue_windows\": %llu, \"first_offset\": %llu, "
         "\"last_offset\": %llu, \"bytes_examined\": %llu, \"va_base\": %llu, \"located\": %d, \"truncated\": %d, "
         "\"records\": [",
         (unsigned long long)r.residue_bytes, (unsigned long long)r.residue_windows, (unsigned long long)r.first_offset,
         (unsigned long long)r.last_offset, (unsigned long long)r.bytes_examined, (unsigned long long)r.va_base,
         r.located, r.truncated);
  for (int k = 0; k < r.nrecords; ++k) {
    const ccm_residue_record& w = r.records[k];
    printf("%s{\"offset\": %lld, \"chunk\": %u, \"mask\": %u}", k ? ", " : "", (long long)w.offset, w.chunk,
           (unsigned)w.mask);
  }
  printf("], \"pages\": ");
  print_pages(ordinal, CCM_BOOK_RESIDUE, r.residue_windows);
  printf("}");
}

// The "cover" object: the fields of k8s_cc_manager_b200.devices.CoverReport, with the first 64 inexact pages.
static void print_cover(const ccm_cover_report& c, int ordinal) {
  static const char* const names[3] = {"first", "check", "readback"};
  printf(", \"cover\": {\"bytes_mapped\": %llu, \"pages_mapped\": %llu, \"va_base\": %llu, \"ms_prove\": %.3f, "
         "\"proved\": %d, \"covered\": %d, \"passes\": [",
         (unsigned long long)c.bytes_mapped, (unsigned long long)c.pages_mapped, (unsigned long long)c.va_base, c.ms_prove,
         c.proved, c.covered);
  for (int k = 0; k < 3; ++k) {
    const ccm_cover_pass& p = c.pass[k];
    printf("%s{\"name\": \"%s\", \"ran\": %d, \"bytes_counted\": %llu, \"bytes_missing\": %llu, \"bytes_extra\": %llu, "
           "\"bytes_outside\": %llu, \"pages_short\": %llu, \"pages_over\": %llu, \"first_short_page\": %llu}",
           k ? ", " : "", names[k], p.ran, (unsigned long long)p.bytes_counted, (unsigned long long)p.bytes_missing,
           (unsigned long long)p.bytes_extra, (unsigned long long)p.bytes_outside, (unsigned long long)p.pages_short,
           (unsigned long long)p.pages_over, (unsigned long long)p.first_short_page);
  }
  printf("], \"pages\": [");
  uint64_t n = 0;
  std::vector<ccm_cover_page> v;
  if (!c.covered && ccm_last_cover_pages(ordinal, nullptr, 0, &n) == CCM_OK) {
    v.resize(n);
    if (n && ccm_last_cover_pages(ordinal, v.data(), n, &n) != CCM_OK) v.clear();
  }
  const size_t keep = 64;   // k8s_cc_manager_b200.devices.COVER_PAGES
  for (size_t k = 0; k < v.size() && k < keep; ++k)
    printf("%s{\"page\": %llu, \"chunk\": %u, \"expected\": %u, \"first\": %u, \"check\": %u, \"readback\": %u}",
           k ? ", " : "", (unsigned long long)v[k].page, v[k].chunk, v[k].expected, v[k].count[0], v[k].count[1],
           v[k].count[2]);
  printf("], \"pages_truncated\": %d}", v.size() > keep);
}

// The "mismatch_triage" object: the fields of k8s_cc_manager_b200.devices.TriageReport for the mismatch page map, with
// the first 64 pages that did not clear (devices.TRIAGE_PAGES).
static void print_mismatch_triage(const ccm_triage_report& t, int ordinal) {
  static const char* const classes[] = {"?", "stays", "returns", "clears"};
  printf(", \"mismatch_triage\": {\"pages_examined\": %llu, \"bytes_examined\": %llu, \"stay_pages\": %llu, "
         "\"stay_bytes\": %llu, \"return_pages\": %llu, \"return_bytes\": %llu, \"clear_pages\": %llu, "
         "\"clear_bytes\": %llu, \"t2_bytes\": %llu, \"t3_bytes\": %llu, \"t2_first_offset\": %llu, "
         "\"t2_last_offset\": %llu, \"t3_first_offset\": %llu, \"t3_last_offset\": %llu, \"va_base\": %llu, "
         "\"ms_hold\": %.3f, \"ms_triage\": %.3f, \"hold_ms\": %u, \"runs\": %d, \"triaged\": %d, \"suspect_pages\": [",
         (unsigned long long)t.pages_examined, (unsigned long long)t.bytes_examined, (unsigned long long)t.stay_pages,
         (unsigned long long)t.stay_bytes, (unsigned long long)t.return_pages, (unsigned long long)t.return_bytes,
         (unsigned long long)t.clear_pages, (unsigned long long)t.clear_bytes, (unsigned long long)t.t2_bytes,
         (unsigned long long)t.t3_bytes, (unsigned long long)t.t2_first_offset, (unsigned long long)t.t2_last_offset,
         (unsigned long long)t.t3_first_offset, (unsigned long long)t.t3_last_offset, (unsigned long long)t.va_base,
         t.ms_hold, t.ms_triage, t.hold_ms, t.runs, t.triaged);
  uint64_t n = 0;
  std::vector<ccm_triage_page> v;
  if (ccm_last_mismatch_triage_pages(ordinal, nullptr, 0, &n) == CCM_OK) {
    v.resize(n);
    if (n && ccm_last_mismatch_triage_pages(ordinal, v.data(), n, &n) != CCM_OK) v.clear();
  }
  const size_t keep = 64;   // k8s_cc_manager_b200.devices.TRIAGE_PAGES
  size_t shown = 0, suspect = 0;
  for (const ccm_triage_page& p : v) {
    if (p.cls == CCM_TRIAGE_CLEARS) continue;
    if (suspect++ >= keep) continue;
    printf("%s{\"page\": %llu, \"chunk\": %u, \"cls\": \"%s\", \"dirt_bytes\": %u, \"t2_bytes\": %u, \"t3_bytes\": %u}",
           shown++ ? ", " : "", (unsigned long long)p.page, p.chunk, classes[p.cls <= 3 ? p.cls : 0], p.dirt_bytes,
           p.t2_bytes, p.t3_bytes);
  }
  printf("], \"suspect_truncated\": %d}", suspect > keep);
}

static int usage(const char* argv0) {
  fprintf(stderr, "usage: %s [--bytes N] [--backend sim|cudasim|sysfs] [--check zero|tagged] [--residue] "
          "[--triage] [--mismatch-triage] [--triage-hold-ms MS] [--prove] [--probe] [--health report|require] "
          "[--relay [--relay-mark-mib N]] (--all | --bdf <bdf> ...)\n", argv0);
  return 2;
}

// The "cover_ledger" object: the fields of k8s_cc_manager_b200.devices.CoverLedger, with the first 64 inexact slots.
static void print_ledger(const ccm_cover_ledger& l, int ordinal) {
  static const char* const names[3] = {"first", "check", "readback"};
  printf(", \"cover_ledger\": {\"bytes_mapped\": %llu, \"slots_mapped\": %llu, \"va_base\": %llu, \"ms_ledger\": %.3f, "
         "\"proved\": %d, \"exact\": %d, \"passes\": [",
         (unsigned long long)l.bytes_mapped, (unsigned long long)l.slots_mapped, (unsigned long long)l.va_base,
         l.ms_ledger, l.proved, l.exact);
  for (int k = 0; k < 3; ++k) {
    const ccm_ledger_pass& p = l.pass[k];
    printf("%s{\"name\": \"%s\", \"ran\": %d, \"slots_short\": %llu, \"slots_over\": %llu, \"bytes_missing\": %llu, "
           "\"bytes_extra\": %llu, \"bytes_outside\": %llu, \"first_short_slot\": %llu, \"first_over_slot\": %llu}",
           k ? ", " : "", names[k], p.ran, (unsigned long long)p.slots_short, (unsigned long long)p.slots_over,
           (unsigned long long)p.bytes_missing, (unsigned long long)p.bytes_extra, (unsigned long long)p.bytes_outside,
           (unsigned long long)p.first_short_slot, (unsigned long long)p.first_over_slot);
  }
  printf("], \"slots\": [");
  uint64_t n = 0;
  std::vector<ccm_ledger_slot> v;
  if (!l.exact && ccm_last_ledger_slots(ordinal, nullptr, 0, &n) == CCM_OK) {
    v.resize(n);
    if (n && ccm_last_ledger_slots(ordinal, v.data(), n, &n) != CCM_OK) v.clear();
  }
  const size_t keep = 64;   // k8s_cc_manager_b200.devices.LEDGER_SLOTS
  for (size_t k = 0; k < v.size() && k < keep; ++k)
    printf("%s{\"slot\": %llu, \"chunk\": %u, \"expected\": %u, \"first\": %u, \"check\": %u, \"readback\": %u}",
           k ? ", " : "", (unsigned long long)v[k].slot, v[k].chunk, v[k].expected, v[k].count[0], v[k].count[1],
           v[k].count[2]);
  printf("], \"slots_truncated\": %d}", v.size() > keep);
}

// The "report_cover" object: the fields of k8s_cc_manager_b200.devices.ReportCoverReport, with the first 64 inexact
// (step, page) entries.
static void print_rcover(const ccm_report_cover& c, int ordinal) {
  static const char* const names[CCM_REPORT_STEPS] = {"LOCATE",      "DIRT_T1",     "DIRT_T2",    "DIRT_T3",
                                                      "MISMATCH_T1", "MISMATCH_T2", "MISMATCH_T3"};
  printf(", \"report_cover\": {\"va_base\": %llu, \"ms_prove\": %.3f, \"proved\": %d, \"covered\": %d, \"steps\": [",
         (unsigned long long)c.va_base, c.ms_prove, c.proved, c.covered);
  for (unsigned k = 0; k < CCM_REPORT_STEPS; ++k) {
    const ccm_report_cover_step& p = c.step[k];
    printf("%s{\"name\": \"%s\", \"ran\": %d, \"launches\": %llu, \"bytes_expected\": %llu, \"bytes_counted\": %llu, "
           "\"bytes_missing\": %llu, \"bytes_extra\": %llu, \"bytes_outside\": %llu, \"pages_short\": %llu, "
           "\"pages_over\": %llu, \"first_short_page\": %llu}",
           k ? ", " : "", names[k], p.ran, (unsigned long long)p.launches, (unsigned long long)p.bytes_expected,
           (unsigned long long)p.bytes_counted, (unsigned long long)p.bytes_missing, (unsigned long long)p.bytes_extra,
           (unsigned long long)p.bytes_outside, (unsigned long long)p.pages_short, (unsigned long long)p.pages_over,
           (unsigned long long)p.first_short_page);
  }
  printf("], \"pages\": [");
  uint64_t n = 0;
  std::vector<ccm_report_cover_page> v;
  if (!c.covered && ccm_last_report_cover_pages(ordinal, nullptr, 0, &n) == CCM_OK) {
    v.resize(n);
    if (n && ccm_last_report_cover_pages(ordinal, v.data(), n, &n) != CCM_OK) v.clear();
  }
  const size_t keep = 64;   // k8s_cc_manager_b200.devices.COVER_PAGES
  for (size_t k = 0; k < v.size() && k < keep; ++k) {
    const int step = v[k].step >= 1 && v[k].step <= (int)CCM_REPORT_STEPS ? v[k].step : 1;
    printf("%s{\"page\": %llu, \"chunk\": %u, \"step\": \"%s\", \"expected\": %u, \"counted\": %u}", k ? ", " : "",
           (unsigned long long)v[k].page, v[k].chunk, names[step - 1], v[k].expected, v[k].counted);
  }
  printf("], \"pages_truncated\": %d}", v.size() > keep);
}

// The "probe" object: the fields of k8s_cc_manager_b200.devices.ProbeReport.
static void print_probe(const ccm_probe_report& p) {
  printf(", \"probe\": {\"windows\": %llu, \"bytes_probed\": %llu, \"mismatch_bytes\": %llu, \"mismatch_windows\": %llu, "
         "\"reread_nonzero_bytes\": %llu, \"seed\": %u, \"launches\": %u, \"va_base\": %llu, \"ms_probe\": %.3f, "
         "\"probed\": %d}",
         (unsigned long long)p.windows, (unsigned long long)p.bytes_probed, (unsigned long long)p.mismatch_bytes,
         (unsigned long long)p.mismatch_windows, (unsigned long long)p.reread_nonzero_bytes, p.seed, p.launches,
         (unsigned long long)p.va_base, p.ms_probe, p.probed);
}

static void print_pcover(const ccm_probe_cover& c, int ordinal);   // after main

// The gate one call runs, in a plain call and in each leg of a relay: its options and its GPUs.
struct GateArgs {
  unsigned long long bytes = 0;
  bool tagged = false, residue = false, triage = false, mismatch_triage = false, prove = false, probe = false;
  unsigned long triage_hold_ms = 100;   // k8s_cc_manager_b200.devices.TRIAGE_HOLD_MS
  int health = 0;                       // ccm_scrub_health's mode: 0 off, 1 report, 2 require
  std::vector<int> devs, ordinals;
  std::vector<std::string> names;
};

// What the relay's second leg adds to that sequence: `armed` runs once every GPU is armed, before the gate (false: the
// gate does not run), `report` prints more members of report i, `tail` more members after "reports".
struct GateHooks {
  std::function<bool()> armed;
  std::function<void(size_t, const ccm_scrub_result&)> report;
  std::function<void()> tail;
};

static int run_gate(const GateArgs& g, const GateHooks& hooks, std::vector<ccm_scrub_result>& res);   // after main
static int relay_first(const GateArgs& g, unsigned long mark_mib);                                       // after main
static int relay(const GateArgs& g, int argc, char** argv);                                              // after main

int main(int argc, char** argv) {
  std::vector<std::string> bdfs;
  unsigned long long bytes = 0;
  bool all = false, tagged = false, residue = false, triage = false, mismatch_triage = false, prove = false,
       probe = false, relay_on = false, relay_first_on = false;
  unsigned long triage_hold_ms = 100;   // k8s_cc_manager_b200.devices.TRIAGE_HOLD_MS
  int health = 0;                       // ccm_scrub_health's mode: 0 off, 1 report, 2 require
  unsigned long mark_mib = 0;           // --relay-mark-mib
  for (int i = 1; i < argc; ++i) {
    std::string a = argv[i];
    if (a == "--all") all = true;
    else if (a == "--residue") residue = true;
    else if (a == "--triage") triage = true;
    else if (a == "--mismatch-triage") mismatch_triage = true;
    else if (a == "--prove") prove = true;
    else if (a == "--probe") probe = true;
    else if (a == "--relay") relay_on = true;
    else if (a == "--relay-first") relay_first_on = true;
    else if (a == "--relay-mark-mib" && i + 1 < argc) {
      mark_mib = strtoul(argv[++i], nullptr, 10);
      if (mark_mib == 0) return usage(argv[0]);
    }
    else if (a == "--triage-hold-ms" && i + 1 < argc) {
      triage_hold_ms = strtoul(argv[++i], nullptr, 10);
      if (triage_hold_ms == 0 || triage_hold_ms > CCM_TRIAGE_MAX_HOLD_MS) return usage(argv[0]);
    }
    else if (a == "--health" && i + 1 < argc) {
      std::string h = argv[++i];
      if (h != "off" && h != "report" && h != "require") return usage(argv[0]);
      health = h == "require" ? 2 : h == "report" ? 1 : 0;
    }
    else if (a == "--bdf" && i + 1 < argc) bdfs.emplace_back(argv[++i]);
    else if (a == "--bytes" && i + 1 < argc) bytes = strtoull(argv[++i], nullptr, 10);
    else if (a == "--check" && i + 1 < argc) {
      std::string c = argv[++i];
      if (c != "zero" && c != "tagged") return usage(argv[0]);
      tagged = c == "tagged";
    }
    else if (a == "--backend" && i + 1 < argc) {
      std::string b = argv[++i];
      int be = b == "sim" ? CCM_BACKEND_SIM : b == "cudasim" ? CCM_BACKEND_CUDASIM : b == "sysfs" ? CCM_BACKEND_SYSFS : -1;
      if (be < 0 || ccm_init(be) != CCM_OK) return usage(argv[0]);
    } else return usage(argv[0]);
  }
  if (!all && bdfs.empty()) return usage(argv[0]);
  if (mismatch_triage && !tagged) {
    fprintf(stderr, "--mismatch-triage needs --check tagged\n");
    return usage(argv[0]);
  }
  if (probe && tagged) {
    fprintf(stderr, "--probe is for --check zero: the tagged check already covers every probe window\n");
    return usage(argv[0]);
  }
  if (relay_on && relay_first_on) return usage(argv[0]);
  if ((relay_on || relay_first_on) && bytes != 0) {
    fprintf(stderr, "--relay is for the whole-HBM gate: it refuses --bytes other than 0\n");
    return usage(argv[0]);
  }
  if (mark_mib && !relay_on && !relay_first_on) {
    fprintf(stderr, "--relay-mark-mib needs --relay\n");
    return usage(argv[0]);
  }

  GateArgs g;
  g.bytes = bytes;
  g.tagged = tagged;
  g.residue = residue;
  g.triage = triage;
  g.mismatch_triage = mismatch_triage;
  g.prove = prove;
  g.probe = probe;
  g.triage_hold_ms = triage_hold_ms;
  g.health = health;
  int n = 0;
  ccm_enumerate(nullptr, 0, &n);
  std::vector<ccm_dev_info> infos(n > 0 ? n : 1);
  ccm_enumerate(infos.data(), n, &n);
  if (all) {
    for (int i = 0; i < n; ++i)
      if (infos[i].kind == CCM_KIND_GPU) {
        g.devs.push_back(infos[i].index);
        g.ordinals.push_back(infos[i].cuda_ordinal);
        g.names.emplace_back(infos[i].bdf);
      }
  } else {
    for (auto& want : bdfs) {
      for (auto& c : want) c = (char)tolower(c);
      int found = -1, ordinal = -1;
      for (int i = 0; i < n; ++i)
        if (infos[i].kind == CCM_KIND_GPU && want == infos[i].bdf) { found = infos[i].index; ordinal = infos[i].cuda_ordinal; }
      if (found < 0) { fprintf(stderr, "unknown GPU %s\n", want.c_str()); return 1; }
      g.devs.push_back(found);
      g.ordinals.push_back(ordinal);
      g.names.push_back(want);
    }
  }
  if (relay_first_on) return relay_first(g, mark_mib);
  if (relay_on) return relay(g, argc, argv);
  std::vector<ccm_scrub_result> res;
  const int rc = run_gate(g, GateHooks(), res);
  ccm_device_release_many((int)g.devs.size(), g.devs.data(), nullptr);  // joins the deferred HBM release, drops the contexts
  return rc;
}

// Arms every GPU as `g` asks, runs the gate, disarms, prints the ONE JSON line and returns the exit code: 0 every GPU
// clean, 3 the gate failed.  With --prove, --probe or --health a GPU that cannot be armed fails the gate before anything
// is scrubbed, and nothing is printed.  `res` receives the results, one per GPU.
static int run_gate(const GateArgs& g, const GateHooks& hooks, std::vector<ccm_scrub_result>& res) {
  const std::vector<int>& devs = g.devs;
  const std::vector<int>& ordinals = g.ordinals;
  const std::vector<std::string>& names = g.names;
  const bool tagged = g.tagged, residue = g.residue, triage = g.triage, mismatch_triage = g.mismatch_triage,
             prove = g.prove, probe = g.probe;
  const int health = g.health;
  res.assign(devs.size() ? devs.size() : 1, ccm_scrub_result());
  std::vector<ccm_tag_result> tags(res.size());
  std::vector<ccm_residue_report> census(residue ? res.size() : 0);
  double wall_ms = 0;
  std::vector<int> parmed;   // ordinals armed for the coverage proof: all of them, or the gate does not run
  std::vector<int> probed;   // ordinals armed for the alias probe: all of them, or the gate does not run
  std::vector<int> harmed;   // ordinals armed for the HBM health report: all of them, or the gate does not run
  std::vector<int> armed;    // ordinals armed for the triage, disarmed once the gate is done
  std::vector<int> marmed;   // and for the mismatch triage
  auto disarm = [&] {
    for (int o : armed) ccm_scrub_triage(o, 0);
    for (int o : marmed) ccm_scrub_mismatch_triage(o, 0);
    for (int o : parmed) ccm_scrub_prove(o, 0);
    for (int o : probed) ccm_scrub_probe(o, 0);
    for (int o : harmed) ccm_scrub_health(o, 0);
  };
  for (size_t i = 0; prove && i < ordinals.size(); ++i) {
    const int rc = ordinals[i] >= 0 ? ccm_scrub_prove(ordinals[i], 1) : CCM_ERR_NO_CUDA;
    if (rc != CCM_OK) {
      fprintf(stderr, "cannot arm the coverage proof on %s: %s\n", names[i].c_str(), ccm_strerror(rc));
      disarm();
      return 3;
    }
    parmed.push_back(ordinals[i]);
  }
  for (size_t i = 0; probe && i < ordinals.size(); ++i) {
    const int rc = ordinals[i] >= 0 ? ccm_scrub_probe(ordinals[i], 1) : CCM_ERR_NO_CUDA;
    if (rc != CCM_OK) {
      fprintf(stderr, "cannot arm the alias probe on %s: %s\n", names[i].c_str(), ccm_strerror(rc));
      disarm();
      return 3;
    }
    probed.push_back(ordinals[i]);
  }
  for (size_t i = 0; health && i < ordinals.size(); ++i) {
    const int rc = ordinals[i] >= 0 ? ccm_scrub_health(ordinals[i], health) : CCM_ERR_NO_CUDA;
    if (rc != CCM_OK) {
      fprintf(stderr, "cannot arm the HBM health report on %s: %s\n", names[i].c_str(), ccm_strerror(rc));
      disarm();
      return 3;
    }
    harmed.push_back(ordinals[i]);
  }
  for (size_t i = 0; triage && i < ordinals.size(); ++i)
    if (ordinals[i] >= 0 && ccm_scrub_triage(ordinals[i], (uint32_t)g.triage_hold_ms) == CCM_OK) armed.push_back(ordinals[i]);
  for (size_t i = 0; mismatch_triage && i < ordinals.size(); ++i)
    if (ordinals[i] >= 0 && ccm_scrub_mismatch_triage(ordinals[i], (uint32_t)g.triage_hold_ms) == CCM_OK)
      marmed.push_back(ordinals[i]);
  if (hooks.armed && !hooks.armed()) {
    disarm();
    return 3;
  }
  if (residue)
    ccm_scrub_verify_many_residue((int)devs.size(), devs.data(), g.bytes, tagged ? tags.data() : nullptr, census.data(),
                                  res.data(), &wall_ms);
  else if (tagged) ccm_scrub_verify_many_tagged((int)devs.size(), devs.data(), g.bytes, tags.data(), res.data(), &wall_ms);
  else ccm_scrub_verify_many((int)devs.size(), devs.data(), g.bytes, res.data(), &wall_ms);
  disarm();
  bool clean = true;
  printf("{\"wall_ms\": %.3f, \"reports\": [", wall_ms);
  for (size_t i = 0; i < devs.size(); ++i) {
    const ccm_scrub_result& r = res[i];
    ccm_probe_report pr;
    const bool ran_probe = probe && ccm_scrub_last_probe(ordinals[i], &pr) == CCM_OK && pr.probed;
    ccm_probe_cover pc;
    const bool probe_proved = prove && ran_probe && ccm_scrub_last_probe_cover(ordinals[i], &pc) == CCM_OK && pc.proved;
    // a proving call that probed and has no probe proof fails in its own report, whoever reads it
    int status = r.status == CCM_OK && prove && ran_probe && !probe_proved ? (int)CCM_ERR_UNCOVERED : r.status;
    ccm_hbm_health hh;
    const bool has_health = health && ccm_scrub_last_health(ordinals[i], &hh) == CCM_OK && hh.mode;
    if (health == 2 && !has_health && status == CCM_OK) status = CCM_ERR_HBM_HEALTH;   // asked for and missing
    clean = clean && status == CCM_OK && r.nonzero_bytes == 0;
    printf("%s{\"bdf\": \"%s\", \"bytes_requested\": %llu, \"bytes_scrubbed\": %llu, \"device_total_bytes\": %llu, "
           "\"nonzero_bytes\": %llu, \"ms_acquire\": %.3f, \"ms_scrub\": %.3f, \"ms_verify\": %.3f, \"ms_release\": %.3f, "
           "\"ms_total\": %.3f, \"segments\": %d, \"status\": %d, \"release_deferred\": %d, "
           "\"device_free_before\": %llu, \"bytes_unreached\": %llu, \"ms_release_wait\": %.3f, \"ms_gpu_span\": %.3f",
           i ? ", " : "", names[i].c_str(), (unsigned long long)r.bytes_requested, (unsigned long long)r.bytes_scrubbed,
           (unsigned long long)r.device_total_bytes, (unsigned long long)r.nonzero_bytes, r.ms_acquire, r.ms_scrub,
           r.ms_verify, r.ms_release, r.ms_total, r.segments, status, r.release_deferred,
           (unsigned long long)r.device_free_before, (unsigned long long)r.bytes_unreached, r.ms_release_wait, r.ms_gpu_span);
    if (tagged) {
      const ccm_tag_result& t = tags[i];
      clean = clean && t.mismatch_bytes == 0;
      printf(", \"check\": \"tagged\", \"tag_seed\": %u, \"mismatch_bytes\": %llu, \"ms_tag\": %.3f, \"ms_check\": %.3f",
             t.seed, (unsigned long long)t.mismatch_bytes, t.ms_tag, t.ms_check);
    }
    ccm_dirt_report d;
    if (r.nonzero_bytes != 0 && ccm_scrub_last_dirt(ordinals[i], &d) == CCM_OK) print_dirt(d, ordinals[i]);
    ccm_mismatch_report m;
    if (tagged && tags[i].mismatch_bytes != 0 && ccm_scrub_last_mismatch(ordinals[i], &m) == CCM_OK) print_mismatch(m, ordinals[i]);
    // --probe refuses --check tagged: at most one of the two prints the mismatch report
    if (ran_probe && pr.mismatch_bytes != 0 && ccm_scrub_last_mismatch(ordinals[i], &m) == CCM_OK) print_mismatch(m, ordinals[i]);
    if (residue) print_residue(census[i], ordinals[i]);
    ccm_triage_report t;
    if (triage && r.nonzero_bytes != 0 && ccm_scrub_last_triage(ordinals[i], &t) == CCM_OK && t.triaged)
      print_triage(t, ordinals[i]);
    if (mismatch_triage && tags[i].mismatch_bytes != 0 && ccm_scrub_last_mismatch_triage(ordinals[i], &t) == CCM_OK &&
        t.triaged)
      print_mismatch_triage(t, ordinals[i]);
    ccm_cover_report c;
    const bool proved = prove && ccm_scrub_last_cover(ordinals[i], &c) == CCM_OK && c.proved;
    if (proved) print_cover(c, ordinals[i]);
    ccm_cover_ledger lg;
    const bool ledgered = proved && ccm_scrub_last_ledger(ordinals[i], &lg) == CCM_OK && lg.proved;
    if (ledgered) print_ledger(lg, ordinals[i]);
    clean = clean && (!prove || (proved && ledgered));   // a proof that was asked for and did not run fails the gate
    if (ran_probe) print_probe(pr);
    if (probe_proved) print_pcover(pc, ordinals[i]);
    ccm_report_cover rc;
    if (prove && ccm_scrub_last_report_cover(ordinals[i], &rc) == CCM_OK && rc.proved) print_rcover(rc, ordinals[i]);
    if (has_health) print_health(hh);
    if (hooks.report) hooks.report(i, r);
    printf("}");
  }
  printf("]");
  if (hooks.tail) hooks.tail();
  printf("}\n");
  fflush(stdout);  // the verdict is out BEFORE the contexts are torn down: a parent can act on it right away
  return clean ? 0 : 3;
}

// ------------------------------------------------------------------------------------------------ the relay
using Clock = std::chrono::steady_clock;
static double ms_since(Clock::time_point t0) {
  return std::chrono::duration<double, std::milli>(Clock::now() - t0).count();
}

// The number after `"key": ` in the object of `line` whose "bdf" is `bdf`; false when there is none.
static bool member(const std::string& line, const std::string& bdf, const char* key, uint64_t* v) {
  const size_t at = line.find("{\"bdf\": \"" + bdf + "\"");
  if (at == std::string::npos) return false;
  const size_t end = line.find('}', at);
  const size_t k = line.find(std::string("\"") + key + "\": ", at);
  if (k == std::string::npos || k > end) return false;
  *v = strtoull(line.c_str() + k + strlen(key) + 4, nullptr, 10);
  return true;
}

// A payload of run_gate with `, "relay": null` closing every report.
static std::string with_null_relay(const std::string& p) {
  const std::string open = "\"reports\": [";
  const size_t at = p.find(open);
  if (at == std::string::npos) return p;
  std::string out = p.substr(0, at + open.size());
  int depth = 0;
  bool str = false, esc = false;
  for (size_t k = at + open.size(); k < p.size(); ++k) {
    const char c = p[k];
    if (str) {
      if (esc) esc = false;
      else if (c == '\\') esc = true;
      else if (c == '"') str = false;
    } else if (c == '"') {
      str = true;
    } else if (c == '{' || c == '[') {
      ++depth;
    } else if (c == '}' || c == ']') {
      if (depth == 0) return out + p.substr(k);   // the end of "reports"
      if (--depth == 0 && c == '}') out += ", \"relay\": null";
    }
    out += c;
  }
  return out;
}

// Leg A (--relay-first): the gate as a plain call runs it, its JSON line on stdout (a pipe to the process that started
// it), then its HBM back with the driver and one "released" line, then the drill's marker when asked for, and then it
// waits for stdin to close.  Its contexts stay until it exits: the second leg's context is created while they exist.
static int relay_first(const GateArgs& g, unsigned long mark_mib) {
  prctl(PR_SET_PDEATHSIG, SIGKILL);   // never outlive the process that started it
  if (getppid() == 1) _exit(3);       // which may be gone already
  std::vector<ccm_scrub_result> res;
  const int rc = run_gate(g, GateHooks(), res);
  printf("{\"released\": [");
  for (size_t i = 0; i < g.devs.size(); ++i) {
    double rel = 0, waited = 0;
    ccm_scrub_release_wait(g.devs[i], &rel, &waited);   // not ccm_device_release_many: the contexts must stay
    uint64_t marked = 0;
    if (mark_mib) {
      ccm_arena_info ai;
      uint64_t nz = 0;
      if (ccm_arena_acquire(g.devs[i], (uint64_t)mark_mib << 20, &ai) == CCM_OK &&
          ccm_arena_fill(g.devs[i], 0xA5, nullptr) == CCM_OK &&
          ccm_arena_verify(g.devs[i], CCM_VERIFY_AUTO, nullptr, nullptr, &nz, nullptr) == CCM_OK)
        marked = nz;
      else
        fprintf(stderr, "cannot hold the %lu MiB marker on %s\n", mark_mib, g.names[i].c_str());
    }
    const ccm_scrub_result& r = res[i];
    printf("%s{\"bdf\": \"%s\", \"device_total_bytes\": %llu, \"device_free_before\": %llu, \"bytes_unreached\": %llu, "
           "\"ms_release\": %.3f, \"ms_waited\": %.3f, \"marked\": %llu}",
           i ? ", " : "", g.names[i].c_str(), (unsigned long long)r.device_total_bytes,
           (unsigned long long)r.device_free_before, (unsigned long long)r.bytes_unreached, rel, waited,
           (unsigned long long)marked);
  }
  printf("], \"clean\": %d}\n", rc == 0);
  fflush(stdout);
  char b[256];
  for (;;) {
    const ssize_t n = read(0, b, sizeof b);
    if (n == 0 || (n < 0 && errno != EINTR)) break;
  }
  _exit(rc);   // the exit frees the contexts (and the marker)
}

// The relay (--relay): leg A in a child started before this process creates any context, leg B here.
static int relay(const GateArgs& g, int argc, char** argv) {
  std::vector<std::string> args{"ccm-scrub"};
  for (int i = 1; i < argc; ++i) args.emplace_back(strcmp(argv[i], "--relay") ? argv[i] : "--relay-first");
  std::vector<char*> av;
  for (auto& a : args) av.push_back(&a[0]);
  av.push_back(nullptr);
  int to_a[2], from_a[2];
  if (pipe2(to_a, O_CLOEXEC) != 0 || pipe2(from_a, O_CLOEXEC) != 0) { perror("pipe2"); return 3; }
  const pid_t parent = getpid();
  const Clock::time_point t0 = Clock::now();
  const pid_t pid = fork();   // fork + exec at once: this process has initialised the driver, and CUDA is not fork-safe
  if (pid < 0) { perror("fork"); return 3; }
  if (pid == 0) {
    prctl(PR_SET_PDEATHSIG, SIGKILL);
    if (getppid() != parent) _exit(127);
    dup2(to_a[0], 0);
    dup2(from_a[1], 1);
    execv("/proc/self/exe", av.data());
    _exit(127);
  }
  close(to_a[0]);
  close(from_a[1]);
  bool reaped = false;
  int a_status = 0;
  auto reap = [&] {
    if (reaped) return;
    close(to_a[1]);
    while (waitpid(pid, &a_status, 0) < 0 && errno == EINTR) {}
    reaped = true;
  };
  // A's JSON line, then its "released" line (none when it could not arm: then its gate did not run)
  FILE* in = fdopen(from_a[0], "r");
  std::string payload, released;
  char* line = nullptr;
  size_t cap = 0;
  ssize_t len;
  while (released.empty() && in && (len = getline(&line, &cap, in)) > 0) {
    std::string l(line, (size_t)len);
    while (!l.empty() && (l.back() == '\n' || l.back() == '\r')) l.pop_back();
    if (l.rfind("{\"released\": ", 0) == 0) released = l;
    else if (l.rfind("{\"wall_ms\": ", 0) == 0) payload = l;
  }
  free(line);
  const double ms_first = ms_since(t0);
  const bool a_clean = released.find("], \"clean\": 1}") != std::string::npos;
  auto first = [&] { printf(", \"first\": %s, \"first_pid\": %d", payload.c_str(), (int)pid); };
  if (payload.empty() || !a_clean) {   // A failed or died: no second leg, the gate has failed anyway
    reap();
    if (in) fclose(in);
    if (payload.empty()) {
      fprintf(stderr, "the first leg (pid %d) printed no report: %s\n", (int)pid,
              WIFEXITED(a_status) ? "its gate did not run" : "it died");
      return 3;
    }
    const std::string own = with_null_relay(payload);
    printf("%s", own.substr(0, own.size() - 1).c_str());   // without its closing brace
    first();
    printf("}\n");
    fflush(stdout);
    return 3;
  }
  const size_t n = g.devs.size();
  std::vector<uint64_t> held(n), tot(n);
  std::vector<bool> have(n, false);
  std::vector<ccm_relay::Settle> settle(n);
  double ms_handover = 0, ms_settle = 0;
  const Clock::time_point t_released = Clock::now();
  GateHooks hooks;
  hooks.armed = [&] {
    // this leg's context exists and is armed: every allocation it needs is made by now
    for (size_t i = 0; i < n; ++i) have[i] = ccm_device_memory(g.ordinals[i], &held[i], &tot[i]) == CCM_OK;
    reap();
    const Clock::time_point t_reaped = Clock::now();
    ms_handover = std::chrono::duration<double, std::milli>(t_reaped - t_released).count();
    if (!WIFEXITED(a_status) || WEXITSTATUS(a_status) != 0) {
      fprintf(stderr, "the first leg (pid %d) did not exit cleanly (status %d): no second leg\n", (int)pid, a_status);
      return false;
    }
    for (;;) {
      const double ms = ms_since(t_reaped);
      bool done = true;
      for (size_t i = 0; i < n; ++i) {
        uint64_t fr = 0, t = 0;
        if (!have[i] || settle[i].done) continue;
        if (ccm_device_memory(g.ordinals[i], &fr, &t) != CCM_OK) { have[i] = false; continue; }
        done = settle[i].read(fr, ms) && done;
      }
      if (done) break;
      std::this_thread::sleep_for(std::chrono::duration<double, std::milli>(ccm_relay::kSettlePollMs));
    }
    ms_settle = ms_since(t_reaped);
    return true;
  };
  bool computed = true;
  hooks.report = [&](size_t i, const ccm_scrub_result& r) {
    ccm_relay::Inputs x;
    x.total = r.device_total_bytes;
    x.b_free_held = held[i];
    x.b_free_settled = settle[i].free_bytes;
    x.b_free_before = r.device_free_before;
    x.b_unreached = r.bytes_unreached;
    const std::string& bdf = g.names[i];
    if (!have[i] || r.device_total_bytes == 0 || !member(released, bdf, "device_free_before", &x.a_free_before) ||
        !member(released, bdf, "bytes_unreached", &x.a_unreached) || !member(released, bdf, "marked", &x.marked)) {
      computed = false;
      printf(", \"relay\": null");
      return;
    }
    const ccm_relay::Relay v = ccm_relay::account(x);
    printf(", \"relay\": {\"total\": %llu, \"a_free_before\": %llu, \"a_unreached\": %llu, \"b_free_held\": %llu, "
           "\"b_free_settled\": %llu, \"b_free_before\": %llu, \"b_unreached\": %llu, \"marked\": %llu, "
           "\"footprint_a\": %llu, \"freed\": %llu, \"held\": %llu, \"growth\": %llu, \"unreached\": %llu, "
           "\"coverage\": %.9f, \"settled\": %d, \"settle_polls\": %d, \"ms_first\": %.3f, \"ms_handover\": %.3f, "
           "\"ms_settle\": %.3f, \"ms_second\": %.3f}",
           (unsigned long long)x.total, (unsigned long long)x.a_free_before, (unsigned long long)x.a_unreached,
           (unsigned long long)x.b_free_held, (unsigned long long)x.b_free_settled, (unsigned long long)x.b_free_before,
           (unsigned long long)x.b_unreached, (unsigned long long)x.marked, (unsigned long long)v.footprint_a,
           (unsigned long long)v.freed, (unsigned long long)v.held, (unsigned long long)v.growth,
           (unsigned long long)v.unreached, v.coverage, settle[i].settled, settle[i].polls, ms_first, ms_handover,
           ms_settle, r.ms_total);
  };
  hooks.tail = first;
  std::vector<ccm_scrub_result> res;
  const int rc = run_gate(g, hooks, res);
  reap();   // when arming failed, the hook never ran
  if (in) fclose(in);
  ccm_device_release_many((int)g.devs.size(), g.devs.data(), nullptr);
  return rc == 0 && computed ? 0 : 3;
}

// The "probe_cover" object: the fields of k8s_cc_manager_b200.devices.ProbeCoverReport, with the first 64 inexact pages.
static void print_pcover(const ccm_probe_cover& c, int ordinal) {
  static const char* const names[3] = {"P1", "P2", "P3"};
  printf(", \"probe_cover\": {\"windows_expected\": %llu, \"va_base\": %llu, \"ms_prove\": %.3f, \"proved\": %d, "
         "\"covered\": %d, \"steps\": [",
         (unsigned long long)c.windows_expected, (unsigned long long)c.va_base, c.ms_prove, c.proved, c.covered);
  for (int k = 0; k < 3; ++k) {
    const ccm_probe_cover_step& p = c.step[k];
    printf("%s{\"name\": \"%s\", \"ran\": %d, \"windows_counted\": %llu, \"windows_missing\": %llu, "
           "\"windows_extra\": %llu, \"windows_outside\": %llu, \"pages_short\": %llu, \"pages_over\": %llu, "
           "\"first_short_page\": %llu}",
           k ? ", " : "", names[k], p.ran, (unsigned long long)p.windows_counted, (unsigned long long)p.windows_missing,
           (unsigned long long)p.windows_extra, (unsigned long long)p.windows_outside, (unsigned long long)p.pages_short,
           (unsigned long long)p.pages_over, (unsigned long long)p.first_short_page);
  }
  printf("], \"pages\": [");
  uint64_t n = 0;
  std::vector<ccm_probe_cover_page> v;
  if (!c.covered && ccm_last_probe_cover_pages(ordinal, nullptr, 0, &n) == CCM_OK) {
    v.resize(n);
    if (n && ccm_last_probe_cover_pages(ordinal, v.data(), n, &n) != CCM_OK) v.clear();
  }
  const size_t keep = 64;   // k8s_cc_manager_b200.devices.COVER_PAGES
  for (size_t k = 0; k < v.size() && k < keep; ++k)
    printf("%s{\"page\": %llu, \"chunk\": %u, \"expected\": %u, \"p1\": %u, \"p2\": %u, \"p3\": %u}",
           k ? ", " : "", (unsigned long long)v[k].page, v[k].chunk, v[k].expected, v[k].count[0], v[k].count[1],
           v[k].count[2]);
  printf("], \"pages_truncated\": %d}", v.size() > keep);
}
