// ccm_health.h — the HBM health rule (include/ccm.h: ccm_hbm_health) and the drills it is tested with.  Plain C++17,
// no CUDA: a CPU test compiles it on its own.  An armed product call takes one snapshot before it maps anything and one
// after its reports, layers the drills on the second (layer), and judges the pair (judge).
#pragma once
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>

#include "ccm.h"

namespace ccm_health {

// The queries the rule needs, in both snapshots: ECC on, the uncorrected counts and the remap state.  The corrected
// counts and the bank histogram are reported and judge nothing.
constexpr uint32_t kNeeded =
    CCM_HBM_Q_ECC_MODE | CCM_HBM_Q_DRAM_UNCORRECTED | CCM_HBM_Q_SRAM_UNCORRECTED | CCM_HBM_Q_REMAPPED_ROWS;
constexpr uint32_t kAllQueries = (1u << CCM_HBM_QUERIES) - 1;
constexpr int32_t kNvmlNotSupported = 3;   // NVML_ERROR_NOT_SUPPORTED
constexpr uint32_t kUnfit = CCM_HBM_R_DRAM_UNCORRECTED | CCM_HBM_R_SRAM_UNCORRECTED | CCM_HBM_R_REMAP_PENDING |
                            CCM_HBM_R_REMAP_FAILURE | CCM_HBM_R_ECC_OFF;

// The "hbm_*" drills of ccm_sim_set (include/ccm.h).
struct Drills {
  uint64_t uncorrected = 0, corrected = 0;
  bool remap_pending = false, remap_failure = false;
  uint32_t unavailable = 0;   // ccm_hbm_query bits
};

// Sets the fields of query `q` (one ccm_hbm_query bit) to 0.
inline void clear_query(ccm_hbm_state* s, uint32_t q) {
  switch (q) {
    case CCM_HBM_Q_ECC_MODE: s->ecc_current = s->ecc_pending = 0; break;
    case CCM_HBM_Q_DRAM_CORRECTED: s->dram_corrected = 0; break;
    case CCM_HBM_Q_DRAM_UNCORRECTED: s->dram_uncorrected = 0; break;
    case CCM_HBM_Q_SRAM_CORRECTED: s->sram_corrected = 0; break;
    case CCM_HBM_Q_SRAM_UNCORRECTED: s->sram_uncorrected = 0; break;
    case CCM_HBM_Q_REMAPPED_ROWS: s->rows_corrected = s->rows_uncorrected = s->remap_pending = s->remap_failure = 0; break;
    case CCM_HBM_Q_REMAP_HISTOGRAM: s->hist_max = s->hist_high = s->hist_partial = s->hist_low = s->hist_none = 0; break;
  }
}

// The drills on top of what NVML returned: the counts and flags first, then the queries reported as not supported
// (those lose what the drills added, as they would on a card that does not answer them).
inline void layer(ccm_hbm_state* s, const Drills& d) {
  s->dram_uncorrected += d.uncorrected;
  s->dram_corrected += d.corrected;
  if (d.remap_pending) s->remap_pending = 1;
  if (d.remap_failure) s->remap_failure = 1;
  for (uint32_t k = 0; k < CCM_HBM_QUERIES; ++k)
    if (d.unavailable & (1u << k)) {
      clear_query(s, 1u << k);
      s->available &= ~(1u << k);
      s->nvml_rc[k] = kNvmlNotSupported;
    }
}

// The report of a call from its two snapshots (mode and ms_health are the caller's).
inline void judge(const ccm_hbm_state& before, const ccm_hbm_state& after, ccm_hbm_health* h) {
  h->before = before;
  h->after = after;
  const uint32_t both = before.available & after.available;
  struct Counter { uint32_t q; uint64_t ccm_hbm_state::*v; int64_t ccm_hbm_health::*d; };
  static const Counter kCounters[4] = {
      {CCM_HBM_Q_DRAM_CORRECTED, &ccm_hbm_state::dram_corrected, &ccm_hbm_health::d_dram_corrected},
      {CCM_HBM_Q_DRAM_UNCORRECTED, &ccm_hbm_state::dram_uncorrected, &ccm_hbm_health::d_dram_uncorrected},
      {CCM_HBM_Q_SRAM_CORRECTED, &ccm_hbm_state::sram_corrected, &ccm_hbm_health::d_sram_corrected},
      {CCM_HBM_Q_SRAM_UNCORRECTED, &ccm_hbm_state::sram_uncorrected, &ccm_hbm_health::d_sram_uncorrected}};
  uint32_t r = 0;
  for (const Counter& c : kCounters) {
    h->*c.d = (both & c.q) ? (int64_t)(after.*c.v - before.*c.v) : 0;
    if ((both & c.q) && after.*c.v < before.*c.v) r |= CCM_HBM_R_WENT_DOWN;
  }
  if (h->d_dram_uncorrected > 0) r |= CCM_HBM_R_DRAM_UNCORRECTED;
  if (h->d_sram_uncorrected > 0) r |= CCM_HBM_R_SRAM_UNCORRECTED;
  if ((after.available & CCM_HBM_Q_REMAPPED_ROWS) && after.remap_pending) r |= CCM_HBM_R_REMAP_PENDING;
  if ((after.available & CCM_HBM_Q_REMAPPED_ROWS) && after.remap_failure) r |= CCM_HBM_R_REMAP_FAILURE;
  if ((after.available & CCM_HBM_Q_ECC_MODE) && !after.ecc_current) r |= CCM_HBM_R_ECC_OFF;
  h->missing_queries = kNeeded & ~both;
  if (h->missing_queries) r |= CCM_HBM_R_NO_ANSWER;
  h->reasons = r;
  h->verdict = (r & kUnfit) ? CCM_HBM_UNFIT : r ? CCM_HBM_UNKNOWN : CCM_HBM_FIT;
}

// The reasons of a report that is not fit, for the error text: "; "-separated, in ccm_hbm_reason order.
inline std::string reasons(const ccm_hbm_health& h) {
  static const char* const kQueryNames[CCM_HBM_QUERIES] = {"ECC mode", "DRAM corrected", "DRAM uncorrected",
                                                           "SRAM corrected", "SRAM uncorrected", "remapped rows",
                                                           "remap histogram"};
  std::string s;
  char b[160];
  auto add = [&](const char* t) { if (!s.empty()) s += "; "; s += t; };
  if (h.reasons & CCM_HBM_R_DRAM_UNCORRECTED) {
    snprintf(b, sizeof b, "uncorrected DRAM errors +%lld during the call", (long long)h.d_dram_uncorrected);
    add(b);
  }
  if (h.reasons & CCM_HBM_R_SRAM_UNCORRECTED) {
    snprintf(b, sizeof b, "uncorrected SRAM errors +%lld during the call", (long long)h.d_sram_uncorrected);
    add(b);
  }
  if (h.reasons & CCM_HBM_R_REMAP_PENDING) add("a row remap is pending: reset the GPU before it holds a tenant's data");
  if (h.reasons & CCM_HBM_R_REMAP_FAILURE) add("a row remap failed: the banks are out of spare rows (RMA)");
  if (h.reasons & CCM_HBM_R_ECC_OFF) add("ECC is off");
  if (h.reasons & CCM_HBM_R_NO_ANSWER) {
    std::string q;
    for (uint32_t k = 0; k < CCM_HBM_QUERIES; ++k)
      if (h.missing_queries & (1u << k)) {
        const int rc = (h.after.available & (1u << k)) ? h.before.nvml_rc[k] : h.after.nvml_rc[k];
        snprintf(b, sizeof b, "%s%s (NVML %d)", q.empty() ? "" : ", ", kQueryNames[k], rc);
        q += b;
      }
    add(("no answer from NVML for " + q).c_str());
  }
  if (h.reasons & CCM_HBM_R_WENT_DOWN) add("an error counter went down between the snapshots (a reset in between)");
  return s;
}

}  // namespace ccm_health
