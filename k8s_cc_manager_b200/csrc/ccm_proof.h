// ccm_proof.h — host-side comparison of the proving kernels' cover maps with what a call holds (include/ccm.h:
// ccm_cover_report, ccm_probe_cover, ccm_report_cover).  Plain C++17, no CUDA: a CPU test compiles it on its own.
// A cover map is np words, word p the bytes counted on the 2 MiB page p from the call's va_base, then the outside slot
// (bytes counted before va_base or past the last page).  A proof requires every page to count exactly what the call
// expects on it, and the outside slot 0.  The coverage ledger (ccm_cover_ledger) is the same per 128 KiB slot.
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <utility>
#include <vector>

#include "ccm.h"

namespace ccm_proof {

constexpr uint64_t kPageBytes = CCM_PAGE_BYTES;
constexpr uint64_t kProbeStride = CCM_PROBE_STRIDE;
constexpr uint64_t kProbeWindow = CCM_PROBE_WINDOW;

// (offset, chunk) of every allocation's first byte, ascending.
using ChunkTable = std::vector<std::pair<uint64_t, uint32_t>>;

// The chunk of `offset`: that of the last allocation that starts at or before it, else the first.  Compared as
// signed: the head window of a raw region that does not start 16-aligned has a negative offset.  (A mapping or a
// segment starts aligned, so the product call never books one.)
inline uint32_t chunk_of(const ChunkTable& chunks, uint64_t offset) {
  auto it = std::upper_bound(chunks.begin(), chunks.end(), offset, [](uint64_t o, const std::pair<uint64_t, uint32_t>& c) {
    return (int64_t)o < (int64_t)c.first;
  });
  if (it != chunks.begin()) --it;
  return it == chunks.end() ? 0u : it->second;
}

// The probe windows of [addr, addr + n): the first 4096-aligned address w0 whose 32 bytes lie inside, and how many
// windows follow it at the stride.
inline void probe_windows_of(uint64_t addr, uint64_t n, uint64_t* w0, uint64_t* nwin) {
  *w0 = (addr + kProbeStride - 1) & ~(kProbeStride - 1);
  *nwin = *w0 + kProbeWindow <= addr + n ? (addr + n - kProbeWindow - *w0) / kProbeStride + 1 : 0;
}

// What a walk over `pieces` (each `bytes` at `offset` from va_base) must count on each of the np pages: the bytes of
// the pieces that lie on it.
template <typename Piece>
std::vector<uint32_t> piece_bytes(const std::vector<Piece>& pieces, uint64_t np) {
  std::vector<uint32_t> exp(np, 0);
  for (const Piece& r : pieces)
    for (uint64_t o = r.offset, end = r.offset + r.bytes; o < end;) {
      const uint64_t p = o / kPageBytes, next = std::min<uint64_t>(end, (p + 1) * kPageBytes);
      if (p < np) exp[p] += (uint32_t)(next - o);
      o = next;
    }
  return exp;
}

// What every step of the probe must count on each of the np pages: CCM_PROBE_WINDOW bytes per window of `chunks`
// (each `bytes` at address `addr`, `offset` from va_base), on the page its offset (c.offset + (window - c.addr)) starts
// on.  A window that crosses a page boundary splits its bytes there, as the kernels' cover_lanes does (it cannot on
// 32-byte-aligned chunk offsets).  Chunks are walked page by page, not window by window: a whole-HBM call has some
// 20 M windows.
template <typename Chunk>
std::vector<uint32_t> probe_bytes(const std::vector<Chunk>& chunks, uint64_t np) {
  std::vector<uint32_t> exp(np, 0);
  for (const Chunk& c : chunks) {
    uint64_t w0 = 0, nwin = 0;
    probe_windows_of(c.addr, c.bytes, &w0, &nwin);
    if (nwin == 0) continue;
    const uint64_t o0 = c.offset + (w0 - c.addr);   // offset of the chunk's first window
    const uint64_t last = o0 + (nwin - 1) * kProbeStride;
    for (uint64_t p = o0 / kPageBytes; p <= last / kPageBytes && p < np; ++p) {
      const uint64_t lo = p * kPageBytes, hi = lo + kPageBytes;
      const uint64_t i0 = lo <= o0 ? 0 : (lo - o0 + kProbeStride - 1) / kProbeStride;
      const uint64_t i1 = std::min<uint64_t>(nwin, (hi - o0 + kProbeStride - 1) / kProbeStride);
      if (i1 <= i0) continue;
      exp[p] += (uint32_t)((i1 - i0) * kProbeWindow);
      const uint64_t end = o0 + (i1 - 1) * kProbeStride + kProbeWindow;   // the page's last window, past its end?
      if (end > hi) {
        exp[p] -= (uint32_t)(end - hi);
        if (p + 1 < np) exp[p + 1] += (uint32_t)(end - hi);
      }
    }
  }
  return exp;
}

// One map against its expectation, in bytes.  counted and extra include the outside slot, as the reports define them.
struct Tally {
  uint64_t counted = 0, missing = 0, extra = 0, outside = 0, pages_short = 0, pages_over = 0, first_short_page = 0;
  bool exact() const { return missing == 0 && extra == 0; }
};

// Compares `map` (exp.size() page words, then the outside slot) with `exp`; appends every inexact page to *inexact,
// ascending.
inline Tally tally(const uint32_t* map, const std::vector<uint32_t>& exp, std::vector<uint64_t>* inexact) {
  Tally t;
  const uint64_t np = exp.size();
  for (uint64_t p = 0; p < np; ++p) {
    const uint32_t c = map[p];
    t.counted += c;
    if (c == exp[p]) continue;
    if (c < exp[p]) {
      if (t.pages_short++ == 0) t.first_short_page = p;
      t.missing += exp[p] - c;
    } else {
      t.pages_over++;
      t.extra += c - exp[p];
    }
    inexact->push_back(p);
  }
  t.outside = map[np];
  t.counted += t.outside;
  t.extra += t.outside;
  return t;
}

// A row of the coverage or the report proof (ccm_cover_pass, ccm_report_cover_step), in bytes.
template <typename Row>
void put_bytes(Row* r, const Tally& t) {
  r->bytes_counted = t.counted;
  r->bytes_missing = t.missing;
  r->bytes_extra = t.extra;
  r->bytes_outside = t.outside;
  r->pages_short = t.pages_short;
  r->pages_over = t.pages_over;
  r->first_short_page = t.first_short_page;
}

// The three maps of the passes or of the probe steps (np + 1 words each, end to end) against one expectation:
// t[k] for every map that ran (ran[k]; the others are not compared), and *pages one entry (ccm_cover_page,
// ccm_probe_cover_page) per page inexact in any of them, ascending, with the counts of those that ran.
template <typename Page>
void tally_three(const uint32_t* maps, uint64_t np, const std::vector<uint32_t>& exp, const bool ran[3],
                 const ChunkTable& chunks, Tally t[3], std::vector<Page>* pages) {
  std::vector<uint64_t> bad;
  for (int k = 0; k < 3; ++k)
    if (ran[k]) t[k] = tally(maps + k * (np + 1), exp, &bad);
  std::sort(bad.begin(), bad.end());
  bad.erase(std::unique(bad.begin(), bad.end()), bad.end());
  pages->clear();
  for (const uint64_t p : bad) {
    Page e;
    memset(&e, 0, sizeof e);
    e.page = p;
    e.chunk = chunk_of(chunks, p * kPageBytes);
    e.expected = exp[p];
    for (int k = 0; k < 3; ++k)
      if (ran[k]) e.count[k] = maps[k * (np + 1) + p];
    pages->push_back(e);
  }
}

// The coverage proof of a call that holds `spans` (offsets tiling [0, bytes_mapped)) from va_base: `maps` are the
// three passes' maps, ran[k] says pass k ran.  Fills *rep (proved = 1; ms_prove is the caller's) and *pages.
template <typename Span>
void fill_cover(const uint32_t* maps, uint64_t np, const std::vector<Span>& spans, uint64_t bytes_mapped,
                uint64_t va_base, const bool ran[3], const ChunkTable& chunks, ccm_cover_report* rep,
                std::vector<ccm_cover_page>* pages) {
  memset(rep, 0, sizeof *rep);
  rep->bytes_mapped = bytes_mapped;
  rep->pages_mapped = (bytes_mapped + kPageBytes - 1) / kPageBytes;
  rep->va_base = va_base;
  rep->proved = 1;
  Tally t[3];
  tally_three(maps, np, piece_bytes(spans, np), ran, chunks, t, pages);
  for (int k = 0; k < 3; ++k) {
    rep->pass[k].ran = ran[k];
    put_bytes(&rep->pass[k], t[k]);
  }
  rep->covered = t[0].exact() && t[1].exact() && t[2].exact();
}

constexpr uint64_t kSlotBytes = CCM_LEDGER_SLOT_BYTES;

// The coverage ledger of a call that mapped bytes_mapped from va_base: `ledgers` are the three passes' ledgers, ns + 1
// words each (ns slots, then the outside slot), end to end; ran[k] says pass k ran.  Every pass that ran must count
// min(kSlotBytes, bytes_mapped - s * kSlotBytes) on every slot s of [0, bytes_mapped), 0 on every other slot and 0 in
// the outside slot.  Fills *rep (proved = 1; ms_ledger is the caller's) and *slots, one entry per slot inexact in any
// pass that ran, ascending.
inline void fill_ledger(const uint32_t* ledgers, uint64_t ns, uint64_t bytes_mapped, uint64_t va_base, const bool ran[3],
                        const ChunkTable& chunks, ccm_cover_ledger* rep, std::vector<ccm_ledger_slot>* slots) {
  memset(rep, 0, sizeof *rep);
  rep->bytes_mapped = bytes_mapped;
  rep->slots_mapped = (bytes_mapped + kSlotBytes - 1) / kSlotBytes;
  rep->va_base = va_base;
  rep->proved = 1;
  rep->exact = 1;
  slots->clear();
  for (uint64_t s = 0; s < ns; ++s) {
    const uint32_t want = s * kSlotBytes < bytes_mapped ? (uint32_t)std::min(kSlotBytes, bytes_mapped - s * kSlotBytes) : 0u;
    bool bad = false;
    for (int k = 0; k < 3; ++k) {
      if (!ran[k]) continue;
      const uint32_t got = ledgers[k * (ns + 1) + s];
      if (got == want) continue;
      bad = true;
      ccm_ledger_pass& p = rep->pass[k];
      if (got < want) {
        if (p.slots_short++ == 0) p.first_short_slot = s;
        p.bytes_missing += want - got;
      } else {
        if (p.slots_over++ == 0) p.first_over_slot = s;
        p.bytes_extra += got - want;
      }
    }
    if (!bad) continue;
    ccm_ledger_slot e;
    memset(&e, 0, sizeof e);
    e.slot = s;
    e.chunk = chunk_of(chunks, s * kSlotBytes);
    e.expected = want;
    for (int k = 0; k < 3; ++k)
      if (ran[k]) e.count[k] = ledgers[k * (ns + 1) + s];
    slots->push_back(e);
  }
  for (int k = 0; k < 3; ++k) {
    ccm_ledger_pass& p = rep->pass[k];
    p.ran = ran[k];
    if (!ran[k]) continue;
    p.bytes_outside = ledgers[k * (ns + 1) + ns];
    p.bytes_extra += p.bytes_outside;
    if (p.bytes_missing || p.bytes_extra) rep->exact = 0;
  }
}

inline uint64_t windows(uint64_t bytes) { return (bytes + kProbeWindow - 1) / kProbeWindow; }

// The probe proof of a call whose probe walked `chunks` (as probe_bytes): `maps` are P1's, P2's and P3's.  Fills *rep
// (proved = 1; ms_prove is the caller's) and *pages.
template <typename Chunk>
void fill_probe_cover(const uint32_t* maps, uint64_t np, const std::vector<Chunk>& chunks, uint64_t va_base,
                      const ChunkTable& owners, ccm_probe_cover* rep, std::vector<ccm_probe_cover_page>* pages) {
  memset(rep, 0, sizeof *rep);
  rep->va_base = va_base;
  rep->proved = 1;
  for (const Chunk& c : chunks) {
    uint64_t w0 = 0, nwin = 0;
    probe_windows_of(c.addr, c.bytes, &w0, &nwin);
    rep->windows_expected += nwin;
  }
  const bool ran[3] = {true, true, true};
  Tally t[3];
  tally_three(maps, np, probe_bytes(chunks, np), ran, owners, t, pages);
  for (int k = 0; k < 3; ++k) {
    ccm_probe_cover_step& ps = rep->step[k];
    ps.ran = 1;
    ps.windows_counted = windows(t[k].counted);
    ps.windows_missing = windows(t[k].missing);
    ps.windows_extra = windows(t[k].extra);
    ps.windows_outside = windows(t[k].outside);
    ps.pages_short = t[k].pages_short;
    ps.pages_over = t[k].pages_over;
    ps.first_short_page = t[k].first_short_page;
  }
  rep->covered = t[0].exact() && t[1].exact() && t[2].exact();
}

// Report steps first .. first + n - 1 (CCM_REPORT_*) that ran to their end over `pieces` (as piece_bytes): `maps` are
// their maps, end to end, and launches[s - 1] the launches of step s.  Fills rep->step[] of each (ran = 1), clears
// rep->covered when one is inexact, and appends one entry per inexact (step, page) to *pages.
template <typename Piece>
void fill_report_steps(const uint32_t* maps, uint64_t np, int first, int n, const std::vector<Piece>& pieces,
                       const uint64_t* launches, const ChunkTable& chunks, ccm_report_cover* rep,
                       std::vector<ccm_report_cover_page>* pages) {
  const std::vector<uint32_t> exp = piece_bytes(pieces, np);
  uint64_t total = 0;
  for (const Piece& r : pieces) total += r.bytes;
  for (int k = 0; k < n; ++k) {
    const int step = first + k;
    const uint32_t* m = maps + k * (np + 1);
    std::vector<uint64_t> bad;
    const Tally t = tally(m, exp, &bad);
    ccm_report_cover_step& ps = rep->step[step - 1];
    ps.ran = 1;
    ps.launches = launches[step - 1];
    ps.bytes_expected = total;
    put_bytes(&ps, t);
    if (!t.exact()) rep->covered = 0;
    for (const uint64_t p : bad)
      pages->push_back(ccm_report_cover_page{p, chunk_of(chunks, p * kPageBytes), step, exp[p], m[p]});
  }
}

}  // namespace ccm_proof
