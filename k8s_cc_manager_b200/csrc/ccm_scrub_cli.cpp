// ccm-scrub — native command-line front end of the HBM scrub gate (links libccm.so).
//
//   ccm-scrub [--bytes N] [--backend sim|cudasim|sysfs] [--check zero|tagged] [--residue] (--all | --bdf <pci address> ...)
//
// Runs the concurrent gate (ccm_scrub_verify_many, or ccm_scrub_verify_many_tagged with --check tagged)
// and prints ONE JSON line with the same fields as k8s_cc_manager_b200.devices.ScrubReport (the
// tagged-gate fields only with --check tagged, "dirt" only for a GPU whose read-back found non-zero bytes: where
// they are, as ccm_scrub_last_dirt reports it; "mismatch" only for a GPU whose tagged check found bytes off their
// tags, as ccm_scrub_last_mismatch reports it; "residue" for every GPU with --residue, which runs the census
// calls, ccm_scrub_verify_many_residue).  Exit 0: every GPU clean; 3: gate failed;
// 2: usage.  Used by the manager for CC_SCRUB_ISOLATION=process (no Python start-up in the
// child) and usable from the legacy shell engine (reference scripts/cc-manager.sh) as a
// post-reset step.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "ccm.h"

// The "dirt" object: the fields of k8s_cc_manager_b200.devices.DirtReport, records with their bytes in hex.
static void print_dirt(const ccm_dirt_report& d) {
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
  printf("]}");
}

// The "mismatch" object: the fields of k8s_cc_manager_b200.devices.MismatchReport, kinds by name.
static void print_mismatch(const ccm_mismatch_report& m) {
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
  printf("]}");
}

// The "residue" object: the fields of k8s_cc_manager_b200.devices.ResidueReport (no bytes: there are none).
static void print_residue(const ccm_residue_report& r) {
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
  printf("]}");
}

static int usage(const char* argv0) {
  fprintf(stderr, "usage: %s [--bytes N] [--backend sim|cudasim|sysfs] [--check zero|tagged] [--residue] "
          "(--all | --bdf <bdf> ...)\n", argv0);
  return 2;
}

int main(int argc, char** argv) {
  std::vector<std::string> bdfs;
  unsigned long long bytes = 0;
  bool all = false, tagged = false, residue = false;
  for (int i = 1; i < argc; ++i) {
    std::string a = argv[i];
    if (a == "--all") all = true;
    else if (a == "--residue") residue = true;
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

  int n = 0;
  ccm_enumerate(nullptr, 0, &n);
  std::vector<ccm_dev_info> infos(n > 0 ? n : 1);
  ccm_enumerate(infos.data(), n, &n);
  std::vector<int> devs, ordinals;
  std::vector<std::string> names;
  if (all) {
    for (int i = 0; i < n; ++i)
      if (infos[i].kind == CCM_KIND_GPU) {
        devs.push_back(infos[i].index);
        ordinals.push_back(infos[i].cuda_ordinal);
        names.emplace_back(infos[i].bdf);
      }
  } else {
    for (auto& want : bdfs) {
      for (auto& c : want) c = (char)tolower(c);
      int found = -1, ordinal = -1;
      for (int i = 0; i < n; ++i)
        if (infos[i].kind == CCM_KIND_GPU && want == infos[i].bdf) { found = infos[i].index; ordinal = infos[i].cuda_ordinal; }
      if (found < 0) { fprintf(stderr, "unknown GPU %s\n", want.c_str()); return 1; }
      devs.push_back(found);
      ordinals.push_back(ordinal);
      names.push_back(want);
    }
  }
  std::vector<ccm_scrub_result> res(devs.size() ? devs.size() : 1);
  std::vector<ccm_tag_result> tags(res.size());
  std::vector<ccm_residue_report> census(residue ? res.size() : 0);
  double wall_ms = 0;
  if (residue)
    ccm_scrub_verify_many_residue((int)devs.size(), devs.data(), bytes, tagged ? tags.data() : nullptr, census.data(),
                                  res.data(), &wall_ms);
  else if (tagged) ccm_scrub_verify_many_tagged((int)devs.size(), devs.data(), bytes, tags.data(), res.data(), &wall_ms);
  else ccm_scrub_verify_many((int)devs.size(), devs.data(), bytes, res.data(), &wall_ms);
  bool clean = true;
  printf("{\"wall_ms\": %.3f, \"reports\": [", wall_ms);
  for (size_t i = 0; i < devs.size(); ++i) {
    const ccm_scrub_result& r = res[i];
    clean = clean && r.status == CCM_OK && r.nonzero_bytes == 0;
    printf("%s{\"bdf\": \"%s\", \"bytes_requested\": %llu, \"bytes_scrubbed\": %llu, \"device_total_bytes\": %llu, "
           "\"nonzero_bytes\": %llu, \"ms_acquire\": %.3f, \"ms_scrub\": %.3f, \"ms_verify\": %.3f, \"ms_release\": %.3f, "
           "\"ms_total\": %.3f, \"segments\": %d, \"status\": %d, \"release_deferred\": %d, "
           "\"device_free_before\": %llu, \"bytes_unreached\": %llu, \"ms_release_wait\": %.3f, \"ms_gpu_span\": %.3f",
           i ? ", " : "", names[i].c_str(), (unsigned long long)r.bytes_requested, (unsigned long long)r.bytes_scrubbed,
           (unsigned long long)r.device_total_bytes, (unsigned long long)r.nonzero_bytes, r.ms_acquire, r.ms_scrub,
           r.ms_verify, r.ms_release, r.ms_total, r.segments, r.status, r.release_deferred,
           (unsigned long long)r.device_free_before, (unsigned long long)r.bytes_unreached, r.ms_release_wait, r.ms_gpu_span);
    if (tagged) {
      const ccm_tag_result& t = tags[i];
      clean = clean && t.mismatch_bytes == 0;
      printf(", \"check\": \"tagged\", \"tag_seed\": %u, \"mismatch_bytes\": %llu, \"ms_tag\": %.3f, \"ms_check\": %.3f",
             t.seed, (unsigned long long)t.mismatch_bytes, t.ms_tag, t.ms_check);
    }
    ccm_dirt_report d;
    if (r.nonzero_bytes != 0 && ccm_scrub_last_dirt(ordinals[i], &d) == CCM_OK) print_dirt(d);
    ccm_mismatch_report m;
    if (tagged && tags[i].mismatch_bytes != 0 && ccm_scrub_last_mismatch(ordinals[i], &m) == CCM_OK) print_mismatch(m);
    if (residue) print_residue(census[i]);
    printf("}");
  }
  printf("]}\n");
  fflush(stdout);  // the verdict is out BEFORE the contexts are torn down: a parent can act on it right away
  ccm_device_release_many((int)devs.size(), devs.data(), nullptr);  // joins the deferred HBM release, drops the contexts
  return clean ? 0 : 3;
}
