// ccm_core.cpp — device table, register backends and the public C ABI of libccm.so.
//
// Replaces the device-access boundary of the reference (external
// NVIDIA/gpu-admin-tools v2025.11.21, reference versions.mk:22; call sites
// reference main.py:155,441,505,511,519,523-524 — table in SURVEY.md §8b).
// The register map of that library is NOT in the reference tree, so the
// read/write semantics here follow what the reference OBSERVES at its call
// sites ("parity unpinned" for the bit-level layout, see DESIGN.md):
//   set_*_mode  stages a value; it becomes current only after reset
//   reset       returns before the device is usable again
//   wait_for_boot blocks until it is; query_* then reads the applied value
#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdarg>
#include <cstdlib>
#include <cstring>
#include <dirent.h>
#include <dlfcn.h>
#include <fstream>
#include <memory>
#include <mutex>
#include <random>
#include <shared_mutex>
#include <sstream>
#include <string>
#include <thread>
#include <vector>

#include "ccm_internal.h"

namespace ccm {

// ------------------------------------------------------------------ error text
static thread_local std::string t_error;
void set_error(const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  t_error = buf;
}
const std::string& last_error() { return t_error; }

using Clock = std::chrono::steady_clock;

// ---------------------------------------------------------------- device model
struct Device {
  ccm_dev_info info{};
  std::mutex mu;  // serialises ops on THIS device only
  // simulated register file
  int cc_mode = CCM_CC_OFF, cc_staged = CCM_CC_OFF;
  int ppcie_mode = CCM_PPCIE_OFF, ppcie_staged = CCM_PPCIE_OFF;
  bool booted = true;
  Clock::time_point boot_ready_at{};
  int reset_ms = 0, boot_ms = 0;
  uint32_t fail_mask = 0;  // ccm_sim_op bits that return CCM_ERR_FAULT
  bool stuck = false;      // reset does not apply staged values
  ScrubDrill drill;        // fault drills of the scrub gate (ccm_internal.h)
  std::string sysfs_path;  // sysfs backend
};

static std::shared_mutex g_table_mu;  // shared for ops, exclusive only for rebuilds
static std::vector<std::unique_ptr<Device>> g_devs;
static int g_backend = -1;
static std::once_flag g_init_once;

// ------------------------------------------------------------------------ trace
static std::mutex g_trace_mu;
static std::vector<std::string> g_trace;
static std::atomic<uint64_t> g_seq{0};

static void trace(const Device& d, const char* op, const char* arg) {
  if (g_backend == CCM_BACKEND_SYSFS) return;
  char line[192];
  uint64_t s = g_seq.fetch_add(1);
  snprintf(line, sizeof line, "%llu %s %s %s", (unsigned long long)s, d.info.bdf, op, arg ? arg : "-");
  std::lock_guard<std::mutex> g(g_trace_mu);
  if (g_trace.size() < (1u << 20)) g_trace.emplace_back(line);
}

static const char* cc_name(int m) {
  switch (m) { case CCM_CC_OFF: return "off"; case CCM_CC_ON: return "on"; case CCM_CC_DEVTOOLS: return "devtools"; }
  return "?";
}
static const char* pp_name(int m) { return m == CCM_PPCIE_ON ? "on" : (m == CCM_PPCIE_OFF ? "off" : "?"); }

// ------------------------------------------------------------ topology builders
static const char* kSimGpuBdf[8] = {"0000:1b:00.0", "0000:43:00.0", "0000:52:00.0", "0000:61:00.0",
                                    "0000:9d:00.0", "0000:c3:00.0", "0000:d1:00.0", "0000:df:00.0"};

static long env_long(const char* name, long dflt) {
  const char* v = getenv(name);
  if (!v || !*v) return dflt;
  return strtol(v, nullptr, 10);
}

static void apply_sim_env(Device& d) {
  d.reset_ms = (int)env_long("CCM_SIM_RESET_MS", 0);
  d.boot_ms = (int)env_long("CCM_SIM_BOOT_MS", 0);
  const char* m = getenv("CCM_SIM_CC_MODE");
  if (m) {
    if (!strcmp(m, "on")) d.cc_mode = CCM_CC_ON;
    else if (!strcmp(m, "devtools")) d.cc_mode = CCM_CC_DEVTOOLS;
    else d.cc_mode = CCM_CC_OFF;
    d.cc_staged = d.cc_mode;
  }
}

static void build_sim(int n_gpus, int n_switches, bool bind_cuda) {
  g_devs.clear();
  // CCM_SIM_BIND_CUDA=0: synthetic GPUs with NO CUDA device behind them (scrub must fail)
  const int ncuda = (bind_cuda && env_long("CCM_SIM_BIND_CUDA", 1) != 0) ? cuda_device_count() : 0;
  for (int i = 0; i < n_gpus; ++i) {
    auto d = std::make_unique<Device>();
    d->info.index = (int)g_devs.size();
    d->info.kind = CCM_KIND_GPU;
    d->info.cc_query_supported = 1;
    d->info.ppcie_query_supported = 1;
    d->info.cuda_ordinal = i < ncuda ? i : -1;
    if (i < 8) snprintf(d->info.bdf, sizeof d->info.bdf, "%s", kSimGpuBdf[i]);
    else snprintf(d->info.bdf, sizeof d->info.bdf, "0001:%02x:00.0", i);
    snprintf(d->info.name, sizeof d->info.name, "NVIDIA H100 (sim)");
    if (d->info.cuda_ordinal >= 0) {
      char bdf[32], name[96];
      uint64_t tot = 0;
      if (cuda_describe(d->info.cuda_ordinal, bdf, sizeof bdf, name, sizeof name, &tot) == CCM_OK)
        d->info.hbm_total_bytes = tot;
    }
    apply_sim_env(*d);
    g_devs.push_back(std::move(d));
  }
  for (int i = 0; i < n_switches; ++i) {
    auto d = std::make_unique<Device>();
    d->info.index = (int)g_devs.size();
    d->info.kind = CCM_KIND_NVSWITCH;
    d->info.cc_query_supported = 0;
    d->info.ppcie_query_supported = 1;
    d->info.cuda_ordinal = -1;
    snprintf(d->info.bdf, sizeof d->info.bdf, "0000:%02x:00.0", 5 + i);
    snprintf(d->info.name, sizeof d->info.name, "NVIDIA NVSwitch (sim)");
    apply_sim_env(*d);
    g_devs.push_back(std::move(d));
  }
}

static void build_cudasim() {
  g_devs.clear();
  const int n = cuda_device_count();
  for (int i = 0; i < n; ++i) {
    auto d = std::make_unique<Device>();
    d->info.index = i;
    d->info.kind = CCM_KIND_GPU;
    d->info.cc_query_supported = 1;
    d->info.ppcie_query_supported = 1;
    d->info.cuda_ordinal = i;
    uint64_t tot = 0;
    if (cuda_describe(i, d->info.bdf, sizeof d->info.bdf, d->info.name, sizeof d->info.name, &tot) != CCM_OK) {
      snprintf(d->info.bdf, sizeof d->info.bdf, "0000:%02x:00.0", i);
      snprintf(d->info.name, sizeof d->info.name, "CUDA device %d", i);
    }
    d->info.hbm_total_bytes = tot;
    apply_sim_env(*d);
    g_devs.push_back(std::move(d));
  }
}

static bool read_hex_file(const std::string& path, unsigned long* out) {
  std::ifstream f(path);
  if (!f) return false;
  std::string s;
  f >> s;
  if (s.empty()) return false;
  *out = strtoul(s.c_str(), nullptr, 16);
  return true;
}

// sysfs: every PCI function with vendor 0x10de whose class is display (0x03xxxx:
// GPUs are 0x030000 / 0x030200) or bridge-other 0x068000 (NVSwitch) — the same
// set the reference describes at main.py:148-150.
static void build_sysfs() {
  g_devs.clear();
  const char* root_env = getenv("CCM_SYSFS_ROOT");
  std::string root = root_env && *root_env ? root_env : "/sys/bus/pci/devices";
  DIR* dir = opendir(root.c_str());
  if (!dir) return;
  std::vector<std::string> names;
  while (dirent* de = readdir(dir)) {
    if (de->d_name[0] == '.') continue;
    names.emplace_back(de->d_name);
  }
  closedir(dir);
  std::sort(names.begin(), names.end());
  const int ncuda = cuda_device_count();
  for (const auto& nm : names) {
    std::string p = root + "/" + nm;
    unsigned long vendor = 0, cls = 0, devid = 0;
    if (!read_hex_file(p + "/vendor", &vendor) || vendor != 0x10de) continue;
    if (!read_hex_file(p + "/class", &cls)) continue;
    const bool is_gpu = (cls >> 16) == 0x03;
    const bool is_sw = (cls >> 8) == 0x0680;
    if (!is_gpu && !is_sw) continue;
    read_hex_file(p + "/device", &devid);
    auto d = std::make_unique<Device>();
    d->info.index = (int)g_devs.size();
    d->info.kind = is_gpu ? CCM_KIND_GPU : CCM_KIND_NVSWITCH;
    d->info.cc_query_supported = is_gpu ? 1 : 0;
    d->info.ppcie_query_supported = 0;  // register map unavailable (see header)
    d->info.cuda_ordinal = -1;
    snprintf(d->info.bdf, sizeof d->info.bdf, "%s", nm.c_str());
    snprintf(d->info.name, sizeof d->info.name, "NVIDIA %s 0x%04lx", is_gpu ? "GPU" : "NVSwitch", devid);
    d->sysfs_path = p;
    for (int o = 0; o < ncuda; ++o) {
      char bdf[32], name[96];
      uint64_t tot = 0;
      if (cuda_describe(o, bdf, sizeof bdf, name, sizeof name, &tot) == CCM_OK && nm == bdf) {
        d->info.cuda_ordinal = o;
        d->info.hbm_total_bytes = tot;
        snprintf(d->info.name, sizeof d->info.name, "%s", name);
      }
    }
    g_devs.push_back(std::move(d));
  }
}

static int do_init(int backend) {
  std::unique_lock<std::shared_mutex> g(g_table_mu);
  if (backend < 0) {
    const char* b = getenv("CCM_BACKEND");
    if (b && !strcmp(b, "sim")) backend = CCM_BACKEND_SIM;
    else if (b && !strcmp(b, "cudasim")) backend = CCM_BACKEND_CUDASIM;
    else if (b && !strcmp(b, "sysfs")) backend = CCM_BACKEND_SYSFS;
    else backend = cuda_device_count() > 0 ? CCM_BACKEND_CUDASIM : CCM_BACKEND_SIM;
  }
  g_backend = backend;
  switch (backend) {
    case CCM_BACKEND_SIM:
      build_sim((int)env_long("CCM_SIM_GPUS", 8), (int)env_long("CCM_SIM_NVSWITCHES", 0), true);
      break;
    case CCM_BACKEND_CUDASIM: build_cudasim(); break;
    case CCM_BACKEND_SYSFS: build_sysfs(); break;
    default: set_error("unknown backend %d", backend); return CCM_ERR_INVALID;
  }
  return CCM_OK;
}

static void ensure_init() {
  std::call_once(g_init_once, [] { do_init(-1); });
}

// Runs `fn(Device&)` with the table held shared and the device locked.
template <class F>
static int with_dev(int dev, F&& fn) {
  ensure_init();
  std::shared_lock<std::shared_mutex> g(g_table_mu);
  if (dev < 0 || (size_t)dev >= g_devs.size()) { set_error("device index %d out of range", dev); return CCM_ERR_NO_DEVICE; }
  Device& d = *g_devs[dev];
  std::lock_guard<std::mutex> l(d.mu);
  return fn(d);
}

int cuda_ordinal_of(int dev) {
  int ord = -1;
  int rc = with_dev(dev, [&](Device& d) { ord = d.info.cuda_ordinal; return CCM_OK; });
  if (rc) return rc;
  if (ord < 0) { set_error("device %d has no CUDA device behind it: the HBM scrub cannot run", dev); return CCM_ERR_NO_CUDA; }
  return ord;
}

static thread_local ScrubDrill t_scrub_drill;  // set for the duration of one scrub_verify_one
const ScrubDrill& current_scrub_drill() { return t_scrub_drill; }
static thread_local ccm_tag_result* t_tag_call = nullptr;  // likewise; nullptr = zero-only call
ccm_tag_result* current_tag_call() { return t_tag_call; }
static thread_local ccm_residue_report* t_residue_call = nullptr;  // likewise; nullptr = no census
ccm_residue_report* current_residue_call() { return t_residue_call; }

int sim_scrub_hook(int dev, ScrubDrill* drill) {
  return with_dev(dev, [&](Device& d) {
    trace(d, "scrub", nullptr);
    if (drill) *drill = g_backend == CCM_BACKEND_SYSFS ? ScrubDrill() : d.drill;
    if (d.fail_mask & CCM_OP_SCRUB) { set_error("injected fault: scrub on %s", d.info.bdf); return (int)CCM_ERR_FAULT; }
    return (int)CCM_OK;
  });
}

// ------------------------------------------------------------------ NVML (dl)
// One loader for every NVML query of the library: libnvidia-ml.so.1 is opened and nvmlInit_v2 called once, and each
// entry point is resolved with dlsym (no link-time NVML).  Only read-only queries are resolved.
struct NvmlCcState { unsigned int environment, ccFeature, devToolsMode; };
struct NvmlRemapHistogram { unsigned int max, high, partial, low, none; };
using NvmlDevice = void*;
struct Nvml {
  void* lib = nullptr;
  int init_rc = -1;   // nvmlInit_v2's return code
  int (*cc_state)(NvmlCcState*) = nullptr;
  int (*handle_by_bus)(const char*, NvmlDevice*) = nullptr;
  int (*ecc_mode)(NvmlDevice, int*, int*) = nullptr;
  int (*error_counter)(NvmlDevice, int, int, int, unsigned long long*) = nullptr;
  int (*remapped_rows)(NvmlDevice, unsigned int*, unsigned int*, unsigned int*, unsigned int*) = nullptr;
  int (*remap_histogram)(NvmlDevice, NvmlRemapHistogram*) = nullptr;
};
constexpr int kNvmlNotSupported = 3;   // NVML_ERROR_NOT_SUPPORTED

// The loaded library, or nullptr with the error text set.
static const Nvml* nvml() {
  static const Nvml n = [] {
    Nvml v;
    v.lib = dlopen("libnvidia-ml.so.1", RTLD_LAZY | RTLD_LOCAL);
    if (!v.lib) return v;
    auto init = (int (*)())dlsym(v.lib, "nvmlInit_v2");
    v.init_rc = init ? init() : -1;
    v.cc_state = (decltype(v.cc_state))dlsym(v.lib, "nvmlSystemGetConfComputeState");
    v.handle_by_bus = (decltype(v.handle_by_bus))dlsym(v.lib, "nvmlDeviceGetHandleByPciBusId_v2");
    v.ecc_mode = (decltype(v.ecc_mode))dlsym(v.lib, "nvmlDeviceGetEccMode");
    v.error_counter = (decltype(v.error_counter))dlsym(v.lib, "nvmlDeviceGetMemoryErrorCounter");
    v.remapped_rows = (decltype(v.remapped_rows))dlsym(v.lib, "nvmlDeviceGetRemappedRows");
    v.remap_histogram = (decltype(v.remap_histogram))dlsym(v.lib, "nvmlDeviceGetRowRemapperHistogram");
    return v;
  }();
  if (!n.lib) { set_error("libnvidia-ml.so.1 not loadable"); return nullptr; }
  if (n.init_rc != 0) { set_error("nvmlInit_v2 failed (%d)", n.init_rc); return nullptr; }
  return &n;
}

// Query-only view of the platform's CC state for the sysfs backend.
static int nvml_cc_state(int* mode) {
  const Nvml* n = nvml();
  if (!n) return CCM_ERR_UNSUPPORTED;
  if (!n->cc_state) { set_error("NVML lacks nvmlSystemGetConfComputeState"); return CCM_ERR_UNSUPPORTED; }
  NvmlCcState s{};
  int rc = n->cc_state(&s);
  if (rc != 0) { set_error("nvmlSystemGetConfComputeState failed (%d)", rc); return rc == kNvmlNotSupported ? CCM_ERR_UNSUPPORTED : CCM_ERR_IO; }
  *mode = s.ccFeature ? (s.devToolsMode ? CCM_CC_DEVTOOLS : CCM_CC_ON) : CCM_CC_OFF;
  return CCM_OK;
}

int hbm_snapshot_bus(const char* bus_id, ccm_hbm_state* out) {
  memset(out, 0, sizeof *out);
  const auto t0 = Clock::now();
  const Nvml* n = nvml();
  int rc = CCM_OK;
  NvmlDevice h = nullptr;
  if (!n) rc = CCM_ERR_UNSUPPORTED;
  else if (!n->handle_by_bus) { set_error("NVML lacks nvmlDeviceGetHandleByPciBusId_v2"); rc = CCM_ERR_UNSUPPORTED; }
  else if (int hr = n->handle_by_bus(bus_id, &h)) { set_error("NVML has no device at %s (%d)", bus_id, hr); rc = CCM_ERR_UNSUPPORTED; }
  if (rc != CCM_OK) {
    for (int32_t& r : out->nvml_rc) r = kNvmlNotSupported;
    out->ms_query = std::chrono::duration<double, std::milli>(Clock::now() - t0).count();
    return rc;
  }
  // Each query: its return code in nvml_rc[k], its bit in `available` when it answered.
  auto note = [&](int k, int qrc, const char* what) {
    out->nvml_rc[k] = qrc;
    if (qrc == 0) out->available |= 1u << k;
    else if (qrc != kNvmlNotSupported && rc == CCM_OK) { set_error("%s on %s failed (%d)", what, bus_id, qrc); rc = CCM_ERR_IO; }
  };
  int cur = 0, pend = 0;
  note(0, n->ecc_mode ? n->ecc_mode(h, &cur, &pend) : kNvmlNotSupported, "nvmlDeviceGetEccMode");
  if (out->available & CCM_HBM_Q_ECC_MODE) { out->ecc_current = cur != 0; out->ecc_pending = pend != 0; }
  constexpr int kCorrected = 0, kUncorrected = 1, kVolatile = 0, kDram = 2, kSram = 7;   // nvml.h enums
  uint64_t* counts[4] = {&out->dram_corrected, &out->dram_uncorrected, &out->sram_corrected, &out->sram_uncorrected};
  for (int k = 0; k < 4; ++k) {
    unsigned long long c = 0;
    note(1 + k, n->error_counter ? n->error_counter(h, k % 2 ? kUncorrected : kCorrected, kVolatile, k < 2 ? kDram : kSram, &c)
                                 : kNvmlNotSupported, "nvmlDeviceGetMemoryErrorCounter");
    if (out->available & (1u << (1 + k))) *counts[k] = c;
  }
  unsigned int corr = 0, unc = 0, pending = 0, failure = 0;
  note(5, n->remapped_rows ? n->remapped_rows(h, &corr, &unc, &pending, &failure) : kNvmlNotSupported,
       "nvmlDeviceGetRemappedRows");
  if (out->available & CCM_HBM_Q_REMAPPED_ROWS) {
    out->rows_corrected = corr;
    out->rows_uncorrected = unc;
    out->remap_pending = pending != 0;
    out->remap_failure = failure != 0;
  }
  NvmlRemapHistogram hist{};
  note(6, n->remap_histogram ? n->remap_histogram(h, &hist) : kNvmlNotSupported, "nvmlDeviceGetRowRemapperHistogram");
  if (out->available & CCM_HBM_Q_REMAP_HISTOGRAM) {
    out->hist_max = hist.max;
    out->hist_high = hist.high;
    out->hist_partial = hist.partial;
    out->hist_low = hist.low;
    out->hist_none = hist.none;
  }
  out->ms_query = std::chrono::duration<double, std::milli>(Clock::now() - t0).count();
  return rc;
}

// ------------------------------------------------------------- register ops
static int check_fault(Device& d, uint32_t op, const char* what) {
  if (d.fail_mask & op) { set_error("injected fault: %s on %s", what, d.info.bdf); return CCM_ERR_FAULT; }
  return CCM_OK;
}
static int check_booted(Device& d, const char* what) {
  // a reset device comes back by itself once its boot time has elapsed; wait_for_boot
  // only blocks until then (a later transition may find devices a failed one left behind)
  if (!d.booted && Clock::now() >= d.boot_ready_at) d.booted = true;
  if (!d.booted) { set_error("%s on %s before wait_for_boot after a reset", what, d.info.bdf); return CCM_ERR_NOT_BOOTED; }
  return CCM_OK;
}

static int op_query_cc(Device& d, int* mode) {
  if (!d.info.cc_query_supported) { set_error("%s does not support CC mode query", d.info.bdf); return CCM_ERR_UNSUPPORTED; }
  if (g_backend == CCM_BACKEND_SYSFS) return nvml_cc_state(mode);
  int rc = check_fault(d, CCM_OP_QUERY_CC, "query_cc_mode");
  if (!rc) rc = check_booted(d, "query_cc_mode");
  if (!rc) *mode = d.cc_mode;
  trace(d, "query_cc_mode", rc ? "error" : cc_name(d.cc_mode));
  return rc;
}
static int op_set_cc(Device& d, int mode) {
  if (mode != CCM_CC_OFF && mode != CCM_CC_ON && mode != CCM_CC_DEVTOOLS) { set_error("invalid CC mode %d", mode); return CCM_ERR_INVALID; }
  if (!d.info.cc_query_supported) { set_error("%s does not support CC mode", d.info.bdf); return CCM_ERR_UNSUPPORTED; }
  if (g_backend == CCM_BACKEND_SYSFS) {
    set_error("staging CC mode needs the gpu-admin-tools register map, which is not part of this build");
    return CCM_ERR_UNSUPPORTED;
  }
  trace(d, "set_cc_mode", cc_name(mode));
  int rc = check_fault(d, CCM_OP_SET_CC, "set_cc_mode");
  if (!rc) rc = check_booted(d, "set_cc_mode");
  if (!rc) d.cc_staged = mode;
  return rc;
}
static int op_query_ppcie(Device& d, int* mode) {
  if (!d.info.ppcie_query_supported) { set_error("%s does not support PPCIe mode query", d.info.bdf); return CCM_ERR_UNSUPPORTED; }
  int rc = check_fault(d, CCM_OP_QUERY_PPCIE, "query_ppcie_mode");
  if (!rc) rc = check_booted(d, "query_ppcie_mode");
  if (!rc) *mode = d.ppcie_mode;
  trace(d, "query_ppcie_mode", rc ? "error" : pp_name(d.ppcie_mode));
  return rc;
}
static int op_set_ppcie(Device& d, int mode) {
  if (mode != CCM_PPCIE_OFF && mode != CCM_PPCIE_ON) { set_error("invalid PPCIe mode %d", mode); return CCM_ERR_INVALID; }
  if (!d.info.ppcie_query_supported) { set_error("%s does not support PPCIe mode", d.info.bdf); return CCM_ERR_UNSUPPORTED; }
  trace(d, "set_ppcie_mode", pp_name(mode));
  int rc = check_fault(d, CCM_OP_SET_PPCIE, "set_ppcie_mode");
  if (!rc) rc = check_booted(d, "set_ppcie_mode");
  if (!rc) d.ppcie_staged = mode;
  return rc;
}
static int op_reset(Device& d) {
  if (g_backend == CCM_BACKEND_SYSFS) {
    // a CUDA context must not be alive on a function that is about to be reset
    if (d.info.cuda_ordinal >= 0) engine_teardown(d.info.cuda_ordinal);
    std::ofstream f(d.sysfs_path + "/reset");
    if (!f) { set_error("cannot open %s/reset", d.sysfs_path.c_str()); return CCM_ERR_IO; }
    f << "1";
    f.flush();
    if (!f) { set_error("write to %s/reset failed", d.sysfs_path.c_str()); return CCM_ERR_IO; }
    d.booted = false;
    return CCM_OK;
  }
  trace(d, "reset_with_os", nullptr);
  int rc = check_fault(d, CCM_OP_RESET, "reset_with_os");
  if (rc) return rc;
  if (d.reset_ms > 0) std::this_thread::sleep_for(std::chrono::milliseconds(d.reset_ms));
  if (!d.stuck) { d.cc_mode = d.cc_staged; d.ppcie_mode = d.ppcie_staged; }
  else { d.cc_staged = d.cc_mode; d.ppcie_staged = d.ppcie_mode; }
  d.booted = false;
  d.boot_ready_at = Clock::now() + std::chrono::milliseconds(d.boot_ms);
  return CCM_OK;
}
static int op_wait_boot(Device& d, int timeout_ms) {
  if (timeout_ms <= 0) timeout_ms = 120000;
  if (g_backend == CCM_BACKEND_SYSFS) {
    const auto deadline = Clock::now() + std::chrono::milliseconds(timeout_ms);
    for (;;) {
      unsigned long vendor = 0;
      if (read_hex_file(d.sysfs_path + "/vendor", &vendor) && vendor == 0x10de) { d.booted = true; return CCM_OK; }
      if (Clock::now() >= deadline) { set_error("%s did not come back within %d ms", d.info.bdf, timeout_ms); return CCM_ERR_TIMEOUT; }
      std::this_thread::sleep_for(std::chrono::milliseconds(50));
    }
  }
  trace(d, "wait_for_boot", nullptr);
  int rc = check_fault(d, CCM_OP_WAIT_BOOT, "wait_for_boot");
  if (rc) return rc;
  if (!d.booted) {
    const auto now = Clock::now();
    if (d.boot_ready_at > now) {
      const auto need = std::chrono::duration_cast<std::chrono::milliseconds>(d.boot_ready_at - now).count();
      if (need > timeout_ms) {
        std::this_thread::sleep_for(std::chrono::milliseconds(timeout_ms));
        set_error("%s did not boot within %d ms", d.info.bdf, timeout_ms);
        return CCM_ERR_TIMEOUT;
      }
      std::this_thread::sleep_until(d.boot_ready_at);
    }
    d.booted = true;
  }
  return CCM_OK;
}

}  // namespace ccm

// ============================================================== public C ABI
using namespace ccm;

extern "C" {

int ccm_abi_version(void) { return CCM_ABI_VERSION; }

const char* ccm_strerror(int status) {
  switch (status) {
    case CCM_OK: return "ok";
    case CCM_ERR_INVALID: return "invalid argument";
    case CCM_ERR_NO_DEVICE: return "no such device";
    case CCM_ERR_UNSUPPORTED: return "operation not supported by this device or backend";
    case CCM_ERR_IO: return "device register / sysfs access failed";
    case CCM_ERR_TIMEOUT: return "timed out waiting for the device to boot";
    case CCM_ERR_CUDA: return "CUDA call failed";
    case CCM_ERR_NOMEM: return "could not obtain the HBM scrub arena";
    case CCM_ERR_DIRTY: return "HBM verify found non-zero bytes after the scrub";
    case CCM_ERR_NO_CUDA: return "no usable CUDA device for the HBM scrub";
    case CCM_ERR_STATE: return "call out of order";
    case CCM_ERR_FAULT: return "injected fault";
    case CCM_ERR_NOT_BOOTED: return "device not booted since its last reset";
    case CCM_ERR_MISMATCH: return "HBM bytes did not hold their address tag (tagged scrub gate)";
    case CCM_ERR_UNCOVERED: return "a scrub gate pass did not walk every mapped byte exactly once (coverage proof)";
    case CCM_ERR_HBM_HEALTH: return "the GPU's HBM ECC or row-remapping state is unfit or unknown (HBM health)";
  }
  return "unknown ccm status";
}

int ccm_last_error(char* buf, size_t cap) {
  const std::string& e = last_error();
  if (buf && cap) {
    size_t n = e.size() < cap - 1 ? e.size() : cap - 1;
    memcpy(buf, e.data(), n);
    buf[n] = 0;
  }
  return (int)e.size();
}

int ccm_init(int backend) {
  std::call_once(g_init_once, [] {});  // an explicit init supersedes the lazy one
  return do_init(backend);
}

int ccm_backend_in_use(void) { ensure_init(); return g_backend; }

int ccm_enumerate(ccm_dev_info* out, int cap, int* n) {
  ensure_init();
  std::shared_lock<std::shared_mutex> g(g_table_mu);
  if (n) *n = (int)g_devs.size();
  if (out)
    for (int i = 0; i < cap && (size_t)i < g_devs.size(); ++i) out[i] = g_devs[i]->info;
  return CCM_OK;
}

int ccm_query_cc_mode(int dev, int* mode) {
  if (!mode) return CCM_ERR_INVALID;
  return with_dev(dev, [&](Device& d) { return op_query_cc(d, mode); });
}
int ccm_set_cc_mode(int dev, int mode) { return with_dev(dev, [&](Device& d) { return op_set_cc(d, mode); }); }
int ccm_query_ppcie_mode(int dev, int* mode) {
  if (!mode) return CCM_ERR_INVALID;
  return with_dev(dev, [&](Device& d) { return op_query_ppcie(d, mode); });
}
int ccm_set_ppcie_mode(int dev, int mode) { return with_dev(dev, [&](Device& d) { return op_set_ppcie(d, mode); }); }
int ccm_reset(int dev) { return with_dev(dev, [&](Device& d) { return op_reset(d); }); }
int ccm_hbm_snapshot(int dev, ccm_hbm_state* out) {
  if (!out) return CCM_ERR_INVALID;
  char bdf[sizeof(ccm_dev_info::bdf)];
  int rc = with_dev(dev, [&](Device& d) { memcpy(bdf, d.info.bdf, sizeof bdf); return (int)CCM_OK; });
  if (rc) { memset(out, 0, sizeof *out); return rc; }
  return hbm_snapshot_bus(bdf, out);
}
int ccm_wait_for_boot(int dev, int timeout_ms) { return with_dev(dev, [&](Device& d) { return op_wait_boot(d, timeout_ms); }); }

// ------------------------------------------------------------------ scrub ABI
static ScrubEngine* engine_of_dev(int dev, int* rc) {
  int ord = cuda_ordinal_of(dev);
  if (ord < 0) { *rc = ord; return nullptr; }
  ScrubEngine* e = engine_for(ord);
  if (!e) { *rc = CCM_ERR_NO_CUDA; return nullptr; }
  *rc = CCM_OK;
  return e;
}
static ScrubEngine* engine_of_ordinal(int ordinal, int* rc) {
  ScrubEngine* e = engine_for(ordinal);
  *rc = e ? CCM_OK : CCM_ERR_NO_CUDA;
  return e;
}

// tag: nullptr for the zero-only gate; otherwise the tagged gate runs, with tag->seed drawn here when 0.
// residue: nullptr, or the census report this call fills.
static int scrub_verify_one(int dev, uint64_t bytes, bool node_fanout, ccm_tag_result* tag, ccm_scrub_result* out,
                            ccm_residue_report* residue = nullptr) {
  if (out) { memset(out, 0, sizeof *out); out->bytes_requested = bytes; }
  if (residue) memset(residue, 0, sizeof *residue);
  if (tag) {
    const uint32_t seed = tag->seed;
    memset(tag, 0, sizeof *tag);
    tag->seed = seed;
    if (tag->seed == 0) {
      std::random_device rd;
      while (tag->seed == 0) tag->seed = (uint32_t)rd();
    }
  }
  ScrubDrill drill;
  int rc = sim_scrub_hook(dev, &drill);
  ScrubEngine* e = rc ? nullptr : engine_of_dev(dev, &rc);
  if (!e) { if (out) out->status = rc; return rc; }
  t_scrub_drill = drill;
  t_tag_call = tag;
  t_residue_call = residue;
  rc = engine_scrub_verify(e, bytes, drill.inject, node_fanout, out);
  t_residue_call = nullptr;
  t_tag_call = nullptr;
  t_scrub_drill = ScrubDrill();
  return rc;
}

int ccm_scrub_verify(int dev, uint64_t bytes, ccm_scrub_result* out) {
  return scrub_verify_one(dev, bytes, false, nullptr, out);
}

int ccm_scrub_verify_tagged(int dev, uint64_t bytes, ccm_tag_result* tag, ccm_scrub_result* out) {
  if (!tag) return CCM_ERR_INVALID;
  return scrub_verify_one(dev, bytes, false, tag, out);
}

int ccm_scrub_release_wait(int dev, double* ms_release, double* ms_waited) {
  if (ms_release) *ms_release = 0;
  if (ms_waited) *ms_waited = 0;
  const int ord = cuda_ordinal_of(dev);
  if (ord < 0) return ord;
  ScrubEngine* e = engine_lookup(ord);  // no engine (or a torn-down one): nothing can be pending — and asking
  return e ? engine_release_wait(e, ms_release, ms_waited) : (int)CCM_OK;  // must not re-create a CUDA context
}

static int scrub_verify_many(int n, const int* devs, uint64_t bytes, ccm_tag_result* tag, ccm_scrub_result* out,
                             double* wall_ms, ccm_residue_report* residue = nullptr) {
  if (n < 0 || (n > 0 && (!devs || !out))) return CCM_ERR_INVALID;
  const auto t0 = Clock::now();
  std::vector<std::thread> th;
  std::vector<std::string> errs(n);
  th.reserve(n);
  for (int i = 0; i < n; ++i)
    th.emplace_back([&, i] {
      int rc = scrub_verify_one(devs[i], bytes, n > 1, tag ? &tag[i] : nullptr, &out[i], residue ? &residue[i] : nullptr);
      if (rc) errs[i] = last_error();
    });
  for (auto& t : th) t.join();
  if (wall_ms) *wall_ms = std::chrono::duration<double, std::milli>(Clock::now() - t0).count();
  for (int i = 0; i < n; ++i)
    if (out[i].status != CCM_OK) { set_error("%s", errs[i].c_str()); return out[i].status; }
  return CCM_OK;
}

int ccm_scrub_verify_many(int n, const int* devs, uint64_t bytes, ccm_scrub_result* out, double* wall_ms) {
  return scrub_verify_many(n, devs, bytes, nullptr, out, wall_ms);
}

int ccm_scrub_verify_many_tagged(int n, const int* devs, uint64_t bytes, ccm_tag_result* tag, ccm_scrub_result* out,
                                 double* wall_ms) {
  if (n > 0 && !tag) return CCM_ERR_INVALID;
  return scrub_verify_many(n, devs, bytes, tag, out, wall_ms);
}

int ccm_scrub_verify_residue(int dev, uint64_t bytes, ccm_tag_result* tag, ccm_residue_report* residue,
                             ccm_scrub_result* out) {
  if (!residue) return CCM_ERR_INVALID;
  return scrub_verify_one(dev, bytes, false, tag, out, residue);
}

int ccm_scrub_verify_many_residue(int n, const int* devs, uint64_t bytes, ccm_tag_result* tag,
                                  ccm_residue_report* residue, ccm_scrub_result* out, double* wall_ms) {
  if (n > 0 && !residue) return CCM_ERR_INVALID;
  return scrub_verify_many(n, devs, bytes, tag, out, wall_ms, residue);
}

int ccm_arena_acquire(int dev, uint64_t bytes, ccm_arena_info* out) {
  int rc; ScrubEngine* e = engine_of_dev(dev, &rc);
  return e ? engine_arena_acquire(e, bytes, out) : rc;
}
int ccm_arena_release(int dev) {
  int rc; ScrubEngine* e = engine_of_dev(dev, &rc);
  return e ? engine_arena_release(e, nullptr) : rc;
}
int ccm_arena_scrub(int dev, int variant, const ccm_launch_cfg* cfg, void* stream, float* ms) {
  int rc; ScrubEngine* e = engine_of_dev(dev, &rc);
  return e ? engine_arena_scrub(e, variant, cfg, stream, ms) : rc;
}
int ccm_arena_verify(int dev, int variant, const ccm_launch_cfg* cfg, void* stream, uint64_t* nonzero, float* ms) {
  int rc; ScrubEngine* e = engine_of_dev(dev, &rc);
  return e ? engine_arena_verify(e, variant, cfg, stream, nonzero, ms) : rc;
}
int ccm_arena_scrub_verify_async(int dev, int sv, int vv, const ccm_launch_cfg* scfg,
                                 const ccm_launch_cfg* vcfg, void* stream) {
  int rc; ScrubEngine* e = engine_of_dev(dev, &rc);
  return e ? engine_arena_scrub_verify_async(e, sv, vv, scfg, vcfg, stream) : rc;
}
int ccm_arena_fetch_count(int dev, void* stream, uint64_t* nonzero) {
  int rc; ScrubEngine* e = engine_of_dev(dev, &rc);
  return e ? engine_arena_fetch_count(e, stream, nonzero) : rc;
}
int ccm_arena_step_times(int dev, int cap, float* scrub_ms, float* verify_ms, int* n) {
  int rc; ScrubEngine* e = engine_of_dev(dev, &rc);
  return e ? engine_arena_step_times(e, cap, scrub_ms, verify_ms, n) : rc;
}
int ccm_arena_fill(int dev, int byte_value, void* stream) {
  int rc; ScrubEngine* e = engine_of_dev(dev, &rc);
  return e ? engine_arena_fill(e, byte_value, stream) : rc;
}
int ccm_arena_fill_random(int dev, uint64_t seed, void* stream) {
  int rc; ScrubEngine* e = engine_of_dev(dev, &rc);
  return e ? engine_arena_fill_random(e, seed, stream) : rc;
}
int ccm_arena_write(int dev, uint64_t offset, const void* host_src, uint64_t bytes) {
  int rc; ScrubEngine* e = engine_of_dev(dev, &rc);
  return e ? engine_arena_rw(e, offset, const_cast<void*>(host_src), bytes, true) : rc;
}
int ccm_arena_read(int dev, uint64_t offset, void* host_dst, uint64_t bytes) {
  int rc; ScrubEngine* e = engine_of_dev(dev, &rc);
  return e ? engine_arena_rw(e, offset, host_dst, bytes, false) : rc;
}

int ccm_region_scrub(int cuda_ordinal, void* dptr, uint64_t bytes, int variant, const ccm_launch_cfg* cfg,
                     void* stream, float* ms) {
  int rc; ScrubEngine* e = engine_of_ordinal(cuda_ordinal, &rc);
  return e ? engine_region_scrub(e, dptr, bytes, variant, cfg, stream, ms) : rc;
}
int ccm_region_verify(int cuda_ordinal, const void* dptr, uint64_t bytes, int variant, const ccm_launch_cfg* cfg,
                      void* stream, uint64_t* nonzero, float* ms) {
  int rc; ScrubEngine* e = engine_of_ordinal(cuda_ordinal, &rc);
  return e ? engine_region_verify(e, dptr, bytes, variant, cfg, stream, nonzero, ms) : rc;
}
int ccm_host_roundtrip(int cuda_ordinal, void* host_buf, uint64_t bytes, uint64_t dev_offset,
                       int sv, int vv, uint64_t* pre, uint64_t* post) {
  if (bytes && !host_buf) return CCM_ERR_INVALID;
  int rc; ScrubEngine* e = engine_of_ordinal(cuda_ordinal, &rc);
  return e ? engine_host_roundtrip(e, host_buf, bytes, dev_offset, sv, vv, pre, post) : rc;
}

int ccm_device_release(int dev) {
  int ord = -1;
  int rc = with_dev(dev, [&](Device& d) { ord = d.info.cuda_ordinal; return (int)CCM_OK; });
  if (rc) return rc;
  return ord >= 0 ? engine_teardown(ord) : (int)CCM_OK;
}

int ccm_device_release_many(int n, const int* devs, double* wall_ms) {
  if (n < 0 || (n > 0 && !devs)) return CCM_ERR_INVALID;
  const auto t0 = Clock::now();
  std::vector<int> rcs(n, CCM_OK);
  std::vector<std::string> errs(n);
  std::vector<std::thread> th;
  th.reserve(n);
  for (int i = 0; i < n; ++i)
    th.emplace_back([&, i] {
      rcs[i] = ccm_device_release(devs[i]);
      if (rcs[i]) errs[i] = last_error();
    });
  for (auto& t : th) t.join();
  if (wall_ms) *wall_ms = std::chrono::duration<double, std::milli>(Clock::now() - t0).count();
  for (int i = 0; i < n; ++i)
    if (rcs[i] != CCM_OK) { set_error("%s", errs[i].c_str()); return rcs[i]; }
  return CCM_OK;
}

uint64_t ccm_kernel_launches(void) { return kernel_launches(); }
const char* ccm_default_kernels(void) { return default_kernel_names(); }

// ------------------------------------------------------------------ sim knobs
int ccm_sim_topology(int n_gpus, int n_switches) {
  std::call_once(g_init_once, [] {});
  if (n_gpus < 0 || n_switches < 0 || n_gpus + n_switches > 4096) return CCM_ERR_INVALID;
  std::unique_lock<std::shared_mutex> g(g_table_mu);
  g_backend = CCM_BACKEND_SIM;
  build_sim(n_gpus, n_switches, true);
  return CCM_OK;
}

static int sim_apply(Device& d, const std::string& k, int64_t v) {
  if (k == "cc_mode") { d.cc_mode = d.cc_staged = (int)v; }
  else if (k == "ppcie_mode") { d.ppcie_mode = d.ppcie_staged = (int)v; }
  else if (k == "cc_supported") d.info.cc_query_supported = v ? 1 : 0;
  else if (k == "ppcie_supported") d.info.ppcie_query_supported = v ? 1 : 0;
  else if (k == "reset_ms") d.reset_ms = (int)v;
  else if (k == "boot_ms") d.boot_ms = (int)v;
  else if (k == "fail_op") d.fail_mask = (uint32_t)v;
  else if (k == "stuck") d.stuck = v != 0;
  else if (k == "cuda_ordinal") d.info.cuda_ordinal = (int)v;
  else if (k == "booted") d.booted = v != 0;
  else if (k == "scrub_inject") d.drill.inject = v < 0 ? 0 : (uint64_t)v;
  else if (k == "tag_inject") d.drill.tag_inject = v < 0 ? 0 : (uint64_t)v;
  else if (k == "scrub_alias") d.drill.alias = v != 0;
  else if (k == "scrub_residue") d.drill.residue = v < 0 ? 0 : (uint64_t)v;
  else if (k == "triage_stay") d.drill.triage_stay = v < 0 ? 0 : (uint64_t)v;
  else if (k == "triage_return") d.drill.triage_return = v < 0 ? 0 : (uint64_t)v;
  else if (k == "cover_skip") d.drill.cover_skip = v < 0 ? 0 : (uint64_t)v;
  else if (k == "probe_mismatch") d.drill.probe_mismatch = v < 0 ? 0 : (uint64_t)v;
  else if (k == "probe_dirt") d.drill.probe_dirt = v < 0 ? 0 : (uint64_t)v;
  else if (k == "probe_skip") d.drill.probe_skip = v < 0 ? 0 : (uint64_t)v;
  else if (k == "probe_skip_step") {
    if (v < 0 || v > 3) { set_error("sim key 'probe_skip_step' takes 0..3, not %lld", (long long)v); return CCM_ERR_INVALID; }
    d.drill.probe_skip_step = v == 0 ? 2 : (int)v;
  }
  else if (k == "report_skip") d.drill.report_skip = v < 0 ? 0 : (uint64_t)v;
  else if (k == "hbm_uncorrected") d.drill.hbm.uncorrected = v < 0 ? 0 : (uint64_t)v;
  else if (k == "hbm_corrected") d.drill.hbm.corrected = v < 0 ? 0 : (uint64_t)v;
  else if (k == "hbm_remap_pending") d.drill.hbm.remap_pending = v != 0;
  else if (k == "hbm_remap_failure") d.drill.hbm.remap_failure = v != 0;
  else if (k == "hbm_unavailable") {
    if (v < 0 || v > (int64_t)ccm_health::kAllQueries) {
      set_error("sim key 'hbm_unavailable' takes ccm_hbm_query bits (0..%u), not %lld", ccm_health::kAllQueries, (long long)v);
      return CCM_ERR_INVALID;
    }
    d.drill.hbm.unavailable = (uint32_t)v;
  }
  else if (k == "report_skip_step") {
    if (v < 0 || v > (int64_t)CCM_REPORT_STEPS) {
      set_error("sim key 'report_skip_step' takes 0..%u, not %lld", CCM_REPORT_STEPS, (long long)v);
      return CCM_ERR_INVALID;
    }
    d.drill.report_skip_step = v == 0 ? (int)CCM_REPORT_DIRT_T3 : (int)v;
  }
  else if (k == "cover_pass") {
    if (v < 0 || v > CCM_PASS_READBACK) { set_error("sim key 'cover_pass' takes 0..3, not %lld", (long long)v); return CCM_ERR_INVALID; }
    d.drill.cover_pass = v == 0 ? (int)CCM_PASS_READBACK : (int)v;
  }
  else if (k == "cover_repeat") {
    if (v < 0 || v > 15) { set_error("sim key 'cover_repeat' takes 0..15, not %lld", (long long)v); return CCM_ERR_INVALID; }
    d.drill.cover_repeat = (uint32_t)v;
  }
  else if (k == "cover_lane_drop") {
    if (v < 0 || v > 512) { set_error("sim key 'cover_lane_drop' takes 0..512, not %lld", (long long)v); return CCM_ERR_INVALID; }
    d.drill.cover_lane_drop = (uint32_t)v;
  }
  else if (k == "scrub_poison" || k == "scrub_flood" || k == "tag_flood") {
    if (v < 0 || v > 255) { set_error("sim key '%s' takes a byte value (0 = off), not %lld", k.c_str(), (long long)v); return CCM_ERR_INVALID; }
    (k == "scrub_poison" ? d.drill.poison : k == "scrub_flood" ? d.drill.flood : d.drill.tag_flood) = (int)v;
  }
  else { set_error("unknown sim key '%s'", k.c_str()); return CCM_ERR_INVALID; }
  return CCM_OK;
}

int ccm_sim_set(int dev, const char* key, int64_t value) {
  if (!key) return CCM_ERR_INVALID;
  ensure_init();
  if (g_backend == CCM_BACKEND_SYSFS) return CCM_OK;
  const std::string k(key);
  if (dev == -1) {
    std::shared_lock<std::shared_mutex> g(g_table_mu);
    for (auto& d : g_devs) {
      std::lock_guard<std::mutex> l(d->mu);
      int rc = sim_apply(*d, k, value);
      if (rc) return rc;
    }
    return CCM_OK;
  }
  return with_dev(dev, [&](Device& d) { return sim_apply(d, k, value); });
}

int ccm_sim_get(int dev, const char* key, int64_t* value) {
  if (!key || !value) return CCM_ERR_INVALID;
  const std::string k(key);
  return with_dev(dev, [&](Device& d) {
    if (k == "cc_mode") *value = d.cc_mode;
    else if (k == "cc_staged") *value = d.cc_staged;
    else if (k == "ppcie_mode") *value = d.ppcie_mode;
    else if (k == "ppcie_staged") *value = d.ppcie_staged;
    else if (k == "booted") *value = d.booted;
    else if (k == "reset_ms") *value = d.reset_ms;
    else if (k == "boot_ms") *value = d.boot_ms;
    else if (k == "fail_op") *value = d.fail_mask;
    else if (k == "stuck") *value = d.stuck;
    else if (k == "cuda_ordinal") *value = d.info.cuda_ordinal;
    else if (k == "scrub_inject") *value = (int64_t)d.drill.inject;
    else if (k == "scrub_poison") *value = d.drill.poison;
    else if (k == "scrub_flood") *value = d.drill.flood;
    else if (k == "tag_inject") *value = (int64_t)d.drill.tag_inject;
    else if (k == "scrub_alias") *value = d.drill.alias;
    else if (k == "scrub_residue") *value = (int64_t)d.drill.residue;
    else if (k == "triage_stay") *value = (int64_t)d.drill.triage_stay;
    else if (k == "triage_return") *value = (int64_t)d.drill.triage_return;
    else if (k == "tag_flood") *value = d.drill.tag_flood;
    else if (k == "cover_skip") *value = (int64_t)d.drill.cover_skip;
    else if (k == "cover_pass") *value = d.drill.cover_pass;
    else if (k == "cover_repeat") *value = d.drill.cover_repeat;
    else if (k == "cover_lane_drop") *value = d.drill.cover_lane_drop;
    else if (k == "probe_mismatch") *value = (int64_t)d.drill.probe_mismatch;
    else if (k == "probe_dirt") *value = (int64_t)d.drill.probe_dirt;
    else if (k == "probe_skip") *value = (int64_t)d.drill.probe_skip;
    else if (k == "probe_skip_step") *value = d.drill.probe_skip_step;
    else if (k == "report_skip") *value = (int64_t)d.drill.report_skip;
    else if (k == "report_skip_step") *value = d.drill.report_skip_step;
    else if (k == "hbm_uncorrected") *value = (int64_t)d.drill.hbm.uncorrected;
    else if (k == "hbm_corrected") *value = (int64_t)d.drill.hbm.corrected;
    else if (k == "hbm_remap_pending") *value = d.drill.hbm.remap_pending;
    else if (k == "hbm_remap_failure") *value = d.drill.hbm.remap_failure;
    else if (k == "hbm_unavailable") *value = d.drill.hbm.unavailable;
    else { set_error("unknown sim key '%s'", k.c_str()); return (int)CCM_ERR_INVALID; }
    return (int)CCM_OK;
  });
}

int ccm_sim_trace(char* buf, size_t cap) {
  std::lock_guard<std::mutex> g(g_trace_mu);
  // concurrent ops append out of seq order; present them sorted by seq
  std::vector<std::string> lines = g_trace;
  std::sort(lines.begin(), lines.end(), [](const std::string& a, const std::string& b) {
    return strtoull(a.c_str(), nullptr, 10) < strtoull(b.c_str(), nullptr, 10);
  });
  std::string all;
  for (auto& l : lines) { all += l; all += '\n'; }
  if (buf && cap) {
    size_t n = all.size() < cap - 1 ? all.size() : cap - 1;
    memcpy(buf, all.data(), n);
    buf[n] = 0;
  }
  return (int)all.size();
}

int ccm_sim_trace_clear(void) {
  std::lock_guard<std::mutex> g(g_trace_mu);
  g_trace.clear();
  g_seq = 0;
  return CCM_OK;
}

}  // extern "C"
