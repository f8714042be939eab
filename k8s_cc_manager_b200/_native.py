"""ctypes binding of libccm.so (include/ccm.h).

This is the ONLY way the Python host code reaches the device shim.  There is no
pure-Python fallback: if the shared library is missing or does not export the ABI
declared in include/ccm.h, importing this module's `lib()` raises — the product
path must fail loudly rather than silently skipping the HBM scrub.
"""
from __future__ import annotations

import ctypes as C
import os
import threading
from pathlib import Path

PKG_DIR = Path(__file__).resolve().parent
LIB_PATH = Path(os.environ.get("CCM_LIB", PKG_DIR / "libccm.so"))

# ---- status codes (include/ccm.h: ccm_status) --------------------------------
OK = 0
ERR_INVALID = -1
ERR_NO_DEVICE = -2
ERR_UNSUPPORTED = -3
ERR_IO = -4
ERR_TIMEOUT = -5
ERR_CUDA = -6
ERR_NOMEM = -7
ERR_DIRTY = -8
ERR_NO_CUDA = -9
ERR_STATE = -10
ERR_FAULT = -11
ERR_NOT_BOOTED = -12
ERR_MISMATCH = -13
ERR_UNCOVERED = -14
ERR_HBM_HEALTH = -15

CC_MODES = {"off": 0, "on": 1, "devtools": 2}
CC_MODE_NAMES = {v: k for k, v in CC_MODES.items()}
PPCIE_MODES = {"off": 0, "on": 1}
PPCIE_MODE_NAMES = {v: k for k, v in PPCIE_MODES.items()}

KIND_GPU, KIND_NVSWITCH = 0, 1
BACKEND_SIM, BACKEND_CUDASIM, BACKEND_SYSFS = 0, 1, 2
BACKENDS = {"sim": BACKEND_SIM, "cudasim": BACKEND_CUDASIM, "sysfs": BACKEND_SYSFS}

SCRUB_AUTO, SCRUB_ST128, SCRUB_ST256, SCRUB_TMA, SCRUB_MEMSET = 0, 1, 2, 3, 4
VERIFY_AUTO, VERIFY_LD128, VERIFY_LD256 = 0, 1, 2
SCRUB_VARIANTS = {"auto": 0, "st128": 1, "st256": 2, "tma": 3, "memset": 4}
VERIFY_VARIANTS = {"auto": 0, "ld128": 1, "ld256": 2}

ABI_VERSION = 2  # include/ccm.h: CCM_ABI_VERSION

OP_QUERY_CC, OP_SET_CC, OP_QUERY_PPCIE, OP_SET_PPCIE, OP_RESET, OP_WAIT_BOOT, OP_SCRUB = 1, 2, 4, 8, 16, 32, 64


class DevInfo(C.Structure):
    _fields_ = [
        ("index", C.c_int32),
        ("kind", C.c_int32),
        ("cc_query_supported", C.c_int32),
        ("ppcie_query_supported", C.c_int32),
        ("cuda_ordinal", C.c_int32),
        ("reserved0", C.c_int32),
        ("hbm_total_bytes", C.c_uint64),
        ("bdf", C.c_char * 32),
        ("name", C.c_char * 96),
    ]


class LaunchCfg(C.Structure):
    _fields_ = [
        ("ctas_per_sm", C.c_int32),
        ("threads_per_cta", C.c_int32),
        ("tile_bytes", C.c_int32),
        ("unroll", C.c_int32),
        ("cache_policy", C.c_int32),
        ("schedule", C.c_int32),
    ]


class ScrubResult(C.Structure):
    _fields_ = [
        ("bytes_requested", C.c_uint64),
        ("bytes_scrubbed", C.c_uint64),
        ("device_total_bytes", C.c_uint64),
        ("nonzero_bytes", C.c_uint64),
        ("ms_acquire", C.c_double),
        ("ms_scrub", C.c_double),
        ("ms_verify", C.c_double),
        ("ms_release", C.c_double),
        ("ms_total", C.c_double),
        ("segments", C.c_int32),
        ("scrub_variant", C.c_int32),
        ("verify_variant", C.c_int32),
        ("sm_count", C.c_int32),
        ("status", C.c_int32),
        ("release_deferred", C.c_int32),
        ("device_free_before", C.c_uint64),
        ("bytes_unreached", C.c_uint64),
        ("ms_release_wait", C.c_double),
        ("ms_gpu_span", C.c_double),
    ]

    def as_dict(self) -> dict:
        return {name: getattr(self, name) for name, _ in self._fields_}


class TagResult(C.Structure):
    """include/ccm.h: ccm_tag_result (seed is in/out: 0 asks the library to draw one)."""
    _fields_ = [
        ("seed", C.c_uint32),
        ("reserved", C.c_uint32),
        ("mismatch_bytes", C.c_uint64),
        ("ms_tag", C.c_double),
        ("ms_check", C.c_double),
        ("va_base", C.c_uint64),
    ]


DIRT_RECORDS = 64  # include/ccm.h: CCM_DIRT_RECORDS


class DirtRecord(C.Structure):
    """include/ccm.h: ccm_dirt_record (one dirty 16-byte window)."""
    _fields_ = [
        ("offset", C.c_uint64),
        ("chunk", C.c_uint32),
        ("mask", C.c_uint16),
        ("reserved", C.c_uint16),
        ("bytes", C.c_uint8 * 16),
    ]


class DirtReport(C.Structure):
    """include/ccm.h: ccm_dirt_report (where a failed read-back found its non-zero bytes)."""
    _fields_ = [
        ("nonzero_bytes", C.c_uint64),
        ("dirty_windows", C.c_uint64),
        ("first_offset", C.c_uint64),
        ("last_offset", C.c_uint64),
        ("va_base", C.c_uint64),
        ("ms_locate", C.c_double),
        ("located", C.c_int32),
        ("nrecords", C.c_int32),
        ("truncated", C.c_int32),
        ("reserved", C.c_int32),
        ("records", DirtRecord * DIRT_RECORDS),
    ]


MISMATCH_KINDS = {1: "zero", 2: "alias", 3: "partial", 4: "foreign"}   # include/ccm.h: ccm_mismatch_kind


class MismatchRecord(C.Structure):
    """include/ccm.h: ccm_mismatch_record (one 16-byte window that did not hold its tags)."""
    _fields_ = [
        ("offset", C.c_uint64),
        ("chunk", C.c_uint32),
        ("mask", C.c_uint16),
        ("kind", C.c_uint16),
        ("source_offset", C.c_uint64),
        ("source_chunk", C.c_uint32),
        ("reserved", C.c_uint32),
        ("bytes", C.c_uint8 * 16),
    ]


class MismatchReport(C.Structure):
    """include/ccm.h: ccm_mismatch_report (where a failed tagged check found bytes off their tags)."""
    _fields_ = [
        ("mismatch_bytes", C.c_uint64),
        ("mismatch_windows", C.c_uint64),
        ("zero_windows", C.c_uint64),
        ("first_offset", C.c_uint64),
        ("last_offset", C.c_uint64),
        ("va_base", C.c_uint64),
        ("seed", C.c_uint32),
        ("located", C.c_int32),
        ("nrecords", C.c_int32),
        ("truncated", C.c_int32),
        ("records", MismatchRecord * DIRT_RECORDS),
    ]


class ResidueRecord(C.Structure):
    """include/ccm.h: ccm_residue_record (one 16-byte window that held non-zero bytes at first touch; no bytes)."""
    _fields_ = [
        ("offset", C.c_uint64),
        ("chunk", C.c_uint32),
        ("mask", C.c_uint16),
        ("reserved", C.c_uint16),
    ]


class ResidueReport(C.Structure):
    """include/ccm.h: ccm_residue_report (what a census call's first pass found before it erased it)."""
    _fields_ = [
        ("residue_bytes", C.c_uint64),
        ("residue_windows", C.c_uint64),
        ("first_offset", C.c_uint64),
        ("last_offset", C.c_uint64),
        ("bytes_examined", C.c_uint64),
        ("va_base", C.c_uint64),
        ("located", C.c_int32),
        ("nrecords", C.c_int32),
        ("truncated", C.c_int32),
        ("reserved", C.c_int32),
        ("records", ResidueRecord * DIRT_RECORDS),
    ]


PAGE_BYTES = 2 << 20  # include/ccm.h: CCM_PAGE_BYTES
BOOK_DIRT, BOOK_MISMATCH, BOOK_RESIDUE = 1, 2, 3   # include/ccm.h: ccm_book


class PageEntry(C.Structure):
    """include/ccm.h: ccm_page_entry (the booked bytes of one 2 MiB page)."""
    _fields_ = [
        ("page", C.c_uint64),
        ("bytes", C.c_uint32),
        ("chunk", C.c_uint32),
    ]


TRIAGE_MAX_HOLD_MS = 10000   # include/ccm.h: CCM_TRIAGE_MAX_HOLD_MS
TRIAGE_CLASSES = {1: "stays", 2: "returns", 3: "clears"}   # include/ccm.h: ccm_triage_class


class TriageReport(C.Structure):
    """include/ccm.h: ccm_triage_report (what kind of dirt a failed read-back found)."""
    _fields_ = [
        ("pages_examined", C.c_uint64),
        ("bytes_examined", C.c_uint64),
        ("stay_pages", C.c_uint64),
        ("stay_bytes", C.c_uint64),
        ("return_pages", C.c_uint64),
        ("return_bytes", C.c_uint64),
        ("clear_pages", C.c_uint64),
        ("clear_bytes", C.c_uint64),
        ("t2_bytes", C.c_uint64),
        ("t3_bytes", C.c_uint64),
        ("t2_first_offset", C.c_uint64),
        ("t2_last_offset", C.c_uint64),
        ("t3_first_offset", C.c_uint64),
        ("t3_last_offset", C.c_uint64),
        ("va_base", C.c_uint64),
        ("ms_hold", C.c_double),
        ("ms_triage", C.c_double),
        ("hold_ms", C.c_uint32),
        ("runs", C.c_int32),
        ("triaged", C.c_int32),
        ("reserved", C.c_int32),
    ]


class TriagePage(C.Structure):
    """include/ccm.h: ccm_triage_page (the class of one page of the dirt page map)."""
    _fields_ = [
        ("page", C.c_uint64),
        ("chunk", C.c_uint32),
        ("cls", C.c_uint32),
        ("dirt_bytes", C.c_uint32),
        ("t2_bytes", C.c_uint32),
        ("t3_bytes", C.c_uint32),
        ("reserved", C.c_uint32),
    ]


COVER_PASSES = ("first", "check", "readback")   # include/ccm.h: ccm_cover_pass_id - 1


class CoverPass(C.Structure):
    """include/ccm.h: ccm_cover_pass (what one pass of a proving call counted against what it mapped)."""
    _fields_ = [
        ("bytes_counted", C.c_uint64),
        ("bytes_missing", C.c_uint64),
        ("bytes_extra", C.c_uint64),
        ("bytes_outside", C.c_uint64),
        ("pages_short", C.c_uint64),
        ("pages_over", C.c_uint64),
        ("first_short_page", C.c_uint64),
        ("ran", C.c_int32),
        ("reserved", C.c_int32),
    ]


class CoverReport(C.Structure):
    """include/ccm.h: ccm_cover_report (the coverage proof of the last product call)."""
    _fields_ = [
        ("bytes_mapped", C.c_uint64),
        ("pages_mapped", C.c_uint64),
        ("va_base", C.c_uint64),
        ("ms_prove", C.c_double),
        ("proved", C.c_int32),
        ("covered", C.c_int32),
        ("passes", CoverPass * 3),
    ]


LEDGER_SLOT_BYTES = 128 << 10   # include/ccm.h: CCM_LEDGER_SLOT_BYTES


class LedgerPass(C.Structure):
    """include/ccm.h: ccm_ledger_pass (what one pass counted per 128 KiB slot against what it mapped)."""
    _fields_ = [
        ("slots_short", C.c_uint64),
        ("slots_over", C.c_uint64),
        ("bytes_missing", C.c_uint64),
        ("bytes_extra", C.c_uint64),
        ("bytes_outside", C.c_uint64),
        ("first_short_slot", C.c_uint64),
        ("first_over_slot", C.c_uint64),
        ("ran", C.c_int32),
        ("reserved", C.c_int32),
    ]


class CoverLedger(C.Structure):
    """include/ccm.h: ccm_cover_ledger (the coverage ledger of the last product call)."""
    _fields_ = [
        ("bytes_mapped", C.c_uint64),
        ("slots_mapped", C.c_uint64),
        ("va_base", C.c_uint64),
        ("ms_ledger", C.c_double),
        ("proved", C.c_int32),
        ("exact", C.c_int32),
        ("passes", LedgerPass * 3),
    ]


class LedgerSlot(C.Structure):
    """include/ccm.h: ccm_ledger_slot (one slot some pass that ran did not count exactly)."""
    _fields_ = [
        ("slot", C.c_uint64),
        ("chunk", C.c_uint32),
        ("expected", C.c_uint32),
        ("count", C.c_uint32 * 3),
        ("reserved", C.c_uint32),
    ]


class CoverPage(C.Structure):
    """include/ccm.h: ccm_cover_page (one page some pass did not count exactly)."""
    _fields_ = [
        ("page", C.c_uint64),
        ("chunk", C.c_uint32),
        ("expected", C.c_uint32),
        ("count", C.c_uint32 * 3),
        ("reserved", C.c_uint32),
    ]


PROBE_STRIDE = 4096   # include/ccm.h: CCM_PROBE_STRIDE
PROBE_WINDOW = 32     # include/ccm.h: CCM_PROBE_WINDOW


class ProbeReport(C.Structure):
    """include/ccm.h: ccm_probe_report (the alias probe of the last product call, or of ccm_region_probe)."""
    _fields_ = [
        ("windows", C.c_uint64),
        ("bytes_probed", C.c_uint64),
        ("mismatch_bytes", C.c_uint64),
        ("mismatch_windows", C.c_uint64),
        ("reread_nonzero_bytes", C.c_uint64),
        ("seed", C.c_uint32),
        ("launches", C.c_uint32),
        ("va_base", C.c_uint64),
        ("ms_probe", C.c_double),
        ("probed", C.c_int32),
        ("reserved", C.c_int32 * 3),
    ]


PROBE_STEPS = ("P1", "P2", "P3")   # include/ccm.h: ccm_probe_cover.step


class ProbeCoverStep(C.Structure):
    """include/ccm.h: ccm_probe_cover_step (what one step of a proven probe counted against the call's windows)."""
    _fields_ = [
        ("windows_counted", C.c_uint64),
        ("windows_missing", C.c_uint64),
        ("windows_extra", C.c_uint64),
        ("windows_outside", C.c_uint64),
        ("pages_short", C.c_uint64),
        ("pages_over", C.c_uint64),
        ("first_short_page", C.c_uint64),
        ("ran", C.c_int32),
        ("reserved", C.c_int32),
    ]


class ProbeCover(C.Structure):
    """include/ccm.h: ccm_probe_cover (the probe proof of the last product call)."""
    _fields_ = [
        ("windows_expected", C.c_uint64),
        ("va_base", C.c_uint64),
        ("ms_prove", C.c_double),
        ("proved", C.c_int32),
        ("covered", C.c_int32),
        ("steps", ProbeCoverStep * 3),
    ]


class ProbeCoverPage(C.Structure):
    """include/ccm.h: ccm_probe_cover_page (one page some probe step did not count exactly)."""
    _fields_ = [
        ("page", C.c_uint64),
        ("chunk", C.c_uint32),
        ("expected", C.c_uint32),
        ("count", C.c_uint32 * 3),
        ("reserved", C.c_uint32),
    ]


# include/ccm.h: ccm_report_cover.step, indexed by ccm_report_step_id - 1
REPORT_STEPS = ("LOCATE", "DIRT_T1", "DIRT_T2", "DIRT_T3", "MISMATCH_T1", "MISMATCH_T2", "MISMATCH_T3")
REPORT_LOCATE, REPORT_DIRT_T1, REPORT_DIRT_T2, REPORT_DIRT_T3, REPORT_MISMATCH_T1, REPORT_MISMATCH_T2, \
    REPORT_MISMATCH_T3 = range(1, 8)


class ReportCoverStep(C.Structure):
    """include/ccm.h: ccm_report_cover_step (what one step of a proven locate pass or triage counted)."""
    _fields_ = [
        ("launches", C.c_uint64),
        ("bytes_expected", C.c_uint64),
        ("bytes_counted", C.c_uint64),
        ("bytes_missing", C.c_uint64),
        ("bytes_extra", C.c_uint64),
        ("bytes_outside", C.c_uint64),
        ("pages_short", C.c_uint64),
        ("pages_over", C.c_uint64),
        ("first_short_page", C.c_uint64),
        ("ran", C.c_int32),
        ("reserved", C.c_int32),
    ]


class ReportCover(C.Structure):
    """include/ccm.h: ccm_report_cover (the report proof of the last product call)."""
    _fields_ = [
        ("va_base", C.c_uint64),
        ("ms_prove", C.c_double),
        ("proved", C.c_int32),
        ("covered", C.c_int32),
        ("steps", ReportCoverStep * len(REPORT_STEPS)),
    ]


class ReportCoverPage(C.Structure):
    """include/ccm.h: ccm_report_cover_page (one page one report step did not count exactly)."""
    _fields_ = [
        ("page", C.c_uint64),
        ("chunk", C.c_uint32),
        ("step", C.c_int32),
        ("expected", C.c_uint32),
        ("counted", C.c_uint32),
    ]


# include/ccm.h: ccm_hbm_query, bit k = 1 << k
HBM_QUERIES = ("ecc_mode", "dram_corrected", "dram_uncorrected", "sram_corrected", "sram_uncorrected", "remapped_rows",
               "remap_histogram")
HBM_REASONS = ("dram_uncorrected", "sram_uncorrected", "remap_pending", "remap_failure", "ecc_off", "no_answer",
               "went_down")   # include/ccm.h: ccm_hbm_reason, bit k = 1 << k
HBM_FIT, HBM_UNFIT, HBM_UNKNOWN = 1, 2, 3   # include/ccm.h: ccm_hbm_verdict
HBM_HEALTH_MODES = {"off": 0, "report": 1, "require": 2}   # ccm_scrub_health's mode


class HbmState(C.Structure):
    """include/ccm.h: ccm_hbm_state (one NVML snapshot of a GPU's ECC and row-remapping state)."""
    _fields_ = [
        ("dram_corrected", C.c_uint64),
        ("dram_uncorrected", C.c_uint64),
        ("sram_corrected", C.c_uint64),
        ("sram_uncorrected", C.c_uint64),
        ("ecc_current", C.c_uint32),
        ("ecc_pending", C.c_uint32),
        ("rows_corrected", C.c_uint32),
        ("rows_uncorrected", C.c_uint32),
        ("remap_pending", C.c_uint32),
        ("remap_failure", C.c_uint32),
        ("hist_max", C.c_uint32),
        ("hist_high", C.c_uint32),
        ("hist_partial", C.c_uint32),
        ("hist_low", C.c_uint32),
        ("hist_none", C.c_uint32),
        ("available", C.c_uint32),
        ("nvml_rc", C.c_int32 * len(HBM_QUERIES)),
        ("reserved", C.c_int32),
        ("ms_query", C.c_double),
    ]


class HbmHealth(C.Structure):
    """include/ccm.h: ccm_hbm_health (the HBM health report of the last product call)."""
    _fields_ = [
        ("before", HbmState),
        ("after", HbmState),
        ("d_dram_corrected", C.c_int64),
        ("d_dram_uncorrected", C.c_int64),
        ("d_sram_corrected", C.c_int64),
        ("d_sram_uncorrected", C.c_int64),
        ("ms_health", C.c_double),
        ("mode", C.c_int32),
        ("verdict", C.c_int32),
        ("reasons", C.c_uint32),
        ("missing_queries", C.c_uint32),
    ]


class ArenaInfo(C.Structure):
    _fields_ = [
        ("bytes", C.c_uint64),
        ("device_total_bytes", C.c_uint64),
        ("device_free_before", C.c_uint64),
        ("segments", C.c_int32),
        ("reserved", C.c_int32),
        ("ms_acquire", C.c_double),
    ]


_P = C.POINTER
_SIGNATURES = {
    # name: (restype, argtypes)
    "ccm_abi_version": (C.c_int, []),
    "ccm_strerror": (C.c_char_p, [C.c_int]),
    "ccm_last_error": (C.c_int, [C.c_char_p, C.c_size_t]),
    "ccm_init": (C.c_int, [C.c_int]),
    "ccm_backend_in_use": (C.c_int, []),
    "ccm_enumerate": (C.c_int, [_P(DevInfo), C.c_int, _P(C.c_int)]),
    "ccm_query_cc_mode": (C.c_int, [C.c_int, _P(C.c_int)]),
    "ccm_set_cc_mode": (C.c_int, [C.c_int, C.c_int]),
    "ccm_query_ppcie_mode": (C.c_int, [C.c_int, _P(C.c_int)]),
    "ccm_set_ppcie_mode": (C.c_int, [C.c_int, C.c_int]),
    "ccm_reset": (C.c_int, [C.c_int]),
    "ccm_wait_for_boot": (C.c_int, [C.c_int, C.c_int]),
    "ccm_scrub_verify": (C.c_int, [C.c_int, C.c_uint64, _P(ScrubResult)]),
    "ccm_scrub_verify_many": (C.c_int, [C.c_int, _P(C.c_int), C.c_uint64, _P(ScrubResult), _P(C.c_double)]),
    "ccm_scrub_verify_tagged": (C.c_int, [C.c_int, C.c_uint64, _P(TagResult), _P(ScrubResult)]),
    "ccm_scrub_verify_many_tagged": (C.c_int, [C.c_int, _P(C.c_int), C.c_uint64, _P(TagResult), _P(ScrubResult),
                                               _P(C.c_double)]),
    "ccm_scrub_release_wait": (C.c_int, [C.c_int, _P(C.c_double), _P(C.c_double)]),
    "ccm_scrub_last_dirt": (C.c_int, [C.c_int, _P(DirtReport)]),
    "ccm_region_locate": (C.c_int, [C.c_int, C.c_void_p, C.c_uint64, C.c_void_p, _P(DirtReport)]),
    "ccm_scrub_last_mismatch": (C.c_int, [C.c_int, _P(MismatchReport)]),
    "ccm_region_tag_check_locate": (C.c_int, [C.c_int, C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p,
                                              _P(MismatchReport)]),
    "ccm_scrub_verify_residue": (C.c_int, [C.c_int, C.c_uint64, _P(TagResult), _P(ResidueReport), _P(ScrubResult)]),
    "ccm_scrub_verify_many_residue": (C.c_int, [C.c_int, _P(C.c_int), C.c_uint64, _P(TagResult), _P(ResidueReport),
                                                _P(ScrubResult), _P(C.c_double)]),
    "ccm_region_census": (C.c_int, [C.c_int, C.c_void_p, C.c_uint64, C.c_int, C.c_uint32, C.c_void_p,
                                    _P(ResidueReport)]),
    "ccm_last_page_map": (C.c_int, [C.c_int, C.c_int, _P(PageEntry), C.c_uint64, _P(C.c_uint64)]),
    "ccm_scrub_triage": (C.c_int, [C.c_int, C.c_uint32]),
    "ccm_scrub_last_triage": (C.c_int, [C.c_int, _P(TriageReport)]),
    "ccm_last_triage_pages": (C.c_int, [C.c_int, _P(TriagePage), C.c_uint64, _P(C.c_uint64)]),
    "ccm_scrub_mismatch_triage": (C.c_int, [C.c_int, C.c_uint32]),
    "ccm_scrub_last_mismatch_triage": (C.c_int, [C.c_int, _P(TriageReport)]),
    "ccm_last_mismatch_triage_pages": (C.c_int, [C.c_int, _P(TriagePage), C.c_uint64, _P(C.c_uint64)]),
    "ccm_scrub_prove": (C.c_int, [C.c_int, C.c_int]),
    "ccm_scrub_last_cover": (C.c_int, [C.c_int, _P(CoverReport)]),
    "ccm_last_cover_pages": (C.c_int, [C.c_int, _P(CoverPage), C.c_uint64, _P(C.c_uint64)]),
    "ccm_scrub_last_ledger": (C.c_int, [C.c_int, _P(CoverLedger)]),
    "ccm_last_ledger_slots": (C.c_int, [C.c_int, _P(LedgerSlot), C.c_uint64, _P(C.c_uint64)]),
    "ccm_scrub_probe": (C.c_int, [C.c_int, C.c_int]),
    "ccm_scrub_last_probe": (C.c_int, [C.c_int, _P(ProbeReport)]),
    "ccm_region_probe": (C.c_int, [C.c_int, C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p, _P(ProbeReport),
                                   _P(MismatchReport)]),
    "ccm_scrub_last_probe_cover": (C.c_int, [C.c_int, _P(ProbeCover)]),
    "ccm_last_probe_cover_pages": (C.c_int, [C.c_int, _P(ProbeCoverPage), C.c_uint64, _P(C.c_uint64)]),
    "ccm_scrub_last_report_cover": (C.c_int, [C.c_int, _P(ReportCover)]),
    "ccm_last_report_cover_pages": (C.c_int, [C.c_int, _P(ReportCoverPage), C.c_uint64, _P(C.c_uint64)]),
    "ccm_hbm_snapshot": (C.c_int, [C.c_int, _P(HbmState)]),
    "ccm_scrub_health": (C.c_int, [C.c_int, C.c_int]),
    "ccm_scrub_last_health": (C.c_int, [C.c_int, _P(HbmHealth)]),
    "ccm_arena_acquire": (C.c_int, [C.c_int, C.c_uint64, _P(ArenaInfo)]),
    "ccm_arena_release": (C.c_int, [C.c_int]),
    "ccm_arena_scrub": (C.c_int, [C.c_int, C.c_int, _P(LaunchCfg), C.c_void_p, _P(C.c_float)]),
    "ccm_arena_verify": (C.c_int, [C.c_int, C.c_int, _P(LaunchCfg), C.c_void_p, _P(C.c_uint64), _P(C.c_float)]),
    "ccm_arena_scrub_verify_async": (C.c_int, [C.c_int, C.c_int, C.c_int, _P(LaunchCfg), _P(LaunchCfg), C.c_void_p]),
    "ccm_arena_fetch_count": (C.c_int, [C.c_int, C.c_void_p, _P(C.c_uint64)]),
    "ccm_arena_step_times": (C.c_int, [C.c_int, C.c_int, _P(C.c_float), _P(C.c_float), _P(C.c_int)]),
    "ccm_arena_fill": (C.c_int, [C.c_int, C.c_int, C.c_void_p]),
    "ccm_arena_fill_random": (C.c_int, [C.c_int, C.c_uint64, C.c_void_p]),
    "ccm_arena_write": (C.c_int, [C.c_int, C.c_uint64, C.c_void_p, C.c_uint64]),
    "ccm_arena_read": (C.c_int, [C.c_int, C.c_uint64, C.c_void_p, C.c_uint64]),
    "ccm_region_scrub": (C.c_int, [C.c_int, C.c_void_p, C.c_uint64, C.c_int, _P(LaunchCfg), C.c_void_p, _P(C.c_float)]),
    "ccm_region_verify": (C.c_int, [C.c_int, C.c_void_p, C.c_uint64, C.c_int, _P(LaunchCfg), C.c_void_p, _P(C.c_uint64), _P(C.c_float)]),
    "ccm_region_tag_fill": (C.c_int, [C.c_int, C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p, _P(C.c_float)]),
    "ccm_region_tag_check_zero": (C.c_int, [C.c_int, C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p, _P(C.c_uint64),
                                            _P(C.c_float)]),
    "ccm_region_prove": (C.c_int, [C.c_int, C.c_void_p, C.c_uint64, C.c_uint32]),
    "ccm_host_roundtrip": (C.c_int, [C.c_int, C.c_void_p, C.c_uint64, C.c_uint64, C.c_int, C.c_int, _P(C.c_uint64), _P(C.c_uint64)]),
    "ccm_device_release": (C.c_int, [C.c_int]),
    "ccm_device_release_many": (C.c_int, [C.c_int, _P(C.c_int), _P(C.c_double)]),
    "ccm_device_memory": (C.c_int, [C.c_int, _P(C.c_uint64), _P(C.c_uint64)]),
    "ccm_kernel_launches": (C.c_uint64, []),
    "ccm_default_kernels": (C.c_char_p, []),
    "ccm_sim_topology": (C.c_int, [C.c_int, C.c_int]),
    "ccm_sim_set": (C.c_int, [C.c_int, C.c_char_p, C.c_int64]),
    "ccm_sim_get": (C.c_int, [C.c_int, C.c_char_p, _P(C.c_int64)]),
    "ccm_sim_trace": (C.c_int, [C.c_char_p, C.c_size_t]),
    "ccm_sim_trace_clear": (C.c_int, []),
}

EXPORTED_SYMBOLS = tuple(_SIGNATURES)

_lib = None
_lib_lock = threading.Lock()


class NativeLibraryError(ImportError):
    """libccm.so is missing or does not match include/ccm.h."""


def lib() -> C.CDLL:
    """Loads libccm.so once and types every entry point.  Raises if unavailable."""
    global _lib
    if _lib is not None:
        return _lib
    with _lib_lock:
        if _lib is not None:
            return _lib
        if not LIB_PATH.exists():
            raise NativeLibraryError(
                f"{LIB_PATH} not found: build it with `python -m k8s_cc_manager_b200.build` "
                "(the CC manager has no host fallback for the device shim)"
            )
        handle = C.CDLL(str(LIB_PATH), mode=C.RTLD_LOCAL)
        for name, (restype, argtypes) in _SIGNATURES.items():
            try:
                fn = getattr(handle, name)
            except AttributeError as exc:
                raise NativeLibraryError(f"{LIB_PATH} does not export {name}") from exc
            fn.restype = restype
            fn.argtypes = argtypes
        if handle.ccm_abi_version() != ABI_VERSION:
            raise NativeLibraryError(f"{LIB_PATH}: ABI version {handle.ccm_abi_version()} != {ABI_VERSION}")
        _lib = handle
    return _lib


def default_kernels() -> tuple:
    """(scrub kernel, verify kernel) AUTO launches, named the way ncu prints them."""
    return tuple(lib().ccm_default_kernels().decode().split(";"))


def strerror(status: int) -> str:
    return lib().ccm_strerror(status).decode()


def last_error() -> str:
    buf = C.create_string_buffer(1024)
    lib().ccm_last_error(buf, len(buf))
    return buf.value.decode(errors="replace")


def launch_cfg(ctas_per_sm: int = 0, threads: int = 0, tile_bytes: int = 0, unroll: int = 0,
               cache_policy: int = 0, schedule: int = 0) -> LaunchCfg:
    """cache_policy: 0 library default, 1 plain, 2 evict_first, 3 streaming, 4 evict_last.
    schedule: 0 library default, 1 static grid-stride, 2 dynamic (atomic chunk grabs)."""
    return LaunchCfg(ctas_per_sm, threads, tile_bytes, unroll, cache_policy, schedule)
