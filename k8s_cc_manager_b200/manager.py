"""CC-mode manager: the reference's transition engine, made concurrent, with the HBM
scrub gate spliced in.

Same surface as the reference entrypoint (reference main.py): class `CCManager` with
the same method names and return values, `create_readiness_file`,
`is_host_cc_enabled`, `main()` with the same flags / env vars, the same input label
(nvidia.com/cc.mode), output labels and exit codes.  What changes is HOW a
transition runs (SURVEY.md §8a rows a1-a7, S):

  reference main.py:502-529          here
  -------------------------------    -------------------------------------------
  for gpu: query/set   (serial)      phase "stage": every GPU at once
  for gpu: reset       (serial)      phase "reset": every staged GPU at once
  for gpu: wait+verify (serial)      phase "boot":  every reset GPU at once
  (nothing)                          phase "scrub": full-HBM zero + read-back on
                                     every reset GPU, concurrently, one CUDA
                                     context per GPU (libccm.so); a GPU whose HBM
                                     does not read back all-zero fails the
                                     transition -> label 'failed'
  set_cc_state_label(mode)           unchanged

Phases are joined before the next one starts, so the reference's ordering
guarantees ("stage all, then reset all, then verify all", main.py:455-459; PPCIe
"set on all devices before any reset", main.py:321-325) still hold.  With
CC_MAX_PARALLEL=1 the engine degenerates to the reference's exact serial
device-op order (that is what the golden-trace parity tests pin).

Fixed on purpose (SURVEY.md §0, §8f N2): the reference calls time.sleep without
importing time (main.py:684), ignores --kubeconfig (main.py:703-707 vs 129-138),
and never validates the mode string before touching hardware.
"""
from __future__ import annotations

import argparse
import inspect
import logging
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path
from typing import Callable, List, Optional, Sequence

from kubernetes import client, config, watch
from kubernetes.client.rest import ApiException

from . import devices as _devices
from .devices import GpuError
from .drain_gate import (
    evict_gpu_operator_components,
    fetch_current_component_labels,
    recover_journaled_labels,
    reschedule_gpu_operator_components,
    set_cc_state_label,
)

logging.basicConfig(level=logging.INFO, format="%(asctime)s - %(name)s - %(levelname)s - %(message)s")
logger = logging.getLogger("k8s-cc-manager")

CC_MODE_CONFIG_LABEL = "nvidia.com/cc.mode"
READINESS_FILE = os.environ.get("CC_READINESS_FILE", "/run/nvidia/validations/.cc-manager-ctr-ready")
VALID_MODES = ("on", "off", "devtools", "ppcie")
SCRUB_SKIPPED_ANNOTATION = "nvidia.com/cc-manager.scrub-skipped"
RESIDUE_MODES = ("off", "report")   # CC_SCRUB_RESIDUE
TRIAGE_MODES = ("off", "report")    # CC_SCRUB_TRIAGE, CC_SCRUB_MISMATCH_TRIAGE
PROOF_MODES = ("off", "require")    # CC_SCRUB_PROOF
ALIAS_PROBE_MODES = ("off", "require")   # CC_SCRUB_ALIAS_PROBE
HBM_HEALTH_MODES = ("off", "report", "require")   # CC_SCRUB_HBM_HEALTH
# How long the dirt and mismatch triages wait before their last re-read of the pages they re-wrote: long enough for an
# agent that still writes this GPU's memory to show itself, short against a transition.
SCRUB_TRIAGE_HOLD_MS = 100

WATCH_TIMEOUT_SECONDS = 300
RECONNECT_DELAY_SECONDS = 5
EVICTION_TIMEOUT_SECONDS = 300


def create_readiness_file() -> None:
    """Touch the file the GPU Operator's validator looks for; never fatal
    (reference main.py:66-78)."""
    try:
        path = Path(READINESS_FILE)
        path.parent.mkdir(parents=True, exist_ok=True)
        path.touch()
        logger.info("Created readiness file: %s", READINESS_FILE)
    except Exception as exc:  # noqa: BLE001 - readiness is best effort
        logger.warning("Failed to create readiness file %s: %s", READINESS_FILE, exc)


def is_host_cc_enabled(sysfs_root: str = "/sys") -> bool:
    """True when the host runs with Intel TDX or AMD SEV-SNP enabled
    (reference main.py:80-103: kvm_intel tdx / kvm_amd sev_snp parameters)."""
    for rel in ("module/kvm_intel/parameters/tdx", "module/kvm_amd/parameters/sev_snp"):
        param = os.path.join(sysfs_root, rel)
        if os.path.exists(param):
            with open(param, "r") as fh:
                if fh.read().strip().lower() in ("y", "1"):
                    return True
    return False


class ScrubFailure(RuntimeError):
    """The HBM scrub gate refused to release a GPU."""


class CCManager:
    """Reconciles the node's GPUs to the CC mode named by the nvidia.com/cc.mode label."""

    def __init__(self, node_name: str, default_mode: str, host_cc: bool, *,
                 kubeconfig: str = "", v1=None,
                 device_source: Optional[Callable[[], tuple]] = None,
                 scrub_mode: Optional[str] = None, scrub_bytes: Optional[int] = None,
                 max_parallel: Optional[int] = None, scrub_check: Optional[str] = None,
                 scrub_residue: Optional[str] = None, scrub_triage: Optional[str] = None,
                 scrub_mismatch_triage: Optional[str] = None, scrub_proof: Optional[str] = None,
                 scrub_alias_probe: Optional[str] = None, scrub_hbm_health: Optional[str] = None):
        env = os.environ
        self.operator_namespace = env.get("OPERATOR_NAMESPACE", "gpu-operator")
        self.evict_operator_components = env.get("EVICT_OPERATOR_COMPONENTS", "true").lower() == "true"
        self.node_name = node_name
        self.default_mode = default_mode
        self.host_cc_capable = host_cc
        self.current_label = None
        self.current_rv = None
        self.last_label = None
        self.max_consecutive_errors = 10

        # --- new knobs (all optional; defaults keep the reference's behaviour + scrub)
        # require: every GPU that went through a reset must pass the gate, a GPU that cannot be
        #          scrubbed fails the transition (fail closed).
        # auto:    GPUs WITHOUT a CUDA device behind them (vfio-bound for passthrough, or CC-on under
        #          a bare-metal driver that cannot run CUDA) are released unscrubbed, loudly: warning
        #          + node annotation; every GPU that can be scrubbed still must pass.
        # skip:    no gate at all (the reference's behaviour).
        self.scrub_mode = (scrub_mode or env.get("CC_SCRUB_MODE", "require")).lower()
        if self.scrub_mode not in ("require", "auto", "skip"):
            raise ValueError(f"CC_SCRUB_MODE must be 'require', 'auto' or 'skip', not {self.scrub_mode!r}")
        if scrub_bytes is None and int(env.get("CC_SCRUB_BYTES", "0")) != 0 and self.scrub_mode != "skip" \
                and env.get("CC_SCRUB_ALLOW_PARTIAL", "false").lower() != "true":
            # a byte-limited scrub is a drill, not a gate: it leaves most of HBM unread
            raise ValueError("CC_SCRUB_BYTES != 0 scrubs only part of HBM; set CC_SCRUB_ALLOW_PARTIAL=true "
                             "to accept that (tests / drills), or leave it 0 for the full-HBM gate")
        self.scrub_bytes = int(scrub_bytes if scrub_bytes is not None else env.get("CC_SCRUB_BYTES", "0"))
        # zero:   zero-fill + read-back.
        # tagged: an address-tagged known answer is written and checked before the zeroing, so memory
        #         the zeroing never reached (a second virtual view of one physical range, a store that
        #         does not land) fails the gate too.  About twice the HBM traffic of 'zero'.
        self.scrub_check = (scrub_check or env.get("CC_SCRUB_CHECK", "zero")).lower()
        if self.scrub_check not in _devices.CHECKS:
            raise ValueError(f"CC_SCRUB_CHECK must be 'zero' or 'tagged', not {self.scrub_check!r}")
        # off:    the gate says nothing about what it erased.
        # report: the gate's first pass also counts and locates what the memory held before it erased it (a census:
        #         one more read of the mapping, no more launches).  Logged and kept in
        #         last_transition["scrub_residue"]; it is a report, never a reason to fail the gate.
        self.scrub_residue = (scrub_residue or env.get("CC_SCRUB_RESIDUE", "off")).lower()
        if self.scrub_residue not in RESIDUE_MODES:
            raise ValueError(f"CC_SCRUB_RESIDUE must be 'off' or 'report', not {self.scrub_residue!r}")
        # off:    a failed read-back reports where the dirt is.
        # report: it also re-zeroes the dirty pages and re-reads them at once and after SCRUB_TRIAGE_HOLD_MS, and says
        #         whether the dirt stays (a hardware or mapping fault), returns (something still writes this GPU's
        #         memory) or clears (a one-time write).  Logged and kept in last_transition["scrub_triage"]; it never
        #         changes the verdict.
        self.scrub_triage = (scrub_triage or env.get("CC_SCRUB_TRIAGE", "off")).lower()
        if self.scrub_triage not in TRIAGE_MODES:
            raise ValueError(f"CC_SCRUB_TRIAGE must be 'off' or 'report', not {self.scrub_triage!r}")
        # off:    a failed tagged check reports where the tags were wrong.
        # report: it also writes the tags over those pages again, checks and zeroes them, and reads them for zeros after
        #         SCRUB_TRIAGE_HOLD_MS, and says whether the mismatch stays (hardware or a broken mapping), returns
        #         (something still writes this GPU's memory) or clears (a one-time write).  Needs CC_SCRUB_CHECK=tagged.
        #         Logged and kept in last_transition["scrub_mismatch_triage"]; it never changes the verdict.
        self.scrub_mismatch_triage = (scrub_mismatch_triage or env.get("CC_SCRUB_MISMATCH_TRIAGE", "off")).lower()
        if self.scrub_mismatch_triage not in TRIAGE_MODES:
            raise ValueError(f"CC_SCRUB_MISMATCH_TRIAGE must be 'off' or 'report', not {self.scrub_mismatch_triage!r}")
        if self.scrub_mismatch_triage == "report" and self.scrub_check != "tagged":
            raise ValueError("CC_SCRUB_MISMATCH_TRIAGE=report triages what the tagged check finds: it needs "
                             f"CC_SCRUB_CHECK=tagged, not {self.scrub_check!r}")
        # off:     the gate's verdict rests on what its kernels counted.
        # require: every pass of the gate also counts, on the device, the bytes it walked on every 2 MiB page, and a GPU
        #          on which a pass missed or repeated a byte fails the gate (ccm_scrub_prove, DESIGN.md §5h).  A check,
        #          not a report: a device that cannot prove its coverage fails the gate.  Logged and kept in
        #          last_transition["scrub_cover"].  Its coverage ledger counts every thread's bytes per 128 KiB slot
        #          (DESIGN.md §5h): a GPU whose ledger is inexact fails the gate.  Logged and kept in
        #          last_transition["scrub_cover_ledger"].  A GPU that failed also proves its locate pass and triages (DESIGN.md
        #          §5k): which pages of its dirt and triage reports rest on a step that missed bytes.  A report, not a
        #          check: it never changes the verdict.  Logged and kept in last_transition["scrub_report_cover"].
        self.scrub_proof = (scrub_proof or env.get("CC_SCRUB_PROOF", "off")).lower()
        if self.scrub_proof not in PROOF_MODES:
            raise ValueError(f"CC_SCRUB_PROOF must be 'off' or 'require', not {self.scrub_proof!r}")
        # off:     the zero gate cannot see a page mapped twice: both views read back zero.
        # require: after a clean read-back, the zero gate also tags, checks and re-reads one 32-byte window per 4 KiB
        #          page (ccm_scrub_probe, DESIGN.md §5i), and a GPU on which a window lost its tags (a page mapped twice)
        #          fails the gate.  A check, not a report: a device that cannot probe fails the gate.  The tagged check
        #          already covers every window, so it is refused with CC_SCRUB_CHECK=tagged.  Logged and kept in
        #          last_transition["scrub_probe"].  With CC_SCRUB_PROOF=require too, the probe is proven (DESIGN.md
        #          §5j): a report whose probe step missed a window fails the gate (and a device call whose probe proof
        #          did not run returns ERR_UNCOVERED).  Logged and kept in last_transition["scrub_probe_cover"].
        self.scrub_alias_probe = (scrub_alias_probe or env.get("CC_SCRUB_ALIAS_PROBE", "off")).lower()
        if self.scrub_alias_probe not in ALIAS_PROBE_MODES:
            raise ValueError(f"CC_SCRUB_ALIAS_PROBE must be 'off' or 'require', not {self.scrub_alias_probe!r}")
        if self.scrub_alias_probe == "require" and self.scrub_check == "tagged":
            raise ValueError("CC_SCRUB_ALIAS_PROBE=require probes the zero gate; CC_SCRUB_CHECK=tagged already checks "
                             "every probe window: use one or the other")
        # off:     the gate judges HBM only by what its kernels read back, and ECC corrects a flipped cell on its way to
        #          them: a memory fault during the gate goes unseen.
        # report:  the gate also reads the GPU's ECC counters and row-remapping state through NVML before and after its
        #          passes (ccm_scrub_health, DESIGN.md §5m).  Logged and kept in last_transition["scrub_hbm_health"].
        # require: a GPU whose uncorrected error count rose during the gate, whose row remap is pending (it needs another
        #          reset before it holds a tenant's data) or failed (RMA), whose ECC is off, or whose state could not be
        #          read, fails the gate.  A check, not a report: a device without the report fails the gate.
        self.scrub_hbm_health = (scrub_hbm_health or env.get("CC_SCRUB_HBM_HEALTH", "off")).lower()
        if self.scrub_hbm_health not in HBM_HEALTH_MODES:
            raise ValueError(f"CC_SCRUB_HBM_HEALTH must be 'off', 'report' or 'require', not {self.scrub_hbm_health!r}")
        self.max_parallel = int(max_parallel if max_parallel is not None else env.get("CC_MAX_PARALLEL", "0"))
        # "full-HBM" is enforced, not assumed: when scrubbing everything (scrub_bytes == 0) a GPU on
        # which less than this fraction of DEVICE memory was zeroed and read back fails the gate
        # (something else still holds HBM, so part of it was NOT scrubbed).  The gate reaches all free
        # HBM down to the last 2 MiB granule: 0.9935 of an H100 80 GB in a process that holds nothing else
        # on the GPU (benchmarks/coverage_probe.py), 0.9915 with torch's context in the same process.  The
        # remainder is the CUDA context's own footprint, which no kernel of that context can map; 0.99 leaves
        # that footprint room to grow by ~0.3 % of the device and fails a GPU that another tenant holds.
        self.scrub_min_coverage = float(env.get("CC_SCRUB_MIN_COVERAGE", "0.99"))
        # A CUDA context must not outlive the gate: it pins HBM, blocks a vfio re-bind and would
        # not survive the next transition's device reset.  (Benchmarks that share the process
        # with other CUDA users switch this off.)
        self.release_cuda_context = env.get("CC_RELEASE_CUDA_CONTEXT", "true").lower() == "true"
        # 'thread': the gate runs inside this process (libccm's concurrent launcher).
        # 'process': it runs in a short-lived `scrub_worker` child, so no CUDA state survives in
        # the daemon and a CUDA fault cannot take the control loop down.
        self.scrub_isolation = env.get("CC_SCRUB_ISOLATION", "thread").lower()
        if self.scrub_isolation not in ("thread", "process"):
            raise ValueError(f"CC_SCRUB_ISOLATION must be 'thread' or 'process', not {self.scrub_isolation!r}")
        self.concurrent_evict_wait = env.get("CC_CONCURRENT_EVICT_WAIT", "false").lower() == "true"
        self.journal_labels = env.get("CC_JOURNAL_COMPONENT_LABELS", "false").lower() == "true"
        self._device_source = device_source or _devices.find_gpus
        self._sleep = time.sleep
        self._pool: Optional[ThreadPoolExecutor] = None
        self._pool_size = 0
        self._gate_gpus: list = []      # GPUs whose gate resources (HBM on its way back, CUDA contexts) are still held
        self.last_transition: dict = {}

        if v1 is not None:
            self.v1 = v1
        else:
            self.v1 = self._connect(kubeconfig)
        logger.info("Initialized CC Manager for node: %s", node_name)
        logger.info("Default CC mode: %s", default_mode or "(none)")
        logger.info("HBM scrub gate: %s (bytes=%s, max_parallel=%s, check=%s)", self.scrub_mode,
                    self.scrub_bytes or "max", self.max_parallel or "all", self.scrub_check)

    @staticmethod
    def _connect(kubeconfig: str):
        """In-cluster config first, then a kubeconfig (reference main.py:129-140);
        unlike the reference, an explicit --kubeconfig path is honoured."""
        try:
            config.load_incluster_config()
            logger.info("Loaded in-cluster Kubernetes configuration")
        except config.ConfigException:
            try:
                if kubeconfig:
                    config.load_kube_config(config_file=kubeconfig)
                    logger.info("Loaded kubeconfig from %s", kubeconfig)
                else:
                    config.load_kube_config()
                    logger.info("Loaded kubeconfig from default location")
            except config.ConfigException as exc:
                logger.error("Failed to load Kubernetes configuration: %s", exc)
                raise
        return client.CoreV1Api()

    # ------------------------------------------------------------------ discovery
    def find_nvidia_devices(self) -> tuple:
        """(devices, count) of ALL NVIDIA PCI functions — GPUs and NVSwitches
        (reference main.py:144-155)."""
        return self._device_source()

    def get_gpus(self) -> list:
        devices, _ = self.find_nvidia_devices()
        return [d for d in devices if d.is_gpu()]

    def get_nvswitches(self) -> list:
        devices, _ = self.find_nvidia_devices()
        return [d for d in devices if d.is_nvswitch()]

    def get_cc_capable_gpus(self) -> list:
        capable = []
        for gpu in self.get_gpus():
            if gpu.is_cc_query_supported:
                capable.append(gpu)
                logger.info("Found CC-capable GPU: %s - %s", gpu.bdf, gpu.name)
            else:
                logger.warning("GPU %s does not support CC mode query", gpu.bdf)
        return capable

    def get_ppcie_capable_devices(self) -> list:
        capable = []
        devices, _ = self.find_nvidia_devices()
        for dev in devices:
            if dev.is_ppcie_query_supported:
                capable.append(dev)
                logger.info("Found PPCIe-capable device: %s - %s", dev.bdf, dev.name)
            else:
                logger.warning("Device %s does not support PPCIe mode query", dev.bdf)
        return capable

    # ------------------------------------------------------------- phase runner
    def _workers(self, n: int) -> int:
        return n if self.max_parallel <= 0 else max(1, min(n, self.max_parallel))

    def _executor(self, n: int) -> ThreadPoolExecutor:
        """One long-lived pool (a thread per device), grown on demand: creating a pool per
        phase costs ~50 us per thread, which is visible next to micro-second register ops."""
        want = self._workers(n)
        if self._pool is None or self._pool_size < want:
            if self._pool is not None:
                self._pool.shutdown(wait=True)
            self._pool = ThreadPoolExecutor(max_workers=want, thread_name_prefix="cc-dev")
            self._pool_size = want
        return self._pool

    def _fan_out(self, items: Sequence, fn: Callable, phase: str) -> list:
        """Run fn(item) for every item — concurrently unless CC_MAX_PARALLEL=1 — and
        join.  The error of the lowest-index failing item is re-raised after the
        join, so a failure is deterministic and no phase is left half-running."""
        items = list(items)
        if not items:
            return []
        started = time.perf_counter()
        try:
            if self._workers(len(items)) == 1:
                return [fn(item) for item in items]  # reference order, stops at first error
            results, errors = [None] * len(items), [None] * len(items)

            def run(i):
                try:
                    results[i] = fn(items[i])
                except BaseException as exc:  # noqa: BLE001 - re-raised below
                    errors[i] = exc

            list(self._executor(len(items)).map(run, range(len(items))))
            for exc in errors:
                if exc is not None:
                    raise exc
            return results
        finally:
            timings = self.last_transition.setdefault("phase_seconds", {})
            timings[phase] = timings.get(phase, 0.0) + (time.perf_counter() - started)

    # ------------------------------------------------------------------- queries
    def mode_is_set(self, gpus: list, mode: str) -> bool:
        """True iff every GPU already reports `mode`; any query error counts as
        "not set" (reference main.py:428-447)."""
        def query(gpu):
            try:
                return gpu.query_cc_mode() == mode
            except Exception as exc:  # noqa: BLE001
                logger.error("Unexpected error getting CC mode on %s: %s", gpu.bdf, exc)
                return False
        # Register reads are micro-seconds: fanning them out costs more than it saves
        # (benchmarks/config1_get_only.py), so the get-only path stays serial and
        # short-circuits exactly like the reference.
        return all(query(g) for g in gpus)

    def ppcie_mode_is_set(self, devices: list) -> bool:
        """reference main.py:298-315."""
        def query(dev):
            try:
                return dev.query_ppcie_mode() == "on"
            except Exception as exc:  # noqa: BLE001
                logger.error("Unexpected error getting PPCIe mode on %s: %s", dev.bdf, exc)
                return False
        return all(query(d) for d in devices)

    # ------------------------------------------------------------ public entry
    def set_cc_mode(self, mode: str) -> bool:
        """Dispatcher (reference main.py:214-263): capability checks, early-outs,
        eviction-gated or direct transition."""
        if not self.host_cc_capable and mode != "off":
            logger.warning("Host doesn't have CC, gpu mode %s specified", mode)
        if mode and mode not in VALID_MODES:
            # The reference would evict and then fail inside the device library;
            # refuse before touching anything, with the same observable outcome.
            logger.error("Invalid CC mode %r (valid: %s)", mode, ", ".join(VALID_MODES))
            set_cc_state_label(self.v1, self.node_name, "failed")
            return False
        if mode == "ppcie":
            return self.set_ppcie_mode()

        gpus = self.get_gpus()
        cc_gpus = self.get_cc_capable_gpus()
        if mode != "off" and len(gpus) != len(cc_gpus):
            missing = {g.bdf for g in gpus} - {g.bdf for g in cc_gpus}
            logger.error("Some GPUs are not cc-capable: %s", missing)
            sys.exit(1)
        if not gpus:
            logger.warning("No GPUs to configure")
            return True
        if not mode:
            logger.info("No CC mode specified, skipping")
            return True
        if not cc_gpus:
            set_cc_state_label(self.v1, self.node_name, "off")
            return True
        if self.mode_is_set(cc_gpus, mode):
            logger.info("All gpus already set to cc %s, skipping", mode)
            return self._publish_already_set(cc_gpus, mode)
        if self.evict_operator_components:
            return self._set_cc_mode_with_eviction(cc_gpus, mode)
        return self._set_cc_mode_direct(cc_gpus, mode)

    def _publish_already_set(self, gpus: list, mode: str) -> bool:
        """reference main.py:255-258: the registers already read `mode`, publish it.  One addition: if the
        node still carries cc.mode.state=failed, the last transition flipped the GPUs and then did NOT pass
        (e.g. the HBM scrub found dirt, or the manager died before the verdict).  Publishing `mode` now would
        turn that failure into a success without a single byte having been checked (ADVICE r1) — so the gate
        runs first.  The check rides on the node read that set_cc_state_label does anyway: the healthy path
        costs exactly the reference's two API verbs, with or without a gate configured."""
        if self.scrub_mode == "skip":
            set_cc_state_label(self.v1, self.node_name, mode)
            return True
        outcome = {"ok": True}

        def regate() -> bool:
            logger.warning("GPUs already read CC mode '%s' but the last transition FAILED: running the HBM scrub "
                           "gate before the state is published", mode)
            self.last_transition = {"mode": mode, "gpus": len(gpus), "phase_seconds": {}, "regate": True}
            t0 = time.perf_counter()
            try:
                self._scrub_gate(gpus)
            except Exception as exc:  # noqa: BLE001 - GpuError, ScrubFailure, anything: stay failed
                logger.error("HBM scrub gate failed again: %s", exc)
                outcome["ok"] = False
            self.last_transition["seconds_to_verdict"] = time.perf_counter() - t0
            return outcome["ok"]

        set_cc_state_label(self.v1, self.node_name, mode, regate=regate)
        self._release_gate_resources()      # no-op unless the gate ran; after the label, as everywhere
        return outcome["ok"]

    def set_ppcie_mode(self) -> bool:
        """Protected-PCIe mode on every GPU and NVSwitch (reference main.py:265-296)."""
        devices, _ = self.find_nvidia_devices()
        ppcie_devices = self.get_ppcie_capable_devices()
        if len(devices) != len(ppcie_devices):
            missing = {d.bdf for d in devices} - {d.bdf for d in ppcie_devices}
            logger.error("Some devices do not support PPCIe mode: %s", missing)
            sys.exit(1)
        if not devices:
            logger.warning("No devices to configure for PPCIe mode")
            return True
        if self.ppcie_mode_is_set(devices):
            logger.info("All devices already in PPCIe mode, skipping")
            set_cc_state_label(self.v1, self.node_name, "ppcie")
            return True
        if self.evict_operator_components:
            return self._set_ppcie_mode_with_eviction(devices)
        return self._set_ppcie_mode_direct(devices)

    # --------------------------------------------------------- transition engine
    def _stage_reset_verify(self, devices: list, *, query: str, stage: str, target: str,
                            what: str) -> list:
        """stage -> (join) -> reset -> (join) -> wait_for_boot + read back.

        `query` / `stage` name the device methods (query_cc_mode/set_cc_mode or the
        PPCIe pair).  Returns the devices that were actually staged and reset.
        """
        def do_stage(dev):
            current = getattr(dev, query)()
            if current == target:
                logger.info("%s %s already in %s mode '%s'", dev.name, dev.bdf, what, target)
                return None
            logger.info("Setting %s mode on %s from '%s' to '%s'", what, dev.bdf, current, target)
            getattr(dev, stage)(target)
            return dev

        staged = [d for d in self._fan_out(devices, do_stage, "stage") if d is not None]
        if not staged:
            return []
        logger.info("Resetting %d device(s) to apply %s mode", len(staged), what)

        def do_reset(dev):
            logger.info("Resetting device %s", dev.bdf)
            dev.reset_with_os()

        self._fan_out(staged, do_reset, "reset")

        def do_boot(dev):
            dev.wait_for_boot()
            seen = getattr(dev, query)()
            if seen != target:
                raise RuntimeError(f"{what} mode verification failed on {dev.bdf}: "
                                   f"expected '{target}', got '{seen}'")
            logger.info("Verified %s mode '%s' on %s", what, target, dev.bdf)

        self._fan_out(staged, do_boot, "boot")
        return staged

    def _scrub_gate(self, reset_devices: list) -> None:
        """NEW stage (SURVEY.md §8a row S): no GPU that went through a CC reset is
        released before its HBM has been zero-filled and read back all-zero.

        Returns as soon as every verdict is in.  What the gate still holds then — HBM on its way
        back to the driver (libccm's reaper) and the CUDA contexts — is given up by
        _release_gate_resources(), which the callers run AFTER the state label is published."""
        gpus = [d for d in reset_devices if d.is_gpu()]
        if not gpus:
            return
        if self.scrub_mode == "skip":
            logger.warning("CC_SCRUB_MODE=skip: releasing %d GPU(s) WITHOUT an HBM scrub", len(gpus))
            self.last_transition["scrub"] = "skipped"
            return
        if self.scrub_mode == "auto":
            blind = [g for g in gpus if not self._can_scrub(g)]
            if blind:
                names = ",".join(g.bdf for g in blind)
                logger.warning("CC_SCRUB_MODE=auto: NO CUDA device behind %s (vfio-bound or CC-on under a driver "
                               "that cannot run CUDA): releasing %d GPU(s) WITHOUT an HBM scrub", names, len(blind))
                self.last_transition["scrub_skipped"] = [g.bdf for g in blind]
                self._annotate({SCRUB_SKIPPED_ANNOTATION: names})
                gpus = [g for g in gpus if self._can_scrub(g)]
                if not gpus:
                    self.last_transition["scrub"] = "skipped"
                    return
            else:
                self._annotate({SCRUB_SKIPPED_ANNOTATION: None})
        self._gate_gpus = list(gpus)
        self._run_scrub(gpus)

    @staticmethod
    def _native_of(gpu):
        """The libccm device that scrubs `gpu`: the device itself, or the one a ScrubbingProxy found by PCI
        address behind a foreign register library; None for anything else."""
        if isinstance(gpu, _devices.NvidiaDevice):
            return gpu
        if isinstance(gpu, _devices.ScrubbingProxy):
            return object.__getattribute__(gpu, "_native")
        return None

    @staticmethod
    def _can_scrub(gpu) -> bool:
        if isinstance(gpu, _devices.ScrubbingProxy):
            return object.__getattribute__(gpu, "_native") is not None
        if isinstance(gpu, _devices.NvidiaDevice):
            return gpu.cuda_ordinal >= 0
        return hasattr(gpu, "scrub_and_verify")

    def _annotate(self, annotations: dict) -> None:
        try:
            self.v1.patch_node(self.node_name, {"metadata": {"annotations": annotations}})
        except Exception as exc:  # noqa: BLE001 - informational only
            logger.warning("Could not update node annotations %s: %s", sorted(annotations), exc)

    def _release_gate_resources(self) -> None:
        """Hands back what the scrub gate held: joins libccm's background HBM release and, with
        CC_RELEASE_CUDA_CONTEXT=true (default), resets each GPU's CUDA primary context — all GPUs
        at once (one native thread each).  Runs after the state label is out, so the driver's
        unmap/release/teardown work overlaps the API round trips instead of delaying the verdict."""
        gpus, self._gate_gpus = self._gate_gpus, []
        if not gpus:
            return
        started = time.perf_counter()

        def attempt(what, fn):
            try:
                fn()
            except Exception as exc:  # noqa: BLE001 - never mask the gate's own verdict
                logger.warning("Could not %s: %s", what, exc)

        in_process = self.scrub_isolation != "process"   # a worker process took its contexts with it
        native = [n for n in map(self._native_of, gpus) if n is not None]      # libccm devices, also behind proxies
        others = [g for g in gpus if self._native_of(g) is None]
        if self.release_cuda_context:
            if native and in_process:
                attempt("release the CUDA contexts", lambda: _devices.release_cuda_contexts(native))
            for gpu in others:
                release = getattr(gpu, "release_cuda_context", None)
                if release is not None:
                    attempt(f"release the CUDA context on {gpu.bdf}", release)
        elif in_process:
            for gpu in gpus:
                wait = getattr(gpu, "wait_scrub_released", None)
                if wait is not None:
                    attempt(f"wait for the HBM release on {gpu.bdf}", wait)
        self.last_transition.setdefault("phase_seconds", {})["release"] = time.perf_counter() - started

    def _scrub_in_worker_process(self, gpus: list) -> list:
        """CC_SCRUB_ISOLATION=process: one child runs the concurrent gate for all GPUs."""
        import json as _json
        import subprocess
        native_cli = Path(__file__).resolve().parent / "ccm-scrub"
        if native_cli.exists() and os.environ.get("CC_SCRUB_WORKER", "native") == "native":
            cmd = [str(native_cli), "--bytes", str(self.scrub_bytes)]   # no interpreter start-up in the child
        else:
            cmd = [sys.executable, "-m", "k8s_cc_manager_b200.scrub_worker", "--bytes", str(self.scrub_bytes)]
        if self.scrub_check != "zero":
            cmd += ["--check", self.scrub_check]
        if self.census:
            cmd += ["--residue"]
        if self.triage:
            cmd += ["--triage", "--triage-hold-ms", str(SCRUB_TRIAGE_HOLD_MS)]
        if self.mismatch_triage:
            cmd += ["--mismatch-triage"] + ([] if self.triage else ["--triage-hold-ms", str(SCRUB_TRIAGE_HOLD_MS)])
        if self.prove:
            cmd += ["--prove"]
        if self.alias_probe:
            cmd += ["--probe"]
        if self.scrub_hbm_health != "off":
            cmd += ["--health", self.scrub_hbm_health]
        for gpu in gpus:
            cmd += ["--bdf", gpu.bdf]
        env = dict(os.environ)
        pkg_parent = str(Path(__file__).resolve().parents[1])
        env["PYTHONPATH"] = pkg_parent + os.pathsep + env.get("PYTHONPATH", "")
        proc = subprocess.run(cmd, capture_output=True, text=True, env=env,
                              timeout=float(os.environ.get("CC_SCRUB_TIMEOUT_SECONDS", "600")))
        lines = [ln for ln in proc.stdout.splitlines() if ln.startswith("{")]
        if proc.returncode not in (0, 3) or not lines:
            raise ScrubFailure(f"scrub worker failed (exit {proc.returncode}): {proc.stderr.strip()[-500:]}")
        payload = _json.loads(lines[-1])
        return [_devices.ScrubReport.from_json(r) for r in payload["reports"]]

    @property
    def prove(self) -> bool:
        return self.scrub_proof == "require"

    @property
    def alias_probe(self) -> bool:
        return self.scrub_alias_probe == "require"

    @property
    def hbm_health_required(self) -> bool:
        return self.scrub_hbm_health == "require"

    def _scrub_call(self, gpu, **kwargs):
        """The one call every per-device gate path makes: with CC_SCRUB_PROOF=require it also asks for the coverage
        proof, with CC_SCRUB_ALIAS_PROBE=require for the alias probe.  A device whose scrub_and_verify cannot take
        `prove` (`probe`) fails the gate: it is never scrubbed without them in its place."""
        if self.prove:
            kwargs["prove"] = True
            try:
                inspect.signature(gpu.scrub_and_verify).bind(self.scrub_bytes, **kwargs)
            except (TypeError, ValueError):
                raise ScrubFailure(f"device {gpu.bdf} cannot prove its HBM coverage (CC_SCRUB_PROOF=require); refusing "
                                   "to release it") from None
        if self.alias_probe:
            kwargs["probe"] = True
            try:
                inspect.signature(gpu.scrub_and_verify).bind(self.scrub_bytes, **kwargs)
            except (TypeError, ValueError):
                raise ScrubFailure(f"device {gpu.bdf} cannot probe its HBM for pages mapped twice "
                                   "(CC_SCRUB_ALIAS_PROBE=require); refusing to release it") from None
        if self.scrub_hbm_health != "off":
            try:
                inspect.signature(gpu.scrub_and_verify).bind(self.scrub_bytes, **kwargs, health=self.scrub_hbm_health)
                kwargs["health"] = self.scrub_hbm_health
            except (TypeError, ValueError):
                if self.hbm_health_required:
                    raise ScrubFailure(f"device {gpu.bdf} cannot report its HBM health (CC_SCRUB_HBM_HEALTH=require); "
                                       "refusing to release it") from None
                logger.warning("Device %s cannot report its HBM health (CC_SCRUB_HBM_HEALTH=report): its gate runs "
                               "without it", gpu.bdf)
        return gpu.scrub_and_verify(self.scrub_bytes, **kwargs)

    def _scrub_many(self, natives: list, **kwargs):
        """The one native fan-out call of the gate, with the coverage proof under CC_SCRUB_PROOF=require and the alias
        probe under CC_SCRUB_ALIAS_PROBE=require."""
        if self.prove:
            kwargs["prove"] = True
        if self.alias_probe:
            kwargs["probe"] = True
        if self.scrub_hbm_health != "off":
            kwargs["health"] = self.scrub_hbm_health
        return _devices.scrub_and_verify_many(natives, self.scrub_bytes, **kwargs)

    def _scrub_checked(self, gpu):
        """The tagged gate on one device.  A device that cannot run it fails the gate: it is never
        scrubbed zero-only in its place."""
        try:
            inspect.signature(gpu.scrub_and_verify).bind(self.scrub_bytes, check=self.scrub_check)
        except (TypeError, ValueError):
            raise ScrubFailure(f"device {gpu.bdf} cannot run the {self.scrub_check} HBM check "
                               f"(CC_SCRUB_CHECK={self.scrub_check}); refusing to release it") from None
        rep = self._scrub_call(gpu, check=self.scrub_check)
        if getattr(rep, "check", "zero") != self.scrub_check:
            raise ScrubFailure(f"device {gpu.bdf} returned a {getattr(rep, 'check', 'zero')} scrub report for "
                               f"CC_SCRUB_CHECK={self.scrub_check}; refusing to release it")
        return rep

    @property
    def census(self) -> bool:
        return self.scrub_residue == "report"

    def _scrub_with_residue(self, gpu):
        """The census call on one device.  A device whose scrub_and_verify cannot take `residue` is scrubbed exactly
        as without the census, with a warning: the census is a report, and its absence never holds a GPU back."""
        try:
            inspect.signature(gpu.scrub_and_verify).bind(self.scrub_bytes, check=self.scrub_check, residue=True)
        except (TypeError, ValueError):
            logger.warning("Device %s cannot report HBM residue (CC_SCRUB_RESIDUE=report): its gate runs without "
                           "the census", gpu.bdf)
            return self._scrub_one(gpu, census=False)
        return self._scrub_call(gpu, check=self.scrub_check, residue=True)

    @property
    def triage(self) -> bool:
        return self.scrub_triage == "report"

    def _scrub_with_triage(self, gpu, census: bool):
        """The triage call on one device (with the census when `census`).  A device whose scrub_and_verify cannot take
        `triage` is scrubbed exactly as without the triage, with a warning: the triage is a report, and its absence
        never holds a GPU back."""
        kwargs = dict(check=self.scrub_check, triage=True, triage_hold_ms=SCRUB_TRIAGE_HOLD_MS)
        if census:
            kwargs["residue"] = True
        try:
            inspect.signature(gpu.scrub_and_verify).bind(self.scrub_bytes, **kwargs)
        except (TypeError, ValueError):
            logger.warning("Device %s cannot triage HBM dirt (CC_SCRUB_TRIAGE=report): its gate runs without the "
                           "triage", gpu.bdf)
            return self._scrub_one(gpu, census)
        rep = self._scrub_call(gpu, **kwargs)
        if getattr(rep, "check", "zero") != self.scrub_check:   # as _scrub_checked: never zero-only in its place
            raise ScrubFailure(f"device {gpu.bdf} returned a {getattr(rep, 'check', 'zero')} scrub report for "
                               f"CC_SCRUB_CHECK={self.scrub_check}; refusing to release it")
        return rep

    @property
    def mismatch_triage(self) -> bool:
        return self.scrub_mismatch_triage == "report"

    def _scrub_with_mismatch_triage(self, gpu):
        """The mismatch triage call on one device (with the dirt triage and the census when they are on).  A device
        whose scrub_and_verify cannot take `mismatch_triage` is scrubbed exactly as without it, with a warning."""
        kwargs = dict(check=self.scrub_check, triage_hold_ms=SCRUB_TRIAGE_HOLD_MS, mismatch_triage=True)
        if self.triage:
            kwargs["triage"] = True
        if self.census:
            kwargs["residue"] = True
        try:
            inspect.signature(gpu.scrub_and_verify).bind(self.scrub_bytes, **kwargs)
        except (TypeError, ValueError):
            logger.warning("Device %s cannot triage HBM tag mismatches (CC_SCRUB_MISMATCH_TRIAGE=report): its gate "
                           "runs without the mismatch triage", gpu.bdf)
            return self._scrub_with_triage(gpu, self.census) if self.triage else self._scrub_one(gpu, self.census)
        rep = self._scrub_call(gpu, **kwargs)
        if getattr(rep, "check", "zero") != self.scrub_check:   # as _scrub_checked: never zero-only in its place
            raise ScrubFailure(f"device {gpu.bdf} returned a {getattr(rep, 'check', 'zero')} scrub report for "
                               f"CC_SCRUB_CHECK={self.scrub_check}; refusing to release it")
        return rep

    def _scrub_one(self, gpu, census: bool):
        if census:
            return self._scrub_with_residue(gpu)
        if self.scrub_check == "zero":
            return self._scrub_call(gpu)   # the call every scrubbing device takes
        return self._scrub_checked(gpu)

    # The window reports a scrub report or GpuError may carry, in the order they are logged: (attribute, key of
    # last_transition that keeps them by bdf, log level, log line).  Residue is what the census found before the gate
    # erased it ("none" included); dirt is where a failed read-back found its non-zero bytes; mismatch is where a
    # failed tagged check found bytes off their tags, and whose tags they hold.
    _REPORT_NOTES = (
        ("residue", "scrub_residue", logging.INFO, "HBM residue on %s: %s"),
        ("dirt", "scrub_dirt", logging.ERROR, "HBM dirt on %s: %s"),
        ("mismatch", "scrub_mismatch", logging.ERROR, "HBM tag mismatch on %s: %s"),
    )
    # Logged after them: whether that dirt stays, returns or clears when its pages are zeroed and read back once more
    # (CC_SCRUB_TRIAGE=report), then whether that mismatch does when its pages are tagged and checked once more
    # (CC_SCRUB_MISMATCH_TRIAGE=report).  They have no page line: each is itself a verdict per page.
    _TRIAGE_NOTES = (("triage", "scrub_triage", logging.ERROR, "HBM dirt triage on %s: %s"),
                     ("mismatch_triage", "scrub_mismatch_triage", logging.ERROR, "HBM mismatch triage on %s: %s"))

    # One more line per report that carries its page map: which 2 MiB pages, and so which allocations, hold its bytes.
    _PAGE_NOTES = {
        "residue": "HBM residue pages on %s: %s",
        "dirt": "HBM dirt pages on %s: %s",
        "mismatch": "HBM tag mismatch pages on %s: %s",
    }

    def _note_reports(self, bdf: str, holder) -> None:
        """Logs every window report `holder` carries and keeps it in last_transition: the gate hands the memory back
        right after the verdict, so this is the only look anyone gets at it.  The coverage proof comes first: INFO when
        every pass covered every byte, ERROR naming the short pass and its pages when not; then its ledger, likewise per
        slot.  The report proof of a GPU
        that failed comes before its dirt and triage lines, which name the pages it left unproven."""
        cover = getattr(holder, "cover", None)
        if cover is not None:
            self.last_transition.setdefault("scrub_cover", {})[bdf] = cover
            logger.log(logging.INFO if cover.covered else logging.ERROR, "HBM coverage proof on %s: %s", bdf,
                       cover.summary())
        ledger = getattr(holder, "ledger", None)
        if ledger is not None:
            self.last_transition.setdefault("scrub_cover_ledger", {})[bdf] = ledger
            logger.log(logging.INFO if ledger.exact else logging.ERROR, "HBM coverage ledger on %s: %s", bdf,
                       ledger.summary())
        probe = getattr(holder, "probe", None)
        if probe is not None:
            self.last_transition.setdefault("scrub_probe", {})[bdf] = probe
            logger.log(logging.INFO if probe.held else logging.ERROR, "HBM alias probe on %s: %s", bdf, probe.summary())
        probe_cover = getattr(holder, "probe_cover", None)
        if probe_cover is not None:
            self.last_transition.setdefault("scrub_probe_cover", {})[bdf] = probe_cover
            logger.log(logging.INFO if probe_cover.covered else logging.ERROR, "HBM alias probe proof on %s: %s", bdf,
                       probe_cover.summary())
        health = getattr(holder, "health", None)
        if health is not None:
            self.last_transition.setdefault("scrub_hbm_health", {})[bdf] = health
            level = logging.INFO if health.fit else logging.ERROR if self.hbm_health_required else logging.WARNING
            logger.log(level, "HBM health on %s: %s", bdf, health.summary())
        report_cover = getattr(holder, "report_cover", None)
        if report_cover is not None:
            self.last_transition.setdefault("scrub_report_cover", {})[bdf] = report_cover
            logger.log(logging.INFO if report_cover.covered else logging.ERROR, "HBM report proof on %s: %s", bdf,
                       report_cover.summary())
        for attr, key, level, line in self._REPORT_NOTES + self._TRIAGE_NOTES:
            report = getattr(holder, attr, None)
            if report is not None:
                self.last_transition.setdefault(key, {})[bdf] = report
                note = report.summary()
                unproven = report_cover.unproven_pages(attr) if report_cover is not None and attr in _devices.REPORT_STEP_OF.values() else []
                if unproven:
                    note += (f" (unproven on pages {', '.join(map(str, unproven))}: a step of the report proof was short "
                             "there)")
                logger.log(level, line, bdf, note)
                pages = getattr(report, "pages", None) if attr in self._PAGE_NOTES else None
                if pages is not None:
                    logger.log(level, self._PAGE_NOTES[attr], bdf, pages.summary())

    def _run_scrub(self, gpus: list) -> None:
        started = time.perf_counter()
        if self.scrub_isolation == "process":
            reports = self._scrub_in_worker_process(gpus)
        elif all(self._native_of(g) is not None for g in gpus) and self._workers(len(gpus)) == len(gpus):
            # ONE native call for the whole node (maps first, then launches: DESIGN.md §6) — also when the
            # register work belongs to a foreign library and libccm only scrubs (ScrubbingProxy)
            natives = [self._native_of(g) for g in gpus]
            if self.mismatch_triage:
                extra = {"residue": True} if self.census else {}
                if self.triage:
                    extra["triage"] = True
                reports, _ = self._scrub_many(natives, check=self.scrub_check, triage_hold_ms=SCRUB_TRIAGE_HOLD_MS,
                                              mismatch_triage=True, **extra)
            elif self.triage:
                extra = {"residue": True} if self.census else {}
                reports, _ = self._scrub_many(natives, check=self.scrub_check, triage=True,
                                              triage_hold_ms=SCRUB_TRIAGE_HOLD_MS, **extra)
            elif self.census:
                reports, _ = self._scrub_many(natives, check=self.scrub_check, residue=True)
            elif self.scrub_check == "zero":
                reports, _ = self._scrub_many(natives)
            else:
                reports, _ = self._scrub_many(natives, check=self.scrub_check)
            for rep, gpu in zip(reports, gpus):
                rep.bdf = gpu.bdf
        else:
            def one(gpu):
                if not hasattr(gpu, "scrub_and_verify"):
                    raise ScrubFailure(f"device {gpu.bdf} offers no HBM scrub; refusing to release it")
                try:
                    if self.mismatch_triage:
                        return self._scrub_with_mismatch_triage(gpu)
                    if self.triage:
                        return self._scrub_with_triage(gpu, self.census)
                    return self._scrub_one(gpu, self.census)
                except GpuError as exc:
                    self._note_reports(gpu.bdf, exc)
                    raise
            reports = self._fan_out(gpus, one, "scrub")
        elapsed = time.perf_counter() - started
        self.last_transition.setdefault("phase_seconds", {})["scrub"] = elapsed
        self.last_transition["scrub"] = reports
        for rep in reports:
            self._note_reports(rep.bdf, rep)
        for rep in reports:
            if self.hbm_health_required:   # the hardware's record comes first: it explains any count below
                health = getattr(rep, "health", None)
                if health is None:
                    raise ScrubFailure(f"HBM scrub on {rep.bdf} carries no HBM health report "
                                       "(CC_SCRUB_HBM_HEALTH=require); refusing to release it")
                if not health.fit:
                    raise ScrubFailure(f"HBM health on {rep.bdf} is {health.verdict_name}: " + "; ".join(health.why()))
            mismatch = getattr(rep, "mismatch_bytes", 0)
            probe_cover = getattr(rep, "probe_cover", None)
            probe_short = probe_cover is not None and not (probe_cover.proved and probe_cover.covered)
            if rep.status != 0 or rep.nonzero_bytes != 0 or mismatch != 0:
                raise ScrubFailure(
                    f"HBM scrub failed on {rep.bdf}: status={rep.status} "
                    f"nonzero_bytes={rep.nonzero_bytes} of {rep.bytes_scrubbed}"
                    + (f" mismatch_bytes={mismatch} (bytes that did not hold their address tag)"
                       if self.scrub_check == "tagged" else "")
                    + (" (a pass did not walk every mapped byte exactly once: see the coverage proof)"
                       if rep.status == _devices.N.ERR_UNCOVERED and not probe_short else "")
                    + (" (a probe window did not hold its tags: see the alias probe)"
                       if getattr(getattr(rep, "probe", None), "mismatch_bytes", 0) else "")
                    + (" (a probe step did not take every window exactly once: see the alias probe proof)"
                       if probe_short else ""))
            if self.prove and getattr(rep, "cover", None) is None:
                raise ScrubFailure(f"HBM scrub on {rep.bdf} carries no coverage proof (CC_SCRUB_PROOF=require); "
                                   "refusing to release it")
            ledger = getattr(rep, "ledger", None)
            if self.prove and ledger is not None and not (ledger.proved and ledger.exact):
                raise ScrubFailure(f"HBM coverage ledger failed on {rep.bdf}: {ledger.summary()}")
            if self.alias_probe and getattr(rep, "probe", None) is None:
                raise ScrubFailure(f"HBM scrub on {rep.bdf} carries no alias probe (CC_SCRUB_ALIAS_PROBE=require); "
                                   "refusing to release it")
            if self.prove and self.alias_probe and probe_short:
                raise ScrubFailure(f"HBM alias probe proof failed on {rep.bdf}: {probe_cover.summary()}")
            if self.scrub_bytes == 0 and rep.coverage < self.scrub_min_coverage:
                raise ScrubFailure(
                    f"HBM scrub on {rep.bdf} covered only {100 * rep.coverage:.2f}% of device memory "
                    f"(< {100 * self.scrub_min_coverage:.1f}%): {(rep.device_total_bytes - rep.bytes_scrubbed) >> 20} MiB "
                    f"were not scrubbed ({rep.bytes_unreached >> 20} MiB free but unmappable, the rest held by other contexts)")
            logger.info("Scrubbed %s: %.1f GiB (%.2f%% of HBM, %d MiB of free HBM unreached) zeroed at %.0f GB/s, "
                        "verified at %.0f GB/s, 0 non-zero bytes",
                        rep.bdf, rep.bytes_scrubbed / 2**30, 100 * rep.coverage, rep.bytes_unreached >> 20,
                        rep.scrub_gbs, rep.verify_gbs)
        logger.info("HBM scrub gate passed on %d GPU(s) in %.3f s", len(reports), elapsed)

    def _set_cc_mode_direct(self, gpus: list, mode: str) -> bool:
        """PPCIe-off pre-step, then CC stage/reset/verify, then the scrub gate
        (reference main.py:449-542)."""
        logger.info("Setting CC mode to '%s' on %d GPU(s)", mode, len(gpus))
        self.last_transition = {"mode": mode, "gpus": len(gpus), "phase_seconds": {}}
        t0 = time.perf_counter()
        try:
            all_devices, _ = self.find_nvidia_devices()
            ppcie_devices = [d for d in all_devices if d.is_ppcie_query_supported]
            reset_for_ppcie = self._stage_reset_verify(
                ppcie_devices, query="query_ppcie_mode", stage="set_ppcie_mode", target="off", what="PPCIe")
            reset_for_cc = self._stage_reset_verify(
                gpus, query="query_cc_mode", stage="set_cc_mode", target=mode, what="CC")
            by_bdf = {d.bdf: d for d in reset_for_ppcie if d.is_gpu()}
            by_bdf.update({d.bdf: d for d in reset_for_cc})
            self._scrub_gate(list(by_bdf.values()))
        except GpuError as exc:
            logger.error("GPU error setting CC mode: %s", exc)
            return self._finish_transition("failed", t0)
        except Exception as exc:  # noqa: BLE001 - any failure marks the node failed
            logger.error("Unexpected error setting CC mode: %s", exc)
            return self._finish_transition("failed", t0)
        logger.info("Successfully set CC mode to '%s' on all GPUs", mode)
        return self._finish_transition(mode, t0)

    def _finish_transition(self, state: str, t0: float) -> bool:
        """Publishes the outcome (reference main.py:531-542), THEN gives the gate's GPU resources
        back; `seconds_to_verdict` is what the label waited for, `seconds` the whole call."""
        self.last_transition["seconds_to_verdict"] = time.perf_counter() - t0
        set_cc_state_label(self.v1, self.node_name, state)
        self._release_gate_resources()
        self.last_transition["seconds"] = time.perf_counter() - t0
        return state != "failed"

    def _set_ppcie_mode_direct(self, devices: list) -> bool:
        """reference main.py:317-391: PPCIe off where it is not (each device on its
        own: set, reset, wait), then stage 'on' everywhere, reset together, verify."""
        logger.info("Setting PPCIe mode on %d device(s)", len(devices))
        self.last_transition = {"mode": "ppcie", "gpus": len(devices), "phase_seconds": {}}
        t0 = time.perf_counter()
        try:
            def force_off(dev):
                current = dev.query_ppcie_mode()
                if current == "off":
                    logger.info("Device %s PPCIe mode already off", dev.bdf)
                    return None
                logger.info("Setting PPCIe mode off on %s (current: %s)", dev.bdf, current)
                dev.set_ppcie_mode("off")
                dev.reset_with_os()
                dev.wait_for_boot()
                return dev

            cycled = [d for d in self._fan_out(devices, force_off, "ppcie-off") if d is not None]
            staged = self._stage_reset_verify(
                devices, query="query_ppcie_mode", stage="set_ppcie_mode", target="on", what="PPCIe")
            by_bdf = {d.bdf: d for d in cycled}
            by_bdf.update({d.bdf: d for d in staged})
            self._scrub_gate(list(by_bdf.values()))
        except GpuError as exc:
            logger.error("GPU error setting PPCIe mode: %s", exc)
            return self._finish_transition("failed", t0)
        except Exception as exc:  # noqa: BLE001
            logger.error("Unexpected error setting PPCIe mode: %s", exc)
            return self._finish_transition("failed", t0)
        logger.info("Successfully set PPCIe mode on all devices")
        return self._finish_transition("ppcie", t0)

    def _with_eviction(self, what: str, transition: Callable[[], bool]) -> bool:
        """Pause operator components, run the transition, restore them — the
        restore runs even when the transition failed (reference main.py:544-578)."""
        component_labels = fetch_current_component_labels(self.v1, self.node_name)
        logger.info("Evicting GPU operator components before %s mode change", what)
        if not evict_gpu_operator_components(
                self.v1, self.node_name, self.operator_namespace, component_labels,
                timeout=EVICTION_TIMEOUT_SECONDS,
                concurrent_wait=self.concurrent_evict_wait, journal_annotation=self.journal_labels):
            logger.error("Failed to evict GPU operator components")
            return False
        result = transition()
        logger.info("Rescheduling GPU operator components")
        if not reschedule_gpu_operator_components(self.v1, self.node_name, component_labels,
                                                  journal_annotation=self.journal_labels):
            logger.error("Failed to reschedule GPU operator components")
            result = False
        return result

    def _set_cc_mode_with_eviction(self, gpus: list, mode: str) -> bool:
        return self._with_eviction("CC", lambda: self._set_cc_mode_direct(gpus, mode))

    def _set_ppcie_mode_with_eviction(self, devices: list) -> bool:
        return self._with_eviction("PPCIe", lambda: self._set_ppcie_mode_direct(devices))

    # ------------------------------------------------------------- control plane
    def get_node_cc_mode_label(self) -> None:
        """Refresh current_label / current_rv from the API server; exits on failure
        (reference main.py:580-598)."""
        try:
            node = self.v1.read_node(self.node_name)
        except ApiException as exc:
            logger.error("Failed to read node labels: %s", exc)
            sys.exit(1)
        labels = node.metadata.labels or {}
        self.last_label = self.current_label
        self.current_label = labels.get(CC_MODE_CONFIG_LABEL, "")
        self.current_rv = node.metadata.resource_version

    def with_default(self, label) -> str:
        if label:
            return label
        logger.info("Applying default CC mode: %s", self.default_mode)
        return self.default_mode

    def recover_interrupted_transition(self) -> bool:
        """SURVEY.md §8f N1.  The reference keeps the operator components' ORIGINAL deploy labels only
        in memory between evict and reschedule (main.py:556-576): a manager that dies in between
        leaves every component 'paused-for-cc-mode-change' for good.  With
        CC_JOURNAL_COMPONENT_LABELS=true the originals are journaled in a node annotation before the
        pause; a journal found at start-up means exactly that crash — the labels are restored (and
        the journal cleared) before anything else, and the normal reconcile below then re-runs the
        transition, re-evicting from the restored values.  Returns True if a journal was replayed."""
        if not self.journal_labels:
            return False
        journaled = recover_journaled_labels(self.v1, self.node_name)
        if journaled is None:
            return False
        logger.warning("Found the component-label journal of an INTERRUPTED transition on node %s: restoring %s",
                       self.node_name, journaled)
        if not reschedule_gpu_operator_components(self.v1, self.node_name, journaled, journal_annotation=True):
            logger.error("Could not restore the journaled component labels; will retry on the next start")
            return False
        return True

    def watch_and_apply(self) -> None:
        """Apply the current label once, signal readiness, then follow the node's
        label forever (reference main.py:600-684)."""
        self.recover_interrupted_transition()
        self.get_node_cc_mode_label()
        self.set_cc_mode(self.with_default(self.current_label))
        create_readiness_file()
        logger.info("Starting watch on node '%s' for label '%s' current_label: %s",
                    self.node_name, CC_MODE_CONFIG_LABEL, self.current_label)

        applied_label = self.current_label
        consecutive_errors = 0
        selector = f"metadata.name={self.node_name}"

        def reconcile(origin: str):
            nonlocal applied_label
            if self.current_label == applied_label:
                return
            logger.info("Label changed: '%s' -> '%s' (%s)", applied_label, self.current_label, origin)
            applied_label = self.current_label
            self.set_cc_mode(self.with_default(self.current_label))

        while True:
            try:
                stream = watch.Watch().stream(
                    self.v1.list_node, field_selector=selector,
                    resource_version=self.current_rv, timeout_seconds=WATCH_TIMEOUT_SECONDS)
                logger.info("Starting watch from ResourceVersion: %s", self.current_rv)
                for event in stream:
                    kind = event["type"]
                    if kind == "ERROR":
                        logger.error("Watch error event: %s", event)
                        consecutive_errors += 1
                        break  # reconnect right away
                    consecutive_errors = 0
                    node = event["object"]
                    rv = getattr(node.metadata, "resource_version", None)
                    if rv:
                        self.current_rv = rv
                    if kind in ("ADDED", "MODIFIED"):
                        self.current_label = (node.metadata.labels or {}).get(CC_MODE_CONFIG_LABEL, "")
                        reconcile(f"event: {kind}")
            except ApiException as exc:
                consecutive_errors += 1
                if consecutive_errors >= self.max_consecutive_errors:
                    logger.error("Watch failed %d times consecutively, treating as fatal error",
                                 consecutive_errors)
                    raise RuntimeError(
                        f"Watch failed after {consecutive_errors} consecutive errors: {exc}") from exc
                if exc.status == 410:
                    logger.warning("ResourceVersion %s is too old (410 Gone). "
                                   "Performing re-sync and starting fresh watch.", self.current_rv)
                    self.get_node_cc_mode_label()
                    reconcile("re-sync")
                logger.info("Reconnecting in %d seconds...", RECONNECT_DELAY_SECONDS)
                self._sleep(RECONNECT_DELAY_SECONDS)

    def run(self) -> None:
        self.watch_and_apply()


def _device_source_from_env():
    """Which library does the register work (query / stage / reset / wait_for_boot)?

    CC_DEVICE_LIBRARY=gpu-admin-tools: NVIDIA/gpu-admin-tools, looked up where the reference looks
        (<app dir>/gpu-admin-tools, reference main.py:30-31); libccm.so adds only the HBM scrub,
        matched by PCI address.
    CC_DEVICE_LIBRARY=libccm: libccm.so for both.
    unset: gpu-admin-tools when that directory exists (the reference image ships it), else libccm.

    The production entrypoint never drives a SIMULATED register file by accident (ADVICE r1: with no
    env set, libccm picks its cudasim/sim backend and the manager would publish cc.mode.state=on
    without having touched hardware): a simulated backend is refused unless CCM_ALLOW_SIM=1."""
    tools = os.environ.get("GPU_ADMIN_TOOLS_PATH") or os.path.join(
        os.path.dirname(os.path.abspath(sys.argv[0] or ".")), "gpu-admin-tools")
    choice = os.environ.get("CC_DEVICE_LIBRARY", "").lower()
    if not choice:
        choice = "gpu-admin-tools" if os.path.isdir(tools) else "libccm"
    if choice == "libccm":
        from . import _native  # noqa: PLC0415
        backend = _native.lib().ccm_backend_in_use()
        if backend in (_native.BACKEND_SIM, _native.BACKEND_CUDASIM) \
                and os.environ.get("CCM_ALLOW_SIM", "").lower() not in ("1", "true", "yes"):
            name = {v: k for k, v in _native.BACKENDS.items()}[backend]
            raise RuntimeError(
                f"libccm selected its SIMULATED register backend ({name}): refusing to manage CC mode on "
                "simulated registers.  Use CC_DEVICE_LIBRARY=gpu-admin-tools (real register access) or "
                "CCM_BACKEND=sysfs, or set CCM_ALLOW_SIM=1 for drills and tests")
        return None
    if choice != "gpu-admin-tools":
        raise ValueError(f"CC_DEVICE_LIBRARY must be 'libccm' or 'gpu-admin-tools', not {choice!r}")
    sys.path.insert(0, tools)
    from pci.devices import find_gpus as foreign_find_gpus  # noqa: PLC0415 - optional dependency
    return _devices.with_scrub(foreign_find_gpus)


def build_arg_parser() -> argparse.ArgumentParser:
    env = os.environ
    parser = argparse.ArgumentParser(description="NVIDIA CC Manager For Kubernetes (H100-native)")
    parser.add_argument("--kubeconfig", default=env.get("KUBECONFIG", ""),
                        help="Absolute path to the kubeconfig file")
    parser.add_argument("--default-cc-mode", "-m", default=env.get("DEFAULT_CC_MODE", "on"),
                        help="CC mode to be set by default when node label nvidia.com/cc.mode is not "
                             "applied. Valid modes: 'on', 'off', 'devtools', 'ppcie'")
    parser.add_argument("--node-name", default=env.get("NODE_NAME", ""),
                        help="Kubernetes node name (default: $NODE_NAME)")
    parser.add_argument("--debug", action="store_true", help="Enable debug logging")
    parser.add_argument("--scrub-mode", default=None, choices=("require", "auto", "skip"),
                        help="HBM scrub gate after every CC transition (default: $CC_SCRUB_MODE or require)")
    parser.add_argument("--scrub-check", default=None, choices=("zero", "tagged"),
                        help="what the scrub gate checks: zero read-back, or an address-tagged known answer "
                             "before it (default: $CC_SCRUB_CHECK or zero)")
    parser.add_argument("--scrub-residue", default=None, choices=RESIDUE_MODES,
                        help="report what the scrub gate found in HBM before it erased it (never fails the gate; "
                             "default: $CC_SCRUB_RESIDUE or off)")
    parser.add_argument("--scrub-triage", default=None, choices=TRIAGE_MODES,
                        help="after a failed read-back, re-zero and re-read the dirty pages and report whether the dirt "
                             "stays, returns or clears (never changes the verdict; default: $CC_SCRUB_TRIAGE or off)")
    parser.add_argument("--scrub-mismatch-triage", default=None, choices=TRIAGE_MODES,
                        help="with --scrub-check tagged, after a failed check, re-tag, check and re-read the pages off "
                             "their tags and report whether the mismatch stays, returns or clears (never changes the "
                             "verdict; default: $CC_SCRUB_MISMATCH_TRIAGE or off)")
    parser.add_argument("--scrub-proof", default=None, choices=PROOF_MODES,
                        help="require: every pass of the scrub gate counts the bytes it walked on every 2 MiB page, and "
                             "a GPU whose pass missed or repeated a byte fails the gate (default: $CC_SCRUB_PROOF or off)")
    parser.add_argument("--scrub-alias-probe", default=None, choices=ALIAS_PROBE_MODES,
                        help="require: after a clean read-back, the zero gate tags, checks and re-reads one 32-byte "
                             "window per 4 KiB page, and a GPU with a page mapped twice fails the gate (not with "
                             "--scrub-check tagged; default: $CC_SCRUB_ALIAS_PROBE or off)")
    parser.add_argument("--scrub-hbm-health", default=None, choices=HBM_HEALTH_MODES,
                        help="report: read the GPUs' ECC counters and row-remapping state before and after the gate; "
                             "require: a GPU whose memory failed during the gate, with a pending or failed row remap, "
                             "ECC off, or a state that cannot be read fails the gate (default: $CC_SCRUB_HBM_HEALTH or "
                             "off)")
    return parser


def main(argv: Optional[List[str]] = None) -> None:
    args = build_arg_parser().parse_args(argv)
    if args.debug:
        logger.setLevel(logging.DEBUG)
        logging.getLogger("nvidia_gpu_tools").setLevel(logging.DEBUG)
        logging.getLogger("k8s_cc_manager_b200").setLevel(logging.DEBUG)
    if not args.node_name:
        logger.error("NODE_NAME environment variable must be set for k8s-cc-manager")
        sys.exit(1)

    default_mode = args.default_cc_mode
    host_cc = is_host_cc_enabled()
    if not host_cc:
        if default_mode != "off":
            logger.warning("Overriding default CC mode: %s to off because the host does not support CC",
                           default_mode)
        default_mode = "off"

    try:
        CCManager(node_name=args.node_name, default_mode=default_mode, host_cc=host_cc,
                  kubeconfig=args.kubeconfig, scrub_mode=args.scrub_mode, scrub_check=args.scrub_check,
                  scrub_residue=args.scrub_residue, scrub_triage=args.scrub_triage,
                  scrub_mismatch_triage=args.scrub_mismatch_triage, scrub_proof=args.scrub_proof,
                  scrub_alias_probe=args.scrub_alias_probe, scrub_hbm_health=args.scrub_hbm_health,
                  device_source=_device_source_from_env()).run()
    except KeyboardInterrupt:
        logger.info("Shutting down...")
        sys.exit(0)
    except Exception as exc:  # noqa: BLE001
        logger.error("Fatal error: %s", exc, exc_info=True)
        sys.exit(1)


if __name__ == "__main__":
    main()
