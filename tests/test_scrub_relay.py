"""The relayed whole-HBM gate on the CPU: the accounting and settle rules (csrc/ccm_relay.h, compiled with g++ -Wall
-Werror) over a table of cases against a Python restatement; ccm-scrub's usage refusals; the relay's failure path on the
sim backend without a CUDA device (leg A fails, no leg B, nothing left running); a --relay-first child that ends when its
stdin closes and when the process that started it dies; and RelayReport's JSON and summary."""
from __future__ import annotations

import json
import os
import shutil
import signal
import subprocess
import sys
import time
from pathlib import Path

import pytest

import test_cover_proof as TC
from k8s_cc_manager_b200 import _native as N
from k8s_cc_manager_b200.devices import RelayReport, ScrubReport, reports_from_payload

ROOT = Path(__file__).resolve().parents[1]
CSRC = ROOT / "k8s_cc_manager_b200" / "csrc"
INCLUDE = ROOT / "include"
CLI = ROOT / "k8s_cc_manager_b200" / "ccm-scrub"
MiB = 1 << 20
GiB = 1 << 30
U64 = (1 << 64) - 1


def gxx():
    cc = shutil.which("g++")
    if cc is None:
        pytest.skip("no g++")
    return cc


def cli():
    if not CLI.exists():
        pytest.skip("ccm-scrub is not built")
    return str(CLI)


# ---------------------------------------------------------------------------------- the rules
RULE_MAIN = r"""
#include <cstdio>
#include <iostream>
#include <string>
#include "ccm_relay.h"
// stdin: "a <8 inputs>" -> the outputs; "s <n> <free ms> x n" -> polls settled done free
int main() {
  std::string kind;
  while (std::cin >> kind) {
    if (kind == "a") {
      ccm_relay::Inputs in;
      std::cin >> in.total >> in.a_free_before >> in.a_unreached >> in.b_free_held >> in.b_free_settled >>
          in.b_free_before >> in.b_unreached >> in.marked;
      const ccm_relay::Relay r = ccm_relay::account(in);
      printf("%llu %llu %llu %llu %llu %.12f\n", (unsigned long long)r.footprint_a, (unsigned long long)r.freed,
             (unsigned long long)r.held, (unsigned long long)r.growth, (unsigned long long)r.unreached, r.coverage);
    } else {
      int n;
      std::cin >> n;
      ccm_relay::Settle s;
      int reads = 0;
      for (int k = 0; k < n; ++k) {
        unsigned long long f;
        double ms;
        std::cin >> f >> ms;
        if (!s.done) { s.read(f, ms); ++reads; }
      }
      printf("%d %d %d %llu %d\n", s.polls, (int)s.settled, (int)s.done, (unsigned long long)s.free_bytes, reads);
    }
  }
  return 0;
}
"""

SETTLE_POLL_MS, SETTLE_FLAT, SETTLE_DEADLINE_MS = 5.0, 4, 2000.0


def account(total, a_free, a_unr, b_held, b_settled, b_before, b_unr, marked=0):
    """The rule of csrc/ccm_relay.h, restated: (footprint_a, freed, held, growth, unreached, coverage)."""
    footprint = max(0, total - a_free)
    freed = max(0, b_settled - b_held)
    held = max(0, footprint - freed)
    growth = max(0, b_settled - b_before)
    unreached = min(U64, held + growth + a_unr + b_unr)
    coverage = 1 - min(unreached, total) / total if total else 0.0
    return footprint, freed, held, growth, unreached, coverage


def settle(series):
    """The settle rule, restated: (polls, settled, done, last free) after feeding (free, ms) reads until it is done."""
    polls = flat = 0
    last = 0
    for free, ms in series:
        flat = flat + 1 if polls and free == last else 1
        last = free
        polls += 1
        if flat >= SETTLE_FLAT:
            return polls, 1, 1, last
        if ms >= SETTLE_DEADLINE_MS:
            return polls, 0, 1, last
    return polls, 0, 0, last


TOTAL = 85_017_493_504
A_FREE = 84_464_041_984
FOOT = TOTAL - A_FREE
CASES = {
    # one GPU alone: A's exit gives back exactly its footprint
    "alone": (TOTAL, A_FREE, 1_245_184, A_FREE - FOOT, A_FREE, A_FREE, 1_245_184, 0),
    # another process holds 3 GiB through both legs: it is what neither leg reached
    "other process": (TOTAL, A_FREE - 3 * GiB, 2 * MiB, A_FREE - 3 * GiB - FOOT, A_FREE - 3 * GiB,
                      A_FREE - 3 * GiB, 2 * MiB, 0),
    # the drill's marker comes back with A's exit: freed exceeds the footprint A started with
    "marker": (TOTAL, A_FREE, 2 * MiB, A_FREE - FOOT - 256 * MiB, A_FREE, A_FREE, 2 * MiB, 256 * MiB),
    # leg B allocated 8 MiB after the hand-over
    "late growth": (TOTAL, A_FREE, 2 * MiB, A_FREE - FOOT, A_FREE, A_FREE - 8 * MiB, 2 * MiB, 0),
    # nonsense reads clamp instead of wrapping
    "free above total": (1000, 2000, 0, 5000, 3000, 9000, 0, 0),
    "settled below held": (1000, 100, 0, 800, 500, 500, 0, 0),
    "huge unreached": (1000, 900, U64 - 5, 0, 0, 0, 10, 0),
    "no total": (0, 0, 0, 0, 0, 0, 0, 0),
}
SETTLES = {
    "rises then flat": [(100, 0), (200, 5), (300, 10), (300, 15), (300, 20), (300, 25), (999, 30)],
    "flat at once": [(500, 0), (500, 5), (500, 10), (500, 15)],
    "never flat": [(k, 5.0 * k) for k in range(500)],
    "too few reads": [(7, 0), (7, 5)],
}


@pytest.fixture(scope="module")
def rule_binary(tmp_path_factory):
    d = tmp_path_factory.mktemp("relay")
    (d / "rule.cpp").write_text(RULE_MAIN)
    subprocess.run([gxx(), "-std=c++17", "-Wall", "-Wextra", "-Werror", "-O1", "-I", str(INCLUDE), "-I", str(CSRC),
                    str(d / "rule.cpp"), "-o", str(d / "rule")], check=True)
    return d / "rule"


def test_the_settle_constants_are_the_restated_ones():
    text = (CSRC / "ccm_relay.h").read_text()
    assert f"kSettlePollMs = {SETTLE_POLL_MS}" in text and f"kSettleFlat = {SETTLE_FLAT};" in text
    assert f"kSettleDeadlineMs = {SETTLE_DEADLINE_MS}" in text and SETTLE_DEADLINE_MS <= 5000


def test_the_accounting_rule_matches_its_restatement(rule_binary):
    text = "".join("a " + " ".join(map(str, c)) + "\n" for c in CASES.values())
    lines = subprocess.run([str(rule_binary)], input=text, capture_output=True, text=True, check=True).stdout.splitlines()
    got = {}
    for (name, case), line in zip(CASES.items(), lines):
        *ints, cov = line.split()
        want = account(*case)
        assert [int(x) for x in ints] == list(want[:5]), name
        assert float(cov) == pytest.approx(want[5], abs=1e-11), name
        got[name] = want
    assert len(lines) == len(CASES)
    assert got["alone"][2] == 0 and got["alone"][1] == FOOT and got["alone"][5] == pytest.approx(1 - 2_490_368 / TOTAL)
    assert got["other process"][2] == 3 * GiB
    assert got["marker"][1] == FOOT + 256 * MiB and got["marker"][2] == 0
    assert got["late growth"][3] == 8 * MiB and got["late growth"][4] == 12 * MiB
    assert got["free above total"][:4] == (0, 0, 0, 0)
    assert got["settled below held"][1] == 0 and got["settled below held"][2] == 900
    assert got["huge unreached"][4] == U64 and got["huge unreached"][5] == 0.0
    assert got["no total"][5] == 0.0


def test_the_settle_rule_matches_its_restatement(rule_binary):
    text = "".join(f"s {len(s)} " + " ".join(f"{f} {ms}" for f, ms in s) + "\n" for s in SETTLES.values())
    lines = subprocess.run([str(rule_binary)], input=text, capture_output=True, text=True, check=True).stdout.splitlines()
    got = {}
    for (name, series), line in zip(SETTLES.items(), lines):
        polls, settled, done, free, _ = (int(x) for x in line.split())
        assert (polls, settled, done, free) == settle(series), name
        got[name] = (polls, settled, done, free)
    assert got["rises then flat"] == (6, 1, 1, 300)
    assert got["flat at once"] == (4, 1, 1, 500)
    assert got["never flat"] == (401, 0, 1, 400)   # the read at the deadline ends the wait
    assert got["too few reads"][2] == 0


# ---------------------------------------------------------------------------------- ccm-scrub
@pytest.mark.parametrize("args", [["--relay", "--bytes", "1"], ["--relay-mark-mib", "8"],
                                  ["--relay-mark-mib", "0", "--relay"], ["--relay", "--relay-first"]],
                         ids=["bytes", "mark-without-relay", "mark-zero", "both-legs"])
def test_usage_refusals(args):
    proc = subprocess.run([cli(), "--backend", "sim", *args, "--all"], capture_output=True, text=True, timeout=60)
    assert proc.returncode == 2 and proc.stdout == "", proc.stderr


def sim_env():
    return dict(os.environ, CCM_SIM_BIND_CUDA="0", CCM_SIM_GPUS="2")


def alive(pid: int) -> bool:
    try:
        state = Path(f"/proc/{pid}/stat").read_text().rsplit(")", 1)[1].split()[0]
    except (FileNotFoundError, ProcessLookupError):
        return False
    return state != "Z"


def test_a_failed_first_leg_ends_the_relay(tmp_path):
    proc = subprocess.run([cli(), "--backend", "sim", "--relay", "--all"], capture_output=True, text=True, timeout=60,
                          env=sim_env())
    assert proc.returncode == 3, proc.stderr
    out = json.loads(proc.stdout.splitlines()[-1])
    assert len(out["reports"]) >= 1 and len(out["reports"]) == len(out["first"]["reports"])
    for rep, first in zip(out["reports"], out["first"]["reports"]):
        assert rep["status"] == N.ERR_NO_CUDA and rep["relay"] is None
        assert {**rep, "relay": None} == {**first, "relay": None}   # leg A's report, verbatim
    assert "relay" not in out["first"]["reports"][0]
    assert not alive(out["first_pid"])
    reps = reports_from_payload(out)
    assert [r.relay for r in reps] == [None] * len(reps)


def test_a_plain_call_prints_no_relay_members():
    proc = subprocess.run([cli(), "--backend", "sim", "--all"], capture_output=True, text=True, timeout=60, env=sim_env())
    out = json.loads(proc.stdout)
    assert proc.returncode == 3 and set(out) == {"wall_ms", "reports"} and "relay" not in out["reports"][0]


def first_leg(stdin, **kw):
    return subprocess.Popen([cli(), "--backend", "sim", "--relay-first", "--all"], stdin=stdin,
                            stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, env=sim_env(), **kw)


def test_the_first_leg_ends_when_its_stdin_closes():
    child = first_leg(subprocess.PIPE)
    try:
        payload = json.loads(child.stdout.readline())
        released = json.loads(child.stdout.readline())
        assert payload["reports"][0]["status"] == N.ERR_NO_CUDA
        assert released["clean"] == 0 and [r["bdf"] for r in released["released"]] == \
            [r["bdf"] for r in payload["reports"]] and released["released"][0]["marked"] == 0
        time.sleep(0.3)
        assert child.poll() is None   # it waits for its stdin to close
        t0 = time.monotonic()
        child.stdin.close()
        assert child.wait(timeout=5) == 3   # its gate failed
        assert time.monotonic() - t0 < 1.0
    finally:
        child.kill()
        child.wait()


STARTER = r"""
import os, subprocess, sys, time
child = subprocess.Popen(sys.argv[1:], stdin=int(os.environ["RELAY_STDIN"]), stdout=subprocess.DEVNULL,
                         stderr=subprocess.DEVNULL, pass_fds=(int(os.environ["RELAY_STDIN"]),))
print(child.pid, flush=True)
time.sleep(120)
"""


def test_the_first_leg_ends_when_the_process_that_started_it_dies():
    r, w = os.pipe()   # this process keeps the write end open: only the starter's death can end the child
    try:
        starter = subprocess.Popen([sys.executable, "-c", STARTER, cli(), "--backend", "sim", "--relay-first", "--all"],
                                   stdout=subprocess.PIPE, text=True, env={**sim_env(), "RELAY_STDIN": str(r)},
                                   pass_fds=(r,))
        pid = int(starter.stdout.readline())
        time.sleep(0.5)
        assert alive(pid)
        os.kill(starter.pid, signal.SIGKILL)
        starter.wait()
        deadline = time.monotonic() + 1.0
        while alive(pid) and time.monotonic() < deadline:
            time.sleep(0.02)
        assert not alive(pid)
    finally:
        os.close(r)
        os.close(w)


# ---------------------------------------------------------------------------------- RelayReport
def relay_json(coverage=0.99997, held=0, first=None):
    total = 85_017_493_504
    d = dict(total=total, a_free_before=84_464_041_984, a_unreached=1_245_184, b_free_held=83_910_590_464,
             b_free_settled=84_464_041_984, b_free_before=84_464_041_984, b_unreached=1_245_184, marked=0,
             footprint_a=553_451_520, freed=553_451_520, held=held, growth=0, unreached=2_490_368 + held,
             coverage=coverage, settled=1, settle_polls=4, ms_first=420.5, ms_handover=95.25, ms_settle=16.0,
             ms_second=190.0)
    if first is not None:
        d["first"] = first
    return d


def test_relay_report_round_trips_and_summarises():
    first = TC.zero_report("0000:01:00.0")
    rep = TC.zero_report("0000:01:00.0")
    rep.relay = RelayReport.from_json(relay_json(first=first.as_json()))
    assert rep.relay.first == first
    again = ScrubReport.from_json(json.loads(json.dumps(rep.as_json())))
    assert again.relay == rep.relay and again == rep
    s = rep.relay.summary()
    assert s.startswith("coverage 0.99997 of 79.2 GiB (2.4 MiB unreached)")
    assert "footprint 527.8 MiB, freed 527.8 MiB, held 0.0 MiB, growth 0.0 MiB" in s
    assert "unmappable A 1.2 MiB, B 1.2 MiB" in s and "first leg 420 ms" in s and "second leg 190 ms" in s
    assert "marker" not in s and "did not settle" not in s
    plain = ScrubReport.from_json(TC.zero_report("0000:01:00.0").as_json())
    assert plain.relay is None and "relay" not in plain.as_json()


def test_reports_from_payload_gives_each_relay_its_first_leg():
    a = [TC.zero_report(b).as_json() for b in ("0000:01:00.0", "0000:02:00.0")]
    b = [dict(x, relay=relay_json()) for x in a]
    b[1]["relay"] = None
    reps = reports_from_payload({"wall_ms": 1.0, "reports": b, "first": {"wall_ms": 1.0, "reports": a},
                                 "first_pid": 1})
    assert reps[0].relay.first == ScrubReport.from_json(a[0]) and reps[1].relay is None
