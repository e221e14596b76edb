"""Time of dev::MockProver::verify_par's check: mock_prove(DeviceOps, ...) -- Ops::check_constraints through b200zk_graph_evaluate,
b200zk_nonzero_rows, b200zk_lookup_missing_rows and b200zk_copy_check -- against the host mock_prove (mock_check, one row at a time
on one core; plonk_b200.hpp), on the synthetic circuit of tests/cpp/test_mock_device.cpp.

usage: mock_time.py [--reps R] [--out FILE] [--ks 16,20] [--plants P]

The circuit (one JSON line per k, on stdout and appended to FILE, default profiles/mock_h100_<power limit>w.jsonl): 32 gates over
8 advice columns and 4 selectors, 4 lookups into a 2^16-row range table (one of them a 2-tuple, one rotated), the 8 advice columns
under copy constraints with random cycles, and P witness cells broken.  The driver (time mode) makes one warm-up call of
mock_prove(DeviceOps), then R calls, each timed by the host clock from a synchronised context to the call's return; the call ends
with the download of the failure lists, so it covers the witness synthesis on the host, the uploads and the checks.  It then times
the host mock_prove once and requires both failure lists to be equal.  The card's name, power limit and maximum SM clock are read
in the same run.
"""
import argparse
import json
import os
import subprocess

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DRIVER = os.path.join(_ROOT, "tests", "cpp", "test_mock_device")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    name, power, clock = [x.strip() for x in q.stdout.strip().splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    ap.add_argument("--ks", default="16,20")
    ap.add_argument("--plants", type=int, default=300)
    a = ap.parse_args()
    info = card()
    out = a.out or os.path.join(_ROOT, "profiles", "mock_h100_%sw.jsonl" % info["power_limit"].split()[0].split(".")[0])
    for k in [int(x) for x in a.ks.split(",")]:
        r = subprocess.run([DRIVER, "time", str(k), "3", str(a.plants), str(a.reps)], capture_output=True, text=True, timeout=3600)
        assert r.returncode == 0 and r.stdout.strip().endswith("OK"), r.stdout + r.stderr
        words = [l.split() for l in r.stdout.splitlines()]
        vals = {w[0]: float(w[1]) for w in words if len(w) == 2 and w[0] in ("device_ms_median", "device_ms_min", "host_ms")}
        summary = next(l for l in r.stdout.splitlines() if "device == host" in l)
        rec = {"k": k, "gates": 32, "lookups": 4, "permutation_columns": 8, "planted_cells": a.plants, "reps": a.reps,
               "failures": int(summary.split("device == host, ")[1].split(" failures")[0]),
               "device_ms_median": round(vals["device_ms_median"], 3), "device_ms_min": round(vals["device_ms_min"], 3),
               "host_ms": round(vals["host_ms"], 1), "device_equals_host": True,
               "speedup_vs_host": round(vals["host_ms"] / vals["device_ms_median"], 1)}
        rec.update(info)
        line = json.dumps(rec)
        print(line, flush=True)
        with open(out, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
