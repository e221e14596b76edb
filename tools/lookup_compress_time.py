"""Time of mv_lookup::Argument::prepare's compression of the lookup tuples with theta: the DeviceOps override of
Ops::compress_expressions (every read column uploaded once, then b200zk_graph_evaluate per side with log_size = k, rot_scale = 1,
then the downloads) against the host default (the fold over the expressions, one row at a time on one core; plonk_b200.hpp).

usage: lookup_compress_time.py [--reps R] [--out FILE] [--shapes layer2,inner_8,inner_64]

Shapes (one JSON line each, on stdout and appended to FILE, default profiles/lookup_compress_h100_<power limit>w.jsonl):
  layer2    k = 25, one lookup: input = one advice column, table = one fixed column
  inner_N   k = 20, N lookups: input (q a_0, q a_1, q a_2) with one selector q shared by all, table (t_0, t_1, t_2); lookup l reads
            the advice columns and table columns 3 (l mod 8) + i, so 8 lookups read 24 + 24 columns and 64 lookups read the same
            columns again, as the inner circuit's lookups share their columns
The C++ driver tests/cpp/test_lookup_compress (time mode) makes two warm-up calls of the DeviceOps override, then R calls, each
timed by the host clock from a synchronised context to the call's return; the call ends with the download of every result column,
so the time covers the uploads, the evaluations and the downloads.  It then times the host default once and requires both outputs
to be equal.  The card's name, power limit and maximum SM clock are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, _ROOT)
sys.path.insert(0, os.path.join(_ROOT, "tests"))
from lookup_compress_model import write_case  # noqa: E402
from lookup_model import small_ints  # noqa: E402
from oracle import oracle as O  # noqa: E402

DRIVER = os.path.join(_ROOT, "tests", "cpp", "test_lookup_compress")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    name, power, clock = [x.strip() for x in q.stdout.strip().splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def shape(name):
    """(k, fixed, advice, sides)"""
    if name == "layer2":
        k = 25
        return k, [O.fill_fr(1 << k, 1)], [O.fill_fr(1 << k, 2)], [[("advice", 0, 0)], [("fixed", 0, 0)]]
    k, lookups = 20, int(name.split("_")[1])
    n = 1 << k
    q = small_ints((np.arange(n) % 4 != 3).astype(np.int64))
    groups = min(lookups, 8)
    advice = [O.fill_fr(n, 100 + i) for i in range(3 * groups)]
    fixed = [q] + [O.fill_fr(n, 200 + i) for i in range(3 * groups)]
    sides = []
    for l in range(lookups):
        g = l % 8
        sides.append([("mul", ("fixed", 0, 0), ("advice", 3 * g + i, 0)) for i in range(3)])
        sides.append([("fixed", 1 + 3 * g + i, 0) for i in range(3)])
    return k, fixed, advice, sides


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    ap.add_argument("--shapes", default="layer2,inner_8,inner_64")
    a = ap.parse_args()
    info = card()
    out = a.out or os.path.join(_ROOT, "profiles", "lookup_compress_h100_%sw.jsonl" % info["power_limit"].split()[0].split(".")[0])
    for name in a.shapes.split(","):
        k, fixed, advice, sides = shape(name)
        with tempfile.TemporaryDirectory() as d:
            src = os.path.join(d, "in.bin")
            write_case(src, k, 0x5EED, [], fixed, advice, [], sides)
            del fixed, advice
            r = subprocess.run([DRIVER, "time", src, str(a.reps)], capture_output=True, text=True, timeout=3600)
        assert r.returncode == 0 and r.stdout.strip().endswith("OK"), r.stdout + r.stderr
        words = [l.split() for l in r.stdout.splitlines()]
        vals = {w[0]: float(w[1]) for w in words if len(w) == 2 and w[0] in ("device_ms_median", "device_ms_min", "host_ms")}
        rec = {"shape": name, "k": k, "lookups": len(sides) // 2, "sides": len(sides), "reps": a.reps,
               "device_ms_median": round(vals["device_ms_median"], 3), "device_ms_min": round(vals["device_ms_min"], 3),
               "host_default_ms": round(vals["host_ms"], 1), "device_equals_host_default": True,
               "speedup_vs_host_default": round(vals["host_ms"] / vals["device_ms_median"], 1)}
        rec.update(info)
        line = json.dumps(rec)
        print(line, flush=True)
        with open(out, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
