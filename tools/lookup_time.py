"""Time of the lookup multiplicity column m(X) (mv_lookup::Argument::prepare): b200zk_lookup_multiplicities on the device against
the host default of Ops::lookup_multiplicities (a std::map index of the table, then one find per input cell; plonk_b200.hpp).

usage: lookup_time.py [--out FILE] [--reps R] [--no-host-layer2]

Shapes (one JSON line each, on stdout and appended to FILE):
  layer2   k = 25, a range table 0 .. 2^24 - 1 in rows 0 .. 2^24 - 1 (every other row zero, a duplicate of row 0 that the
           first-row rule does not count on), one input column of 2^25 rows: ~60 % zeros, the rest drawn from the range
  inner_N  k = 20, a 2^16-row range table (the other rows zero), N = 1, 2, 4 input columns of the same witness-like kind
usable = 2^k - 10 (the blinding rows of a create_proof).  Device: two warm-up calls, then R calls, each timed by CUDA events on the
context stream and by the host clock up to the call's return (which includes the 8-byte read-back of first_missing, so the
device work has finished).  Host: the C++ driver tests/cpp/test_lookup_multiplicities (host mode) times the host default around
the call alone, once.  The device m is compared with the host default's m (and with tests/lookup_model.py's) element for element.
The card's name and power limit are read in the same run.
"""
import argparse
import importlib
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, _ROOT)
sys.path.insert(0, os.path.join(_ROOT, "tests"))
zk = importlib.import_module("scroll-prover_b200")
from lookup_model import numpy_model, small_ints  # noqa: E402

DRIVER = os.path.join(_ROOT, "tests", "cpp", "test_lookup_multiplicities")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    name, power, clock = [x.strip() for x in q.stdout.strip().splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def shape(k: int, range_rows: int, n_inputs: int, seed: int):
    n, usable = 1 << k, (1 << k) - 10
    rng = np.random.default_rng(seed)
    table = np.zeros((n, 4), np.uint64)  # rows past the range hold zero, a duplicate of row 0 (as an unassigned fixed cell)
    table[:range_rows] = small_ints(np.arange(range_rows))
    inputs = []
    for _ in range(n_inputs):
        v = rng.integers(0, range_rows, n)
        v[rng.random(n) < 0.6] = 0
        inputs.append(small_ints(v))
    return inputs, table, usable


def host_default(inputs, table, k, usable):
    with tempfile.TemporaryDirectory() as d:
        src, dst = os.path.join(d, "in.bin"), os.path.join(d, "out.bin")
        with open(src, "wb") as f:
            f.write(np.array([k, len(inputs)], np.uint32).tobytes() + np.array([usable], np.uint64).tobytes())
            for col in [table] + list(inputs):
                f.write(np.ascontiguousarray(col).tobytes())
        r = subprocess.run([DRIVER, "host", src, dst], capture_output=True, text=True, timeout=3600)
        assert r.returncode == 0 and r.stdout.strip().endswith("OK"), r.stdout + r.stderr
        ms = float([l for l in r.stdout.splitlines() if l.startswith("host_ms")][0].split()[1])
        raw = np.fromfile(dst, np.uint64)
        assert raw[0] == 0, "the host default found an input outside the table"
        return ms, raw[1:].reshape(-1, 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--no-host-layer2", action="store_true", help="skip the host default at k = 25 (minutes on one core)")
    a = ap.parse_args()
    info = card()
    ctx = zk.Context(0)
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    cases = [("layer2", 25, 1 << 24, 1), ("inner_1", 20, 1 << 16, 1), ("inner_2", 20, 1 << 16, 2), ("inner_4", 20, 1 << 16, 4)]
    for name, k, range_rows, n_inputs in cases:
        inputs, table, usable = shape(k, range_rows, n_inputs, 1000 + k + n_inputs)
        with torch.cuda.stream(stream):
            dev = lambda x: torch.from_numpy(np.ascontiguousarray(x).view(np.int64)).cuda()
            d_in, d_t = [dev(c) for c in inputs], dev(table)
            out = torch.empty((1 << k, 4), dtype=torch.int64, device="cuda")
            torch.cuda.synchronize()
            for _ in range(2):
                assert ctx.lookup_multiplicities(d_in, d_t, k, usable, out) is None
            ev_ms, wall_ms = [], []
            for _ in range(a.reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0 = time.perf_counter()
                e0.record(stream)
                miss = ctx.lookup_multiplicities(d_in, d_t, k, usable, out)
                e1.record(stream)
                wall_ms.append((time.perf_counter() - t0) * 1e3)
                e1.synchronize()
                ev_ms.append(e0.elapsed_time(e1))
                assert miss is None
            m = out.cpu().numpy().view(np.uint64)
            del d_in, d_t, out
            torch.cuda.empty_cache()
        m_model, miss_model = numpy_model(inputs, table, k, usable)
        assert miss_model is None and np.array_equal(m, m_model), name
        rec = {"shape": name, "k": k, "usable": usable, "range_rows": range_rows, "n_inputs": n_inputs, "reps": a.reps,
               "device_ms_median": round(statistics.median(ev_ms), 3), "device_ms_min": round(min(ev_ms), 3),
               "call_wall_ms_median": round(statistics.median(wall_ms), 3), "device_m_equals_model": True}
        if name == "layer2" and a.no_host_layer2:
            rec["host_default_ms"] = "not measured"
        else:
            host_ms, m_host = host_default(inputs, table, k, usable)
            rec["host_default_ms"] = round(host_ms, 1)
            rec["device_m_equals_host_default"] = bool(np.array_equal(m, m_host))
            assert rec["device_m_equals_host_default"], name
            rec["speedup_vs_host_default"] = round(host_ms / statistics.median(ev_ms), 1)
        rec.update(info)
        line = json.dumps(rec)
        print(line, flush=True)
        if a.out:
            with open(a.out, "a") as f:
                f.write(line + "\n")
    ctx.set_stream(None)
    ctx.close()


if __name__ == "__main__":
    main()
