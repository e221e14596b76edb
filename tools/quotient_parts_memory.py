"""Device memory and time of a layer-shaped evaluate_h, whole coset against coset parts (JSON lines on stdout).

usage: quotient_parts_memory.py K [C] [--parts-only]

C resident columns (default 20) of 2^K coefficients, J = 4 (the chunk protocol's quotient.num_chunk), three programs: the
gate program of tools/quotient_time.py, the permutation section (two sets of two columns) and a two-input log-derivative lookup
(tests/h_terms_programs.py), each reading its columns from the C resident ones.
  whole: coeff_to_extended of every column (C x J x 2^K elements), the programs over the extended coset, the division by
         X^n - 1 and extended_to_coeff;
  parts: per part j, every column's part (C x 2^K), the programs on the part, then extended_parts_to_coeff with the division.
Each path runs twice in a fresh context (a warm-up, then the timed run; host clock around device work that ends in a
synchronise).  Peak memory is the device's used memory (torch.cuda.mem_get_info: the library's own allocations and torch's pool)
at its highest point, sampled after every allocation, minus the used memory before the path's context was created.  A path that
does not fit reports "fits": false.  Where both fit, the two h outputs (J x 2^K coefficients) are compared element by element.
The card's name and power limit are read in the same run.  For a path that fails, peak_GiB is what was held when the allocation
failed.
"""
import gc
import importlib
import json
import os
import subprocess
import sys
import time

import torch

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, _ROOT)
sys.path.insert(0, os.path.join(_ROOT, "tools"))
sys.path.insert(0, os.path.join(_ROOT, "tests"))
zk = importlib.import_module("scroll-prover_b200")
from h_terms_programs import logup_terms_program, permutation_terms_program  # noqa: E402
from quick_time import rand_fr  # noqa: E402
from quotient_time import gate_program  # noqa: E402

GIB = float(1 << 30)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    name, power, clock = [x.strip() for x in q.stdout.strip().splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def programs(ctx):
    fr = zk.fr_from_int
    gate = ctx.graph(gate_program(16, 4), [fr(1)], [0, 1, 2, 3])
    pc, pk, pr = permutation_terms_program(2, 2, 4, -6)
    lc, lk, lr = logup_terms_program(2)
    return [gate, ctx.graph(pc, [fr(v) for v in pk], pr), ctx.graph(lc, [fr(v) for v in lk], lr)]


def tables(cols):
    """column tables of the three programs, drawn from the C resident columns"""
    pick = lambda idx: [cols[i % len(cols)] for i in idx]
    return [dict(fixed=pick([4, 5]), advice=pick([0, 1, 2, 3])),                                     # gate: 2 fixed, 4 advice
            dict(fixed=pick([6, 7, 8, 9, 10, 11, 12]), advice=pick([13, 14, 0, 1, 2, 3])),          # perm: sigma x4 l0 l_last l_act | z x2 v x4
            dict(fixed=pick([10, 11, 12]), advice=pick([15, 16, 17, 18, 19]))]                      # lookup: l0 l_last l_act | f x2 t m phi


class Peak:
    def __init__(self):
        free, self.total = torch.cuda.mem_get_info()
        self.base = self.total - free
        self.used = self.base

    def __call__(self):
        free, _ = torch.cuda.mem_get_info()
        self.used = max(self.used, self.total - free)

    def gib(self):
        return (self.used - self.base) / GIB


def run_path(kind, K, C):
    """(record, h) -- h the J pieces of 2^K coefficients, or None when the path does not fit"""
    J, n, ek = 4, 1 << K, K + 2
    gc.collect()
    torch.cuda.empty_cache()
    peak = Peak()
    ctx = zk.Context(0)
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    ctx.set_stream(stream.cuda_stream)
    rec = {"path": kind, "k": K, "extended_k": ek, "J": J, "columns": C}
    h = None
    try:
        d = zk.EvaluationDomain(ctx, J + 1, K)
        fr = zk.fr_from_int
        args = dict(beta=fr(5), gamma=fr(7), theta=fr(11), y=fr(0x1234567), extended_omega=d.extended_omega)
        progs = programs(ctx)
        coeffs = [rand_fr(n, 100 + i) for i in range(C)]
        peak()

        def whole():
            ext = [d.coeff_to_extended(c) for c in coeffs]
            vals = torch.zeros((J * n, 4), dtype=torch.int64, device="cuda")
            peak()
            for g, tab in zip(progs, tables(ext)):
                g.evaluate(vals, ek, J, **tab, **args)
            peak()
            del ext
            zn, wn = pow(zk._ZETA, n, zk.R_MOD), pow(zk.fr_to_int(d.extended_omega), n, zk.R_MOD)
            tinv = torch.stack([torch.from_numpy(fr(pow((zn * pow(wn, j, zk.R_MOD) - 1) % zk.R_MOD, -1, zk.R_MOD)).view("int64"))
                                for j in range(J)]).cuda()
            tcol = tinv.repeat(n, 1)
            peak()
            ctx.poly_mul(vals, tcol, out=vals)
            del tcol
            ctx.best_fft(vals, d.extended_omega_inv, ek, inverse_scale=True, coset_mode=zk.COSET_POST)
            peak()
            return [vals[t * n:(t + 1) * n] for t in range(J)]

        def parts():
            out = []
            for j in range(J):
                cols = [d.coeff_to_extended_part(c, j) for c in coeffs]
                v = torch.zeros((n, 4), dtype=torch.int64, device="cuda")
                peak()
                for g, tab in zip(progs, tables(cols)):
                    g.evaluate_part(v, K, ek, j, **tab, **args)
                out.append(v)
                peak()
                del cols
            d.extended_parts_to_coeff(out, divide_by_vanishing=True)
            peak()
            return out

        fn = whole if kind == "whole" else parts
        fn()  # warm-up
        ctx.synchronize()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        h = fn()
        ctx.synchronize()
        torch.cuda.synchronize()
        rec.update(fits=True, s=round(time.perf_counter() - t0, 4))
    except (torch.OutOfMemoryError, zk.B200zkError) as e:
        if isinstance(e, zk.B200zkError) and e.code != zk.E_OOM:
            raise
        peak()  # what was held when the allocation failed
        rec.update(fits=False, error=str(e).splitlines()[0][:160])
        h = None
    rec["peak_GiB"] = round(peak.gib(), 2)
    if h is not None:
        h = [t.cpu() for t in h]  # keep for the comparison, free the device
    for g in locals().get("progs", []):
        g.release()
    ctx.close()
    torch.cuda.set_stream(torch.cuda.default_stream())
    torch.cuda.empty_cache()
    return rec, h


def main():
    argv = [a for a in sys.argv[1:] if not a.startswith("--")]
    K = int(argv[0])
    C = int(argv[1]) if len(argv) > 1 else 20
    info = card()
    kinds = ["parts"] if "--parts-only" in sys.argv else ["whole", "parts"]
    results = {}
    for kind in kinds:
        rec, h = run_path(kind, K, C)
        results[kind] = h
        print(json.dumps({**rec, **info}), flush=True)
    if results.get("whole") is not None and results.get("parts") is not None:
        equal = all(torch.equal(a, b) for a, b in zip(results["whole"], results["parts"]))
        print(json.dumps({"k": K, "columns": C, "h_equal": equal, **info}), flush=True)


if __name__ == "__main__":
    main()
