"""Times the MSM bucket sort (profile classes msm_count, msm_scan, msm_scatter) beside msm_accumulate and the whole MSM, for
the MSM plans of the chunk-proof step: a 2^20 precomputed-table batch of msm_srs_max_batch columns, 2^24 plain bases at
c = 19 and 2^25 plain bases at c = 20, each with uniform and witness-like scalars (60 % zero, 30 % below 2^16).

    python tools/msm_sort_time.py [--out FILE] [--reps R]     # on the GPU

One JSON line per shape, with the card name, power limit and clocks read in the same run.  The default output is
profiles/msm_sort_h100_<power limit>w.jsonl.  Kernel times are per MSM (per batch for the 2^20 shape), from CUDA events
around each profile class in a profiled pass; `msm_ms` is the median of R unprofiled MSMs timed with CUDA events."""
import argparse
import importlib
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
zk = importlib.import_module("scroll-prover_b200")

SORT = ("msm_count", "msm_scan", "msm_scatter")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, limit, smax, sm = [x.strip() for x in q.split(",")]
    return {"device": name, "power_limit_w": float(limit), "sm_clock_max_mhz": int(smax), "sm_clock_mhz": int(sm)}


def rand_fr(n, gen):
    t = torch.randint(-(2**63), 2**63 - 1, (n, 4), dtype=torch.int64, device="cuda", generator=gen)
    t[:, 3] &= 0x0FFFFFFFFFFFFFFF  # < 2^252 < r: valid Montgomery limbs
    return t


def witness_like(ctx, n, gen):
    sel = torch.rand(n, device="cuda", generator=gen)
    small = torch.randint(0, 1 << 16, (n,), dtype=torch.int64, device="cuda", generator=gen)
    raw = torch.zeros((n, 4), dtype=torch.int64, device="cuda")
    raw[:, 0] = torch.where((sel >= 0.6) & (sel < 0.9), small, torch.zeros_like(small))
    torch.cuda.synchronize()
    mont = ctx.poly_scale(raw, zk.fr_from_int(1 << 256))
    uni = rand_fr(n, gen)
    torch.cuda.synchronize()
    return torch.where((sel >= 0.9).unsqueeze(1), uni, mont).contiguous()


def measure(ctx, run, reps):
    run()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        run()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ctx.profile_enable(True)
    ctx.profile_reset()
    for _ in range(reps):
        run()
    torch.cuda.synchronize()
    prof = ctx.profile_read()
    ctx.profile_enable(False)
    ks = {k: prof[k]["ms"] / reps for k in SORT + ("msm_accumulate",) if k in prof}
    return sorted(ts)[len(ts) // 2], ks


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    ctx = zk.Context(0)
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    ctx.set_stream(stream.cuda_stream)
    gen = torch.Generator(device="cuda").manual_seed(0x5047)
    lines = []
    for log_n, c, pre in ((20, 17, True), (24, 19, False), (25, 20, False)):
        n = 1 << log_n
        g = torch.empty((n, 8), dtype=torch.int64, device="cuda")
        ctx.g1_generator_mul_batch(rand_fr(n, gen), out=g)
        torch.cuda.synchronize()
        ctx.srs_set_precompute(pre)
        srs = ctx.srs_register(g, zk.SRS_G_LAGRANGE)
        ctx.srs_set_precompute(True)
        del g
        ctx.msm_set_window(0 if pre else c)
        for kind in ("uniform", "witness"):
            make = (lambda: rand_fr(n, gen)) if kind == "uniform" else (lambda: witness_like(ctx, n, gen))
            col = make()
            srs.msm(col)
            st = ctx.msm_last_stats()
            batch = max(1, min(32, (1 << 28) // (n * st["n_windows"]))) if pre else 1
            cols = [col] + [make() for _ in range(batch - 1)]
            torch.cuda.synchronize()
            ctx.msm_total_adds(reset=True)
            srs.msm_batch(cols)
            adds = ctx.msm_total_adds(reset=True)
            ms, ks = measure(ctx, lambda: srs.msm_batch(cols), args.reps)
            line = {"shape": f"2^{log_n} {'precomputed' if pre else 'plain'} c={st['window_bits']} batch={batch} {kind}",
                    "log_n": log_n, "c": st["window_bits"], "precomputed": pre, "batch": batch, "scalars": kind,
                    "entries": adds, "msm_ms": ms, "kernel_ms": ks, "sort_ms": sum(ks.get(k, 0.0) for k in SORT)}
            line.update(card())
            lines.append(line)
            print(json.dumps(line), flush=True)
            del cols, col
        ctx.msm_set_window(0)
        srs.release()
        torch.cuda.empty_cache()
    out = args.out or os.path.join(ROOT, "profiles", f"msm_sort_h100_{lines[0]['power_limit_w']:.0f}w.jsonl")
    with open(out, "w") as f:
        for l in lines:
            f.write(json.dumps(l) + "\n")


if __name__ == "__main__":
    main()
