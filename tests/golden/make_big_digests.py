"""Writes tests/golden/big_digests.json: SHA-256 digests of the ORACLE's outputs at BASELINE sizes (MSM 2^22 / 2^24 uniform and
witness-like, iNTT 2^24 and 2^25, coset NTT 2^26, g_to_lagrange 2^14 / 2^16) on fixed seeded inputs.  tests/test_gpu_exact_big.py
and tests/test_gpu_chunk_shapes.py (iNTT 2^25) hold the CUDA path to the live oracle AND to these committed digests, so later
rounds cannot drift.  CPU only; takes a few minutes.

    python tests/golden/make_big_digests.py
"""
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import oracle as O  # noqa: E402

GEN_THREADS = 8  # fill_points_chain starts one chain per thread: the bases depend on this number, so it is fixed


def sha(a) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def msm_case(log_n: int, witness_like: bool, threads: int):
    n = 1 << log_n
    bases = O.fill_points_chain(n, 9000 + log_n, GEN_THREADS)
    scal = O.fill_fr(n, 9100 + log_n + (50 if witness_like else 0), witness_like)
    return bases, scal, O.g1_to_affine(O.best_multiexp(scal, bases, threads))


def ntt_inputs(k: int):
    return O.fill_fr(1 << k, 9200 + k)


def main():
    threads = os.cpu_count() or 8
    out = {}
    for log_n in (22, 24):
        for wl in (False, True):
            _, _, res = msm_case(log_n, wl, threads)
            out[f"msm_{log_n}_{'witness' if wl else 'uniform'}"] = sha(res)
            print(log_n, wl, out[f"msm_{log_n}_{'witness' if wl else 'uniform'}"], flush=True)
    k = 24
    dom = O.EvaluationDomain(5, k)
    a = ntt_inputs(k)
    coeff = dom.lagrange_to_coeff(a, threads)
    out["lagrange_to_coeff_24"] = sha(coeff)
    out["coeff_to_extended_26"] = sha(dom.coeff_to_extended(coeff, threads))
    k = 25
    out["lagrange_to_coeff_25"] = sha(O.EvaluationDomain(5, k).lagrange_to_coeff(ntt_inputs(k), threads))
    print("ntt done", flush=True)
    for kk in (14, 16):
        g = O.fill_points_chain(1 << kk, 9300 + kk, GEN_THREADS)
        out[f"g_to_lagrange_{kk}"] = sha(O.g_to_lagrange(g, kk, threads))
        print("g_to_lagrange", kk, flush=True)
    json.dump(out, open(os.path.join(ROOT, "tests", "golden", "big_digests.json"), "w"), indent=1)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
