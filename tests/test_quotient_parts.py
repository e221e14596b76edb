"""create_proof with a proving key that stores no extended cosets (plonk_b200.hpp, keygen(..., keep_cosets = false)): evaluate_h
runs one coset part at a time.  h(X) is unique, so the proofs must be the whole-coset prover's, byte for byte.

CPU: over the CPU oracle (tests/cpp/oracle_parts_ops.hpp), the by-parts proof hashes to the COMMITTED digest of the whole-coset
session (tests/golden/plonk_session_digests.json) and verifies; with the Poseidon transcript it equals the whole-coset proof.
GPU: the same through the C ABI (b200zk_coeff_to_extended_part, b200zk_graph_evaluate_part, b200zk_extended_parts_to_coeff).
The circuits are those of tests/cpp/test_plonk_session.cpp.
"""
import hashlib
import json
import os
import subprocess

import pytest

from test_plonk_session import CASES, GPU_CASES, key

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "test_quotient_parts.cpp")
BIN = os.path.join(ROOT, "tests", "cpp", "test_quotient_parts")
DIGESTS = os.path.join(ROOT, "tests", "golden", "plonk_session_digests.json")


def binary():
    deps = [SRC] + [os.path.join(ROOT, "tests", "cpp", f) for f in ("test_plonk_session.cpp", "oracle_ops.hpp", "oracle_parts_ops.hpp")] + \
        [os.path.join(ROOT, "scroll-prover_b200", h) for h in ("plonk_b200.hpp", "halo2_b200.hpp", "pairing_bn254.hpp", "serde_bn254.hpp")]
    if not os.path.exists(BIN) or any(os.path.getmtime(d) > os.path.getmtime(BIN) for d in deps):
        subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "liboracle.so"])
        lib, orc = os.path.join(ROOT, "scroll-prover_b200"), os.path.join(ROOT, "oracle")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-o", BIN, SRC, "-L" + lib, "-lb200zk", "-Wl,-rpath," + lib, "-L" + orc, "-loracle",
                               "-Wl,-rpath," + orc])
    return BIN


def run(mode, k, seed, variant):
    r = subprocess.run([binary(), mode, str(k), str(seed), str(variant)], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and r.stdout.strip().endswith("OK"), r.stdout[-2000:] + r.stderr[-2000:]
    proofs = {l.split()[1]: bytes.fromhex(l.split()[2]) for l in r.stdout.splitlines() if l.startswith("proof_sha_input")}
    return proofs, r.stdout


@pytest.mark.parametrize("k,seed,variant", CASES)
def test_proof_by_parts_over_the_oracle_matches_the_committed_digest(k, seed, variant):
    proofs, out = run("oracle", k, seed, variant)
    assert "poseidon proof by parts identical to the whole-coset one" in out
    assert hashlib.sha256(proofs["parts_oracle"]).hexdigest() == json.load(open(DIGESTS))[key(k, seed, variant)]


@pytest.mark.gpu
@pytest.mark.parametrize("k,seed,variant", GPU_CASES)
def test_proof_by_parts_on_the_device_is_the_oracle_proof(k, seed, variant):
    proofs, out = run("both", k, seed, variant)
    assert "device proof by parts identical to the oracle's" in out
    assert proofs["parts_device"] == proofs["parts_oracle"]
    digests = json.load(open(DIGESTS))
    if key(k, seed, variant) in digests:
        assert hashlib.sha256(proofs["parts_device"]).hexdigest() == digests[key(k, seed, variant)]


@pytest.mark.gpu
@pytest.mark.parametrize("k,variant", [(14, 1), (16, 2), (14, 3)])
def test_device_only_session_by_parts_equals_the_whole_coset_session(k, variant):
    """2^14 / 2^16 rows through the C ABI alone, Poseidon transcript: the proof by parts is the whole-coset proof of the same seed,
    and the halo2-style verifier and the snark-verifier mirror accept it."""
    _, out = run("device", k, 3, variant)
    assert "identical to the whole-coset proof, accepted by both verifiers" in out
