"""The C++ host mirror of the reference API (scroll-prover_b200/halo2_b200.hpp) exercised through the C ABI."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "test_halo2_b200.cpp")
BIN = os.path.join(ROOT, "tests", "cpp", "test_halo2_b200")


def _build(out=BIN):
    libdir = os.path.join(ROOT, "scroll-prover_b200")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-o", out, SRC, "-L" + libdir, "-lb200zk",
                           "-Wl,-rpath," + libdir])
    return out


def test_cpp_mirror_compiles_against_the_abi():
    _build()
    assert os.path.exists(BIN)


@pytest.mark.gpu
def test_cpp_mirror_runs_on_gpu_from_a_private_build(tmp_path):
    """built from the current sources into a directory of its own: the run needs no write access to the source tree"""
    binary = _build(str(tmp_path / "test_halo2_b200"))
    r = subprocess.run([binary], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout + r.stderr


def test_cpp_mirror_host_only_parts_on_the_cpu(zk):
    """No GPU needed: EvaluationDomain::new(5, 25) against the reference's chunk.protocol dump, and the C++ permutation /
    lookup program generators lowered through b200zk_graph_check to exactly the instruction / slot counts of their Python twins."""
    import json
    import sys

    import numpy as np

    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from h_terms_programs import logup_terms_program, permutation_terms_program

    src = os.path.join(ROOT, "tests", "cpp", "test_host_only.cpp")
    binary = os.path.join(ROOT, "tests", "cpp", "test_host_only")
    libdir = os.path.join(ROOT, "scroll-prover_b200")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-o", binary, src, "-L" + libdir, "-lb200zk", "-Wl,-rpath," + libdir])
    dom = json.load(open(os.path.join(ROOT, "tests", "golden", "reference_fixtures.json")))["chunk_protocol"]["domain"]
    hx = lambda limbs: np.array(limbs, dtype=np.uint64).tobytes().hex()
    c, k, r = permutation_terms_program(3, 3, 8, -6)
    perm = zk.graph_check(c, len(k), len(r))
    c, k, r = logup_terms_program(3)
    look = zk.graph_check(c, len(k), len(r))
    res = subprocess.run([binary, hx(dom["gen"]), hx(dom["gen_inv"]), hx(dom["n_inv"]), str(perm["n_instructions"]), str(perm["n_slots"]),
                          str(look["n_instructions"]), str(look["n_slots"])], capture_output=True, text=True, timeout=120)
    assert res.returncode == 0 and "HOST OK" in res.stdout, res.stdout + res.stderr
