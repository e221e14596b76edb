"""mv_lookup::Argument::prepare's compression of the lookup tuples with theta, checked without a device:

- the host default of Ops::compress_expressions in plonk_b200.hpp (the C++ driver tests/cpp/test_lookup_compress.cpp, `host` mode)
  against a Python big-integer fold (tests/lookup_compress_model.py) on random tuples: constants, negation, a + (-b), products,
  scaled, challenges, fixed / advice / instance queries at rotations -3 .. 3, k down to 1 where a rotation exceeds 2^k;
- the programs keygen lowers for the same tuples (compression_program), run by the host-emulated interpreter (csrc/graph.hpp,
  csrc/graph_exec.cuh) and by the oracle's interpreter with log_size = k and rot_scale = 1, against the same fold;
- create_proof with the compression done by the oracle's interpreter running the keygen programs reproduces the committed session
  digests (tests/golden/plonk_session_digests.json), with whole-coset keys and keys without cosets.
"""
import hashlib
import json
import os
import random
import subprocess

import numpy as np
import pytest

from lookup_compress_model import every_kind, fold_model, random_expr, read_host_output, to_ints, write_case
from lookup_model import R_MOD
from oracle import oracle as O
from quotient_programs import C_HORNER, C_SUB, S_CONST, S_THETA
from test_graph_host_emul import host_eval, lib  # noqa: F401  (lib: the host-emulation fixture)
from test_plonk_session import CASES, key

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "test_lookup_compress.cpp")
BIN = os.path.join(ROOT, "tests", "cpp", "test_lookup_compress")
DIGESTS = os.path.join(ROOT, "tests", "golden", "plonk_session_digests.json")
SHAPE = (3, 3, 2, 2)  # fixed, advice, instance columns; challenges


def binary():
    deps = [SRC] + [os.path.join(ROOT, "tests", "cpp", f) for f in ("test_plonk_session.cpp", "oracle_ops.hpp", "oracle_parts_ops.hpp")] + \
        [os.path.join(ROOT, "scroll-prover_b200", h) for h in ("plonk_b200.hpp", "halo2_b200.hpp", "pairing_bn254.hpp", "serde_bn254.hpp")]
    if not os.path.exists(BIN) or any(os.path.getmtime(d) > os.path.getmtime(BIN) for d in deps):
        subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "liboracle.so"])
        lib_dir, orc = os.path.join(ROOT, "scroll-prover_b200"), os.path.join(ROOT, "oracle")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-o", BIN, SRC, "-L" + lib_dir, "-lb200zk", "-Wl,-rpath," + lib_dir,
                               "-L" + orc, "-loracle", "-Wl,-rpath," + orc])
    return BIN


def random_case(seed, k, tuple_sizes, shape=SHAPE):
    """(theta, challenges, fixed, advice, instance, sides): random columns, every tuple_sizes[i]-expression side at depth <= 3"""
    rng = random.Random(seed)
    nf, na, ni, nc = shape
    cols = [O.fill_fr(1 << k, seed * 100 + i) for i in range(nf + na + ni)]
    challenges = [rng.randrange(R_MOD) for _ in range(nc)]
    sides = [[random_expr(rng, 3, shape) for _ in range(m)] for m in tuple_sizes]
    return rng.randrange(R_MOD), challenges, cols[:nf], cols[nf:nf + na], cols[nf + na:], sides


def run_host(tmp_path, k, case):
    theta, challenges, fixed, advice, instance, sides = case
    src, dst = tmp_path / "in.bin", tmp_path / "out.bin"
    write_case(src, k, theta, challenges, fixed, advice, instance, sides)
    r = subprocess.run([binary(), "host", str(src), str(dst)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and r.stdout.strip().endswith("OK"), r.stdout + r.stderr
    return read_host_output(dst, k, len(sides))


def model(k, case):
    theta, challenges, fixed, advice, instance, sides = case
    cols = {"fixed": [to_ints(c) for c in fixed], "advice": [to_ints(c) for c in advice], "instance": [to_ints(c) for c in instance]}
    return [fold_model(s, cols, challenges, theta, 1 << k) for s in sides]


def interpreters(lib, k, case, program):
    """(host emulation, oracle) of one compression program on the 2^k Lagrange rows"""
    theta, challenges, fixed, advice, instance, _ = case
    calcs, consts, rotations = program
    z = O.fr_from_int(0)
    ch = O.frs_from_ints(challenges) if challenges else np.zeros((0, 4), np.uint64)
    th = O.fr_from_int(theta)
    values = np.zeros((1 << k, 4), np.uint64)
    oracle = O.graph_evaluate(calcs, consts, rotations, fixed, advice, instance, ch, z, z, th, z, None, values, k, 1)
    rc, emul, _, err = host_eval(lib, calcs, consts, rotations, fixed, advice, instance, ch, [z, z, th, z], None, values, k, 1)
    assert rc == 0, err
    return emul, oracle


@pytest.mark.parametrize("k,seed,tuple_sizes", [(1, 1, [1, 2, 3, 4]), (2, 2, [4, 1]), (3, 3, [2, 3]), (5, 4, [1, 4, 2]),
                                                (8, 5, [3]), (10, 6, [2, 1])])
def test_host_default_and_programs_follow_the_fold(lib, tmp_path, k, seed, tuple_sizes):  # noqa: F811
    case = random_case(seed, k, tuple_sizes)
    case[5].append(every_kind(SHAPE))
    want = model(k, case)
    got, programs = run_host(tmp_path, k, case)
    for s, (w, g, p) in enumerate(zip(want, got, programs)):
        assert np.array_equal(g, w), f"host default, side {s}"
        emul, oracle = interpreters(lib, k, case, p)
        assert np.array_equal(emul, w), f"host-emulated interpreter, side {s}"
        assert np.array_equal(oracle, w), f"oracle interpreter, side {s}"


def test_lowering_is_one_horner_over_the_tuple_with_theta(tmp_path):
    """Horner(0, [e_0 .. e_{m-1}], Theta) as the last calculation, and a + (-b) lowered to SUB"""
    case = random_case(9, 3, [])
    case[5].append(every_kind(SHAPE))
    _, [(calcs, consts, _)] = run_host(tmp_path, 3, case)
    op, start, factor, parts = calcs[-1]
    assert op == C_HORNER and len(parts) == 3 and factor[0] == S_THETA
    assert start[0] == S_CONST and not consts[start[1]].any()
    assert any(c[0] == C_SUB for c in calcs)


@pytest.mark.parametrize("k,seed,variant", CASES)
def test_keygen_programs_reproduce_the_committed_session_digests(k, seed, variant):
    r = subprocess.run([binary(), "session", str(k), str(seed), str(variant)], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and r.stdout.strip().endswith("OK"), r.stdout[-2000:] + r.stderr[-2000:]
    proofs = {l.split()[1]: bytes.fromhex(l.split()[2]) for l in r.stdout.splitlines() if l.startswith("proof_sha_input")}
    want = json.load(open(DIGESTS))[key(k, seed, variant)]
    assert hashlib.sha256(proofs["whole"]).hexdigest() == want
    assert hashlib.sha256(proofs["parts"]).hexdigest() == want
