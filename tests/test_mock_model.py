"""The model of MockProver's three device checks (tests/mock_model.py), checked without a device:

- against the host mock_prove of plonk_b200.hpp on the three session circuits, honest and with sabotages 1-4: the C++ driver
  tests/cpp/test_mock_device.cpp (`host` mode) writes each case's gate values, compressed lookup tuples, permutation columns and
  successor array with the host's failure list, and the model must rebuild that list element for element;
- its contract on hand-made cases: ascending order, cap truncation, j * 2^k + i indexing, only rows below usable, successor
  comparison, against loops written out below.
"""
import os
import subprocess

import numpy as np
import pytest

from lookup_model import random_fr
from mock_model import _as_keys, copy_check, lookup_missing_rows, mock_failures, nonzero_rows, random_cycles, read_host_dump, sparse_values

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "test_mock_device.cpp")
BIN = os.path.join(ROOT, "tests", "cpp", "test_mock_device")


def binary():
    deps = [SRC, os.path.join(ROOT, "tests", "cpp", "test_plonk_session.cpp")] + [
        os.path.join(ROOT, "scroll-prover_b200", h) for h in ("plonk_b200.hpp", "halo2_b200.hpp")]
    if not os.path.exists(BIN) or any(os.path.getmtime(d) > os.path.getmtime(BIN) for d in deps):
        lib, orc = os.path.join(ROOT, "scroll-prover_b200"), os.path.join(ROOT, "oracle")
        subprocess.check_call(["make", "-s", "-C", orc, "liboracle.so"])
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-o", BIN, SRC, "-L" + lib, "-lb200zk", "-Wl,-rpath," + lib, "-L" + orc,
                               "-loracle", "-Wl,-rpath," + orc])
    return BIN


SESSION_CASES = [(4, 1, 1), (6, 1, 1), (5, 2, 2), (7, 4, 2), (5, 3, 3), (6, 1, 3)]


@pytest.mark.parametrize("k,seed,variant", SESSION_CASES)
def test_model_rebuilds_the_host_mock_prove(k, seed, variant, tmp_path):
    out = tmp_path / "cases.bin"
    r = subprocess.run([binary(), "host", str(k), str(seed), str(variant), str(out)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and r.stdout.strip().endswith("OK"), r.stdout + r.stderr
    cases = read_host_dump(out)
    assert len(cases) == 5
    assert cases[0]["failures"] == []  # the honest witness
    for sabotage, case in enumerate(cases):
        assert case["k"] == k and case["usable"] < 1 << k
        assert mock_failures(case) == case["failures"], sabotage
        if sabotage:
            assert case["failures"], sabotage
    assert {f[0] for c in cases for f in c["failures"]} >= {0, 1}


def test_nonzero_rows_contract():
    rng = np.random.default_rng(1)
    v = sparse_values(rng, 1000, 0.05)
    want = [i for i in range(1000) if any(int(x) for x in v[i])]
    count, rows = nonzero_rows(v)
    assert count == len(want) and rows.tolist() == want
    for cap in (0, 1, len(want) - 1, len(want), len(want) + 5):
        c, r = nonzero_rows(v, cap)
        assert c == len(want) and r.tolist() == want[:cap]
    assert nonzero_rows(np.zeros((64, 4), np.uint64))[0] == 0
    assert nonzero_rows(np.ones((64, 4), np.uint64))[1].tolist() == list(range(64))


def test_lookup_missing_rows_contract():
    rng = np.random.default_rng(2)
    k, n, usable = 5, 32, 27
    table = random_fr(rng, n)
    table[3] = table[20]  # a duplicated value
    inputs = [table[rng.integers(0, usable, n)] for _ in range(3)]
    inputs[0][4] = table[30]  # only in a table row >= usable: missing
    inputs[2][0] = random_fr(rng, 1)[0]
    inputs[1][usable] = random_fr(rng, 1)[0]  # rows >= usable are not checked
    inputs[2][n - 1] = random_fr(rng, 1)[0]
    keys = {bytes(table[r].tobytes()) for r in range(usable)}
    want = [j * n + i for j in range(3) for i in range(usable) if bytes(inputs[j][i].tobytes()) not in keys]
    assert want == [4, 2 * n]
    count, rows = lookup_missing_rows(inputs, table, k, usable)
    assert count == 2 and rows.tolist() == want
    assert lookup_missing_rows(inputs, table, k, usable, 1)[1].tolist() == want[:1]
    assert lookup_missing_rows(inputs, table, k, 0)[0] == 0


def test_copy_check_contract():
    rng = np.random.default_rng(3)
    for n_cols, k, mism in [(1, 1, 0), (2, 3, 3), (5, 6, 40)]:
        cols, nxt = random_cycles(rng, n_cols, k, mism)
        vals = np.concatenate(cols)
        want = [f for f in range(n_cols << k) if not np.array_equal(vals[f], vals[int(nxt[f])])]
        count, rows = copy_check(cols, nxt, k)
        assert count == len(want) and rows.tolist() == want
        assert sorted(nxt.tolist()) == list(range(n_cols << k))  # a permutation: every cell is in exactly one cycle
        if mism == 0:
            assert count == 0


def test_lookup_search_equals_lexicographic_membership():
    """the limb-0 search of the model against np.isin on whole rows, including table values that share limb 0 (the fallback)"""
    from lookup_model import make_case

    rng = np.random.default_rng(4)
    for k, shape in [(8, "dup"), (10, "range"), (9, "skew")]:
        inputs, table, usable = make_case(shape, k, 2, 40 + k, (1 << k) - 5)
        inputs[0][rng.integers(0, usable, 9)] = random_fr(rng, 9)
        for col in inputs:
            want = np.flatnonzero(~np.isin(_as_keys(col[:usable]), _as_keys(table[:usable])))
            count, rows = lookup_missing_rows([col], table, k, usable)
            assert count == len(want) and rows.tolist() == want.tolist()
    table = random_fr(rng, 16)
    table[5, 0] = table[2, 0]  # two distinct values share limb 0
    col = table[rng.integers(0, 16, 16)]
    col[3] = table[2] ^ np.array([0, 1, 0, 0], np.uint64)  # limb 0 of a table value, another value
    want = [i for i in range(16) if not any(np.array_equal(col[i], table[r]) for r in range(16))]
    assert lookup_missing_rows([col], table, 4, 16)[1].tolist() == want == [3]
