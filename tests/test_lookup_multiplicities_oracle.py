"""The rule of the lookup multiplicity column m(X) (mv_lookup::Argument::prepare), checked without a device:

- the host default of Ops::lookup_multiplicities in plonk_b200.hpp (the C++ driver tests/cpp/test_lookup_multiplicities.cpp,
  `host` mode) against a Python dict model written out below, on the corner cases of the rule;
- tests/lookup_model.py's vectorised model (the reference of the GPU tests at large k) against the same dict model;
- m closes the log-derivative running sum: with the oracle's logup_running_sum, phi[usable] = 0 on a satisfied lookup.
"""
import os
import subprocess

import numpy as np
import pytest

from lookup_model import make_case, mont, numpy_model, random_fr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "test_lookup_multiplicities.cpp")
BIN = os.path.join(ROOT, "tests", "cpp", "test_lookup_multiplicities")


def binary():
    deps = [SRC] + [os.path.join(ROOT, "scroll-prover_b200", h) for h in ("plonk_b200.hpp", "halo2_b200.hpp")]
    if not os.path.exists(BIN) or any(os.path.getmtime(d) > os.path.getmtime(BIN) for d in deps):
        lib = os.path.join(ROOT, "scroll-prover_b200")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-o", BIN, SRC, "-L" + lib, "-lb200zk", "-Wl,-rpath," + lib])
    return BIN


def host_default(inputs, table, k, usable, tmp_path):
    """Ops::lookup_multiplicities' host body: (m, panicked)"""
    src, dst = tmp_path / "in.bin", tmp_path / "out.bin"
    with open(src, "wb") as f:
        f.write(np.array([k, len(inputs)], np.uint32).tobytes() + np.array([usable], np.uint64).tobytes())
        for col in [table] + list(inputs):
            f.write(np.ascontiguousarray(col, np.uint64).tobytes())
    r = subprocess.run([binary(), "host", str(src), str(dst)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and r.stdout.strip().endswith("OK"), r.stdout + r.stderr
    raw = np.fromfile(dst, np.uint64)
    if raw[0] == 1:
        assert "lookup input is not in the table" in r.stdout
        return None, True
    return raw[1:].reshape(-1, 4), False


def dict_rule(inputs, table, k, usable):
    """the rule row by row: the first usable table row of each value takes the counts; first_missing = j * 2^k + i"""
    first = {}
    for r in range(usable):
        first.setdefault(bytes(table[r].tobytes()), r)
    counts, first_missing = {}, None
    for j, col in enumerate(inputs):
        for i in range(usable):
            r = first.get(bytes(col[i].tobytes()))
            if r is None:
                first_missing = (j << k) + i if first_missing is None else first_missing
            else:
                counts[r] = counts.get(r, 0) + 1
    m = np.zeros((1 << k, 4), np.uint64)
    for r, c in counts.items():
        m[r] = mont(c)
    return m, first_missing


def corner_cases():
    """(name, inputs, table, k, usable)"""
    rng = np.random.default_rng(7)
    out = []
    k, n = 6, 64
    # duplicated table values: the first usable row holding a value takes all its counts
    t = random_fr(rng, n)
    t[10] = t[3]
    t[40] = t[3]
    t[20] = t[33]
    col = t[rng.integers(0, 57, n)]
    col[:6] = t[[3, 10, 40, 33, 20, 3]]
    out.append(("duplicates", [col], t, k, 57))
    # a value present only at rows >= usable: missing, reported at the smallest (input, row)
    t2 = random_fr(rng, n)
    a, b = t2[rng.integers(0, 57, n)], t2[rng.integers(0, 57, n)]
    a[30] = t2[60]
    b[5] = t2[61]
    out.append(("only_unusable_rows", [a, b], t2, k, 57))
    b2 = b.copy()
    a2 = t2[rng.integers(0, 57, n)]
    out.append(("missing_in_second_input", [a2, b2], t2, k, 57))
    # several inputs, and every input the same column
    t3 = random_fr(rng, n)
    out.append(("several_inputs", [t3[rng.integers(0, 50, n)] for _ in range(5)], t3, k, 50))
    same = t3[rng.integers(0, 50, n)]
    out.append(("all_inputs_equal", [same, same.copy(), same.copy()], t3, k, 50))
    # zero values in table and inputs (the disabled rows of a range check), including a zero only above usable
    t4 = random_fr(rng, n)
    t4[12] = 0
    t4[50] = 0
    z = t4[rng.integers(0, 57, n)]
    z[::3] = 0
    out.append(("zeros", [z], t4, k, 57))
    t5 = random_fr(rng, n)
    t5[60] = 0
    z5 = t5[rng.integers(0, 57, n)]
    z5[9] = 0
    out.append(("zero_only_unusable", [z5], t5, k, 57))
    # usable = 2^k: every row counts, the last row included
    t6 = random_fr(rng, n)
    c6 = t6[rng.integers(0, n, n)]
    c6[n - 1] = t6[n - 1]
    out.append(("usable_full", [c6, t6.copy()], t6, k, n))
    out.append(("usable_zero", [c6], t6, k, 0))
    out.append(("k0", [t6[:1].copy()], t6[:1].copy(), 0, 1))
    return out


CASES = corner_cases()


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_host_default_follows_the_rule(case, tmp_path):
    name, inputs, table, k, usable = case
    m_ref, miss_ref = dict_rule(inputs, table, k, usable)
    m, panicked = host_default(inputs, table, k, usable, tmp_path)
    assert panicked == (miss_ref is not None)
    if not panicked:
        assert np.array_equal(m, m_ref)
    expect_missing = {"only_unusable_rows": 30, "missing_in_second_input": (1 << 6) + 5, "zero_only_unusable": 9}
    assert miss_ref == expect_missing.get(name)
    if name == "duplicates":
        assert not m_ref[10].any() and not m_ref[40].any() and not m_ref[33].any() and m_ref[3].any() and m_ref[20].any()


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_vectorised_model_equals_the_rule(case):
    _, inputs, table, k, usable = case
    m_ref, miss_ref = dict_rule(inputs, table, k, usable)
    m, miss = numpy_model(inputs, table, k, usable)
    assert miss == miss_ref
    if miss is None:
        assert np.array_equal(m, m_ref)


@pytest.mark.parametrize("shape,k,n_inputs,usable", [("dup", 9, 1, 500), ("range", 10, 2, 1017), ("skew", 8, 3, None),
                                                     ("dup", 7, 8, None), ("range", 5, 1, 20)])
def test_generated_shapes(shape, k, n_inputs, usable, tmp_path):
    inputs, table, usable = make_case(shape, k, n_inputs, 11, usable)
    m_ref, miss_ref = dict_rule(inputs, table, k, usable)
    assert miss_ref is None
    m, miss = numpy_model(inputs, table, k, usable)
    assert miss is None and np.array_equal(m, m_ref)
    mh, panicked = host_default(inputs, table, k, usable, tmp_path)
    assert not panicked and np.array_equal(mh, m_ref)


@pytest.mark.parametrize("name", ["duplicates", "several_inputs", "all_inputs_equal", "zeros"])
def test_multiplicities_close_the_running_sum(name):
    """phi[0] = 0, phi[i+1] = phi[i] + sum_j 1/(f_j[i] + beta) - m[i]/(t[i] + beta): a satisfied lookup closes at row usable,
    and moving one table row's count onto another row breaks it"""
    from oracle import oracle as O

    _, inputs, table, k, usable = next(c for c in CASES if c[0] == name)
    m, miss = dict_rule(inputs, table, k, usable)
    assert miss is None and usable < (1 << k)
    beta, zero = O.fill_fr(1, 31337)[0], np.zeros(4, np.uint64)
    assert not O.logup_running_sum(inputs, table, m, beta, k, zero)[usable].any()
    hit = np.nonzero(m.any(axis=1))[0]
    r = int(hit[0])
    s = next(x for x in range(usable) if not np.array_equal(table[x], table[r]) and not np.array_equal(m[x], m[r]))
    bad = m.copy()
    bad[r], bad[s] = m[s], m[r]
    assert not np.array_equal(bad, m)
    assert O.logup_running_sum(inputs, table, bad, beta, k, zero)[usable].any()
