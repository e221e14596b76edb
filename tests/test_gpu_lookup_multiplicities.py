"""b200zk_lookup_multiplicities (csrc/lookup.cu), the m(X) column of mv_lookup::Argument::prepare, bit for bit against the rule
(tests/lookup_model.py, itself checked against a row-by-row model and the host default of Ops::lookup_multiplicities in
tests/test_lookup_multiplicities_oracle.py): random tables with duplicates, the range-check shape, skewed inputs, 1 and 8 inputs,
first_missing, argument errors; and DeviceOps::lookup_multiplicities against the Ops host default through the C++ driver."""
import subprocess

import numpy as np
import pytest

from lookup_model import make_case, numpy_model, random_fr
from test_lookup_multiplicities_oracle import binary

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def one_stream(ctx):
    """torch tensors in and out: the library runs on torch's current stream for the duration of a test"""
    import torch

    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        ctx.set_stream(s.cuda_stream)
        yield
        ctx.synchronize()
    ctx.set_stream(None)


def dev(a):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint64).view(np.int64)).cuda()


def host(t):
    return t.cpu().numpy().view(np.uint64)


def run(ctx, inputs, table, k, usable):
    import torch

    out = torch.full(((1 << k), 4), -1, dtype=torch.int64, device="cuda")  # every row must be written
    miss = ctx.lookup_multiplicities([dev(c) for c in inputs], dev(table), k, usable, out)
    return host(out), miss


def check(ctx, inputs, table, k, usable):
    m_ref, miss_ref = numpy_model(inputs, table, k, usable)
    m, miss = run(ctx, inputs, table, k, usable)
    assert miss == miss_ref
    if miss is None:
        assert np.array_equal(m, m_ref)
    return m


@pytest.mark.parametrize("k", range(1, 21))
def test_random_tables_with_duplicates(ctx, k):
    n = 1 << k
    for usable in sorted({n, max(1, n - 7)}):
        inputs, table, usable = make_case("dup", k, 1, 100 + k, usable)
        check(ctx, inputs, table, k, usable)


@pytest.mark.parametrize("k", [1, 2, 5, 8, 12, 16, 20])
@pytest.mark.parametrize("shape", ["range", "skew"])
def test_range_check_and_skewed_inputs(ctx, k, shape):
    n = 1 << k
    inputs, table, usable = make_case(shape, k, 1, 200 + k, max(1, n - 5))
    check(ctx, inputs, table, k, usable)


@pytest.mark.parametrize("shape", ["dup", "range", "skew"])
def test_eight_inputs(ctx, shape):
    for k in (3, 11, 20):
        inputs, table, usable = make_case(shape, k, 8, 300 + k, (1 << k) - 3)
        check(ctx, inputs, table, k, usable)


def test_one_value_two_to_the_twenty_times(ctx):
    """2^20 copies of one input value: the whole count lands on one row (the first usable row of the value)"""
    k = 20
    inputs, table, usable = make_case("skew", k, 1, 7)
    table[5] = table[usable // 2]  # an earlier duplicate of the hot value takes the count
    m = check(ctx, inputs, table, k, usable)
    first = int(np.nonzero((table[:usable] == table[5]).all(axis=1))[0][0])
    assert first <= 5 and np.count_nonzero(m.any(axis=1)) == 1 and m[first].any()


@pytest.mark.parametrize("shape,n_inputs", [("dup", 1), ("range", 1), ("skew", 1), ("skew", 8)])
def test_at_two_to_the_twenty_four(ctx, shape, n_inputs):
    k = 24
    inputs, table, usable = make_case(shape, k, n_inputs, 24, (1 << k) - 9)
    check(ctx, inputs, table, k, usable)


@pytest.mark.parametrize("k,n_inputs", [(4, 1), (10, 3), (16, 8), (20, 2)])
def test_first_missing(ctx, k, n_inputs):
    n = 1 << k
    rng = np.random.default_rng(k)
    inputs, table, usable = make_case("dup", k, n_inputs, 400 + k, n - 4)
    # a value held only by a row >= usable in the last column, then values in no row earlier and earlier
    j0, i0 = n_inputs - 1, int(rng.integers(0, usable))
    inputs[j0][i0] = table[n - 1]
    check(ctx, inputs, table, k, usable)
    inputs[0][usable - 1] = random_fr(rng, 1)[0]
    _, miss = run(ctx, inputs, table, k, usable)
    assert miss == numpy_model(inputs, table, k, usable)[1] == (i0 if n_inputs == 1 and i0 < usable - 1 else usable - 1)
    inputs[0][0] = random_fr(rng, 1)[0]
    assert run(ctx, inputs, table, k, usable)[1] == 0
    # a missing value at a row >= usable does not count
    inputs2, table2, _ = make_case("dup", k, 1, 500 + k, n - 4)
    inputs2[0][n - 1] = random_fr(rng, 1)[0]
    check(ctx, inputs2, table2, k, usable)


def test_argument_errors(ctx, zk):
    import torch

    k = 4
    inputs, table, usable = make_case("dup", k, 1, 9)
    col, tab = dev(inputs[0]), dev(table)
    out = torch.zeros((1 << k, 4), dtype=torch.int64, device="cuda")
    bad = [
        lambda: ctx.lookup_multiplicities([inputs[0]], tab, k, usable, out),  # a host input column
        lambda: ctx.lookup_multiplicities([col], table, k, usable, out),  # a host table
        lambda: ctx.lookup_multiplicities([col], tab, k, usable, np.zeros((1 << k, 4), np.uint64)),  # a host output
        lambda: ctx.lookup_multiplicities([col], tab, 29, usable, out),  # k > 28
        lambda: ctx.lookup_multiplicities([], tab, k, usable, out),  # no inputs
        lambda: ctx.lookup_multiplicities([col] * 65, tab, k, usable, out),  # more than 64 inputs
        lambda: ctx.lookup_multiplicities([col], tab, k, (1 << k) + 1, out),  # usable > 2^k
    ]
    for call in bad:
        with pytest.raises(zk.B200zkError) as e:
            call()
        assert e.value.code == zk.E_INVALID
    assert ctx.lookup_multiplicities([col], tab, k, usable, out) is None  # the context is still usable


@pytest.mark.parametrize("k,seed", [(3, 1), (10, 2), (16, 3)])
def test_device_ops_equal_the_host_default(k, seed):
    r = subprocess.run([binary(), "random", str(k), str(seed)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and r.stdout.strip().endswith("OK"), r.stdout[-2000:] + r.stderr[-2000:]
    assert r.stdout.count("device m == host m; unsatisfied lookup -> \"lookup input is not in the table") == 2
