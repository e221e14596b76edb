"""dev::MockProver::verify_par's checks on the device (csrc/mock.cu): b200zk_nonzero_rows, b200zk_lookup_missing_rows and
b200zk_copy_check bit for bit against tests/mock_model.py (itself pinned to the host mock_prove in tests/test_mock_model.py) for
k = 1 .. 20 and 24, with cap 0, below the count and above it, all-zero and all-failing inputs and rows in device memory; every
argument error; and mock_prove(DeviceOps, ...) against the host mock_prove through the C++ driver, on the session circuits and on
a synthetic circuit at k = 20."""
import subprocess

import numpy as np
import pytest

from lookup_model import make_case, random_fr
from mock_model import copy_check, lookup_missing_rows, nonzero_rows, random_cycles, sparse_values
from test_mock_model import SESSION_CASES, binary

pytestmark = pytest.mark.gpu

KS = list(range(1, 21)) + [24]


@pytest.fixture(autouse=True)
def one_stream(ctx):
    """torch tensors in and out: the library runs on torch's current stream for the duration of a test.  The blocks torch
    cached for this test's stream can only be reused on that stream, so they are handed back to the device afterwards: later
    tests in the session (the 2^28 transform needs 40 GiB free) must find the memory these tests used."""
    import torch

    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        ctx.set_stream(s.cuda_stream)
        yield
        ctx.synchronize()
    ctx.set_stream(None)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def dev(a):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint64).view(np.int64)).cuda()


def caps(count):
    return [None, 0, max(0, count // 2), count + 3]


def same(got, want, cap):
    """(count, rows) of the device against the model's full list, for one cap"""
    count, rows = got
    w_count, w_rows = want
    assert count == w_count
    rows = rows.cpu().numpy().view(np.uint64) if hasattr(rows, "cpu") else np.asarray(rows, np.uint64)
    expect = w_rows if cap is None else w_rows[:cap]
    assert np.array_equal(rows, expect), (len(rows), len(expect))


@pytest.mark.parametrize("k", KS)
def test_nonzero_rows(ctx, k):
    import torch

    rng = np.random.default_rng(k)
    n = 1 << k
    for density in (0.0, 0.002, 0.3, 1.0):
        v = sparse_values(rng, n, density)
        dv = dev(v)
        want = nonzero_rows(v)
        for cap in caps(want[0]):
            same(ctx.nonzero_rows(dv, cap), want, cap)
        out = torch.full((want[0] + 1,), -1, dtype=torch.int64, device="cuda")  # the list written to device memory
        same(ctx.nonzero_rows(dv, out=out), want, None)
        assert int(out[-1]) == -1
    assert ctx.nonzero_rows(dev(np.zeros((n, 4), np.uint64)))[0] == 0


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("n_inputs", [1, 8])
def test_lookup_missing_rows(ctx, k, n_inputs):
    if k == 24 and n_inputs == 8:
        pytest.skip("8 inputs at 2^24 rows: 4 GiB of host test data")
    rng = np.random.default_rng(100 * k + n_inputs)
    n = 1 << k
    usable = max(1, n - 7)
    inputs, table, usable = make_case("dup", k, n_inputs, 500 + k, usable)  # duplicated table values
    for j in range(n_inputs):  # misses below usable, and values only in table rows >= usable; rows >= usable are never listed
        hit = rng.integers(0, n, size=min(n, 1 + n // 64))
        inputs[j][hit] = random_fr(rng, len(hit))
        if usable < n:
            inputs[j][rng.integers(0, usable)] = table[n - 1]
    di, dt = [dev(c) for c in inputs], dev(table)
    want = lookup_missing_rows(inputs, table, k, usable)
    assert want[0] > 0
    for cap in caps(want[0]):
        same(ctx.lookup_missing_rows(di, dt, k, usable, cap), want, cap)
    # every usable row failing, and none
    fresh = [random_fr(rng, n) for _ in range(n_inputs)]
    same(ctx.lookup_missing_rows([dev(c) for c in fresh], dt, k, usable), lookup_missing_rows(fresh, table, k, usable), None)
    assert ctx.lookup_missing_rows([dt] * n_inputs, dt, k, usable)[0] == 0


@pytest.mark.parametrize("k", KS)
def test_copy_check(ctx, k):
    rng = np.random.default_rng(7 * k)
    n_cols = 1 if k == 24 else (6 if k <= 16 else 3)
    cols, nxt = random_cycles(rng, n_cols, k, mismatches=1 + (n_cols << k) // 500)
    dc, dn = [dev(c) for c in cols], dev(nxt)
    want = copy_check(cols, nxt, k)
    for cap in caps(want[0]):
        same(ctx.copy_check(dc, dn, k, cap), want, cap)
    # every cell failing: distinct values, each cell's successor the next cell
    vals = [random_fr(rng, 1 << k) for _ in range(n_cols)]
    shift = (np.arange(n_cols << k, dtype=np.uint64) + 1) % (n_cols << k)
    if (n_cols << k) > 1:
        same(ctx.copy_check([dev(c) for c in vals], dev(shift), k), copy_check(vals, shift, k), None)
        assert ctx.copy_check([dev(c) for c in vals], dev(shift), k, 0)[0] == n_cols << k


def test_argument_errors(ctx, zk):
    k, n = 4, 16
    inputs, table, usable = make_case("dup", k, 1, 9)
    col, tab = dev(inputs[0]), dev(table)
    nxt = dev(np.arange(n, dtype=np.uint64))
    lib = zk.lib()
    import ctypes as C

    count = C.c_uint64()
    bad = [
        lambda: ctx.nonzero_rows(inputs[0]),  # a host column
        lambda: ctx._ck(lib.b200zk_nonzero_rows(ctx._h, C.c_void_p(col.data_ptr()), n, None, 4, C.byref(count))),  # null rows, cap > 0
        lambda: ctx._ck(lib.b200zk_nonzero_rows(ctx._h, C.c_void_p(col.data_ptr()), n, None, 0, None)),  # null count_out
        lambda: ctx.lookup_missing_rows([inputs[0]], tab, k, usable),  # a host input column
        lambda: ctx.lookup_missing_rows([col], table, k, usable),  # a host table
        lambda: ctx.lookup_missing_rows([col], tab, 29, usable),  # k > 28
        lambda: ctx.lookup_missing_rows([], tab, k, usable),  # no inputs
        lambda: ctx.lookup_missing_rows([col] * 65, tab, k, usable),  # more than 64 inputs
        lambda: ctx.lookup_missing_rows([col], tab, k, n + 1),  # usable > 2^k
        lambda: ctx.copy_check([inputs[0]], nxt, k),  # a host column
        lambda: ctx.copy_check([col], np.arange(n, dtype=np.uint64), k),  # a host next array
        lambda: ctx.copy_check([], nxt, k),  # no columns
        lambda: ctx.copy_check([col], nxt, 29),  # k > 28
        lambda: ctx.copy_check([col], dev(np.where(np.arange(n) == 5, n, np.arange(n)).astype(np.uint64)), k),  # next out of range
        lambda: ctx.copy_check([col, col], dev(np.full(2 * n, 2 * n + 100, np.uint64)), k),  # every next out of range
    ]
    for call in bad:
        with pytest.raises(zk.B200zkError) as e:
            call()
        assert e.value.code == zk.E_INVALID
    # the context keeps working
    assert ctx.nonzero_rows(col)[0] == nonzero_rows(inputs[0])[0]
    assert ctx.lookup_missing_rows([col], tab, k, usable)[0] == 0
    assert ctx.copy_check([col], nxt, k)[0] == 0


def run_driver(*args, timeout=900):
    r = subprocess.run([binary(), *map(str, args)], capture_output=True, text=True, timeout=timeout)
    assert r.returncode == 0 and r.stdout.strip().endswith("OK"), r.stdout[-3000:] + r.stderr[-3000:]
    return r.stdout


@pytest.mark.parametrize("k,seed,variant", SESSION_CASES + [(6, 5, 1), (8, 9, 2), (7, 11, 3)])
def test_device_ops_mock_prove_equals_the_host(k, seed, variant):
    out = run_driver("device", k, seed, variant)
    assert out.count("device == host") == 5


def test_synthetic_circuit_at_two_to_the_twenty():
    out = run_driver("synthetic", 20, 3, 300, timeout=1800)
    line = next(l for l in out.splitlines() if "device == host" in l)
    assert "gates=32 lookups=4 permutation=8" in line
    total = int(line.split("device == host, ")[1].split(" failures")[0])
    assert 300 <= total <= 10000, line
