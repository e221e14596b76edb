"""Models of dev::MockProver::verify_par's three device checks (csrc/mock.cu), each a list of failing flat indices in ascending order
of which the first min(cap, count) are returned with the count:

- nonzero_rows(values):                           rows whose field element is not zero (a gate's failing rows);
- lookup_missing_rows(inputs, table, k, usable):  j * 2^k + i of every (input j, row i < usable) whose value is in no usable table
                                                  row (rows >= usable of the inputs are never reported, rows >= usable of the table
                                                  never match);
- copy_check(cols, nxt, k):                       c * 2^k + r of every cell whose value differs from that of cell nxt[c * 2^k + r].

Field elements are (n, 4) uint64 Montgomery limbs and are compared limb for limb.  mock_failures() assembles MockProver's list from
the three checks in the order of plonk_b200.hpp's mock_check: gates, then lookups, then permutation columns."""
import numpy as np

from lookup_model import random_fr

GATE, LOOKUP, PERMUTATION = 0, 1, 2


def _listed(flags, cap):
    rows = np.flatnonzero(flags).astype(np.uint64)
    return len(rows), rows if cap is None else rows[:cap]


def _as_keys(a):
    """(m, 4) uint64 -> one structured key per row (compared field by field, so np.isin sorts them lexicographically)"""
    a = np.ascontiguousarray(a, dtype=np.uint64)
    return a.view([("l0", "<u8"), ("l1", "<u8"), ("l2", "<u8"), ("l3", "<u8")]).reshape(-1)


def nonzero_rows(values, cap=None):
    return _listed(np.asarray(values, dtype=np.uint64).any(axis=1), cap)


def _in_table(values, table):
    """row-wise membership of `values` in `table` ((m, 4) uint64 each).  The table is sorted by limb 0 and searched with it, the
    other limbs confirm; when two distinct table values share limb 0 that search is ambiguous and the lexicographic np.isin
    decides instead (slower, and it never happens with random or small-integer data)."""
    if len(table) == 0:
        return np.zeros(len(values), bool)
    order = np.argsort(table[:, 0], kind="stable")
    ts = table[order]
    same0 = ts[1:, 0] == ts[:-1, 0]
    if not np.all((ts[1:] == ts[:-1]).all(axis=1)[same0]):
        return np.isin(_as_keys(values), _as_keys(table))
    keys, qo = np.ascontiguousarray(ts[:, 0]), np.argsort(values[:, 0])
    pos = np.empty(len(values), np.int64)
    pos[qo] = np.minimum(np.searchsorted(keys, values[qo, 0]), len(ts) - 1)  # sorted queries: a merge, not random probes
    return (ts[pos] == values).all(axis=1)


def lookup_missing_rows(inputs, table, k: int, usable: int, cap=None):
    n = 1 << k
    tab = np.ascontiguousarray(np.asarray(table, dtype=np.uint64)[:usable])
    flags = np.zeros(len(inputs) * n, bool)
    for j, col in enumerate(inputs):
        flags[j * n: j * n + usable] = ~_in_table(np.asarray(col, dtype=np.uint64)[:usable], tab)
    return _listed(flags, cap)


def copy_check(cols, nxt, k: int, cap=None):
    vals = np.concatenate([np.asarray(c, dtype=np.uint64) for c in cols])
    nxt = np.asarray(nxt, dtype=np.uint64)
    assert len(nxt) == len(cols) << k and (nxt < len(nxt)).all()
    return _listed((vals != vals[nxt.astype(np.int64)]).any(axis=1), cap)


def mock_failures(case):
    """MockProver's failure list [(kind, index, row)] from the inputs of the three checks (a read_host_dump case)"""
    k, n, u = case["k"], 1 << case["k"], case["usable"]
    out = []
    for g, v in enumerate(case["gates"]):
        out += [(GATE, g, int(r)) for r in nonzero_rows(v)[1]]
    for li, (inp, tab) in enumerate(case["lookups"]):
        out += [(LOOKUP, li, int(r)) for r in lookup_missing_rows([inp], tab, k, u)[1]]
    if case["perm"]:
        out += [(PERMUTATION, int(f) // n, int(f) % n) for f in copy_check(case["perm"], case["next"], k)[1]]
    return out


def read_host_dump(path):
    """the cases tests/cpp/test_mock_device.cpp `host` writes (its header comment gives the layout)"""
    raw = open(path, "rb").read()
    pos = 0

    def take(dtype, count):
        nonlocal pos
        a = np.frombuffer(raw, dtype=dtype, count=count, offset=pos)
        pos += a.nbytes
        return a

    cases = []
    while pos < len(raw):
        k = int(take(np.uint32, 1)[0])
        n = 1 << k
        usable = int(take(np.uint64, 1)[0])
        n_gates, n_lookups, n_perm = (int(x) for x in take(np.uint32, 3))
        col = lambda: take(np.uint64, 4 * n).reshape(n, 4)
        gates = [col() for _ in range(n_gates)]
        lookups = [(col(), col()) for _ in range(n_lookups)]
        perm = [col() for _ in range(n_perm)]
        nxt = take(np.uint64, n_perm * n)
        n_fail = int(take(np.uint64, 1)[0])
        failures = []
        for _ in range(n_fail):
            kind, index = (int(x) for x in take(np.uint32, 2))
            failures.append((kind, index, int(take(np.uint64, 1)[0])))
        cases.append(dict(k=k, usable=usable, gates=gates, lookups=lookups, perm=perm, next=nxt, failures=failures))
    return cases


# ---------------------------------------------------------------- test data
def sparse_values(rng, n: int, density: float):
    """n field elements, each nonzero with probability `density` (a random one of its limbs nonzero, or all of them)"""
    v = np.zeros((n, 4), np.uint64)
    hit = np.flatnonzero(rng.random(n) < density)
    v[hit] = random_fr(rng, len(hit))
    one_limb = hit[rng.random(len(hit)) < 0.5]  # a value with three zero limbs is still nonzero
    keep = rng.integers(0, 4, len(one_limb))
    mask = np.zeros((len(one_limb), 4), bool)
    mask[np.arange(len(one_limb)), keep] = True
    v[one_limb] = np.where(mask, v[one_limb] | np.uint64(1), np.uint64(0))
    return v


def random_cycles(rng, n_cols: int, k: int, mismatches: int):
    """(cols, nxt): the n_cols * 2^k cells cut into random cycles (lengths 1 .. 16) whose cells hold one value each; then
    `mismatches` random cells get another value"""
    total = n_cols << k
    order = rng.permutation(total)
    lengths = []
    left = total
    while left:
        lengths.append(min(left, int(rng.integers(1, 17))))
        left -= lengths[-1]
    lengths = np.array(lengths)
    starts = np.concatenate([[0], np.cumsum(lengths)[:-1]])
    cycle_of = np.repeat(np.arange(len(lengths)), lengths)
    pos = np.arange(total)
    succ_pos = np.where(pos + 1 == starts[cycle_of] + lengths[cycle_of], starts[cycle_of], pos + 1)
    nxt = np.empty(total, np.uint64)
    nxt[order] = order[succ_pos]
    vals = np.empty((total, 4), np.uint64)
    vals[order] = random_fr(rng, len(lengths))[cycle_of]
    bad = rng.choice(total, size=min(mismatches, total), replace=False)
    vals[bad] = random_fr(rng, len(bad))
    return [vals[c << k:(c + 1) << k] for c in range(n_cols)], nxt
