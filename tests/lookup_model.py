"""Models of mv_lookup::Argument::prepare's multiplicity column m(X), the rule of Ops::lookup_multiplicities in
scroll-prover_b200/plonk_b200.hpp: every (input j, row i < usable) counts once on the FIRST usable table row holding its value;
rows >= usable (and rows no input hits) stay zero; first_missing = j * 2^k + i of the smallest (j, i) whose value is in no
usable table row, None when there is none.  Values are compared limb for limb; m is Montgomery Fr, (2^k, 4) uint64.

dict_model is the rule written out row by row (small k); numpy_model is the same rule vectorised, for the sizes of the GPU
tests.  Both return (m, first_missing); m is only meaningful when first_missing is None."""
import numpy as np

R_MOD = 0x30644E72E131A029B85045B68181585D2833E84879B9709143E1F593F0000001


def mont(v: int) -> np.ndarray:
    v = (v % R_MOD) * (1 << 256) % R_MOD
    return np.array([(v >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(4)], dtype=np.uint64)


def counts_to_m(counts) -> np.ndarray:
    counts = np.asarray(counts)
    m = np.zeros((len(counts), 4), np.uint64)
    nz = np.nonzero(counts)[0]
    if len(nz):
        values, inv = np.unique(counts[nz], return_inverse=True)
        m[nz] = np.stack([mont(int(c)) for c in values])[inv]
    return m


def dict_model(inputs, table, k: int, usable: int):
    n = 1 << k
    index = {}
    for r in range(usable):
        index.setdefault(table[r].tobytes(), r)
    counts = [0] * n
    first_missing = None
    for j, col in enumerate(inputs):
        for i in range(usable):
            r = index.get(col[i].tobytes())
            if r is None:
                if first_missing is None:
                    first_missing = (j << k) + i
                continue
            counts[r] += 1
    return counts_to_m(counts), first_missing


def numpy_model(inputs, table, k: int, usable: int):
    """Sort the usable table rows by limb 0 (stable, so the smallest row of a value comes first), search every input by limb 0
    and confirm the other limbs.  Two distinct table values with the same limb 0 would defeat the search: that is asserted
    against rather than handled (it does not occur in random or small-integer data)."""
    n = 1 << k
    table = np.asarray(table, dtype=np.uint64)
    t = table[:usable]
    order = np.argsort(t[:, 0], kind="stable")
    ts = t[order]
    same0 = ts[1:, 0] == ts[:-1, 0]
    assert np.all((ts[1:] == ts[:-1]).all(axis=1)[same0]), "numpy_model: two table values share limb 0"
    start = np.ones(len(ts), bool)
    start[1:] = ~same0
    first_row, keys = order[start], ts[start, 0]
    counts = np.zeros(n, np.int64)
    first_missing = None
    for j, col in enumerate(inputs):
        v = np.asarray(col, dtype=np.uint64)[:usable]
        if len(keys) == 0:
            found, rows = np.zeros(len(v), bool), np.zeros(len(v), np.int64)
        else:
            pos = np.minimum(np.searchsorted(keys, v[:, 0]), len(keys) - 1)
            rows = first_row[pos]
            found = (keys[pos] == v[:, 0]) & (t[rows] == v).all(axis=1)
        if first_missing is None and not found.all():
            first_missing = (j << k) + int(np.argmin(found))
        counts += np.bincount(rows[found], minlength=n)
    return counts_to_m(counts), first_missing


# ---------------------------------------------------------------- test data
_P = np.array([(R_MOD >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(4)], dtype=np.uint64)


def _add_mod(a, b):
    """(a + b) mod p for (N, 4) arrays of reduced limbs"""
    out = np.empty_like(a)
    carry = np.zeros(len(a), np.uint64)
    for i in range(4):
        s = a[:, i] + b[:, i]
        c1 = (s < a[:, i]).astype(np.uint64)
        s2 = s + carry
        c2 = (s2 < s).astype(np.uint64)
        out[:, i], carry = s2, c1 | c2
    # subtract p where out >= p (no carry out of limb 3 is possible: p < 2^254)
    ge = np.ones(len(a), bool)
    decided = np.zeros(len(a), bool)
    for i in (3, 2, 1, 0):
        gt, lt = out[:, i] > _P[i], out[:, i] < _P[i]
        ge = np.where(~decided & lt, False, ge)
        decided |= gt | lt
    borrow = np.zeros(len(a), np.uint64)
    res = out.copy()
    for i in range(4):
        d = out[:, i] - _P[i]
        b1 = (out[:, i] < _P[i]).astype(np.uint64)
        d2 = d - borrow
        b2 = (d < borrow).astype(np.uint64)
        res[:, i], borrow = d2, b1 | b2
    return np.where(ge[:, None], res, out)


def small_ints(values) -> np.ndarray:
    """Montgomery limbs of the integers `values` (< 2^24), as range-check cells hold them"""
    values = np.asarray(values, dtype=np.int64)
    assert values.min(initial=0) >= 0 and values.max(initial=0) < (1 << 24)
    lo = np.stack([mont(v) for v in range(1 << 12)])
    hi = np.stack([mont(v << 12) for v in range(1 << 12)])
    return _add_mod(hi[values >> 12], lo[values & 0xFFF])


def random_fr(rng: np.random.Generator, count: int) -> np.ndarray:
    """reduced field elements with uniformly random low limbs (limb 3 below p's)"""
    a = rng.integers(0, 1 << 64, size=(count, 4), dtype=np.uint64, endpoint=False)
    a[:, 3] %= _P[3]
    return a


def make_case(shape: str, k: int, n_inputs: int, seed: int, usable: int | None = None):
    """(inputs, table, usable) of one shape:
    dup    random table with duplicated values (a pool of usable/4), inputs drawn from its usable rows
    range  range table 0 .. usable-1 as small integers, inputs ~60 % zeros and the rest from the range (witness-like)
    skew   dup table; every input cell one value, except for the odd rows of the odd columns (half the inputs one value)
    Rows >= usable of the table and of the inputs hold fresh random values."""
    n = 1 << k
    usable = n if usable is None else usable
    rng = np.random.default_rng(seed)
    table = random_fr(rng, n)
    if shape == "range":
        table[:usable] = small_ints(np.arange(usable) % (1 << 24))
    elif usable:
        pool = random_fr(rng, max(1, usable // 4))
        table[:usable] = pool[rng.integers(0, len(pool), usable)]
    inputs = []
    for j in range(n_inputs):
        col = random_fr(rng, n)
        if usable:
            if shape == "range":
                v = rng.integers(0, usable, usable)
                v[rng.random(usable) < 0.6] = 0
                col[:usable] = table[v]
            elif shape == "skew":
                col[:usable] = table[usable // 2]
                if j % 2:
                    col[1:usable:2] = table[rng.integers(0, usable, len(range(1, usable, 2)))]
            else:
                col[:usable] = table[rng.integers(0, usable, usable)]
        inputs.append(col)
    return inputs, table, usable
