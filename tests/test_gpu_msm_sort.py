"""The MSM bucket sort (csrc/msm.cu: msm_count -> bin scan -> msm_partition -> msm_bin_sort / msm_big_*) on every shape the
accumulate side depends on, checked through the MSM result against the oracle (or, where the oracle would take minutes,
against a closed form over repeated known points):

plain bases (one bucket set per window) and precomputed SRS tables (one set, table offset in the entry); batches of 1 to 32
columns; sliced commits (a first offset into the SRS); n from 1 up, not a multiple of any tile; every window 2..24;
all-zero, single-value (one giant bucket, hence one giant bin) and witness-like columns; the (1 << c) - v sign edge."""
import numpy as np
import pytest

from oracle import oracle as O
from msm_sort_model import recode_counts

pytestmark = pytest.mark.gpu
SEED = 0x5EEDB2005047


def aff(j):
    return O.g1_to_affine(j)


def sign_edge(c, count):
    """scalars whose recoding hits v == 2^c (a zero digit that carries) and the other ends of the digit range"""
    out = []
    for k in range(1, 254 // c + 1):
        for v in ((1 << (c * k)) - 1, (1 << (c * k)) - (1 << (c - 1)), (1 << (c * k)) + (1 << (c - 1)) + 1):
            if 0 < v < O.R_MOD:
                out.append(v)
    out += [O.R_MOD - 1, O.R_MOD - (1 << c), 1 << (c - 1), (1 << (c - 1)) + 1]
    return np.stack([O.fr_from_int(v) for v in out[:count]])


def eight_point_bases(ctx, n):
    """bases P_i = (3 + i % 8) G, so that sum s_i P_i has a closed form"""
    pts8 = ctx.g1_generator_mul_batch(np.stack([O.fr_from_int(3 + i) for i in range(8)]))
    return np.tile(pts8, ((n + 7) // 8, 1))[:n]


@pytest.mark.parametrize("c", [2, 3, 7, 9, 10, 13, 17, 20, 21, 24])
def test_every_window_with_sign_edges(ctx, c):
    n = 3001
    bases = O.fill_points(n, SEED + c, 16)
    scal = O.fill_fr(n, SEED + 100 + c, witness_like=(c % 2 == 1))
    edge = sign_edge(c, 200)
    scal[: len(edge)] = edge
    exp = aff(O.best_multiexp(scal, bases, threads=16))
    ctx.msm_set_window(c)
    try:
        ctx.msm_total_adds(reset=True)
        got = ctx.best_multiexp(scal, bases)
        adds = ctx.msm_total_adds(reset=True)
        assert ctx.msm_last_stats()["window_bits"] == c
    finally:
        ctx.msm_set_window(0)
    assert np.array_equal(aff(got), exp), c
    vals = [O.fr_to_int(s) for s in scal]
    assert adds == sum(recode_counts(v, c) for v in vals)  # M, the entry count the bench's roofline uses


@pytest.mark.parametrize("n", [1, 2, 31, 8191, 8193, 40961])
@pytest.mark.parametrize("kind", ["uniform", "witness", "zero", "single"])
def test_plain_bases_sizes_and_distributions(ctx, n, kind):
    bases = O.fill_points(n, SEED + n, 16)
    if kind == "zero":
        scal = np.zeros((n, 4), np.uint64)
    elif kind == "single":
        scal = np.tile(O.fr_from_int(0xDEADBEEF12345), (n, 1))
    else:
        scal = O.fill_fr(n, SEED + 7 * n, witness_like=(kind == "witness"))
    got = ctx.best_multiexp(scal, bases)
    assert np.array_equal(aff(got), aff(O.best_multiexp(scal, bases, threads=16))), (n, kind)


def test_precomputed_tables_batches_and_slices(ctx):
    """precomputed SRS (one bucket set, entry = i + w * stride): batches of 1, 5 and 32 columns, a short prefix and a slice
    at an offset; the batch mixes zero, single-value, witness-like and uniform columns"""
    n = (1 << 16) + 5
    bases = O.fill_points_chain(n, 4711, 16)
    srs = ctx.srs_register(bases)
    m = n - 3  # not a multiple of any tile
    cols = []
    for j in range(32):
        if j % 9 == 4:
            c = np.zeros((m, 4), np.uint64)
        elif j % 9 == 7:
            c = np.tile(O.fr_from_int(j + 2), (m, 1))
        else:
            c = O.fill_fr(m, SEED + 300 + j, witness_like=(j % 2 == 0))
        cols.append(c)
    exp = [aff(O.best_multiexp(c, bases[:m], threads=16)) for c in cols]
    for count in (1, 5, 32):
        got = srs.msm_batch(cols[:count])
        for j in range(count):
            assert np.array_equal(aff(got[j]), exp[j]), (count, j)
    # a slice of the tables: sum_i s_i P_{first + i}
    first, ln = 4000, (1 << 16) - 4000
    s = cols[1][:ln]
    assert np.array_equal(aff(srs.msm_range(s, first)), aff(O.best_multiexp(s, bases[first:first + ln], threads=16)))
    srs.release()


def test_one_bin_holds_every_entry(ctx):
    """a column of one repeated scalar: every window's digits fall in one bucket, so each bin is far above the one-block
    limit and goes through the multi-block path"""
    n = 1 << 19
    bases = eight_point_bases(ctx, n)
    v = 0x1234_5678_9ABC_DEF0_1122_3344
    sc = np.tile(O.fr_from_int(v), (n, 1))
    got = ctx.best_multiexp(sc, bases)
    k = v * sum(3 + i % 8 for i in range(n)) % O.R_MOD
    exp = aff(O.g1_mul(O.g1_from_affine(O.g1_generator()), O.fr_from_int(k)))
    assert np.array_equal(aff(got), exp)


def test_bucket_of_2_20_entries_inside_a_batch(ctx):
    """precomputed 2^20 tables: a batch of ordinary columns with one column whose 2^20 scalars are all 1 (one bucket of
    2^20 entries in window 0, every other window empty)"""
    n = 1 << 20
    bases = eight_point_bases(ctx, n)
    srs = ctx.srs_register(bases)
    rng = np.random.default_rng(SEED)
    small = rng.integers(0, 1 << 62, size=(n,), dtype=np.uint64)
    cols = [np.tile(O.fr_from_int(1), (n, 1))]
    # ordinary columns with a closed form: v_i < 2^62 given in canonical form, converted on the device (x * R^2 / R)
    raw = np.zeros((n, 4), np.uint64)
    raw[:, 0] = small
    r2 = O.fr_from_int(1 << 256)
    mont = ctx.poly_scale(raw, r2)
    cols += [mont, np.zeros((n, 4), np.uint64), mont[::-1].copy()]
    got = srs.msm_batch(cols)
    weights = np.array([3 + i % 8 for i in range(n)], dtype=object)
    vals = small.astype(object)
    G = O.g1_from_affine(O.g1_generator())
    ks = [int(weights.sum()), int((vals * weights).sum()), 0, int((vals[::-1] * weights).sum())]
    for j, k in enumerate(ks):
        exp = aff(O.g1_mul(G, O.fr_from_int(k % O.R_MOD)))
        assert np.array_equal(aff(got[j]), exp), j
    srs.release()


def test_column_pipeline_commits(ctx, zk):
    """run_column_jobs (mode 0 commitments, batched inside the library) over zero, single-value and witness-like columns"""
    k = 13
    n = 1 << k
    gl = O.fill_points_chain(n, 8080, 16)
    s_gl = ctx.srs_register(gl, zk.SRS_G_LAGRANGE)
    dom = zk.EvaluationDomain(ctx, 5, k)
    cols = [np.zeros((n, 4), np.uint64), np.tile(O.fr_from_int(5), (n, 1))]
    cols += [O.fill_fr(n, SEED + 900 + i, witness_like=(i % 2 == 0)) for i in range(6)]
    jobs = [(c, s_gl, 0, None, None) for c in cols]
    res = zk.run_column_jobs(ctx, jobs, k, omega_inv=dom.omega_inv, extended_omega=dom.extended_omega,
                             extended_omega_inv=dom.extended_omega_inv, extended_k=k + 2)
    ctx.synchronize()
    for i, c in enumerate(cols):
        assert np.array_equal(aff(res[i]), aff(O.best_multiexp(c, gl, threads=16))), i
    s_gl.release()
