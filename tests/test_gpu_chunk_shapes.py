"""Every element of the chunk proof's largest transforms and commitments, checked with O(n) host work per case (-m gpu).

The prover's layers run at k = 20, 24 and 25, so its transforms reach 2^27 points (three- and four-pass NTT plans) and its
commitments 2^25 bases (the plain MSM path at c = 20).  A live oracle run at those sizes takes minutes per case, so:

- A transform y_j = sum_i a_i c^i w^(ij) is checked through eval(y, r) = (r^N - 1) sum_i a_i c^i / (w^i r - 1) at a
  random r (oracle/dft_identity.c; tests/test_dft_identity.py holds it to the oracle's transforms).  An inverse transform
  is checked through the forward relation of its output.  A wrong element passes with probability <= N / |Fr| ~ 2^-226,
  and each NTT case shows that one changed output element fails the check.
- An MSM runs over bases P_i = s_i G with known discrete logs, so its result must be <a, s> G.  Each case asserts the
  window the library chose (msm_last_stats), so the intended plan is the one checked.

Each case runs on a context of its own, closed afterwards, so twiddle tables and scratch of one case do not stay behind
for the next.  A case that needs more free device memory than the card has is skipped, with the amounts."""
import json
import os
import sys

import numpy as np
import pytest

from oracle import oracle as O
from oracle import pyref as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import make_big_digests as G  # noqa: E402  (the input recipes live beside the digests)

pytestmark = pytest.mark.gpu
DIGESTS = json.load(open(os.path.join(ROOT, "tests", "golden", "big_digests.json")))
THREADS = os.cpu_count() or 8
SEED = 0xC4A2_0000
GiB = 1 << 30
FR = 32  # bytes per field element
ONE = O.const_fr("fr_ONE")
ZETA = O.const_fr("fr_ZETA")
GEN = O.g1_from_affine(O.g1_generator())


def omega_for(log_n):
    return O.fr_from_int(P.omega_for(log_n))


def point(seed):
    return O.fill_fr(1, seed)[0]


@pytest.fixture
def lctx(zk):
    import torch

    c = zk.Context(0)
    yield c
    c.close()
    torch.cuda.empty_cache()


def need_free(nbytes, what):
    import torch

    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < nbytes:
        pytest.skip(f"{what} needs {nbytes / GiB:.0f} GiB of free device memory; {free / GiB:.1f} GiB free")


def to_host(t):
    return t.cpu().numpy().view(np.uint64)


def rand_dev(n, seed):
    """n uniform field elements (raw limbs < 2^252 < r, so valid Montgomery values) drawn on the device"""
    import torch

    g = torch.Generator(device="cuda").manual_seed(seed)
    a = torch.randint(-(2 ** 63), 2 ** 63 - 1, (n, 4), dtype=torch.int64, device="cuda", generator=g)
    a[:, 3] &= 0x0FFFFFFFFFFFFFFF
    return a


def assert_transform(y, a, c, w, N, r, name, out_is_y, mutate=True):
    """y_j = sum_i a_i c^i w^(ij) for every j < N.  out_is_y names the side the device wrote (y for a forward transform,
    a for an inverse one); with mutate, that side with one element changed must fail the same check."""
    lhs, rhs = O.eval_polynomial_mt(y, r), O.dft_eval_rhs(a, c, w, r, N)
    assert np.array_equal(lhs, rhs), name
    if not mutate:
        return
    out = y if out_is_y else a
    i = len(out) * 5 // 7
    saved = out[i].copy()
    out[i] = O.fr_add(out[i], ONE)
    try:
        bad = O.eval_polynomial_mt(y, r) if out_is_y else O.dft_eval_rhs(a, c, w, r, N)
        assert not np.array_equal(bad, rhs if out_is_y else lhs), f"{name}: a changed output element passed"
    finally:
        out[i] = saved


# --------------------------------------------------------------------------- NTT
@pytest.mark.parametrize("log_n", range(19, 29))
def test_best_fft_every_plan(lctx, log_n):
    """best_fft forward at every size from 2^19 (three passes) to 2^28 (four passes: 7,7,7,7)"""
    import torch

    n = 1 << log_n
    need_free(3 * FR * n + GiB, f"a 2^{log_n} transform")  # data, pass scratch, twiddle table
    a_dev = rand_dev(n, log_n)
    a = to_host(a_dev)
    w = omega_for(log_n)
    torch.cuda.synchronize()
    lctx.best_fft(a_dev, w, log_n)
    lctx.synchronize()
    y = to_host(a_dev)
    del a_dev
    assert_transform(y, a, ONE, w, n, point(SEED + log_n), f"best_fft 2^{log_n}", out_is_y=True)


@pytest.mark.parametrize("k", [20, 24, 25])
def test_column_transform_chain(lctx, zk, k):
    """lagrange_to_coeff (2^k), coeff_to_extended (2^(k+2)), extended_to_coeff (2^(k+2)) on one device-resident column"""
    import torch

    dom, od = zk.EvaluationDomain(lctx, 5, k), O.EvaluationDomain(5, k)
    n, N = 1 << k, 1 << dom.extended_k
    need_free(FR * (n + 4 * N) + GiB, f"the k = {k} chain")  # column, coset, pass scratch, two twiddle tables
    v_dev = rand_dev(n, 100 + k)
    v = to_host(v_dev)
    torch.cuda.synchronize()
    dom.lagrange_to_coeff(v_dev)
    ext = dom.coeff_to_extended(v_dev)
    lctx.synchronize()
    coeff, e = to_host(v_dev), to_host(ext)
    del v_dev
    assert_transform(v, coeff, ONE, od.omega, n, point(SEED + 200 + k), f"lagrange_to_coeff 2^{k}", out_is_y=False)
    assert_transform(e, coeff, ZETA, od.extended_omega, N, point(SEED + 300 + k), f"coeff_to_extended 2^{N.bit_length() - 1}",
                     out_is_y=True)
    dom.extended_to_coeff(ext)
    lctx.synchronize()
    b = to_host(ext)
    del ext
    assert not b[n:].any(), "extended_to_coeff: coefficients above 2^k"
    assert np.array_equal(b[:n], coeff)
    assert_transform(e, b[:n], ZETA, od.extended_omega, N, point(SEED + 400 + k), "extended_to_coeff", out_is_y=False)


def test_coset_parts_k25(lctx, zk):
    """coeff_to_extended_part for every part j < J = 4 (the last one in place) and extended_parts_to_coeff at k = 25"""
    import torch

    k = 25
    dom, od = zk.EvaluationDomain(lctx, 5, k), O.EvaluationDomain(5, k)
    n, N, J = 1 << k, 1 << dom.extended_k, dom.n_parts
    assert J == 4
    need_free(FR * (J + 1) * n + FR * N + 2 * GiB, "the k = 25 coset parts")
    coeff_dev = rand_dev(n, 500)
    coeff = to_host(coeff_dev)
    parts = [torch.empty_like(coeff_dev) for _ in range(J - 1)]
    torch.cuda.synchronize()
    for j in range(J - 1):
        dom.coeff_to_extended_part(coeff_dev, j, out=parts[j])
    dom.coeff_to_extended_part(coeff_dev, J - 1, out=coeff_dev)
    parts.append(coeff_dev)
    lctx.synchronize()
    for j in range(J):
        g_j = O.fr_mul(ZETA, O.fr_pow_u64(od.extended_omega, j))
        assert_transform(to_host(parts[j]), coeff, g_j, od.omega, n, point(SEED + 510 + j), f"coeff_to_extended_part {j}",
                         out_is_y=True)
    del parts, coeff_dev
    # the inverse on arbitrary values: part j holds the extended coset's rows j + J*r
    vals_dev = [rand_dev(n, 520 + j) for j in range(J)]
    vals = np.stack([to_host(t) for t in vals_dev], axis=1).reshape(-1, 4)  # interleaved: row r*J + j = vals_dev[j][r]
    torch.cuda.synchronize()
    dom.extended_parts_to_coeff(vals_dev)
    lctx.synchronize()
    b = np.concatenate([to_host(t) for t in vals_dev])  # parts[t] = coefficients [t*n, (t+1)*n)
    del vals_dev
    assert_transform(vals, b, ZETA, od.extended_omega, N, point(SEED + 530), "extended_parts_to_coeff", out_is_y=False)


def test_lagrange_to_coeff_25_exact(lctx, zk):
    """every element of lagrange_to_coeff(2^25) against the live oracle and the committed digest"""
    import torch

    k = 25
    a = G.ntt_inputs(k)
    exp = O.EvaluationDomain(5, k).lagrange_to_coeff(a, THREADS)
    got = torch.from_numpy(a.view(np.int64)).cuda()
    torch.cuda.synchronize()
    zk.EvaluationDomain(lctx, 5, k).lagrange_to_coeff(got)
    lctx.synchronize()
    got = to_host(got)
    assert np.array_equal(got, exp)
    assert G.sha(got) == DIGESTS["lagrange_to_coeff_25"]


# --------------------------------------------------------------------------- MSM over bases with known discrete logs
@pytest.fixture(scope="module")
def logs():
    """s_i of the bases P_i = s_i G (2^25 of them; the smaller handles use a prefix)"""
    return O.fill_fr(1 << 25, SEED + 1)


def known_bases(ctx, s, n):
    """P_i = s_i G for i < n on the device, 64 of them compared with the oracle's scalar multiplication"""
    import torch

    p = torch.empty((n, 8), dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    ctx.g1_generator_mul_batch(s[:n], out=p)
    ctx.synchronize()
    idx = np.unique(np.linspace(0, n - 1, 64).astype(np.int64))
    sample = p[torch.from_numpy(idx).cuda()].cpu().numpy().view(np.uint64)
    for row, i in zip(sample, idx):
        assert np.array_equal(row, O.g1_to_affine(O.g1_mul(GEN, s[i]))), i
    return p


def expect(a, s):
    """<a, s> G (affine)"""
    return O.g1_to_affine(O.g1_mul(GEN, O.compute_inner_product(a, s)))


def register(ctx, s, n, precompute):
    import torch

    p = known_bases(ctx, s, n)
    ctx.srs_set_precompute(precompute)
    try:
        srs = ctx.srs_register(p)
    finally:
        ctx.srs_set_precompute(True)
    del p
    torch.cuda.empty_cache()
    return srs


def window(ctx):
    return ctx.msm_last_stats()["window_bits"]


def skip_unless_tables_fit(n, c):
    """srs_register keeps the W = 254 / c + 1 tables only when they take < 0.35 x the free device memory"""
    import torch

    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    tables = 64 * n * (254 // c + 1)
    if tables >= 0.35 * free:
        pytest.skip(f"the precomputed 2^{n.bit_length() - 1} handle needs {tables / GiB:.0f} GiB < 0.35 x free memory; "
                    f"{free / GiB:.1f} GiB free, so the library registers plain bases")


def test_msm_plain_2_25(lctx, logs):
    """the plain path at n = 2^25 (c = 20, the layer2 commitments), four columns, then a 2^24 commit over its first half"""
    n = 1 << 25
    need_free(14 * GiB, "the plain 2^25 MSM")
    srs = register(lctx, logs, n, precompute=False)
    try:
        v = O.fill_fr(1, SEED + 11)
        cols = {"uniform": O.fill_fr(n, SEED + 12), "witness-like": O.fill_fr(n, SEED + 13, witness_like=True),
                "one repeated value": np.repeat(v, n, axis=0), "all zero": np.zeros((n, 4), np.uint64)}
        for name, a in cols.items():
            got = O.g1_to_affine(srs.msm(a))
            assert window(lctx) == 20, name
            assert np.array_equal(got, expect(a, logs)), name
        del cols
        a = O.fill_fr(n // 2, SEED + 14)
        got = O.g1_to_affine(srs.msm(a))  # the first 2^24 bases of the 2^25 handle (layer1's coefficient commits)
        assert window(lctx) == 17
        assert np.array_equal(got, expect(a, logs[: n // 2]))
    finally:
        srs.release()


def test_msm_precomputed_2_24(lctx, logs):
    n = 1 << 24
    skip_unless_tables_fit(n, 22)
    srs = register(lctx, logs, n, precompute=True)
    try:
        a = O.fill_fr(n, SEED + 21, witness_like=True)
        a[3::5] = O.fill_fr(len(a[3::5]), SEED + 22)
        got = O.g1_to_affine(srs.msm(a))
        assert window(lctx) == 22
        assert np.array_equal(got, expect(a, logs[:n]))
    finally:
        srs.release()


def test_msm_precomputed_2_20_batches_range_and_boundary(lctx, logs):
    """the precomputed 2^20 handle (c = 17): batches of 16, 17 (msm_max_batch) and 18 (two pipelines) columns, a range at a
    non-zero offset, and the srs_pre_c boundary: n = 2^16 uses the tables, n = 2^16 - 1 the plain bases (table 0)"""
    n = 1 << 20
    skip_unless_tables_fit(n, 17)
    s = logs[:n]
    srs = register(lctx, logs, n, precompute=True)
    try:
        cols = [O.fill_fr(n, SEED + 30 + i, witness_like=(i % 3 == 1)) for i in range(18)]
        cols[5][:] = cols[5][0]  # one giant bucket per window
        cols[9][:] = 0
        exp = [expect(c, s) for c in cols]
        for count in (16, 17, 18):
            out = srs.msm_batch(cols[:count])
            assert window(lctx) == 17, count
            for j in range(count):
                assert np.array_equal(O.g1_to_affine(out[j]), exp[j]), (count, j)
        first, m = 3 * (1 << 16) + 5, 1 << 19
        a = O.fill_fr(m, SEED + 50)
        got = O.g1_to_affine(srs.msm_range(a, first))
        assert window(lctx) == 17
        assert np.array_equal(got, expect(a, s[first:first + m]))
        bases = known_bases(lctx, logs, 1 << 16).cpu().numpy().view(np.uint64)
        for m, c in (((1 << 16), 17), ((1 << 16) - 1, 11)):
            a = O.fill_fr(m, SEED + 60 + c)
            got = O.g1_to_affine(srs.msm(a))
            assert window(lctx) == c, m
            assert np.array_equal(got, O.g1_to_affine(O.best_multiexp(a, bases[:m], THREADS))), m
            assert np.array_equal(got, expect(a, s[:m])), m
    finally:
        srs.release()


# --------------------------------------------------------------------------- the column pipeline at the layers' shapes
def test_column_jobs_inner_k20(lctx, zk, logs):
    """inner layer: 40 pinned host columns (groups of 16, 16, 8) mixing mode 2 and mode 0 over the precomputed 2^20
    handle; the same call with the two-stream overlap off gives identical bits"""
    import torch

    k = 20
    n = 1 << k
    skip_unless_tables_fit(n, 17)
    dom, od = zk.EvaluationDomain(lctx, 5, k), O.EvaluationDomain(5, k)
    N = 1 << dom.extended_k
    s = logs[:n]
    srs = register(lctx, logs, n, precompute=True)
    checked = (0, 20, 39)  # one column of each group
    try:
        cols = [O.fill_fr(n, SEED + 100 + i, witness_like=(i % 2 == 0)) for i in range(40)]
        pinned = [torch.from_numpy(c.view(np.int64)).pin_memory() for c in cols]
        modes = [0 if i % 4 == 1 else 2 for i in range(40)]
        assert all(modes[i] == 2 for i in checked)

        def run():
            co = {i: torch.empty((n, 4), dtype=torch.int64, device="cuda") for i in checked}
            eo = {i: torch.empty((N, 4), dtype=torch.int64, device="cuda") for i in checked}
            jobs = [(pinned[i], srs, modes[i], co.get(i), eo.get(i)) for i in range(40)]
            torch.cuda.synchronize()
            res = zk.run_column_jobs(lctx, jobs, k, omega_inv=dom.omega_inv, extended_omega=dom.extended_omega,
                                     extended_k=dom.extended_k)
            lctx.synchronize()
            return res, {i: (to_host(co[i]), to_host(eo[i])) for i in checked}

        res, outs = run()
        for i in range(40):
            assert np.array_equal(O.g1_to_affine(res[i]), expect(cols[i], s)), i
        for i in checked:
            coeff, ext = outs[i]
            assert_transform(cols[i], coeff, ONE, od.omega, n, point(SEED + 600 + i), f"coefficients {i}", out_is_y=False,
                             mutate=False)
            assert_transform(ext, coeff, ZETA, od.extended_omega, N, point(SEED + 700 + i), f"extended {i}", out_is_y=True,
                             mutate=False)
        lctx.set_overlap(False)
        try:
            res2, outs2 = run()
        finally:
            lctx.set_overlap(True)
        assert np.array_equal(res2, res)
        for i in checked:
            assert np.array_equal(outs2[i][0], outs[i][0]) and np.array_equal(outs2[i][1], outs[i][1]), i
    finally:
        srs.release()


def test_column_jobs_layer2_k25(lctx, zk, logs):
    """layer2: a mode 2 job (pinned host column over the plain 2^25 handle), a mode 5 job (device coefficients -> 2^27
    coset) and a mode 4 job (2^27 device values -> coefficients, in place)"""
    import torch

    k = 25
    n = 1 << k
    need_free(44 * GiB, "the k = 25 column pipeline")
    dom, od = zk.EvaluationDomain(lctx, 5, k), O.EvaluationDomain(5, k)
    N = 1 << dom.extended_k
    srs = register(lctx, logs, n, precompute=False)
    try:
        col = O.fill_fr(n, SEED + 800, witness_like=True)
        col[1::3] = O.fill_fr(len(col[1::3]), SEED + 801)
        pinned = torch.from_numpy(col.view(np.int64)).pin_memory()
        c5_dev = rand_dev(n, 810)
        q_dev = rand_dev(N, 811)
        c5, q_in = to_host(c5_dev), to_host(q_dev)
        co2 = torch.empty((n, 4), dtype=torch.int64, device="cuda")
        eo2 = torch.empty((N, 4), dtype=torch.int64, device="cuda")
        eo5 = torch.empty((N, 4), dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        res = zk.run_column_jobs(lctx, [(pinned, srs, 2, co2, eo2), (c5_dev, None, 5, None, eo5), (q_dev, None, 4, q_dev, None)],
                                 k, omega_inv=dom.omega_inv, extended_omega=dom.extended_omega,
                                 extended_omega_inv=dom.extended_omega_inv, extended_k=dom.extended_k)
        lctx.synchronize()
        assert window(lctx) == 20
        assert np.array_equal(O.g1_to_affine(res[0]), expect(col, logs)) and not res[1:].any()
        coeff = to_host(co2)
        assert_transform(col, coeff, ONE, od.omega, n, point(SEED + 820), "mode 2 coefficients", out_is_y=False, mutate=False)
        del co2, c5_dev
        assert_transform(to_host(eo2), coeff, ZETA, od.extended_omega, N, point(SEED + 821), "mode 2 extended", out_is_y=True,
                         mutate=False)
        del eo2
        assert_transform(to_host(eo5), c5, ZETA, od.extended_omega, N, point(SEED + 822), "mode 5", out_is_y=True, mutate=False)
        del eo5
        assert_transform(q_in, to_host(q_dev), ZETA, od.extended_omega, N, point(SEED + 823), "mode 4", out_is_y=False,
                         mutate=False)
    finally:
        srs.release()
