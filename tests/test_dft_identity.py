"""The O(n) transform check (oracle/dft_identity.c, a test helper): for y_j = sum_{i<m} a_i c^i w^(ij), j < N,

    eval_polynomial(y, r) == (r^N - 1) * sum_i a_i c^i / (w^i r - 1)      (r^N != 1).

tests/test_gpu_chunk_shapes.py checks every element of the prover's largest transforms with it, so here the helper is
held to the oracle's own transforms (best_fft, EvaluationDomain) for N = 2^1 .. 2^14 in every shape those checks use:
plain, zero-padded (m < N), coset (c = zeta), coset part j (c = zeta w_ext^j, w = w_ext^J), the forward relation of an
inverse transform's output, and m > N.  A y with one element changed or two elements swapped must fail."""
import numpy as np
import pytest

from oracle import oracle as O
from oracle import pyref as P

SEED = 0xD1F7_0000


def omega_for(log_n):
    return O.fr_from_int(P.omega_for(log_n))


def powers(c, m):
    out = np.zeros((m, 4), np.uint64)
    cur = O.const_fr("fr_ONE")
    for i in range(m):
        out[i] = cur
        cur = O.fr_mul(cur, c)
    return out


def scaled_fft(a, c, omega, log_n):
    """y_j = sum_{i<len(a)} a_i c^i omega^(ij) for j < 2^log_n, with the oracle's best_fft (len(a) <= 2^log_n)"""
    buf = np.zeros((1 << log_n, 4), np.uint64)
    cp = powers(c, len(a))
    for i in range(len(a)):
        buf[i] = O.fr_mul(a[i], cp[i])
    return O.best_fft(buf, omega, log_n)


def holds(y, a, c, omega, r, N):
    return np.array_equal(O.eval_polynomial(y, r), O.dft_eval_rhs(a, c, omega, r, N, threads=4))


def cases(log_n):
    """(name, y, a, c, omega, N): y is the transform of a under (c, omega, N), computed by the oracle's transforms"""
    N = 1 << log_n
    one = O.const_fr("fr_ONE")
    w = omega_for(log_n)
    a = O.fill_fr(N, SEED + log_n)
    yield "plain", O.best_fft(a, w, log_n), a, one, w, N
    m = N // 2 + 1 if N > 2 else 1
    yield "zero-padded", scaled_fft(a[:m], one, w, log_n), a[:m], one, w, N
    zeta = O.const_fr("fr_ZETA")
    yield "coset", scaled_fft(a, zeta, w, log_n), a, zeta, w, N
    # lagrange_to_coeff: its output a' satisfies the plain forward relation with its input
    dom_n = O.EvaluationDomain(5, log_n)
    yield "inverse", a, dom_n.lagrange_to_coeff(a), one, dom_n.omega, N
    if log_n >= 3:  # EvaluationDomain(5, k): extended_k = k + 2, J = 4 parts
        k = log_n - 2
        dom = O.EvaluationDomain(5, k)
        coeff = O.fill_fr(1 << k, SEED + 100 + log_n)
        ext = dom.coeff_to_extended(coeff)
        yield "coeff_to_extended", ext, coeff, dom.g_coset, dom.extended_omega, N
        yield "extended_to_coeff", ext, dom.extended_to_coeff(ext), dom.g_coset, dom.extended_omega, N
        J = 4
        w_part = O.fr_pow_u64(dom.extended_omega, J)
        for j in range(J):
            g_j = O.fr_mul(dom.g_coset, O.fr_pow_u64(dom.extended_omega, j))
            yield f"part{j}", ext[j::J], coeff, g_j, w_part, N // J
        # m > N: one part of the transform of a full-length (N) coefficient vector
        j = 3
        g_j = O.fr_mul(dom.g_coset, O.fr_pow_u64(dom.extended_omega, j))
        yield "part of full", scaled_fft(a, dom.g_coset, dom.extended_omega, log_n)[j::J], a, g_j, w_part, N // J


@pytest.mark.parametrize("log_n", range(1, 15))
def test_identity_matches_oracle_transforms(log_n):
    r = O.fill_fr(1, SEED + 200 + log_n)[0]
    seen = set()
    for name, y, a, c, w, N in cases(log_n):
        seen.add(name)
        assert holds(y, a, c, w, r, N), name
        # one element changed: the identity fails
        bad = y.copy()
        i = (7 * log_n) % len(bad)
        bad[i] = O.fr_add(bad[i], O.const_fr("fr_ONE"))
        assert not holds(bad, a, c, w, r, N), name
        # two (different) elements swapped: the identity fails
        if len(y) >= 2:
            p, q = 0, len(y) - 1
            if not np.array_equal(y[p], y[q]):
                sw = y.copy()
                sw[[p, q]] = sw[[q, p]]
                assert not holds(sw, a, c, w, r, N), name
        # and a changed input element on the right side fails too
        bad_a = a.copy()
        bad_a[-1] = O.fr_add(bad_a[-1], O.const_fr("fr_ONE"))
        assert not holds(y, bad_a, c, w, r, N), name
    assert len(seen) == (4 if log_n < 3 else 11)


@pytest.mark.parametrize("n", [0, 1, 5, 1024, 1025, 70001])
def test_threaded_horner_matches_eval_polynomial(n):
    y = O.fill_fr(n, SEED + 400 + n)
    r = O.fill_fr(1, SEED + 401)[0]
    for t in (1, 3, 8):
        assert np.array_equal(O.eval_polynomial_mt(y, r, threads=t), O.eval_polynomial(y, r))


def test_identity_rejects_bad_roots():
    a = O.fill_fr(8, SEED + 300)
    one = O.const_fr("fr_ONE")
    w = omega_for(3)
    with pytest.raises(ValueError, match="omega"):
        O.dft_eval_rhs(a, one, omega_for(4), O.fill_fr(1, 1)[0], 8)  # omega^8 != 1
    with pytest.raises(ValueError, match="r\\^N"):
        O.dft_eval_rhs(a, one, w, O.fr_pow_u64(w, 5), 8)  # r^8 == 1: the identity says nothing
    # threads do not change the result (slices start at arbitrary indices)
    big = O.fill_fr(5000, SEED + 301)
    r = O.fill_fr(1, SEED + 302)[0]
    w13 = omega_for(13)
    zeta = O.const_fr("fr_ZETA")
    ref = O.dft_eval_rhs(big, zeta, w13, r, 1 << 13, threads=1)
    for t in (2, 3, 7, 64):
        assert np.array_equal(O.dft_eval_rhs(big, zeta, w13, r, 1 << 13, threads=t), ref)
