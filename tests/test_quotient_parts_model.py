"""The quotient by coset parts, checked on the CPU against the whole-coset definitions.

With n = 2^k, J = 2^(extended_k - k) and w = w_ext^J, the extended coset zeta<w_ext> is the union of the J cosets
g_j<w>, g_j = zeta * w_ext^j, and extended index j + J*r is row r of part j.  The library computes a part with one size-n
transform (csrc/ntt.cu, PART kernels), turns J parts back into coefficients with per-part inverse transforms and a J-point
inverse DFT across the parts (csrc/quotient.cu, parts_idft_kernel), and runs the GraphEvaluator on one part.  These tests
restate each step with big integers (oracle/pyref.py) and compare it with coeff_to_extended / extended_to_coeff /
halo2_graph_evaluate of the whole coset; the part's programs run on the oracle's interpreter through tests/part_programs.py.
"""
import random

import numpy as np
import pytest

from oracle import oracle as O
from oracle import pyref as P
from part_programs import on_part
from quotient_programs import C_HORNER, C_MUL, S_INTER, S_X, random_program

R = P.R_MOD
CASES = [(k, logj) for logj in (1, 2, 3) for k in (2, 3, 4) if k + logj <= 6]  # n <= 16, J in {2, 4, 8}, J*n <= 64


def rand_poly(seed, n):
    rng = random.Random(seed)
    return [rng.randrange(R) for _ in range(n)]


def part_forward(a, k, ext_k, j):
    """The PART forward transform: coefficient i times g_j^i = zeta^(i mod 3) * w_ext^(j*i), then a size-n DFT with w."""
    we = P.omega_for(ext_k)
    J = 1 << (ext_k - k)
    pre = [x * pow(P.ZETA, i % 3, R) * pow(we, j * i, R) % R for i, x in enumerate(a)]
    return P.dft(pre, pow(we, J, R))


def radix2_idft(vals, w_inv):
    """The in-register network of parts_idft_kernel: bit-reversed load, radix-2 DIT stages with w_J^-(k*J/len)."""
    J = len(vals)
    logj = J.bit_length() - 1
    brev = lambda x: int(format(x, f"0{logj}b")[::-1], 2) if logj else 0
    a = [vals[brev(j)] for j in range(J)]
    tw = [pow(w_inv, m, R) for m in range(J // 2)]
    length = 2
    while length <= J:
        for b in range(0, J, length):
            for kk in range(length // 2):
                u, v = a[b + kk], a[b + kk + length // 2]
                if kk:
                    v = v * tw[kk * (J // length)] % R
                a[b + kk], a[b + kk + length // 2] = (u + v) % R, (u - v) % R
        length <<= 1
    return a


def parts_to_coeff(parts, k, ext_k, divide_by_vanishing):
    """b200zk_extended_parts_to_coeff restated: per part an inverse size-n DFT with post-scale n^-1 g_j^-i (times
    ((g_j)^n - 1)^-1), then for every i a J-point inverse DFT across the parts scaled by J^-1 zeta^(-n*t)."""
    n, J = 1 << k, 1 << (ext_k - k)
    we = P.omega_for(ext_k)
    w_inv = pow(pow(we, J, R), -1, R)
    out = []
    for j, e in enumerate(parts):
        gj = P.ZETA * pow(we, j, R) % R
        s = pow(n, -1, R)
        if divide_by_vanishing:
            s = s * pow((pow(gj, n, R) - 1) % R, -1, R) % R
        gi = pow(gj, -1, R)
        out.append([x * s % R * pow(gi, i, R) % R for i, x in enumerate(P.dft(e, w_inv))])
    wj_inv = pow(pow(we, n, R), -1, R)
    zn_inv = pow(pow(P.ZETA, n, R), -1, R)
    j_inv = pow(J, -1, R)
    res = [[0] * n for _ in range(J)]
    for i in range(n):
        col = radix2_idft([out[j][i] for j in range(J)], wj_inv)
        for t in range(J):
            res[t][i] = col[t] * j_inv % R * pow(zn_inv, t, R) % R
    return res


@pytest.mark.parametrize("k,logj", CASES)
def test_part_transform_is_the_subsampled_whole_transform(k, logj):
    n, ext_k, J = 1 << k, k + logj, 1 << logj
    a = rand_poly(10 * k + logj, n)
    whole = P.coeff_to_extended(a, k, ext_k)
    for j in range(J):
        assert part_forward(a, k, ext_k, j) == whole[j::J]


@pytest.mark.parametrize("divide", [False, True])
@pytest.mark.parametrize("k,logj", CASES)
def test_parts_to_coeff_is_extended_to_coeff_of_the_interleaved_parts(k, logj, divide):
    n, ext_k, J = 1 << k, k + logj, 1 << logj
    N = n * J
    we = P.omega_for(ext_k)
    ext = rand_poly(100 + 10 * k + logj, N)  # any values: the inverse is exact for every vector, not only low degree
    parts = [ext[j::J] for j in range(J)]
    got = parts_to_coeff(parts, k, ext_k, divide)
    if divide:  # divide_by_vanishing_poly: (zeta w_ext^idx)^n - 1 on the coset
        ext = [v * pow((pow(P.ZETA * pow(we, idx, R) % R, n, R) - 1) % R, -1, R) % R for idx, v in enumerate(ext)]
    want = P.extended_to_coeff(ext, ext_k)
    assert [c for part in got for c in part] == want


@pytest.mark.parametrize("k,logj", CASES)
def test_parts_round_trip_recovers_the_polynomial(k, logj):
    n, ext_k, J = 1 << k, k + logj, 1 << logj
    h = rand_poly(7 + k + logj, n * J)  # J*n coefficients: every part is needed
    we = P.omega_for(ext_k)
    parts = [[P.eval_poly(h, P.ZETA * pow(we, j + J * r, R) % R) for r in range(n)] for j in range(J)]
    got = parts_to_coeff(parts, k, ext_k, False)
    assert [c for part in got for c in part] == h


@pytest.mark.parametrize("J", [2, 4, 8, 16])
def test_radix2_network_is_the_inverse_dft(J):
    w = P.omega_for(J.bit_length() - 1)
    vals = rand_poly(J, J)
    w_inv = pow(w, -1, R)
    assert radix2_idft(vals, w_inv) == P.dft(vals, w_inv)


@pytest.mark.parametrize("k,logj", [(3, 1), (4, 2), (5, 3), (6, 4)])
def test_pass0_power_from_the_half_table(k, logj):
    """ext_pow in csrc/ntt.cu: w_ext^e for e < N from the top level of the universal table, which holds w_ext^m for m < N/2
    only, with w_ext^(m + N/2) = -w_ext^m; the forward exponent is j*i (< N, no reduction), the inverse one (-j*i) mod N."""
    ext_k = k + logj
    N, n, J = 1 << ext_k, 1 << k, 1 << logj
    we = P.omega_for(ext_k)
    half = [pow(we, m, R) for m in range(N // 2)]

    def ext_pow(e):
        w = half[e & (N // 2 - 1)]
        return (R - w) % R if e >= N // 2 else w

    for j in range(J):
        for i in range(n):
            assert j * i < N
            assert ext_pow(j * i) == pow(we, j * i, R)
            assert ext_pow((-j * i) & (N - 1)) == pow(we, -j * i, R)


@pytest.mark.parametrize("k,logj,seed", [(3, 1, 1), (3, 2, 2), (4, 2, 3), (3, 3, 4), (2, 2, 5)])
def test_program_on_a_part_is_a_row_subset_of_the_whole_coset(k, logj, seed):
    """part j of halo2_graph_evaluate over the extended coset (rot_scale J) == the program moved onto the part
    (ExtendedX scaled by w_ext^j) evaluated over 2^k rows with omega = w_ext^J and rot_scale 1"""
    n, ext_k, J = 1 << k, k + logj, 1 << logj
    N = n * J
    calcs, constants, rotations = random_program(seed, 60, 2, 3, 1, 2, 4, chain_bias=0.5)
    rotations = [0, -1, 1, n + 1]  # -1 wraps at row 0, +1 at row n-1, n+1 wraps for every row
    last = len(calcs) - 1
    calcs = calcs + [(C_MUL, (S_X, 0, 0), (S_INTER, last, 0), None),  # ExtendedX in every result, also as Horner factor / part
                     (C_HORNER, (S_INTER, last + 1, 0), (S_X, 0, 0), [(S_X, 0, 0), (S_INTER, 0, 0)])]
    rng = random.Random(seed)
    mk = lambda cnt: [O.fill_fr(N, rng.randrange(1 << 30)) for _ in range(cnt)]
    fx, ad, ins = mk(2), mk(3), mk(1)
    ch = O.fill_fr(2, 77)
    bgty = [O.fill_fr(1, 1000 + i)[0] for i in range(4)]
    prev = O.fill_fr(N, 4242)
    consts = O.frs_from_ints(constants)
    we = P.omega_for(ext_k)
    whole = O.graph_evaluate(calcs, consts, rotations, fx, ad, ins, ch, *bgty, O.fr_from_int(we), prev, ext_k, J)
    for j in range(J):
        sub = lambda cols: [np.ascontiguousarray(c[j::J]) for c in cols]
        pc, pk = on_part(calcs, constants, pow(we, j, R))
        got = O.graph_evaluate(pc, O.frs_from_ints(pk), rotations, sub(fx), sub(ad), sub(ins), ch, *bgty,
                               O.fr_from_int(pow(we, J, R)), np.ascontiguousarray(prev[j::J]), k, 1)
        assert np.array_equal(got, whole[j::J])


def test_moving_a_program_without_extended_x_changes_nothing():
    calcs = [(C_MUL, (S_INTER, 0, 0), (S_INTER, 0, 0), None)]
    assert on_part(calcs, [3], 5) == (calcs, [3])
