"""The quotient by coset parts on the device (csrc/ntt.cu PART kernels, csrc/quotient.cu parts_idft_kernel and
b200zk_graph_evaluate_part), checked bit-exactly against the oracle's whole-coset transforms and against the device's
whole-coset evaluate_h chain.

With n = 2^k and J = 2^(extended_k - k), part j of the extended coset is zeta * w_ext^j * <w_ext^J>: rows j, j + J, j + 2J, ...
of the whole coset.
"""
import random

import numpy as np
import pytest

from h_terms_programs import logup_terms_program, permutation_terms_program
from oracle import oracle as O
from quotient_programs import C_MUL, R_MOD, S_ADVICE, S_CONST, random_program

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def one_stream(ctx):
    """Device-resident outputs are asynchronous on the context stream: put the library on torch's current stream so that
    clones, kernels and .cpu() copies are ordered on one stream."""
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


def domains(zk, ctx, k, logj):
    """EvaluationDomain(J + 1, k): extended_k = k + log2 J and quotient_poly_degree = J, so that the oracle's extended_to_coeff
    keeps all J*n coefficients."""
    J = 1 << logj
    d, do = zk.EvaluationDomain(ctx, J + 1, k), O.EvaluationDomain(J + 1, k)
    assert d.extended_k == do.extended_k == k + logj and d.n_parts == J
    return d, do


def scale_by(a, s, k):
    """a * s for a constant s, by the oracle's interpreter (one Mul calculation)"""
    z = O.fr_from_int(0)
    return O.graph_evaluate([(C_MUL, (S_ADVICE, 0, 0), (S_CONST, 0, 0), None)], np.asarray([s]), [0], [], [a], [],
                            np.zeros((0, 4), np.uint64), z, z, z, z, None, np.zeros_like(a), k, 1)


@pytest.mark.parametrize("logj", [1, 2, 3])
@pytest.mark.parametrize("k", [3, 10, 16, 20])
def test_parts_match_the_oracle(ctx, zk, k, logj):
    J, n = 1 << logj, 1 << k
    d, do = domains(zk, ctx, k, logj)
    a = O.fill_fr(n, 31 * k + logj)
    whole = do.coeff_to_extended(a, threads=8)
    parts_host, parts_dev = [], []
    for j in range(J):
        want = whole[j::J]
        got = d.coeff_to_extended_part(a, j)                  # host in, host out
        assert np.array_equal(got, want), f"part {j} (host)"
        out = dev(np.zeros((n, 4), np.uint64))
        d.coeff_to_extended_part(dev(a), j, out=out)          # device in, device out
        assert np.array_equal(host(out), want), f"part {j} (device)"
        inplace = dev(a)
        d.coeff_to_extended_part(inplace, j, out=inplace)     # in place
        assert np.array_equal(host(inplace), want), f"part {j} (in place)"
        parts_host.append(got)
        parts_dev.append(inplace)
    # parts -> coefficients: extended_to_coeff of the interleaved coset, all J*n coefficients
    coeffs = do.extended_to_coeff(whole, threads=8)
    assert len(coeffs) == J * n
    d.extended_parts_to_coeff(parts_dev)
    assert np.array_equal(np.concatenate([host(p) for p in parts_dev]), coeffs)
    # with the division by X^n - 1 (the constant t_evaluations[j] on part j), host memory, one part left on the device
    divided = np.concatenate([scale_by(np.ascontiguousarray(whole[j::J]), do.t_evaluations[j], k) for j in range(J)])
    inter = np.empty_like(whole)
    for j in range(J):
        inter[j::J] = divided[j * n:(j + 1) * n]
    want_div = do.extended_to_coeff(inter, threads=8)
    mixed = [p.copy() for p in parts_host]
    mixed[0] = dev(mixed[0])
    d.extended_parts_to_coeff(mixed, divide_by_vanishing=True)
    got_div = np.concatenate([host(mixed[0])] + mixed[1:])
    assert np.array_equal(got_div, want_div)


def _columns(seed, n, count):
    rng = random.Random(seed)
    return [O.fill_fr(n, rng.randrange(1 << 30)) for _ in range(count)]


def _programs(n_blind=4):
    gate = random_program(17, 150, 2, 3, 1, 2, 4, chain_bias=0.5)
    perm = permutation_terms_program(2, 2, 3, -(n_blind + 1))
    look = logup_terms_program(2)
    return gate, perm, look


def _tables(cols):
    """column tables of the three programs, drawn from one pool of 9 columns:
    gate: fixed [c4 c5], advice [c0 c1 c2], instance [c3]
    perm: advice [z0 z1 v0 v1 v2] = [c6 c7 c0 c1 c2], fixed [s0 s1 s2 l0 l_last l_active] = [c3 c4 c5 c6 c7 c8]
    look: advice [f0 f1 t m phi] = [c1 c2 c3 c4 c5], fixed [l0 l_last l_active] = [c6 c7 c8]"""
    c = cols
    return [
        dict(fixed=[c[4], c[5]], advice=[c[0], c[1], c[2]], instance=[c[3]]),
        dict(fixed=[c[3], c[4], c[5], c[6], c[7], c[8]], advice=[c[6], c[7], c[0], c[1], c[2]], instance=[]),
        dict(fixed=[c[6], c[7], c[8]], advice=[c[1], c[2], c[3], c[4], c[5]], instance=[]),
    ]


def test_graph_evaluate_part_matches_the_subsampled_whole_coset(ctx, zk):
    k, logj = 10, 2
    J, n = 1 << logj, 1 << k
    d = zk.EvaluationDomain(ctx, J + 1, k)
    ext = [dev(c) for c in _columns(5, n * J, 9)]
    ch = O.fill_fr(2, 77)
    beta, gamma, theta, y = [O.fill_fr(1, 1000 + i)[0] for i in range(4)]
    prev = O.fill_fr(n * J, 4242)
    for (calcs, constants, rotations), tab in zip(_programs(), _tables(ext)):
        g = ctx.graph(calcs, O.frs_from_ints(constants), rotations)
        whole = dev(prev)
        g.evaluate(whole, d.extended_k, J, challenges=ch, beta=beta, gamma=gamma, theta=theta, y=y,
                   extended_omega=d.extended_omega, **tab)
        want = host(whole)
        for j in range(J):
            part = dev(np.ascontiguousarray(prev[j::J]))
            sub = {key: [c[j::J].contiguous() for c in cols] for key, cols in tab.items()}
            g.evaluate_part(part, k, d.extended_k, j, challenges=ch, beta=beta, gamma=gamma, theta=theta, y=y,
                            extended_omega=d.extended_omega, **sub)
            assert np.array_equal(host(part), want[j::J]), f"part {j}"
        g.release()


def test_full_chain_by_parts_equals_the_whole_coset_chain(ctx, zk):
    """evaluate_h at 2^22 rows, J = 4: every column's part from its coefficients, the gate, permutation and lookup programs
    folded with y, then the parts to coefficients with the vanishing division -- against coeff_to_extended, the same programs
    over the whole coset, the division and extended_to_coeff.  Every one of the 2^24 coefficients must be equal."""
    import torch

    k, logj = 22, 2
    J, n = 1 << logj, 1 << k
    d = zk.EvaluationDomain(ctx, J + 1, k)
    coeffs = [dev(c) for c in _columns(9, n, 9)]
    ch = O.fill_fr(2, 78)
    beta, gamma, theta, y = [O.fill_fr(1, 2000 + i)[0] for i in range(4)]
    progs = [ctx.graph(c, O.frs_from_ints(k_), r) for c, k_, r in _programs()]
    args = dict(challenges=ch, beta=beta, gamma=gamma, theta=theta, y=y, extended_omega=d.extended_omega)

    ext = [d.coeff_to_extended(c) for c in coeffs]
    whole = torch.zeros((n * J, 4), dtype=torch.int64, device="cuda")
    for g, tab in zip(progs, _tables(ext)):
        g.evaluate(whole, d.extended_k, J, **tab, **args)
    del ext
    tinv = [pow((pow(O.fr_to_int(d.g_coset), n, R_MOD) * pow(O.fr_to_int(d.extended_omega), n * j, R_MOD) - 1) % R_MOD, -1, R_MOD)
            for j in range(J)]
    tcol = dev(O.frs_from_ints(tinv)).repeat(n, 1)
    ctx.poly_mul(whole, tcol, out=whole)
    del tcol
    ctx.best_fft(whole, d.extended_omega_inv, d.extended_k, inverse_scale=True, coset_mode=zk.COSET_POST)
    want = host(whole)
    del whole

    parts = []
    for j in range(J):
        cols = [d.coeff_to_extended_part(c, j) for c in coeffs]
        vals = torch.zeros((n, 4), dtype=torch.int64, device="cuda")
        for g, tab in zip(progs, _tables(cols)):
            g.evaluate_part(vals, k, d.extended_k, j, **tab, **args)
        parts.append(vals)
        del cols
    d.extended_parts_to_coeff(parts, divide_by_vanishing=True)
    got = np.concatenate([host(p) for p in parts])
    assert np.array_equal(got, want)
    for g in progs:
        g.release()


def test_part_argument_errors(ctx, zk):
    k = 4
    n = 1 << k
    d = zk.EvaluationDomain(ctx, 5, k)  # J = 4
    a = O.fill_fr(n, 3)
    with pytest.raises(zk.B200zkError) as ei:
        d.coeff_to_extended_part(a, 4)
    assert ei.value.code == zk.E_INVALID
    big = zk.EvaluationDomain(ctx, 33, k)  # J = 32
    assert big.n_parts == 32
    with pytest.raises(zk.B200zkError) as ei:
        big.coeff_to_extended_part(a, 0)
    assert ei.value.code == zk.E_UNSUPPORTED
    with pytest.raises(zk.B200zkError) as ei:
        big.extended_parts_to_coeff([a.copy() for _ in range(32)])
    assert ei.value.code == zk.E_UNSUPPORTED
    g = ctx.graph([(C_MUL, (S_ADVICE, 0, 0), (S_CONST, 0, 0), None)], O.frs_from_ints([3]), [0])
    vals = dev(np.zeros((n, 4), np.uint64))
    with pytest.raises(zk.B200zkError) as ei:  # part >= J
        g.evaluate_part(vals, k, k + 2, 4, advice=[dev(a)], extended_omega=d.extended_omega)
    assert ei.value.code == zk.E_INVALID
    with pytest.raises(zk.B200zkError) as ei:  # J = 32
        g.evaluate_part(vals, k, k + 5, 0, advice=[dev(a)], extended_omega=big.extended_omega)
    assert ei.value.code == zk.E_UNSUPPORTED
    with pytest.raises(zk.B200zkError) as ei:  # columns must be device memory
        g.evaluate_part(vals, k, k + 2, 1, advice=[a], extended_omega=d.extended_omega)
    assert ei.value.code == zk.E_INVALID
    g.release()
