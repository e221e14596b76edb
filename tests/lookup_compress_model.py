"""Random mv-lookup tuples for Ops::compress_expressions (scroll-prover_b200/plonk_b200.hpp) and the big-integer model of its rule:
out[r] = fold(acc * theta + e(r)) over the tuple, e read from the Lagrange values at (r + rotation) mod 2^k, challenges by index.

An expression is a nested tuple: ("const", v) | ("fixed" | "advice" | "instance", column, rotation) | ("challenge", i) | ("neg", e) |
("sum", a, b) | ("sub", a, b) (upstream's a + (-b)) | ("mul", a, b) | ("scaled", e, v), with v an integer < R_MOD.  write_case
writes the case file of tests/cpp/test_lookup_compress.cpp; read_host_output parses what its host mode writes back."""
import random

import numpy as np

from lookup_model import R_MOD, mont

R_INV = pow(1 << 256, -1, R_MOD)
(K_CONSTANT, K_FIXED, K_ADVICE, K_INSTANCE, K_NEGATED, K_SUM, K_PRODUCT, K_SCALED, K_CHALLENGE) = range(9)  # Expr::Kind
QUERY = {"fixed": K_FIXED, "advice": K_ADVICE, "instance": K_INSTANCE}


def random_expr(rng: random.Random, depth: int, shape):
    """shape = (n_fixed, n_advice, n_instance, n_challenges); rotations -3 .. 3"""
    nf, na, ni, nc = shape
    if depth == 0 or rng.random() < 0.3:
        leaves = ["const"] + ["fixed"] * (nf > 0) * 2 + ["advice"] * (na > 0) * 2 + ["instance"] * (ni > 0) + ["challenge"] * (nc > 0)
        kind = rng.choice(leaves)
        if kind == "const":
            return ("const", rng.choice([0, 1, 2, R_MOD - 1, rng.randrange(R_MOD)]))
        if kind == "challenge":
            return ("challenge", rng.randrange(nc))
        return (kind, rng.randrange({"fixed": nf, "advice": na, "instance": ni}[kind]), rng.randint(-3, 3))
    op = rng.choice(["neg", "sum", "sub", "mul", "mul", "scaled"])
    if op == "neg":
        return ("neg", random_expr(rng, depth - 1, shape))
    if op == "scaled":
        return ("scaled", random_expr(rng, depth - 1, shape), rng.randrange(R_MOD))
    return (op, random_expr(rng, depth - 1, shape), random_expr(rng, depth - 1, shape))


def every_kind(shape):
    """one tuple that holds every expression kind, a SUB and the extreme rotations"""
    return [("sub", ("mul", ("fixed", 0, -3), ("advice", 0, 3)), ("scaled", ("instance", 0, 1), 5)),
            ("sum", ("neg", ("challenge", shape[3] - 1)), ("const", 7)),
            ("mul", ("advice", shape[1] - 1, -1), ("sum", ("fixed", shape[0] - 1, 2), ("instance", shape[2] - 1, -2)))]


def encode(e) -> bytes:
    kind = e[0]
    u32 = lambda v: np.array([v], np.uint32).tobytes()
    fr = lambda v: mont(v).tobytes()
    if kind == "const":
        return u32(K_CONSTANT) + fr(e[1])
    if kind in QUERY:
        return u32(QUERY[kind]) + u32(e[1]) + np.array([e[2]], np.int32).tobytes()
    if kind == "challenge":
        return u32(K_CHALLENGE) + u32(e[1])
    if kind == "neg":
        return u32(K_NEGATED) + encode(e[1])
    if kind == "sub":
        return u32(K_SUM) + encode(e[1]) + u32(K_NEGATED) + encode(e[2])
    if kind == "scaled":
        return u32(K_SCALED) + encode(e[1]) + fr(e[2])
    return u32(K_SUM if kind == "sum" else K_PRODUCT) + encode(e[1]) + encode(e[2])


def to_ints(col) -> list:
    """canonical integers of Montgomery limbs, (n, 4) uint64"""
    col = np.asarray(col, np.uint64)
    return [(int(a) | int(b) << 64 | int(c) << 128 | int(d) << 192) * R_INV % R_MOD for a, b, c, d in col]


def evaluate(e, cols, challenges, n):
    """the expression on every row, as canonical integers; cols = {"fixed": [[int]], ...}"""
    kind = e[0]
    if kind == "const":
        return [e[1]] * n
    if kind in QUERY:
        c, rot = cols[kind][e[1]], e[2]
        return [c[(r + rot) % n] for r in range(n)]
    if kind == "challenge":
        return [challenges[e[1]]] * n
    if kind == "neg":
        return [(-v) % R_MOD for v in evaluate(e[1], cols, challenges, n)]
    if kind == "scaled":
        return [v * e[2] % R_MOD for v in evaluate(e[1], cols, challenges, n)]
    a, b = evaluate(e[1], cols, challenges, n), evaluate(e[2], cols, challenges, n)
    if kind == "sum":
        return [(x + y) % R_MOD for x, y in zip(a, b)]
    if kind == "sub":
        return [(x - y) % R_MOD for x, y in zip(a, b)]
    return [x * y % R_MOD for x, y in zip(a, b)]


def fold_model(tuple_, cols, challenges, theta, n):
    """Montgomery limbs (n, 4) of fold(acc * theta + e) over the tuple"""
    acc = [0] * n
    for e in tuple_:
        acc = [(a * theta + v) % R_MOD for a, v in zip(acc, evaluate(e, cols, challenges, n))]
    return np.stack([mont(v) for v in acc])


def write_case(path, k, theta, challenges, fixed, advice, instance, sides):
    """theta, challenges: canonical integers; columns: Montgomery limbs (2^k, 4); sides: lists of expressions"""
    with open(path, "wb") as f:
        f.write(np.array([k, len(fixed), len(advice), len(instance), len(challenges), len(sides)], np.uint32).tobytes())
        for v in [theta] + list(challenges):
            f.write(mont(v).tobytes())
        for col in list(fixed) + list(advice) + list(instance):
            assert col.shape == (1 << k, 4)
            f.write(np.ascontiguousarray(col, np.uint64).tobytes())
        for side in sides:
            f.write(np.array([len(side)], np.uint32).tobytes())
            for e in side:
                f.write(encode(e))


def read_host_output(path, k, n_sides):
    """(columns, programs); a program is (calcs, constants, rotations) in oracle.graph_evaluate's form"""
    raw = open(path, "rb").read()
    n = 1 << k
    cols = np.frombuffer(raw[:32 * n * n_sides], np.uint64).reshape(n_sides, n, 4)
    pos, programs = 32 * n * n_sides, []

    def take(width, dtype):
        nonlocal pos
        cnt = int(np.frombuffer(raw[pos:pos + 4], np.uint32)[0])
        a = np.frombuffer(raw[pos + 4:pos + 4 + cnt * width], dtype)
        pos += 4 + cnt * width
        return a, cnt

    for _ in range(n_sides):
        c, nc = take(36, np.uint32)
        p, npart = take(12, np.uint32)
        consts, ncon = take(32, np.uint64)
        rots, _ = take(4, np.int32)
        c, p = c.reshape(nc, 9), p.reshape(npart, 3)
        calcs = [(int(x[0]), tuple(int(v) for v in x[1:4]), tuple(int(v) for v in x[4:7]),
                  [tuple(int(v) for v in q) for q in p[x[7]:x[7] + x[8]]] if x[8] else None) for x in c]
        programs.append((calcs, consts.reshape(ncon, 4).copy(), [int(r) for r in rots]))
    assert pos == len(raw)
    return cols, programs
