"""A GraphEvaluator program moved onto one coset part of the extended domain, for the CPU oracle.

The oracle's interpreter (oracle/halo2_quotient.c, halo2_graph_evaluate) evaluates ExtendedX as zeta * omega^row.  On part j
of the extended coset the point of row r is g_j * w^r = (zeta * w^r) * w_ext^j, so the same interpreter run over 2^k rows with
omega = w = w_ext^J and rot_scale = 1 evaluates the part once every ExtendedX operand is multiplied by the constant w_ext^j.
`on_part` does that rewrite: a new first calculation t = ExtendedX * c (c appended to the constants), every ExtendedX operand
replaced by t and every intermediate index shifted by one; the last calculation, whose value the interpreter stores, stays last.
The C++ twin is rewrite_for_part in tests/cpp/oracle_parts_ops.hpp.
"""
from quotient_programs import C_MUL, S_CONST, S_INTER, S_X


def on_part(calcs, constants, factor):
    """(calcs, constants) of the program with ExtendedX scaled by `factor` (an integer mod r)"""
    if not any(src is not None and src[0] == S_X for op, a, b, parts in calcs for src in [a, b, *(parts or [])]):
        return list(calcs), list(constants)
    c = len(constants)

    def move(src):
        if src is None:
            return None
        if src[0] == S_X:
            return (S_INTER, 0, 0)
        if src[0] == S_INTER:
            return (S_INTER, src[1] + 1, src[2])
        return src

    out = [(C_MUL, (S_X, 0, 0), (S_CONST, c, 0), None)]
    out += [(op, move(a), move(b), [move(p) for p in parts] if parts is not None else None) for op, a, b, parts in calcs]
    return out, list(constants) + [factor]
