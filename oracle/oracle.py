"""ORACLE — TEST INFRASTRUCTURE ONLY.

ctypes binding of oracle/liboracle.so (the CPU restatement of halo2curves /
halo2_proofs for the hot path; see oracle/bn254_oracle.h for the reference pins).
Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
legs may import this module.  The product (scroll-prover_b200/) never does.

Field elements travel as numpy uint64 arrays of shape (n, 4) (raw Montgomery limbs,
memcpy-compatible with halo2curves Fr/Fq); affine points as (n, 8); Jacobian as (12,).
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "liboracle.so")


def build(force: bool = False) -> str:
    srcs = ["bn254_field.c", "bn254_curve.c", "halo2_arith.c", "halo2_domain.c", "halo2_quotient.c", "dft_identity.c",
            "bn254_oracle.h", "fp_template.h"]
    stale = force or not os.path.exists(_SO) or any(
        os.path.getmtime(os.path.join(_HERE, s)) > os.path.getmtime(_SO) for s in srcs
    )
    if stale:
        subprocess.check_call(["make", "-s", "-C", _HERE, "-B", "liboracle.so"])
    return _SO


def _load():
    build()
    try:
        lib = C.CDLL(_SO)
        # -march=native binary from another host may SIGILL; probe with a trivial call in a subprocess
    except OSError:
        build(force=True)
        lib = C.CDLL(_SO)
    return lib


def _selfcheck_isa():
    """The .so is built -march=native; if it travelled from a different CPU, rebuild in place."""
    code = (
        "import ctypes,sys;l=ctypes.CDLL(%r);a=(ctypes.c_uint64*4)(1,0,0,0);"
        "r=(ctypes.c_uint64*4)();l.fr_mul(r,a,a)" % _SO
    )
    import sys

    rc = subprocess.call([sys.executable, "-c", code], stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    if rc != 0:
        build(force=True)


if os.path.exists(_SO):
    _selfcheck_isa()
lib = _load()

u64p = C.POINTER(C.c_uint64)
u8p = C.POINTER(C.c_uint8)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


R_MOD = 0x30644E72E131A029B85045B68181585D2833E84879B9709143E1F593F0000001
Q_MOD = 0x30644E72E131A029B85045B68181585D97816A916871CA8D3C208C16D87CFD47
R_MONT = 1 << 256


def limbs_to_int(a) -> int:
    a = np.asarray(a, dtype=np.uint64).reshape(-1)
    return sum(int(x) << (64 * i) for i, x in enumerate(a))


def int_to_limbs(v: int, n: int = 4) -> np.ndarray:
    return np.array([(v >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(n)], dtype=np.uint64)


def fr_from_int(v: int) -> np.ndarray:
    return int_to_limbs((v % R_MOD) * R_MONT % R_MOD)


def fr_to_int(a) -> int:
    return limbs_to_int(a) * pow(R_MONT, -1, R_MOD) % R_MOD


def fq_from_int(v: int) -> np.ndarray:
    return int_to_limbs((v % Q_MOD) * R_MONT % Q_MOD)


def fq_to_int(a) -> int:
    return limbs_to_int(a) * pow(R_MONT, -1, Q_MOD) % Q_MOD


def frs_from_ints(vs) -> np.ndarray:
    return np.stack([fr_from_int(v) for v in vs]) if len(vs) else np.zeros((0, 4), np.uint64)


def frs_to_ints(a) -> list:
    return [fr_to_int(x) for x in np.asarray(a).reshape(-1, 4)]


def const_fr(name: str) -> np.ndarray:
    return np.ctypeslib.as_array((C.c_uint64 * 4).in_dll(lib, name)).copy()


# ---------------------------------------------------------------- field wrappers
def _binop(fn):
    def f(a, b):
        a = np.ascontiguousarray(a, np.uint64)
        b = np.ascontiguousarray(b, np.uint64)
        r = np.zeros(4, np.uint64)
        fn(_p(r), _p(a), _p(b))
        return r

    return f


fr_mul = _binop(lib.fr_mul)
fr_add = _binop(lib.fr_add)
fr_sub = _binop(lib.fr_sub)
fq_mul = _binop(lib.fq_mul)
fq_add = _binop(lib.fq_add)
fq_sub = _binop(lib.fq_sub)


def fr_inv(a):
    a = np.ascontiguousarray(a, np.uint64)
    r = np.zeros(4, np.uint64)
    lib.fr_inv(_p(r), _p(a))
    return r


def fr_pow_u64(a, e: int):
    a = np.ascontiguousarray(a, np.uint64)
    r = np.zeros(4, np.uint64)
    ee = int_to_limbs(e)
    lib.fr_pow(_p(r), _p(a), _p(ee))
    return r


def fr_to_repr(a) -> bytes:
    a = np.ascontiguousarray(a, np.uint64)
    out = (C.c_uint8 * 32)()
    lib.fr_to_repr(out, _p(a))
    return bytes(out)


def fq_to_repr(a) -> bytes:
    a = np.ascontiguousarray(a, np.uint64)
    out = (C.c_uint8 * 32)()
    lib.fq_to_repr(out, _p(a))
    return bytes(out)


def fr_batch_invert(v):
    v = np.ascontiguousarray(v, np.uint64).copy()
    s = np.zeros_like(v)
    lib.fr_batch_invert(_p(v), C.c_uint64(len(v)), _p(s))
    return v


# ---------------------------------------------------------------- curve wrappers
def g1_generator() -> np.ndarray:
    r = np.zeros(8, np.uint64)
    lib.g1_generator(_p(r))
    return r


def g1_affine_is_on_curve(p) -> bool:
    p = np.ascontiguousarray(p, np.uint64)
    return bool(lib.g1_affine_is_on_curve(_p(p)))


def g1_to_affine(j) -> np.ndarray:
    j = np.ascontiguousarray(j, np.uint64)
    r = np.zeros(8, np.uint64)
    lib.g1_to_affine(_p(r), _p(j))
    return r


def g1_from_affine(a) -> np.ndarray:
    a = np.ascontiguousarray(a, np.uint64)
    r = np.zeros(12, np.uint64)
    lib.g1_from_affine(_p(r), _p(a))
    return r


def g1_add(p, q) -> np.ndarray:
    p = np.ascontiguousarray(p, np.uint64)
    q = np.ascontiguousarray(q, np.uint64)
    r = np.zeros(12, np.uint64)
    lib.g1_add(_p(r), _p(p), _p(q))
    return r


def g1_add_mixed(p, q) -> np.ndarray:
    p = np.ascontiguousarray(p, np.uint64)
    q = np.ascontiguousarray(q, np.uint64)
    r = np.zeros(12, np.uint64)
    lib.g1_add_mixed(_p(r), _p(p), _p(q))
    return r


def g1_double(p) -> np.ndarray:
    p = np.ascontiguousarray(p, np.uint64)
    r = np.zeros(12, np.uint64)
    lib.g1_double(_p(r), _p(p))
    return r


def g1_mul(p, s) -> np.ndarray:
    p = np.ascontiguousarray(p, np.uint64)
    s = np.ascontiguousarray(s, np.uint64)
    r = np.zeros(12, np.uint64)
    lib.g1_mul(_p(r), _p(p), _p(s))
    return r


def g1_compress(a) -> bytes:
    a = np.ascontiguousarray(a, np.uint64)
    out = (C.c_uint8 * 32)()
    lib.g1_affine_to_compressed(out, _p(a))
    return bytes(out)


def g1_decompress(b: bytes):
    buf = (C.c_uint8 * 32).from_buffer_copy(b)
    r = np.zeros(8, np.uint64)
    ok = lib.g1_affine_from_compressed(_p(r), buf)
    return r if ok else None


def g1_batch_normalize(js) -> np.ndarray:
    js = np.ascontiguousarray(js, np.uint64).reshape(-1, 12)
    out = np.zeros((len(js), 8), np.uint64)
    lib.g1_batch_normalize(_p(out), _p(js), C.c_uint64(len(js)))
    return out


# ---------------------------------------------------------------- halo2_proofs::arithmetic
def multiexp_serial(coeffs, bases) -> np.ndarray:
    coeffs = np.ascontiguousarray(coeffs, np.uint64).reshape(-1, 4)
    bases = np.ascontiguousarray(bases, np.uint64).reshape(-1, 8)
    assert len(coeffs) == len(bases)
    acc = np.zeros(12, np.uint64)
    lib.g1_identity(_p(acc))
    lib.halo2_multiexp_serial(_p(coeffs), _p(bases), C.c_uint64(len(coeffs)), _p(acc))
    return acc


def best_multiexp(coeffs, bases, threads: int = 1) -> np.ndarray:
    coeffs = np.ascontiguousarray(coeffs, np.uint64).reshape(-1, 4)
    bases = np.ascontiguousarray(bases, np.uint64).reshape(-1, 8)
    assert len(coeffs) == len(bases)  # assert_eq!(coeffs.len(), bases.len())
    out = np.zeros(12, np.uint64)
    lib.halo2_best_multiexp(_p(coeffs), _p(bases), C.c_uint64(len(coeffs)), C.c_int(threads), _p(out))
    return out


def best_fft(a, omega, log_n: int, threads: int = 1) -> np.ndarray:
    a = np.ascontiguousarray(a, np.uint64).reshape(-1, 4).copy()
    assert len(a) == 1 << log_n  # assert_eq!(a.len(), 1 << log_n)
    omega = np.ascontiguousarray(omega, np.uint64)
    lib.halo2_best_fft(_p(a), _p(omega), C.c_uint32(log_n), C.c_int(threads))
    return a


def best_fft_g1(a, omega, log_n: int, threads: int = 1) -> np.ndarray:
    a = np.ascontiguousarray(a, np.uint64).reshape(-1, 12).copy()
    assert len(a) == 1 << log_n
    omega = np.ascontiguousarray(omega, np.uint64)
    lib.halo2_best_fft_g1(_p(a), _p(omega), C.c_uint32(log_n), C.c_int(threads))
    return a


def eval_polynomial(poly, point) -> np.ndarray:
    poly = np.ascontiguousarray(poly, np.uint64).reshape(-1, 4)
    point = np.ascontiguousarray(point, np.uint64)
    r = np.zeros(4, np.uint64)
    lib.halo2_eval_polynomial(_p(r), _p(poly), C.c_uint64(len(poly)), _p(point))
    return r


def kate_division(a, b) -> np.ndarray:
    a = np.ascontiguousarray(a, np.uint64).reshape(-1, 4)
    b = np.ascontiguousarray(b, np.uint64)
    q = np.zeros((max(len(a) - 1, 0), 4), np.uint64)
    lib.halo2_kate_division(_p(q), _p(a), C.c_uint64(len(a)), _p(b))
    return q


def compute_inner_product(a, b) -> np.ndarray:
    a = np.ascontiguousarray(a, np.uint64).reshape(-1, 4)
    b = np.ascontiguousarray(b, np.uint64).reshape(-1, 4)
    r = np.zeros(4, np.uint64)
    lib.halo2_compute_inner_product(_p(r), _p(a), _p(b), C.c_uint64(len(a)))
    return r


# ---------------------------------------------------------------- EvaluationDomain
class _DomainStruct(C.Structure):
    _fields_ = [
        ("n", C.c_uint64),
        ("k", C.c_uint32),
        ("extended_k", C.c_uint32),
        ("quotient_poly_degree", C.c_uint32),
        ("omega", C.c_uint64 * 4),
        ("omega_inv", C.c_uint64 * 4),
        ("extended_omega", C.c_uint64 * 4),
        ("extended_omega_inv", C.c_uint64 * 4),
        ("g_coset", C.c_uint64 * 4),
        ("g_coset_inv", C.c_uint64 * 4),
        ("ifft_divisor", C.c_uint64 * 4),
        ("extended_ifft_divisor", C.c_uint64 * 4),
        ("barycentric_weight", C.c_uint64 * 4),
        ("n_t_evaluations", C.c_uint32),
        ("t_evaluations", (C.c_uint64 * 4) * 64),
    ]


class EvaluationDomain:
    """halo2_proofs::poly::EvaluationDomain::new(j, k)"""

    def __init__(self, j: int, k: int):
        self._s = _DomainStruct()
        rc = lib.halo2_domain_new(C.byref(self._s), C.c_uint32(j), C.c_uint32(k))
        if rc != 0:
            raise ValueError(f"EvaluationDomain::new({j},{k}) failed rc={rc}")
        self.k, self.extended_k, self.n = self._s.k, self._s.extended_k, self._s.n
        self.quotient_poly_degree = self._s.quotient_poly_degree
        for f in ("omega", "omega_inv", "extended_omega", "extended_omega_inv", "g_coset", "g_coset_inv",
                  "ifft_divisor", "extended_ifft_divisor", "barycentric_weight"):
            setattr(self, f, np.array(list(getattr(self._s, f)), dtype=np.uint64))
        self.t_evaluations = np.array([list(self._s.t_evaluations[i]) for i in range(self._s.n_t_evaluations)], dtype=np.uint64)

    def lagrange_to_coeff(self, a, threads: int = 1):
        a = np.ascontiguousarray(a, np.uint64).reshape(-1, 4).copy()
        assert len(a) == self.n
        lib.halo2_lagrange_to_coeff(C.byref(self._s), _p(a), C.c_int(threads))
        return a

    def coeff_to_extended(self, a, threads: int = 1):
        a = np.ascontiguousarray(a, np.uint64).reshape(-1, 4)
        assert len(a) == self.n
        out = np.zeros((1 << self.extended_k, 4), np.uint64)
        lib.halo2_coeff_to_extended(C.byref(self._s), _p(a), _p(out), C.c_int(threads))
        return out

    def extended_to_coeff(self, a, threads: int = 1):
        a = np.ascontiguousarray(a, np.uint64).reshape(-1, 4).copy()
        assert len(a) == 1 << self.extended_k
        lib.halo2_extended_to_coeff(C.byref(self._s), _p(a), C.c_int(threads))
        return a[: self.n * self.quotient_poly_degree]

    def distribute_powers_zeta(self, a, into_coset: bool):
        a = np.ascontiguousarray(a, np.uint64).reshape(-1, 4).copy()
        lib.halo2_distribute_powers_zeta(C.byref(self._s), _p(a), C.c_uint64(len(a)), C.c_int(1 if into_coset else 0))
        return a


# ---------------------------------------------------------------- ParamsKZG
def params_setup(k: int, tau, threads: int = 8, lagrange: bool = True):
    tau = np.ascontiguousarray(tau, np.uint64)
    n = 1 << k
    g = np.zeros((n, 8), np.uint64)
    gl = np.zeros((n, 8), np.uint64) if lagrange else None
    lib.halo2_params_setup(C.c_uint32(k), _p(tau), _p(g), _p(gl) if lagrange else None, C.c_int(threads))
    return g, gl


def g_to_lagrange(g, k: int, threads: int = 8):
    g = np.ascontiguousarray(g, np.uint64).reshape(-1, 8)
    out = np.zeros_like(g)
    lib.halo2_g_to_lagrange(_p(g), _p(out), C.c_uint32(k), C.c_int(threads))
    return out


def commit(bases, poly, threads: int = 1):
    poly = np.ascontiguousarray(poly, np.uint64).reshape(-1, 4)
    return best_multiexp(poly, np.asarray(bases)[: len(poly)], threads)


# ---------------------------------------------------------------- test vectors
def fill_fr(n: int, seed: int, witness_like: bool = False) -> np.ndarray:
    out = np.zeros((n, 4), np.uint64)
    lib.oracle_fill_fr(_p(out), C.c_uint64(n), C.c_uint64(seed), C.c_int(1 if witness_like else 0))
    return out


def fill_points(n: int, seed: int, threads: int = 8) -> np.ndarray:
    out = np.zeros((n, 8), np.uint64)
    lib.oracle_fill_points(_p(out), C.c_uint64(n), C.c_uint64(seed), C.c_int(threads))
    return out


def fill_points_chain(n: int, seed: int, threads: int = 8) -> np.ndarray:
    """distinct valid points P_0 + i*D, cheap to generate at 2^24+ (CPU-baseline inputs only)"""
    out = np.zeros((n, 8), np.uint64)
    lib.oracle_fill_points_chain(_p(out), C.c_uint64(n), C.c_uint64(seed), C.c_int(threads))
    return out


# ---- test helper, not a restatement of the reference (dft_identity.c)
def dft_eval_rhs(a, c, omega, r, N: int, threads: int | None = None) -> np.ndarray:
    """(r^N - 1) * sum_i a_i c^i / (omega^i r - 1): equals eval_polynomial(y, r) for the transform
    y_j = sum_i a_i c^i omega^(ij), j < N.  O(len(a)) on all host threads; raises if omega^N != 1 or r^N == 1."""
    a = np.ascontiguousarray(a, np.uint64).reshape(-1, 4)
    c, omega, r = (np.ascontiguousarray(x, np.uint64).reshape(4) for x in (c, omega, r))
    out = np.zeros(4, np.uint64)
    rc = lib.oracle_dft_eval_rhs(_p(out), _p(a), C.c_uint64(len(a)), _p(c), _p(omega), _p(r), C.c_uint64(N),
                                 C.c_int(threads or os.cpu_count() or 8))
    if rc != 0:
        raise ValueError({-1: "omega^N != 1", -2: "r^N == 1"}[rc])
    return out


def eval_polynomial_mt(poly, point, threads: int | None = None) -> np.ndarray:
    """eval_polynomial(poly, point) with the Horner loop split over all host threads (same value)."""
    poly = np.ascontiguousarray(poly, np.uint64).reshape(-1, 4)
    point = np.ascontiguousarray(point, np.uint64).reshape(4)
    r = np.zeros(4, np.uint64)
    lib.oracle_eval_polynomial_mt(_p(r), _p(poly), C.c_uint64(len(poly)), _p(point), C.c_int(threads or os.cpu_count() or 8))
    return r


# ---- quotient construction (halo2_quotient.c) ------------------------------------------------------------------
# program = (calcs, constants, rotations); calcs: list of (op, a, b, parts) with sources (kind, index, rotation)
SRC = {n: i for i, n in enumerate(["constant", "intermediate", "fixed", "advice", "instance", "challenge", "beta", "gamma",
                                   "theta", "y", "previous", "x"])}
CALC = {n: i for i, n in enumerate(["add", "sub", "mul", "square", "double", "negate", "horner", "store"])}


class _ValueSource(C.Structure):
    _fields_ = [("kind", C.c_uint32), ("index", C.c_uint32), ("rotation", C.c_uint32)]


class _Calculation(C.Structure):
    _fields_ = [("op", C.c_uint32), ("a", _ValueSource), ("b", _ValueSource), ("parts_offset", C.c_uint32),
                ("parts_len", C.c_uint32)]


def pack_program(calcs, vs_type=_ValueSource, calc_type=_Calculation):
    parts = []
    arr = (calc_type * max(1, len(calcs)))()
    for i, (op, a, b, ps) in enumerate(calcs):
        arr[i].op = op
        arr[i].a = vs_type(*a)
        arr[i].b = vs_type(*(b if b is not None else (0, 0, 0)))
        arr[i].parts_offset = len(parts)
        arr[i].parts_len = len(ps or [])
        parts.extend(ps or [])
    parr = (vs_type * max(1, len(parts)))(*[vs_type(*q) for q in parts])
    return arr, parr, len(parts)


def _colptrs(cols):
    cols = [np.ascontiguousarray(c, dtype=np.uint64) for c in cols]
    arr = (C.c_void_p * max(1, len(cols)))(*[c.ctypes.data for c in cols])
    return arr, cols


def graph_evaluate(calcs, constants, rotations, fixed, advice, instance, challenges, beta, gamma, theta, y,
                   extended_omega, values, log_size: int, rot_scale: int) -> np.ndarray:
    arr, parr, _ = pack_program(calcs)
    consts = np.ascontiguousarray(np.asarray(constants, dtype=np.uint64).reshape(-1, 4))
    rots = np.ascontiguousarray(np.asarray(rotations, dtype=np.int32))
    fp, _f = _colptrs(fixed)
    ap, _a = _colptrs(advice)
    ip, _i = _colptrs(instance)
    ch = np.ascontiguousarray(np.asarray(challenges, dtype=np.uint64).reshape(-1, 4))
    out = np.ascontiguousarray(values, dtype=np.uint64).copy()
    sc = [np.ascontiguousarray(v, dtype=np.uint64) for v in (beta, gamma, theta, y)]
    eo = None if extended_omega is None else np.ascontiguousarray(extended_omega, dtype=np.uint64)
    rc = lib.halo2_graph_evaluate(arr, len(calcs), parr, _p(consts), _p(rots), len(rots), fp, ap, ip, _p(ch), _p(sc[0]),
                                  _p(sc[1]), _p(sc[2]), _p(sc[3]), None if eo is None else _p(eo), _p(out), log_size,
                                  rot_scale)
    assert rc == 0
    return out


def prefix_scan(op: int, a, init) -> np.ndarray:
    a = np.ascontiguousarray(a, dtype=np.uint64)
    out = np.zeros_like(a)
    lib.halo2_prefix_scan(op, _p(a), C.c_uint64(len(a)), _p(np.ascontiguousarray(init, dtype=np.uint64)), _p(out))
    return out


def permutation_product(values, sigma, beta, gamma, delta_omega_start, delta, omega, k: int, z_init) -> np.ndarray:
    vp, _v = _colptrs(values)
    sp, _s = _colptrs(sigma)
    out = np.zeros((1 << k, 4), np.uint64)
    sc = [np.ascontiguousarray(v, dtype=np.uint64) for v in (beta, gamma, delta_omega_start, delta, omega, z_init)]
    rc = lib.halo2_permutation_product(vp, sp, len(values), _p(sc[0]), _p(sc[1]), _p(sc[2]), _p(sc[3]), _p(sc[4]), k,
                                       _p(sc[5]), _p(out))
    assert rc == 0
    return out


def logup_running_sum(inputs, table, m, beta, k: int, phi_init) -> np.ndarray:
    ip, _i = _colptrs(inputs)
    out = np.zeros((1 << k, 4), np.uint64)
    t = np.ascontiguousarray(table, dtype=np.uint64)
    mm = np.ascontiguousarray(m, dtype=np.uint64)
    sc = [np.ascontiguousarray(v, dtype=np.uint64) for v in (beta, phi_init)]
    rc = lib.halo2_logup_running_sum(ip, len(inputs), _p(t), _p(mm), _p(sc[0]), k, _p(sc[1]), _p(out))
    assert rc == 0
    return out


def permutation_h_terms(z_cosets, chunk_len: int, value_cosets, sigma_cosets, l0, l_last, l_active_row, beta, gamma, y, delta,
                        extended_omega, last_rotation: int, values, log_size: int, rot_scale: int) -> np.ndarray:
    zp, _z = _colptrs(z_cosets)
    vp, _v = _colptrs(value_cosets)
    sp, _s = _colptrs(sigma_cosets)
    ls = [np.ascontiguousarray(c, dtype=np.uint64) for c in (l0, l_last, l_active_row)]
    sc = [np.ascontiguousarray(c, dtype=np.uint64) for c in (beta, gamma, y, delta, extended_omega)]
    out = np.ascontiguousarray(values, dtype=np.uint64).copy()
    rc = lib.halo2_permutation_h_terms(zp, len(z_cosets), chunk_len, vp, sp, len(value_cosets), _p(ls[0]), _p(ls[1]), _p(ls[2]),
                                       _p(sc[0]), _p(sc[1]), _p(sc[2]), _p(sc[3]), _p(sc[4]), C.c_int32(last_rotation), _p(out),
                                       log_size, C.c_int32(rot_scale))
    assert rc == 0
    return out


def logup_h_terms(input_cosets, table_coset, m_coset, phi_coset, l0, l_last, l_active_row, beta, y, values, log_size: int,
                  rot_scale: int) -> np.ndarray:
    ip, _i = _colptrs(input_cosets)
    cs = [np.ascontiguousarray(c, dtype=np.uint64) for c in (table_coset, m_coset, phi_coset, l0, l_last, l_active_row, beta, y)]
    out = np.ascontiguousarray(values, dtype=np.uint64).copy()
    rc = lib.halo2_logup_h_terms(ip, len(input_cosets), *[_p(c) for c in cs], _p(out), log_size, C.c_int32(rot_scale))
    assert rc == 0
    return out
