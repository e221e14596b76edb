/*
 * ORACLE — TEST INFRASTRUCTURE ONLY (see oracle/README.md).
 *
 * CPU restatement of the polynomial-arithmetic hot path underneath
 * scroll-prover: halo2curves::bn256::{Fr,Fq,G1Affine,G1} and
 * halo2_proofs::{arithmetic, poly::domain, poly::kzg::commitment}.
 * Upstream sources are un-vendored git dependencies (pins:
 * /root/reference/Cargo.lock:1886-1888 halo2_proofs 1.1.0 @ scroll-tech/halo2 e5ddf67,
 * /root/reference/Cargo.lock:1911-1913 halo2curves 0.1.0 @ 112f5b9); this file
 * restates their published algorithms (SURVEY.md Appendix A).
 *
 * PARITY STATUS: constants, encodings and curve equation are pinned by the
 * reference's fixtures (tests/test_oracle_fixtures.py); direct MSM/NTT
 * input->output pairs are NOT shipped by the reference => "parity unpinned" at
 * that level; those are cross-checked against an independent pure-Python
 * big-integer model (oracle/pyref.py) and algebraic identities instead.
 */
#ifndef BN254_ORACLE_H
#define BN254_ORACLE_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct { uint64_t l[4]; } fr_t; /* BN254 scalar field, Montgomery limbs */
typedef struct { uint64_t l[4]; } fq_t; /* BN254 base field,   Montgomery limbs */

typedef struct { fq_t x, y; } g1_affine_t;   /* identity = (0,0); 64 B == params RawBytes */
typedef struct { fq_t x, y, z; } g1_t;       /* Jacobian, identity z == 0; 96 B */

/* ---- field (bn254_field.c) ---- */
extern const fr_t fr_ONE, fr_R2, fr_ROOT_OF_UNITY, fr_ZETA, fr_GENERATOR;
extern const fq_t fq_ONE, fq_R2;
#define FR_S 28

#define DECL_FP(P, T)                                              \
    void P##_add(T *r, const T *a, const T *b);                    \
    void P##_sub(T *r, const T *a, const T *b);                    \
    void P##_neg(T *r, const T *a);                                \
    void P##_dbl(T *r, const T *a);                                \
    void P##_mul(T *r, const T *a, const T *b);                    \
    void P##_sqr(T *r, const T *a);                                \
    void P##_to_repr(uint8_t out[32], const T *a);                 \
    int P##_from_repr(T *r, const uint8_t in[32]);                 \
    int P##_is_zero(const T *a);                                   \
    int P##_eq(const T *a, const T *b);                            \
    void P##_pow(T *r, const T *a, const uint64_t e[4]);           \
    int P##_inv(T *r, const T *a);                                 \
    void P##_batch_invert(T *v, uint64_t n, T *scratch);           \
    void P##_from_u64(T *r, uint64_t v);
DECL_FP(fr, fr_t)
DECL_FP(fq, fq_t)
#undef DECL_FP

/* ---- curve (bn254_curve.c) ---- */
void g1_identity(g1_t *r);
int g1_is_identity(const g1_t *p);
void g1_from_affine(g1_t *r, const g1_affine_t *p);
int g1_affine_is_identity(const g1_affine_t *p);
int g1_affine_is_on_curve(const g1_affine_t *p);
void g1_affine_neg(g1_affine_t *r, const g1_affine_t *p);
void g1_double(g1_t *r, const g1_t *p);
void g1_add(g1_t *r, const g1_t *p, const g1_t *q);
void g1_add_mixed(g1_t *r, const g1_t *p, const g1_affine_t *q);
void g1_neg(g1_t *r, const g1_t *p);
void g1_to_affine(g1_affine_t *r, const g1_t *p);
void g1_batch_normalize(g1_affine_t *out, const g1_t *in, uint64_t n);
void g1_mul(g1_t *r, const g1_t *p, const fr_t *s); /* double-and-add over to_repr bits */
int g1_eq(const g1_t *a, const g1_t *b);           /* projective equality */
void g1_generator(g1_affine_t *r);
/* compressed 32 B: x LE canonical | bit254 = lsb(y) | bit255 = identity */
void g1_affine_to_compressed(uint8_t out[32], const g1_affine_t *p);
int g1_affine_from_compressed(g1_affine_t *r, const uint8_t in[32]);

/* ---- halo2_proofs::arithmetic (halo2_arith.c) ---- */
void halo2_multiexp_serial(const fr_t *coeffs, const g1_affine_t *bases, uint64_t n, g1_t *acc);
void halo2_best_multiexp(const fr_t *coeffs, const g1_affine_t *bases, uint64_t n, int threads, g1_t *out);
void halo2_best_fft(fr_t *a, const fr_t *omega, uint32_t log_n, int threads);
void halo2_best_fft_g1(g1_t *a, const fr_t *omega, uint32_t log_n, int threads);
void halo2_eval_polynomial(fr_t *r, const fr_t *poly, uint64_t n, const fr_t *point);
void halo2_kate_division(fr_t *q, const fr_t *a, uint64_t n, const fr_t *b); /* q has n-1 */
void halo2_compute_inner_product(fr_t *r, const fr_t *a, const fr_t *b, uint64_t n);

/* ---- halo2_proofs::poly::EvaluationDomain (halo2_domain.c) ---- */
typedef struct {
    uint64_t n;
    uint32_t k, extended_k, quotient_poly_degree;
    fr_t omega, omega_inv, extended_omega, extended_omega_inv;
    fr_t g_coset, g_coset_inv, ifft_divisor, extended_ifft_divisor;
    fr_t barycentric_weight;
    uint32_t n_t_evaluations;
    fr_t t_evaluations[64];
} halo2_domain_t;
int halo2_domain_new(halo2_domain_t *d, uint32_t j, uint32_t k);
void halo2_distribute_powers_zeta(const halo2_domain_t *d, fr_t *a, uint64_t len, int into_coset);
void halo2_lagrange_to_coeff(const halo2_domain_t *d, fr_t *a, int threads);                 /* len n, in place */
void halo2_coeff_to_extended(const halo2_domain_t *d, const fr_t *a, fr_t *out, int threads); /* n -> 2^ext_k */
void halo2_extended_to_coeff(const halo2_domain_t *d, fr_t *a, int threads);                 /* in place; valid prefix n*qpd */

/* ---- halo2_proofs::poly::kzg::commitment::ParamsKZG (halo2_params.c) ---- */
/* unsafe_setup-style synthetic SRS with known tau: g[i] = tau^i G, g_lagrange[i] = L_i(tau) G */
void halo2_params_setup(uint32_t k, const fr_t *tau, g1_affine_t *g, g1_affine_t *g_lagrange, int threads);
void halo2_g_to_lagrange(const g1_affine_t *g, g1_affine_t *g_lagrange, uint32_t k, int threads);
void halo2_commit(const g1_affine_t *bases, const fr_t *poly, uint64_t n, int threads, g1_t *out);

/* ---- halo2_proofs::plonk quotient construction (halo2_quotient.c) ---- */
/* plonk::evaluation::{ValueSource, Calculation} in upstream declaration order (+ ExtendedX, see halo2_quotient.c) */
enum { HALO2_SRC_CONSTANT = 0, HALO2_SRC_INTERMEDIATE, HALO2_SRC_FIXED, HALO2_SRC_ADVICE, HALO2_SRC_INSTANCE,
       HALO2_SRC_CHALLENGE, HALO2_SRC_BETA, HALO2_SRC_GAMMA, HALO2_SRC_THETA, HALO2_SRC_Y, HALO2_SRC_PREVIOUS_VALUE,
       HALO2_SRC_EXTENDED_X };
enum { HALO2_CALC_ADD = 0, HALO2_CALC_SUB, HALO2_CALC_MUL, HALO2_CALC_SQUARE, HALO2_CALC_DOUBLE, HALO2_CALC_NEGATE,
       HALO2_CALC_HORNER, HALO2_CALC_STORE };
typedef struct { uint32_t kind, index, rotation; } halo2_value_source_t;
typedef struct {
    uint32_t op;
    halo2_value_source_t a, b; /* Horner: a = start value, b = factor */
    uint32_t parts_offset, parts_len;
} halo2_calculation_t;
int halo2_graph_evaluate(const halo2_calculation_t *calcs, uint32_t n_calcs, const halo2_value_source_t *parts,
                         const fr_t *constants, const int32_t *rotations, uint32_t n_rotations, const fr_t *const *fixed,
                         const fr_t *const *advice, const fr_t *const *instance, const fr_t *challenges, const fr_t *beta,
                         const fr_t *gamma, const fr_t *theta, const fr_t *y, const fr_t *extended_omega, fr_t *values,
                         uint32_t log_size, int32_t rot_scale);
void halo2_prefix_scan(int op, const fr_t *in, uint64_t n, const fr_t *init, fr_t *out);
int halo2_permutation_product(const fr_t *const *values, const fr_t *const *sigma, uint32_t n_cols, const fr_t *beta,
                              const fr_t *gamma, const fr_t *delta_omega_start, const fr_t *delta, const fr_t *omega,
                              uint32_t k, const fr_t *z_init, fr_t *z_out);
int halo2_logup_running_sum(const fr_t *const *inputs, uint32_t n_inputs, const fr_t *table, const fr_t *m,
                            const fr_t *beta, uint32_t k, const fr_t *phi_init, fr_t *phi_out);

int halo2_permutation_h_terms(const fr_t *const *z_cosets, uint32_t n_sets, uint32_t chunk_len, const fr_t *const *value_cosets,
                              const fr_t *const *sigma_cosets, uint32_t n_cols, const fr_t *l0, const fr_t *l_last,
                              const fr_t *l_active_row, const fr_t *beta, const fr_t *gamma, const fr_t *y, const fr_t *delta,
                              const fr_t *extended_omega, int32_t last_rotation, fr_t *values, uint32_t log_size,
                              int32_t rot_scale);
int halo2_logup_h_terms(const fr_t *const *input_cosets, uint32_t n_inputs, const fr_t *table_coset, const fr_t *m_coset,
                        const fr_t *phi_coset, const fr_t *l0, const fr_t *l_last, const fr_t *l_active_row, const fr_t *beta,
                        const fr_t *y, fr_t *values, uint32_t log_size, int32_t rot_scale);

/* ---- deterministic test-vector generator shared with the GPU tests (xorshift64*) ---- */
void oracle_fill_fr(fr_t *out, uint64_t n, uint64_t seed, int witness_like);
void oracle_fill_points(g1_affine_t *out, uint64_t n, uint64_t seed, int threads);
void oracle_fill_points_chain(g1_affine_t *out, uint64_t n, uint64_t seed, int threads);

/* ---- test helper, not a restatement of the reference (dft_identity.c) ---- */
/* out = (r^N - 1) * sum_{i<m} a_i c^i / (w^i r - 1), which equals sum_{j<N} y_j r^j for y_j = sum_i a_i c^i w^(ij):
 * an O(m) check of a whole transform.  Returns 0, -1 if w^N != 1, -2 if r^N == 1. */
int oracle_dft_eval_rhs(fr_t *out, const fr_t *a, uint64_t m, const fr_t *c, const fr_t *w, const fr_t *r, uint64_t N,
                        int threads);
/* halo2_eval_polynomial(y, n, r) split over threads (the left side of the identity at 2^28 elements) */
void oracle_eval_polynomial_mt(fr_t *out, const fr_t *y, uint64_t n, const fr_t *r, int threads);

#ifdef __cplusplus
}
#endif
#endif
