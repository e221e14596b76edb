/*
 * TEST HELPER — not a restatement of the reference (see oracle/README.md).
 *
 * An O(m) check of a whole discrete Fourier transform.  Let y_j = sum_{i<m} a_i c^i w^(ij) for j < N, with w an N-th
 * root of unity (w^N = 1).  Then for any r with r^N != 1
 *
 *     sum_{j<N} y_j r^j = (r^N - 1) * sum_{i<m} a_i c^i / (w^i r - 1),
 *
 * because sum_{j<N} (w^i r)^j = ((w^i r)^N - 1) / (w^i r - 1) and (w^i r)^N = r^N.  The left side is the Horner
 * evaluation of y at r (halo2_eval_polynomial); this file computes the right side.  Every forward transform the
 * prover issues has this shape (plain: c = 1; zero-padded: m < N; coset: c = zeta; coset part j: c = zeta w_ext^j,
 * w = w_ext^J; m > N also holds), and an inverse transform is checked through the forward relation of its output.
 * Both sides are polynomials of degree < N in r, so a y that differs in any element passes with probability at most
 * N / |Fr| for a random r.
 */
#include <pthread.h>
#include <stdlib.h>
#include <string.h>

#include "bn254_oracle.h"

#define DFT_BLOCK 1024 /* denominators inverted together (one field inversion per block) */

typedef struct {
    const fr_t *a, *c, *w, *r;
    uint64_t lo, hi;
    fr_t acc;
} dft_job_t;

static void fr_pow_u64_(fr_t *out, const fr_t *x, uint64_t e) {
    const uint64_t ee[4] = {e, 0, 0, 0};
    fr_pow(out, x, ee);
}

static void *dft_worker(void *arg) {
    dft_job_t *j = (dft_job_t *)arg;
    fr_t cp, wp, den[DFT_BLOCK], num[DFT_BLOCK], scratch[DFT_BLOCK];
    fr_pow_u64_(&cp, j->c, j->lo); /* c^i and w^i at the first index of this slice */
    fr_pow_u64_(&wp, j->w, j->lo);
    memset(&j->acc, 0, sizeof j->acc);
    for (uint64_t i0 = j->lo; i0 < j->hi; i0 += DFT_BLOCK) {
        uint64_t len = j->hi - i0 < DFT_BLOCK ? j->hi - i0 : DFT_BLOCK;
        for (uint64_t t = 0; t < len; ++t) {
            fr_mul(&den[t], &wp, j->r);
            fr_sub(&den[t], &den[t], &fr_ONE);
            fr_mul(&num[t], &j->a[i0 + t], &cp);
            fr_mul(&cp, &cp, j->c);
            fr_mul(&wp, &wp, j->w);
        }
        fr_batch_invert(den, len, scratch);
        for (uint64_t t = 0; t < len; ++t) {
            fr_t q;
            fr_mul(&q, &num[t], &den[t]);
            fr_add(&j->acc, &j->acc, &q);
        }
    }
    return NULL;
}

/* the left side on all host threads: slice t (from index lo_t) is a Horner evaluation h_t, and y(r) = sum_t r^lo_t h_t */
typedef struct {
    const fr_t *y, *r;
    uint64_t lo, hi;
    fr_t acc;
} horner_job_t;

static void *horner_worker(void *arg) {
    horner_job_t *j = (horner_job_t *)arg;
    halo2_eval_polynomial(&j->acc, j->y + j->lo, j->hi - j->lo, j->r);
    fr_t s;
    fr_pow_u64_(&s, j->r, j->lo);
    fr_mul(&j->acc, &j->acc, &s);
    return NULL;
}

void oracle_eval_polynomial_mt(fr_t *out, const fr_t *y, uint64_t n, const fr_t *r, int threads) {
    if (threads < 1) threads = 1;
    if ((uint64_t)threads > n / DFT_BLOCK + 1) threads = (int)(n / DFT_BLOCK + 1);
    horner_job_t *jobs = (horner_job_t *)malloc(sizeof(horner_job_t) * threads);
    pthread_t *tids = (pthread_t *)malloc(sizeof(pthread_t) * threads);
    uint64_t chunk = (n + threads - 1) / threads;
    for (int t = 0; t < threads; ++t) {
        uint64_t lo = (uint64_t)t * chunk, hi = lo + chunk;
        jobs[t] = (horner_job_t){y, r, lo < n ? lo : n, hi < n ? hi : n, {{0, 0, 0, 0}}};
        if (t) pthread_create(&tids[t], NULL, horner_worker, &jobs[t]);
    }
    horner_worker(&jobs[0]);
    fr_t sum = jobs[0].acc;
    for (int t = 1; t < threads; ++t) {
        pthread_join(tids[t], NULL);
        fr_add(&sum, &sum, &jobs[t].acc);
    }
    *out = sum;
    free(jobs);
    free(tids);
}

/* out = (r^N - 1) * sum_{i<m} a_i c^i / (w^i r - 1).  Returns 0, -1 if w^N != 1, -2 if r^N == 1. */
int oracle_dft_eval_rhs(fr_t *out, const fr_t *a, uint64_t m, const fr_t *c, const fr_t *w, const fr_t *r, uint64_t N,
                        int threads) {
    fr_t wN, rN;
    fr_pow_u64_(&wN, w, N);
    if (!fr_eq(&wN, &fr_ONE)) return -1;
    fr_pow_u64_(&rN, r, N);
    fr_sub(&rN, &rN, &fr_ONE);
    if (fr_is_zero(&rN)) return -2;
    if (threads < 1) threads = 1;
    if ((uint64_t)threads > m / DFT_BLOCK + 1) threads = (int)(m / DFT_BLOCK + 1);
    dft_job_t *jobs = (dft_job_t *)malloc(sizeof(dft_job_t) * threads);
    pthread_t *tids = (pthread_t *)malloc(sizeof(pthread_t) * threads);
    uint64_t chunk = (m + threads - 1) / threads;
    for (int t = 0; t < threads; ++t) {
        uint64_t lo = (uint64_t)t * chunk, hi = lo + chunk;
        jobs[t] = (dft_job_t){a, c, w, r, lo < m ? lo : m, hi < m ? hi : m, {{0, 0, 0, 0}}};
        if (t) pthread_create(&tids[t], NULL, dft_worker, &jobs[t]);
    }
    dft_worker(&jobs[0]);
    fr_t sum = jobs[0].acc;
    for (int t = 1; t < threads; ++t) {
        pthread_join(tids[t], NULL);
        fr_add(&sum, &sum, &jobs[t].acc);
    }
    fr_mul(out, &sum, &rN);
    free(jobs);
    free(tids);
    return 0;
}
