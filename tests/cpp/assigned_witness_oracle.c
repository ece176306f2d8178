/* CPU restatement of halo2-base's own witness form, for the tests (tests/assigned_oracle.py builds it into a temporary
 * directory and links it against the oracle's field arithmetic, oracle/_build/liboracle.so).  It is walked the way the
 * Rust code walks it, not the way the kernels do:
 * 1. the Vec<Assigned<Fr>> the inputs stand for: Rational(values[index[i]], den[i]) at index[i], Trivial(values[j]) elsewhere;
 * 2. batch_invert_assigned: the denominators of the Rational cells in column order, one BatchInvert::batch_invert over them
 *    (orc_batch_invert: zeros stay zero), then every cell = numerator * (inverse of its denominator, or 1 without one);
 * 3. LookupAnyManager::assign_raw (halo2-base/src/virtual_region/lookups.rs:130-155): the i-th looked-up cell is the
 *    AssignedValue at lk_index[i], copied to lookup column i % L, row i / L of lk_cols (L x 2^k, pre-zeroed).
 * Returns 0; -1 where orc_assign_lookups returns -1 (rows overflow, or lookups without columns); -2 for an index >= N;
 * -3 for Rational indices that do not strictly increase. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef uint64_t u64;
void orc_f_mul(int w, const u64 *a, const u64 *b, u64 *r, size_t n); /* liboracle: w = 1 is Fr, Montgomery limbs */
void orc_batch_invert(u64 *a, size_t n);

enum { TRIVIAL = 1, RATIONAL = 2 };
typedef struct { int tag; u64 num[4], den[4]; } assigned_t;

int aw_assigned_witness(const u64 *values, size_t N, const u64 *index, const u64 *den, size_t R, const u64 *lk_index, size_t n_lookup,
                        unsigned k, size_t L, u64 *out, u64 *lk_cols) {
    for (size_t i = 0; i < R; i++) {
        if (index[i] >= N) return -2;
        if (i > 0 && index[i] <= index[i - 1]) return -3;
    }
    for (size_t i = 0; i < n_lookup; i++)
        if (lk_index[i] >= N) return -2;
    assigned_t *cells = (assigned_t *)calloc(N ? N : 1, sizeof(assigned_t));
    for (size_t j = 0; j < N; j++) { cells[j].tag = TRIVIAL; memcpy(cells[j].num, values + 4 * j, 32); }
    for (size_t i = 0; i < R; i++) { cells[index[i]].tag = RATIONAL; memcpy(cells[index[i]].den, den + 4 * i, 32); }
    /* batch_invert_assigned */
    u64 *denoms = (u64 *)malloc((N ? N : 1) * 32);
    size_t nd = 0;
    for (size_t j = 0; j < N; j++)
        if (cells[j].tag == RATIONAL) memcpy(denoms + 4 * nd++, cells[j].den, 32);
    orc_batch_invert(denoms, nd);
    size_t di = 0;
    for (size_t j = 0; j < N; j++) {
        if (cells[j].tag == RATIONAL) orc_f_mul(1, cells[j].num, denoms + 4 * di++, out + 4 * j, 1);
        else memcpy(out + 4 * j, cells[j].num, 32);
    }
    free(denoms);
    free(cells);
    /* assign_raw */
    size_t rows = (size_t)1 << k;
    if (L) memset(lk_cols, 0, L * rows * 32);
    if (L == 0) return n_lookup == 0 ? 0 : -1;
    for (size_t i = 0; i < n_lookup; i++) {
        size_t c = i % L, r = i / L;
        if (r >= rows) return -1;
        memcpy(lk_cols + 4 * (c * rows + r), out + 4 * lk_index[i], 32);
    }
    return 0;
}
