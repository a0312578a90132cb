// sorobn_b200 -- soft evidence: the likelihood slots of a program, filled before its first step.
//
// A soft-evidence variable v carries a per-row likelihood lambda_v over its states (planner.py, "Soft
// evidence"): one batched leaf factor [card_v][ld], rows innermost, that the step kernels read like any other
// batched operand.  sbn_soft_pack fills those slots from the caller's likelihood matrix, `[n_rows][ld_lik]`
// row-major with the soft variables' states as columns (variables sorted by name, states in domain order).
//
// Each variable's row is divided by its maximum, so that every entry is at most 1 and every intermediate of
// the program stays <= 1 (DESIGN.md "Precision and fp32 range"): the float32 range rule, the NaN flags and the
// float64 rescue keep their meaning.  The divided-out maxima come back as sum_v log(max_v) per row, in double,
// for log P(e, lambda).  An all-zero row stores zeros and -inf: the row is impossible, like impossible hard
// evidence.
//
// Thread = one evidence row; each store of a state is 32 consecutive rows of a warp (coalesced).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

// desc: (row offset of the variable's slot in the batched arena, in entries per row; card) per soft variable
template <typename T>
__global__ void __launch_bounds__(256) sbn_soft_pack(const T *__restrict__ lik, int64_t ld_lik, int32_t n_rows,
                                                     int32_t n_soft, const int32_t *__restrict__ desc,
                                                     T *__restrict__ arena, int64_t ld, double *__restrict__ log_max) {
    const int64_t b = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (b >= n_rows) return;
    const T *row = lik + b * ld_lik;
    double acc = 0.0;
    for (int v = 0, col = 0; v < n_soft; ++v) {
        const int64_t off = desc[2 * v];
        const int card = desc[2 * v + 1];
        T m = T(0);
        for (int j = 0; j < card; ++j) {
            const T x = row[col + j];
            m = x > m ? x : m;
        }
        T *dst = arena + off * ld + b;
        for (int j = 0; j < card; ++j) dst[j * ld] = m > T(0) ? row[col + j] / m : T(0);
        acc += log(static_cast<double>(m));  // -inf for an all-zero row
        col += card;
    }
    log_max[b] = acc;
}

// The log-domain pack of MPE and marginal MAP programs (float programs only: they have no float64 twin).  It reads
// the caller's likelihoods in double, so that any finite non-negative scale -- 1e-50 or 1e40 -- reaches it intact,
// and stores each entry as log(x / max) computed in double and rounded once to float, -inf for x == 0.  An all-zero
// row is -inf throughout, so its max log P comes out -inf (impossible).  Same thread mapping and descriptors as
// sbn_soft_pack, and the same sum_v log(max_v) per row in double, which the host adds back to the program's max
// log P.
__global__ void __launch_bounds__(256) sbn_soft_pack_log(const double *__restrict__ lik, int64_t ld_lik, int32_t n_rows,
                                                         int32_t n_soft, const int32_t *__restrict__ desc,
                                                         float *__restrict__ arena, int64_t ld,
                                                         double *__restrict__ log_max) {
    const int64_t b = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (b >= n_rows) return;
    const double *row = lik + b * ld_lik;
    double acc = 0.0;
    for (int v = 0, col = 0; v < n_soft; ++v) {
        const int64_t off = desc[2 * v];
        const int card = desc[2 * v + 1];
        double m = 0.0;
        for (int j = 0; j < card; ++j) {
            const double x = row[col + j];
            m = x > m ? x : m;
        }
        float *dst = arena + off * ld + b;
        for (int j = 0; j < card; ++j) {
            const double x = row[col + j];
            dst[j * ld] = x > 0.0 ? __double2float_rn(log(x / m)) : -INFINITY;
        }
        acc += log(m);  // -inf for an all-zero row
        col += card;
    }
    log_max[b] = acc;
}
