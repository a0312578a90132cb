// sorobn_b200 -- sm_90a derivative readout of gradient programs (planner.py KIND_DERIV = 6).
//
// One launch reads, for ONE soft variable s, the derivative of log P(observed, lik) by its likelihood:
//
//     D_s(x, b) = sum_z  prod_i  in_i[ zoff_i(z) + x * ts_i + evoff_i(b) ]  /  P_b
//
// over the bucket that lambda_s entered, with every input of that bucket except lambda_s itself (the
// planner leaves it out), and P_b = P(observed) of row b.  The result is exact where lambda_s(x) = 0.
//
// It is the marginals readout (sbn_marginal.cuh, `sbn_readout_body`): one thread per row, the host-built
// joint-state offset table `zoff`, tables staged in shared memory by bulk-TMA, the products summed in T over
// runs of SBN_MARG_PART joint states and then in double.  Only the epilogue differs: instead of normalising
// the segment, each entry is divided by P_b in double and rounded to T once, and a row whose P_b is below
// `min_total` (or zero / NaN) is written NaN; the host re-runs it in float64.
#pragma once
#include "sbn_kernels.cuh"
#include "sbn_marginal.cuh"

struct SbnDeriv {
    SbnMarginal m;          // `out` is the soft variable's first output row; `card` its states
    const void *prob;       // P(observed) of every row: prob[b] (batched) or prob[0]
    int32_t prob_batched;
};

template <typename T, int C>
__global__ void __launch_bounds__(SBN_MARG_THREADS) sbn_deriv_step(const __grid_constant__ SbnDeriv p) {
    sbn_readout_body<T, C, true>(p.m, p.prob, p.prob_batched);
}

// C = the smallest instantiated accumulator count that covers the soft variable (8 and passes beyond)
template <typename T>
inline cudaError_t sbn_deriv_launch(const SbnDeriv &d, size_t smem, cudaStream_t stream) {
    const unsigned grid = static_cast<unsigned>((d.m.n_rows + SBN_MARG_THREADS - 1) / SBN_MARG_THREADS);
    if (d.m.card <= 2) sbn_deriv_step<T, 2><<<grid, SBN_MARG_THREADS, smem, stream>>>(d);
    else if (d.m.card <= 4) sbn_deriv_step<T, 4><<<grid, SBN_MARG_THREADS, smem, stream>>>(d);
    else sbn_deriv_step<T, 8><<<grid, SBN_MARG_THREADS, smem, stream>>>(d);
    return cudaGetLastError();
}

inline cudaError_t sbn_deriv_set_attrs() {
    cudaError_t e = cudaFuncSetAttribute(sbn_deriv_step<float, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, SBN_SMEM_BUDGET);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(sbn_deriv_step<float, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, SBN_SMEM_BUDGET);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(sbn_deriv_step<float, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize, SBN_SMEM_BUDGET);
    return e;
}
