// sorobn_b200 -- sm_90a readout kernel of marginals programs (planner.py KIND_MARGINAL = 2).
//
// One launch reads the marginal of ONE target t from a bucket of the bucket tree:
//
//     M_t(s, b) = sum_z  prod_i  in_i[ zoff_i(z) + s * ts_i + evoff_i(b) ]   (, b)
//
// where z runs over the joint states of the bucket's other variables, and writes the row's
// segment normalised, M_t / sum_s M_t, straight into the run's posterior output.  The bucket
// belief (a factor over every variable of the bucket) is never materialised.
//
//   * one thread = one evidence row, rows innermost: a warp reads 32 consecutive rows of one
//     operand entry (128 bytes) per load, the layout every step kernel uses;
//   * `zoff` ([n_in][cz], first variable fastest) is the row-invariant part of every operand's
//     offset, precomputed on the host like the step kernels' zoff / tile_off;
//   * inputs 0 .. n_common-1 lack the target axis (ts = 0): they are loaded once per z, the
//     others once per (z, s);
//   * C accumulators per thread, one per target state; a target with more than C states is done
//     in passes of C states (the raw values are written, then re-read and normalised);
//   * a readout sums cz joint states per entry with no MAX_Z bound (625 on the benchmark grid, up to
//     2^21), and a float32 running sum of that many terms misses the 1e-6 relative promise.  So the
//     products are summed in T over runs of SBN_MARG_PART joint states, and those partial sums in
//     double; the segment total, the range rule and the division are double too, and each entry is
//     rounded to T once (a raw value of a multi-pass target twice: when it is written, and after the
//     division).  A double add per product would need a float->double conversion per product, a
//     low-throughput instruction on sm_90: that variant made the benchmark grid's marginals program
//     4.5 % slower (100k rows, H100 80GB HBM3 at a 400 W power limit);
//   * tables (CPTs, evidence-independent factors) are staged in shared memory by bulk-TMA when
//     they fit SBN_SMEM_BUDGET (float only), otherwise gathered through L1;
//   * the range rule of sbn_normalise: a row whose segment total, or smallest non-zero entry, is
//     below `min_total` (or zero / NaN) is written as NaN; the host re-runs such rows in float64.
#pragma once
#include "sbn_kernels.cuh"

#define SBN_MARG_THREADS 128
#define SBN_MARG_PART 32  // joint states summed in T before the double accumulator takes the partial sum

struct SbnMargIn {
    const void *ptr;                 // table / slot base (device), float or double
    int32_t batched;                 // 1: entry e of row b is at e * ld + b
    int32_t ts;                      // stride of the target axis (0 = input lacks it)
    int32_t n_ev;
    int32_t smem_off;                // float offset of the staged copy, -1 = read global
    int32_t stage_floats;
    int32_t pad_;
    int32_t ev_col[SBN_MAX_EV];
    int32_t ev_stride[SBN_MAX_EV];
    int32_t ev_card[SBN_MAX_EV];
};

struct SbnMarginal {
    void *out;              // the target's first posterior row: [card][ld_out]
    int64_t ld_out;
    const uint8_t *ev;
    int64_t ld_ev;
    int64_t ld;             // row pitch of batched operands
    const int32_t *zoff;    // [n_in][cz]
    double min_total;
    int32_t n_rows;
    int32_t n_in;
    int32_t n_common;       // inputs without the target axis (they come first)
    int32_t card;           // target states
    int32_t cz;             // joint states summed out
    int32_t smem_floats;
    SbnMargIn in[SBN_MAX_IN];
};

// The body of the marginals readout and of the derivative readout of gradient programs (sbn_deriv.cuh).
// D = false: the segment is normalised (above).  D = true: each entry is divided by the row's P(observed),
// prob[b] (prob_batched) or prob[0], in double, and rounded to T once; a row whose P(observed) is below
// min_total (or zero / NaN) is written NaN.
template <typename T, int C, bool D>
__device__ __forceinline__ void sbn_readout_body(const SbnMarginal &p, const void *prob, int32_t prob_batched) {
    extern __shared__ __align__(16) float s_tab[];
    __shared__ __align__(8) uint64_t s_bar;
    sbn_pdl_entry();

    const bool staged = p.smem_floats > 0;
    if (staged) {
        if (threadIdx.x == 0) {
            sbn_mbar_init(&s_bar, 1);
            sbn_fence_mbar_init();
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            sbn_mbar_expect_tx(&s_bar, static_cast<uint32_t>(p.smem_floats) * 4u);
            for (int i = 0; i < p.n_in; ++i)
                if (p.in[i].smem_off >= 0)
                    sbn_tma_bulk_g2s(s_tab + p.in[i].smem_off, p.in[i].ptr, static_cast<uint32_t>(p.in[i].stage_floats) * 4u,
                                     &s_bar);
        }
    }

    const int64_t b = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    const bool live = b < p.n_rows;

    // operand i, entry e, this row:  src[i][e * mul[i]]  (src already points at the row / evidence offset)
    const T *src[SBN_MAX_IN];
    int64_t mul[SBN_MAX_IN];
#pragma unroll
    for (int i = 0; i < SBN_MAX_IN; ++i) {
        src[i] = nullptr;
        mul[i] = 1;
        if (i < p.n_in && live) {
            const SbnMargIn &in = p.in[i];
            if (in.batched) {
                src[i] = static_cast<const T *>(in.ptr) + b;
                mul[i] = p.ld;
            } else {
                int64_t evo = 0;
                for (int k = 0; k < in.n_ev; ++k)
                    evo += static_cast<int64_t>(min(static_cast<int>(p.ev[static_cast<int64_t>(in.ev_col[k]) * p.ld_ev + b]),
                                                    in.ev_card[k] - 1)) * in.ev_stride[k];
                if constexpr (std::is_same<T, float>::value) {
                    if (in.smem_off >= 0) src[i] = s_tab + in.smem_off + evo;
                    else src[i] = static_cast<const T *>(in.ptr) + evo;
                } else {
                    src[i] = static_cast<const T *>(in.ptr) + evo;
                }
            }
        }
    }
    if (staged) sbn_mbar_wait(&s_bar, 0);
    if (!live) return;

    T *const out = static_cast<T *>(p.out) + b;
    const int n_in = p.n_in, n_common = p.n_common, cz = p.cz, card = p.card;
    // float: runs of SBN_MARG_PART joint states; double: one run (the partial sum is the sum)
    constexpr int kRun = std::is_same<T, float>::value ? SBN_MARG_PART : (1 << 30);
    double total = 0.0, lo = p.min_total;  // D: `total` holds the row's P(observed)
    if constexpr (D) {
        total = static_cast<double>(static_cast<const T *>(prob)[prob_batched ? b : 0]);
        if (!(total >= p.min_total)) {  // out of range, zero or NaN
            for (int s = 0; s < card; ++s) out[static_cast<int64_t>(s) * p.ld_out] = static_cast<T>(__int_as_float(0x7fc00000));
            return;
        }
    }
    double acc[C];  // after the last pass: its sums (all of them when card <= C)
    for (int s0 = 0; s0 < card; s0 += C) {
#pragma unroll
        for (int s = 0; s < C; ++s) acc[s] = 0.0;
        for (int z0 = 0; z0 < cz; z0 += kRun) {
            T part[C];
#pragma unroll
            for (int s = 0; s < C; ++s) part[s] = T(0);
            const int z1 = z0 + min(kRun, cz - z0);
            for (int z = z0; z < z1; ++z) {
                int e[SBN_MAX_IN];
#pragma unroll
                for (int i = 0; i < SBN_MAX_IN; ++i)
                    if (i < n_in) e[i] = __ldg(p.zoff + static_cast<int64_t>(i) * cz + z) + s0 * p.in[i].ts;
                T common = T(1);
#pragma unroll
                for (int i = 0; i < SBN_MAX_IN; ++i)
                    if (i < n_common) common *= src[i][e[i] * mul[i]];
#pragma unroll
                for (int s = 0; s < C; ++s) {
                    if (s0 + s < card) {
                        T v = common;
#pragma unroll
                        for (int i = 0; i < SBN_MAX_IN; ++i)
                            if (i >= n_common && i < n_in) v *= src[i][static_cast<int64_t>(e[i] + s * p.in[i].ts) * mul[i]];
                        part[s] += v;
                    }
                }
            }
#pragma unroll
            for (int s = 0; s < C; ++s) acc[s] += static_cast<double>(part[s]);
        }
        if constexpr (D) {
#pragma unroll
            for (int s = 0; s < C; ++s)
                if (s0 + s < card) out[static_cast<int64_t>(s0 + s) * p.ld_out] = static_cast<T>(acc[s] / total);
        } else {
#pragma unroll
            for (int s = 0; s < C; ++s) {
                if (s0 + s < card) {
                    total += acc[s];
                    if (acc[s] > 0.0 && acc[s] < lo) lo = acc[s];
                    if (card > C) out[static_cast<int64_t>(s0 + s) * p.ld_out] = static_cast<T>(acc[s]);
                }
            }
        }
    }
    if constexpr (!D) {
        // false for NaN too (in this order the shared body compiles to the standalone kernel's instructions)
        const bool ok = lo >= p.min_total && total >= p.min_total;
        const T nan = static_cast<T>(__int_as_float(0x7fc00000));
        if (card <= C) {
#pragma unroll
            for (int s = 0; s < C; ++s)
                if (s < card) out[static_cast<int64_t>(s) * p.ld_out] = ok ? static_cast<T>(acc[s] / total) : nan;
        } else {
            for (int s = 0; s < card; ++s) {
                T *o = out + static_cast<int64_t>(s) * p.ld_out;
                *o = ok ? static_cast<T>(static_cast<double>(*o) / total) : nan;
            }
        }
    }
}

template <typename T, int C>
__global__ void __launch_bounds__(SBN_MARG_THREADS) sbn_marginal_step(const __grid_constant__ SbnMarginal p) {
    sbn_readout_body<T, C, false>(p, nullptr, 0);
}

// C = the smallest instantiated accumulator count that covers the target (8 and passes beyond)
template <typename T>
inline cudaError_t sbn_marginal_launch(const SbnMarginal &m, size_t smem, cudaStream_t stream) {
    const unsigned grid = static_cast<unsigned>((m.n_rows + SBN_MARG_THREADS - 1) / SBN_MARG_THREADS);
    if (m.card <= 2) sbn_marginal_step<T, 2><<<grid, SBN_MARG_THREADS, smem, stream>>>(m);
    else if (m.card <= 4) sbn_marginal_step<T, 4><<<grid, SBN_MARG_THREADS, smem, stream>>>(m);
    else sbn_marginal_step<T, 8><<<grid, SBN_MARG_THREADS, smem, stream>>>(m);
    return cudaGetLastError();
}

inline cudaError_t sbn_marginal_set_attrs() {
    cudaError_t e = cudaFuncSetAttribute(sbn_marginal_step<float, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, SBN_SMEM_BUDGET);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(sbn_marginal_step<float, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, SBN_SMEM_BUDGET);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(sbn_marginal_step<float, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize, SBN_SMEM_BUDGET);
    return e;
}
