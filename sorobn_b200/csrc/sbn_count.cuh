// sorobn_b200 -- sm_90a count step of counts programs (planner.py KIND_COUNT = 3): the E-step of EM.
//
// One launch adds, for ONE CPT family, the expected counts of every row into a count table:
//
//     counts[key(b) + coff(s)] += sum_z prod_i in_i[ zoff_i(z) + soff_i(s) + evoff_i(b) ] / P_b
//
// where s runs over the joint states of the family's unobserved members M_v, z over the other
// variables of the bucket the family is read from, key(b) gathers the row's codes of the observed
// members and P_b = P(observed cells of b).  A family the program observes completely has no
// inputs: every row adds 1 at key(b).  The per-row family posteriors never reach HBM.
//
//   * the inner loop is the marginals readout's (sbn_marginal.cuh): one thread per row, host-built
//     offset tables (`zoff` [n_in][cz], `soff` [n_in][cs], `coff` [cs]), tables staged in shared
//     memory by bulk-TMA, products summed in T over runs of SBN_MARG_PART joint states and then in
//     double; each contribution is divided by P_b in double;
//   * a row with P_b below `min_total` (or zero / NaN) adds nothing; the host re-runs it in float64;
//   * no floating-point atomics, so that a result is bitwise reproducible: a fixed grid of persistent
//     CTAs walks the blocks of SBN_COUNT_THREADS rows in a fixed order (block blockIdx.x, then
//     + gridDim.x, ...).  In a warp, the lanes whose rows share a key are found once per block
//     (__match_any_sync); per state s, their contributions are summed in lane order (a shuffle
//     butterfly, also fixed, when all 32 share the key) and the group's lowest lane adds the sum to
//     the warp's own partial table in global memory.  `sbn_count_reduce` then adds the partial
//     tables into the count table, in partial-table order.
//
// `sbn_count_weighted_step` is the same step with a per-row double weight w_b (gradient programs,
// planner.py KIND_COUNT of version 10): each contribution is multiplied by w_b / P_b, and a fully
// observed family adds w_b.  Weights may be negative; the reduction order is the unweighted one.
//
// `sbn_joint_step` (joint programs, planner.py KIND_JOINT = 7) is the same per-row computation with an epilogue
// that stores instead of reducing: for ONE group of variables,
//
//     out[s * ld_out + b] = sum_z prod_i in_i[ zoff_i(z) + soff_i(s) + evoff_i(b) ] / P_b
//
// over the group's unobserved members s (their compact joint index, the first member fastest), rows innermost
// so that a warp's stores coalesce.  The division is in double and the result is rounded to T once; a row whose
// P_b is below `min_total` (or zero / NaN) is written NaN.  A group of more than C joint states runs in passes
// of C: the normaliser is known up front, so each pass stores its entries and nothing is re-read.  There is no
// key, no partial table and no atomic: two runs are bitwise equal.
#pragma once
#include "sbn_kernels.cuh"
#include "sbn_marginal.cuh"

#define SBN_COUNT_THREADS 128
#define SBN_COUNT_WARPS (SBN_COUNT_THREADS / 32)

struct SbnCountIn {
    const void *ptr;                 // table / slot base (device), float or double
    int32_t batched;                 // 1: entry e of row b is at e * ld + b
    int32_t n_ev;
    int32_t smem_off;                // float offset of the staged copy, -1 = read global
    int32_t stage_floats;
    int32_t ev_col[SBN_MAX_EV];
    int32_t ev_stride[SBN_MAX_EV];
    int32_t ev_card[SBN_MAX_EV];
};

struct SbnCount {
    double *partial;        // [gridDim.x * SBN_COUNT_WARPS][n_entries]
    const uint8_t *ev;
    int64_t ld_ev;
    int64_t ld;             // row pitch of batched operands
    const void *prob;       // P(observed) of every row: prob[b] (batched) or prob[0]
    const int32_t *zoff;    // [n_in][cz]
    const int32_t *soff;    // [n_in][cs]
    const int32_t *coff;    // [cs]
    double min_total;
    int32_t prob_batched;
    int32_t n_rows;
    int32_t n_in;
    int32_t n_common;       // inputs without any family axis (they come first)
    int32_t cs;             // joint states of the unobserved family members
    int32_t cz;             // joint states summed out
    int32_t n_entries;      // entries of the family's count table
    int32_t smem_floats;
    int32_t n_key;
    int32_t key_col[SBN_MAX_EV];
    int32_t key_stride[SBN_MAX_EV];
    int32_t key_card[SBN_MAX_EV];
    SbnCountIn in[SBN_MAX_IN];
};

// Sum of `v` over the lanes of `grp` (the lanes that share this lane's key), in a fixed order; the result
// is meaningful in the group's lowest lane.
__device__ __forceinline__ double sbn_group_sum(double v, unsigned grp) {
    if (grp == 0xffffffffu) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        return v;
    }
    double s = 0.0;
#pragma unroll
    for (int j = 0; j < 32; ++j) {
        const double x = __shfl_sync(0xffffffffu, v, j);
        if ((grp >> j) & 1u) s += x;
    }
    return s;
}

// The body of the count kernels and of the joint readout; W: rows weighted by weight[b]; J: the joint readout,
// which stores each row's entries at out[s * ld_out + b] instead of adding them to the warp's partial table
template <typename T, int C, bool W, bool J = false>
__device__ __forceinline__ void sbn_count_body(const SbnCount &p, const double *__restrict__ weight,
                                               T *__restrict__ out = nullptr, int64_t ld_out = 0) {
    extern __shared__ __align__(16) float s_tab[];
    __shared__ __align__(8) uint64_t s_bar;
    sbn_pdl_entry();

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    double *const part = J ? nullptr : p.partial + (static_cast<int64_t>(blockIdx.x) * SBN_COUNT_WARPS + warp) * p.n_entries;
    if constexpr (!J)
        for (int e = lane; e < p.n_entries; e += 32) part[e] = 0.0;

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
        sbn_mbar_wait(&s_bar, 0);
    }
    __syncwarp();

    const int n_in = p.n_in, n_common = p.n_common, cz = p.cz, cs = p.cs;
    constexpr int kRun = std::is_same<T, float>::value ? SBN_MARG_PART : (1 << 30);
    const int64_t n_blocks = (static_cast<int64_t>(p.n_rows) + SBN_COUNT_THREADS - 1) / SBN_COUNT_THREADS;
    for (int64_t blk = blockIdx.x; blk < n_blocks; blk += gridDim.x) {
        const int64_t b = blk * SBN_COUNT_THREADS + threadIdx.x;
        int key = -1;  // -1: no contribution (past the last row, or out of range)
        double inv = 0.0;
        double one = 1.0;  // what a fully observed family adds (joint readout: P_b)
        if (b < p.n_rows) {
            const double pr = static_cast<double>(static_cast<const T *>(p.prob)[p.prob_batched ? b : 0]);
            if (pr >= p.min_total) {  // false for NaN too
                if constexpr (J) {
                    one = pr;
                } else if constexpr (W) {
                    one = weight[b];
                    inv = one / pr;
                } else {
                    inv = 1.0 / pr;
                }
                key = 0;
                for (int k = 0; k < p.n_key; ++k)
                    key += min(static_cast<int>(p.ev[static_cast<int64_t>(p.key_col[k]) * p.ld_ev + b]), p.key_card[k] - 1) *
                           p.key_stride[k];
            }
        }
        const unsigned grp = J ? 0u : __match_any_sync(0xffffffffu, key);
        const bool lead = key >= 0 && lane == __ffs(grp) - 1;

        if (!J && n_in == 0) {  // a histogram of the keys
            const double v = sbn_group_sum(key >= 0 ? one : 0.0, grp);
            if (lead) part[key] += v;
            __syncwarp();
            continue;
        }
        const T *src[SBN_MAX_IN];
        int64_t mul[SBN_MAX_IN];
#pragma unroll
        for (int i = 0; i < SBN_MAX_IN; ++i) {
            src[i] = nullptr;
            mul[i] = 1;
            if (i < n_in && key >= 0) {
                const SbnCountIn &in = p.in[i];
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
        for (int s0 = 0; s0 < cs; s0 += C) {
            double acc[C];
#pragma unroll
            for (int s = 0; s < C; ++s) acc[s] = 0.0;
            if (key >= 0) {
                for (int z0 = 0; z0 < cz; z0 += kRun) {
                    T part_s[C];
#pragma unroll
                    for (int s = 0; s < C; ++s) part_s[s] = T(0);
                    const int z1 = z0 + min(kRun, cz - z0);
                    for (int z = z0; z < z1; ++z) {
                        int e[SBN_MAX_IN];
#pragma unroll
                        for (int i = 0; i < SBN_MAX_IN; ++i)
                            if (i < n_in) e[i] = __ldg(p.zoff + static_cast<int64_t>(i) * cz + z);
                        T common = T(1);
#pragma unroll
                        for (int i = 0; i < SBN_MAX_IN; ++i)
                            if (i < n_common) common *= src[i][static_cast<int64_t>(e[i]) * mul[i]];
#pragma unroll
                        for (int s = 0; s < C; ++s) {
                            if (s0 + s < cs) {
                                T v = common;
#pragma unroll
                                for (int i = 0; i < SBN_MAX_IN; ++i)
                                    if (i >= n_common && i < n_in)
                                        v *= src[i][static_cast<int64_t>(e[i] + __ldg(p.soff + static_cast<int64_t>(i) * cs + s0 + s)) * mul[i]];
                                part_s[s] += v;
                            }
                        }
                    }
#pragma unroll
                    for (int s = 0; s < C; ++s) acc[s] += static_cast<double>(part_s[s]);
                }
            }
            if constexpr (J) {
                if (b < p.n_rows) {
#pragma unroll
                    for (int s = 0; s < C; ++s)
                        if (s0 + s < cs)
                            out[static_cast<int64_t>(s0 + s) * ld_out + b] =
                                key >= 0 ? static_cast<T>(acc[s] / one) : static_cast<T>(__int_as_float(0x7fc00000));
                }
                continue;
            }
#pragma unroll
            for (int s = 0; s < C; ++s) {
                if (s0 + s < cs) {  // warp-uniform
                    const double v = sbn_group_sum(acc[s] * inv, grp);
                    if (lead) part[key + __ldg(p.coff + s0 + s)] += v;
                }
            }
            __syncwarp();
        }
    }
}

template <typename T, int C>
__global__ void __launch_bounds__(SBN_COUNT_THREADS) sbn_count_step(const __grid_constant__ SbnCount p) {
    sbn_count_body<T, C, false>(p, nullptr);
}

template <typename T, int C>
__global__ void __launch_bounds__(SBN_COUNT_THREADS) sbn_count_weighted_step(const __grid_constant__ SbnCount p,
                                                                              const double *__restrict__ weight) {
    sbn_count_body<T, C, true>(p, weight);
}

// `out` is the group's first output row; p.partial, p.coff and the key are unused
template <typename T, int C>
__global__ void __launch_bounds__(SBN_COUNT_THREADS) sbn_joint_step(const __grid_constant__ SbnCount p, T *__restrict__ out,
                                                                     int64_t ld_out) {
    sbn_count_body<T, C, false, true>(p, nullptr, out, ld_out);
}

// count[e] += sum over the partial tables, in partial-table order
__global__ void sbn_count_reduce(const double *__restrict__ partial, int64_t n_parts, int32_t n_entries,
                                 double *__restrict__ counts) {
    const int64_t e = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (e >= n_entries) return;
    double s = 0.0;
    for (int64_t g = 0; g < n_parts; ++g) s += partial[g * n_entries + e];
    counts[e] += s;
}

// The run's per-row output: P(observed), NaN where it is out of range
template <typename T>
__global__ void sbn_count_prob(const T *__restrict__ prob, int32_t prob_batched, int32_t n_rows, double min_total,
                               T *__restrict__ out) {
    const int64_t b = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (b >= n_rows) return;
    const T v = prob[prob_batched ? b : 0];
    out[b] = static_cast<double>(v) >= min_total ? v : static_cast<T>(__int_as_float(0x7fc00000));
}

// `weight` non-null: the weighted step (gradient programs)
template <typename T>
inline cudaError_t sbn_count_launch(const SbnCount &c, int64_t grid, size_t smem, double *counts, cudaStream_t stream,
                                    const double *weight = nullptr) {
    const unsigned g = static_cast<unsigned>(grid);
    if (weight) {
        if (c.cs <= 2) sbn_count_weighted_step<T, 2><<<g, SBN_COUNT_THREADS, smem, stream>>>(c, weight);
        else if (c.cs <= 4) sbn_count_weighted_step<T, 4><<<g, SBN_COUNT_THREADS, smem, stream>>>(c, weight);
        else sbn_count_weighted_step<T, 8><<<g, SBN_COUNT_THREADS, smem, stream>>>(c, weight);
    } else if (c.cs <= 2) sbn_count_step<T, 2><<<g, SBN_COUNT_THREADS, smem, stream>>>(c);
    else if (c.cs <= 4) sbn_count_step<T, 4><<<g, SBN_COUNT_THREADS, smem, stream>>>(c);
    else sbn_count_step<T, 8><<<g, SBN_COUNT_THREADS, smem, stream>>>(c);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    const int threads = 256;
    sbn_count_reduce<<<static_cast<unsigned>((c.n_entries + threads - 1) / threads), threads, 0, stream>>>(
        c.partial, grid * SBN_COUNT_WARPS, c.n_entries, counts);
    return cudaGetLastError();
}

// One CTA per SBN_COUNT_THREADS rows; C = the smallest instantiated accumulator count that covers the group (8 and
// passes beyond)
template <typename T>
inline cudaError_t sbn_joint_launch(const SbnCount &c, size_t smem, T *out, int64_t ld_out, cudaStream_t stream) {
    const unsigned g = static_cast<unsigned>((static_cast<int64_t>(c.n_rows) + SBN_COUNT_THREADS - 1) / SBN_COUNT_THREADS);
    if (c.cs <= 2) sbn_joint_step<T, 2><<<g, SBN_COUNT_THREADS, smem, stream>>>(c, out, ld_out);
    else if (c.cs <= 4) sbn_joint_step<T, 4><<<g, SBN_COUNT_THREADS, smem, stream>>>(c, out, ld_out);
    else sbn_joint_step<T, 8><<<g, SBN_COUNT_THREADS, smem, stream>>>(c, out, ld_out);
    return cudaGetLastError();
}

inline cudaError_t sbn_joint_set_attrs() {
    cudaError_t e = cudaFuncSetAttribute(sbn_joint_step<float, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, SBN_SMEM_BUDGET);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(sbn_joint_step<float, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, SBN_SMEM_BUDGET);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(sbn_joint_step<float, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize, SBN_SMEM_BUDGET);
    return e;
}

inline cudaError_t sbn_count_set_attrs() {
    cudaError_t e = cudaFuncSetAttribute(sbn_count_step<float, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, SBN_SMEM_BUDGET);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(sbn_count_step<float, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, SBN_SMEM_BUDGET);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(sbn_count_step<float, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize, SBN_SMEM_BUDGET);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(sbn_count_weighted_step<float, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, SBN_SMEM_BUDGET);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(sbn_count_weighted_step<float, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, SBN_SMEM_BUDGET);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(sbn_count_weighted_step<float, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize, SBN_SMEM_BUDGET);
    return e;
}
