// sorobn_b200 -- sm_90a argmax step of MPE programs (planner.py KIND_ARGMAX = 5): max-sum decoding.
//
// An MPE program (planner.build_mpe_plan, version 8) ships the logs of its tables.  Its upward pass runs the
// step kernels with the max-sum policy (SbnMaxSum, sbn_kernels.cuh): out = max_x sum_i in_i.  Then, top-down,
// one launch per bucket decodes, for every row b, the joint state X of the bucket's eliminated variables:
//
//     w(z) = sum_i in_i[ zoff_i(z) + termoff_i(b) ]        z = 0 .. cz - 1 (first variable fastest)
//
// where termoff gathers the row's observed codes and the codes earlier steps decoded for the row -- the
// bucket's separator -- exactly as a sample step does (sbn_sample.cuh, with one draw).  The pick is the
// first z with the largest w(z): z walks upwards and a later state wins only by a strict `>`.
//
//   * one thread = one row, the grid and the bulk-TMA table staging of sbn_sample_step;
//   * w(z) = ((0 + in_0) + in_1) + ... in input order, in float: additions only, so a CPU replay
//     (oracle/program_interp.py) is bitwise equal.  An impossible row (every w = -inf) decodes to state 0; its
//     max log P(x, e), in the program's p_slot, is -inf.
#pragma once
#include "sbn_kernels.cuh"
#include "sbn_sample.cuh"

__global__ void __launch_bounds__(SBN_SAMPLE_THREADS) sbn_argmax_step(const __grid_constant__ SbnSample p) {
    extern __shared__ __align__(16) float s_tab[];
    __shared__ __align__(8) uint64_t s_bar;
    sbn_pdl_entry();
    const bool staged = sbn_decode_stage(p, s_tab, &s_bar);

    const int64_t b = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    const bool live = b < p.n_rows;
    if (staged) sbn_mbar_wait(&s_bar, 0);
    if (!live) return;

    const float *src[SBN_MAX_IN];
    int64_t mul[SBN_MAX_IN];
    sbn_decode_operands<float>(p, s_tab, b, 0, src, mul);
    const int n_in = p.n_in, cz = p.cz;
    auto weight = [&](int z) {
        float w = 0.f;
#pragma unroll
        for (int i = 0; i < SBN_MAX_IN; ++i)
            if (i < n_in) w += src[i][static_cast<int64_t>(__ldg(p.zoff + static_cast<int64_t>(i) * cz + z)) * mul[i]];
        return w;
    };
    float best = weight(0);
    int pick = 0;
    for (int z = 1; z < cz; ++z) {
        const float w = weight(z);
        if (w > best) {
            best = w;
            pick = z;
        }
    }
    for (int j = 0; j < p.n_x; ++j) {
        const int c = p.x_card[j];
        p.drawn[static_cast<int64_t>(p.d_first + j) * p.ld_drawn + b] = static_cast<uint8_t>(pick % c);
        pick /= c;
    }
}

inline cudaError_t sbn_argmax_launch(const SbnSample &s, size_t smem, cudaStream_t stream) {
    const dim3 grid(static_cast<unsigned>((s.n_rows + SBN_SAMPLE_THREADS - 1) / SBN_SAMPLE_THREADS));
    sbn_argmax_step<<<grid, SBN_SAMPLE_THREADS, smem, stream>>>(s);
    return cudaGetLastError();
}

inline cudaError_t sbn_argmax_set_attrs() {
    return cudaFuncSetAttribute(sbn_argmax_step, cudaFuncAttributeMaxDynamicSharedMemorySize, SBN_SMEM_BUDGET);
}
