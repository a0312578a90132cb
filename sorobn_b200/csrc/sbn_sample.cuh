// sorobn_b200 -- sm_90a sample step of sample programs (planner.py KIND_SAMPLE = 4): backward sampling.
//
// One launch draws, for every (row b, draw d), the joint state X of ONE bucket's eliminated variables:
//
//     w(z) = prod_i in_i[ zoff_i(z) + termoff_i(b, d) ]        z = 0 .. cz - 1 (first variable fastest)
//
// where termoff gathers the row's observed codes and the codes of the variables earlier steps drew for
// (b, d) -- the bucket's separator -- and picks z with probability w(z) / sum_z w(z).  The bucket belief
// is never materialised: the upward pass left its factors in the slot arena.
//
//   * one thread = one (row, draw); rows innermost (blockIdx.x), draws on blockIdx.y (and + gridDim.y beyond
//     65535 draws): a warp reads 32 consecutive rows of one operand entry when their drawn separators agree;
//   * `zoff` ([n_in][cz]) is the row-invariant part of every operand's offset, built on the host; a
//     batched operand's gathered offset is multiplied by the row pitch;
//   * the arithmetic is fixed, so that a CPU replay (oracle/program_interp.py) follows it exactly: w(z) is
//     the product of the entries in input order in T (multiplies only); the total and the cumulative sums
//     are double sums in z order.  The pick is the first z with cum(z) > u * total, else the last z with
//     w(z) > 0.  The weights are walked twice (the total, then the cumulative sums) instead of being held:
//     cz reaches 256;
//   * u = ((w0 >> 5) * 2^26 + (w1 >> 6)) * 2^-53, (w0, w1) = the first two words of Philox-4x32-10 with
//     key (seed lo, seed hi) and counter (step, d, row lo, row hi), row = row_base + b.  The seed and
//     row_base are read from device memory, so a captured graph replays with new ones;
//   * tables are staged in shared memory by bulk-TMA when they fit SBN_SMEM_BUDGET (float only);
//   * a total below `min_total` (or zero / NaN) flags the row (flag[b] = 1; every draw of the row writes
//     the same value, so no atomics); the host re-runs flagged rows in float64.
#pragma once
#include "sbn_gibbs.cuh"
#include "sbn_kernels.cuh"

#define SBN_SAMPLE_THREADS 128
#define SBN_SAMPLE_MAX_TERMS 16  // gathered (col stride card) terms per input (planner.SAMPLE_MAX_TERMS)
#define SBN_SAMPLE_MAX_X 8       // variables drawn by one step

struct SbnSampleIn {
    const void *ptr;                 // table / slot base (device), float or double
    int32_t batched;                 // 1: entry e of row b is at e * ld + b
    int32_t n_ev;                    // gathered (col stride card) terms
    int32_t smem_off;                // float offset of the staged copy, -1 = read global
    int32_t stage_floats;
    int32_t ev_col[SBN_SAMPLE_MAX_TERMS];    // < SbnSample::n_ev: evidence column; otherwise drawn-code row
                                             // ev_col - SbnSample::n_ev
    int32_t ev_stride[SBN_SAMPLE_MAX_TERMS];
    int32_t ev_card[SBN_SAMPLE_MAX_TERMS];
};

struct SbnSample {
    const uint8_t *ev;
    int64_t ld_ev;
    uint8_t *drawn;         // [n_sampled][n_draws][ld_drawn]
    int64_t ld_drawn;
    int64_t ld;             // row pitch of batched operands
    const int32_t *zoff;    // [n_in][cz]
    const uint32_t *args;   // seed lo, seed hi, row_base lo, row_base hi
    uint8_t *flag;          // [n_rows]
    double min_total;
    int32_t n_rows;
    int32_t n_draws;
    int32_t n_ev;
    int32_t n_in;
    int32_t cz;             // joint states of the drawn variables
    int32_t n_x;
    int32_t d_first;        // drawn-code row of the first drawn variable
    int32_t step;           // index of this step among the sample steps (Philox counter word 0)
    int32_t smem_floats;
    int32_t x_card[SBN_SAMPLE_MAX_X];
    SbnSampleIn in[SBN_MAX_IN];
};

// The operands of one (row b, draw d) of a sample or argmax step (sbn_mpe.cuh): entry e of operand i is
// src[i][e * mul[i]], the row's observed codes and the codes decoded before this step already gathered.
template <typename T>
__device__ __forceinline__ void sbn_decode_operands(const SbnSample &p, const float *s_tab, int64_t b, int d,
                                                    const T *(&src)[SBN_MAX_IN], int64_t (&mul)[SBN_MAX_IN]) {
#pragma unroll
    for (int i = 0; i < SBN_MAX_IN; ++i) {
        src[i] = nullptr;
        mul[i] = 1;
        if (i < p.n_in) {
            const SbnSampleIn &in = p.in[i];
            int64_t off = 0;
            for (int t = 0; t < in.n_ev; ++t) {
                const int col = in.ev_col[t];
                const int code = col < p.n_ev ? p.ev[static_cast<int64_t>(col) * p.ld_ev + b]
                                               : p.drawn[(static_cast<int64_t>(col - p.n_ev) * p.n_draws + d) * p.ld_drawn + b];
                off += static_cast<int64_t>(min(code, in.ev_card[t] - 1)) * in.ev_stride[t];
            }
            if (in.batched) {
                src[i] = static_cast<const T *>(in.ptr) + b + off * p.ld;
                mul[i] = p.ld;
            } else if constexpr (std::is_same<T, float>::value) {
                src[i] = (in.smem_off >= 0 ? s_tab + in.smem_off : static_cast<const T *>(in.ptr)) + off;
            } else {
                src[i] = static_cast<const T *>(in.ptr) + off;
            }
        }
    }
}

// Stage the launch's tables in shared memory by bulk-TMA (sample and argmax steps).  Returns whether the
// CTA has to wait on `bar` before it reads them.
__device__ __forceinline__ bool sbn_decode_stage(const SbnSample &p, float *s_tab, uint64_t *bar) {
    const bool staged = p.smem_floats > 0;
    if (staged) {
        if (threadIdx.x == 0) {
            sbn_mbar_init(bar, 1);
            sbn_fence_mbar_init();
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            sbn_mbar_expect_tx(bar, static_cast<uint32_t>(p.smem_floats) * 4u);
            for (int i = 0; i < p.n_in; ++i)
                if (p.in[i].smem_off >= 0)
                    sbn_tma_bulk_g2s(s_tab + p.in[i].smem_off, p.in[i].ptr, static_cast<uint32_t>(p.in[i].stage_floats) * 4u,
                                     bar);
        }
    }
    return staged;
}

// One (row b, draw d) of the launch below
template <typename T>
__device__ __forceinline__ void sbn_sample_draw(const SbnSample &p, const float *s_tab, int64_t b, int d) {
    const T *src[SBN_MAX_IN];
    int64_t mul[SBN_MAX_IN];
    sbn_decode_operands<T>(p, s_tab, b, d, src, mul);
    const int n_in = p.n_in, cz = p.cz;
    auto weight = [&](int z) {
        T w = T(1);
        if (n_in > 0) w = src[0][static_cast<int64_t>(__ldg(p.zoff + z)) * mul[0]];
#pragma unroll
        for (int i = 1; i < SBN_MAX_IN; ++i)
            if (i < n_in) w *= src[i][static_cast<int64_t>(__ldg(p.zoff + static_cast<int64_t>(i) * cz + z)) * mul[i]];
        return w;
    };
    double total = 0.0;
    for (int z = 0; z < cz; ++z) total += static_cast<double>(weight(z));

    const uint64_t row = (static_cast<uint64_t>(__ldg(p.args + 3)) << 32 | __ldg(p.args + 2)) + static_cast<uint64_t>(b);
    uint32_t ctr[4] = {static_cast<uint32_t>(p.step), static_cast<uint32_t>(d), static_cast<uint32_t>(row),
                       static_cast<uint32_t>(row >> 32)};
    sbn_philox(ctr, __ldg(p.args + 0), __ldg(p.args + 1));
    const double u = (static_cast<double>(ctr[0] >> 5) * 67108864.0 + static_cast<double>(ctr[1] >> 6)) * (1.0 / 9007199254740992.0);
    const double thr = u * total;

    double cum = 0.0;
    int pick = -1, last_pos = 0;
    for (int z = 0; z < cz; ++z) {
        const T w = weight(z);
        cum += static_cast<double>(w);
        if (w > T(0)) last_pos = z;
        if (cum > thr) {
            pick = z;
            break;
        }
    }
    if (pick < 0) pick = last_pos;
    if (!(total >= p.min_total)) p.flag[b] = 1;  // NaN too

    for (int j = 0; j < p.n_x; ++j) {
        const int c = p.x_card[j];
        p.drawn[(static_cast<int64_t>(p.d_first + j) * p.n_draws + d) * p.ld_drawn + b] = static_cast<uint8_t>(pick % c);
        pick /= c;
    }
}

template <typename T>
__global__ void __launch_bounds__(SBN_SAMPLE_THREADS) sbn_sample_step(const __grid_constant__ SbnSample p) {
    extern __shared__ __align__(16) float s_tab[];
    __shared__ __align__(8) uint64_t s_bar;
    sbn_pdl_entry();
    const bool staged = sbn_decode_stage(p, s_tab, &s_bar);

    const int64_t b = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    const bool live = b < p.n_rows;
    if (staged) sbn_mbar_wait(&s_bar, 0);
    if (!live) return;
    for (int d = blockIdx.y; d < p.n_draws; d += gridDim.y) sbn_sample_draw<T>(p, s_tab, b, d);
}

// The run's per-row output: P(observed), NaN where it is out of range or a sample step flagged the row
template <typename T>
__global__ void sbn_sample_prob(const T *__restrict__ prob, int32_t prob_batched, const uint8_t *__restrict__ flag,
                                int32_t n_rows, double min_total, T *__restrict__ out) {
    const int64_t b = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (b >= n_rows) return;
    const T v = prob[prob_batched ? b : 0];
    out[b] = static_cast<double>(v) >= min_total && !flag[b] ? v : static_cast<T>(__int_as_float(0x7fc00000));
}

template <typename T>
inline cudaError_t sbn_sample_launch(const SbnSample &s, size_t smem, cudaStream_t stream) {
    const dim3 grid(static_cast<unsigned>((s.n_rows + SBN_SAMPLE_THREADS - 1) / SBN_SAMPLE_THREADS),
                    static_cast<unsigned>(std::min(s.n_draws, 65535)));
    sbn_sample_step<T><<<grid, SBN_SAMPLE_THREADS, smem, stream>>>(s);
    return cudaGetLastError();
}

inline cudaError_t sbn_sample_set_attrs() {
    return cudaFuncSetAttribute(sbn_sample_step<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, SBN_SMEM_BUDGET);
}
