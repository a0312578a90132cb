// sorobn_b200 -- sm_90a kernels for the factor-product / sum-out step.
//
// One launch computes, for every output entry o and evidence row b,
//
//     out[o, b] = sum_x prod_i in_i[ off_i(o) + x * sx_i + evoff_i(b) ]   (, b)
//
// which fuses `pointwise_mul` (/root/reference/sorobn/bayes_net.py:253-256: an
// index join per pair of factors) with `sum_out` (bayes_net.py:54-103: a groupby-sum)
// and with the evidence filter of bayes_net.py:772-774 (here a per-row gather).
//
// Data layout (DESIGN.md "HBM layout"):
//   * batched factor  : float [scope..., ld]  -- evidence rows innermost, ld % 32 == 0,
//                       so a warp reads 128 consecutive rows of one scope entry with
//                       one 128-bit load per lane;
//   * table / shared  : float [scope...]      -- a CPT or an evidence-independent
//                       factor; small ones are staged in shared memory by a bulk-TMA
//                       copy (cp.async.bulk -> SASS UBLKCP) and gathered per lane;
//   * evidence codes  : uint8 [n_ev, ld_ev].
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

#include "../../include/sorobn_b200.h"

#ifndef SBN_FOLD_NORMALISE
#define SBN_FOLD_NORMALISE 0   // 1: normalisation inside the posterior step's epilogue (costs ~10 % on every tiled launch: off)
#endif
#define SBN_THREADS 128      // threads per CTA of the batched kernel (4 rows each)
#define SBN_ROWS_PER_CTA (SBN_THREADS * 4)
#define SBN_SMEM_BUDGET (64 * 1024)   // staged tables of an ordinary launch (several CTAs per SM)
#define SBN_SMEM_BIG (200 * 1024)     // ... of a launch around one big CPT: one CTA per SM

struct SbnInput {
    const float *ptr;                // table / slot base (device)
    int32_t batched;                 // 1: element offsets are in rows (x ld) plus b
    int32_t sx;                      // stride of the eliminated axis
    int32_t n_ev;                    // evidence axes gathered per row
    int32_t smem_off;                // float offset of the staged copy, -1 = read global
    int32_t stage_floats;            // floats copied by the bulk-TMA (multiple of 4)
    int32_t pad_;
    int32_t ev_col[SBN_MAX_EV];
    int32_t ev_stride[SBN_MAX_EV];
    int32_t ev_card[SBN_MAX_EV];     // codes are clamped to card-1 (no out-of-bounds gather)
    int32_t stride[SBN_MAX_AXES];    // stride per output axis (0 = factor lacks the axis)
};

struct SbnStep {
    float *out;
    const uint8_t *ev;
    int64_t ld_ev;
    int64_t ld;          // row pitch of batched buffers (floats), multiple of 32
    int32_t n_rows;      // valid evidence rows (<= ld)
    int32_t n_in;
    int32_t n_axes;
    int32_t cx;          // states of the eliminated variable (1 = product only)
    int32_t n_out;       // prod(card)
    int32_t tile1;       // axis-1 digits handled by one CTA
    int32_t n_tile1;     // ceil(card[1] / tile1)
    int32_t n_bblocks;   // CTAs along the row axis
    int32_t smem_floats; // staged floats in total
    int32_t tiles_per_cta;            // tiled kernel: consecutive tiles one CTA walks
    const int32_t *tile_off;          // tiled kernel: [n_tiles][n_in + 2] = out entry, na | nb << 8, input offsets
    int32_t n_tiles;
    int32_t n_chunks;                 // tiled kernel: ceil(n_tiles / tiles_per_cta)
    const int32_t *zoff;              // several eliminated variables: [n_in][cx] element offsets of
                                      // their joint states (nullptr: one variable, offset = x * sx)
    // slab variant of the tiled kernel (expanding products, see sbn_step_tiled<..., SLAB = true>)
    const int32_t *slab_off;          // [n_slab] element offsets of the A-side slab entries
    int32_t n_slab;                   // cx * slab_ma
    int32_t slab_ma;                  // A-side entries per eliminated state in one slab
    int32_t slab_smem_off;            // float offset of the slab inside dynamic shared memory
    int32_t cx_inner;                 // states of the FIRST eliminated variable (block of the preload schedule)
    const int32_t *slices;            // sliced staging: [n_chunks][n_in][3] = first float, floats, smem offset
    // fused normalisation (tiled kernel, the posterior step when its whole output is ONE tile): instead of
    // storing the un-normalised tile, write posterior / total (range-checked like sbn_normalise) to norm_out
    float *norm_out;                  // [Q][norm_ld], or nullptr
    float *norm_totals;               // P(event) per row, or nullptr
    int64_t norm_ld;
    float norm_min;
    int32_t pad_norm_;
    int32_t card[SBN_MAX_AXES];
    SbnInput in[SBN_MAX_IN];
};

// ------------------------------------------------------------------ PTX helpers
__device__ __forceinline__ uint32_t sbn_smem_u32(const void *p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void sbn_mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(sbn_smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void sbn_fence_mbar_init() {
    // make the init visible to the async (TMA) proxy
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void sbn_mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(sbn_smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void sbn_tma_bulk_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar) {
    // 1-D bulk tensor-memory-accelerator copy global -> shared, completion on mbarrier
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     sbn_smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(sbn_smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void sbn_mbar_wait(uint64_t *bar, uint32_t phase) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(sbn_smem_u32(bar)),
        "r"(phase)
        : "memory");
}

// Programmatic dependent launch (opt-in on the host side): let the next kernel of the stream
// be scheduled as soon as every CTA of this one has started, and do not touch anything a
// predecessor wrote before it has completed.  Both are no-ops for a plain launch.
// Split form: a kernel whose prologue reads only data no launch of the run writes (CPTs, tables computed at
// program creation, tile tables, evidence codes) signals its dependents first, does that prologue -- table staging,
// evidence offsets -- while its predecessor drains, and waits just before it touches a batched factor.
__device__ __forceinline__ void sbn_pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void sbn_pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

__device__ __forceinline__ void sbn_pdl_entry() {
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    asm volatile("griddepcontrol.wait;" ::: "memory");
}

// FMA of two evidence rows held in a register pair.  sm_90 has no packed fp32 FMA, so this is two scalar
// FFMA with the same rounding (one fused multiply-add per row).
__device__ __forceinline__ void sbn_fma2(float (&acc)[2], const float (&a)[2], const float (&b)[2]) {
    acc[0] = fmaf(a[0], b[0], acc[0]);
    acc[1] = fmaf(a[1], b[1], acc[1]);
}

__device__ __forceinline__ float4 sbn_mul4(float4 a, float4 b) {
    return make_float4(a.x * b.x, a.y * b.y, a.z * b.z, a.w * b.w);
}

// Reduction policy of the batched and flat step kernels: how the inputs of one term combine (`times`,
// starting from `one`) and how the terms of the eliminated states reduce (`plus`, starting from `zero`).
// Sum-product is the default of every instantiation.  The policy is an optional trailing template argument
// (SbnPolicy below), so that the sum-product kernels keep their names -- `sbn_step_batched<2, 4>`, as
// profiles and tests/kernel_census.py read them -- and their code.  Max-sum (`out = max_x sum_i in_i`) runs the
// log-domain programs of the most probable explanation (planner.build_mpe_plan): additions and maxima
// only, so there is no FMA to contract and a CPU replay in float32 is bitwise equal.
//
// The kernels reduce through an accumulator: `Acc<T>` starts at `start<T>()`, takes every term with
// `add` and gives the output with `finish` (`Acc4`, `start4`, `add4`, `finish4`: the same for the four rows
// of a float4).  For a semiring (SbnSemiring below) the accumulator is the value itself, `add` is `plus` and
// `finish` returns it, so the sum-product and max-sum kernels compile to the code they had.  Log-sum-exp
// (SbnLogSumExp) needs a running maximum and a rescaled sum.
template <typename R>
struct SbnSemiring {
    template <typename T> using Acc = T;
    template <typename T> static __device__ __forceinline__ T start() { return R::template zero<T>(); }
    template <typename T> static __device__ __forceinline__ void add(T &a, T t) { a = R::plus(a, t); }
    template <typename T> static __device__ __forceinline__ T finish(T a) { return a; }
    using Acc4 = float4;
    static __device__ __forceinline__ float4 start4() {
        const float z = R::template zero<float>();
        return make_float4(z, z, z, z);
    }
    static __device__ __forceinline__ void add4(float4 &a, float4 t) {
        a.x = R::plus(a.x, t.x);
        a.y = R::plus(a.y, t.y);
        a.z = R::plus(a.z, t.z);
        a.w = R::plus(a.w, t.w);
    }
    static __device__ __forceinline__ float4 finish4(float4 a) { return a; }
};
struct SbnSumProduct : SbnSemiring<SbnSumProduct> {
    template <typename T> static __device__ __forceinline__ T one() { return T(1); }
    template <typename T> static __device__ __forceinline__ T zero() { return T(0); }
    template <typename T> static __device__ __forceinline__ T times(T a, T b) { return a * b; }
    template <typename T> static __device__ __forceinline__ T plus(T a, T b) { return a + b; }
    static __device__ __forceinline__ float4 times4(float4 a, float4 b) { return sbn_mul4(a, b); }
};
struct SbnMaxSum : SbnSemiring<SbnMaxSum> {
    template <typename T> static __device__ __forceinline__ T one() { return T(0); }
    template <typename T> static __device__ __forceinline__ T zero() { return static_cast<T>(__int_as_float(0xff800000)); }
    template <typename T> static __device__ __forceinline__ T times(T a, T b) { return a + b; }
    template <typename T> static __device__ __forceinline__ T plus(T a, T b) {
        if constexpr (std::is_same<T, float>::value) return fmaxf(a, b);
        else return fmax(a, b);
    }
    static __device__ __forceinline__ float4 times4(float4 a, float4 b) {
        return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
    }
};
// Log-sum-exp (`out = log sum_x exp(sum_i in_i)`): the buckets of summed-out variables of the marginal MAP
// programs (planner.build_map_plan).  The terms combine as in max-sum; the reduction is online: m is the
// largest term so far and s = sum exp(t - m), rescaled by exp(m_old - m_new) when m grows, and the output is
// m + log(s).  Every exp argument is <= 0, so nothing overflows, and s >= 1 once a term is finite.  A term of
// -inf adds nothing, so a bucket of impossible states gives -inf, never NaN.  expf / logf are the accurate
// library functions (the library is built without fast math).
struct SbnLogSumExp {
    template <typename T> static __device__ __forceinline__ T one() { return T(0); }
    template <typename T> static __device__ __forceinline__ T times(T a, T b) { return a + b; }
    static __device__ __forceinline__ float4 times4(float4 a, float4 b) {
        return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
    }
    template <typename T> struct Acc {
        T m, s;
    };
    template <typename T> static __device__ __forceinline__ T neg_inf() {
        return static_cast<T>(__int_as_float(0xff800000));
    }
    template <typename T> static __device__ __forceinline__ T exp_(T x) {
        if constexpr (std::is_same<T, float>::value) return expf(x);
        else return exp(x);
    }
    template <typename T> static __device__ __forceinline__ T log_(T x) {
        if constexpr (std::is_same<T, float>::value) return logf(x);
        else return log(x);
    }
    template <typename T> static __device__ __forceinline__ Acc<T> start() { return {neg_inf<T>(), T(0)}; }
    template <typename T> static __device__ __forceinline__ void add(Acc<T> &a, T t) {
        if (t > a.m) {
            a.s = a.s * exp_(a.m - t) + T(1);
            a.m = t;
        } else if (t > neg_inf<T>()) {
            a.s += exp_(t - a.m);
        }
    }
    template <typename T> static __device__ __forceinline__ T finish(Acc<T> a) {
        return a.m == neg_inf<T>() ? a.m : a.m + log_(a.s);
    }
    struct Acc4 {
        Acc<float> x, y, z, w;
    };
    static __device__ __forceinline__ Acc4 start4() {
        const Acc<float> a = start<float>();
        return {a, a, a, a};
    }
    static __device__ __forceinline__ void add4(Acc4 &a, float4 t) {
        add(a.x, t.x);
        add(a.y, t.y);
        add(a.z, t.z);
        add(a.w, t.w);
    }
    static __device__ __forceinline__ float4 finish4(const Acc4 &a) {
        return make_float4(finish(a.x), finish(a.y), finish(a.z), finish(a.w));
    }
};
template <typename... R>
struct SbnPolicy {
    using type = SbnSumProduct;
};
template <typename R>
struct SbnPolicy<R> {
    using type = R;
};

// ------------------------------------------------------------- batched step kernel
// The general fallback (more than 4 inputs, two inputs spanning the tile, tables too
// large for shared memory, tile table too large): no limits beyond SBN_MAX_IN / SBN_MAX_AXES.
// Grid: 1-D, blockIdx.x = tile * n_bblocks + bblock (row blocks fastest so that
// neighbouring CTAs stream neighbouring rows of the same scope entries).
// One CTA = 512 evidence rows x one tile of outputs: all card[0] digits of axis 0,
// `tile1` digits of axis 1, one combination of the remaining axes; the mixed-radix
// decomposition of the tile index happens in registers (CTA-uniform).
// Thread = 4 consecutive rows (one float4) looping over the tile, one output per
// iteration; the eliminated axis is reduced in-thread (strided float4 loads, each fully
// coalesced across the warp); operands shared by consecutive outputs are L1 hits.
// Policy: none (sum-product), SbnMaxSum for the log-domain MPE programs, or SbnLogSumExp for the summed
// buckets of the marginal MAP programs.
template <int N_IN, int CX, typename... Policy>
__global__ void __launch_bounds__(SBN_THREADS) sbn_step_batched(const __grid_constant__ SbnStep p) {
    using R = typename SbnPolicy<Policy...>::type;
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
#pragma unroll
            for (int i = 0; i < N_IN; ++i) {
                if (p.in[i].smem_off >= 0) {
                    sbn_tma_bulk_g2s(s_tab + p.in[i].smem_off, p.in[i].ptr,
                                     static_cast<uint32_t>(p.in[i].stage_floats) * 4u, &s_bar);
                }
            }
        }
    }

    const int bblock = blockIdx.x % p.n_bblocks;
    int r = blockIdx.x / p.n_bblocks;  // tile id
    const int b = (bblock * SBN_THREADS + threadIdx.x) * 4;
    const bool live = b < p.n_rows;  // b % 4 == 0: the float4 holds at least one valid row

    const int c0 = p.n_axes > 0 ? p.card[0] : 1;
    const int c1 = p.n_axes > 1 ? p.card[1] : 1;
    const int t1 = r % p.n_tile1;
    r /= p.n_tile1;
    const int d1_begin = t1 * p.tile1;
    const int d1_end = min(c1, d1_begin + p.tile1);
    const int o_rest = r * c0 * c1;  // output is contiguous in axis order

    // mixed-radix digits of the remaining axes -> per-input base offsets (CTA-uniform)
    int off[N_IN];
#pragma unroll
    for (int i = 0; i < N_IN; ++i) off[i] = 0;
    for (int j = 2; j < p.n_axes; ++j) {
        const int c = p.card[j];
        const int d = r % c;
        r /= c;
#pragma unroll
        for (int i = 0; i < N_IN; ++i) off[i] += d * p.in[i].stride[j];
    }

    // per-row evidence offsets of the gathered tables
    int evo[N_IN][4];
#pragma unroll
    for (int i = 0; i < N_IN; ++i) {
        evo[i][0] = evo[i][1] = evo[i][2] = evo[i][3] = 0;
        if (!p.in[i].batched && live) {
            for (int k = 0; k < p.in[i].n_ev; ++k) {
                const uint8_t *col = p.ev + static_cast<int64_t>(p.in[i].ev_col[k]) * p.ld_ev + b;
                const int s = p.in[i].ev_stride[k];
                const int top = p.in[i].ev_card[k] - 1;
#pragma unroll
                for (int l = 0; l < 4; ++l) {
                    const int code = (b + l < p.n_rows) ? min(static_cast<int>(col[l]), top) : 0;
                    evo[i][l] += code * s;
                }
            }
        }
    }

    if (staged) sbn_mbar_wait(&s_bar, 0);
    if (!live) return;

    const int cx = CX > 0 ? CX : p.cx;
    const int64_t ld = p.ld;

    for (int d1 = d1_begin; d1 < d1_end; ++d1) {
        int e0[N_IN];
#pragma unroll
        for (int i = 0; i < N_IN; ++i) e0[i] = off[i] + d1 * (p.n_axes > 1 ? p.in[i].stride[1] : 0);
        for (int d0 = 0; d0 < c0; ++d0) {
            const float o1 = R::template one<float>();
            typename R::Acc4 acc = R::start4();
            auto term = [&](int x) {
                float4 prod = make_float4(o1, o1, o1, o1);
#pragma unroll
                for (int i = 0; i < N_IN; ++i) {
                    const int e = e0[i] + (p.zoff ? __ldg(p.zoff + i * cx + x) : x * p.in[i].sx);
                    float4 v;
                    if (p.in[i].batched) {
                        v = *reinterpret_cast<const float4 *>(p.in[i].ptr + static_cast<int64_t>(e) * ld + b);
                    } else if (p.in[i].smem_off >= 0) {
                        const float *t = s_tab + p.in[i].smem_off + e;
                        v = make_float4(t[evo[i][0]], t[evo[i][1]], t[evo[i][2]], t[evo[i][3]]);
                    } else {
                        const float *t = p.in[i].ptr + e;
                        v = make_float4(__ldg(t + evo[i][0]), __ldg(t + evo[i][1]), __ldg(t + evo[i][2]),
                                        __ldg(t + evo[i][3]));
                    }
                    prod = R::times4(prod, v);
                }
                R::add4(acc, prod);
            };
            if constexpr (CX > 0) {
#pragma unroll
                for (int x = 0; x < CX; ++x) term(x);
            } else {
#pragma unroll 4
                for (int x = 0; x < cx; ++x) term(x);
            }
            *reinterpret_cast<float4 *>(p.out + static_cast<int64_t>(o_rest + d1 * c0 + d0) * ld + b) = R::finish4(acc);
#pragma unroll
            for (int i = 0; i < N_IN; ++i) e0[i] += p.n_axes > 0 ? p.in[i].stride[0] : 0;
        }
    }
}


// --------------------------------------------------- batched step kernel, float64
// The robust fallback for evidence rows below the float32 range (SBN_MIN_TOTAL_F32): same
// contract and grid as sbn_step_batched, scalars are double (tables, scratch and output),
// 2 rows per thread (one 128-bit load), tables read through L1 (no staging).
template <int N_IN>
__global__ void __launch_bounds__(SBN_THREADS) sbn_step_batched_f64(const __grid_constant__ SbnStep p) {
    sbn_pdl_entry();
    const int bblock = blockIdx.x % p.n_bblocks;
    int r = blockIdx.x / p.n_bblocks;  // tile id
    const int b = (bblock * SBN_THREADS + threadIdx.x) * 2;
    if (b >= p.n_rows) return;
    const int c0 = p.n_axes > 0 ? p.card[0] : 1;
    const int c1 = p.n_axes > 1 ? p.card[1] : 1;
    const int t1 = r % p.n_tile1;
    r /= p.n_tile1;
    const int d1_begin = t1 * p.tile1;
    const int d1_end = min(c1, d1_begin + p.tile1);
    const int o_rest = r * c0 * c1;
    int off[N_IN];
#pragma unroll
    for (int i = 0; i < N_IN; ++i) off[i] = 0;
    for (int j = 2; j < p.n_axes; ++j) {
        const int c = p.card[j];
        const int d = r % c;
        r /= c;
#pragma unroll
        for (int i = 0; i < N_IN; ++i) off[i] += d * p.in[i].stride[j];
    }
    int evo[N_IN][2];
#pragma unroll
    for (int i = 0; i < N_IN; ++i) {
        evo[i][0] = evo[i][1] = 0;
        if (!p.in[i].batched) {
            for (int k = 0; k < p.in[i].n_ev; ++k) {
                const uint8_t *col = p.ev + static_cast<int64_t>(p.in[i].ev_col[k]) * p.ld_ev + b;
                const int s = p.in[i].ev_stride[k];
                const int top = p.in[i].ev_card[k] - 1;
#pragma unroll
                for (int l = 0; l < 2; ++l) evo[i][l] += ((b + l < p.n_rows) ? min(static_cast<int>(col[l]), top) : 0) * s;
            }
        }
    }
    const int64_t ld = p.ld;
    double *const out = reinterpret_cast<double *>(p.out);
    for (int d1 = d1_begin; d1 < d1_end; ++d1) {
        for (int d0 = 0; d0 < c0; ++d0) {
            double a0 = 0.0, a1 = 0.0;
            for (int x = 0; x < p.cx; ++x) {
                double p0 = 1.0, p1 = 1.0;
#pragma unroll
                for (int i = 0; i < N_IN; ++i) {
                    const int e = off[i] + d0 * (p.n_axes > 0 ? p.in[i].stride[0] : 0) +
                                  d1 * (p.n_axes > 1 ? p.in[i].stride[1] : 0) +
                                  (p.zoff ? __ldg(p.zoff + i * p.cx + x) : x * p.in[i].sx);
                    const double *src = reinterpret_cast<const double *>(p.in[i].ptr);
                    if (p.in[i].batched) {
                        const double2 v = *reinterpret_cast<const double2 *>(src + static_cast<int64_t>(e) * ld + b);
                        p0 *= v.x;
                        p1 *= v.y;
                    } else {
                        p0 *= __ldg(src + e + evo[i][0]);
                        p1 *= __ldg(src + e + evo[i][1]);
                    }
                }
                a0 += p0;
                a1 += p1;
            }
            *reinterpret_cast<double2 *>(out + static_cast<int64_t>(o_rest + d1 * c0 + d0) * ld + b) = make_double2(a0, a1);
        }
    }
}

// --------------------------------------------------------------- tiled step kernel
// The fast path.  Same contract as sbn_step_batched, different blocking:
//
//   * tile = T digits of output axis 0 x T digits of axis 1 (one combination of the other
//     axes), accumulated in registers for V = 2 consecutive evidence rows per thread;
//   * every input is classed by which of the two tile axes it carries: a factor that lacks
//     axis 0 is loaded once per tile column instead of once per output, one that lacks
//     both once per tile -- the planner orders the axes to minimise these loads
//     (planner.py `_tile_axes`), which turns the 2*cx loads per output of the naive loop
//     into (T + T) * cx per T*T outputs for a product of two batched factors;
//   * the mixed-radix decomposition of the tile index is row-invariant, so it is done
//     once on the host: `tile_off` holds, per tile, the output entry and every input's
//     element offset.  A CTA walks `tiles_per_cta` consecutive tiles for its 256 rows, so
//     operands shared by neighbouring tiles are L1 hits;
//   * tables (CPTs, evidence-independent factors) are staged in shared memory by bulk-TMA
//     and gathered with the row's evidence offset.
template <int V>
struct SbnVec;
template <>
struct SbnVec<2> {
    using type = float2;
};
template <>
struct SbnVec<4> {
    using type = float4;
};

template <int V>
__device__ __forceinline__ void sbn_ldv(float (&r)[V], const float *ptr) {
    const typename SbnVec<V>::type t = *reinterpret_cast<const typename SbnVec<V>::type *>(ptr);
    memcpy(r, &t, sizeof t);
}
// Streaming store (st.global.cs, evict-first): an output is next read by a later launch,
// after hundreds of MB of other traffic, so it should not displace from L2 the operands
// that co-resident CTAs are about to re-read.
template <int V>
__device__ __forceinline__ void sbn_stv(float *ptr, const float (&r)[V]) {
    typename SbnVec<V>::type t;
    memcpy(&t, r, sizeof t);
    __stcs(reinterpret_cast<typename SbnVec<V>::type *>(ptr), t);
}

#define SBN_TILED_THREADS 128

// Inputs arrive sorted by the host: NU that carry neither tile axis, then NA that carry
// axis 0 only, then NB that carry axis 1 only, then NC (0 or 1) that carries both.  Per
// eliminated state x:
//     a[d0] = prod_U in(x) * prod_A in(x, d0)      T values
//     b[d1] = prod_B in(x, d1)                     T values
//     acc[d0][d1] += a[d0] * b[d1] (* c(x, d0, d1))  T*T FFMA
// An input on the C side is read once per output and per x -- each of its entries exactly
// once overall: that is the streaming operand of a sum-out.
//
// CX > 0 (compile-time number of eliminated states) selects the *preload* schedule: every
// operand of the tile, for all x, is fetched into registers before the first FFMA, so a
// thread keeps CX * (NA * T + NB * T + NU) loads in flight instead of one x-step's worth
// (the kernel is latency-bound otherwise: ~16 warps per SM because of the accumulators).
// With a C-side input (T*T loads per x already) only the x-loop schedule is built.
// When several variables are eliminated at once, x runs over their joint states and the
// per-input element offset comes from `zoff` instead of x * sx; the preload schedule then
// preloads one block of CX states (the first eliminated variable) per joint state of the rest.
//
// SLAB = true is the variant for *expanding* products (both the A-side and the B-side batched
// factor have private axes beyond the tile, e.g. 3125 <- B625 x B625): every A entry is needed
// by several B blocks and vice versa, and the caches do not hold the 250 KB per CTA that would
// take.  Tiles are grouped by the digits the two factors share; for one such group a thread
// first copies ITS rows of the whole A-side slab into its own shared-memory column (no
// barrier: a thread only ever reads back what it wrote), then walks the group's tiles reading
// A from shared memory and B blocks through registers (reloaded only when the block
// changes).  Both factors are then read from HBM exactly once.
template <int NU, int NA, int NB, int NC, int T, int V, int CX, bool SLAB = false, bool MX = false>
__global__ void __launch_bounds__(SBN_TILED_THREADS, (CX > 0 ? ((MX && (NU + NA + NB + NC <= 2 || CX <= 5)) ? 3 : 2) : (NC > 0 ? 3 : 4)))
    sbn_step_tiled(const __grid_constant__ SbnStep p) {
    constexpr int N_IN = NU + NA + NB + NC;
    constexpr int TB = (NB > 0 || NC > 0) ? T : 1;  // no input with axis 1: single-axis output
    constexpr int ROW_WORDS = N_IN + 2 + (SLAB ? 3 : 0);  // int32 per tile_off row
    static_assert(NC <= 1, "one input may span both tile axes");
    static_assert(CX == 0 || NC == 0, "the preload schedule does not cover a C-side input");
    static_assert(!SLAB || (NA == 1 && NB == 1 && NC == 0 && CX > 0), "slab variant: one A, one B, preload");
    static_assert(!MX || (CX > 0 && !SLAB), "MX: several eliminated variables on the preload schedule");
    extern __shared__ __align__(16) float s_tab[];
    __shared__ __align__(8) uint64_t s_bar;
    sbn_pdl_launch_dependents();

    // Tile chunks vary fastest: the CTAs resident at any moment then cover all tiles of a
    // few row blocks, so operands shared between tiles are re-read from L2, not from HBM.
    const int rblock = blockIdx.x / p.n_chunks;
    const int chunk = blockIdx.x % p.n_chunks;

    // Tables are staged whole, or -- when they are too big -- only the part this chunk's tiles
    // touch (p.slices; the planner lays such a table out so that the part is contiguous).
    int tab_off[N_IN];  // shared-memory float offset of element 0 of table i (may be negative)
#pragma unroll
    for (int i = 0; i < N_IN; ++i) tab_off[i] = p.in[i].smem_off;
    const bool staged = p.smem_floats > 0;
    if (staged) {
        if (threadIdx.x == 0) {
            sbn_mbar_init(&s_bar, 1);
            sbn_fence_mbar_init();
        }
        __syncthreads();
        if (p.slices) {
            const int32_t *sl = p.slices + static_cast<int64_t>(chunk) * (N_IN * 3);
            uint32_t total = 0;
#pragma unroll
            for (int i = 0; i < N_IN; ++i) {
                tab_off[i] = __ldg(sl + i * 3 + 2) - __ldg(sl + i * 3);
                total += static_cast<uint32_t>(__ldg(sl + i * 3 + 1)) * 4u;
            }
            if (threadIdx.x == 0) {
                sbn_mbar_expect_tx(&s_bar, total);
#pragma unroll
                for (int i = 0; i < N_IN; ++i) {
                    const int len = __ldg(sl + i * 3 + 1);
                    if (len > 0)
                        sbn_tma_bulk_g2s(s_tab + __ldg(sl + i * 3 + 2), p.in[i].ptr + __ldg(sl + i * 3),
                                         static_cast<uint32_t>(len) * 4u, &s_bar);
                }
            }
        } else if (threadIdx.x == 0) {
            sbn_mbar_expect_tx(&s_bar, static_cast<uint32_t>(p.smem_floats) * 4u);
#pragma unroll
            for (int i = 0; i < N_IN; ++i) {
                if (p.in[i].smem_off >= 0) {
                    sbn_tma_bulk_g2s(s_tab + p.in[i].smem_off, p.in[i].ptr,
                                     static_cast<uint32_t>(p.in[i].stage_floats) * 4u, &s_bar);
                }
            }
        }
    }

    const int b = (rblock * static_cast<int>(blockDim.x) + threadIdx.x) * V;
    const bool live = b < p.n_rows;  // b % V == 0 and ld % 32 == 0: the vector stays inside the pitch

    const float *gsrc[N_IN];  // global, row b (batched inputs)
    int evo[N_IN][V];         // shared-memory float offset of the table copy + this row's evidence offset
#pragma unroll
    for (int i = 0; i < N_IN; ++i) {
        gsrc[i] = p.in[i].ptr + b;
#pragma unroll
        for (int l = 0; l < V; ++l) evo[i][l] = tab_off[i];
        if (!p.in[i].batched && live) {
            for (int k = 0; k < p.in[i].n_ev; ++k) {
                const uint8_t *col = p.ev + static_cast<int64_t>(p.in[i].ev_col[k]) * p.ld_ev + b;
                const int s = p.in[i].ev_stride[k];
                const int top = p.in[i].ev_card[k] - 1;
#pragma unroll
                for (int l = 0; l < V; ++l) {
                    const int code = (b + l < p.n_rows) ? min(static_cast<int>(col[l]), top) : 0;
                    evo[i][l] += code * s;
                }
            }
        }
    }

    if (staged) sbn_mbar_wait(&s_bar, 0);
    if (!live) return;
    // everything above read tables, tile tables and evidence codes only; the batched operands below were written
    // by earlier launches of this run
    sbn_pdl_wait();

    const int ld = static_cast<int>(p.ld);
    const int c0 = p.n_axes > 0 ? p.card[0] : 1;
    const int t_begin = chunk * p.tiles_per_cta;
    const int t_end = min(p.n_tiles, t_begin + p.tiles_per_cta);
    float *const outp = p.out + b;
    const int cx = p.cx;

    // element offset of eliminated state x in input i
    auto xoff = [&](int i, int x) { return p.zoff ? __ldg(p.zoff + i * cx + x) : x * p.in[i].sx; };
    // V rows of input i at element offset e
    auto fetch = [&](int i, int e, float (&r)[V]) {
        if (p.in[i].batched) {
            sbn_ldv<V>(r, gsrc[i] + static_cast<int64_t>(e) * ld);
        } else {
#pragma unroll
            for (int l = 0; l < V; ++l) r[l] = s_tab[evo[i][l] + e];
        }
    };

    // slab state: this thread's column of the A-side slab, the B block kept in registers
    float *const slab = s_tab + p.slab_smem_off + threadIdx.x * V;
    const int slab_pitch = static_cast<int>(blockDim.x) * V;  // floats between consecutive slab entries
    int cur_slab = -1, cur_bblock = -1;
    float rb_keep[SLAB ? CX : 1][SLAB ? TB : 1][V];

    for (int t = t_begin; t < t_end; ++t) {
        const int32_t *row = p.tile_off + static_cast<int64_t>(t) * ROW_WORDS;
        const int o_base = __ldg(row);
        const int nab = __ldg(row + 1);
        const int na = nab & 0xff, nb = nab >> 8;
        int base[N_IN];
#pragma unroll
        for (int i = 0; i < N_IN; ++i) base[i] = __ldg(row + 2 + i);
        int a_slab_idx = 0;
        if constexpr (SLAB) {
            const int slab_id = __ldg(row + N_IN + 2);
            a_slab_idx = __ldg(row + N_IN + 3);
            if (slab_id != cur_slab) {
                // copy this thread's rows of the group's A-side slab: global -> registers -> shared
                const int a_super = __ldg(row + N_IN + 4);
                constexpr int i = NU;  // the A-side input
                // asynchronous copies (cp.async -> LDGSTS): no staging registers, every entry of
                // the slab in flight at once; visible to this thread after wait_group
                for (int k = 0; k < p.n_slab; ++k) {
                    const float *src = gsrc[i] + static_cast<int64_t>(a_super + __ldg(p.slab_off + k)) * ld;
                    asm volatile("cp.async.ca.shared.global [%0], [%1], %2;" ::"r"(sbn_smem_u32(slab + k * slab_pitch)),
                                 "l"(src), "n"(V * 4)
                                 : "memory");
                }
                asm volatile("cp.async.commit_group;" ::: "memory");
                asm volatile("cp.async.wait_group 0;" ::: "memory");
                cur_slab = slab_id;
            }
        }

        float acc[T][TB][V];
#pragma unroll
        for (int d0 = 0; d0 < T; ++d0)
#pragma unroll
            for (int d1 = 0; d1 < TB; ++d1)
#pragma unroll
                for (int l = 0; l < V; ++l) acc[d0][d1][l] = 0.f;

        // FULL = whole T x TB tile.  Otherwise digits past the edge re-read the last valid
        // entry (clamped, so every load stays in bounds) and only the stores are predicated.
        auto run_tile = [&](auto full_tag) {
            constexpr bool FULL = decltype(full_tag)::value;
            int k0[T], k1[TB];  // element-offset multipliers of the tile digits
#pragma unroll
            for (int d = 0; d < T; ++d) k0[d] = FULL ? d : min(d, na - 1);
#pragma unroll
            for (int d = 0; d < TB; ++d) k1[d] = FULL ? d : min(d, nb - 1);

            if constexpr (CX > 0) {
              // Several eliminated variables: the first one (CX states, stride sx) is the block
              // that is preloaded, the joint states of the others are walked by `xo` with their
              // offsets from zoff -- the accumulators stay in registers across blocks.
              // (MX = false: one variable, one block -- the loop and the offsets fold away)
              for (int xo = 0; xo < (MX ? cx : 1); xo += CX) {
                int ob[N_IN];
#pragma unroll
                for (int i = 0; i < N_IN; ++i) ob[i] = MX ? base[i] + __ldg(p.zoff + i * cx + xo) : base[i];
                // ---- preload schedule: all loads first ...
                float ra[NA > 0 ? NA : 1][CX][T][V], rb[NB > 0 ? NB : 1][CX][TB][V], ru[NU > 0 ? NU : 1][CX][V];
                if constexpr (SLAB) {
                    // B block: registers, reloaded only when the block changes
                    constexpr int ib = NU + NA;
                    if (base[ib] != cur_bblock) {
                        const int s1 = p.in[ib].stride[1], sx = p.in[ib].sx;
#pragma unroll
                        for (int x = 0; x < CX; ++x)
#pragma unroll
                            for (int d = 0; d < TB; ++d) fetch(ib, base[ib] + x * sx + k1[d] * s1, rb_keep[x][d]);
                        cur_bblock = FULL ? base[ib] : -1;  // a clamped (partial) block is not reusable
                    }
#pragma unroll
                    for (int x = 0; x < CX; ++x)
#pragma unroll
                        for (int d = 0; d < TB; ++d)
#pragma unroll
                            for (int l = 0; l < V; ++l) rb[0][x][d][l] = rb_keep[x][d][l];
                    // A block: this thread's column of the slab
#pragma unroll
                    for (int x = 0; x < CX; ++x)
#pragma unroll
                        for (int d = 0; d < T; ++d) {
                            sbn_ldv<V>(ra[0][x][d], slab + (a_slab_idx + k0[d] + x * p.slab_ma) * slab_pitch);
                        }
                } else {
#pragma unroll
                    for (int j = 0; j < NA; ++j) {
                        const int i = NU + j;
                        const int s0 = p.in[i].stride[0], sx = p.in[i].sx;
#pragma unroll
                        for (int x = 0; x < CX; ++x)
#pragma unroll
                            for (int d = 0; d < T; ++d) fetch(i, ob[i] + x * sx + k0[d] * s0, ra[j][x][d]);
                    }
#pragma unroll
                    for (int j = 0; j < NB; ++j) {
                        const int i = NU + NA + j;
                        const int s1 = p.in[i].stride[1], sx = p.in[i].sx;
#pragma unroll
                        for (int x = 0; x < CX; ++x)
#pragma unroll
                            for (int d = 0; d < TB; ++d) fetch(i, ob[i] + x * sx + k1[d] * s1, rb[j][x][d]);
                    }
                }
#pragma unroll
                for (int i = 0; i < NU; ++i) {
                    const int sx = p.in[i].sx;
#pragma unroll
                    for (int x = 0; x < CX; ++x) fetch(i, ob[i] + x * sx, ru[i][x]);
                }
                // ---- ... then the arithmetic
#pragma unroll
                for (int x = 0; x < CX; ++x) {
                    float a[T][V], bb[TB][V];
#pragma unroll
                    for (int d = 0; d < T; ++d)
#pragma unroll
                        for (int l = 0; l < V; ++l) {
                            float v = 1.f;
#pragma unroll
                            for (int j = 0; j < NA; ++j) v = (j == 0) ? ra[j][x][d][l] : v * ra[j][x][d][l];
#pragma unroll
                            for (int i = 0; i < NU; ++i) v *= ru[i][x][l];
                            a[d][l] = v;
                        }
#pragma unroll
                    for (int d = 0; d < TB; ++d)
#pragma unroll
                        for (int l = 0; l < V; ++l) {
                            float v = 1.f;
#pragma unroll
                            for (int j = 0; j < NB; ++j) v = (j == 0) ? rb[j][x][d][l] : v * rb[j][x][d][l];
                            bb[d][l] = v;
                        }
#pragma unroll
                    for (int d0 = 0; d0 < T; ++d0)
#pragma unroll
                        for (int d1 = 0; d1 < TB; ++d1) {
                            if constexpr (V == 2) {
                                sbn_fma2(acc[d0][d1], a[d0], bb[d1]);
                            } else {
#pragma unroll
                                for (int l = 0; l < V; ++l) acc[d0][d1][l] = fmaf(a[d0][l], bb[d1][l], acc[d0][d1][l]);
                            }
                        }
                }
              }
            } else {
#pragma unroll 2
                for (int x = 0; x < cx; ++x) {
                    float a[T][V], bb[TB][V];
#pragma unroll
                    for (int d = 0; d < T; ++d)
#pragma unroll
                        for (int l = 0; l < V; ++l) a[d][l] = 1.f;
#pragma unroll
                    for (int d = 0; d < TB; ++d)
#pragma unroll
                        for (int l = 0; l < V; ++l) bb[d][l] = 1.f;
                    // ---- C side first: the largest batch of independent loads
                    float rc[NC > 0 ? T : 1][NC > 0 ? TB : 1][V];
                    if constexpr (NC > 0) {
                        constexpr int i = NU + NA + NB;
                        const int e = base[i] + xoff(i, x);
                        const int s0 = p.in[i].stride[0], s1 = p.in[i].stride[1];
#pragma unroll
                        for (int d0 = 0; d0 < T; ++d0)
#pragma unroll
                            for (int d1 = 0; d1 < TB; ++d1) fetch(i, e + k0[d0] * s0 + k1[d1] * s1, rc[d0][d1]);
                    }
                    // ---- A side
#pragma unroll
                    for (int j = 0; j < NA; ++j) {
                        const int i = NU + j;
                        const int e = base[i] + xoff(i, x);
                        const int s0 = p.in[i].stride[0];
                        float r[T][V];
#pragma unroll
                        for (int d = 0; d < T; ++d) fetch(i, e + k0[d] * s0, r[d]);
#pragma unroll
                        for (int d = 0; d < T; ++d)
#pragma unroll
                            for (int l = 0; l < V; ++l) a[d][l] *= r[d][l];
                    }
                    // ---- U side folds into a[]
#pragma unroll
                    for (int i = 0; i < NU; ++i) {
                        float r[V];
                        fetch(i, base[i] + xoff(i, x), r);
#pragma unroll
                        for (int d = 0; d < T; ++d)
#pragma unroll
                            for (int l = 0; l < V; ++l) a[d][l] *= r[l];
                    }
                    // ---- B side
#pragma unroll
                    for (int j = 0; j < NB; ++j) {
                        const int i = NU + NA + j;
                        const int e = base[i] + xoff(i, x);
                        const int s1 = p.in[i].stride[1];
                        float r[TB][V];
#pragma unroll
                        for (int d = 0; d < TB; ++d) fetch(i, e + k1[d] * s1, r[d]);
#pragma unroll
                        for (int d = 0; d < TB; ++d)
#pragma unroll
                            for (int l = 0; l < V; ++l) bb[d][l] *= r[d][l];
                    }
                    // ---- outer product into the accumulators
#pragma unroll
                    for (int d0 = 0; d0 < T; ++d0)
#pragma unroll
                        for (int d1 = 0; d1 < TB; ++d1) {
                            if constexpr (NC == 0 && V == 2) {
                                sbn_fma2(acc[d0][d1], a[d0], bb[d1]);
                            } else {
#pragma unroll
                                for (int l = 0; l < V; ++l) {
                                    if constexpr (NC > 0)
                                        acc[d0][d1][l] = fmaf(a[d0][l] * bb[d1][l], rc[d0][d1][l], acc[d0][d1][l]);
                                    else
                                        acc[d0][d1][l] = fmaf(a[d0][l], bb[d1][l], acc[d0][d1][l]);
                                }
                            }
                        }
                }
            }
#if SBN_FOLD_NORMALISE
            if (p.norm_out != nullptr) {
                // The tile IS the row's whole posterior: posterior / posterior.sum() (bayes_net.py:789-790)
                // here, same summation order and range check as sbn_normalise (SBN_MIN_TOTAL_F32).
                float total[V], lo[V];
#pragma unroll
                for (int l = 0; l < V; ++l) {
                    total[l] = 0.f;
                    lo[l] = p.norm_min;
                }
#pragma unroll
                for (int d1 = 0; d1 < TB; ++d1)
#pragma unroll
                    for (int d0 = 0; d0 < T; ++d0)
                        if (FULL || (d0 < na && d1 < nb)) {
#pragma unroll
                            for (int l = 0; l < V; ++l) {
                                const float v = acc[d0][d1][l];
                                total[l] += v;
                                if (v > 0.f && v < lo[l]) lo[l] = v;
                            }
                        }
                const float nan = __int_as_float(0x7fc00000);
#pragma unroll
                for (int l = 0; l < V; ++l) {
                    if (b + l >= p.n_rows) continue;
                    const bool ok = total[l] >= p.norm_min && lo[l] >= p.norm_min;  // false for NaN too
                    if (p.norm_totals) p.norm_totals[b + l] = ok ? total[l] : nan;
#pragma unroll
                    for (int d1 = 0; d1 < TB; ++d1)
#pragma unroll
                        for (int d0 = 0; d0 < T; ++d0)
                            if (FULL || (d0 < na && d1 < nb))
                                p.norm_out[static_cast<int64_t>(o_base + d1 * c0 + d0) * p.norm_ld + b + l] = ok ? acc[d0][d1][l] / total[l] : nan;
                }
                return;
            }
#endif
#pragma unroll
            for (int d1 = 0; d1 < TB; ++d1)
#pragma unroll
                for (int d0 = 0; d0 < T; ++d0)
                    if (FULL || (d0 < na && d1 < nb))
                        sbn_stv<V>(outp + static_cast<int64_t>(o_base + d1 * c0 + d0) * ld, acc[d0][d1]);
        };
        if (na == T && nb == TB) {
            run_tile(std::true_type{});
        } else {
            run_tile(std::false_type{});
        }
    }
}

// ---------------------------------------------------------------- flat step kernel
// Evidence-independent factors (and single-row "flat" programs): one thread per
// output entry, mixed-radix decomposition of the entry index in registers, the
// eliminated axis reduced in-thread.  Evidence offsets are uniform (row 0).
// T = float inside batched programs, double for single-event programs (those are
// launch-latency bound, so they get the reference's own precision and range for free).
// Policy: the reduction policy, as for sbn_step_batched.
template <typename T, typename... Policy>
__global__ void __launch_bounds__(256) sbn_step_flat(const __grid_constant__ SbnStep p) {
    using R = typename SbnPolicy<Policy...>::type;
    sbn_pdl_entry();
    const int64_t o = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (o >= p.n_out) return;
    int off[SBN_MAX_IN];
#pragma unroll
    for (int i = 0; i < SBN_MAX_IN; ++i) {
        off[i] = 0;
        if (i < p.n_in) {
            for (int k = 0; k < p.in[i].n_ev; ++k)
                off[i] += min(static_cast<int>(p.ev[static_cast<int64_t>(p.in[i].ev_col[k]) * p.ld_ev]),
                              p.in[i].ev_card[k] - 1) *
                          p.in[i].ev_stride[k];
        }
    }
    int r = static_cast<int>(o);
    for (int j = 0; j < p.n_axes; ++j) {
        const int c = p.card[j];
        const int d = r % c;
        r /= c;
#pragma unroll
        for (int i = 0; i < SBN_MAX_IN; ++i)
            if (i < p.n_in) off[i] += d * p.in[i].stride[j];
    }
    typename R::template Acc<T> acc = R::template start<T>();
    for (int x = 0; x < p.cx; ++x) {
        T prod = R::template one<T>();
#pragma unroll
        for (int i = 0; i < SBN_MAX_IN; ++i)
            if (i < p.n_in)
                prod = R::times(prod, __ldg(reinterpret_cast<const T *>(p.in[i].ptr) + off[i] +
                                            (p.zoff ? __ldg(p.zoff + i * p.cx + x) : x * p.in[i].sx)));
        R::add(acc, prod);
    }
    reinterpret_cast<T *>(p.out)[o] = R::finish(acc);
}

// ---------------------------------------------------------------------- normalise
// posterior[q, b] = post[q, b] / sum_q post[q, b]   (bayes_net.py:789-790)
// One thread per evidence row; reads are coalesced across rows for every q.
// A row is written as NaN -- the caller re-runs it in float64 (BayesNet.query_many does) or
// treats it as impossible evidence -- when its normaliser, or its smallest NON-ZERO
// un-normalised entry, is below SBN_MIN_TOTAL (zero / NaN normalisers included).
// Why 1e-30: every factor entry is <= 1, so an addend that contributes more than 1e-7 of an
// entry E >= 1e-30 is itself >= 1e-37, a normal fp32 number carrying full precision; what
// underflowed on the way is bounded by ~1e5 operations x 1.4e-45 (the denormal quantum)
// = 1e-40 absolute, 1e-10 relative to E.  The bound is checked per ENTRY, not only on the
// total: the stated tolerance is 1e-6 relative on every posterior entry, and an entry of
// 1e-37 next to a total of 1e-28 (posterior 1e-9) would carry two or three digits.
// What this cannot see is an entry that underflowed to exactly 0 (true value < 1.4e-45 with a
// total >= 1e-30, i.e. a posterior below 1.4e-15): it is reported as the structural zero it is
// indistinguishable from; `BayesNet.query` (one event) always runs in float64.
#define SBN_MIN_TOTAL_F32 1e-30f

template <typename T>
__global__ void __launch_bounds__(256)
sbn_normalise(const T *__restrict__ post, int64_t ld, int post_batched, int Q, T *__restrict__ out, int64_t ld_out,
              int n_rows, T min_total, T *__restrict__ totals) {
    const int64_t b = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (b >= n_rows) return;
    const int64_t pitch = post_batched ? ld : 1;
    const int64_t base = post_batched ? b : 0;
    T total = T(0), lo = min_total;  // lo: smallest non-zero entry, if any is below min_total
    for (int q = 0; q < Q; ++q) {
        const T v = post[q * pitch + base];
        total += v;
        if (v > T(0) && v < lo) lo = v;
    }
    // the normaliser is P(event) for this row (bayes_net.py:790 divides by it; predict_proba,
    // bayes_net.py:934, returns it); out of range it is reported as NaN like the posterior
    const bool ok = total >= min_total && lo >= min_total;  // false for NaN too
    const T nan = static_cast<T>(__int_as_float(0x7fc00000));
    if (totals) totals[b] = ok ? total : nan;
    for (int q = 0; q < Q; ++q) out[q * ld_out + b] = ok ? post[q * pitch + base] / total : nan;
}
