// sorobn_b200 -- row-block join kernel (see sbn_join.h).
#include "sbn_join.h"

#include <cuda.h>

#include <algorithm>
#include <cstring>

#include "sbn_internal.h"
#include "sbn_kernels.cuh"
#include "sbn_launch.h"
#include "sbn_tma.h"

namespace {

constexpr int kT = 5;            // tile edge = states of the first eliminated variable (the MX block)
constexpr int kSmemMax = 220 * 1024;

struct SbnJoinParams {
    CUtensorMap tm[SBN_JOIN_MAX_BATCHED];  // batched operands, see sbn_tma_encode_rows
    SbnStep s;                             // the step as build_params() lays it out for the tiled kernel
    int32_t boff[SBN_MAX_IN];              // batched input i: float offset of its block inside a stage
    int32_t map_in[SBN_JOIN_MAX_BATCHED];  // input of each tensor map
    int32_t n_maps;
    int32_t rows;                          // R: evidence rows per block
    int32_t stage_floats;                  // multiple of 32 (128-byte aligned stages)
    uint32_t stage_bytes;                  // bytes the boxes of one stage deliver
    int32_t n_blocks;                      // ceil(n_rows / R)
};

__device__ __forceinline__ void tma_3d(float *dst, const CUtensorMap *map, int32_t row, uint64_t *bar) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %4}], [%2];" ::"r"(
                     sbn_smem_u32(dst)),
                 "l"(reinterpret_cast<uint64_t>(map)), "r"(sbn_smem_u32(bar)), "r"(row), "r"(0)
                 : "memory");
}

// Inputs in the tiled kernel's order: NU without a tile axis, NA with axis 0, NB with axis 1.
// Dynamic shared memory: [stage 0][stage 1][tables]; a stage holds, per batched input, [entry][R rows].
template <int NU, int NA, int NB>
__global__ void __launch_bounds__(SBN_JOIN_MAX_THREADS, 1) sbn_join_kernel(const __grid_constant__ SbnJoinParams p) {
    constexpr int T = kT, CX = kT, S = SBN_JOIN_STAGES;
    constexpr int N_IN = NU + NA + NB;
    constexpr int TB = NB > 0 ? T : 1;
    constexpr int ROW_WORDS = N_IN + 2;
    const SbnStep &s = p.s;
    extern __shared__ __align__(128) float s_mem[];
    __shared__ __align__(8) uint64_t s_full[S], s_tab;
    sbn_pdl_launch_dependents();

    const int R = p.rows;
    float *const tab = s_mem + S * p.stage_floats;
    const bool staged = s.smem_floats > 0;
    if (threadIdx.x == 0) {
#pragma unroll
        for (int k = 0; k < S; ++k) sbn_mbar_init(&s_full[k], 1);
        sbn_mbar_init(&s_tab, 1);
        sbn_fence_mbar_init();
    }
    __syncthreads();
    if (threadIdx.x == 0 && staged) {
        sbn_mbar_expect_tx(&s_tab, static_cast<uint32_t>(s.smem_floats) * 4u);
#pragma unroll
        for (int i = 0; i < N_IN; ++i)
            if (!s.in[i].batched) sbn_tma_bulk_g2s(tab + s.in[i].smem_off, s.in[i].ptr, static_cast<uint32_t>(s.in[i].stage_floats) * 4u, &s_tab);
    }
    auto issue = [&](int stage, int blk) {
        float *const dst = s_mem + stage * p.stage_floats;
        sbn_mbar_expect_tx(&s_full[stage], p.stage_bytes);
        for (int m = 0; m < p.n_maps; ++m) tma_3d(dst + p.boff[p.map_in[m]], &p.tm[m], blk * R, &s_full[stage]);
    };
    // tables and tile tables are not written by any launch of the run; the batched operands and the output are
    sbn_pdl_wait();
    if (threadIdx.x == 0)
        for (int k = 0; k < S; ++k)
            if (blockIdx.x + k * gridDim.x < p.n_blocks) issue(k, blockIdx.x + k * gridDim.x);

    // thread = (row r of the block, tile t); the tile's offsets do not change from block to block
    const int r = threadIdx.x % R, t = threadIdx.x / R;
    const int32_t *const row = s.tile_off + static_cast<int64_t>(t) * ROW_WORDS;
    const int o_base = __ldg(row);
    int base[N_IN];
#pragma unroll
    for (int i = 0; i < N_IN; ++i) base[i] = __ldg(row + 2 + i);
    const int c0 = s.card[0];
    const int cx = s.cx;
    if (staged) sbn_mbar_wait(&s_tab, 0);

    for (int it = 0, blk = blockIdx.x; blk < p.n_blocks; ++it, blk += gridDim.x) {
        const int stage = it % S;
        const int b = blk * R + r;
        const bool live = b < s.n_rows;
        // per input: where element e of this row lives -- src[i] + e * mul[i]
        const float *src[N_IN];
        int mul[N_IN];
        const float *const stg = s_mem + stage * p.stage_floats;
#pragma unroll
        for (int i = 0; i < N_IN; ++i) {
            if (s.in[i].batched) {
                src[i] = stg + p.boff[i] + r;
                mul[i] = R;
            } else {
                int e = s.in[i].smem_off;
                for (int k = 0; k < s.in[i].n_ev; ++k) {
                    const int code = live ? min(static_cast<int>(s.ev[static_cast<int64_t>(s.in[i].ev_col[k]) * s.ld_ev + b]), s.in[i].ev_card[k] - 1) : 0;
                    e += code * s.in[i].ev_stride[k];
                }
                src[i] = tab + e;
                mul[i] = 1;
            }
        }
        sbn_mbar_wait(&s_full[stage], static_cast<uint32_t>((it / S) & 1));

        // the tiled kernel's MX schedule, operation for operation (sbn_step_tiled<..., MX = true>)
        float acc[T][TB];
#pragma unroll
        for (int d0 = 0; d0 < T; ++d0)
#pragma unroll
            for (int d1 = 0; d1 < TB; ++d1) acc[d0][d1] = 0.f;
        for (int xo = 0; xo < cx; xo += CX) {
            int ob[N_IN];
#pragma unroll
            for (int i = 0; i < N_IN; ++i) ob[i] = base[i] + __ldg(s.zoff + i * cx + xo);
#pragma unroll
            for (int x = 0; x < CX; ++x) {
                float a[T], bb[TB];
#pragma unroll
                for (int d = 0; d < T; ++d) {
                    float v = 1.f;
#pragma unroll
                    for (int j = 0; j < NA; ++j) {
                        const int i = NU + j;
                        const float r_ = src[i][(ob[i] + x * s.in[i].sx + d * s.in[i].stride[0]) * mul[i]];
                        v = (j == 0) ? r_ : v * r_;
                    }
#pragma unroll
                    for (int i = 0; i < NU; ++i) v *= src[i][(ob[i] + x * s.in[i].sx) * mul[i]];
                    a[d] = v;
                }
#pragma unroll
                for (int d = 0; d < TB; ++d) {
                    float v = 1.f;
#pragma unroll
                    for (int j = 0; j < NB; ++j) {
                        const int i = NU + NA + j;
                        const float r_ = src[i][(ob[i] + x * s.in[i].sx + d * s.in[i].stride[1]) * mul[i]];
                        v = (j == 0) ? r_ : v * r_;
                    }
                    bb[d] = v;
                }
#pragma unroll
                for (int d0 = 0; d0 < T; ++d0)
#pragma unroll
                    for (int d1 = 0; d1 < TB; ++d1) acc[d0][d1] = fmaf(a[d0], bb[d1], acc[d0][d1]);
            }
        }
        if (live) {
#pragma unroll
            for (int d1 = 0; d1 < TB; ++d1)
#pragma unroll
                for (int d0 = 0; d0 < T; ++d0) __stcs(s.out + static_cast<int64_t>(o_base + d1 * c0 + d0) * s.ld + b, acc[d0][d1]);
        }
        // every thread is done with this stage: refill it with the block S steps ahead
        __syncthreads();
        if (threadIdx.x == 0 && blk + S * static_cast<int>(gridDim.x) < p.n_blocks) issue(stage, blk + S * gridDim.x);
    }
}

// The input combinations of the tiled kernel's preload schedule (launch_tiled): at most three inputs, or
// two without a tile axis beside one per axis.
#define SBN_JOIN_COMBOS(X) \
    X(0, 1, 0) X(0, 1, 1) X(0, 1, 2) X(0, 2, 0) X(0, 2, 1) X(1, 1, 0) X(1, 1, 1) X(1, 2, 0) X(2, 1, 0) X(2, 1, 1)

bool instantiated(int nu, int na, int nb) {
#define SBN_JOIN_HAS(U, A, B) \
    if (nu == U && na == A && nb == B) return true;
    SBN_JOIN_COMBOS(SBN_JOIN_HAS)
#undef SBN_JOIN_HAS
    return false;
}

struct JoinShape {
    int rows = 0;
    int stage_floats = 0;
    uint32_t stage_bytes = 0;
    size_t smem = 0;
    int32_t boff[SBN_MAX_IN] = {};
    int e_lo[SBN_MAX_IN] = {};
};

// largest divisor of n that is <= 256 and leaves a quotient <= 256 (the two entry dimensions of a box), or 0
int split_entries(int64_t n) {
    for (int d = 256; d >= 1; --d)
        if (n % d == 0) return n / d <= 256 ? d : 0;
    return 0;
}

bool shape_of(const sbn_program *P, const StepDesc &st, const SbnStep &q, JoinShape *js) {
    if (P->f64 || !P->use_tiled || !P->use_preload) return false;
    // the tiled kernel's MX instantiation (launch_tiled_c): tile edge 5 = states of the first eliminated variable,
    // joint-state offsets, no slab, no slices, no folded normalisation
    if (st.kind != 1 || st.tile != kT || st.nc != 0 || q.tile_off == nullptr || q.zoff == nullptr || q.cx_inner != kT || q.cx % kT != 0)
        return false;
    if (q.slab_off != nullptr || q.slices != nullptr || q.norm_out != nullptr) return false;
    if (!(st.in.size() <= 3 || (st.nu == 2 && st.na == 1 && st.nb == 1)) || !instantiated(st.nu, st.na, st.nb)) return false;
    // whole tiles only (the tiled kernel's FULL path)
    const int64_t n_tiles = st.n_tiles;
    const int tb = st.nb > 0 ? kT : 1;
    for (int64_t t = 0; t < n_tiles; ++t)
        if (P->h_tile_words[static_cast<size_t>(st.tile_off_pos + t * (q.n_in + 2) + 1)] != (kT | tb << 8)) return false;
    // R rows x n_tiles threads: enough of them to keep the SM busy, one CTA per SM
    const int rows = n_tiles * 16 >= 128 ? 16 : 32;
    if (n_tiles * rows < 128 || n_tiles * rows > SBN_JOIN_MAX_THREADS) return false;
    int n_batched = 0;
    int64_t stage = 0;
    for (int i = 0; i < q.n_in; ++i) {
        const InDesc &in = st.in[st.order[i]];
        if (!in.batched) {
            if (q.in[i].smem_off < 0) return false;  // every table staged whole
            continue;
        }
        if (++n_batched > SBN_JOIN_MAX_BATCHED) return false;
        const int64_t n_e = P->slots[in.id].size;
        js->e_lo[i] = split_entries(n_e);
        if (js->e_lo[i] == 0) return false;
        js->boff[i] = static_cast<int32_t>(stage);
        stage += round_up(n_e * rows, 32);
        js->stage_bytes += static_cast<uint32_t>(n_e * rows * 4);
    }
    if (n_batched != SBN_JOIN_MAX_BATCHED) return false;
    js->rows = rows;
    js->stage_floats = static_cast<int>(stage);
    js->smem = static_cast<size_t>(SBN_JOIN_STAGES * stage + q.smem_floats) * 4;
    if (js->smem > kSmemMax) return false;
    // enough row blocks for two per SM: below that the tiled kernel's many small CTAs fill the GPU better
    return q.n_rows >= 2LL * P->n_sms * rows;
}

template <int NU, int NA, int NB>
cudaError_t set_attr() {
    return cudaFuncSetAttribute(sbn_join_kernel<NU, NA, NB>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemMax);
}

}  // namespace

int sbn_join_rows(const sbn_program *P, const StepDesc &st, const SbnStep &q) {
    JoinShape js;
    return shape_of(P, st, q, &js) ? js.rows : 0;
}

cudaError_t sbn_join_set_attrs() {
    cudaError_t e = cudaSuccess;
#define SBN_JOIN_ATTR(U, A, B) \
    if (e == cudaSuccess) e = set_attr<U, A, B>();
    SBN_JOIN_COMBOS(SBN_JOIN_ATTR)
#undef SBN_JOIN_ATTR
    return e;
}

cudaError_t sbn_join_launch(sbn_program *P, const StepDesc &st, const SbnStep &q, cudaStream_t stream) {
    JoinShape js;
    if (!shape_of(P, st, q, &js)) return cudaErrorInvalidValue;
    SbnJoinParams p;
    memset(&p, 0, sizeof p);
    p.s = q;
    p.rows = js.rows;
    p.stage_floats = js.stage_floats;
    p.stage_bytes = js.stage_bytes;
    p.n_blocks = static_cast<int32_t>((q.n_rows + js.rows - 1) / js.rows);
    for (int i = 0; i < q.n_in; ++i) {
        p.boff[i] = js.boff[i];
        if (!q.in[i].batched) continue;
        const int64_t n_e = P->slots[st.in[st.order[i]].id].size;
        if (!sbn_tma_encode_rows(&p.tm[p.n_maps], q.in[i].ptr, q.ld, q.n_rows, n_e, js.rows, js.e_lo[i])) return cudaErrorInvalidValue;
        p.map_in[p.n_maps++] = i;
    }
    const dim3 g(static_cast<unsigned>(std::min<int64_t>(p.n_blocks, P->n_sms))), b(static_cast<unsigned>(js.rows * st.n_tiles));
    const int key = st.nu * 100 + st.na * 10 + st.nb;
    switch (key) {
#define SBN_JOIN_CASE(U, A, B)                                                \
    case U * 100 + A * 10 + B:                                                \
        sbn_launch(sbn_join_kernel<U, A, B>, g, b, js.smem, stream, p);       \
        break;
        SBN_JOIN_COMBOS(SBN_JOIN_CASE)
#undef SBN_JOIN_CASE
        default: return cudaErrorInvalidValue;
    }
    return cudaGetLastError();
}
