// sorobn_b200 -- tensor-map TMA pipeline kernel for the HBM-bound elimination steps (see sbn_tma.h).
#include "sbn_tma.h"

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "sbn_internal.h"

namespace {

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t phase) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(phase)
        : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
// one box of a 2-D tensor map: coordinates (row, entry), completion on the stage's mbarrier
__device__ __forceinline__ void tma_2d(void *dst, const CUtensorMap *map, int32_t c0, int32_t c1, uint64_t *bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
                     smem_u32(dst)),
                 "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
                 : "memory");
}

// a whole operand block of a tile in ONE instruction: box (256 rows, tn tile digits, CX eliminated
// states, 1) of the 4-D view (rows, digit stride, state stride, entry) of the factor
__device__ __forceinline__ void tma_4d(void *dst, const CUtensorMap *map, int32_t c0, int32_t c3, uint64_t *bar) {
    asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %4, %5}], [%2];" ::"r"(
                     smem_u32(dst)),
                 "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(0), "r"(c3)
                 : "memory");
}

// Dynamic shared memory: [stage 0 .. stage S-1 (each stage_floats, 1 KB boxes)] [tables]
template <int T, int CX>
__global__ void __launch_bounds__(SBN_TMA_THREADS, 2) sbn_step_tma(const __grid_constant__ SbnTmaParams p) {
    extern __shared__ __align__(1024) float s_mem[];
    __shared__ __align__(8) uint64_t s_full[SBN_TMA_MAX_STAGES], s_empty[SBN_TMA_MAX_STAGES], s_tab;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int S = p.n_stages;
    float *const tab = s_mem + static_cast<int64_t>(S) * p.stage_floats;

    if (threadIdx.x == 0) {
        for (int s = 0; s < S; ++s) {
            mbar_init(&s_full[s], 1);
            mbar_init(&s_empty[s], SBN_TMA_CONSUMERS);
        }
        mbar_init(&s_tab, 1);
        fence_mbar_init();
    }
    __syncthreads();
    if (threadIdx.x == 0 && p.n_tables > 0) {
        mbar_expect_tx(&s_tab, static_cast<uint32_t>(p.table_floats) * 4u);
        for (int k = 0; k < p.n_tables; ++k) bulk_g2s(tab + p.tab[k].off, p.tab[k].src, static_cast<uint32_t>(p.tab[k].floats) * 4u, &s_tab);
    }

    // contiguous item range of this CTA; item = row block * n_tiles + tile
    const int64_t per = (p.n_items + gridDim.x - 1) / gridDim.x;
    const int64_t i0 = static_cast<int64_t>(blockIdx.x) * per, i1 = min(p.n_items, i0 + per);

    if (warp == SBN_TMA_CONSUMERS) {
        // ------------------------------------------------------------------ producer warp
        int s = 0;
        uint32_t n = 0;  // uses of stage s so far
        for (int64_t i = i0; i < i1; ++i) {
            const int rb = static_cast<int>(i / p.n_tiles), t = static_cast<int>(i - static_cast<int64_t>(rb) * p.n_tiles);
            const int32_t *trow = p.tile_off + static_cast<int64_t>(t) * p.row_words;
            // one stage per block of CX eliminated states (one block unless several variables are summed out)
            for (int blk = 0; blk < p.n_blocks; ++blk) {
                if (n > 0) mbar_wait(&s_empty[s], (n - 1) & 1);
                float *stage = s_mem + static_cast<int64_t>(s) * p.stage_floats;
                if (lane == 0) mbar_expect_tx(&s_full[s], static_cast<uint32_t>(p.n_boxes) * (SBN_TMA_ROWS * 4u));
                __syncwarp();
                if (p.big_boxes) {
                    // one 4-D box per batched operand
                    if (lane < p.n_maps) {
                        int slot = -1, seen = 0;
#pragma unroll
                        for (int q = 0; q < SBN_TMA_SLOTS; q += 2)
                            if (p.in[q].kind == 2) {
                                if (seen == lane && slot < 0) slot = q;
                                ++seen;
                            }
                        const SbnTmaIn &in = p.in[slot];
                        const int boff = p.zoff ? __ldg(p.zoff + in.col * p.cx + blk * CX) : 0;
                        tma_4d(stage + in.off, &p.tm[lane], rb * SBN_TMA_ROWS, __ldg(trow + 2 + in.col) + boff, &s_full[s]);
                    }
                } else
                for (int b = lane; b < p.n_boxes; b += 32) {
                    const int j = b < p.nk0 ? 0 : 1;
                    const int k = j ? b - p.nk0 : b;
                    // the slot of tensor map j: the first batched one in slot order (U0, A0, B0), or the second
                    int slot = -1, seen = 0;
#pragma unroll
                    for (int q = 0; q < SBN_TMA_SLOTS; q += 2)
                        if (p.in[q].kind == 2) {
                            if (seen == j && slot < 0) slot = q;
                            ++seen;
                        }
                    const SbnTmaIn &in = p.in[slot];
                    const int x = k / in.tn, d = k - x * in.tn;
                    const int boff = p.zoff ? __ldg(p.zoff + in.col * p.cx + blk * CX) : 0;
                    const int entry = __ldg(trow + 2 + in.col) + boff + x * in.sx + d * in.sd;
                    tma_2d(stage + in.off + k * SBN_TMA_ROWS, &p.tm[j], rb * SBN_TMA_ROWS, entry, &s_full[s]);
                }
                if (++s == S) {
                    s = 0;
                    ++n;
                }
            }
        }
        return;
    }

    // ---------------------------------------------------------------------- consumer warps
    const int r = (warp * 32 + lane) * 2;  // this thread's two rows inside the item's row block
    int evo[SBN_TMA_SLOTS][2];
    int cur_rb = -1;
    if (p.n_tables > 0) mbar_wait(&s_tab, 0);
    int s = 0;
    uint32_t n = 0;
    for (int64_t i = i0; i < i1; ++i) {
        const int rb = static_cast<int>(i / p.n_tiles), t = static_cast<int>(i - static_cast<int64_t>(rb) * p.n_tiles);
        const int64_t row = static_cast<int64_t>(rb) * SBN_TMA_ROWS + r;
        if (rb != cur_rb) {
            // evidence offsets of the gathered tables for this thread's two rows
            cur_rb = rb;
#pragma unroll
            for (int q = 0; q < SBN_TMA_SLOTS; ++q) {
                evo[q][0] = evo[q][1] = 0;
                if (p.in[q].kind == 1) {
                    evo[q][0] = evo[q][1] = p.in[q].off;
                    for (int e = 0; e < p.in[q].n_ev; ++e) {
                        const uint8_t *colp = p.ev + static_cast<int64_t>(p.in[q].ev_col[e]) * p.ld_ev + row;
                        const int top = p.in[q].ev_card[e] - 1, st = p.in[q].ev_stride[e];
#pragma unroll
                        for (int l = 0; l < 2; ++l) evo[q][l] += (row + l < p.n_rows ? min(static_cast<int>(colp[l]), top) : 0) * st;
                    }
                }
            }
        }
        const int32_t *trow = p.tile_off + static_cast<int64_t>(t) * p.row_words;
        const int o_base = __ldg(trow);
        int base[SBN_TMA_SLOTS];
#pragma unroll
        for (int q = 0; q < SBN_TMA_SLOTS; ++q) base[q] = p.in[q].kind == 1 ? __ldg(trow + 2 + p.in[q].col) : 0;

        float acc[T][T][2];
#pragma unroll
        for (int d0 = 0; d0 < T; ++d0)
#pragma unroll
            for (int d1 = 0; d1 < T; ++d1) acc[d0][d1][0] = acc[d0][d1][1] = 0.f;
      for (int blk = 0; blk < p.n_blocks; ++blk) {
        const float *stage = s_mem + static_cast<int64_t>(s) * p.stage_floats;
        int bbase[SBN_TMA_SLOTS];  // tables: element offset of this block of eliminated states
#pragma unroll
        for (int q = 0; q < SBN_TMA_SLOTS; ++q)
            bbase[q] = base[q] + ((p.zoff && p.in[q].kind == 1) ? __ldg(p.zoff + p.in[q].col * p.cx + blk * CX) : 0);
        mbar_wait(&s_full[s], n & 1);
        // value(s) of slot q for eliminated state x and tile digit d (0 for the U class), both rows
        auto val = [&](int q, int x, int d) -> float2 {
            const SbnTmaIn &in = p.in[q];
            if (in.kind == 2) return *reinterpret_cast<const float2 *>(stage + in.off + (x * in.tn + d) * SBN_TMA_ROWS + r);
            const int e = bbase[q] + x * in.sx + d * in.sd;
            return make_float2(tab[evo[q][0] + e], tab[evo[q][1] + e]);
        };
#pragma unroll
        for (int x = 0; x < CX; ++x) {
            float2 u = make_float2(1.f, 1.f);
            if (p.in[0].kind) u = val(0, x, 0);
            if (p.in[1].kind) {
                const float2 v = val(1, x, 0);
                u.x *= v.x;
                u.y *= v.y;
            }
            float2 a[T], b[T];
#pragma unroll
            for (int d = 0; d < T; ++d) {
                a[d] = val(2, x, d);
                a[d].x *= u.x;
                a[d].y *= u.y;
            }
            if (p.in[3].kind) {
#pragma unroll
                for (int d = 0; d < T; ++d) {
                    const float2 v = val(3, x, d);
                    a[d].x *= v.x;
                    a[d].y *= v.y;
                }
            }
#pragma unroll
            for (int d = 0; d < T; ++d) b[d] = val(4, x, d);
            if (p.in[5].kind) {
#pragma unroll
                for (int d = 0; d < T; ++d) {
                    const float2 v = val(5, x, d);
                    b[d].x *= v.x;
                    b[d].y *= v.y;
                }
            }
#pragma unroll
            for (int d0 = 0; d0 < T; ++d0)
#pragma unroll
                for (int d1 = 0; d1 < T; ++d1) {
                    acc[d0][d1][0] = fmaf(a[d0].x, b[d1].x, acc[d0][d1][0]);
                    acc[d0][d1][1] = fmaf(a[d0].y, b[d1].y, acc[d0][d1][1]);
                }
        }
        // the stage may be refilled as soon as every consumer warp has read it
        __syncwarp();
        if (lane == 0) mbar_arrive(&s_empty[s]);
        if (++s == S) {
            s = 0;
            ++n;
        }
      }
        if (row < p.n_rows) {
            float *outp = p.out + row;
#pragma unroll
            for (int d1 = 0; d1 < T; ++d1)
#pragma unroll
                for (int d0 = 0; d0 < T; ++d0)
                    __stcs(reinterpret_cast<float2 *>(outp + static_cast<int64_t>(o_base + d1 * p.c0 + d0) * p.ld),
                           make_float2(acc[d0][d1][0], acc[d0][d1][1]));
        }
    }
}

// ------------------------------------------------------------------ host
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                  const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = [] {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) {
            cudaGetLastError();
            p = nullptr;
        }
        return reinterpret_cast<EncodeTiledFn>(p);
    }();
    return fn;
}

int env_int(const char *name, int fallback) {
    const char *e = getenv(name);
    return e ? atoi(e) : fallback;
}

bool combo(int T, int cx) { return (T == 5 && cx == 5) || (T == 4 && (cx == 4 || cx == 8)) || (T == 3 && cx == 3) || (T == 2 && cx == 2); }

template <int T, int CX>
cudaError_t launch(const SbnTmaParams &q, int grid, size_t smem, cudaStream_t stream) {
    sbn_step_tma<T, CX><<<grid, SBN_TMA_THREADS, smem, stream>>>(q);
    return cudaGetLastError();
}
template <int T, int CX>
cudaError_t set_attr() {
    return cudaFuncSetAttribute(sbn_step_tma<T, CX>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
}

}  // namespace

bool sbn_tma_encode_rows(CUtensorMap *map, const float *base, int64_t ld, int64_t n_rows, int64_t entries, int box_rows, int e_lo) {
    if (!encode_fn() || e_lo <= 0 || entries % e_lo != 0) return false;
    const cuuint64_t dims[3] = {static_cast<cuuint64_t>(n_rows), static_cast<cuuint64_t>(e_lo), static_cast<cuuint64_t>(entries / e_lo)};
    const cuuint64_t strides[2] = {static_cast<cuuint64_t>(ld) * 4, static_cast<cuuint64_t>(ld) * 4 * e_lo};
    const cuuint32_t box[3] = {static_cast<cuuint32_t>(box_rows), static_cast<cuuint32_t>(e_lo), static_cast<cuuint32_t>(entries / e_lo)};
    const cuuint32_t estr[3] = {1, 1, 1};
    return encode_fn()(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float *>(base), dims, strides, box, estr,
                       CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                       CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

bool sbn_tma_encode_view(CUtensorMap *map, const float *base, int64_t ld, int64_t n_rows, int rank, const int64_t *dims,
                         const int64_t *strides, const int *box, int box_rows) {
    if (!encode_fn() || rank < 1 || rank > 4) return false;
    cuuint64_t gdim[5], gstride[4];
    cuuint32_t gbox[5], estr[5];
    gdim[0] = static_cast<cuuint64_t>(n_rows);
    gbox[0] = static_cast<cuuint32_t>(box_rows);
    estr[0] = 1;
    for (int k = 0; k < rank; ++k) {
        gdim[k + 1] = static_cast<cuuint64_t>(dims[k]);
        gstride[k] = static_cast<cuuint64_t>(dims[k] > 1 ? strides[k] : 1) * static_cast<cuuint64_t>(ld) * 4;
        gbox[k + 1] = static_cast<cuuint32_t>(box[k]);
        estr[k + 1] = 1;
    }
    return encode_fn()(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, static_cast<cuuint32_t>(rank + 1), const_cast<float *>(base), gdim, gstride,
                       gbox, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                       CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

cudaError_t sbn_tma_set_attrs() {
    cudaError_t e = set_attr<5, 5>();
    if (e == cudaSuccess) e = set_attr<4, 4>();
    if (e == cudaSuccess) e = set_attr<4, 8>();
    if (e == cudaSuccess) e = set_attr<3, 3>();
    if (e == cudaSuccess) e = set_attr<2, 2>();
    return e;
}

// A step this kernel takes: planned for the tiled kernel, two tile axes, whole tiles, ONE eliminated
// variable whose states are unrolled, one or two batched operands (each the first of its class),
// tables small enough to sit beside the ring.
bool sbn_tma_eligible(const sbn_program *P, const StepDesc &st) {
    if (!encode_fn() || P->f64 || !P->use_tma) return false;
    if (st.kind != 1 || st.tile <= 0 || st.nc != 0 || st.big_tables || st.slice_pos >= 0) return false;
    if (st.ecards.empty() || !combo(st.tile, st.ecards[0])) return false;
    if (st.ecards.size() > 1 && st.zoff_tiled_pos < 0) return false;
    if (st.cards.size() < 2 || st.na < 1 || st.nb < 1) return false;
    if (st.cards[0] % st.tile || st.cards[1] % st.tile) return false;
    if (st.nu > 2 || st.na > 2 || st.nb > 2) return false;
    int n_batched = 0, batched_in_class[3] = {0, 0, 0};
    int64_t tables = 0;
    for (size_t i = 0; i < st.in.size(); ++i) {
        const InDesc &in = st.in[st.order[i]];
        const int cls = static_cast<int>(i) < st.nu ? 0 : static_cast<int>(i) < st.nu + st.na ? 1 : 2;
        if (in.batched) {
            ++n_batched;
            if (++batched_in_class[cls] > 1) return false;  // one batched operand per class (it takes the class's first slot)
        } else {
            tables += in.is_slot ? P->slots[in.id].padded : P->table_padded[in.id];
        }
    }
    if (n_batched < 1 || n_batched > 2) return false;
    if (tables * 4 > 48 * 1024) return false;
    static const int min_out = env_int("SOROBN_B200_TMA_MINOUT", 250);  // small outputs: the one-wave launches win
    return st.n_out >= min_out;
}

cudaError_t sbn_tma_launch(sbn_program *P, const StepDesc &st, const uint8_t *d_ev, int64_t ld_ev, int64_t n_rows,
                           cudaStream_t stream) {
    SbnTmaParams q;
    memset(&q, 0, sizeof q);
    const int T = st.tile, cx = st.ecards[0];  // states of one block; st.cx of them in all
    q.cx = st.cx;
    q.n_blocks = st.cx / cx;
    q.zoff = st.ecards.size() > 1 ? P->d_tile_off + st.zoff_tiled_pos : nullptr;
    q.out = P->slots[st.out_slot].ptr;
    q.ev = d_ev;
    q.ld_ev = ld_ev;
    q.ld = P->ld;
    q.n_rows = static_cast<int32_t>(n_rows);
    q.n_tiles = static_cast<int32_t>(st.n_tiles);
    q.row_words = static_cast<int32_t>(st.in.size()) + 2;
    q.c0 = st.cards[0];
    q.tile_off = P->d_tile_off + st.tile_off_pos;
    const int64_t n_rblocks = (n_rows + SBN_TMA_ROWS - 1) / SBN_TMA_ROWS;
    q.n_items = n_rblocks * st.n_tiles;

    int next_slot[3] = {0, 2, 4};
    int n_maps = 0, stage_floats = 0, table_floats = 0, n_boxes = 0;
    struct Batched {
        int slot_id, tn, sd, sx;
    };
    std::vector<Batched> batched_desc;
    // slot order inside a class: the batched operand first (only slots U0 / A0 / B0 read the TMA ring)
    std::vector<size_t> visit;
    for (int pass = 0; pass < 2; ++pass)
        for (size_t i = 0; i < st.in.size(); ++i)
            if (st.in[st.order[i]].batched == (pass == 0)) visit.push_back(i);
    for (size_t i : visit) {
        const InDesc &in = st.in[st.order[i]];
        const int cls = static_cast<int>(i) < st.nu ? 0 : static_cast<int>(i) < st.nu + st.na ? 1 : 2;
        SbnTmaIn &d = q.in[next_slot[cls]++];
        d.col = static_cast<int32_t>(i);
        d.sx = in.sx;
        d.sd = cls == 1 ? in.strides[0] : cls == 2 ? in.strides[1] : 0;
        if (in.batched) {
            d.kind = 2;
            d.tmap = n_maps;
            d.tn = cls == 0 ? 1 : T;
            d.off = stage_floats;
            const int nk = cx * d.tn;
            if (n_maps == 0) q.nk0 = nk;
            stage_floats += nk * SBN_TMA_ROWS;
            n_boxes += nk;
            batched_desc.push_back({in.id, d.tn, d.sd, d.sx});
            ++n_maps;
        } else {
            d.kind = 1;
            d.off = table_floats;
            d.n_ev = static_cast<int32_t>(in.ev.size());
            for (size_t a = 0; a < in.ev.size(); ++a) {
                d.ev_col[a] = in.ev[a].col;
                d.ev_stride[a] = in.ev[a].stride;
                d.ev_card[a] = in.ev[a].card;
            }
            SbnTmaTable &tb = q.tab[q.n_tables++];
            const int64_t padded = in.is_slot ? P->slots[in.id].padded : P->table_padded[in.id];
            tb.src = in.is_slot ? P->slots[in.id].ptr : P->d_tables + P->tables[in.id].first;
            tb.floats = static_cast<int32_t>(padded);
            tb.off = table_floats;
            table_floats += static_cast<int>(padded);
        }
    }
    // Tensor maps.  Preferred: a 4-D view (rows, tile digit, eliminated state, entry) of the factor whose
    // box (256, tn, CX, 1) is the whole operand block of a tile -- ONE TMA instruction per operand
    // and stage (25 one-entry boxes per stage saturate the TMA unit's issue rate before HBM).
    // The view needs non-zero strides for both axes; otherwise fall back to (rows, entries) with
    // one-entry boxes.
    static const int big_env = env_int("SOROBN_B200_TMA_BIGBOX", 1);
    bool big = big_env != 0;
    for (const Batched &b : batched_desc)
        if (b.sx <= 0 || (b.tn > 1 && b.sd <= 0)) big = false;
    for (int attempt = 0; attempt < 2; ++attempt) {
        bool ok = true;
        for (size_t m = 0; m < batched_desc.size() && ok; ++m) {
            const Batched &b = batched_desc[m];
            const cuuint64_t ld = static_cast<cuuint64_t>(P->ld), n_e = static_cast<cuuint64_t>(P->slots[b.slot_id].size);
            CUresult r;
            if (big) {
                const cuuint64_t dims[4] = {ld, static_cast<cuuint64_t>(b.tn), static_cast<cuuint64_t>(cx), n_e};
                const cuuint64_t strides[3] = {(b.tn > 1 ? static_cast<cuuint64_t>(b.sd) : 1) * ld * 4, static_cast<cuuint64_t>(b.sx) * ld * 4, ld * 4};
                const cuuint32_t box[4] = {SBN_TMA_ROWS, static_cast<cuuint32_t>(b.tn), static_cast<cuuint32_t>(cx), 1};
                const cuuint32_t estr[4] = {1, 1, 1, 1};
                r = encode_fn()(&q.tm[m], CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, P->slots[b.slot_id].ptr, dims, strides, box, estr,
                                CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                                CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            } else {
                const cuuint64_t dims[2] = {ld, n_e};
                const cuuint64_t strides[1] = {ld * 4};
                const cuuint32_t box[2] = {SBN_TMA_ROWS, 1};
                const cuuint32_t estr[2] = {1, 1};
                r = encode_fn()(&q.tm[m], CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, P->slots[b.slot_id].ptr, dims, strides, box, estr,
                                CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                                CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            }
            if (r != CUDA_SUCCESS) ok = false;
        }
        if (ok) break;
        if (!big) return cudaErrorInvalidValue;
        big = false;  // the driver refused the 4-D view: one-entry boxes
    }
    q.big_boxes = big ? 1 : 0;
    q.n_maps = n_maps;
    q.stage_floats = stage_floats;
    q.n_boxes = n_boxes;
    q.table_floats = table_floats;
    // ring depth: three stages when two CTAs still fit an SM, else two
    static const int stages_env = env_int("SOROBN_B200_TMA_STAGES", 0);
    int S = stages_env > 0 ? std::min(stages_env, SBN_TMA_MAX_STAGES) : 3;
    auto smem_of = [&](int s) { return static_cast<size_t>(s) * stage_floats * 4 + static_cast<size_t>(table_floats) * 4; };
    while (S > 2 && smem_of(S) > 110 * 1024) --S;
    if (smem_of(S) > 200 * 1024) return cudaErrorInvalidConfiguration;
    q.n_stages = S;
    const int sms = P->n_sms;
    const int per_sm = smem_of(S) + 2048 <= 113 * 1024 ? 2 : 1;
    const int grid = static_cast<int>(std::min<int64_t>(q.n_items, static_cast<int64_t>(sms) * per_sm));
    const size_t smem = smem_of(S);
    if (T == 5) return launch<5, 5>(q, grid, smem, stream);
    if (T == 4 && cx == 4) return launch<4, 4>(q, grid, smem, stream);
    if (T == 4) return launch<4, 8>(q, grid, smem, stream);
    if (T == 3) return launch<3, 3>(q, grid, smem, stream);
    return launch<2, 2>(q, grid, smem, stream);
}
