// sorobn_b200 -- the on-chip segment kernel and its host-side planning (see sbn_chain.h).
#include "sbn_chain.h"

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <type_traits>

#include "sbn_internal.h"

// dynamic shared memory of the segment kernel: [evidence codes][table buffer 0][table buffer 1][arena]
extern __shared__ __align__(16) uint8_t sbn_smem[];

namespace {

// ------------------------------------------------------------------ PTX helpers
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
__device__ __forceinline__ void tma_bulk_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
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

__device__ __forceinline__ void bar_compute(int n_threads) { asm volatile("bar.sync 1, %0;" ::"r"(n_threads) : "memory"); }

__device__ __forceinline__ float lds_f(uint32_t off) { return *reinterpret_cast<const float *>(sbn_smem + off); }
// operands outside shared memory (the CTA's scratch, the slot arena) are streamed: they bypass L1,
// which is left to the tile tables every row block re-reads
__device__ __forceinline__ float ldg_f(const char *p, uint32_t off) { return __ldcg(reinterpret_cast<const float *>(p + off)); }
__device__ __forceinline__ void stg_f(char *p, uint32_t off, float v) { __stcg(reinterpret_cast<float *>(p + off), v); }

__device__ __forceinline__ uint32_t lds_u(uint32_t off) { return *reinterpret_cast<const uint32_t *>(sbn_smem + off); }

// ---- step records (shared memory, uint32 words; built by sbn_chain_bind) ----------------------
//   header  [0] fast | T << 3 | out_space << 6 | n_in << 9   [1] present   [2] cx   [3] n_tiles
//           [4] out_off  [5] out_eb  [6] out_c0b  [7] ksplit  [8,9] out_ptr
//           [10] tile rows (byte offset from the records' base)  [11] joint-state offsets (same; 0 = none)
//           [14] word offsets of slots 0..3 (8 bits each)  [15] of slots 4..6
//   slot    [0] space | col << 4 | n_ev << 8  [1] off  [2] sxb  [3] sab  [4] sbb  [5,6] ptr  [7] -
//           then per evidence axis: col | card << 16, byte stride
//   tile rows: [n_tiles][2 + n_in] = out byte offset, na | nb << 8, input byte offsets
// Everything is read with LDS: addresses are byte offsets into sbn_smem, never generic pointers.
#define SBN_REC_HDR 16
#define SBN_REC_SLOT 8

struct StepRec {
    uint32_t b;      // byte offset of the record inside sbn_smem
    uint32_t base;   // byte offset of the records' base (tile rows / offsets are relative to it)
    __device__ __forceinline__ uint32_t wd(int i) const { return lds_u(b + 4 * i); }
    __device__ __forceinline__ int fast() const { return wd(0) & 7; }
    __device__ __forceinline__ int T() const { return (wd(0) >> 3) & 7; }
    __device__ __forceinline__ int out_space() const { return (wd(0) >> 6) & 7; }
    __device__ __forceinline__ int n_in() const { return (wd(0) >> 9) & 15; }
    __device__ __forceinline__ int present() const { return static_cast<int>(wd(1)); }
    __device__ __forceinline__ int cx() const { return static_cast<int>(wd(2)); }
    __device__ __forceinline__ int n_tiles() const { return static_cast<int>(wd(3)); }
    __device__ __forceinline__ uint32_t out_off() const { return wd(4); }
    __device__ __forceinline__ uint32_t out_eb() const { return wd(5); }
    __device__ __forceinline__ uint32_t out_c0b() const { return wd(6); }
    __device__ __forceinline__ int ksplit() const { return static_cast<int>(wd(7)); }
    __device__ __forceinline__ char *out_ptr() const { return reinterpret_cast<char *>(static_cast<uint64_t>(wd(8)) | static_cast<uint64_t>(wd(9)) << 32); }
    __device__ __forceinline__ uint32_t tiles_b() const { return base + wd(10); }
    __device__ __forceinline__ bool has_xoff() const { return wd(11) != 0; }
    __device__ __forceinline__ uint32_t xoff_b() const { return base + wd(11); }
    __device__ __forceinline__ uint32_t slot(int k) const { return b + 4 * ((wd(14 + (k >> 2)) >> (8 * (k & 3))) & 0xff); }
};
__device__ __forceinline__ int slot_space(uint32_t sw) { return lds_u(sw) & 15; }
__device__ __forceinline__ int slot_col(uint32_t sw) { return (lds_u(sw) >> 4) & 15; }
__device__ __forceinline__ const char *slot_ptr(uint32_t sw) {
    return reinterpret_cast<const char *>(static_cast<uint64_t>(lds_u(sw + 20)) | static_cast<uint64_t>(lds_u(sw + 24)) << 32);
}
// byte offset inside shared memory of element 0 of a shared-memory operand for this lane (tables:
// plus the row's evidence offset)
__device__ __forceinline__ uint32_t slot_smem_base(uint32_t sw, uint32_t ring_b, uint32_t arena_b, int lane) {
    const uint32_t w0 = lds_u(sw), off = lds_u(sw + 4);
    if ((w0 & 15) == SBN_SP_TABLE) {
        const int n_ev = (w0 >> 8) & 15;
        uint32_t evo = 0;
#pragma unroll 4
        for (int e = 0; e < n_ev; ++e) {
            const uint32_t cc = lds_u(sw + 4 * (SBN_REC_SLOT + 2 * e));
            evo += static_cast<uint32_t>(min(static_cast<int>(sbn_smem[(cc & 0xffff) * SBN_CHAIN_ROWS + lane]), static_cast<int>(cc >> 16) - 1)) *
                   lds_u(sw + 4 * (SBN_REC_SLOT + 2 * e + 1));
        }
        return ring_b + off + evo;
    }
    return arena_b + off + lane * 4;
}

struct StepCtx {
    uint32_t ring_b, arena_b;
    char *scratch;
    const char *any_global;
    int lane, warp, n_warps, n_threads;
    int64_t row;
    bool live;
};

// One elimination step for this CTA's 32 rows, any shape: warps share the tiles, lanes are rows.
//   out[o, b] = sum_x prod_i in_i[off_i(o) + xoff_i(x) (+ evoff_i(b))]
// Inputs sit in fixed class slots (U0 U1: no tile axis, A0 A1: axis 0, B0 B1: axis 1, C0: both);
// absent slots and the memory space of a present one are CTA-uniform branches.  The code is shaped
// for the largest tile edge (5): a smaller edge runs through the clamps / predicates of partial tiles.
// ksplit > 1 (few tiles, many eliminated states): the states of a tile are split over ksplit warps
// whose partial sums meet in the output through atomic adds.
constexpr int TG = 5;
__device__ __noinline__ void chain_step_generic(StepRec rec, StepCtx c) {
    constexpr int T = TG;
    const int present = rec.present();
    uint32_t so[SBN_CHAIN_SLOTS], sxb[SBN_CHAIN_SLOTS], sab[SBN_CHAIN_SLOTS], sbb[SBN_CHAIN_SLOTS];
    const char *gp[SBN_CHAIN_SLOTS];
    int col[SBN_CHAIN_SLOTS];
    bool sm[SBN_CHAIN_SLOTS];
#pragma unroll
    for (int k = 0; k < SBN_CHAIN_SLOTS; ++k) {
        so[k] = sxb[k] = sab[k] = sbb[k] = 0;
        gp[k] = c.any_global;  // unused slots are never read
        col[k] = 0;
        sm[k] = true;
        if ((present >> k) & 1) {
            const uint32_t sw = rec.slot(k);
            const int space = slot_space(sw);
            if (space == SBN_SP_TABLE || space == SBN_SP_SMEM) {
                so[k] = slot_smem_base(sw, c.ring_b, c.arena_b, c.lane);
            } else if (space == SBN_SP_GLOBAL) {
                gp[k] = slot_ptr(sw) + c.row * 4;
                sm[k] = false;
            } else {
                gp[k] = c.scratch + lds_u(sw + 4) + c.lane * 4;
                sm[k] = false;
            }
            sxb[k] = lds_u(sw + 8);
            sab[k] = lds_u(sw + 12);
            sbb[k] = lds_u(sw + 16);
            col[k] = slot_col(sw);
        }
        __builtin_assume(__isGlobal(gp[k]));
    }
    const bool out_sm = rec.out_space() == SBN_SP_SMEM, out_global = rec.out_space() == SBN_SP_GLOBAL;
    const uint32_t out_so = c.arena_b + rec.out_off() + c.lane * 4;
    char *out_gp = out_global ? rec.out_ptr() + c.row * 4 : out_sm ? const_cast<char *>(c.any_global) : c.scratch + rec.out_off() + c.lane * 4;
    __builtin_assume(__isGlobal(out_gp));
    const uint32_t oeb = rec.out_eb(), oc0b = rec.out_c0b();
    const int cx = rec.cx(), n_tiles = rec.n_tiles(), row_words = rec.n_in() + 2, ks = rec.ksplit();
    const bool xoffs = rec.has_xoff();
    const uint32_t xoff_b = rec.xoff_b(), tiles_b = rec.tiles_b();
    const bool hU0 = present & 1, hU1 = present & 2, hA0 = present & 4, hA1 = present & 8, hB0 = present & 16,
               hB1 = present & 32, hC = present & 64;
    const bool may_store = !out_global || c.live;

    if (ks > 1) {
        // zero the output, then every warp adds its share
        for (int t = c.warp; t < n_tiles; t += c.n_warps) {
            const uint32_t trow = tiles_b + static_cast<uint32_t>(t * row_words) * 4;
            const uint32_t o_off = lds_u(trow), nab = lds_u(trow + 4);
            const int na = nab & 0xff, nb = nab >> 8;
            for (int d1 = 0; d1 < nb; ++d1)
                for (int d0 = 0; d0 < na; ++d0) {
                    if (out_sm) *reinterpret_cast<float *>(sbn_smem + out_so + o_off + d1 * oc0b + d0 * oeb) = 0.f;
                    else if (may_store) stg_f(out_gp, o_off + d1 * oc0b + d0 * oeb, 0.f);
                }
        }
        bar_compute(c.n_threads);
    }
    const int n_items = n_tiles * ks;
    for (int item = c.warp; item < n_items; item += c.n_warps) {
        const int t = item / ks, j = item - t * ks;
        const int x_begin = static_cast<int>(static_cast<int64_t>(cx) * j / ks), x_end = static_cast<int>(static_cast<int64_t>(cx) * (j + 1) / ks);
        const uint32_t trow = tiles_b + static_cast<uint32_t>(t * row_words) * 4;
        const uint32_t o_off = lds_u(trow);
        const uint32_t nab = lds_u(trow + 4);
        const int na = nab & 0xff, nb = nab >> 8;
        uint32_t base[SBN_CHAIN_SLOTS];
#pragma unroll
        for (int k = 0; k < SBN_CHAIN_SLOTS; ++k) base[k] = ((present >> k) & 1) ? lds_u(trow + 4 * (2 + col[k])) : 0u;
        float acc[T][T];
#pragma unroll
        for (int d0 = 0; d0 < T; ++d0)
#pragma unroll
            for (int d1 = 0; d1 < T; ++d1) acc[d0][d1] = 0.f;
        // digits past the tile edge re-read the last valid entry (clamped: every load stays in
        // bounds); only the stores are predicated
        auto k0 = [&](int d) -> uint32_t { return min(d, na - 1); };
        auto k1 = [&](int d) -> uint32_t { return min(d, nb - 1); };
#pragma unroll 1
        for (int x = x_begin; x < x_end; ++x) {
            auto xo = [&](int k) -> uint32_t {
                return base[k] + (xoffs ? lds_u(xoff_b + 4 * (col[k] * cx + x)) : static_cast<uint32_t>(x) * sxb[k]);
            };
            float u = 1.f;
            if (hU0) u = sm[0] ? lds_f(so[0] + xo(0)) : ldg_f(gp[0], xo(0));
            if (hU1) u *= sm[1] ? lds_f(so[1] + xo(1)) : ldg_f(gp[1], xo(1));
            float a[T], b[T];
            if (hA0) {
                const uint32_t e = xo(2);
#pragma unroll
                for (int d = 0; d < T; ++d) a[d] = (sm[2] ? lds_f(so[2] + e + k0(d) * sab[2]) : ldg_f(gp[2], e + k0(d) * sab[2])) * u;
            } else {
#pragma unroll
                for (int d = 0; d < T; ++d) a[d] = u;
            }
            if (hA1) {
                const uint32_t e = xo(3);
#pragma unroll
                for (int d = 0; d < T; ++d) a[d] *= sm[3] ? lds_f(so[3] + e + k0(d) * sab[3]) : ldg_f(gp[3], e + k0(d) * sab[3]);
            }
            if (hB0) {
                const uint32_t e = xo(4);
#pragma unroll
                for (int d = 0; d < T; ++d) b[d] = sm[4] ? lds_f(so[4] + e + k1(d) * sbb[4]) : ldg_f(gp[4], e + k1(d) * sbb[4]);
            } else {
#pragma unroll
                for (int d = 0; d < T; ++d) b[d] = 1.f;
            }
            if (hB1) {
                const uint32_t e = xo(5);
#pragma unroll
                for (int d = 0; d < T; ++d) b[d] *= sm[5] ? lds_f(so[5] + e + k1(d) * sbb[5]) : ldg_f(gp[5], e + k1(d) * sbb[5]);
            }
            if (hC) {
                const uint32_t e = xo(6);
#pragma unroll
                for (int d1 = 0; d1 < T; ++d1) {
                    if (d1 < nb) {
#pragma unroll
                        for (int d0 = 0; d0 < T; ++d0) {
                            const uint32_t o = e + k0(d0) * sab[6] + k1(d1) * sbb[6];
                            const float cv = sm[6] ? lds_f(so[6] + o) : ldg_f(gp[6], o);
                            acc[d0][d1] = fmaf(a[d0] * b[d1], cv, acc[d0][d1]);
                        }
                    }
                }
            } else {
#pragma unroll
                for (int d1 = 0; d1 < T; ++d1) {
                    if (d1 < nb) {
#pragma unroll
                        for (int d0 = 0; d0 < T; ++d0) acc[d0][d1] = fmaf(a[d0], b[d1], acc[d0][d1]);
                    }
                }
            }
        }
#pragma unroll
        for (int d1 = 0; d1 < T; ++d1)
#pragma unroll
            for (int d0 = 0; d0 < T; ++d0)
                if (d0 < na && d1 < nb) {
                    const uint32_t o = o_off + d1 * oc0b + d0 * oeb;
                    if (ks > 1) {
                        if (out_sm) atomicAdd(reinterpret_cast<float *>(sbn_smem + out_so + o), acc[d0][d1]);
                        else if (may_store) atomicAdd(reinterpret_cast<float *>(out_gp + o), acc[d0][d1]);
                    } else if (out_sm) {
                        *reinterpret_cast<float *>(sbn_smem + out_so + o) = acc[d0][d1];
                    } else if (may_store) {
                        stg_f(out_gp, o, acc[d0][d1]);
                    }
                }
    }
}

// The common shape, specialised: two-axis tile, full T x T tiles, the first eliminated variable has
// T states -- its T states are unrolled, the joint states of further eliminated variables are
// walked block by block with the accumulators kept in registers.  Every operand is in shared
// memory (tables and arena) except possibly A0 (GA) and B0 (GB), which then live in the CTA's
// scratch / the slot arena.  Per operand load: one integer multiply-add and one LDS (or LDG.cg).
template <int T, bool GA, bool GB>
__device__ __noinline__ void chain_step_fast(StepRec rec, StepCtx c) {
    const int present = rec.present();
    const bool hU0 = present & 1, hU1 = present & 2, hA1 = present & 8, hB1 = present & 32;
    uint32_t s_u0 = 0, s_u1 = 0, s_a0 = 0, s_a1 = 0, s_b0 = 0, s_b1 = 0;
    uint32_t x_u0 = 0, x_u1 = 0, x_a0, x_a1 = 0, x_b0, x_b1 = 0, d_a0, d_a1 = 0, d_b0, d_b1 = 0;
    int c_u0 = 0, c_u1 = 0, c_a0, c_a1 = 0, c_b0, c_b1 = 0;
    const char *g_a0 = c.any_global, *g_b0 = c.any_global;
    if (hU0) { const uint32_t sw = rec.slot(0); s_u0 = slot_smem_base(sw, c.ring_b, c.arena_b, c.lane); x_u0 = lds_u(sw + 8); c_u0 = slot_col(sw); }
    if (hU1) { const uint32_t sw = rec.slot(1); s_u1 = slot_smem_base(sw, c.ring_b, c.arena_b, c.lane); x_u1 = lds_u(sw + 8); c_u1 = slot_col(sw); }
    {
        const uint32_t sw = rec.slot(2);
        if (GA) g_a0 = slot_space(sw) == SBN_SP_GLOBAL ? slot_ptr(sw) + c.row * 4 : c.scratch + lds_u(sw + 4) + c.lane * 4;
        else s_a0 = slot_smem_base(sw, c.ring_b, c.arena_b, c.lane);
        x_a0 = lds_u(sw + 8); d_a0 = lds_u(sw + 12); c_a0 = slot_col(sw);
    }
    if (hA1) { const uint32_t sw = rec.slot(3); s_a1 = slot_smem_base(sw, c.ring_b, c.arena_b, c.lane); x_a1 = lds_u(sw + 8); d_a1 = lds_u(sw + 12); c_a1 = slot_col(sw); }
    {
        const uint32_t sw = rec.slot(4);
        if (GB) g_b0 = slot_space(sw) == SBN_SP_GLOBAL ? slot_ptr(sw) + c.row * 4 : c.scratch + lds_u(sw + 4) + c.lane * 4;
        else s_b0 = slot_smem_base(sw, c.ring_b, c.arena_b, c.lane);
        x_b0 = lds_u(sw + 8); d_b0 = lds_u(sw + 16); c_b0 = slot_col(sw);
    }
    __builtin_assume(__isGlobal(g_a0));
    __builtin_assume(__isGlobal(g_b0));
    if (hB1) { const uint32_t sw = rec.slot(5); s_b1 = slot_smem_base(sw, c.ring_b, c.arena_b, c.lane); x_b1 = lds_u(sw + 8); d_b1 = lds_u(sw + 16); c_b1 = slot_col(sw); }

    const bool out_sm = rec.out_space() == SBN_SP_SMEM, out_global = rec.out_space() == SBN_SP_GLOBAL;
    const uint32_t out_so = c.arena_b + rec.out_off() + c.lane * 4;
    char *out_gp = out_global ? rec.out_ptr() + c.row * 4 : out_sm ? const_cast<char *>(c.any_global) : c.scratch + rec.out_off() + c.lane * 4;
    __builtin_assume(__isGlobal(out_gp));
    const uint32_t oeb = rec.out_eb(), oc0b = rec.out_c0b();
    const int cx = rec.cx(), n_tiles = rec.n_tiles(), row_words = rec.n_in() + 2;
    const bool xoffs = rec.has_xoff();
    const uint32_t xoff_b = rec.xoff_b(), tiles_b = rec.tiles_b();

    for (int t = c.warp; t < n_tiles; t += c.n_warps) {
        const uint32_t trow = tiles_b + static_cast<uint32_t>(t * row_words) * 4;
        const uint32_t r_o = lds_u(trow);
        const uint32_t r_u0 = hU0 ? lds_u(trow + 4 * (2 + c_u0)) : 0u, r_u1 = hU1 ? lds_u(trow + 4 * (2 + c_u1)) : 0u;
        const uint32_t r_a0 = lds_u(trow + 4 * (2 + c_a0)), r_a1 = hA1 ? lds_u(trow + 4 * (2 + c_a1)) : 0u;
        const uint32_t r_b0 = lds_u(trow + 4 * (2 + c_b0)), r_b1 = hB1 ? lds_u(trow + 4 * (2 + c_b1)) : 0u;
        float acc[T][T];
#pragma unroll
        for (int d0 = 0; d0 < T; ++d0)
#pragma unroll
            for (int d1 = 0; d1 < T; ++d1) acc[d0][d1] = 0.f;
        for (int blk = 0; blk < cx; blk += T) {
            // element 0 of this block of T eliminated states, per operand
            uint32_t e_u0 = s_u0 + r_u0, e_u1 = s_u1 + r_u1, e_a0 = s_a0 + r_a0, e_a1 = s_a1 + r_a1, e_b0 = s_b0 + r_b0,
                     e_b1 = s_b1 + r_b1;
            if (xoffs) {
                if (hU0) e_u0 += lds_u(xoff_b + 4 * (c_u0 * cx + blk));
                if (hU1) e_u1 += lds_u(xoff_b + 4 * (c_u1 * cx + blk));
                e_a0 += lds_u(xoff_b + 4 * (c_a0 * cx + blk));
                if (hA1) e_a1 += lds_u(xoff_b + 4 * (c_a1 * cx + blk));
                e_b0 += lds_u(xoff_b + 4 * (c_b0 * cx + blk));
                if (hB1) e_b1 += lds_u(xoff_b + 4 * (c_b1 * cx + blk));
            }
#pragma unroll
            for (int x = 0; x < T; ++x) {
                float a[T], b[T];
#pragma unroll
                for (int d = 0; d < T; ++d) a[d] = GA ? ldg_f(g_a0, e_a0 + x * x_a0 + d * d_a0) : lds_f(e_a0 + x * x_a0 + d * d_a0);
#pragma unroll
                for (int d = 0; d < T; ++d) b[d] = GB ? ldg_f(g_b0, e_b0 + x * x_b0 + d * d_b0) : lds_f(e_b0 + x * x_b0 + d * d_b0);
                if (hU0) {
                    float u = lds_f(e_u0 + x * x_u0);
                    if (hU1) u *= lds_f(e_u1 + x * x_u1);
#pragma unroll
                    for (int d = 0; d < T; ++d) b[d] *= u;
                }
                if (hA1) {
#pragma unroll
                    for (int d = 0; d < T; ++d) a[d] *= lds_f(e_a1 + x * x_a1 + d * d_a1);
                }
                if (hB1) {
#pragma unroll
                    for (int d = 0; d < T; ++d) b[d] *= lds_f(e_b1 + x * x_b1 + d * d_b1);
                }
#pragma unroll
                for (int d1 = 0; d1 < T; ++d1)
#pragma unroll
                    for (int d0 = 0; d0 < T; ++d0) acc[d0][d1] = fmaf(a[d0], b[d1], acc[d0][d1]);
            }
        }
        if (out_sm) {
#pragma unroll
            for (int d1 = 0; d1 < T; ++d1)
#pragma unroll
                for (int d0 = 0; d0 < T; ++d0)
                    *reinterpret_cast<float *>(sbn_smem + out_so + r_o + d1 * oc0b + d0 * oeb) = acc[d0][d1];
        } else if (!out_global || c.live) {
#pragma unroll
            for (int d1 = 0; d1 < T; ++d1)
#pragma unroll
                for (int d0 = 0; d0 < T; ++d0) stg_f(out_gp, r_o + d1 * oc0b + d0 * oeb, acc[d0][d1]);
        }
    }
}

constexpr int kChainStages = SBN_CHAIN_STAGES;        // table staging runs this many steps ahead of the arithmetic
constexpr int kChainMaxThreads = 512;  // 128 registers: with 13..16 warps one SM sub-partition (16K registers) hosts 4 of them

// Roles: warps 0 .. n_cw-1 compute (they meet at named barrier 1), the last warp is the producer --
// one lane of it keeps the table ring full: for step g + kChainStages - 1 it waits until the
// stage's previous tenant (step g - 1) has been left by every compute warp (`empty` mbarrier) and
// issues the bulk-TMA copies that complete on the stage's `full` mbarrier.
__global__ void __launch_bounds__(kChainMaxThreads, 1) sbn_chain_kernel(const __grid_constant__ SbnChainParams p) {
    __shared__ __align__(8) uint64_t s_full[kChainStages], s_empty[kChainStages];
    const uint32_t rec_b = static_cast<uint32_t>(p.ev_bytes);
    const uint32_t ring_b = rec_b + static_cast<uint32_t>(p.rec_words) * 4u;
    const uint32_t arena_b = ring_b + static_cast<uint32_t>(p.ring_bytes);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_cw = (blockDim.x >> 5) - 1;
    const int n_ct = n_cw * 32;
    const int n_steps = p.n_steps;
    const int my_blocks = (p.n_rblocks - static_cast<int>(blockIdx.x) + static_cast<int>(gridDim.x) - 1) / static_cast<int>(gridDim.x);
    const int64_t g_end = static_cast<int64_t>(my_blocks) * n_steps;

    {
        uint32_t *recs = reinterpret_cast<uint32_t *>(sbn_smem + rec_b);
        for (int i = threadIdx.x; i < p.rec_words; i += blockDim.x) recs[i] = __ldg(p.recs + i);
    }
    if (threadIdx.x == 0) {
        for (int k = 0; k < kChainStages; ++k) {
            mbar_init(&s_full[k], 1);
            mbar_init(&s_empty[k], 1);
        }
        fence_mbar_init();
    }
    __syncthreads();

    if (warp == n_cw) {
        // ------------------------------------------------------------------ producer
        if (lane != 0) return;
        int s = 0;
        for (int64_t g = 0; g < g_end; ++g) {
            const int stage = static_cast<int>(g % kChainStages);
            if (g >= kChainStages) mbar_wait(&s_empty[stage], static_cast<uint32_t>(((g / kChainStages) - 1) & 1));
            const SbnChainStage *sg = p.stages + s;
            const uint32_t bytes = sg->bytes;
            if (bytes == 0) {
                mbar_arrive(&s_full[stage]);
            } else {
                mbar_expect_tx(&s_full[stage], bytes);
                for (int k = 0; k < sg->n; ++k)
                    tma_bulk_g2s(sbn_smem + ring_b + sg->copy[k].dst_off, sg->copy[k].src, sg->copy[k].bytes, &s_full[stage]);
            }
            s = s + 1 == n_steps ? 0 : s + 1;
        }
        return;
    }

    // ---------------------------------------------------------------------- compute warps
    StepCtx c;
    c.ring_b = ring_b;
    c.arena_b = arena_b;
    c.scratch = reinterpret_cast<char *>(p.scratch + static_cast<int64_t>(blockIdx.x) * p.scratch_floats);
    c.any_global = reinterpret_cast<const char *>(p.recs);
    c.lane = lane;
    c.warp = warp;
    c.n_warps = n_cw;
    c.n_threads = n_ct;
    int64_t g = 0;
    for (int it = 0; it < my_blocks; ++it) {
        const int rb = static_cast<int>(blockIdx.x) + it * static_cast<int>(gridDim.x);
        c.row = static_cast<int64_t>(rb) * SBN_CHAIN_ROWS + lane;
        c.live = c.row < p.n_rows;
        const int64_t row_c = c.live ? c.row : p.n_rows - 1;  // padding lanes compute on the last valid row's codes
        for (int k = warp; k < p.n_ev; k += n_cw) sbn_smem[k * SBN_CHAIN_ROWS + lane] = p.ev[static_cast<int64_t>(k) * p.ld_ev + row_c];
        bar_compute(n_ct);
        for (int s = 0; s < n_steps; ++s, ++g) {
            const long long t_begin = p.prof ? clock64() : 0;
            const int stage = static_cast<int>(g % kChainStages);
            StepRec rec{rec_b + 4 * lds_u(rec_b + 4 * s), rec_b};
            mbar_wait(&s_full[stage], static_cast<uint32_t>((g / kChainStages) & 1));
            const long long t_wait = p.prof ? clock64() : 0;
            const int fast = rec.fast();
            if (fast == 0) {
                chain_step_generic(rec, c);
            } else {
#define SBN_FAST(TV)                                                  \
    case TV:                                                          \
        if (fast == 1) chain_step_fast<TV, false, false>(rec, c);     \
        else if (fast == 2) chain_step_fast<TV, true, false>(rec, c); \
        else if (fast == 3) chain_step_fast<TV, false, true>(rec, c); \
        else chain_step_fast<TV, true, true>(rec, c);                 \
        break;
                switch (rec.T()) {
                    SBN_FAST(2)
                    SBN_FAST(3)
                    SBN_FAST(4)
                    SBN_FAST(5)
                }
#undef SBN_FAST
            }
            const long long t_work = p.prof ? clock64() : 0;
            bar_compute(n_ct);
            if (threadIdx.x == 0) mbar_arrive(&s_empty[stage]);  // every compute warp has left the stage's tables
            if (p.prof && lane == 0) {
                // per step: [0] cycles of warp 0 from entry to past the barrier, [1] sum over warps of busy cycles
                if (warp == 0) atomicAdd(p.prof + 4 * s, static_cast<unsigned long long>(clock64() - t_begin));
                atomicAdd(p.prof + 4 * s + 1, static_cast<unsigned long long>(t_work - t_begin));
                atomicAdd(p.prof + 4 * s + 2, static_cast<unsigned long long>(t_wait - t_begin));
                if (warp == n_cw - 1) atomicAdd(p.prof + 4 * s + 3, static_cast<unsigned long long>(t_work - t_wait));
            }
        }
        if (p.post_space >= 0) {
            // posterior / posterior.sum() (bayes_net.py:789-790), range-checked like sbn_normalise
            if (warp == 0 && c.live) {
                const bool psm = p.post_space == SBN_SP_SMEM;
                const uint32_t po = (psm ? arena_b : 0u) + p.post_off + lane * 4;
                auto post = [&](int q) -> float {
                    return psm ? lds_f(po + q * (SBN_CHAIN_ROWS * 4)) : ldg_f(c.scratch, po + q * (SBN_CHAIN_ROWS * 4));
                };
                float total = 0.f, lo = p.min_total;
                for (int q = 0; q < p.Q; ++q) {
                    const float v = post(q);
                    total += v;
                    if (v > 0.f && v < lo) lo = v;
                }
                const bool ok = total >= p.min_total && lo >= p.min_total;
                const float nan = __int_as_float(0x7fc00000);
                if (p.totals) p.totals[c.row] = ok ? total : nan;
                for (int q = 0; q < p.Q; ++q) p.out[static_cast<int64_t>(q) * p.ld_out + c.row] = ok ? post(q) / total : nan;
            }
            bar_compute(n_ct);
        }
    }
}

// ------------------------------------------------------------------ host: allocation of homes
// First-fit free list over a range of floats (blocks of whole [entries][32] factors).
struct FreeList {
    struct Block {
        int64_t off, size;
    };
    std::vector<Block> free_;
    int64_t peak = 0;
    explicit FreeList(int64_t capacity) { free_.push_back({0, capacity}); }
    int64_t alloc(int64_t size) {  // -1 when nothing fits
        for (size_t i = 0; i < free_.size(); ++i) {
            if (free_[i].size >= size) {
                const int64_t off = free_[i].off;
                free_[i].off += size;
                free_[i].size -= size;
                if (free_[i].size == 0) free_.erase(free_.begin() + i);
                peak = std::max(peak, off + size);
                return off;
            }
        }
        return -1;
    }
    void release(int64_t off, int64_t size) {
        size_t i = 0;
        while (i < free_.size() && free_[i].off < off) ++i;
        free_.insert(free_.begin() + i, {off, size});
        for (size_t j = 0; j + 1 < free_.size();) {  // coalesce
            if (free_[j].off + free_[j].size == free_[j + 1].off) {
                free_[j].size += free_[j + 1].size;
                free_.erase(free_.begin() + j + 1);
            } else {
                ++j;
            }
        }
    }
};

int env_int(const char *name, int fallback) {
    const char *e = getenv(name);
    return e ? atoi(e) : fallback;
}

int64_t step_table_floats(const sbn_program *P, const StepDesc &st) {
    int64_t t = 0;
    for (const InDesc &in : st.in)
        if (!in.batched) t += in.is_slot ? P->slots[in.id].padded : P->table_padded[in.id];
    return t;
}

// a step the segment kernel can run: planned for the tiled kernel (<= 4 inputs sorted into
// U / A / B / C classes, tile table built), tables small enough to be staged whole
bool chainable(const sbn_program *P, const StepDesc &st, int64_t tab_max) {
    if (st.kind != 1 || st.tile <= 0 || st.big_tables || st.slice_pos >= 0) return false;
    if (st.nu > 2 || st.na > 2 || st.nb > 2 || st.nc > 1 || st.in.size() > 4) return false;
    static const int min_out = env_int("SOROBN_B200_CHAIN_MINOUT", 0), max_out = env_int("SOROBN_B200_CHAIN_MAXOUT", 1 << 30);
    if (st.n_out < min_out || st.n_out > max_out) return false;  // experiments: segments of big-frontier steps only
    return step_table_floats(P, st) <= tab_max;
}

int input_class(const StepDesc &st, int i) { return i < st.nu ? 0 : i < st.nu + st.na ? 1 : i < st.nu + st.na + st.nb ? 2 : 3; }

int chain_grid(const sbn_program *P, const SbnSegment &seg) {
    const int sms = P->n_sms;
    int per_sm = 1;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, sbn_chain_kernel, seg.threads, seg.smem_bytes) != cudaSuccess || per_sm < 1) {
        cudaGetLastError();
        per_sm = 1;
    }
    return sms * per_sm;
}

}  // namespace

void sbn_chain_plan(sbn_program *P) {
    for (SbnSegment *s : P->segments) delete s;
    P->segments.clear();
    P->seg_first.assign(P->steps.size(), -1);
    if (P->mode != 1 || P->f64) return;
    // Segments are planned for every batched program (cheap) but only USED when the program's
    // use_chain switch is on: SOROBN_B200_CHAIN=1 or sbn_program_set_tiled(prog, 7).  The default stays
    // the per-step launches (DESIGN.md "On-chip segments").
    static const int min_steps = env_int("SOROBN_B200_CHAIN_MIN", 4);
    static const int tab_kb = env_int("SOROBN_B200_CHAIN_TAB_KB", 32);  // tables of one step
    const int64_t tab_max = static_cast<int64_t>(tab_kb) * 1024 / 4;
    const int n_steps = static_cast<int>(P->steps.size());

    // consumer of every intermediate (each has exactly one)
    std::vector<int> consumer(n_steps, -1);
    {
        std::vector<int> writer(P->slots.size(), -1);
        for (int s = 0; s < n_steps; ++s) {
            for (const InDesc &in : P->steps[s].in)
                if (in.is_slot && writer[in.id] >= 0) consumer[writer[in.id]] = s;
            writer[P->steps[s].out_slot] = s;
        }
    }

    // runs of chainable batched steps; table-only steps in between were hoisted to program
    // creation and do not break a run, any other batched step does
    std::vector<std::vector<int>> runs(1);
    for (int k = 0; k < n_steps; ++k) {
        const StepDesc &st = P->steps[k];
        if (st.kind == 0) continue;
        if (chainable(P, st, tab_max)) runs.back().push_back(k);
        else if (!runs.back().empty()) runs.emplace_back();
    }
    for (const std::vector<int> &run : runs) {
        if (static_cast<int>(run.size()) < min_steps) continue;
        SbnSegment *seg = new SbnSegment();
        seg->first = run.front();
        seg->last = run.back();
        seg->steps = run;
        // table ring: the tables of SBN_CHAIN_STAGES consecutive steps (cyclically: the row blocks
        // repeat the sequence) must not overlap.  Bump allocation with wrap-around, verified, grown
        // until it holds; a segment shorter than the pipeline gets one fixed slice per stage.
        const int n_run = static_cast<int>(run.size());
        std::vector<int64_t> tbytes(n_run);
        int64_t tmax = 16, rec_words = n_run;
        for (int i = 0; i < n_run; ++i) {
            const StepDesc &st = P->steps[run[i]];
            tbytes[i] = round_up(step_table_floats(P, st) * 4, 16);
            tmax = std::max(tmax, tbytes[i]);
            rec_words += SBN_REC_HDR;
            for (const InDesc &in : st.in) rec_words += SBN_REC_SLOT + 2 * static_cast<int64_t>(in.ev.size());
            rec_words += st.n_tiles * (static_cast<int64_t>(st.in.size()) + 2);
            if (st.zoff_tiled_pos >= 0) rec_words += static_cast<int64_t>(st.in.size()) * st.cx;
        }
        seg->ring_off.assign(n_run, 0);
        if (n_run < SBN_CHAIN_STAGES) {
            // shorter than the pipeline: every step keeps its own region; re-staging it for the next
            // row block rewrites the same bytes (the tables do not depend on the rows)
            int64_t cursor = 0;
            for (int i = 0; i < n_run; ++i) {
                seg->ring_off[i] = cursor;
                cursor += tbytes[i];
            }
            seg->ring_bytes = round_up(std::max<int64_t>(cursor, 16), 16);
        } else {
            int64_t window = 0;
            for (int i = 0; i < n_run; ++i) {
                int64_t w = 0;
                for (int d = 0; d < SBN_CHAIN_STAGES; ++d) w += tbytes[(i + d) % n_run];
                window = std::max(window, w);
            }
            int64_t R = round_up(window, 1024);
            for (;; R += 2048) {
                int64_t cursor = 0;
                for (int i = 0; i < n_run; ++i) {
                    if (cursor + tbytes[i] > R) cursor = 0;
                    seg->ring_off[i] = cursor;
                    cursor += tbytes[i];
                }
                bool ok = true;
                for (int i = 0; i < n_run && ok; ++i)
                    for (int d = 1; d < SBN_CHAIN_STAGES && ok; ++d) {
                        const int j = (i + d) % n_run;
                        const int64_t a0 = seg->ring_off[i], a1 = a0 + tbytes[i], b0 = seg->ring_off[j], b1 = b0 + tbytes[j];
                        if (tbytes[i] > 0 && tbytes[j] > 0 && a0 < b1 && b0 < a1) ok = false;
                    }
                if (ok || R > 128 * 1024) break;
            }
            seg->ring_bytes = R;
        }
        const int64_t ring_bytes = seg->ring_bytes;
        seg->rec_words = round_up(rec_words, 4);
        const int64_t ev_bytes = round_up(static_cast<int64_t>(std::max(P->n_ev, 1)) * SBN_CHAIN_ROWS, 16);
        const int64_t fixed = 256 + ev_bytes + seg->rec_words * 4 + ring_bytes;
        if (fixed + 4 * SBN_CHAIN_ROWS * 4 > SBN_CHAIN_SMEM) {
            delete seg;
            continue;
        }
        const int64_t arena_cap = (SBN_CHAIN_SMEM - fixed) / 4 / SBN_CHAIN_ROWS * SBN_CHAIN_ROWS;
        FreeList arena(arena_cap), scratch(int64_t(1) << 40);
        struct Home {
            int space = SBN_SP_GLOBAL;
            int64_t off = 0, size = 0;
        };
        std::vector<Home> home(n_steps);
        std::vector<int> writer(P->slots.size(), -1);
        for (int k = 0; k < seg->first; ++k) writer[P->steps[k].out_slot] = k;
        auto inside = [&](int w) { return w >= seg->first && P->steps[w].kind == 1; };
        for (int k = seg->first; k <= seg->last; ++k) {
            const StepDesc &st = P->steps[k];
            if (st.kind == 0) {
                writer[st.out_slot] = k;
                continue;
            }
            const bool is_post = k == n_steps - 1;
            const bool internal = is_post || (consumer[k] >= 0 && consumer[k] <= seg->last);
            Home h;
            h.size = st.n_out * SBN_CHAIN_ROWS;
            if (internal) {
                h.off = arena.alloc(h.size);
                h.space = SBN_SP_SMEM;
                if (h.off < 0) {
                    h.off = scratch.alloc(h.size);
                    h.space = SBN_SP_SCRATCH;
                }
            } else {
                seg->hbm_bytes_per_row += st.n_out * 4;
            }
            home[k] = h;
            SbnChainHome ch;
            ch.step = k;
            ch.out_space = h.space;
            ch.out_off = h.off;
            // class slots: U0 U1 | A0 A1 | B0 B1 | C0; st.order lists the inputs U.., A.., B.., C
            int next_slot[4] = {0, 2, 4, 6};
            for (int i = 0; i < static_cast<int>(st.in.size()); ++i) {
                const InDesc &in = st.in[st.order[i]];
                ch.slot[i] = next_slot[input_class(st, i)]++;
                if (!in.batched) {
                    ch.space[i] = SBN_SP_TABLE;
                } else if (writer[in.id] >= 0 && inside(writer[in.id])) {
                    ch.space[i] = home[writer[in.id]].space;
                    ch.off[i] = home[writer[in.id]].off;
                } else {
                    ch.space[i] = SBN_SP_GLOBAL;
                    seg->hbm_bytes_per_row += P->slots[in.id].size * 4;
                }
            }
            seg->homes.push_back(ch);
            for (const InDesc &in : st.in) {  // inputs die with this step (single consumer)
                if (!in.batched) continue;
                const int w = writer[in.id];
                if (w >= 0 && inside(w)) {
                    if (home[w].space == SBN_SP_SMEM) arena.release(home[w].off, home[w].size);
                    else if (home[w].space == SBN_SP_SCRATCH) scratch.release(home[w].off, home[w].size);
                }
            }
            writer[st.out_slot] = k;
            if (is_post) {
                seg->ends_in_posterior = true;
                seg->post_space = h.space;
                seg->post_off = h.off;
            }
        }
        seg->arena_floats = arena.peak;
        seg->scratch_floats = round_up(scratch.peak, 64);
        seg->smem_bytes = static_cast<size_t>(ev_bytes + seg->rec_words * 4 + ring_bytes + seg->arena_floats * 4);
        // warps share the tiles of a step: 13 of them take the 25 tiles of a 625-entry output in two rounds
        int64_t max_tiles = 1;
        for (int k : run) max_tiles = std::max(max_tiles, P->steps[k].n_tiles);
        static const int warps_env = env_int("SOROBN_B200_CHAIN_WARPS", 0);
        int warps = warps_env > 0 ? warps_env : 13;
        if (warps_env <= 0 && max_tiles < warps) warps = static_cast<int>(std::max<int64_t>(2, max_tiles));
        seg->threads = std::min(kChainMaxThreads, (warps + 1) * 32);  // + the producer warp
        for (int k : run) P->seg_first[k] = -2;  // inside a segment, not its head
        P->seg_first[seg->first] = static_cast<int>(P->segments.size());
        P->segments.push_back(seg);
        static const int debug = env_int("SOROBN_B200_CHAIN_DEBUG", 0);
        if (debug) {
            int n_smem = 0, n_scr = 0, n_glob = 0;
            for (const SbnChainHome &ch : seg->homes) {
                n_smem += ch.out_space == SBN_SP_SMEM;
                n_scr += ch.out_space == SBN_SP_SCRATCH;
                n_glob += ch.out_space == SBN_SP_GLOBAL;
            }
            fprintf(stderr, "[sbn_chain] segment %zu: steps %d..%d (%zu batched), outputs smem/scratch/hbm %d/%d/%d, arena %lld B, "
                            "table ring %lld B, scratch %lld B per CTA, %d threads, %zu B smem, hbm %lld B/row\n",
                    P->segments.size() - 1, seg->first, seg->last, seg->steps.size(), n_smem, n_scr, n_glob,
                    (long long)seg->arena_floats * 4, (long long)ring_bytes, (long long)seg->scratch_floats * 4,
                    seg->threads, seg->smem_bytes, (long long)seg->hbm_bytes_per_row);
        }
    }
}

cudaError_t sbn_chain_set_attrs() {
    return cudaFuncSetAttribute(sbn_chain_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SBN_CHAIN_SMEM - 64);
}

// Build the device descriptors: every offset in bytes, premultiplied by the row pitch of the space
// the operand lives in.  Needs the slot arena (pointers, ld), so it runs after sbn_program_reserve.
cudaError_t sbn_chain_bind(sbn_program *P) {
    if (P->segments.empty()) return cudaSuccess;
    P->chain_fits = true;
    int64_t scratch = 0;
    int max_grid = 1;
    for (SbnSegment *seg : P->segments) {
        scratch = std::max(scratch, seg->scratch_floats);
        max_grid = std::max(max_grid, chain_grid(P, *seg));
    }
    cudaFree(P->d_chain_scratch);
    P->d_chain_scratch = nullptr;
    if (scratch > 0) {
        cudaError_t e = cudaMalloc(&P->d_chain_scratch, static_cast<size_t>(scratch) * max_grid * 4);
        if (e != cudaSuccess) return e;
    }
    const int64_t ld = P->ld;
    auto pitch_of = [&](int space) -> int64_t { return space == SBN_SP_TABLE ? 1 : space == SBN_SP_GLOBAL ? ld : SBN_CHAIN_ROWS; };
    for (SbnSegment *seg : P->segments) {
        struct Pitches {
            int64_t out;
            int64_t in[4];
        };
        std::vector<Pitches> pitch_of_step;
        seg->host.assign(seg->homes.size(), SbnChainStep());
        for (size_t idx = 0; idx < seg->homes.size(); ++idx) {
            const SbnChainHome &ch = seg->homes[idx];
            const StepDesc &st = P->steps[ch.step];
            SbnChainStep &cs = seg->host[idx];
            memset(&cs, 0, sizeof cs);
            const int n_in = static_cast<int>(st.in.size());
            const int64_t out_pitch = pitch_of(ch.out_space);
            cs.out_ptr = P->slots[st.out_slot].ptr;
            cs.out_space = ch.out_space;
            cs.out_off = static_cast<uint32_t>(ch.out_off * 4);
            cs.out_eb = static_cast<uint32_t>(out_pitch * 4);
            cs.out_c0b = static_cast<uint32_t>((st.cards.empty() ? 1 : st.cards[0]) * out_pitch * 4);
            if (ch.out_space == SBN_SP_GLOBAL && st.n_out * ld * 4 >= (int64_t(1) << 32)) P->chain_fits = false;
            cs.T = st.tile;
            cs.cx = st.cx;
            cs.n_in = n_in;
            cs.n_tiles = static_cast<int32_t>(st.n_tiles);
            int64_t tab_off = 0;
            int64_t pitch[4] = {1, 1, 1, 1};
            for (int i = 0; i < n_in; ++i) {
                const InDesc &in = st.in[st.order[i]];
                SbnChainIn &ci = cs.in[ch.slot[i]];
                cs.present |= 1 << ch.slot[i];
                pitch[i] = pitch_of(ch.space[i]);
                ci.space = ch.space[i];
                ci.col = i;
                ci.sxb = static_cast<uint32_t>(in.sx * pitch[i] * 4);
                ci.sab = static_cast<uint32_t>((in.strides.size() > 0 ? in.strides[0] : 0) * pitch[i] * 4);
                ci.sbb = static_cast<uint32_t>((in.strides.size() > 1 ? in.strides[1] : 0) * pitch[i] * 4);
                ci.n_ev = static_cast<int32_t>(in.ev.size());
                for (size_t a = 0; a < in.ev.size(); ++a) {
                    ci.ev_col[a] = in.ev[a].col;
                    ci.ev_stride_b[a] = static_cast<uint32_t>(in.ev[a].stride * 4);
                    ci.ev_card[a] = in.ev[a].card;
                }
                if (ch.space[i] == SBN_SP_TABLE) {
                    const int64_t padded = in.is_slot ? P->slots[in.id].padded : P->table_padded[in.id];
                    ci.ptr = in.is_slot ? P->slots[in.id].ptr : P->d_tables + P->tables[in.id].first;
                    ci.off = static_cast<uint32_t>(seg->ring_off[idx] + tab_off * 4);
                    ci.stage_bytes = static_cast<int32_t>(padded * 4);
                    tab_off += padded;
                } else if (ch.space[i] == SBN_SP_GLOBAL) {
                    ci.ptr = P->slots[in.id].ptr;
                    if (P->slots[in.id].size * ld * 4 >= (int64_t(1) << 32)) P->chain_fits = false;
                } else {
                    ci.off = static_cast<uint32_t>(ch.off[i] * 4);
                }
            }
            cs.table_bytes = static_cast<int32_t>(tab_off * 4);
            {
                // specialised shape?  (see chain_step_fast)
                const int T = st.tile;
                bool ok = st.nc == 0 && st.na >= 1 && st.nb >= 1 && st.cards.size() >= 2 && !st.ecards.empty() &&
                          st.ecards[0] == T && st.cards[0] % T == 0 && st.cards[1] % T == 0;
                int fast = 1;  // 1 + (A0 outside shared memory) + 2 * (B0 outside shared memory)
                for (int i = 0; i < n_in && ok; ++i) {
                    const bool gmem = ch.space[i] == SBN_SP_GLOBAL || ch.space[i] == SBN_SP_SCRATCH;
                    if (gmem && ch.slot[i] == 2) fast += 1;
                    else if (gmem && ch.slot[i] == 4) fast += 2;
                    else if (gmem) ok = false;
                }
                static const int fast_env = env_int("SOROBN_B200_CHAIN_FAST", 1);
                cs.fast = ok && fast_env ? fast : 0;
            }
            pitch_of_step.push_back({out_pitch, {pitch[0], pitch[1], pitch[2], pitch[3]}});
        }
        cudaError_t e = cudaSuccess;
        // step records for the compute warps and staging lists for the producer lane
        const int n_cw = seg->threads / 32 - 1;
        std::vector<uint32_t> recs(seg->host.size(), 0);
        std::vector<SbnChainStage> stages(seg->host.size());
        auto put64 = [](std::vector<uint32_t> &v, size_t at, const void *ptr) {
            const uint64_t u = reinterpret_cast<uint64_t>(ptr);
            v[at] = static_cast<uint32_t>(u);
            v[at + 1] = static_cast<uint32_t>(u >> 32);
        };
        for (size_t idx = 0; idx < seg->host.size(); ++idx) {
            const SbnChainStep &cs = seg->host[idx];
            const size_t at = recs.size();
            recs[idx] = static_cast<uint32_t>(at);
            recs.resize(at + SBN_REC_HDR, 0);
            int ks = 1;
            if (cs.fast == 0 && cs.n_tiles * 2 <= n_cw && cs.cx >= 16) ks = std::max(1, std::min(n_cw / cs.n_tiles, cs.cx / 4));
            static const int split_env = env_int("SOROBN_B200_CHAIN_SPLIT", 1);
            if (!split_env) ks = 1;
            recs[at + 0] = static_cast<uint32_t>(cs.fast | cs.T << 3 | cs.out_space << 6 | cs.n_in << 9);
            recs[at + 1] = static_cast<uint32_t>(cs.present);
            recs[at + 2] = static_cast<uint32_t>(cs.cx);
            recs[at + 3] = static_cast<uint32_t>(cs.n_tiles);
            recs[at + 4] = cs.out_off;
            recs[at + 5] = cs.out_eb;
            recs[at + 6] = cs.out_c0b;
            recs[at + 7] = static_cast<uint32_t>(ks);
            put64(recs, at + 8, cs.out_ptr);
            SbnChainStage &sg = stages[idx];
            memset(&sg, 0, sizeof sg);
            for (int k = 0; k < SBN_CHAIN_SLOTS; ++k) {
                if (!((cs.present >> k) & 1)) continue;
                const SbnChainIn &ci = cs.in[k];
                const size_t sw = recs.size();
                if (sw - at > 255) return cudaErrorInvalidValue;
                recs[at + 14 + (k >> 2)] |= static_cast<uint32_t>(sw - at) << (8 * (k & 3));
                recs.resize(sw + SBN_REC_SLOT + 2 * ci.n_ev, 0);
                recs[sw + 0] = static_cast<uint32_t>(ci.space | ci.col << 4 | ci.n_ev << 8);
                recs[sw + 1] = ci.off;
                recs[sw + 2] = ci.sxb;
                recs[sw + 3] = ci.sab;
                recs[sw + 4] = ci.sbb;
                put64(recs, sw + 5, ci.ptr);
                for (int a = 0; a < ci.n_ev; ++a) {
                    recs[sw + SBN_REC_SLOT + 2 * a] = static_cast<uint32_t>(ci.ev_col[a]) | static_cast<uint32_t>(ci.ev_card[a]) << 16;
                    recs[sw + SBN_REC_SLOT + 2 * a + 1] = ci.ev_stride_b[a];
                }
                if (ci.space == SBN_SP_TABLE) {
                    sg.copy[sg.n].src = ci.ptr;
                    sg.copy[sg.n].dst_off = ci.off;
                    sg.copy[sg.n].bytes = static_cast<uint32_t>(ci.stage_bytes);
                    sg.bytes += static_cast<uint32_t>(ci.stage_bytes);
                    sg.n++;
                }
            }
        }
        // tile rows and joint-state offsets, in bytes, behind the records (all of it lives in shared memory)
        for (size_t idx = 0; idx < seg->host.size(); ++idx) {
            const StepDesc &st = P->steps[seg->homes[idx].step];
            const Pitches &pt = pitch_of_step[idx];
            const int n_in = static_cast<int>(st.in.size());
            const size_t at = recs[idx];
            recs[at + 10] = static_cast<uint32_t>(recs.size() * 4);
            const int32_t *src = P->h_tile_words.data() + st.tile_off_pos;
            for (int64_t t = 0; t < st.n_tiles; ++t) {
                const int32_t *r = src + t * (n_in + 2);
                recs.push_back(static_cast<uint32_t>(static_cast<int64_t>(r[0]) * pt.out * 4));
                recs.push_back(static_cast<uint32_t>(r[1]));
                for (int i = 0; i < n_in; ++i) recs.push_back(static_cast<uint32_t>(static_cast<int64_t>(r[2 + i]) * pt.in[i] * 4));
            }
            if (st.zoff_tiled_pos >= 0) {
                recs[at + 11] = static_cast<uint32_t>(recs.size() * 4);
                const int32_t *z = P->h_tile_words.data() + st.zoff_tiled_pos;
                for (int i = 0; i < n_in; ++i)
                    for (int x = 0; x < st.cx; ++x) recs.push_back(static_cast<uint32_t>(static_cast<int64_t>(z[i * st.cx + x]) * pt.in[i] * 4));
            }
        }
        if (static_cast<int64_t>(recs.size()) > seg->rec_words) return cudaErrorInvalidValue;
        recs.resize(static_cast<size_t>(seg->rec_words), 0);
        cudaFree(seg->d_recs);
        cudaFree(seg->d_stages);
        seg->d_recs = nullptr;
        seg->d_stages = nullptr;
        e = cudaMalloc(&seg->d_recs, recs.size() * 4);
        if (e != cudaSuccess) return e;
        e = cudaMalloc(&seg->d_stages, stages.size() * sizeof(SbnChainStage));
        if (e != cudaSuccess) return e;
        e = cudaMemcpyAsync(seg->d_recs, recs.data(), recs.size() * 4, cudaMemcpyHostToDevice, P->stream);
        if (e != cudaSuccess) return e;
        e = cudaMemcpyAsync(seg->d_stages, stages.data(), stages.size() * sizeof(SbnChainStage), cudaMemcpyHostToDevice, P->stream);
        if (e != cudaSuccess) return e;
        e = cudaStreamSynchronize(P->stream);  // the host vectors die with this iteration
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

cudaError_t sbn_chain_launch(sbn_program *P, const SbnSegment &seg, const uint8_t *d_ev, int64_t ld_ev, int64_t n_rows,
                             float *d_out, int64_t ld_out, cudaStream_t stream) {
    SbnChainParams q;
    memset(&q, 0, sizeof q);
    q.recs = seg.d_recs;
    q.stages = seg.d_stages;
    q.rec_words = static_cast<int32_t>(seg.rec_words);
    q.n_steps = static_cast<int32_t>(seg.host.size());
    q.n_ev = P->n_ev;
    q.ev = d_ev;
    q.ld_ev = ld_ev;
    q.ld = P->ld;
    q.n_rows = static_cast<int32_t>(n_rows);
    q.n_rblocks = static_cast<int32_t>((n_rows + SBN_CHAIN_ROWS - 1) / SBN_CHAIN_ROWS);
    q.scratch = P->d_chain_scratch;
    q.scratch_floats = seg.scratch_floats;
    q.ev_bytes = static_cast<int32_t>(round_up(static_cast<int64_t>(std::max(P->n_ev, 1)) * SBN_CHAIN_ROWS, 16));
    q.ring_bytes = static_cast<int32_t>(seg.ring_bytes);
    q.post_space = seg.ends_in_posterior ? seg.post_space : -1;
    q.post_off = static_cast<uint32_t>(seg.post_off * 4);
    q.Q = P->Q;
    q.min_total = 1e-30f;
    q.out = d_out;
    q.ld_out = ld_out;
    q.totals = P->d_total;
    const int grid = static_cast<int>(std::min<int64_t>(chain_grid(P, seg), q.n_rblocks));
    static const int prof = env_int("SOROBN_B200_CHAIN_PROF", 0);
    if (prof) {  // developer aid: per-step cycle counts, printed after the launch (synchronises!)
        unsigned long long *d_prof = nullptr;
        const size_t n = seg.host.size() * 4;
        cudaMalloc(&d_prof, n * 8);
        cudaMemsetAsync(d_prof, 0, n * 8, stream);
        q.prof = d_prof;
        sbn_chain_kernel<<<grid, seg.threads, seg.smem_bytes, stream>>>(q);
        std::vector<unsigned long long> h(n);
        cudaMemcpyAsync(h.data(), d_prof, n * 8, cudaMemcpyDeviceToHost, stream);
        cudaStreamSynchronize(stream);
        cudaFree(d_prof);
        const double per_cta = static_cast<double>((q.n_rblocks + grid - 1) / grid) * grid;
        double tot = 0;
        for (size_t i = 0; i < seg.host.size(); ++i) tot += h[4 * i] / per_cta;
        fprintf(stderr, "[sbn_chain] per-step cycles per row block (warp 0 wall | mean busy per warp | mean table wait | last warp's step function), total %.0f\n", tot);
        for (size_t i = 0; i < seg.host.size(); ++i) {
            const SbnChainStep &cs = seg.host[i];
            fprintf(stderr, "  step %3d fast=%d T=%d cx=%3d tiles=%4d present=0x%02x out_space=%d  %8.0f | %8.0f | %8.0f | %8.0f\n", seg.steps[i], cs.fast,
                    cs.T, cs.cx, cs.n_tiles, cs.present, cs.out_space, h[4 * i] / per_cta,
                    h[4 * i + 1] / per_cta / (seg.threads / 32 - 1), h[4 * i + 2] / per_cta / (seg.threads / 32 - 1), h[4 * i + 3] / per_cta);
        }
        return cudaGetLastError();
    }
    sbn_chain_kernel<<<grid, seg.threads, seg.smem_bytes, stream>>>(q);
    return cudaGetLastError();
}

void sbn_chain_free(sbn_program *P) {
    for (SbnSegment *seg : P->segments) {
        cudaFree(seg->d_recs);
        cudaFree(seg->d_stages);
        delete seg;
    }
    P->segments.clear();
    cudaFree(P->d_chain_scratch);
    P->d_chain_scratch = nullptr;
}
