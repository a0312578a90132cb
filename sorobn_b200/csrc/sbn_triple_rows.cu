// sorobn_b200 -- row-block variant of the expanding product (see sbn_pair.h, SbnTripleRows).
#include <cuda.h>

#include <algorithm>
#include <cstdlib>
#include <cstring>

#include "sbn_internal.h"
#include "sbn_kernels.cuh"
#include "sbn_launch.h"
#include "sbn_pair.h"
#include "sbn_tma.h"

namespace {

constexpr int kT = SBN_PAIR_T;
constexpr int kR = SBN_TRIPLE_ROWS_R;
constexpr int kCombos = SBN_TRIPLE_ROWS_COMBOS;
constexpr int kStages = 8;                                      // ring depth: 8 x 24 KB
constexpr int kBoxFloats = 2016;                                // kT^3 x kR = 2000 floats, rounded up to 128 B
constexpr int kStageFloats = 3 * kBoxFloats;                    // one box each of A, B, C
constexpr int kThreads = ((kR * kCombos + 31) / 32 + 1) * 32;   // consumer warps + the producer warp
constexpr size_t kSmem = static_cast<size_t>(kStages) * kStageFloats * 4;

struct SbnTripleRowsParams {
    CUtensorMap tm[3];             // A, B, C: view (row, e1, e2, p, u), box (R, T, T, 1, u digits)
    float *out;
    int64_t ld;
    int32_t n_rows, n_blocks, n_combos;
    uint32_t stage_bytes;          // bytes the three boxes of one stage deliver
    int32_t o_z, o_s;              // entry strides of z and s in the output
    int32_t uoff[3][kCombos];      // float offset of combination c's T x T block inside the operand's box
    int32_t o_off[kCombos];        // output entry of combination c at z = s = 0
};

__device__ __forceinline__ void tma_5d(float *dst, const CUtensorMap *map, int32_t row, int32_t p, uint64_t *bar) {
    asm volatile(
        "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %4, %5, %4}], [%2];" ::"r"(
            sbn_smem_u32(dst)),
        "l"(reinterpret_cast<uint64_t>(map)), "r"(sbn_smem_u32(bar)), "r"(row), "r"(0), "r"(p)
        : "memory");
}

__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(sbn_smem_u32(bar)) : "memory");
}

// Dynamic shared memory: kStages stages of [A box][B box][C box]; a box is [u][e2][e1][R rows] (p fixed), so
// X[e2][e1] of combination c and row r sits at uoff[X][c] + (e2 * T + e1) * R + r:
//   A[k][j]: e1 = j, e2 = k      B[j][s]: e1 = s, e2 = j      C[k][z]: e1 = z, e2 = k
// Warps 0 .. kThreads / 32 - 2 compute (thread = row r x combination c, R rows per combination); the last warp
// issues the boxes, one stage per (row block, p), as soon as the consumer warps have released the stage.
__global__ void __launch_bounds__(kThreads, 1) sbn_triple_rows_kernel(const __grid_constant__ SbnTripleRowsParams p) {
    constexpr int T = kT, R = kR;
    extern __shared__ __align__(128) float s_mem[];
    __shared__ __align__(8) uint64_t s_full[kStages], s_empty[kStages];
    sbn_pdl_launch_dependents();
    const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
    const int n_consumers = static_cast<int>(blockDim.x) / 32 - 1;
    if (threadIdx.x == 0) {
#pragma unroll
        for (int k = 0; k < kStages; ++k) {
            sbn_mbar_init(&s_full[k], 1);
            sbn_mbar_init(&s_empty[k], static_cast<uint32_t>(n_consumers));
        }
        sbn_fence_mbar_init();
    }
    __syncthreads();
    // the operands were written, and the output may still be read, by earlier launches of this run
    sbn_pdl_wait();

    if (warp == n_consumers) {
        if (lane == 0) {
            int it = 0;
            for (int blk = blockIdx.x; blk < p.n_blocks; blk += gridDim.x)
                for (int pp = 0; pp < T; ++pp, ++it) {
                    const int stage = it % kStages;
                    if (it >= kStages) sbn_mbar_wait(&s_empty[stage], static_cast<uint32_t>((it / kStages - 1) & 1));
                    float *const dst = s_mem + stage * kStageFloats;
                    sbn_mbar_expect_tx(&s_full[stage], p.stage_bytes);
#pragma unroll
                    for (int m = 0; m < 3; ++m) tma_5d(dst + m * kBoxFloats, &p.tm[m], blk * R, pp, &s_full[stage]);
                }
        }
        return;
    }

    // the lanes past R x n_combos (a partial last consumer warp) repeat the last combination and store nothing
    const int r = threadIdx.x % R;
    const int c = min(static_cast<int>(threadIdx.x) / R, p.n_combos - 1);
    const bool active = static_cast<int>(threadIdx.x) < R * p.n_combos;
    const int ua = p.uoff[0][c] + r, ub = kBoxFloats + p.uoff[1][c] + r, uc = 2 * kBoxFloats + p.uoff[2][c] + r;
    // element offsets fit 32 bits (sbn_pair_fits)
    const uint32_t ld = static_cast<uint32_t>(p.ld);
    const uint32_t ob = static_cast<uint32_t>(p.o_off[c]) * ld, oz = static_cast<uint32_t>(p.o_z) * ld,
                   os = static_cast<uint32_t>(p.o_s) * ld;
    int it = 0;
    for (int blk = blockIdx.x; blk < p.n_blocks; blk += gridDim.x) {
        float acc[T][T];  // [z][s]
#pragma unroll
        for (int z = 0; z < T; ++z)
#pragma unroll
            for (int s = 0; s < T; ++s) acc[z][s] = 0.f;
#pragma unroll 1
        for (int pp = 0; pp < T; ++pp, ++it) {
            const int stage = it % kStages;
            const float *const sm = s_mem + stage * kStageFloats;
            sbn_mbar_wait(&s_full[stage], static_cast<uint32_t>((it / kStages) & 1));
            // sbn_triple_kernel's loop body, operation for operation, on the shared-memory copies
            float A[T][T], B[T][T], C[T][T];  // A[k][j]  B[j][s]  C[k][z]
#pragma unroll
            for (int j = 0; j < T; ++j)
#pragma unroll
                for (int s = 0; s < T; ++s) B[j][s] = sm[ub + (j * T + s) * R];
#pragma unroll
            for (int k = 0; k < T; ++k)
#pragma unroll
                for (int j = 0; j < T; ++j) A[k][j] = sm[ua + (k * T + j) * R];
#pragma unroll
            for (int k = 0; k < T; ++k)
#pragma unroll
                for (int z = 0; z < T; ++z) C[k][z] = sm[uc + (k * T + z) * R];
            // every value of this stage is in registers: release it to the producer
            __syncwarp();
            if (lane == 0) mbar_arrive(&s_empty[stage]);
#pragma unroll
            for (int k = 0; k < T; ++k) {
                float n[T];  // N[k][s] = sum_j A[k][j] B[j][s]
#pragma unroll
                for (int s = 0; s < T; ++s) {
                    float v = A[k][0] * B[0][s];
#pragma unroll
                    for (int j = 1; j < T; ++j) v = fmaf(A[k][j], B[j][s], v);
                    n[s] = v;
                }
#pragma unroll
                for (int z = 0; z < T; ++z)
#pragma unroll
                    for (int s = 0; s < T; ++s) acc[z][s] = fmaf(C[k][z], n[s], acc[z][s]);
            }
        }
        const int b = blk * R + r;
        if (active && b < p.n_rows) {
            float *const op = p.out + b;
#pragma unroll
            for (int z = 0; z < T; ++z)
#pragma unroll
                for (int s = 0; s < T; ++s) __stcs(op + (ob + z * oz + s * os), acc[z][s]);
        }
    }
}

// The digit of one operand's extra axis per combination: offs[c] = dig[c] x stride, dig < T.  false when the
// offsets are not of that form.
bool walk_axis(const int64_t *offs, int n, int32_t *card, int32_t *stride, int32_t *dig) {
    int64_t st = 0;
    for (int c = 0; c < n; ++c)
        if (offs[c] < 0) return false;
        else if (offs[c] > 0 && (st == 0 || offs[c] < st)) st = offs[c];
    int32_t top = 0;
    for (int c = 0; c < n; ++c) {
        const int64_t d = st > 0 ? offs[c] / st : 0;
        if (st > 0 && offs[c] % st != 0) return false;
        if (d >= kT) return false;
        dig[c] = static_cast<int32_t>(d);
        top = std::max(top, dig[c]);
    }
    *card = top + 1;
    *stride = static_cast<int32_t>(st > 0 ? st : 1);
    return true;
}

bool rows_enabled() {
    // read at every launch (not cached), so that an A/B run can switch it between two graph captures
    const char *e = getenv("SOROBN_B200_TRIPLE_ROWS");
    return e ? atoi(e) != 0 : true;
}

}  // namespace

void sbn_triple_rows_plan(const SbnTripleParams &q, const int32_t *tiles, SbnTripleRows *rows) {
    memset(rows, 0, sizeof *rows);
    const int64_t n = static_cast<int64_t>(q.n_tiles) * q.group;
    if (n < SBN_TRIPLE_ROWS_MIN_COMBOS || n > kCombos) return;
    const int nc = static_cast<int>(n);
    int64_t offs[3][kCombos];
    for (int c = 0; c < nc; ++c) {
        const int t = c % q.n_tiles, g = c / q.n_tiles;
        offs[0][c] = static_cast<int64_t>(tiles[4 * t + 1]) + static_cast<int64_t>(g) * q.a_g;
        offs[1][c] = tiles[4 * t + 2];
        offs[2][c] = tiles[4 * t + 3];
        rows->o_off[c] = static_cast<int32_t>(tiles[4 * t] + static_cast<int64_t>(g) * q.o_g);
    }
    for (int m = 0; m < 3; ++m)
        if (!walk_axis(offs[m], nc, &rows->u_card[m], &rows->u_stride[m], rows->u_dig[m])) return;
    rows->n_combos = nc;
    rows->ok = 1;
}

cudaError_t sbn_triple_rows_set_attrs() {
    return cudaFuncSetAttribute(sbn_triple_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kSmem));
}

bool sbn_triple_rows_launch(const sbn_program *P, const SbnTripleRows &rows, const SbnTripleParams &q, cudaStream_t stream) {
    if (!rows.ok || !rows_enabled()) return false;
    const int64_t n_blocks = (static_cast<int64_t>(q.n_rows) + kR - 1) / kR;
    // fewer blocks than two per SM: sbn_triple_kernel's many small CTAs fill the GPU better
    if (n_blocks < 2LL * P->n_sms) return false;
    SbnTripleRowsParams p;
    memset(&p, 0, sizeof p);
    // per operand: (e1, e2, p) strides in the kernel's box order, then the axis the combinations walk
    const float *const base[3] = {q.a, q.b, q.c};
    const int64_t strides[3][4] = {{q.a_j, q.a_k, q.a_p, rows.u_stride[0]},
                                   {q.b_s, q.b_j, q.b_p, rows.u_stride[1]},
                                   {q.c_z, q.c_k, q.c_p, rows.u_stride[2]}};
    uint32_t bytes = 0;
    for (int m = 0; m < 3; ++m) {
        const int64_t dims[4] = {kT, kT, kT, rows.u_card[m]};
        const int box[4] = {kT, kT, 1, rows.u_card[m]};
        if (!sbn_tma_encode_view(&p.tm[m], base[m], q.ld, q.n_rows, 4, dims, strides[m], box, kR)) return false;
        bytes += static_cast<uint32_t>(kR * kT * kT * rows.u_card[m] * 4);
        for (int c = 0; c < rows.n_combos; ++c) p.uoff[m][c] = rows.u_dig[m][c] * kT * kT * kR;
    }
    p.out = q.out;
    p.ld = q.ld;
    p.n_rows = q.n_rows;
    p.n_blocks = static_cast<int32_t>(n_blocks);
    p.n_combos = rows.n_combos;
    p.stage_bytes = bytes;
    p.o_z = q.o_z;
    p.o_s = q.o_s;
    for (int c = 0; c < rows.n_combos; ++c) p.o_off[c] = rows.o_off[c];
    const dim3 g(static_cast<unsigned>(std::min<int64_t>(n_blocks, P->n_sms)));
    const dim3 b(static_cast<unsigned>(((kR * rows.n_combos + 31) / 32 + 1) * 32));
    sbn_launch(sbn_triple_rows_kernel, g, b, kSmem, stream, p);
    return true;
}
