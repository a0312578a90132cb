// sorobn_b200 -- an expanding product contracted by its consumer in one launch (sbn_pair.h, SbnContractParams).
#include <algorithm>

#include "sbn_kernels.cuh"
#include "sbn_launch.h"
#include "sbn_pair.h"

namespace {

constexpr int kR = SBN_CONTRACT_R;
constexpr int kT = SBN_PAIR_T;
constexpr int kMaxThreads = kR * SBN_CONTRACT_MAX_WARPS;
constexpr size_t kSmemMax = static_cast<size_t>(SBN_CONTRACT_MAX_OPERAND) * kR * 4 + static_cast<size_t>(SBN_CONTRACT_MAX_E) * 16;

__device__ __forceinline__ void cp_async16(float *dst, const float *src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(sbn_smem_u32(dst)), "l"(src) : "memory");
}

// CTA = kR evidence rows x n_tiles x kz outputs, CJ = states of step 1's eliminated variable; thread (threadIdx.x = row, threadIdx.y = tile x kz + z digit).
// Dynamic shared memory: A, B, C columns [entry][kR], then the joint-state table [n_e] x int4.
template <bool PROD2, int CJ>
__global__ void __launch_bounds__(kMaxThreads) sbn_contract_kernel(const __grid_constant__ SbnContractParams p) {
    extern __shared__ __align__(16) float s_mem[];
    sbn_pdl_launch_dependents();
    const int n_cols = p.n_a + p.n_b + p.n_c;
    const float *const s_a = s_mem;
    const float *const s_b = s_a + p.n_a * kR;
    const float *const s_c = s_b + p.n_b * kR;
    int4 *const s_e = reinterpret_cast<int4 *>(s_mem + n_cols * kR);
    const int tid = threadIdx.y * kR + threadIdx.x;
    const int n_thr = kR * static_cast<int>(blockDim.y);
    // the offset tables were written when the program was created, not by any launch of the run
    const int4 *const words = reinterpret_cast<const int4 *>(p.words);
    for (int i = tid; i < p.n_e; i += n_thr) s_e[i] = __ldg(words + i);
    const int tile = threadIdx.y / p.kz, z = threadIdx.y % p.kz;
    const int4 tw = __ldg(words + p.n_e + tile);
    const int64_t b0 = static_cast<int64_t>(blockIdx.x) * kR;
    sbn_pdl_wait();

    // the block's rows of every operand entry: kR / 4 16-byte pieces per entry, each from HBM once (the row pitch
    // is a multiple of kR, so the rows past n_rows are still inside it; their results are not stored)
    constexpr int kPieces = kR / 4;
    for (int i = tid; i < n_cols * kPieces; i += n_thr) {
        const int col = i / kPieces, piece = i % kPieces;
        const float *src = col < p.n_a ? p.a + static_cast<int64_t>(col) * p.ld
                           : col < p.n_a + p.n_b ? p.b + static_cast<int64_t>(col - p.n_a) * p.ld
                                                 : p.c + static_cast<int64_t>(col - p.n_a - p.n_b) * p.ld;
        cp_async16(s_mem + col * kR + piece * 4, src + b0 + piece * 4);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncthreads();

    const int r = threadIdx.x;
    const int64_t b = b0 + r;
    if (b >= p.n_rows) return;
    const float *const rb = s_b + tw.y + z * p.b_z + r;
    const float *const rc = s_c + tw.z + z * p.c_z + r;
    // per j: this thread's column of A, and its B entry at j (j x the column stride folded in once)
    const float *ra[CJ];
    int bj[CJ];
#pragma unroll
    for (int j = 0; j < CJ; ++j) ra[j] = s_a + tw.x + r + j * p.a_j, bj[j] = j * p.b_j;
    float acc = 0.f, bv[CJ];
#pragma unroll
    for (int j = 0; j < CJ; ++j) bv[j] = 0.f;
    // A and C are read at every joint state (on the grid they move at every one); B only when the state moves it.
    // No branch depends on an earlier load, so the unrolled iterations issue their loads ahead of the arithmetic.
    int pb = -1;
#pragma unroll 4
    for (int e = 0; e < p.n_e; ++e) {
        const int4 w = s_e[e];
        float av[CJ];
#pragma unroll
        for (int j = 0; j < CJ; ++j) av[j] = ra[j][w.x];
        const float cv = rc[w.z];
        const bool moved = w.y != pb;
        pb = w.y;
#pragma unroll
        for (int j = 0; j < CJ; ++j)
            if (moved) bv[j] = rb[w.y + bj[j]];
        // step 1's entry M[o, e]: the tiled kernel's chain over j, from 0.f
        float m = 0.f;
#pragma unroll
        for (int j = 0; j < CJ; ++j) m = fmaf(av[j], bv[j], m);
        // step 2's term: the tiled kernel's a[d] = M x C (both on the A side), then fmaf(a, 1.f, acc) -- or M and C
        // on different sides: fmaf(M, C, acc)
        if constexpr (PROD2) acc = fmaf(__fmul_rn(m, cv), 1.f, acc);
        else acc = fmaf(m, cv, acc);
    }
    __stcs(p.out + static_cast<int64_t>(tw.w + z * p.o_z) * p.ld + b, acc);
}

}  // namespace

cudaError_t sbn_contract_launch(const SbnContractParams &q, cudaStream_t stream) {
    const int64_t grid = (static_cast<int64_t>(q.n_rows) + kR - 1) / kR;
    if (grid >= (1LL << 31)) return cudaErrorInvalidConfiguration;
    const size_t smem = static_cast<size_t>(q.n_a + q.n_b + q.n_c) * kR * 4 + static_cast<size_t>(q.n_e) * 16;
    const dim3 g(static_cast<unsigned>(grid)), b(kR, q.n_tiles * q.kz);
#define SBN_CONTRACT_CASE(J)                                                      \
    case J:                                                                       \
        if (q.prod2) sbn_launch(sbn_contract_kernel<true, J>, g, b, smem, stream, q);  \
        else sbn_launch(sbn_contract_kernel<false, J>, g, b, smem, stream, q);         \
        break;
    switch (q.cj) {
        SBN_CONTRACT_CASE(2)
        SBN_CONTRACT_CASE(3)
        SBN_CONTRACT_CASE(4)
        SBN_CONTRACT_CASE(5)
        default: return cudaErrorInvalidValue;
    }
#undef SBN_CONTRACT_CASE
    return cudaGetLastError();
}

template <bool PROD2, int CJ>
static cudaError_t set_attr() {
    return cudaFuncSetAttribute(sbn_contract_kernel<PROD2, CJ>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kSmemMax));
}

cudaError_t sbn_contract_set_attrs() {
    cudaError_t e = cudaSuccess;
    for (cudaError_t r : {set_attr<true, 2>(), set_attr<true, 3>(), set_attr<true, 4>(), set_attr<true, 5>(), set_attr<false, 2>(),
                          set_attr<false, 3>(), set_attr<false, 4>(), set_attr<false, 5>()})
        if (e == cudaSuccess) e = r;
    return e;
}
