// sorobn_b200 -- step-kernel instantiations: one input spans both tile axes (NC = 1), and the plain batched kernel
// (one of four translation units that share the ~290 instantiations of sbn_step_tiled; see sbn_launch.h)
#include "sbn_launch_impl.cuh"

cudaError_t sbn_tiled_c_launch(int key, const SbnStep &q, int tile, bool preload, int64_t grid, cudaStream_t stream) {
    switch (key) {
        case 1: return launch_tiled_c<0, 0, 0, 1>(q, tile, preload, grid, stream);
        case 11: return launch_tiled_c<0, 0, 1, 1>(q, tile, preload, grid, stream);
        case 101: return launch_tiled_c<0, 1, 0, 1>(q, tile, preload, grid, stream);
        case 111: return launch_tiled_c<0, 1, 1, 1>(q, tile, preload, grid, stream);
        case 1001: return launch_tiled_c<1, 0, 0, 1>(q, tile, preload, grid, stream);
        case 1011: return launch_tiled_c<1, 0, 1, 1>(q, tile, preload, grid, stream);
        case 1101: return launch_tiled_c<1, 1, 0, 1>(q, tile, preload, grid, stream);
        case 1111: return launch_tiled_c<1, 1, 1, 1>(q, tile, preload, grid, stream);
    }
    return cudaErrorInvalidValue;
}

cudaError_t sbn_tiled_c_set_attrs() {
    cudaError_t e = cudaSuccess;
    if (e == cudaSuccess) e = set_tiled_attr_c<0, 0, 0, 1>();
    if (e == cudaSuccess) e = set_tiled_attr_c<0, 0, 1, 1>();
    if (e == cudaSuccess) e = set_tiled_attr_c<0, 1, 0, 1>();
    if (e == cudaSuccess) e = set_tiled_attr_c<0, 1, 1, 1>();
    if (e == cudaSuccess) e = set_tiled_attr_c<1, 0, 0, 1>();
    if (e == cudaSuccess) e = set_tiled_attr_c<1, 0, 1, 1>();
    if (e == cudaSuccess) e = set_tiled_attr_c<1, 1, 0, 1>();
    if (e == cudaSuccess) e = set_tiled_attr_c<1, 1, 1, 1>();
    return e;
}

cudaError_t sbn_batched_launch(const SbnStep &q, int64_t grid, cudaStream_t stream) {
    switch (q.n_in) {
        case 1: return launch_batched_n<1>(q, grid, stream);
        case 2: return launch_batched_n<2>(q, grid, stream);
        case 3: return launch_batched_n<3>(q, grid, stream);
        case 4: return launch_batched_n<4>(q, grid, stream);
        case 5: return launch_batched_n<5>(q, grid, stream);
        case 6: return launch_batched_n<6>(q, grid, stream);
        case 7: return launch_batched_n<7>(q, grid, stream);
        case 8: return launch_batched_n<8>(q, grid, stream);
    }
    return cudaErrorInvalidValue;
}

// The log-domain instantiations: max-sum (MPE programs, and the MAP buckets of marginal MAP programs) and
// log-sum-exp (the summed buckets of marginal MAP programs), the generic eliminated-state loop only
namespace {
template <int N_IN, typename R>
cudaError_t launch_batched_policy_n(const SbnStep &q, int64_t grid, cudaStream_t stream) {
    sbn_launch(sbn_step_batched<N_IN, 0, R>, dim3(static_cast<unsigned>(grid)), dim3(SBN_THREADS),
               static_cast<size_t>(q.smem_floats) * 4, stream, q);
    return cudaGetLastError();
}

template <typename R>
cudaError_t launch_batched_policy(const SbnStep &q, int64_t grid, cudaStream_t stream) {
    switch (q.n_in) {
        case 1: return launch_batched_policy_n<1, R>(q, grid, stream);
        case 2: return launch_batched_policy_n<2, R>(q, grid, stream);
        case 3: return launch_batched_policy_n<3, R>(q, grid, stream);
        case 4: return launch_batched_policy_n<4, R>(q, grid, stream);
        case 5: return launch_batched_policy_n<5, R>(q, grid, stream);
        case 6: return launch_batched_policy_n<6, R>(q, grid, stream);
        case 7: return launch_batched_policy_n<7, R>(q, grid, stream);
        case 8: return launch_batched_policy_n<8, R>(q, grid, stream);
    }
    return cudaErrorInvalidValue;
}
}  // namespace

cudaError_t sbn_batched_maxsum_launch(const SbnStep &q, int64_t grid, cudaStream_t stream) {
    return launch_batched_policy<SbnMaxSum>(q, grid, stream);
}

cudaError_t sbn_batched_logsumexp_launch(const SbnStep &q, int64_t grid, cudaStream_t stream) {
    return launch_batched_policy<SbnLogSumExp>(q, grid, stream);
}

cudaError_t sbn_batched_logdomain_set_attrs() {
    cudaError_t e = cudaSuccess;
#define SBN_M(N, R)                                                                                        \
    if (e == cudaSuccess)                                                                                  \
        e = cudaFuncSetAttribute(sbn_step_batched<N, 0, R>, cudaFuncAttributeMaxDynamicSharedMemorySize, \
                                 SBN_SMEM_BUDGET);
    SBN_M(1, SbnMaxSum) SBN_M(2, SbnMaxSum) SBN_M(3, SbnMaxSum) SBN_M(4, SbnMaxSum)
    SBN_M(5, SbnMaxSum) SBN_M(6, SbnMaxSum) SBN_M(7, SbnMaxSum) SBN_M(8, SbnMaxSum)
    SBN_M(1, SbnLogSumExp) SBN_M(2, SbnLogSumExp) SBN_M(3, SbnLogSumExp) SBN_M(4, SbnLogSumExp)
    SBN_M(5, SbnLogSumExp) SBN_M(6, SbnLogSumExp) SBN_M(7, SbnLogSumExp) SBN_M(8, SbnLogSumExp)
#undef SBN_M
    return e;
}

cudaError_t sbn_batched_set_attrs() {
    cudaError_t e = set_smem_attr_n<1>();
    if (e == cudaSuccess) e = set_smem_attr_n<2>();
    if (e == cudaSuccess) e = set_smem_attr_n<3>();
    if (e == cudaSuccess) e = set_smem_attr_n<4>();
    if (e == cudaSuccess) e = set_smem_attr_n<5>();
    if (e == cudaSuccess) e = set_smem_attr_n<6>();
    if (e == cudaSuccess) e = set_smem_attr_n<7>();
    if (e == cudaSuccess) e = set_smem_attr_n<8>();
    return e;
}
