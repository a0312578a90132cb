// sorobn_b200 -- launch entry points of the step-kernel instantiations.
//
// The register-tiled kernel is instantiated per (inputs without tile axis, with axis 0, with axis 1,
// with both) x tile edge x schedule: ~290 kernels.  They are spread over four translation units
// (sbn_tiled_u0/u1/u2/c.cu) so that nvcc compiles them in parallel; this header is all sbn_api.cu sees.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <cstdlib>
#include <cstring>

struct SbnStep;

constexpr int kRowsPerThread = 2;                 // evidence rows per thread of the tiled kernel
constexpr int kSlabThreads = 64;                  // CTA size of the slab variant (x kRowsPerThread rows)
constexpr int64_t kSlabSmemMax = 96 * 1024;       // bytes of shared memory one slab may take

// CTA size of the regular tiled launches (the kernel reads blockDim.x); 128 unless overridden
// for experiments
inline int tiled_threads() {
    static const int v = [] {
        const char *e = getenv("SOROBN_B200_TILED_THREADS");
        const int t = e ? atoi(e) : 0;
        return (t == 32 || t == 64 || t == 128) ? t : 128;
    }();
    return v;
}

// Launch with the programmatic-dependent-launch attribute when enabled: the kernel may then be
// scheduled while its predecessor on the stream is still draining; it calls
// griddepcontrol.wait before touching anything a predecessor wrote (see sbn_pdl_entry).
inline bool pdl_enabled() {
    static const bool v = [] {
        const char *e = getenv("SOROBN_B200_PDL");
        return e ? atoi(e) != 0 : false;
    }();
    return v;
}

template <typename Kernel, typename... Args>
void sbn_launch(Kernel kernel, dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args... args) {
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof cfg);
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl_enabled() ? 1 : 0;
    cudaLaunchKernelEx(&cfg, kernel, args...);
}

// key = NU * 1000 + NA * 100 + NB * 10 + NC
cudaError_t sbn_tiled_u0_launch(int key, const SbnStep &q, int tile, bool preload, int64_t grid, cudaStream_t stream);
cudaError_t sbn_tiled_u1_launch(int key, const SbnStep &q, int tile, bool preload, int64_t grid, cudaStream_t stream);
cudaError_t sbn_tiled_u2_launch(int key, const SbnStep &q, int tile, bool preload, int64_t grid, cudaStream_t stream);
cudaError_t sbn_tiled_c_launch(int key, const SbnStep &q, int tile, bool preload, int64_t grid, cudaStream_t stream);
cudaError_t sbn_slab_launch(int nu, const SbnStep &q, int tile, int64_t grid, cudaStream_t stream);
cudaError_t sbn_batched_launch(const SbnStep &q, int64_t grid, cudaStream_t stream);
cudaError_t sbn_batched_maxsum_launch(const SbnStep &q, int64_t grid, cudaStream_t stream);  // MPE and MAP programs
cudaError_t sbn_batched_logsumexp_launch(const SbnStep &q, int64_t grid, cudaStream_t stream);  // MAP programs
cudaError_t sbn_tiled_u0_set_attrs();
cudaError_t sbn_tiled_u1_set_attrs();
cudaError_t sbn_tiled_u2_set_attrs();   // + the slab variants
cudaError_t sbn_tiled_c_set_attrs();
cudaError_t sbn_batched_set_attrs();
cudaError_t sbn_batched_logdomain_set_attrs();  // the max-sum and log-sum-exp instantiations
