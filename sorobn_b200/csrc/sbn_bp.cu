// sorobn_b200 -- loopy belief propagation, one evidence row per thread (sorobn_b200/bp.py defines the algorithm
// and the words; DESIGN.md "Loopy belief propagation").
//
// Rows are independent fixed-point problems, so one thread runs one row through every sweep inside one launch,
// with no grid-wide synchronisation (the shape of sbn_gibbs.cuh):
//   * the compiled words are staged in shared memory: every thread of a warp walks the same records, so control
//     flow and the word reads are uniform (broadcast);
//   * the factor tables are staged in shared memory when they fit beside the words, else read through the
//     read-only path;
//   * the per-row message state lives in a device scratch laid out [message entry][row], so the 32 rows of a warp
//     read and write 128 consecutive bytes of each entry; offsets are 64-bit;
//   * a row that converged (or met a zero) leaves its loop.
// Both directions of every message are stored (mu at entries [0, E), nu at [E, 2E)): step 1 reads nu and writes
// mu, step 2 reads mu and writes nu, so every entry is updated in place.  Storing only mu and forming nu on the
// fly would halve the state but multiply step 1's reads by the variable degrees.
// The max-product instantiations (version-2 words, the most probable explanation) run the same sweep with a max in
// step 1, then decode every variable and score the decode in the same thread.
// Expected counts (version-3 words) run the sum-product sweep over every CPT, then a second kernel,
// sbn_bp_counts_kernel, reads the stored messages back: per row the family beliefs, their sum into per-warp count
// tables (no floating-point atomics, the pattern of sbn_count.cuh) and the Bethe log-likelihood.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <vector>

#include "sbn_internal.h"

namespace {

constexpr int32_t kMagic = 0x53424250;  // "SBBP" (bp.MAGIC)
constexpr int kHeader = 12;
constexpr int kThreads = 128;
constexpr int kMaxCard = 256;  // bp.MAX_CARD
constexpr int kSmemLimit = 200 * 1024;
constexpr int64_t kScratchBudget = 1LL << 30;  // bytes of message state per chunk
constexpr double kTiny = 0x1p-32;             // the rescale of sbn_gibbs.cuh
constexpr double kRescale = 0x1p64;
constexpr int64_t kPartialBudget = 256LL << 20;  // bytes of per-warp count tables of the readout
constexpr int kCountWarps = kThreads / 32;

// The states loop of a message: unrolled over the MAXC registers of the narrow kernel (each state guarded by
// x < c), or bounded by the card c in the wide kernel, whose arrays live in local memory.
#define BP_XN (MAXC <= 8 ? MAXC : c)

struct BpArgs {
    const int32_t *words;
    int n_words;
    const float *tables;
    int n_table_floats;
    int tables_in_smem;
    const uint8_t *ev;  // [n_ev][ld]
    float *msg;         // [2E][ld]
    float *out;         // [Q][ld]
    int32_t *iters;     // [ld]
    int64_t ld, n_rows;
    int n_iterations;
    float damping, tol;
    uint8_t *codes;  // max-product: [n_var][ld]
    double *log_p;   // max-product: [ld]; expected counts: NaN for a dead row, then its log Z_B
};

// Product of the mu of a variable's edges except `skip` (-1: all of them) into p[], rescaled against underflow;
// returns the sum of p[0 .. c).  The product runs in double: the rescale keeps its largest state in range, but with
// many neighbours a smaller state can fall more than 2^126 below the largest before later factors bring it back
// (60 disagreeing children of one variable do), and in float32 it would lose its digits in the subnormals.
template <int MAXC>
__device__ __forceinline__ double bp_product(const int32_t *edges, int deg, int skip, int c, const float *mu,
                                             int64_t ld, double (&p)[MAXC]) {
#pragma unroll
    for (int x = 0; x < BP_XN; ++x) p[x] = 1.0;
    for (int k = 0; k < deg; ++k) {
        if (k == skip) continue;
        const float *m = mu + static_cast<int64_t>(edges[k]) * ld;
        double top = 0.0;
#pragma unroll
        for (int x = 0; x < BP_XN; ++x)
            if (x < c) {
                p[x] *= static_cast<double>(m[static_cast<int64_t>(x) * ld]);
                top = fmax(top, p[x]);
            }
        if (top < kTiny) {
#pragma unroll
            for (int x = 0; x < BP_XN; ++x) p[x] *= kRescale;
        }
    }
    double s = 0.0;
#pragma unroll
    for (int x = 0; x < BP_XN; ++x)
        if (x < c) s += p[x];
    return s;
}

}  // namespace

// MAX = false: sum-product, version-1 words, beliefs of the targets; MAX = true: max-product, version-2 words,
// codes and log P of the decode (bp.py "Max-product"); CNT = true: sum-product over version-3 words (bp.py "Expected
// counts"), the messages left in the scratch for sbn_bp_counts_kernel and log_p[row] = NaN for a dead row, else 0.
template <int MAXC, bool MAX, bool CNT = false>
__global__ void __launch_bounds__(kThreads) sbn_bp_kernel(const __grid_constant__ BpArgs a) {
    extern __shared__ __align__(16) uint8_t s_raw[];
    int32_t *w = reinterpret_cast<int32_t *>(s_raw);
    float *s_tab = reinterpret_cast<float *>(s_raw + ((a.n_words * 4 + 15) & ~15));
    for (int i = threadIdx.x; i < a.n_words; i += blockDim.x) w[i] = a.words[i];
    if (a.tables_in_smem)
        for (int i = threadIdx.x; i < a.n_table_floats; i += blockDim.x) s_tab[i] = a.tables[i];
    __syncthreads();
    const int64_t row = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (row >= a.n_rows) return;
    const bool tsm = a.tables_in_smem != 0;
    const float *__restrict__ gtab = a.tables;
    auto table = [&](int e) -> float { return tsm ? s_tab[e] : __ldg(gtab + e); };

    const int n_fac = w[3], n_var = w[4], E = w[5], n_tgt = w[6], Q = w[7];
    const int fac_pos = w[9], var_pos = w[10], tgt_pos = w[11];
    const int64_t ld = a.ld;
    float *mu = a.msg + row;
    float *nu = a.msg + static_cast<int64_t>(E) * ld + row;
    const uint8_t *ev = a.ev + row;
    const float lam = a.damping, keep = 1.f - a.damping;

    // uniform start: every edge's mu and nu
    for (int f = 0, p = fac_pos; f < n_fac; ++f) {
        const int n_mem = w[p + 2], n_evax = w[p + 3];
        for (int i = 0; i < n_mem; ++i) {
            const int c = w[p + 4 + 3 * i], e = w[p + 6 + 3 * i];
            const float u = 1.f / static_cast<float>(c);
            for (int x = 0; x < c; ++x) {
                mu[static_cast<int64_t>(e + x) * ld] = u;
                nu[static_cast<int64_t>(e + x) * ld] = u;
            }
        }
        p += 4 + 3 * n_mem + 3 * n_evax;
    }

    bool dead = false;
    if constexpr (MAX || CNT) {
        // a family whose members are all observed, at an entry of probability 0: the row's evidence is impossible,
        // and no message would ever see it (the sweep skips such factors)
        for (int f = 0, p = fac_pos; f < n_fac; ++f) {
            const int n_mem = w[p + 2], n_evax = w[p + 3];
            if (n_mem == 0) {
                int idx = w[p + 1];
                for (int k = 0; k < n_evax; ++k) {
                    const int32_t *ax = w + p + 4 + 3 * k;
                    idx += min(static_cast<int>(ev[static_cast<int64_t>(ax[0]) * ld]), ax[2] - 1) * ax[1];
                }
                if (!(table(idx) > 0.f)) dead = true;
            }
            p += 4 + 3 * n_mem + 3 * n_evax;
        }
    }
    // max-product: a pattern that observes every node has nothing to decode, and a row dead before its first sweep
    // runs none; both record 0
    const int sweeps = (MAX || CNT) && (n_var == 0 || dead) ? 0 : a.n_iterations;
    int recorded = (MAX || CNT) && (n_var == 0 || dead) ? 0 : a.n_iterations + 1;
    for (int t = 1; t <= sweeps; ++t) {
        // ---- step 1: every factor-to-variable message, damped, and the residual
        float r = 0.f;
        for (int f = 0, p = fac_pos; f < n_fac; ++f) {
            const int n_mem = w[p + 2], n_evax = w[p + 3];
            if ((MAX || CNT) && n_mem == 0) {  // an all-observed family: only the score (or the readout) reads it
                p += 4 + 3 * n_evax;
                continue;
            }
            const int32_t *mem = w + p + 4;
            const int32_t *ax = mem + 3 * n_mem;
            int base = w[p + 1];
            for (int k = 0; k < n_evax; ++k) {
                const int code = min(static_cast<int>(ev[static_cast<int64_t>(ax[3 * k]) * ld]), ax[3 * k + 2] - 1);
                base += code * ax[3 * k + 1];
            }
            int T = 1;
            for (int i = 0; i < n_mem; ++i) T *= mem[3 * i];
            for (int i = 0; i < n_mem; ++i) {
                const int c = mem[3 * i], si = mem[3 * i + 1], e = mem[3 * i + 2];
                const int n_other = T / c;
                float s[MAXC];
#pragma unroll
                for (int x = 0; x < BP_XN; ++x) s[x] = 0.f;
                for (int j = 0; j < n_other; ++j) {
                    // decode j over the other members (first fastest): their states, table offset and nu product
                    int rem = j, idx = base;
                    float prod = 1.f;
                    for (int u = 0; u < n_mem; ++u) {
                        if (u == i) continue;
                        const int cu = mem[3 * u];
                        const int xu = rem % cu;
                        rem /= cu;
                        idx += xu * mem[3 * u + 1];
                        prod *= nu[static_cast<int64_t>(mem[3 * u + 2] + xu) * ld];
                    }
#pragma unroll
                    for (int x = 0; x < BP_XN; ++x)
                        if (x < c) {
                            if constexpr (MAX)
                                s[x] = fmaxf(s[x], table(idx + x * si) * prod);
                            else
                                s[x] += table(idx + x * si) * prod;
                        }
                }
                float S = 0.f;
#pragma unroll
                for (int x = 0; x < BP_XN; ++x)
                    if (x < c) S += s[x];
                // divide (not multiply by 1 / S): the sum of the other members' nu products is not rescaled and
                // may be subnormal, where 1 / S overflows while every ratio s[x] / S is finite
                if (!(S > 0.f)) dead = true;
                float *m = mu + static_cast<int64_t>(e) * ld;
#pragma unroll
                for (int x = 0; x < BP_XN; ++x)
                    if (x < c) {
                        const float old = m[static_cast<int64_t>(x) * ld];
                        const float v = keep * (s[x] / S) + lam * old;
                        r = fmaxf(r, fabsf(v - old));
                        m[static_cast<int64_t>(x) * ld] = v;
                    }
            }
            p += 4 + 3 * n_mem + 3 * n_evax;
        }
        if (dead) {
            recorded = t;
            break;
        }
        // ---- step 2: every variable-to-factor message from the new mu
        for (int v = 0, p = var_pos; v < n_var && !dead; ++v) {
            const int c = w[p + 1], deg = w[p + 2];
            const int32_t *edges = w + p + 3;
            for (int k = 0; k < deg; ++k) {
                double q[MAXC];
                const double S = bp_product<MAXC>(edges, deg, k, c, mu, ld, q);
                if (!(S > 0.0)) dead = true;
                float *n = nu + static_cast<int64_t>(edges[k]) * ld;
#pragma unroll
                for (int x = 0; x < BP_XN; ++x)
                    if (x < c) n[static_cast<int64_t>(x) * ld] = static_cast<float>(q[x] / S);
            }
            p += 3 + deg;
        }
        if (dead) {
            recorded = t;
            break;
        }
        if (r < a.tol) {
            recorded = t;
            break;
        }
    }
    a.iters[row] = recorded;
    if constexpr (MAX) {
        // ---- decode: every variable's first state of largest belief product, from the last sweep's mu.  The code
        // is left in the first nu entry of each of the variable's edges (no sweep reads nu any more), where the
        // score finds it through the factor's member records.
        for (int k = 0; k < n_tgt && !dead; ++k) {
            const int p = w[tgt_pos + 2 * k];
            const int c = w[p + 1], deg = w[p + 2];
            double q[MAXC];
            const double S = bp_product<MAXC>(w + p + 3, deg, -1, c, mu, ld, q);
            if (!(S > 0.0)) {
                dead = true;
                break;
            }
            int best = 0;
            double top = q[0];
#pragma unroll
            for (int x = 1; x < BP_XN; ++x)
                if (x < c && q[x] > top) {
                    top = q[x];
                    best = x;
                }
            a.codes[static_cast<int64_t>(w[tgt_pos + 2 * k + 1]) * ld + row] = static_cast<uint8_t>(best);
            for (int j = 0; j < deg; ++j) nu[static_cast<int64_t>(w[p + 3 + j]) * ld] = static_cast<float>(best);
        }
        // ---- score: log P(decode, e) over every factor, 0-member ones included
        double lp = 0.0;
        for (int f = 0, p = fac_pos; f < n_fac && !dead; ++f) {
            const int n_mem = w[p + 2], n_evax = w[p + 3];
            const int32_t *mem = w + p + 4;
            const int32_t *ax = mem + 3 * n_mem;
            int idx = w[p + 1];
            for (int i = 0; i < n_mem; ++i)
                idx += static_cast<int>(nu[static_cast<int64_t>(mem[3 * i + 2]) * ld]) * mem[3 * i + 1];
            for (int k = 0; k < n_evax; ++k) {
                const int code = min(static_cast<int>(ev[static_cast<int64_t>(ax[3 * k]) * ld]), ax[3 * k + 2] - 1);
                idx += code * ax[3 * k + 1];
            }
            lp += log(static_cast<double>(table(idx)));
            p += 4 + 3 * n_mem + 3 * n_evax;
        }
        if (dead) {
            lp = __longlong_as_double(0x7ff8000000000000LL);
            for (int k = 0; k < n_tgt; ++k) a.codes[static_cast<int64_t>(w[tgt_pos + 2 * k + 1]) * ld + row] = 0;
        }
        a.log_p[row] = lp;
    } else if constexpr (CNT) {
        a.log_p[row] = dead ? __longlong_as_double(0x7ff8000000000000LL) : 0.0;
    } else {
        // ---- beliefs of the targets from the last sweep's mu
        for (int k = 0; k < n_tgt && !dead; ++k) {
            const int p = w[tgt_pos + 2 * k];
            const int c = w[p + 1], deg = w[p + 2];
            double q[MAXC];
            const double S = bp_product<MAXC>(w + p + 3, deg, -1, c, mu, ld, q);
            if (!(S > 0.0)) {
                dead = true;
                break;
            }
            float *o = a.out + static_cast<int64_t>(w[tgt_pos + 2 * k + 1]) * ld + row;
#pragma unroll
            for (int x = 0; x < BP_XN; ++x)
                if (x < c) o[static_cast<int64_t>(x) * ld] = static_cast<float>(q[x] / S);
        }
        if (dead)
            for (int q = 0; q < Q; ++q) a.out[static_cast<int64_t>(q) * ld + row] = __int_as_float(0x7fc00000);
    }
}

namespace {

// Sum of `v` over the lanes of `grp` (the lanes that share this lane's key) in lane order, or by a fixed butterfly
// when all 32 share it (sbn_count.cuh's sbn_group_sum); the result is meaningful in the group's lowest lane.
__device__ __forceinline__ double bp_group_sum(double v, unsigned grp) {
    if (grp == 0xffffffffu) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        return v;
    }
    double s = 0.0;
#pragma unroll
    for (int j = 0; j < 32; ++j) {
        const double x = __shfl_sync(0xffffffffu, v, j);
        if ((grp >> j) & 1u) s += x;
    }
    return s;
}

// f(x_f, e) prod_i nu_{i->f}(x_i) in double, for the configuration j of a factor's members (first member fastest;
// members are innermost in the table, so the entry is base + j)
__device__ __forceinline__ double bp_family_term(const int32_t *mem, int n_mem, int j, double f, const float *nu,
                                                 int64_t ld) {
    double p = f;
    for (int i = 0; i < n_mem; ++i) {
        const int c = mem[3 * i];
        p *= static_cast<double>(nu[static_cast<int64_t>(mem[3 * i + 2] + j % c) * ld]);
        j /= c;
    }
    return p;
}

}  // namespace

// The expected-counts readout of version-3 words (bp.py "Expected counts"), after the CNT sweep: a fixed grid of
// persistent CTAs walks the blocks of kThreads rows in a fixed order (block blockIdx.x, then + gridDim.x, ...), one
// row per thread.  A live row (log_p not NaN) first forms, in double, every variable belief's entropy term and every
// family belief's normaliser and energy term: log Z_B, or dead when a sum is 0.  Then every factor, uniformly over the
// warp: the lanes whose rows share the factor's evidence key (its table entry at the row's codes) are found by
// __match_any_sync, each entry's belief is summed over the group in lane order, and the group's lowest lane adds the
// sum to the warp's own count table `partial` [gridDim.x * kCountWarps][n_table_floats], indexed like the blob.
template <int MAXC>
__global__ void __launch_bounds__(kThreads) sbn_bp_counts_kernel(const __grid_constant__ BpArgs a,
                                                                 double *__restrict__ partial) {
    extern __shared__ __align__(16) uint8_t s_raw[];
    int32_t *w = reinterpret_cast<int32_t *>(s_raw);
    float *s_tab = reinterpret_cast<float *>(s_raw + ((a.n_words * 4 + 15) & ~15));
    for (int i = threadIdx.x; i < a.n_words; i += blockDim.x) w[i] = a.words[i];
    if (a.tables_in_smem)
        for (int i = threadIdx.x; i < a.n_table_floats; i += blockDim.x) s_tab[i] = a.tables[i];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    double *const part = partial + (static_cast<int64_t>(blockIdx.x) * kCountWarps + warp) * a.n_table_floats;
    for (int e = lane; e < a.n_table_floats; e += 32) part[e] = 0.0;
    __syncthreads();
    const bool tsm = a.tables_in_smem != 0;
    const float *__restrict__ gtab = a.tables;
    auto table = [&](int e) -> float { return tsm ? s_tab[e] : __ldg(gtab + e); };

    const int n_fac = w[3], n_var = w[4], E = w[5];
    const int fac_pos = w[9], var_pos = w[10];
    const int64_t ld = a.ld;
    const int64_t n_blocks = (a.n_rows + kThreads - 1) / kThreads;
    for (int64_t blk = blockIdx.x; blk < n_blocks; blk += gridDim.x) {
        const int64_t row = blk * kThreads + threadIdx.x;
        const bool in = row < a.n_rows;
        const int64_t r = in ? row : 0;
        const float *mu = a.msg + r;
        const float *nu = a.msg + static_cast<int64_t>(E) * ld + r;
        const uint8_t *ev = a.ev + r;
        bool live = in && !isnan(a.log_p[r]);
        auto key_of = [&](int p, int n_mem, int n_evax) {
            int base = w[p + 1];
            const int32_t *ax = w + p + 4 + 3 * n_mem;
            for (int k = 0; k < n_evax; ++k)
                base += min(static_cast<int>(ev[static_cast<int64_t>(ax[3 * k]) * ld]), ax[3 * k + 2] - 1) * ax[3 * k + 1];
            return base;
        };

        // ---- log Z_B: sum_v (d_v - 1) sum_x b_v log b_v ...
        double lz = 0.0;
        for (int v = 0, p = var_pos; v < n_var && live; ++v) {
            const int c = w[p + 1], deg = w[p + 2];
            double q[MAXC];
            const double S = bp_product<MAXC>(w + p + 3, deg, -1, c, mu, ld, q);
            if (!(S > 0.0)) {
                live = false;
                break;
            }
            double h = 0.0;
#pragma unroll
            for (int x = 0; x < BP_XN; ++x)
                if (x < c) {
                    const double b = q[x] / S;
                    if (b > 0.0) h += b * log(b);
                }
            lz += static_cast<double>(deg - 1) * h;
            p += 3 + deg;
        }
        // ... + sum_f sum_x b_f (log f - log b_f) = H_f / S_f + log S_f with p = f prod nu, S_f = sum p,
        // H_f = sum p (log f - log p); a 0-member factor adds log f(e)
        for (int f = 0, p = fac_pos; f < n_fac && live; ++f) {
            const int n_mem = w[p + 2], n_evax = w[p + 3];
            const int base = key_of(p, n_mem, n_evax);
            if (n_mem == 0) {
                lz += log(static_cast<double>(table(base)));
            } else {
                int T = 1;
                for (int i = 0; i < n_mem; ++i) T *= w[p + 4 + 3 * i];
                double S = 0.0, H = 0.0;
                for (int j = 0; j < T; ++j) {
                    const double fx = static_cast<double>(table(base + j));
                    const double t = bp_family_term(w + p + 4, n_mem, j, fx, nu, ld);
                    S += t;
                    if (t > 0.0) H += t * (log(fx) - log(t));
                }
                if (!(S > 0.0)) live = false;
                else lz += H / S + log(S);
            }
            p += 4 + 3 * n_mem + 3 * n_evax;
        }
        if (in) a.log_p[row] = live ? lz : __longlong_as_double(0x7ff8000000000000LL);

        // ---- counts: every factor's belief at the row's evidence key, summed per group of lanes
        for (int f = 0, p = fac_pos; f < n_fac; ++f) {
            const int n_mem = w[p + 2], n_evax = w[p + 3];
            const int key = live ? key_of(p, n_mem, n_evax) : -1;
            const unsigned grp = __match_any_sync(0xffffffffu, key);
            const bool lead = key >= 0 && lane == __ffs(grp) - 1;
            if (n_mem == 0) {
                const double v = bp_group_sum(live ? 1.0 : 0.0, grp);
                if (lead) part[key] += v;
            } else {
                int T = 1;
                for (int i = 0; i < n_mem; ++i) T *= w[p + 4 + 3 * i];
                double S = 0.0;
                if (live)
                    for (int j = 0; j < T; ++j)
                        S += bp_family_term(w + p + 4, n_mem, j, static_cast<double>(table(key + j)), nu, ld);
                for (int j = 0; j < T; ++j) {
                    const double b =
                        live ? bp_family_term(w + p + 4, n_mem, j, static_cast<double>(table(key + j)), nu, ld) / S : 0.0;
                    const double v = bp_group_sum(b, grp);
                    if (lead) part[key + j] += v;
                }
            }
            __syncwarp();
            p += 4 + 3 * n_mem + 3 * n_evax;
        }
    }
}

// counts[e] += the sum of partial[g][e] over the count tables g: each of the 8 warps of a CTA sums the tables
// g = warp, warp + 8, ... in order for 32 entries, then lane-wise the 8 sums in warp order: a fixed order.
__global__ void __launch_bounds__(256) sbn_bp_counts_reduce(const double *__restrict__ partial, int64_t n_parts,
                                                            int32_t n_entries, double *__restrict__ counts) {
    __shared__ double s[8][32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t e = static_cast<int64_t>(blockIdx.x) * 32 + lane;
    double v = 0.0;
    if (e < n_entries)
        for (int64_t g = warp; g < n_parts; g += 8) v += partial[g * n_entries + e];
    s[warp][lane] = v;
    __syncthreads();
    if (warp == 0 && e < n_entries) {
        double t = 0.0;
#pragma unroll
        for (int k = 0; k < 8; ++k) t += s[k][lane];
        counts[e] += t;
    }
}

struct sbn_bp {
    int device = 0;
    std::vector<int32_t> words;
    int n_table_floats = 0;
    int version = 1;
    int n_ev = 0, E = 0, Q = 0, max_card = 1;
    int smem = 0;
    bool tables_in_smem = false;
    int32_t *d_words = nullptr;
    float *d_tables = nullptr;
    int64_t cap = 0;  // rows per chunk
    uint8_t *d_ev = nullptr;
    float *d_msg = nullptr, *d_out = nullptr;
    int32_t *d_iters = nullptr;
    uint8_t *d_codes = nullptr;  // version 2
    double *d_log_p = nullptr;   // versions 2 and 3
    int n_sm = 1;
    int count_grid = 0;            // version 3: CTAs of the readout (the count tables it has room for)
    double *d_partial = nullptr;   // [count_grid * kCountWarps][n_table_floats]
    double *d_counts = nullptr;    // [n_table_floats]: the running total over a call's chunks
    cudaStream_t stream = nullptr;
};

namespace {

#define SBN_BP_CUDA(call)                                                                                        \
    do {                                                                                                       \
        cudaError_t e_ = (call);                                                                               \
        if (e_ != cudaSuccess)                                                                                 \
            return sbn_fail(e_ == cudaErrorMemoryAllocation ? SBN_E_NOMEM : SBN_E_CUDA, "%s failed: %s (%s:%d)", \
                            #call, cudaGetErrorString(e_), __FILE__, __LINE__);                                \
    } while (0)

// Bounds-check every word (bp.py layout); fills the version, n_ev, E, Q and the widest message.  Versions 2
// (max-product) and 3 (expected counts) allow factors of 0 members and 0 variables and edges, and their targets must
// be every variable record in order at q_offset k, each member edge of a factor exactly one variable's: the score
// finds the decoded codes through them.
int validate(const int32_t *w, int64_t n, int64_t n_tables, sbn_bp &b) {
    if (n < kHeader) return sbn_fail(SBN_E_INVALID, "bp words: %lld words, the header has %d", static_cast<long long>(n), kHeader);
    if (n >= (1LL << 30)) return sbn_fail(SBN_E_INVALID, "bp words: %lld words", static_cast<long long>(n));
    if (w[0] != kMagic || w[1] < 1 || w[1] > 3) return sbn_fail(SBN_E_INVALID, "bp words: bad magic or version %d", w[1]);
    const bool mpe = w[1] != 1;  // the version-2 rules
    const int lo = mpe ? 0 : 1;  // the least n_var, E, targets, Q and members of a factor
    const int n_ev = w[2], n_fac = w[3], n_var = w[4], E = w[5], n_tgt = w[6], Q = w[7];
    if (n_ev < 0 || n_fac < 1 || n_var < lo || E < lo || n_tgt < lo || Q < lo || w[8] != n_tables ||
        (mpe && (n_tgt != n_var || Q != n_var)))
        return sbn_fail(SBN_E_INVALID, "bp words: bad header (n_ev %d, factors %d, variables %d, E %d, targets %d, Q %d, "
                        "table floats %d of %lld)", n_ev, n_fac, n_var, E, n_tgt, Q, w[8], static_cast<long long>(n_tables));
    if (w[9] != kHeader || w[10] < w[9] || w[11] < w[10] || static_cast<int64_t>(w[11]) + 2LL * n_tgt != n)
        return sbn_fail(SBN_E_INVALID, "bp words: bad section positions %d %d %d", w[9], w[10], w[11]);
    int64_t p = w[9];
    int64_t edge_end = 0;
    int max_card = 1;
    for (int f = 0; f < n_fac; ++f) {
        if (p + 4 > w[10]) return sbn_fail(SBN_E_INVALID, "bp words: factor %d runs past its section", f);
        const int64_t off = w[p + 1];
        const int n_mem = w[p + 2], n_evax = w[p + 3];
        if (n_mem < lo || n_evax < 0 || p + 4 + 3LL * (n_mem + n_evax) > w[10])
            return sbn_fail(SBN_E_INVALID, "bp words: factor %d has %d members and %d evidence axes", f, n_mem, n_evax);
        int64_t span = 1;  // entries the factor's table spans
        for (int i = 0; i < n_mem; ++i) {
            const int c = w[p + 4 + 3 * i], s = w[p + 5 + 3 * i], e = w[p + 6 + 3 * i];
            if (c < 1 || c > kMaxCard || s != span || e < 0 || static_cast<int64_t>(e) + c > E)
                return sbn_fail(SBN_E_INVALID, "bp words: factor %d member %d (card %d, stride %d, edge %d)", f, i, c, s, e);
            span *= c;
            edge_end = std::max<int64_t>(edge_end, static_cast<int64_t>(e) + c);
            max_card = std::max(max_card, c);
            if (span >= (1LL << 31)) return sbn_fail(SBN_E_INVALID, "bp words: factor %d is too large", f);
        }
        for (int k = 0; k < n_evax; ++k) {
            const int32_t *ax = w + p + 4 + 3 * n_mem + 3 * k;
            if (ax[0] < 0 || ax[0] >= n_ev || ax[1] != span || ax[2] < 1 || ax[2] > 256)
                return sbn_fail(SBN_E_INVALID, "bp words: factor %d evidence axis %d (col %d, stride %d, card %d)", f, k,
                                ax[0], ax[1], ax[2]);
            span *= ax[2];
            if (span >= (1LL << 31)) return sbn_fail(SBN_E_INVALID, "bp words: factor %d is too large", f);
        }
        if (off < 0 || off + span > n_tables)
            return sbn_fail(SBN_E_INVALID, "bp words: factor %d table [%lld, +%lld) outside %lld floats", f,
                            static_cast<long long>(off), static_cast<long long>(span), static_cast<long long>(n_tables));
        p += 4 + 3 * (n_mem + n_evax);
    }
    if (p != w[10] || edge_end != E) return sbn_fail(SBN_E_INVALID, "bp words: factor section does not end at its edges");
    // version 2: the card of the factor member whose edge starts at e (E is now bounded by the checked records)
    std::vector<int> member_card(mpe ? E : 0, 0);
    for (int64_t q = w[9]; mpe && q < w[10]; q += 4 + 3 * (w[q + 2] + w[q + 3]))
        for (int i = 0; i < w[q + 2]; ++i) member_card[w[q + 6 + 3 * i]] = w[q + 4 + 3 * i];
    std::vector<int> var_at(n, -1), var_pos;
    for (int v = 0; v < n_var; ++v) {
        if (p + 3 > w[11]) return sbn_fail(SBN_E_INVALID, "bp words: variable %d runs past its section", v);
        const int c = w[p + 1], deg = w[p + 2];
        if (c < 1 || c > kMaxCard || deg < 1 || p + 3 + deg > w[11])
            return sbn_fail(SBN_E_INVALID, "bp words: variable %d (card %d, degree %d)", v, c, deg);
        for (int k = 0; k < deg; ++k) {
            const int e = w[p + 3 + k];
            if (e < 0 || static_cast<int64_t>(e) + c > E || (mpe && member_card[e] != c))
                return sbn_fail(SBN_E_INVALID, "bp words: variable %d edge %d at %d", v, k, e);
            if (mpe) member_card[e] = 0;  // claimed
        }
        var_at[p] = c;
        var_pos.push_back(static_cast<int>(p));
        p += 3 + deg;
    }
    if (p != w[11]) return sbn_fail(SBN_E_INVALID, "bp words: variable section does not end at the targets");
    if (mpe && std::any_of(member_card.begin(), member_card.end(), [](int c) { return c != 0; }))
        return sbn_fail(SBN_E_INVALID, "bp words: a factor member's edge belongs to no variable");
    for (int k = 0; k < n_tgt; ++k) {
        const int vp = w[p + 2 * k], q = w[p + 2 * k + 1];
        if (vp < 0 || vp >= n || var_at[vp] < 0 || q < 0 || q + (mpe ? 1 : var_at[vp]) > Q ||
            (mpe && (vp != var_pos[k] || q != k)))
            return sbn_fail(SBN_E_INVALID, "bp words: target %d (record %d, q_offset %d)", k, vp, q);
    }
    b.version = w[1];
    b.n_ev = n_ev;
    b.E = E;
    b.Q = Q;
    b.max_card = max_card;
    return SBN_OK;
}

template <bool MAX, bool CNT>
void launch(const BpArgs &a, int max_card, unsigned grid, int smem, cudaStream_t stream) {
    if (max_card <= 8)
        sbn_bp_kernel<8, MAX, CNT><<<grid, kThreads, smem, stream>>>(a);
    else
        sbn_bp_kernel<kMaxCard, MAX, CNT><<<grid, kThreads, smem, stream>>>(a);
}

int reserve(sbn_bp *b, int64_t rows);

// The error of a run call given words of another version: the call that runs them
int wrong_call(int version) {
    if (version == 1) return sbn_fail(SBN_E_INVALID, "sum-product (version 1) words run through sbn_bp_run_host");
    if (version == 2) return sbn_fail(SBN_E_INVALID, "max-product (version 2) words run through sbn_bp_mpe_host");
    return sbn_fail(SBN_E_INVALID, "expected-counts (version 3) words run through sbn_bp_counts_host");
}

// The argument checks, the reservation and the chunk loop of the run calls: upload a chunk's codes, run it,
// download its iterations, and queue the download of its outputs by `fetch(r0, n)`; one synchronise at the end.
template <bool MAX, bool CNT, typename Fetch>
int run_rows(sbn_bp *b, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, int32_t n_iterations, float damping, float tol,
             int64_t ld_out, int32_t *iterations, Fetch fetch) {
    if (n_rows < 0 || ld_ev < n_rows || ld_out < n_rows)
        return sbn_fail(SBN_E_INVALID, "bad shape: %lld rows, pitches %lld / %lld", static_cast<long long>(n_rows),
                        static_cast<long long>(ld_ev), static_cast<long long>(ld_out));
    if (n_iterations < 1 || n_iterations == 0x7fffffff)
        return sbn_fail(SBN_E_INVALID, "n_iterations must be in [1, 2^31 - 2], not %d", n_iterations);
    if (!(damping >= 0.f && damping < 1.f)) return sbn_fail(SBN_E_INVALID, "damping must be in [0, 1), not %g", damping);
    if (!(tol >= 0.f) || std::isinf(tol)) return sbn_fail(SBN_E_INVALID, "tol must be finite and >= 0, not %g", tol);
    if (n_rows == 0) return SBN_OK;
    SBN_BP_CUDA(cudaSetDevice(b->device));
    int64_t want = n_rows;
    if (const char *s = std::getenv("SOROBN_B200_CHUNK_ROWS")) {
        const long long cap = std::atoll(s);
        if (cap > 0) want = std::min<int64_t>(want, cap);
    }
    int rc = reserve(b, want);
    if (rc != SBN_OK) return rc;
    const int64_t chunk = std::min(b->cap, want);
    for (int64_t r0 = 0; r0 < n_rows; r0 += chunk) {
        const int64_t n = std::min(chunk, n_rows - r0);
        if (b->n_ev > 0)
            SBN_BP_CUDA(cudaMemcpy2DAsync(b->d_ev, b->cap, ev + r0, ld_ev, n, b->n_ev, cudaMemcpyHostToDevice, b->stream));
        BpArgs a{b->d_words, static_cast<int>(b->words.size()), b->d_tables, b->n_table_floats, b->tables_in_smem ? 1 : 0,
                 b->d_ev, b->d_msg, b->d_out, b->d_iters, b->cap, n, n_iterations, damping, tol, b->d_codes, b->d_log_p};
        launch<MAX, CNT>(a, b->max_card, static_cast<unsigned>((n + kThreads - 1) / kThreads), b->smem, b->stream);
        SBN_BP_CUDA(cudaGetLastError());
        rc = fetch(r0, n);
        if (rc != SBN_OK) return rc;
        SBN_BP_CUDA(cudaMemcpyAsync(iterations + r0, b->d_iters, n * 4, cudaMemcpyDeviceToHost, b->stream));
    }
    SBN_BP_CUDA(cudaStreamSynchronize(b->stream));
    return SBN_OK;
}

int reserve(sbn_bp *b, int64_t rows) {
    if (rows <= b->cap) return SBN_OK;
    const int64_t per_row = std::max<int64_t>(1, 2LL * b->E * 4);  // E = 0: a max-product pattern with nothing to decode
    int64_t cap = std::max<int64_t>(kThreads, kScratchBudget / per_row / kThreads * kThreads);
    cap = std::min(cap, round_up(rows, kThreads));
    if (cap <= b->cap) return SBN_OK;
    cudaFree(b->d_ev);
    cudaFree(b->d_msg);
    cudaFree(b->d_out);
    cudaFree(b->d_iters);
    cudaFree(b->d_codes);
    cudaFree(b->d_log_p);
    cudaFree(b->d_partial);
    b->d_ev = nullptr;
    b->d_msg = b->d_out = nullptr;
    b->d_iters = nullptr;
    b->d_codes = nullptr;
    b->d_log_p = nullptr;
    b->d_partial = nullptr;
    b->cap = 0;
    b->count_grid = 0;
    SBN_BP_CUDA(cudaMalloc(&b->d_ev, std::max<int64_t>(1, b->n_ev) * cap));
    SBN_BP_CUDA(cudaMalloc(&b->d_msg, std::max<int64_t>(1, 2LL * b->E) * cap * 4));
    SBN_BP_CUDA(cudaMalloc(&b->d_iters, cap * 4));
    if (b->version == 2) {
        SBN_BP_CUDA(cudaMalloc(&b->d_codes, std::max<int64_t>(1, b->Q) * cap));
        SBN_BP_CUDA(cudaMalloc(&b->d_log_p, cap * 8));
    } else if (b->version == 3) {
        // the readout's grid: 8 CTAs per SM at most, fewer when their count tables would pass kPartialBudget
        const int64_t table_bytes = std::max<int64_t>(1, static_cast<int64_t>(b->n_table_floats) * 8 * kCountWarps);
        const int64_t grid = std::max<int64_t>(1, std::min<int64_t>({cap / kThreads, 8LL * b->n_sm,
                                                                      kPartialBudget / table_bytes}));
        SBN_BP_CUDA(cudaMalloc(&b->d_log_p, cap * 8));
        SBN_BP_CUDA(cudaMalloc(&b->d_partial, grid * table_bytes));
        b->count_grid = static_cast<int>(grid);
    } else {
        SBN_BP_CUDA(cudaMalloc(&b->d_out, static_cast<int64_t>(b->Q) * cap * 4));
    }
    b->cap = cap;
    return SBN_OK;
}

}  // namespace

extern "C" {

int sbn_bp_create(int device, const int32_t *words, int64_t n_words, const float *tables, int64_t n_table_floats,
                  sbn_bp **out) {
    if (!words || !out || (n_table_floats > 0 && !tables)) return sbn_fail(SBN_E_INVALID, "null argument");
    *out = nullptr;
    sbn_bp probe;
    int rc = validate(words, n_words, n_table_floats, probe);
    if (rc != SBN_OK) return rc;
    const int64_t words_bytes = (n_words * 4 + 15) & ~15LL;
    if (words_bytes > kSmemLimit)
        return sbn_fail(SBN_E_INVALID, "bp words: %lld words do not fit the kernel's shared memory",
                        static_cast<long long>(n_words));
    int n_dev = 0;
    if (cudaGetDeviceCount(&n_dev) != cudaSuccess || n_dev == 0) return sbn_fail(SBN_E_NODEVICE, "no CUDA device available");
    if (device < 0 || device >= n_dev) return sbn_fail(SBN_E_NODEVICE, "device %d out of range (%d visible)", device, n_dev);
    sbn_bp *b = new sbn_bp();
    b->device = device;
    b->words.assign(words, words + n_words);
    b->n_table_floats = static_cast<int>(n_table_floats);
    b->version = probe.version;
    b->n_ev = probe.n_ev;
    b->E = probe.E;
    b->Q = probe.Q;
    b->max_card = probe.max_card;
    b->tables_in_smem = words_bytes + n_table_floats * 4 <= kSmemLimit;
    b->smem = static_cast<int>(words_bytes + (b->tables_in_smem ? n_table_floats * 4 : 0));
    auto bail = [&](int code) {
        sbn_bp_destroy(b);
        return code;
    };
#define SBN_BP_CUDA_B(call)                                                                                             \
    do {                                                                                                              \
        cudaError_t e_ = (call);                                                                                      \
        if (e_ != cudaSuccess)                                                                                        \
            return bail(sbn_fail(e_ == cudaErrorMemoryAllocation ? SBN_E_NOMEM : SBN_E_CUDA, "%s failed: %s (%s:%d)", \
                                 #call, cudaGetErrorString(e_), __FILE__, __LINE__));                                 \
    } while (0)
    SBN_BP_CUDA_B(cudaSetDevice(device));
    cudaDeviceProp prop;
    SBN_BP_CUDA_B(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0)
        return bail(sbn_fail(SBN_E_NODEVICE, "device %d is sm_%d%d; this library is built for sm_90a only", device,
                             prop.major, prop.minor));
    SBN_BP_CUDA_B(cudaFuncSetAttribute(sbn_bp_kernel<8, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit));
    SBN_BP_CUDA_B(cudaFuncSetAttribute(sbn_bp_kernel<kMaxCard, false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       kSmemLimit));
    SBN_BP_CUDA_B(cudaFuncSetAttribute(sbn_bp_kernel<8, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit));
    SBN_BP_CUDA_B(cudaFuncSetAttribute(sbn_bp_kernel<kMaxCard, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       kSmemLimit));
    SBN_BP_CUDA_B(cudaFuncSetAttribute(sbn_bp_kernel<8, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       kSmemLimit));
    SBN_BP_CUDA_B(cudaFuncSetAttribute(sbn_bp_kernel<kMaxCard, false, true>,
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit));
    SBN_BP_CUDA_B(cudaFuncSetAttribute(sbn_bp_counts_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit));
    SBN_BP_CUDA_B(cudaFuncSetAttribute(sbn_bp_counts_kernel<kMaxCard>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       kSmemLimit));
    SBN_BP_CUDA_B(cudaDeviceGetAttribute(&b->n_sm, cudaDevAttrMultiProcessorCount, device));
    SBN_BP_CUDA_B(cudaStreamCreateWithFlags(&b->stream, cudaStreamNonBlocking));
    SBN_BP_CUDA_B(cudaMalloc(&b->d_words, n_words * 4));
    SBN_BP_CUDA_B(cudaMemcpy(b->d_words, words, n_words * 4, cudaMemcpyHostToDevice));
    if (n_table_floats > 0) {
        SBN_BP_CUDA_B(cudaMalloc(&b->d_tables, n_table_floats * 4));
        SBN_BP_CUDA_B(cudaMemcpy(b->d_tables, tables, n_table_floats * 4, cudaMemcpyHostToDevice));
    }
    if (b->version == 3) SBN_BP_CUDA_B(cudaMalloc(&b->d_counts, std::max<int64_t>(1, n_table_floats) * 8));
#undef SBN_BP_CUDA_B
    *out = b;
    return SBN_OK;
}

int sbn_bp_run_host(sbn_bp *b, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, int32_t n_iterations, float damping,
                    float tol, float *out, int64_t ld_out, int32_t *iterations) {
    if (!b || !out || !iterations || (b->n_ev > 0 && !ev)) return sbn_fail(SBN_E_INVALID, "null argument");
    if (b->version != 1) return wrong_call(b->version);
    return run_rows<false, false>(b, ev, ld_ev, n_rows, n_iterations, damping, tol, ld_out, iterations, [&](int64_t r0, int64_t n) {
        SBN_BP_CUDA(cudaMemcpy2DAsync(out + r0, ld_out * 4, b->d_out, b->cap * 4, n * 4, b->Q, cudaMemcpyDeviceToHost,
                                      b->stream));
        return SBN_OK;
    });
}

int sbn_bp_mpe_host(sbn_bp *b, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, int32_t n_iterations, float damping,
                    float tol, uint8_t *codes, int64_t ld_codes, double *log_p, int32_t *iterations) {
    if (!b || !log_p || !iterations || (b->n_ev > 0 && !ev) || (b->Q > 0 && !codes))
        return sbn_fail(SBN_E_INVALID, "null argument");
    if (b->version != 2) return wrong_call(b->version);
    return run_rows<true, false>(b, ev, ld_ev, n_rows, n_iterations, damping, tol, ld_codes, iterations, [&](int64_t r0, int64_t n) {
        if (b->Q > 0)
            SBN_BP_CUDA(cudaMemcpy2DAsync(codes + r0, ld_codes, b->d_codes, b->cap, n, b->Q, cudaMemcpyDeviceToHost,
                                          b->stream));
        SBN_BP_CUDA(cudaMemcpyAsync(log_p + r0, b->d_log_p, n * 8, cudaMemcpyDeviceToHost, b->stream));
        return SBN_OK;
    });
}

int sbn_bp_counts_host(sbn_bp *b, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, int32_t n_iterations, float damping,
                       float tol, double *counts, double *log_z, int32_t *iterations) {
    if (!b || !log_z || !iterations || (b->n_ev > 0 && !ev) || (b->n_table_floats > 0 && !counts))
        return sbn_fail(SBN_E_INVALID, "null argument");
    if (b->version != 3) return wrong_call(b->version);
    std::fill(counts, counts + b->n_table_floats, 0.0);
    return run_rows<false, true>(b, ev, ld_ev, n_rows, n_iterations, damping, tol, n_rows, iterations,
                                 [&](int64_t r0, int64_t n) {
        const int64_t n_tab = b->n_table_floats;
        if (r0 == 0 && n_tab > 0) SBN_BP_CUDA(cudaMemsetAsync(b->d_counts, 0, n_tab * 8, b->stream));
        const int64_t grid = std::min<int64_t>(b->count_grid, (n + kThreads - 1) / kThreads);
        BpArgs a{b->d_words, static_cast<int>(b->words.size()), b->d_tables, b->n_table_floats, b->tables_in_smem ? 1 : 0,
                 b->d_ev, b->d_msg, nullptr, b->d_iters, b->cap, n, n_iterations, damping, tol, nullptr, b->d_log_p};
        if (b->max_card <= 8)
            sbn_bp_counts_kernel<8><<<static_cast<unsigned>(grid), kThreads, b->smem, b->stream>>>(a, b->d_partial);
        else
            sbn_bp_counts_kernel<kMaxCard><<<static_cast<unsigned>(grid), kThreads, b->smem, b->stream>>>(a, b->d_partial);
        SBN_BP_CUDA(cudaGetLastError());
        if (n_tab > 0) {
            sbn_bp_counts_reduce<<<static_cast<unsigned>((n_tab + 31) / 32), 256, 0, b->stream>>>(
                b->d_partial, grid * kCountWarps, static_cast<int32_t>(n_tab), b->d_counts);
            SBN_BP_CUDA(cudaGetLastError());
        }
        SBN_BP_CUDA(cudaMemcpyAsync(log_z + r0, b->d_log_p, n * 8, cudaMemcpyDeviceToHost, b->stream));
        if (r0 + n == n_rows && n_tab > 0)
            SBN_BP_CUDA(cudaMemcpyAsync(counts, b->d_counts, n_tab * 8, cudaMemcpyDeviceToHost, b->stream));
        return SBN_OK;
    });
}

int sbn_bp_set_tables(sbn_bp *b, const float *tables, int64_t n_table_floats) {
    if (!b || (n_table_floats > 0 && !tables)) return sbn_fail(SBN_E_INVALID, "null argument");
    if (n_table_floats != b->n_table_floats)
        return sbn_fail(SBN_E_INVALID, "bp tables: %lld floats, the words were compiled for %d",
                        static_cast<long long>(n_table_floats), b->n_table_floats);
    if (n_table_floats == 0) return SBN_OK;
    SBN_BP_CUDA(cudaSetDevice(b->device));
    SBN_BP_CUDA(cudaStreamSynchronize(b->stream));
    SBN_BP_CUDA(cudaMemcpy(b->d_tables, tables, n_table_floats * 4, cudaMemcpyHostToDevice));
    return SBN_OK;
}

void sbn_bp_destroy(sbn_bp *b) {
    if (!b) return;
    cudaSetDevice(b->device);
    if (b->stream) cudaStreamSynchronize(b->stream);
    cudaFree(b->d_words);
    cudaFree(b->d_tables);
    cudaFree(b->d_ev);
    cudaFree(b->d_msg);
    cudaFree(b->d_out);
    cudaFree(b->d_iters);
    cudaFree(b->d_codes);
    cudaFree(b->d_log_p);
    cudaFree(b->d_partial);
    cudaFree(b->d_counts);
    if (b->stream) cudaStreamDestroy(b->stream);
    delete b;
}

}  // extern "C"
