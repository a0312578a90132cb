// sorobn_b200 -- contingency tables and decomposable family scores over a resident complete data set
// (structure learning's hot path: sorobn_b200/structure.py, DESIGN.md "Structure learning").
//
// The data set lives on the device as uint8 state codes [n_vars][ld], rows innermost (the evidence layout),
// uploaded once by sbn_tally_create.  A batch of families (child, parents) is counted exactly into one uint64
// arena, each family's table [.., parent 1, child] with the child fastest:
//
//   * shared path (sbn_tally_count): families are packed, in the caller's order, into groups whose tables fit
//     SBN_TALLY_SMEM_BINS uint32 bins together and whose members are at most kMaxStage distinct columns.  A CTA
//     takes blocks of kRows rows, stages that block's codes of the group's columns in shared memory once, and
//     bins every family of the group from there: each code byte is read from HBM once per group.  A table of
//     at most kVoteBins entries is counted by warp votes (one ballot per bin and 32 rows, lane b accumulating
//     bin b), which never serialises on a shared address; one of at most kMatchBins by warp-aggregated
//     increments (__match_any_sync: the lanes of one bin elect a leader that adds their number), so a hot bin
//     costs one atomic per warp and sub-row; a larger one by plain shared atomics.  The CTA flushes its
//     non-zero bins with 64-bit global atomics at the end.
//   * global path (sbn_tally_count_global): a family whose table alone exceeds the budget counts with 64-bit global
//     atomics straight from HBM.
//
// sbn_tally_score then reduces every table of the batch to its BIC or BDeu score in double, one CTA per family;
// sbn_tally_test reduces every table of a batch of conditional-independence tests to its G^2 or X^2 statistic,
// degrees of freedom and p-value, one CTA per test (constraint-based learning, structure.pc).
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

#include "sbn_internal.h"

namespace {

constexpr int kRows = 1024;      // rows per staged block; the device pitch is a multiple of it
constexpr int kThreads = 512;    // group kernel CTA
constexpr int kWarps = kThreads / 32;
constexpr int kMaxStage = 64;    // distinct staged columns of one group (kMaxStage * kRows bytes of shared memory)
constexpr int kVoteBins = 16;    // tables of at most this many entries are counted by warp votes
constexpr int kMatchBins = 256;  // up to this many, by warp-aggregated increments (one atomic per distinct bin)
constexpr int kMaxAxes = 22;     // members with more than one state: 2^22 >= every table the ABI accepts
constexpr int kDescWords = 4 + 2 * kMaxAxes;  // off, T, n_ax, pad | (slot, stride) per axis
constexpr int kScoreThreads = 128;
constexpr int kTestThreads = 256;
constexpr int kTestWarps = kTestThreads / 32;
constexpr int kThreadStratum = 32;  // strata of at most this many cells are reduced one per thread, larger ones one per warp
constexpr unsigned kFull = 0xffffffffu;

struct FamScore {
    long long off;  // first entry of the family's table in the arena
    int T, r;       // entries, states of the child
};

// Lane a < n_ax holds axis a's (byte offset of its staged row or column, stride); idx[i] = the table entry of row
// `r + i` for the four rows whose codes are the bytes of the 32-bit words read at base + offset + r.
__device__ __forceinline__ void tally_index(const uint8_t *base, int64_t r, int n_ax, long long ax_off, int ax_stride,
                                            uint32_t idx[4]) {
    idx[0] = idx[1] = idx[2] = idx[3] = 0;
    for (int a = 0; a < n_ax; ++a) {
        const long long off = __shfl_sync(kFull, ax_off, a);
        const uint32_t st = static_cast<uint32_t>(__shfl_sync(kFull, ax_stride, a));
        const uint32_t w = *reinterpret_cast<const uint32_t *>(base + off + r);
        idx[0] += (w & 0xffu) * st;
        idx[1] += ((w >> 8) & 0xffu) * st;
        idx[2] += ((w >> 16) & 0xffu) * st;
        idx[3] += (w >> 24) * st;
    }
}

}  // namespace

__global__ void __launch_bounds__(kThreads, 2)
sbn_tally_count(const uint8_t *__restrict__ codes, int64_t ld, int64_t n_rows, const int32_t *__restrict__ gvars,
                int n_gvars, const int32_t *__restrict__ desc, int n_fam, int slices, int n_bins,
                unsigned long long *__restrict__ out) {
    extern __shared__ __align__(16) unsigned char smem[];
    uint32_t *hist = reinterpret_cast<uint32_t *>(smem);
    uint8_t *stage = smem + ((n_bins * 4 + 15) & ~15);
    for (int i = threadIdx.x; i < n_bins; i += blockDim.x) hist[i] = 0;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t n_blocks = (n_rows + kRows - 1) / kRows;
    const int slice_rows = kRows / slices;
    const int n_items = n_fam * slices;
    constexpr int kVec = kRows / 16;
    for (int64_t blk = blockIdx.x; blk < n_blocks; blk += gridDim.x) {
        __syncthreads();  // the previous block's counting (and the zeroing) is done before the stage is rewritten
        const int64_t row0 = blk * kRows;
        for (int i = threadIdx.x; i < n_gvars * kVec; i += blockDim.x) {
            const int g = i / kVec, c = i - g * kVec;
            reinterpret_cast<uint4 *>(stage)[i] =
                __ldg(reinterpret_cast<const uint4 *>(codes + static_cast<int64_t>(gvars[g]) * ld + row0) + c);
        }
        __syncthreads();
        const int n_valid = static_cast<int>(min(static_cast<int64_t>(kRows), n_rows - row0));
        for (int item = warp; item < n_items; item += kWarps) {
            const int f = item / slices, s = item - f * slices;
            const int32_t *d = desc + static_cast<int64_t>(f) * kDescWords;
            const int off = d[0], T = d[1], n_ax = d[2];
            const long long ax_off = lane < n_ax ? static_cast<long long>(d[4 + 2 * lane]) * kRows : 0;
            const int ax_stride = lane < n_ax ? d[5 + 2 * lane] : 0;
            const int lo = s * slice_rows, hi = min(lo + slice_rows, n_valid);
            if (T <= kVoteBins) {
                uint32_t acc = 0;
                for (int b0 = lo; b0 < hi; b0 += 128) {
                    const int r = b0 + 4 * lane;
                    uint32_t idx[4];
                    tally_index(stage, r, n_ax, ax_off, ax_stride, idx);
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const bool valid = r + i < hi;
                        for (int b = 0; b < T; ++b) {
                            const unsigned bal = __ballot_sync(kFull, valid && idx[i] == static_cast<uint32_t>(b));
                            if (lane == b) acc += __popc(bal);
                        }
                    }
                }
                if (lane < T && acc) atomicAdd(hist + off + lane, acc);
            } else if (T <= kMatchBins) {
                for (int b0 = lo; b0 < hi; b0 += 128) {
                    const int r = b0 + 4 * lane;
                    uint32_t idx[4];
                    tally_index(stage, r, n_ax, ax_off, ax_stride, idx);
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const bool valid = r + i < hi;
                        const unsigned peers = __match_any_sync(kFull, valid ? idx[i] : 0xffffffffu);
                        if (valid && lane == __ffs(peers) - 1) atomicAdd(hist + off + idx[i], __popc(peers));
                    }
                }
            } else {
                for (int b0 = lo; b0 < hi; b0 += 128) {
                    const int r = b0 + 4 * lane;
                    uint32_t idx[4];
                    tally_index(stage, r, n_ax, ax_off, ax_stride, idx);
#pragma unroll
                    for (int i = 0; i < 4; ++i)
                        if (r + i < hi) atomicAdd(hist + off + idx[i], 1u);
                }
            }
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < n_bins; i += blockDim.x)
        if (hist[i]) atomicAdd(out + i, static_cast<unsigned long long>(hist[i]));
}

__global__ void __launch_bounds__(256)
sbn_tally_count_global(const uint8_t *__restrict__ codes, int64_t ld, int64_t n_rows, const int32_t *__restrict__ d,
                       unsigned long long *__restrict__ out) {
    const int lane = threadIdx.x & 31;
    const int n_ax = d[2];
    const long long ax_off = lane < n_ax ? static_cast<long long>(d[4 + 2 * lane]) * ld : 0;
    const int ax_stride = lane < n_ax ? d[5 + 2 * lane] : 0;
    const int64_t step = 4LL * gridDim.x * blockDim.x;
    // whole warps iterate together (the axis shuffles); a lane past the last row reads nothing
    for (int64_t b0 = 4LL * (static_cast<int64_t>(blockIdx.x) * blockDim.x + (threadIdx.x & ~31)); b0 < n_rows; b0 += step) {
        const int64_t r = b0 + 4 * lane;
        uint32_t idx[4];
        tally_index(codes, r < n_rows ? r : 0, n_ax, ax_off, ax_stride, idx);
#pragma unroll
        for (int i = 0; i < 4; ++i)
            if (r + i < n_rows) atomicAdd(out + idx[i], 1ull);
    }
}

__global__ void __launch_bounds__(kScoreThreads)
sbn_tally_score(const unsigned long long *__restrict__ counts, const FamScore *__restrict__ fams, int kind, double ess,
                double n_rows, double *__restrict__ scores) {
    __shared__ double part[kScoreThreads];
    const FamScore fm = fams[blockIdx.x];
    const int r = fm.r, q = fm.T / fm.r;
    const double a_j = ess / q, a_jk = ess / fm.T;
    const double lg_j = kind == 1 ? lgamma(a_j) : 0.0, lg_jk = kind == 1 ? lgamma(a_jk) : 0.0;
    double acc = 0.0;
    // a parent configuration without rows adds exactly 0 to either score
    for (int j = threadIdx.x; j < q; j += blockDim.x) {
        const unsigned long long *c = counts + fm.off + static_cast<long long>(j) * r;
        unsigned long long nj = 0;
        for (int k = 0; k < r; ++k) nj += c[k];
        if (nj == 0) continue;
        const double dj = static_cast<double>(nj);
        if (kind == 0) {
            for (int k = 0; k < r; ++k)
                if (c[k]) {
                    const double n = static_cast<double>(c[k]);
                    acc += n * log(n / dj);
                }
        } else {
            acc += lg_j - lgamma(dj + a_j);
            for (int k = 0; k < r; ++k)
                if (c[k]) acc += lgamma(static_cast<double>(c[k]) + a_jk) - lg_jk;
        }
    }
    part[threadIdx.x] = acc;
    __syncthreads();
    for (int w = kScoreThreads / 2; w > 0; w >>= 1) {
        if (threadIdx.x < w) part[threadIdx.x] += part[threadIdx.x + w];
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        double s = part[0];
        if (kind == 0) s -= 0.5 * log(n_rows) * static_cast<double>(q) * static_cast<double>(r - 1);
        scores[blockIdx.x] = s;
    }
}

namespace {

// log(1 + d) - d, by its series where the two terms would cancel
__device__ double log1pmx(double d) {
    if (fabs(d) > 0.5) return log1p(d) - d;
    double pw = d, sum = 0.0;
    for (int k = 2; k < 100; ++k) {
        pw *= -d;
        const double term = pw / k;
        sum += term;
        if (fabs(term) <= 1e-17 * fabs(sum)) break;
    }
    return sum;
}

// Q(a, x), the regularised upper incomplete gamma function, for a > 0 and x > 0: the series of P below a + 1, the
// continued fraction of Q (modified Lentz) above.  The prefactor x^a e^-x / Gamma(a) is taken in the log domain;
// from a = 10 on through Stirling's series, a log1pmx((x - a) / a) + ln(a / 2 pi) / 2 - (the correction to
// Stirling), which keeps its absolute error near 1e-13 at a = 2^21 where a ln x and lgamma(a) are both ~3e7.
__device__ __noinline__ double upper_gamma_q(double a, double x) {
    double lp;
    if (a < 10.0) {
        lp = a * log(x) - x - lgamma(a);
    } else {
        const double ia = 1.0 / a, ia2 = ia * ia;
        const double corr = ia * (1.0 / 12 - ia2 * (1.0 / 360 - ia2 * (1.0 / 1260 - ia2 / 1680)));
        lp = a * log1pmx((x - a) * ia) + 0.5 * log(a / (2.0 * 3.14159265358979323846)) - corr;
    }
    if (x < a + 1.0) {
        double ap = a, del = 1.0 / a, sum = del;
        for (int n = 0; n < 1000000; ++n) {
            ap += 1.0;
            del *= x / ap;
            sum += del;
            if (fabs(del) <= 1e-17 * fabs(sum)) break;
        }
        return 1.0 - sum * exp(lp);
    }
    constexpr double kTiny = 1e-300;
    double b = x + 1.0 - a, c = 1.0 / kTiny, d = 1.0 / b, h = d;
    for (int i = 1; i < 1000000; ++i) {
        const double an = -i * (i - a);
        b += 2.0;
        d = an * d + b;
        if (fabs(d) < kTiny) d = kTiny;
        c = b + an / c;
        if (fabs(c) < kTiny) c = kTiny;
        d = 1.0 / d;
        const double del = d * c;
        h *= del;
        if (fabs(del - 1.0) <= 1e-16) break;
    }
    return exp(lp) * h;
}

// The contribution of one cell with count n, margins nx = N_xz and ny = N_yz in a stratum of nz rows: G^2 / 2
// (the factor 2 is applied to the sum) over the non-zero cells, X^2 over the cells whose expected count is > 0.
__device__ __forceinline__ double test_cell(int kind, double n, double nx, double ny, double nz) {
    if (kind == SBN_TEST_G2) return n > 0.0 ? n * log(n * nz / (nx * ny)) : 0.0;
    if (nx == 0.0 || ny == 0.0) return 0.0;
    const double e = nx * ny / nz, r = n - e;
    return r * r / e;
}

}  // namespace

// One CTA per test: the table [..][y][x] of test `blockIdx.x` (x fastest) is a run of strata of rx * ry entries.
// A stratum of at most kThreadStratum cells is reduced by one thread, recomputing its margins per cell; a larger
// one by one warp, with its margins in shared memory.  Thread (warp) i takes strata i, i + 256 (8), ..; each
// thread sums its cells in a fixed order and the CTA adds the threads in a fixed tree, so the result is bitwise
// reproducible.  Margins and dof are exact integers (every count is below 2^32).
__global__ void __launch_bounds__(kTestThreads)
sbn_tally_test(const unsigned long long *__restrict__ counts, const FamScore *__restrict__ fams,
               const int32_t *__restrict__ ry_of, int kind, double *__restrict__ out) {
    __shared__ uint32_t marg[kTestWarps][2][256];
    __shared__ double part[kTestThreads];
    __shared__ long long dpart[kTestThreads];
    const FamScore fm = fams[blockIdx.x];
    const int rx = fm.r, ry = ry_of[blockIdx.x], S = rx * ry;
    const long long n_strata = fm.T / S;
    const unsigned long long *tab = counts + fm.off;
    double acc = 0.0;
    long long dof = 0;
    if (S <= kThreadStratum) {
        for (long long z = threadIdx.x; z < n_strata; z += kTestThreads) {
            const unsigned long long *c = tab + z * S;
            unsigned long long nz = 0;
            int a = 0, b = 0;
            for (int x = 0; x < rx; ++x) {
                unsigned long long s = 0;
                for (int y = 0; y < ry; ++y) s += c[y * rx + x];
                a += s > 0;
                nz += s;
            }
            if (nz == 0) continue;  // an empty stratum adds nothing
            for (int y = 0; y < ry; ++y) {
                unsigned long long s = 0;
                for (int x = 0; x < rx; ++x) s += c[y * rx + x];
                b += s > 0;
            }
            dof += static_cast<long long>(a - 1) * (b - 1);
            const double dz = static_cast<double>(nz);
            for (int y = 0; y < ry; ++y) {
                unsigned long long ny = 0;
                for (int x = 0; x < rx; ++x) ny += c[y * rx + x];
                for (int x = 0; x < rx; ++x) {
                    unsigned long long nx = 0;
                    for (int y2 = 0; y2 < ry; ++y2) nx += c[y2 * rx + x];
                    acc += test_cell(kind, static_cast<double>(c[y * rx + x]), static_cast<double>(nx),
                                     static_cast<double>(ny), dz);
                }
            }
        }
    } else {
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        uint32_t *mx = marg[warp][0], *my = marg[warp][1];
        for (long long z = warp; z < n_strata; z += kTestWarps) {
            const unsigned long long *c = tab + z * S;
            unsigned long long nz = 0;
            int a = 0, b = 0;
            for (int x = lane; x < rx; x += 32) {
                unsigned long long s = 0;
                for (int y = 0; y < ry; ++y) s += c[y * rx + x];
                mx[x] = static_cast<uint32_t>(s);
                a += s > 0;
                nz += s;
            }
            for (int y = lane; y < ry; y += 32) {
                unsigned long long s = 0;
                for (int x = 0; x < rx; ++x) s += c[y * rx + x];
                my[y] = static_cast<uint32_t>(s);
                b += s > 0;
            }
            for (int o = 16; o > 0; o >>= 1) {
                nz += __shfl_xor_sync(kFull, nz, o);
                a += __shfl_xor_sync(kFull, a, o);
                b += __shfl_xor_sync(kFull, b, o);
            }
            __syncwarp();
            if (nz != 0) {
                if (lane == 0) dof += static_cast<long long>(a - 1) * (b - 1);
                const double dz = static_cast<double>(nz);
                for (int i = lane; i < S; i += 32) {
                    const int y = i / rx, x = i - y * rx;
                    acc += test_cell(kind, static_cast<double>(c[i]), static_cast<double>(mx[x]),
                                     static_cast<double>(my[y]), dz);
                }
            }
            __syncwarp();  // every lane is done with the margins before the next stratum rewrites them
        }
    }
    part[threadIdx.x] = acc;
    dpart[threadIdx.x] = dof;
    __syncthreads();
    for (int w = kTestThreads / 2; w > 0; w >>= 1) {
        if (threadIdx.x < w) {
            part[threadIdx.x] += part[threadIdx.x + w];
            dpart[threadIdx.x] += dpart[threadIdx.x + w];
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        const double stat = kind == SBN_TEST_G2 ? 2.0 * part[0] : part[0];
        const long long df = dpart[0];
        double p = 1.0;
        if (df > 0 && stat > 0.0) p = upper_gamma_q(0.5 * static_cast<double>(df), 0.5 * stat);
        out[3LL * blockIdx.x] = stat;
        out[3LL * blockIdx.x + 1] = static_cast<double>(df);
        out[3LL * blockIdx.x + 2] = p;
    }
}

namespace {

// One parsed batch: the descriptors of every family (groups' families consecutive), the staged columns of every
// group, and how each group or global family is launched.
struct Launch {
    bool global;
    int first;           // first family (descriptor index)
    int n_fam, n_bins;   // shared path: families, bins of the group
    int gvar_first, n_gvars;
    long long out;       // arena offset of the first entry
};
struct Batch {
    std::vector<int32_t> desc;
    std::vector<int32_t> gvars;
    std::vector<FamScore> fams;
    std::vector<Launch> launches;
    long long n_counts = 0;
};

}  // namespace

struct sbn_tally {
    int device = 0;
    int n_sms = 1;
    int n_vars = 0;
    int64_t n_rows = 0, ld = 0;
    std::vector<int32_t> card;
    uint8_t *d_codes = nullptr;
    unsigned long long *d_counts = nullptr;
    int64_t counts_cap = 0;
    void *d_words = nullptr;  // descriptors, staged columns, score records, scores
    int64_t words_cap = 0;
    void *d_tests = nullptr;  // the y cards of a batch of tests, then its [n_tests][3] results
    int64_t tests_cap = 0;
    cudaStream_t stream = nullptr;
};

namespace {

#define SBN_TALLY_CUDA(call)                                                                                      \
    do {                                                                                                        \
        cudaError_t e_ = (call);                                                                                \
        if (e_ != cudaSuccess)                                                                                  \
            return sbn_fail(e_ == cudaErrorMemoryAllocation ? SBN_E_NOMEM : SBN_E_CUDA, "%s failed: %s (%s:%d)", \
                            #call, cudaGetErrorString(e_), __FILE__, __LINE__);                                 \
    } while (0)

// Parse and bounds-check the family words (k, child, parent 1, .., parent k-1 per family) and pack the batch.
int parse_batch(const sbn_tally *t, const int32_t *words, int64_t n_words, Batch &B) {
    if (!words || n_words <= 0) return sbn_fail(SBN_E_INVALID, "no family words");
    std::vector<int> slot(t->n_vars, -1);
    std::vector<char> seen(t->n_vars, 0);
    Launch cur{false, 0, 0, 0, 0, 0, 0};
    auto close_group = [&]() {
        if (cur.n_fam) B.launches.push_back(cur);
        for (int g = cur.gvar_first; g < static_cast<int>(B.gvars.size()); ++g) slot[B.gvars[g]] = -1;
        cur = Launch{false, static_cast<int>(B.fams.size()), 0, 0, static_cast<int>(B.gvars.size()), 0, B.n_counts};
    };
    int64_t p = 0;
    while (p < n_words) {
        const int f = static_cast<int>(B.fams.size());
        const int32_t k = words[p++];
        if (k < 1 || k > t->n_vars || p + k > n_words)
            return sbn_fail(SBN_E_INVALID, "family %d: %d members (%d columns, %lld words left)", f, k, t->n_vars,
                            static_cast<long long>(n_words - p));
        long long T = 1;
        int n_ax = 0, n_new = 0;
        for (int i = 0; i < k; ++i) {
            const int32_t v = words[p + i];
            if (v < 0 || v >= t->n_vars) return sbn_fail(SBN_E_INVALID, "family %d: column %d of %d", f, v, t->n_vars);
            if (seen[v]) {
                for (int j = 0; j < i; ++j) seen[words[p + j]] = 0;
                return sbn_fail(SBN_E_INVALID, "family %d: column %d appears twice", f, v);
            }
            seen[v] = 1;
            T *= t->card[v];
            if (T > SBN_TALLY_MAX_TABLE) {
                for (int j = 0; j <= i; ++j) seen[words[p + j]] = 0;
                return sbn_fail(SBN_E_INVALID, "family %d: table of more than %d entries", f, SBN_TALLY_MAX_TABLE);
            }
            if (t->card[v] > 1) {
                ++n_ax;
                if (slot[v] < 0) ++n_new;
            }
        }
        for (int i = 0; i < k; ++i) seen[words[p + i]] = 0;
        const bool global = T > SBN_TALLY_SMEM_BINS;
        if (global || cur.n_bins + T > SBN_TALLY_SMEM_BINS || cur.n_gvars + n_new > kMaxStage) close_group();
        B.desc.resize(B.desc.size() + kDescWords, 0);
        int32_t *d = B.desc.data() + static_cast<int64_t>(f) * kDescWords;
        d[0] = global ? 0 : cur.n_bins;
        d[1] = static_cast<int32_t>(T);
        d[2] = n_ax;
        long long stride = 1;
        int a = 0;
        for (int i = 0; i < k; ++i) {
            const int32_t v = words[p + i];
            if (t->card[v] > 1) {
                if (global) {
                    d[4 + 2 * a] = v;
                } else {
                    if (slot[v] < 0) {
                        slot[v] = cur.n_gvars++;
                        B.gvars.push_back(v);
                    }
                    d[4 + 2 * a] = slot[v];
                }
                d[5 + 2 * a] = static_cast<int32_t>(stride);
                ++a;
            }
            stride *= t->card[v];
        }
        B.fams.push_back(FamScore{B.n_counts, static_cast<int>(T), t->card[words[p]]});
        if (global) {
            B.launches.push_back(Launch{true, f, 1, static_cast<int>(T), 0, 0, B.n_counts});
            B.n_counts += T;
            close_group();
        } else {
            cur.n_fam++;
            cur.n_bins += static_cast<int>(T);
            B.n_counts += T;
        }
        p += k;
    }
    close_group();
    return SBN_OK;
}

// Upload the batch, zero the arena and count every family of it into d_counts; d_scores (if any) follows the words
int run_counts(sbn_tally *t, const Batch &B, FamScore **d_fams, double **d_scores) {
    SBN_TALLY_CUDA(cudaSetDevice(t->device));
    const int64_t desc_bytes = round_up(static_cast<int64_t>(B.desc.size()) * 4, 256);
    const int64_t gvar_bytes = round_up(std::max<int64_t>(1, B.gvars.size()) * 4, 256);
    const int64_t fam_bytes = round_up(static_cast<int64_t>(B.fams.size()) * sizeof(FamScore), 256);
    const int64_t score_bytes = round_up(static_cast<int64_t>(B.fams.size()) * 8, 256);
    const int64_t need = desc_bytes + gvar_bytes + fam_bytes + score_bytes;
    if (need > t->words_cap) {
        if (t->d_words) SBN_TALLY_CUDA(cudaFree(t->d_words));
        t->d_words = nullptr;
        t->words_cap = 0;
        SBN_TALLY_CUDA(cudaMalloc(&t->d_words, need));
        t->words_cap = need;
    }
    if (B.n_counts > t->counts_cap) {
        if (t->d_counts) SBN_TALLY_CUDA(cudaFree(t->d_counts));
        t->d_counts = nullptr;
        t->counts_cap = 0;
        SBN_TALLY_CUDA(cudaMalloc(&t->d_counts, B.n_counts * sizeof(unsigned long long)));
        t->counts_cap = B.n_counts;
    }
    char *base = static_cast<char *>(t->d_words);
    int32_t *d_desc = reinterpret_cast<int32_t *>(base);
    int32_t *d_gvars = reinterpret_cast<int32_t *>(base + desc_bytes);
    *d_fams = reinterpret_cast<FamScore *>(base + desc_bytes + gvar_bytes);
    *d_scores = reinterpret_cast<double *>(base + desc_bytes + gvar_bytes + fam_bytes);
    SBN_TALLY_CUDA(cudaMemcpyAsync(d_desc, B.desc.data(), B.desc.size() * 4, cudaMemcpyHostToDevice, t->stream));
    if (!B.gvars.empty())
        SBN_TALLY_CUDA(cudaMemcpyAsync(d_gvars, B.gvars.data(), B.gvars.size() * 4, cudaMemcpyHostToDevice, t->stream));
    SBN_TALLY_CUDA(cudaMemcpyAsync(*d_fams, B.fams.data(), B.fams.size() * sizeof(FamScore), cudaMemcpyHostToDevice,
                                   t->stream));
    SBN_TALLY_CUDA(cudaMemsetAsync(t->d_counts, 0, B.n_counts * sizeof(unsigned long long), t->stream));
    const int64_t n_blocks = (t->n_rows + kRows - 1) / kRows;
    for (const Launch &L : B.launches) {
        const int32_t *d = d_desc + static_cast<int64_t>(L.first) * kDescWords;
        if (L.global) {
            const int64_t grid = std::min<int64_t>(8LL * t->n_sms, (t->n_rows + 1023) / 1024);
            sbn_tally_count_global<<<static_cast<int>(grid), 256, 0, t->stream>>>(t->d_codes, t->ld, t->n_rows, d,
                                                                           t->d_counts + L.out);
        } else {
            const int smem = ((L.n_bins * 4 + 15) & ~15) + L.n_gvars * kRows;
            int per_sm = 0;
            SBN_TALLY_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, sbn_tally_count, kThreads, smem));
            const int64_t grid = std::min<int64_t>(static_cast<int64_t>(std::max(per_sm, 1)) * t->n_sms, n_blocks);
            int slices = 1;
            while (slices < 8 && L.n_fam * slices * 2 <= kWarps) slices *= 2;
            sbn_tally_count<<<static_cast<int>(grid), kThreads, smem, t->stream>>>(
                t->d_codes, t->ld, t->n_rows, d_gvars + L.gvar_first, L.n_gvars, d, L.n_fam, slices, L.n_bins,
                t->d_counts + L.out);
        }
        SBN_TALLY_CUDA(cudaGetLastError());
    }
    return SBN_OK;
}

}  // namespace

extern "C" {

int sbn_tally_create(int device, const uint8_t *codes, int64_t ld, int32_t n_vars, int64_t n_rows, const int32_t *cards,
                     sbn_tally **out) {
    if (!codes || !cards || !out) return sbn_fail(SBN_E_INVALID, "null argument");
    *out = nullptr;
    if (n_vars < 1 || n_rows < 1 || ld < n_rows)
        return sbn_fail(SBN_E_INVALID, "bad shape: %d columns, %lld rows, pitch %lld", n_vars,
                        static_cast<long long>(n_rows), static_cast<long long>(ld));
    if (n_rows >= (1LL << 32)) return sbn_fail(SBN_E_INVALID, "%lld rows: at most 2^32 - 1", static_cast<long long>(n_rows));
    for (int v = 0; v < n_vars; ++v) {
        if (cards[v] < 1 || cards[v] > 256) return sbn_fail(SBN_E_INVALID, "column %d has %d states", v, cards[v]);
        const uint8_t *row = codes + static_cast<int64_t>(v) * ld;
        uint8_t top = 0;
        for (int64_t b = 0; b < n_rows; ++b) top = std::max(top, row[b]);
        if (top >= cards[v]) return sbn_fail(SBN_E_INVALID, "column %d holds code %d of %d states", v, top, cards[v]);
    }
    int n_dev = 0;
    if (cudaGetDeviceCount(&n_dev) != cudaSuccess || n_dev == 0) return sbn_fail(SBN_E_NODEVICE, "no CUDA device available");
    if (device < 0 || device >= n_dev) return sbn_fail(SBN_E_NODEVICE, "device %d out of range (%d visible)", device, n_dev);
    sbn_tally *t = new sbn_tally();
    t->device = device;
    t->n_vars = n_vars;
    t->n_rows = n_rows;
    t->ld = round_up(n_rows, kRows);
    t->card.assign(cards, cards + n_vars);
    auto bail = [&](int code) {
        sbn_tally_destroy(t);
        return code;
    };
#define SBN_TALLY_CUDA_T(call)                                                                                          \
    do {                                                                                                              \
        cudaError_t e_ = (call);                                                                                      \
        if (e_ != cudaSuccess)                                                                                        \
            return bail(sbn_fail(e_ == cudaErrorMemoryAllocation ? SBN_E_NOMEM : SBN_E_CUDA, "%s failed: %s (%s:%d)", \
                                 #call, cudaGetErrorString(e_), __FILE__, __LINE__));                                 \
    } while (0)
    SBN_TALLY_CUDA_T(cudaSetDevice(device));
    cudaDeviceProp prop;
    SBN_TALLY_CUDA_T(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0)
        return bail(sbn_fail(SBN_E_NODEVICE, "device %d is sm_%d%d; this library is built for sm_90a only", device,
                             prop.major, prop.minor));
    t->n_sms = prop.multiProcessorCount;
    SBN_TALLY_CUDA_T(cudaFuncSetAttribute(sbn_tally_count, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          SBN_TALLY_SMEM_BINS * 4 + kMaxStage * kRows));
    SBN_TALLY_CUDA_T(cudaStreamCreateWithFlags(&t->stream, cudaStreamNonBlocking));
    const size_t bytes = static_cast<size_t>(n_vars) * static_cast<size_t>(t->ld);
    SBN_TALLY_CUDA_T(cudaMalloc(&t->d_codes, bytes));
    SBN_TALLY_CUDA_T(cudaMemsetAsync(t->d_codes, 0, bytes, t->stream));  // the pitch's padding reads as state 0
    SBN_TALLY_CUDA_T(cudaMemcpy2DAsync(t->d_codes, t->ld, codes, ld, n_rows, n_vars, cudaMemcpyHostToDevice, t->stream));
    SBN_TALLY_CUDA_T(cudaStreamSynchronize(t->stream));
#undef SBN_TALLY_CUDA_T
    *out = t;
    return SBN_OK;
}

int sbn_tally_counts(sbn_tally *t, const int32_t *words, int64_t n_words, uint64_t *counts, int64_t n_counts) {
    if (!t || !counts) return sbn_fail(SBN_E_INVALID, "null argument");
    Batch B;
    int rc = parse_batch(t, words, n_words, B);
    if (rc != SBN_OK) return rc;
    if (n_counts != B.n_counts)
        return sbn_fail(SBN_E_INVALID, "the families have %lld table entries, not %lld", B.n_counts,
                        static_cast<long long>(n_counts));
    FamScore *d_fams;
    double *d_scores;
    rc = run_counts(t, B, &d_fams, &d_scores);
    if (rc != SBN_OK) return rc;
    SBN_TALLY_CUDA(cudaMemcpyAsync(counts, t->d_counts, B.n_counts * sizeof(uint64_t), cudaMemcpyDeviceToHost, t->stream));
    SBN_TALLY_CUDA(cudaStreamSynchronize(t->stream));
    return SBN_OK;
}

int sbn_tally_scores(sbn_tally *t, const int32_t *words, int64_t n_words, int kind, double ess, double *scores,
                     int64_t n_families) {
    if (!t || !scores) return sbn_fail(SBN_E_INVALID, "null argument");
    if (kind != SBN_SCORE_BIC && kind != SBN_SCORE_BDEU) return sbn_fail(SBN_E_INVALID, "unknown score kind %d", kind);
    if (kind == SBN_SCORE_BDEU && !(ess > 0.0 && std::isfinite(ess)))
        return sbn_fail(SBN_E_INVALID, "BDeu needs a positive equivalent sample size, not %g", ess);
    Batch B;
    int rc = parse_batch(t, words, n_words, B);
    if (rc != SBN_OK) return rc;
    if (n_families != static_cast<int64_t>(B.fams.size()))
        return sbn_fail(SBN_E_INVALID, "the words hold %zu families, not %lld", B.fams.size(),
                        static_cast<long long>(n_families));
    FamScore *d_fams;
    double *d_scores;
    rc = run_counts(t, B, &d_fams, &d_scores);
    if (rc != SBN_OK) return rc;
    sbn_tally_score<<<static_cast<unsigned>(B.fams.size()), kScoreThreads, 0, t->stream>>>(
        t->d_counts, d_fams, kind, ess, static_cast<double>(t->n_rows), d_scores);
    SBN_TALLY_CUDA(cudaGetLastError());
    SBN_TALLY_CUDA(cudaMemcpyAsync(scores, d_scores, B.fams.size() * sizeof(double), cudaMemcpyDeviceToHost, t->stream));
    SBN_TALLY_CUDA(cudaStreamSynchronize(t->stream));
    return SBN_OK;
}

int sbn_tally_tests(sbn_tally *t, const int32_t *words, int64_t n_words, int kind, double *out, int64_t n_tests) {
    if (!t || !out) return sbn_fail(SBN_E_INVALID, "null argument");
    if (kind != SBN_TEST_G2 && kind != SBN_TEST_CHI2) return sbn_fail(SBN_E_INVALID, "unknown test kind %d", kind);
    Batch B;
    int rc = parse_batch(t, words, n_words, B);
    if (rc != SBN_OK) return rc;
    if (n_tests != static_cast<int64_t>(B.fams.size()))
        return sbn_fail(SBN_E_INVALID, "the words hold %zu tests, not %lld", B.fams.size(), static_cast<long long>(n_tests));
    // parse_batch has checked every test's words; a test needs x and y
    std::vector<int32_t> ry(B.fams.size());
    for (int64_t p = 0, f = 0; p < n_words; p += 1 + words[p], ++f) {
        if (words[p] < 2) return sbn_fail(SBN_E_INVALID, "test %lld: %d members, at least x and y are needed",
                                          static_cast<long long>(f), words[p]);
        ry[f] = t->card[words[p + 2]];
    }
    FamScore *d_fams;
    double *d_scores;
    rc = run_counts(t, B, &d_fams, &d_scores);
    if (rc != SBN_OK) return rc;
    const int64_t ry_bytes = round_up(n_tests * 4, 256);
    const int64_t need = ry_bytes + n_tests * 3 * static_cast<int64_t>(sizeof(double));
    if (need > t->tests_cap) {
        if (t->d_tests) SBN_TALLY_CUDA(cudaFree(t->d_tests));
        t->d_tests = nullptr;
        t->tests_cap = 0;
        SBN_TALLY_CUDA(cudaMalloc(&t->d_tests, need));
        t->tests_cap = need;
    }
    int32_t *d_ry = static_cast<int32_t *>(t->d_tests);
    double *d_out = reinterpret_cast<double *>(static_cast<char *>(t->d_tests) + ry_bytes);
    SBN_TALLY_CUDA(cudaMemcpyAsync(d_ry, ry.data(), n_tests * 4, cudaMemcpyHostToDevice, t->stream));
    sbn_tally_test<<<static_cast<unsigned>(n_tests), kTestThreads, 0, t->stream>>>(t->d_counts, d_fams, d_ry, kind, d_out);
    SBN_TALLY_CUDA(cudaGetLastError());
    SBN_TALLY_CUDA(cudaMemcpyAsync(out, d_out, n_tests * 3 * sizeof(double), cudaMemcpyDeviceToHost, t->stream));
    SBN_TALLY_CUDA(cudaStreamSynchronize(t->stream));
    return SBN_OK;
}

void sbn_tally_destroy(sbn_tally *t) {
    if (!t) return;
    cudaSetDevice(t->device);
    if (t->stream) cudaStreamSynchronize(t->stream);
    cudaFree(t->d_codes);
    cudaFree(t->d_counts);
    cudaFree(t->d_words);
    cudaFree(t->d_tests);
    if (t->stream) cudaStreamDestroy(t->stream);
    delete t;
}

}  // extern "C"
