// sorobn_b200 -- Gibbs sampling on the device (BASELINE.json configs[4]).
//
// Mirrors `BayesNet._gibbs_sampling` (/root/reference/sorobn/bayes_net.py:665-737):
//   * start from a forward sample with the event variables clamped (bayes_net.py:715,
//     `self.sample(init=event)` -> `_forward_sample`, :518-548);
//   * every iteration takes the next non-event variable in a fixed cycle (sorted by name,
//     :697 and :718) and resamples it from P(var | Markov blanket) (:724-729);
//   * after every iteration the current state of the query variables is recorded (:732-733);
//   * the answer is the frequency of each joint query state (:736-737).
// The reference precomputes one table per variable over its whole Markov boundary with pandas
// (:699-712); here the conditional is evaluated on the fly, which needs only the CPT of the
// variable and of its children:
//     P(v = x | blanket)  ~  P(x | pa(v)) * prod_{c in children(v)} P(c | pa(c) with v = x)
// One thread runs one chain (one evidence row): a chain is a serial dependency (every update reads
// the state the previous one wrote), so its speed is the LATENCY of one update, and 10k chains are
// 10k independent latency chains -- splitting an update over lanes would add instructions without
// shortening that chain.  What shortens it is keeping everything an update touches on chip:
//   * the resampling cycle is compiled on the host into one record per position (variable,
//     cardinality, CPT base, (parent, stride) pairs, per child its CPT base / own state / stride of
//     the variable / other (parent, stride) pairs) -- one broadcast shared-memory read per word
//     instead of the pointer chase through the CSR arrays in global memory;
//   * every CPT is staged in shared memory when the network's tables fit (42 KB for the 100-node
//     benchmark grid), the chain states live there as [variable][chain] bytes (conflict-free);
//   * the weights of the <= 8 states stay in registers (SBN_GIBBS_MAX_CARD falls back to local memory).
// 64 chains per CTA: 10k chains make 157 CTAs, one or two per SM on all 132 SMs of an H100.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define SBN_GIBBS_THREADS 128       // forward-sampling kernel
#define SBN_GIBBS_CHAINS 64         // chains (threads) per CTA of the Gibbs kernel
#define SBN_GIBBS_MAX_CARD 64

struct SbnGibbs {
    int32_t n_vars;
    int32_t n_cycle;             // non-event variables
    int32_t n_query;
    int32_t Q;                   // joint query states
    int32_t n_ev;
    int32_t pad_;
    const int32_t *card;         // [n_vars]
    const int32_t *cpt_off;      // [n_vars] float offset of each CPT (axes [*parents, var], var fastest)
    const int32_t *par_ptr;      // [n_vars + 1] CSR of parents
    const int32_t *par_idx;      //   parent ids
    const int32_t *par_stride;   //   stride of that parent in the child's CPT
    const int32_t *chi_ptr;      // [n_vars + 1] CSR of children
    const int32_t *chi_idx;      //   child ids
    const int32_t *chi_stride;   //   stride of the variable inside that child's CPT
    const int32_t *cycle;        // [n_cycle] variable ids in cycle order
    const int32_t *prog;         // compiled cycle: [n_cycle] record positions, then the records (see sbn_gibbs_kernel)
    int32_t prog_words;
    int32_t tables_in_smem;      // 1: every CPT is staged in shared memory (table_floats of them)
    int32_t table_floats;
    int32_t pad2_;
    const int32_t *query;        // [n_query] query variable ids, slowest first
    const int32_t *ev_var;       // [n_ev] evidence variable ids (column order of `ev`)
    const float *tables;
    const uint8_t *ev;           // [n_ev][ld_ev] state codes
    int64_t ld_ev;
    float *out;                  // [Q][ld_out] frequencies
    int64_t ld_out;
    int64_t n_chains;
    int64_t n_iterations;
    uint64_t seed;
};

// Philox-4x32-10 (Salmon et al. 2011): counter-based, so chain c / draw k is reproducible.
__device__ __forceinline__ void sbn_philox(uint32_t (&ctr)[4], uint32_t k0, uint32_t k1) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint32_t hi0 = __umulhi(0xD2511F53u, ctr[0]), lo0 = 0xD2511F53u * ctr[0];
        const uint32_t hi1 = __umulhi(0xCD9E8D57u, ctr[2]), lo1 = 0xCD9E8D57u * ctr[2];
        const uint32_t n0 = hi1 ^ ctr[1] ^ k0, n2 = hi0 ^ ctr[3] ^ k1;
        ctr[0] = n0;
        ctr[1] = lo1;
        ctr[2] = n2;
        ctr[3] = lo0;
        k0 += 0x9E3779B9u;
        k1 += 0xBB67AE85u;
    }
}

struct SbnRng {
    uint32_t buf[4];
    uint32_t k0, k1, chain_lo, chain_hi;
    uint32_t counter;
    int have;
    __device__ void init(uint64_t seed, uint64_t chain) {
        k0 = static_cast<uint32_t>(seed);
        k1 = static_cast<uint32_t>(seed >> 32);
        chain_lo = static_cast<uint32_t>(chain);
        chain_hi = static_cast<uint32_t>(chain >> 32);
        counter = 0;
        have = 0;
    }
    __device__ float uniform() {  // (0, 1]
        if (have == 0) {
            buf[0] = counter++;
            buf[1] = 0;
            buf[2] = chain_lo;
            buf[3] = chain_hi;
            sbn_philox(buf, k0, k1);
            have = 4;
        }
        --have;  // a select chain keeps buf[] in registers (dynamic indexing would put it in local memory)
        const uint32_t u = have == 3 ? buf[3] : have == 2 ? buf[2] : have == 1 ? buf[1] : buf[0];
        return (static_cast<float>(u >> 8) + 1.0f) * (1.0f / 16777216.0f);
    }
};

// Record of one cycle position (int32 words; built by sbn_gibbs_create):
//   [0] variable | card << 16   [1] float offset of its CPT row base   [2] n_parents | n_children << 8
//   n_parents x (parent variable, stride)
//   per child: [CPT base] [child variable] [stride of the variable in the child's CPT] [n_other]
//              n_other x (other parent variable, stride)
// Un-normalised P(v = x | Markov blanket) for x < card into w[] (bayes_net.py:699-712 computes the
// same table ahead of time with pandas; here it is evaluated for the current state only).
template <int MAXC, typename StateFn, typename TableFn>
__device__ __forceinline__ int sbn_gibbs_weights(const int32_t *__restrict__ r, StateFn state, TableFn table, float (&w)[MAXC]) {
    const int v_c = r[0];
    const int c = v_c >> 16;
    int base = r[1];
    const int np = r[2] & 0xff, nc = r[2] >> 8;
    r += 3;
    for (int k = 0; k < np; ++k, r += 2) base += state(r[0]) * r[1];
#pragma unroll
    for (int x = 0; x < MAXC; ++x) w[x] = x < c ? table(base + x) : 0.f;
    for (int j = 0; j < nc; ++j) {
        int cb = r[0] + state(r[1]);
        const int sv = r[2], no = r[3];
        r += 4;
        for (int k = 0; k < no; ++k, r += 2) cb += state(r[0]) * r[1];
#pragma unroll
        for (int x = 0; x < MAXC; ++x)
            if (x < c) w[x] *= table(cb + x * sv);
    }
    return v_c;
}

template <int MAXC>
__global__ void __launch_bounds__(SBN_GIBBS_CHAINS) sbn_gibbs_kernel(const __grid_constant__ SbnGibbs p) {
    extern __shared__ __align__(16) uint8_t s_raw[];
    // layout: program words | tables (optional) | state [n_vars][T] bytes | counts [Q][T] uint32
    constexpr int T = SBN_GIBBS_CHAINS;
    int32_t *s_prog = reinterpret_cast<int32_t *>(s_raw);
    float *s_tab = reinterpret_cast<float *>(s_prog + ((p.prog_words + 3) / 4) * 4);
    uint8_t *s_state0 = reinterpret_cast<uint8_t *>(s_tab + (p.tables_in_smem ? ((p.table_floats + 3) / 4) * 4 : 0));
    uint8_t *state = s_state0 + threadIdx.x;
    uint32_t *counts = reinterpret_cast<uint32_t *>(s_state0 + ((static_cast<size_t>(p.n_vars) * T + 15) / 16) * 16) + threadIdx.x;
    for (int i = threadIdx.x; i < p.prog_words; i += T) s_prog[i] = p.prog[i];
    if (p.tables_in_smem)
        for (int i = threadIdx.x; i < p.table_floats; i += T) s_tab[i] = p.tables[i];
    __syncthreads();

    const int64_t chain = static_cast<int64_t>(blockIdx.x) * T + threadIdx.x;
    if (chain >= p.n_chains) return;
    const bool tsm = p.tables_in_smem != 0;
    const float *__restrict__ gtab = p.tables;
    auto table = [&](int e) -> float { return tsm ? s_tab[e] : __ldg(gtab + e); };
    auto st = [&](int v) -> int { return state[v * T]; };
    SbnRng rng;
    rng.init(p.seed, static_cast<uint64_t>(chain));
    for (int q = 0; q < p.Q; ++q) counts[q * T] = 0;

    // ---- initial state: forward sample, event variables clamped (bayes_net.py:518-548)
    for (int v = 0; v < p.n_vars; ++v) state[v * T] = 0xff;
    for (int k = 0; k < p.n_ev; ++k) {
        const int v = p.ev_var[k];
        state[v * T] = min(static_cast<int>(p.ev[static_cast<int64_t>(k) * p.ld_ev + chain]), p.card[v] - 1);
    }
    for (int v = 0; v < p.n_vars; ++v) {  // variable ids are topological
        if (state[v * T] != 0xff) continue;
        int base = p.cpt_off[v];
        for (int k = p.par_ptr[v]; k < p.par_ptr[v + 1]; ++k) base += state[p.par_idx[k] * T] * p.par_stride[k];
        const int c = p.card[v];
        float u = rng.uniform(), acc = 0.f;
        int pick = c - 1;
        for (int x = 0; x < c; ++x) {
            acc += table(base + x);
            if (u <= acc) {
                pick = x;
                break;
            }
        }
        state[v * T] = static_cast<uint8_t>(pick);
    }
    // joint query index = sum_k state[query_k] * qstride_k; the last query variable is fastest
    int qvar[4], qstr[4];
    const int nq = min(p.n_query, 4);
    {
        int stride = 1;
        for (int k = p.n_query - 1; k >= 0; --k) {
            if (k < 4) {
                qvar[k] = p.query[k];
                qstr[k] = stride;
            }
            stride *= p.card[p.query[k]];
        }
    }

    // ---- the chain
    int cyc = 0;
    for (int64_t it = 0; it < p.n_iterations; ++it) {
        float w[MAXC];
        const int v_c = sbn_gibbs_weights<MAXC>(s_prog + s_prog[cyc], st, table, w);
        const int v = v_c & 0xffff, c = v_c >> 16;
        cyc = cyc + 1 == p.n_cycle ? 0 : cyc + 1;
        float cum[MAXC];
        float total = 0.f;
#pragma unroll
        for (int x = 0; x < MAXC; ++x) {
            total += w[x];
            cum[x] = total;
        }
        if (total > 0.f) {  // an all-zero conditional (deterministic CPTs) keeps the current value
            const float u = rng.uniform() * total;
            // first x with u <= cum[x] == number of x with cum[x] < u (cum is flat, = total >= u,
            // beyond the cardinality; a zero-weight state repeats its predecessor's cum and is never picked)
            int pick = 0;
#pragma unroll
            for (int x = 0; x < MAXC; ++x) pick += cum[x] < u ? 1 : 0;
            state[v * T] = static_cast<uint8_t>(min(pick, c - 1));
        }
        // record the joint state of the query variables (bayes_net.py:732-733)
        int qi = 0;
        if (p.n_query <= 4) {
#pragma unroll
            for (int k = 0; k < 4; ++k)
                if (k < nq) qi += state[qvar[k] * T] * qstr[k];
        } else {
            for (int k = 0; k < p.n_query; ++k) qi = qi * p.card[p.query[k]] + state[p.query[k] * T];
        }
        counts[qi * T] += 1;
    }
    const float inv = 1.0f / static_cast<float>(p.n_iterations);
    for (int q = 0; q < p.Q; ++q) p.out[static_cast<int64_t>(q) * p.ld_out + chain] = static_cast<float>(counts[q * T]) * inv;
}

// ---- the same chain, straight-line: networks whose variables have at most 8 states, 4 parents,
// 4 children and 4 (parent, stride) terms per CPT get a FIXED-size record per cycle position:
//   [0] variable | card << 16   [1] -   then SBN_GF_GROUPS groups (the variable's own CPT, then
//   its children) of [base, stride of the variable, 4 x (state index, stride)]
// padded with a dummy state slot that is always 0 and a dummy 1.0 table entry (stride 0).  Every
// word of the record, every state byte and every table entry of an update is then an independent
// load: the update's latency is three dependent shared-memory reads deep instead of one per loop
// iteration of the generic kernel.  Arithmetic and random
// stream are the generic kernel's, bit for bit (padding multiplies by 1.0f).
#define SBN_GF_GROUPS 5
#define SBN_GF_TERMS 4
#define SBN_GF_WORDS (2 + SBN_GF_GROUPS * (2 + 2 * SBN_GF_TERMS))

__global__ void __launch_bounds__(SBN_GIBBS_CHAINS) sbn_gibbs_flat_kernel(const __grid_constant__ SbnGibbs p) {
    extern __shared__ __align__(16) uint8_t s_raw[];
    // layout: records [n_cycle][SBN_GF_WORDS] | tables | state [n_vars + 1][T] bytes | counts [Q][T] uint32
    constexpr int T = SBN_GIBBS_CHAINS, MAXC = 8;
    int32_t *s_prog = reinterpret_cast<int32_t *>(s_raw);
    float *s_tab = reinterpret_cast<float *>(s_prog + ((p.prog_words + 3) / 4) * 4);
    uint8_t *s_state0 = reinterpret_cast<uint8_t *>(s_tab + ((p.table_floats + 3) / 4) * 4);
    uint8_t *state = s_state0 + threadIdx.x;
    uint32_t *counts = reinterpret_cast<uint32_t *>(s_state0 + ((static_cast<size_t>(p.n_vars + 1) * T + 15) / 16) * 16) + threadIdx.x;
    for (int i = threadIdx.x; i < p.prog_words; i += T) s_prog[i] = p.prog[i];
    for (int i = threadIdx.x; i < p.table_floats; i += T) s_tab[i] = p.tables[i];
    __syncthreads();

    const int64_t chain = static_cast<int64_t>(blockIdx.x) * T + threadIdx.x;
    if (chain >= p.n_chains) return;
    SbnRng rng;
    rng.init(p.seed, static_cast<uint64_t>(chain));
    for (int q = 0; q < p.Q; ++q) counts[q * T] = 0;

    // ---- initial state: forward sample, event variables clamped (bayes_net.py:518-548)
    for (int v = 0; v < p.n_vars; ++v) state[v * T] = 0xff;
    state[p.n_vars * T] = 0;  // the dummy slot padding terms read
    for (int k = 0; k < p.n_ev; ++k) {
        const int v = p.ev_var[k];
        state[v * T] = min(static_cast<int>(p.ev[static_cast<int64_t>(k) * p.ld_ev + chain]), p.card[v] - 1);
    }
    for (int v = 0; v < p.n_vars; ++v) {  // variable ids are topological
        if (state[v * T] != 0xff) continue;
        int base = p.cpt_off[v];
        for (int k = p.par_ptr[v]; k < p.par_ptr[v + 1]; ++k) base += state[p.par_idx[k] * T] * p.par_stride[k];
        const int c = p.card[v];
        float u = rng.uniform(), acc = 0.f;
        int pick = c - 1;
        for (int x = 0; x < c; ++x) {
            acc += s_tab[base + x];
            if (u <= acc) {
                pick = x;
                break;
            }
        }
        state[v * T] = static_cast<uint8_t>(pick);
    }
    int qvar[4] = {0, 0, 0, 0}, qstr[4] = {0, 0, 0, 0};
    {
        int stride = 1;
#pragma unroll
        for (int k = 3; k >= 0; --k)
            if (k < p.n_query) {
                qvar[k] = p.query[k];
                qstr[k] = stride;
                stride *= p.card[p.query[k]];
            }
    }

    // ---- the chain
    int cyc = 0;
    for (int64_t it = 0; it < p.n_iterations; ++it) {
        const int4 *r4 = reinterpret_cast<const int4 *>(s_prog + cyc * SBN_GF_WORDS);
        cyc = cyc + 1 == p.n_cycle ? 0 : cyc + 1;
        int rw[SBN_GF_WORDS];
#pragma unroll
        for (int i = 0; i < SBN_GF_WORDS / 4; ++i) {
            const int4 t = r4[i];
            rw[4 * i] = t.x;
            rw[4 * i + 1] = t.y;
            rw[4 * i + 2] = t.z;
            rw[4 * i + 3] = t.w;
        }
        const float u01 = rng.uniform();  // independent of the loads: overlaps them
        const int v = rw[0] & 0xffff, c = rw[0] >> 16;
        float w[MAXC];
#pragma unroll
        for (int x = 0; x < MAXC; ++x) w[x] = 1.f;
#pragma unroll
        for (int g = 0; g < SBN_GF_GROUPS; ++g) {
            const int *gw = rw + 2 + g * (2 + 2 * SBN_GF_TERMS);
            int base = gw[0];
#pragma unroll
            for (int k = 0; k < SBN_GF_TERMS; ++k) base += state[gw[2 + 2 * k] * T] * gw[3 + 2 * k];
            const int sv = gw[1];
#pragma unroll
            for (int x = 0; x < MAXC; ++x)
                if (x < c) w[x] = g == 0 ? s_tab[base + x * sv] : w[x] * s_tab[base + x * sv];
        }
        float cum[MAXC];
        float total = 0.f;
#pragma unroll
        for (int x = 0; x < MAXC; ++x) {
            total += x < c ? w[x] : 0.f;
            cum[x] = total;
        }
        if (total > 0.f) {  // an all-zero conditional (deterministic CPTs) keeps the current value
            const float u = u01 * total;
            int pick = 0;
#pragma unroll
            for (int x = 0; x < MAXC; ++x) pick += cum[x] < u ? 1 : 0;
            state[v * T] = static_cast<uint8_t>(min(pick, c - 1));
        }
        // record the joint state of the query variables (bayes_net.py:732-733)
        int qi = 0;
#pragma unroll
        for (int k = 0; k < 4; ++k) qi += state[qvar[k] * T] * qstr[k];
        counts[qi * T] += 1;
    }
    const float inv = 1.0f / static_cast<float>(p.n_iterations);
    for (int q = 0; q < p.Q; ++q) p.out[static_cast<int64_t>(q) * p.ld_out + chain] = static_cast<float>(counts[q * T]) * inv;
}

// The conditional the chain samples from, for one given joint state: P(v | blanket) normalised.
// Same device function as the chain (tests pin it to the reference's precomputed tables).
__global__ void sbn_gibbs_conditional_kernel(const SbnGibbs p, int pos, const uint8_t *__restrict__ joint, float *__restrict__ out) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    float w[SBN_GIBBS_MAX_CARD];
    const float *gtab = p.tables;
    auto table = [&](int e) -> float { return gtab[e]; };
    auto st = [&](int v) -> int { return joint[v]; };
    const int c = sbn_gibbs_weights<SBN_GIBBS_MAX_CARD>(p.prog + p.prog[pos], st, table, w) >> 16;
    float total = 0.f;
    for (int x = 0; x < c; ++x) total += w[x];
    for (int x = 0; x < c; ++x) out[x] = total > 0.f ? w[x] / total : __int_as_float(0x7fc00000);
}


// ------------------------------------------------- forward-sampling based estimators
// `BayesNet._forward_sample` (bayes_net.py:518-548) draws the variables in topological
// order; a variable named in `init` takes that value instead of being drawn, and the sample's
// "likelihood" is the product of P(value | parents) over ALL variables, i.e. the joint
// probability of the sample.
//   algo 1, likelihood weighting (bayes_net.py:621-663): samples with init = event; the
//           answer is, per joint query state, the MEAN likelihood of the samples that landed
//           there, normalised over the states (the reference's estimator, kept as is);
//   algo 2, rejection sampling (bayes_net.py:577-619): unconstrained samples; those that
//           contradict the event are dropped; the answer is the frequency of each query state
//           among the kept ones (NaN when none is kept: the reference returns an empty Series).
// One CTA per evidence row, its threads share the row's samples; per-state sums live in
// shared memory (atomics, low contention).
__global__ void __launch_bounds__(SBN_GIBBS_THREADS) sbn_forward_kernel(const __grid_constant__ SbnGibbs p, int algo) {
    extern __shared__ uint8_t s_raw[];
    const int T = SBN_GIBBS_THREADS;
    uint8_t *state = s_raw + threadIdx.x;                                             // [n_vars][T]
    uint8_t *evcode = s_raw + static_cast<size_t>(p.n_vars) * T;                      // [n_vars], 0xff = free
    float *acc_sum = reinterpret_cast<float *>(s_raw + ((static_cast<size_t>(p.n_vars) * (T + 1) + 15) / 16) * 16);  // [Q]
    uint32_t *acc_cnt = reinterpret_cast<uint32_t *>(acc_sum + p.Q);                  // [Q]
    const int64_t row = blockIdx.x;

    for (int v = threadIdx.x; v < p.n_vars; v += T) evcode[v] = 0xff;
    for (int q = threadIdx.x; q < p.Q; q += T) {
        acc_sum[q] = 0.f;
        acc_cnt[q] = 0;
    }
    __syncthreads();
    for (int k = threadIdx.x; k < p.n_ev; k += T) {
        const int v = p.ev_var[k];
        evcode[v] = static_cast<uint8_t>(min(static_cast<int>(p.ev[static_cast<int64_t>(k) * p.ld_ev + row]), p.card[v] - 1));
    }
    __syncthreads();

    for (int64_t it = threadIdx.x; it < p.n_iterations; it += T) {
        SbnRng rng;
        rng.init(p.seed, static_cast<uint64_t>(row) * static_cast<uint64_t>(p.n_iterations) + static_cast<uint64_t>(it));
        float lik = 1.f;
        bool keep = true;
        for (int v = 0; v < p.n_vars; ++v) {
            int base = p.cpt_off[v];
            for (int k = p.par_ptr[v]; k < p.par_ptr[v + 1]; ++k) base += state[p.par_idx[k] * T] * p.par_stride[k];
            const int c = p.card[v];
            int x;
            if (algo == 1 && evcode[v] != 0xff) {
                x = evcode[v];
            } else {
                const float u = rng.uniform();
                float acc = 0.f;
                x = c - 1;
                for (int j = 0; j < c; ++j) {
                    acc += __ldg(p.tables + base + j);
                    if (u <= acc) {
                        x = j;
                        break;
                    }
                }
                if (algo == 2 && evcode[v] != 0xff && x != evcode[v]) keep = false;
            }
            lik *= __ldg(p.tables + base + x);
            state[v * T] = static_cast<uint8_t>(x);
        }
        int qi = 0;
        for (int k = 0; k < p.n_query; ++k) qi = qi * p.card[p.query[k]] + state[p.query[k] * T];
        if (algo == 1) {
            atomicAdd(&acc_sum[qi], lik);
            atomicAdd(&acc_cnt[qi], 1u);
        } else if (keep) {
            atomicAdd(&acc_cnt[qi], 1u);
        }
    }
    __syncthreads();
    // normalise: likelihood -> per-state mean, then over the states; rejection -> frequency
    __shared__ float s_total;
    if (threadIdx.x == 0) {
        float total = 0.f;
        for (int q = 0; q < p.Q; ++q) {
            const float v = algo == 1 ? (acc_cnt[q] ? acc_sum[q] / static_cast<float>(acc_cnt[q]) : 0.f)
                                      : static_cast<float>(acc_cnt[q]);
            acc_sum[q] = v;
            total += v;
        }
        s_total = total;
    }
    __syncthreads();
    for (int q = threadIdx.x; q < p.Q; q += T)
        p.out[static_cast<int64_t>(q) * p.ld_out + row] = s_total > 0.f ? acc_sum[q] / s_total : __int_as_float(0x7fc00000);
}
