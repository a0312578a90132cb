// sorobn_b200 -- engine internals shared by the translation units of libsorobn_b200.so
// (sbn_api.cu: parsing, classic step launches, C ABI; sbn_chain.cu: the on-chip segment kernel).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>
#include <utility>
#include <vector>

#include "../../include/sorobn_b200.h"

struct EvAxis {
    int col, stride, card;
};
struct InDesc {
    bool is_slot;
    int id;
    bool batched;
    int sx;                      // stride of the eliminated axis when there is exactly one
    std::vector<EvAxis> ev;
    std::vector<int> estrides;   // stride per eliminated axis
    std::vector<int> strides;
};
struct StepDesc {
    int kind;
    int out_slot;
    int cx;                      // joint states of the eliminated variables (1 = product only)
    int64_t n_out;
    std::vector<int> cards;
    std::vector<int> ecards;     // cardinality per eliminated variable
    int64_t zoff_pos = -1;       // >= 0: int32 offset of the [n_in][cx] joint-state offset table
    int64_t zoff_tiled_pos = -1; // the same table with rows in the tiled kernel's input order
    std::vector<InDesc> in;
    // tiled fast path (sbn_step_tiled): tile edge, tile count, offset-table position
    int tile = 0;            // 0 = not eligible, use sbn_step_batched
    int nu = 0, na = 0, nb = 0, nc = 0;  // inputs without a tile axis / with axis 0 / axis 1 / both
    std::vector<int> order;      // kernel input slot -> index into `in` (U, then A, then B)
    int64_t n_tiles = 0;
    int64_t tile_off_pos = 0;  // int32 offset into sbn_program::d_tile_off
    // slab variant (expanding products): tiles grouped by the digits A and B share
    bool slab = false;
    bool big_tables = false;     // staged tables exceed SBN_SMEM_BUDGET: one CTA per SM (see smem_big)
    int slab_ma = 0, n_slab = 0;
    int64_t slab_off_pos = 0;
    int64_t slab_tile_off_pos = 0;  // tile table in slab order (rows of n_in + 5 words)
    int64_t tiles_per_super = 0, n_super = 0;
    // sliced staging (tables beyond SBN_SMEM_BUDGET): per chunk of `slice_tpc` tiles, per input,
    // (first float, floats, shared-memory offset) of the part of the table those tiles touch
    int64_t slice_pos = -1;
    int64_t slice_tpc = 0;
    int64_t slice_smem = 0;      // floats of shared memory of the largest chunk
    // readout of a marginals program (kind 2, sbn_marginal.cuh): first posterior row of the target's segment;
    // `in` is reordered so that the n_common inputs without the target axis come first
    int64_t q_offset = -1;
    int n_common = 0;
    // count step of a counts program (kind 3, sbn_count.cuh): q_offset is the family's first count-table entry,
    // `key` gathers the observed members, `cstrides` place the unobserved ones; [n_in][cs] / [cs] offset tables
    std::vector<EvAxis> key;
    std::vector<int> cstrides;
    int64_t span = 0;          // entries of the family's count table
    int64_t soff_pos = -1, coff_pos = -1;
    // sample step of a sample program (kind 4, sbn_sample.cuh): the `ecards` variables are drawn (not summed
    // out) into drawn-code rows q_offset ..; an input's `ev` terms may name drawn rows (col >= n_ev).
    // An argmax step of an MPE program (kind 5, sbn_mpe.cuh) has the same layout and decodes instead.
    // kind-0 / 1 step of a marginal MAP program: its eliminated variables are summed out by log-sum-exp (else maximised)
    bool logsumexp = false;
};
struct Slot {
    bool batched;
    int64_t size;     // floats per row (batched) or in total
    int64_t padded;   // size rounded up to 4 floats (bulk-TMA granularity)
    float *ptr;
};

inline int64_t round_up(int64_t v, int64_t m) { return (v + m - 1) / m * m; }

// Record the message sbn_last_error returns (printf format) and return `code`: the error convention of every
// entry point, for the translation units outside sbn_api.cu
int sbn_fail(int code, const char *fmt, ...);

struct SbnSegment;  // sbn_chain.h
struct SbnPair;     // sbn_pair.h

// What a program computes, fixed by its header version (4 .. 11 in this order)
enum ProgramKind {
    kPosterior,  // kind-0 / 1 steps, then the normalised posterior slot
    kMarginals,  // kind-2 readouts write the posterior, already normalised; no posterior slot
    kCounts,     // kind-3 steps add expected counts, post_slot holds P(observed)
    kSample,     // kind-4 steps draw codes, post_slot holds P(observed)
    kMpe,        // log tables, max-sum upward pass, kind-5 argmax steps decode into the drawn-code buffer with
                 // one draw, post_slot holds max log P(x, e)
    kMap,        // marginal MAP: an MPE program whose kind-0 / 1 steps each sum out (log-sum-exp) or maximise,
                 // post_slot holds max log P(x_MAP, e); it runs through the MPE entry point
    kGrad,       // gradient: a counts program whose kind-3 steps are weighted per row, plus kind-6 derivative
                 // readouts written to rows 1 .. of the output; row 0 and post_slot hold P(observed)
    kJoint,      // joint: a counts program whose steps are kind-7 per-row readouts of groups of variables into the
                 // output [Q][ld]; post_slot holds P(observed), the run's per-row P(observed) goes to d_total
};

// Programs on log tables (MPE and marginal MAP): float32 only, the log-domain step kernels only
inline bool sbn_log_domain(ProgramKind k) { return k == kMpe || k == kMap; }

// Every address and size a captured graph bakes in: it is replayed only for an equal key
struct GraphKey {
    const void *ev = nullptr;
    int64_t ld_ev = 0, n_rows = 0;
    const void *out = nullptr;
    int64_t ld_out = 0;
    const void *partial = nullptr;  // counts program: the per-warp partial tables
    const void *drawn = nullptr;    // sample / MPE program: the drawn-code buffer, its draws and pitch
    int64_t n_draws = 0, ld_drawn = 0;
    const void *lik = nullptr;      // soft-evidence program: the likelihoods the pack reads, and their pitch
    int64_t ld_lik = 0;
    const void *weight = nullptr;   // gradient program: the row weights of the count steps
    bool operator==(const GraphKey &o) const {
        return ev == o.ev && out == o.out && ld_ev == o.ld_ev && n_rows == o.n_rows && ld_out == o.ld_out &&
               partial == o.partial && drawn == o.drawn && n_draws == o.n_draws && ld_drawn == o.ld_drawn &&
               lik == o.lik && ld_lik == o.ld_lik && weight == o.weight;
    }
};
struct CachedGraph {
    cudaGraphExec_t exec = nullptr;
    GraphKey key;
    int64_t launches = 0;  // kernel launches one replay stands for (sbn_program::launches)
};

struct sbn_program {
    int device = 0;
    int n_sms = 1;     // multiprocessors of `device`: the grid-size heuristics count waves in them
    bool f64 = false;  // single-event programs computed and returned in double
    ProgramKind kind = kPosterior;
    int mode = 0, n_ev = 0, Q = 0, post_slot = 0, post_batched = 0;
    int64_t n_counts = 0;    // counts program: entries of the count table
    int64_t n_table_floats = 0;  // size of the table blob (sbn_program_set_tables replaces it in place)
    double *d_counts = nullptr;   // counts program: the run's count table [n_counts]
    int64_t partial_doubles = 0;  // counts / gradient program: doubles of the per-warp partial tables a call allocates
    int n_sampled = 0;            // sample / MPE program: drawn-code rows (one per unobserved variable)
    uint8_t *d_drawn = nullptr;   // sample program: drawn codes [n_sampled][n_draws][ld_drawn], then flags [ld_drawn]
    int64_t drawn_bytes = 0;
    uint32_t *d_sample_args = nullptr;  // seed lo, seed hi, row_base lo, row_base hi of the current chunk
    // soft evidence (any batched program, sbn_soft.cuh): (slot, card) of every likelihood, in
    // likelihood-column order; their pack descriptors; the staging buffer of host likelihoods [reserved][n_lik]
    // (double when f64) and sum log(max) [ld] of the last run
    std::vector<std::pair<int, int>> soft;
    int n_lik = 0;
    int32_t *d_soft = nullptr;
    void *d_lik = nullptr;
    double *d_log_max = nullptr;
    // gradient program: per step, whether P(observed) depends on it (the steps a forward run issues); the staging
    // buffer of host weights [reserved]; the forward run's own graph
    std::vector<char> forward;
    double *d_weight = nullptr;
    CachedGraph forward_graph;
    std::vector<std::pair<int64_t, int64_t>> tables;  // (offset, size) in floats
    std::vector<int64_t> table_padded;
    float *d_tables = nullptr;
    std::vector<Slot> slots;
    std::vector<StepDesc> steps;

    int64_t reserved_rows = 0;  // chunk capacity
    int64_t ld = 0;             // row pitch of batched scratch (floats)
    float *d_arena = nullptr;   // batched scratch
    float *d_shared = nullptr;  // unbatched scratch
    int32_t *d_tile_off = nullptr;  // per-step tile offset tables of the tiled kernel
    float *d_total = nullptr;   // per-row normaliser = P(event) of the last run [ld] (double when f64)
    uint8_t *d_ev = nullptr;    // staging for run_host  [n_ev][ld]
    float *d_out = nullptr;     //                         [Q][ld]   (double when f64)
    cudaStream_t stream = nullptr;
    // Branch streams for graph capture: the steps form a tree (every intermediate is consumed
    // once), so independent sub-trees are captured on different streams and become parallel
    // branches of the CUDA graph.
    static constexpr int kBranches = 4;
    cudaStream_t branch[kBranches] = {nullptr, nullptr, nullptr, nullptr};
    std::vector<cudaEvent_t> step_done;  // one event per step (+ normalise), capture-only
    std::vector<cudaEvent_t> pipe_events;  // run_host pipelining: fork, (upload done, kernels done) per column range, joins
    bool use_branches = false;  // measured: no gain on the grid plan (one long chain); opt-in

    bool use_graph = true;
    bool use_tiled = true;
    bool use_slab = true;
    bool use_preload = true;  // tiled kernel: operand preload schedule where instantiated (else the x-loop)
    CachedGraph graph;       // one run of rows on the device
    CachedGraph pipe_graph;  // the pipelined host run (pinned host buffers)

    int64_t launches = 0;
    int64_t setup_launches = 0;  // evidence-independent launches issued once at creation

    // on-chip segments (sbn_chain.h): runs of batched steps executed by one persistent kernel
    std::vector<SbnSegment *> segments;
    std::vector<int> seg_first;      // per step: >= 0 = head of that segment, -2 = inside one, -1 = classic launch
    float *d_chain_scratch = nullptr;
    bool use_chain = true;
    bool use_tma = true;             // tensor-map TMA pipeline kernel for the steps it covers (sbn_tma.h)
    bool chain_fits = true;          // false when a slot-arena operand of a segment needs > 32-bit byte offsets
    std::vector<int32_t> h_tile_words;  // host copy of d_tile_off

    // paired steps (sbn_pair.h): a step and its consumer as one launch, the intermediate in registers
    std::vector<SbnPair *> pairs;
    std::vector<int> pair_first;     // per step: >= 0 = first step of that pair, -2 = its second step, -1 = on its own
    float *d_pair_canon = nullptr;   // canonical coefficient arrays of all pairs
    int32_t *d_pair_tiles = nullptr; // their tile tables
    bool use_pair = true;
    bool pairs_avoid_segments = false;  // planned with the on-chip segments switched on: no pair touches a segment's step
};

