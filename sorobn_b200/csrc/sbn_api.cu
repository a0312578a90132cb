// sorobn_b200 -- C-ABI engine: program parsing, scratch management, launches.
//
// Host-side counterpart of `BayesNet._variable_elimination`
// (/root/reference/sorobn/bayes_net.py:739-794): the reference walks the hidden
// variables in Python and calls pandas for every product / sum-out; here the walk was
// frozen by sorobn_b200/planner.py into a list of steps and this file replays it as
// kernel launches (optionally captured in a CUDA graph) for a batch of evidence rows.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "sbn_chain.h"
#include "sbn_count.cuh"
#include "sbn_deriv.cuh"
#include "sbn_gibbs.cuh"
#include "sbn_internal.h"
#include "sbn_join.h"
#include "sbn_kernels.cuh"
#include "sbn_launch.h"
#include "sbn_marginal.cuh"
#include "sbn_mpe.cuh"
#include "sbn_pair.h"
#include "sbn_sample.cuh"
#include "sbn_soft.cuh"
#include "sbn_tma.h"

namespace {

thread_local std::string g_err;

void set_error(const char *fmt, va_list ap) {
    char buf[512];
    vsnprintf(buf, sizeof buf, fmt, ap);
    g_err = buf;
}

int fail(int code, const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    set_error(fmt, ap);
    va_end(ap);
    return code;
}

#define SBN_CUDA(call)                                                                              \
    do {                                                                                            \
        cudaError_t e_ = (call);                                                                    \
        if (e_ != cudaSuccess)                                                                      \
            return fail(SBN_E_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, \
                        __LINE__);                                                                  \
    } while (0)

constexpr int32_t kMagic = 0x53424E31;
constexpr int kVersion = 4;
constexpr int kVersionMarginals = 5;  // planner.build_marginals_plan: kind-2 readouts, no posterior slot
constexpr int kVersionCounts = 6;     // planner.build_counts_plan: kind-3 count steps, P(observed) in the posterior slot
constexpr int kVersionSample = 7;     // planner.build_sample_plan: kind-4 sample steps, P(observed) in the posterior slot
constexpr int kVersionMpe = 8;        // planner.build_mpe_plan: log tables, max-sum steps, kind-5 argmax steps,
                                      // max log P(x, e) in the posterior slot
constexpr int kVersionMap = 9;        // planner.build_map_plan: version 8 plus a reduction word on kind-0 / 1 steps
                                      // (1 = log-sum-exp, 0 = max), max log P(x_MAP, e) in the posterior slot
constexpr int kVersionGrad = 10;      // planner.build_pattern_plan(kind "grad"): version 6 with weighted count steps plus
                                      // kind-6 derivative readouts, P(observed) in the posterior slot
static_assert(kVersionMpe - kVersion == kMpe, "one program kind per header version, in order");
static_assert(kVersionMap - kVersion == kMap, "one program kind per header version, in order");
constexpr int kVersionJoint = 11;     // planner.build_joint_plan: version 6 with kind-7 per-row joint readouts in place of
                                      // the count steps, P(observed) in the posterior slot
static_assert(kVersionGrad - kVersion == kGrad, "one program kind per header version, in order");
static_assert(kVersionJoint - kVersion == kJoint, "one program kind per header version, in order");
constexpr int64_t kMarginalZoffMax = 1 << 24;  // int32 words of one readout's joint-state offset table
constexpr int kMaxElim = 3;
constexpr int kMaxZ = 256;
constexpr int kHeaderWords = 12;

}  // namespace

int sbn_fail(int code, const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    set_error(fmt, ap);
    va_end(ap);
    return code;
}

namespace {

int parse(sbn_program *P, const int32_t *w, int64_t n) {
    if (n < kHeaderWords) return fail(SBN_E_INVALID, "program shorter than its header");
    if (w[0] != kMagic) return fail(SBN_E_INVALID, "bad program magic 0x%x", w[0]);
    if (w[1] < kVersion || w[1] > kVersionJoint)
        return fail(SBN_E_INVALID, "program version %d, engine expects %d, %d, %d, %d, %d, %d, %d or %d", w[1], kVersion,
                    kVersionMarginals, kVersionCounts, kVersionSample, kVersionMpe, kVersionMap, kVersionGrad, kVersionJoint);
    P->kind = static_cast<ProgramKind>(w[1] - kVersion);
    // a gradient program parses as a counts program plus its derivative readouts (kind 6)
    const bool grad = P->kind == kGrad;
    const bool marginals = P->kind == kMarginals, counts = P->kind == kCounts || grad, mpe = sbn_log_domain(P->kind);
    const bool map = P->kind == kMap;
    // a joint program: the counts program's passes with kind-7 readouts in place of the count steps
    const bool joint = P->kind == kJoint;
    // sample, MPE and marginal MAP programs share the words of their last steps
    const bool decodes = P->kind == kSample || mpe;
    P->mode = w[2];
    P->n_ev = w[3];
    const int n_tables = w[4], n_slots = w[5], n_steps = w[6];
    P->Q = w[7];
    P->post_slot = w[8];
    P->post_batched = w[9];
    if (P->mode != 0 && P->mode != 1) return fail(SBN_E_INVALID, "bad mode %d", P->mode);
    if (P->n_ev < 0 || n_tables < 0 || n_slots <= 0 || n_steps <= 0 || P->Q <= 0)
        return fail(SBN_E_INVALID, "bad header counts");
    if (counts) {
        P->n_counts = w[10];
        if ((!grad && P->Q != 1) || P->n_counts <= 0 || P->mode != (grad ? 1 : P->mode))
            return fail(SBN_E_INVALID, grad ? "bad gradient header" : "bad counts header");
    }
    if (joint && (w[10] != 0 || P->mode != 1)) return fail(SBN_E_INVALID, "bad joint header");
    if (decodes) {
        P->n_sampled = w[10];
        if (P->Q != 1 || P->mode != 1 || P->n_sampled < 0)
            return fail(SBN_E_INVALID, map ? "bad MAP header" : mpe ? "bad MPE header" : "bad sample header");
    }
    // sample program: kind-4 steps draw codes; MPE / MAP program: kind-5 steps decode them (same words)
    const int decode_kind = mpe ? 5 : 4;
    int n_drawn = 0;  // sample / MPE program: drawn-code rows written by the sample / argmax steps so far
    if (marginals ? (P->post_slot != -1 || P->post_batched != 0) : (P->post_slot < 0 || P->post_slot >= n_slots))
        return fail(SBN_E_INVALID, "post slot out of range");
    int64_t p = kHeaderWords;
    auto need = [&](int64_t k) { return p + k <= n; };
    if (!need(2LL * n_tables + 2LL * n_slots)) return fail(SBN_E_INVALID, "truncated table/slot section");
    for (int t = 0; t < n_tables; ++t) {
        const int64_t off = w[p], size = w[p + 1];
        p += 2;
        if (off < 0 || size <= 0 || (off % 4) != 0) return fail(SBN_E_INVALID, "bad table %d", t);
        P->tables.push_back({off, size});
        P->table_padded.push_back(round_up(size, 4));
    }
    for (int s = 0; s < n_slots; ++s) {
        const int batched = w[p];
        const int64_t size = w[p + 1];
        p += 2;
        if ((batched != 0 && batched != 1) || size <= 0) return fail(SBN_E_INVALID, "bad slot %d", s);
        if (batched && P->mode == 0) return fail(SBN_E_INVALID, "batched slot in a flat program");
        P->slots.push_back({batched != 0, size, round_up(size, 4), nullptr});
    }
    // (a gradient program's slot holds P(observed); its other output rows are written by the readouts)
    if (!marginals && ((P->slots[P->post_slot].batched ? 1 : 0) != P->post_batched || P->slots[P->post_slot].size < (grad || joint ? 1 : P->Q)))
        return fail(SBN_E_INVALID, "posterior slot mismatch");
    {
        // soft evidence: (slot, card) of every likelihood, filled before step 0 (sbn_soft.cuh); n_soft is word 10
        // of versions 4 and 5, word 11 of the others (their word 10 holds n_counts / n_sampled)
        const int n_soft = P->kind == kPosterior || marginals ? w[10] : w[11];
        if (n_soft < 0 || (n_soft > 0 && P->mode != 1) || !need(2LL * n_soft))
            return fail(SBN_E_INVALID, "bad soft-evidence section");
        for (int v = 0; v < n_soft; ++v) {
            const int slot = w[p], card = w[p + 1];
            p += 2;
            if (slot < 0 || slot >= n_slots || !P->slots[slot].batched || card < 1 || P->slots[slot].size < card)
                return fail(SBN_E_INVALID, "bad likelihood %d", v);
            for (const auto &o : P->soft)
                if (o.first == slot) return fail(SBN_E_INVALID, "two likelihoods share slot %d", slot);
            P->soft.push_back({slot, card});
            P->n_lik += card;
        }
    }
    if (grad && P->Q != 1 + P->n_lik) return fail(SBN_E_INVALID, "a gradient program writes 1 + %d rows, not %d", P->n_lik, P->Q);
    std::vector<int> written(marginals || grad || joint ? P->Q : 0, 0);  // posterior entries (gradient: output rows) written by the readouts
    for (int s = 0; s < n_steps; ++s) {
        if (!need(5)) return fail(SBN_E_INVALID, "truncated step %d", s);
        StepDesc st;
        st.kind = w[p];
        const int n_in = w[p + 1];
        st.out_slot = w[p + 2];
        const int n_axes = w[p + 3];
        const int n_elim = w[p + 4];
        st.cx = 1;
        p += 5;
        const bool readout = st.kind == 2 || (grad && st.kind == 6);  // kind 6: the layout of kind 2
        const bool count = st.kind == 3;
        const bool draw = decodes && st.kind == decode_kind;
        const bool jread = joint && st.kind == 7;  // the layout of kind 2, any number of output axes
        if (st.kind != 0 && st.kind != 1 && !(readout && (marginals || grad)) && !(count && counts) && !draw && !jread)
            return fail(SBN_E_INVALID, "step %d: bad kind", s);
        if (draw) {
            // the drawn variables are the step's `n_elim` axes; they fill the next drawn-code rows
            if (!need(1)) return fail(SBN_E_INVALID, "truncated step %d", s);
            st.q_offset = w[p++];
            if (st.out_slot != -1 || n_axes != 0 || n_elim < 1 || n_elim > SBN_SAMPLE_MAX_X || st.q_offset != n_drawn ||
                n_drawn + n_elim > P->n_sampled)
                return fail(SBN_E_INVALID, mpe ? "step %d: bad argmax step" : "step %d: bad sample step", s);
        }
        if (map && (st.kind == 0 || st.kind == 1)) {
            // the reduction of the eliminated variables: 1 = log-sum-exp, 0 = max (and every product-only step)
            if (!need(1)) return fail(SBN_E_INVALID, "truncated step %d", s);
            const int reduce = w[p++];
            if (reduce != 0 && reduce != 1) return fail(SBN_E_INVALID, "step %d: bad reduction %d", s, reduce);
            st.logsumexp = reduce == 1;
        }
        if (count) {
            // c_offset, the observed members' gathers and the count-table strides of the output axes
            if (!need(2)) return fail(SBN_E_INVALID, "truncated step %d", s);
            st.q_offset = w[p];
            const int n_key = w[p + 1];
            p += 2;
            if (st.out_slot != -1 || n_axes < 0 || n_axes > SBN_MAX_AXES || n_elim < 0 || n_elim > 64 || n_key < 0 ||
                n_key > SBN_MAX_EV || (n_in == 0 && (n_axes != 0 || n_elim != 0)))
                return fail(SBN_E_INVALID, "step %d: bad count step", s);
            if (!need(3LL * n_key + n_axes)) return fail(SBN_E_INVALID, "truncated step %d", s);
            int64_t span = 1;
            for (int k = 0; k < n_key; ++k) {
                EvAxis a{w[p], w[p + 1], w[p + 2]};
                p += 3;
                if (a.col < 0 || a.col >= P->n_ev || a.stride < 0 || a.card < 1 || a.card > 256)
                    return fail(SBN_E_INVALID, "step %d: bad key axis", s);
                span += static_cast<int64_t>(a.card - 1) * a.stride;
                st.key.push_back(a);
            }
            for (int j = 0; j < n_axes; ++j) {
                if (w[p + j] < 0) return fail(SBN_E_INVALID, "step %d: negative count stride", s);
                st.cstrides.push_back(w[p + j]);
            }
            p += n_axes;
            if (!need(n_axes)) return fail(SBN_E_INVALID, "truncated step %d", s);
            for (int j = 0; j < n_axes; ++j) {
                if (w[p + j] < 1) return fail(SBN_E_INVALID, "step %d: axis card %d", s, w[p + j]);
                span += static_cast<int64_t>(w[p + j] - 1) * st.cstrides[j];
            }
            if (st.q_offset < 0 || span >= (1LL << 31) || st.q_offset + span > P->n_counts)
                return fail(SBN_E_INVALID, "step %d: count-table entries outside the table", s);
            st.span = span;
        }
        if (jread) {
            // the group's unobserved members are the output axes, written at output rows q_offset .. q_offset + n_out - 1
            if (!need(1)) return fail(SBN_E_INVALID, "truncated step %d", s);
            st.q_offset = w[p++];
            if (st.out_slot != -1 || n_axes < 1 || n_axes > SBN_MAX_AXES || n_elim < 0 || n_elim > 64 || n_in < 1)
                return fail(SBN_E_INVALID, "step %d: bad joint readout", s);
        }
        if (readout) {
            // one output axis (the target), written at posterior rows q_offset .. q_offset + card - 1
            if (!need(1)) return fail(SBN_E_INVALID, "truncated step %d", s);
            st.q_offset = w[p++];
            if (st.out_slot != -1 || n_axes != 1 || n_elim < 0 || n_elim > 64)
                return fail(SBN_E_INVALID, "step %d: bad readout step", s);
        }
        if (st.kind == 1 && P->mode == 0) return fail(SBN_E_INVALID, "step %d: batched step in a flat program", s);
        if (n_in < (count ? 0 : 1) || n_in > SBN_MAX_IN) return fail(SBN_E_INVALID, "step %d: %d inputs", s, n_in);
        if (n_axes < 0 || n_axes > SBN_MAX_AXES) return fail(SBN_E_INVALID, "step %d: %d axes", s, n_axes);
        const bool writes_slot = !readout && !count && !draw && !jread;
        if (writes_slot && (n_elim < 0 || n_elim > kMaxElim)) return fail(SBN_E_INVALID, "step %d: %d eliminated axes", s, n_elim);
        if (writes_slot && (st.out_slot < 0 || st.out_slot >= n_slots)) return fail(SBN_E_INVALID, "step %d: out slot", s);
        if (!need(n_axes + n_elim)) return fail(SBN_E_INVALID, "truncated step %d", s);
        st.n_out = 1;
        for (int j = 0; j < n_axes; ++j) {
            const int c = w[p + j];
            if (c < 1) return fail(SBN_E_INVALID, "step %d: axis card %d", s, c);
            st.n_out *= c;
            if (st.n_out >= (1LL << 31) || ((count || jread) && st.n_out > kMarginalZoffMax / SBN_MAX_IN))
                return fail(SBN_E_INVALID, "step %d: output too large", s);
            st.cards.push_back(c);
        }
        p += n_axes;
        for (int k = 0; k < n_elim; ++k) {
            const int c = w[p + k];
            if (c < 1 || (draw && c > 256)) return fail(SBN_E_INVALID, "step %d: eliminated card %d", s, c);
            if (static_cast<int64_t>(st.cx) * c > (readout || count || jread ? kMarginalZoffMax / SBN_MAX_IN : kMaxZ))
                return fail(SBN_E_INVALID, "step %d: too many eliminated states", s);
            st.cx *= c;
            st.ecards.push_back(c);
        }
        p += n_elim;
        if (readout) {
            if (st.q_offset < (grad ? 1 : 0) || st.q_offset + st.n_out > P->Q)
                return fail(SBN_E_INVALID, "step %d: segment outside the posterior", s);
            for (int64_t q = st.q_offset; q < st.q_offset + st.n_out; ++q) written[q]++;
        } else if (count) {
            if (static_cast<int64_t>(st.cx) * st.n_out >= (1LL << 31)) return fail(SBN_E_INVALID, "step %d: count step too large", s);
        } else if (jread) {
            if (static_cast<int64_t>(st.cx) * st.n_out >= (1LL << 31)) return fail(SBN_E_INVALID, "step %d: joint readout too large", s);
            if (st.q_offset < 0 || st.q_offset + st.n_out > P->Q) return fail(SBN_E_INVALID, "step %d: rows outside the output", s);
            for (int64_t q = st.q_offset; q < st.q_offset + st.n_out; ++q) written[q]++;
        } else if (!draw) {
            const Slot &os = P->slots[st.out_slot];
            if (os.batched != (st.kind == 1)) return fail(SBN_E_INVALID, "step %d: out slot kind mismatch", s);
            if (os.size < st.n_out) return fail(SBN_E_INVALID, "step %d: out slot too small", s);
        }
        const bool per_row = st.kind == 1 || ((readout || count || draw || jread) && P->mode == 1);  // batched operands allowed
        for (int i = 0; i < n_in; ++i) {
            if (!need(4)) return fail(SBN_E_INVALID, "truncated step %d input %d", s, i);
            InDesc in;
            in.is_slot = w[p] != 0;
            in.id = w[p + 1];
            in.batched = w[p + 2] != 0;
            in.sx = 0;
            const int n_ev = w[p + 3];
            p += 4;
            if (n_ev < 0 || n_ev > (draw ? SBN_SAMPLE_MAX_TERMS : SBN_MAX_EV))
                return fail(SBN_E_INVALID, "step %d input %d: %d ev axes", s, i, n_ev);
            if (!need(3LL * n_ev + n_elim + n_axes)) return fail(SBN_E_INVALID, "truncated step %d input %d", s, i);
            int64_t size;
            if (in.is_slot) {
                if (in.id < 0 || in.id >= n_slots) return fail(SBN_E_INVALID, "step %d input %d: slot id", s, i);
                if (in.id == st.out_slot) return fail(SBN_E_INVALID, "step %d: output aliases input %d", s, i);
                if (P->slots[in.id].batched != in.batched)
                    return fail(SBN_E_INVALID, "step %d input %d: batched flag mismatch", s, i);
                size = P->slots[in.id].size;
            } else {
                if (in.id < 0 || in.id >= n_tables) return fail(SBN_E_INVALID, "step %d input %d: table id", s, i);
                if (in.batched) return fail(SBN_E_INVALID, "step %d input %d: batched table", s, i);
                size = P->tables[in.id].second;
            }
            if (in.batched && !per_row) return fail(SBN_E_INVALID, "step %d: batched input in flat step", s);
            if (in.batched && n_ev && !draw) return fail(SBN_E_INVALID, "step %d input %d: batched input with ev axes", s, i);
            if (n_ev && !per_row && P->mode != 0)
                return fail(SBN_E_INVALID, "step %d input %d: evidence axes in an unbatched step", s, i);
            int64_t max_off = 0;
            for (int k = 0; k < n_ev; ++k) {
                EvAxis a{w[p], w[p + 1], w[p + 2]};
                p += 3;
                // a sample step also gathers the codes drawn by the steps before it (col >= n_ev); a batched
                // operand only those: its observed columns are part of its rows already
                const int n_cols = draw ? P->n_ev + n_drawn : P->n_ev;
                if (a.col < 0 || a.col >= n_cols || (in.batched && a.col < P->n_ev) || a.stride < 0 || a.card < 1 || a.card > 256)
                    return fail(SBN_E_INVALID, "step %d input %d: bad ev axis", s, i);
                max_off += static_cast<int64_t>(a.card - 1) * a.stride;
                in.ev.push_back(a);
            }
            for (int k = 0; k < n_elim; ++k) {
                const int sk = w[p + k];
                if (sk < 0) return fail(SBN_E_INVALID, "step %d input %d: negative stride", s, i);
                max_off += static_cast<int64_t>(st.ecards[k] - 1) * sk;
                in.estrides.push_back(sk);
            }
            p += n_elim;
            if (n_elim >= 1) in.sx = in.estrides[0];  // zoff enumerates joint states with this variable fastest
            for (int j = 0; j < n_axes; ++j) {
                const int sj = w[p + j];
                if (sj < 0) return fail(SBN_E_INVALID, "step %d input %d: negative stride", s, i);
                max_off += static_cast<int64_t>(st.cards[j] - 1) * sj;
                in.strides.push_back(sj);
            }
            p += n_axes;
            if (max_off >= size) return fail(SBN_E_INVALID, "step %d input %d: reads past its buffer", s, i);
            st.in.push_back(std::move(in));
        }
        if (count || jread) {  // inputs without any family (group) axis first: loaded once per joint state z
            auto no_axis = [](const InDesc &in) { return std::all_of(in.strides.begin(), in.strides.end(), [](int v) { return v == 0; }); };
            std::stable_partition(st.in.begin(), st.in.end(), no_axis);
            st.n_common = static_cast<int>(std::count_if(st.in.begin(), st.in.end(), no_axis));
        }
        if (draw) n_drawn += n_elim;  // at most kMaxZ joint states: checked with the eliminated cards
        if (readout) {
            std::stable_partition(st.in.begin(), st.in.end(), [](const InDesc &in) { return in.strides[0] == 0; });
            st.n_common = static_cast<int>(std::count_if(st.in.begin(), st.in.end(), [](const InDesc &in) { return in.strides[0] == 0; }));
        }
        P->steps.push_back(std::move(st));
    }
    if (p != n) return fail(SBN_E_INVALID, "trailing words in program");
    if (P->mode == 1) {
        // evidence-independent tables are computed once per program (run_table_steps): their slots
        // must not be recycled (planner: _assign_slots keep_unbatched)
        std::vector<int> writes(P->slots.size(), 0);
        for (const StepDesc &st : P->steps)
            if (st.kind == 0 && ++writes[st.out_slot] > 1)
                return fail(SBN_E_INVALID, "unbatched slot %d is written twice in a batched program", st.out_slot);
    }
    if (decodes) {
        // every drawn-code row is written; the sample / argmax steps run last, after the last write of the
        // posterior slot (P(observed), or max log P(x, e))
        if (n_drawn != P->n_sampled) return fail(SBN_E_INVALID, "%d of %d drawn-code rows are written", n_drawn, P->n_sampled);
        int writer = -1, first = static_cast<int>(P->steps.size());
        for (size_t i = 0; i < P->steps.size(); ++i) {
            if (P->steps[i].kind == decode_kind) {
                if (first > static_cast<int>(i)) first = static_cast<int>(i);
            } else {
                if (first < static_cast<int>(i)) return fail(SBN_E_INVALID, "step %zu comes after a sample step", i);
                if (P->steps[i].out_slot == P->post_slot) writer = static_cast<int>(i);
            }
        }
        if (writer < 0) return fail(SBN_E_INVALID, "P(observed) is not written before the sample steps");
    } else if (marginals) {
        for (int q = 0; q < P->Q; ++q)
            if (written[q] != 1) return fail(SBN_E_INVALID, "posterior entry %d is written %d times", q, written[q]);
    } else if (counts || joint) {
        // P(observed) is written before the first count step and not overwritten before the last one (the last
        // derivative readout of a gradient program; the last joint readout)
        int first = -1, last = -1, writer = -1;
        for (size_t i = 0; i < P->steps.size(); ++i) {
            if (P->steps[i].kind >= 2) {
                if (first < 0) first = static_cast<int>(i);
                last = static_cast<int>(i);
            } else if (P->steps[i].out_slot == P->post_slot) {
                writer = static_cast<int>(i);
            }
        }
        if (first < 0) return fail(SBN_E_INVALID, joint ? "a joint program without a readout" : "a counts program without a count step");
        if (joint)
            for (int q = 0; q < P->Q; ++q)
                if (written[q] != 1) return fail(SBN_E_INVALID, "output row %d is written %d times", q, written[q]);
        if (writer < 0 || writer > first) return fail(SBN_E_INVALID, "P(observed) is not written before the count steps");
        for (int i = first; i <= last; ++i)
            if (P->steps[i].kind < 2) return fail(SBN_E_INVALID, "step %d comes between the count steps", i);
        if (grad) {
            for (int q = 1; q < P->Q; ++q)
                if (written[q] != 1) return fail(SBN_E_INVALID, "output row %d is written %d times", q, written[q]);
            // the forward run: the steps P(observed) depends on, through the last writer of every slot it reads
            std::vector<int> last_writer(P->slots.size(), -1);
            std::vector<std::vector<int>> deps(P->steps.size());
            for (int i = 0; i < writer + 1; ++i) {
                for (const InDesc &in : P->steps[i].in)
                    if (in.is_slot && last_writer[in.id] >= 0) deps[i].push_back(last_writer[in.id]);
                last_writer[P->steps[i].out_slot] = i;
            }
            P->forward.assign(P->steps.size(), 0);
            std::vector<int> stack = {writer};
            while (!stack.empty()) {
                const int i = stack.back();
                stack.pop_back();
                if (P->forward[i]) continue;
                P->forward[i] = 1;
                for (int d : deps[i]) stack.push_back(d);
            }
        }
    } else if (P->steps.back().out_slot != P->post_slot) {
        return fail(SBN_E_INVALID, "last step does not write the posterior");
    }
    for (const auto &sv : P->soft) {
        // a likelihood slot holds the pack's values from before step 0: its first access is a read (a later step
        // may reuse the slot once the likelihood's readers are done)
        for (const StepDesc &st : P->steps) {
            bool read = false;
            for (const InDesc &in : st.in) read |= in.is_slot && in.id == sv.first;
            if (read) break;
            if (st.kind <= 1 && st.out_slot == sv.first)
                return fail(SBN_E_INVALID, "likelihood slot %d is written before it is read", sv.first);
        }
    }
    return SBN_OK;
}

constexpr int kTiledMaxIn = 4;
constexpr int64_t kTileTableMax = 1 << 23;  // int32 words per step

// Tables staged per CTA: SBN_SMEM_BUDGET keeps several CTAs per SM.  Opt-in experiment
// (SOROBN_B200_SMEM_BIG=<KB>, up to 200): a launch around a larger CPT (8^5 entries = 128 KB) stages
// it with ONE CTA per SM walking every tile of its rows.  4 warps per SM are latency-bound on the
// shared-memory gathers, so the default leaves such tables to the L1/L2 gathers of the plain kernel.
int64_t smem_big() {
    static const int64_t v = [] {
        const char *e = getenv("SOROBN_B200_SMEM_BIG");
        const int64_t kb = e ? atoll(e) : SBN_SMEM_BUDGET / 1024;
        return std::max<int64_t>(SBN_SMEM_BUDGET, std::min<int64_t>(kb * 1024, SBN_SMEM_BIG));
    }();
    return v;
}

// Slab variant of the tiled kernel: eligible when the launch multiplies one batched factor on
// the A side with one on the B side (plus at most one table without tile axes), both with
// private axes beyond the tile.  Emits the tile table in slab order (shared digits, then the
// B-private digits and B blocks, then the A-private digits and A blocks) and the slab's entry
// offsets.  Returns false when the step does not qualify (the caller then emits the plain
// tile table).
// Sliced staging.  The planner ships a CPT that is too big for shared memory with the output
// axes >= 2 outermost (planner.py `_relayout_big_tables`), so the tiles of one chunk touch a
// contiguous part of it.  Find the largest chunk whose parts fit SBN_SMEM_BUDGET and record, per
// chunk and input, which floats to stage and where.
int64_t slice_budget() {
    static const int64_t v = [] {
        const char *e = getenv("SOROBN_B200_SLICE_KB");
        // 32 KB: more CTAs per SM than 64 KB, while a launch with two 128 KB CPTs still fits
        // (at 16 KB it would leave the tiled kernel)
        const int64_t kb = e ? atoll(e) : 32;
        return std::max<int64_t>(1024, std::min<int64_t>(kb * 1024, SBN_SMEM_BUDGET));
    }();
    return v;
}
bool plan_slices(sbn_program *P, StepDesc &st, int T, std::vector<int32_t> *words) {
    const int n_in = static_cast<int>(st.in.size());
    const int n_axes = static_cast<int>(st.cards.size());
    const int row_words = n_in + 2;
    std::vector<int64_t> span(n_in, 0), size(n_in, 0);
    for (int i = 0; i < n_in; ++i) {
        const InDesc &in = st.in[st.order[i]];
        if (in.batched) continue;
        size[i] = in.is_slot ? P->slots[in.id].padded : P->table_padded[in.id];
        int64_t sp = 0;
        for (size_t k = 0; k < st.ecards.size(); ++k) sp += static_cast<int64_t>(st.ecards[k] - 1) * in.estrides[k];
        if (n_axes > 0) sp += static_cast<int64_t>(std::min(T, st.cards[0]) - 1) * in.strides[0];
        if (n_axes > 1) sp += static_cast<int64_t>(std::min(T, st.cards[1]) - 1) * in.strides[1];
        for (const EvAxis &a : in.ev) sp += static_cast<int64_t>(a.card - 1) * a.stride;
        span[i] = sp;
    }
    for (int64_t tpc = st.n_tiles; tpc >= 1; tpc = (tpc == 1 ? 0 : (tpc + 1) / 2)) {
        const int64_t chunks = (st.n_tiles + tpc - 1) / tpc;
        std::vector<int32_t> rec;
        rec.reserve(static_cast<size_t>(chunks) * n_in * 3);
        int64_t worst = 0;
        for (int64_t c = 0; c < chunks; ++c) {
            int64_t smem = 0;
            for (int i = 0; i < n_in; ++i) {
                if (st.in[st.order[i]].batched) {
                    rec.insert(rec.end(), {0, 0, -1});
                    continue;
                }
                int64_t lo = INT64_MAX, hi = 0;
                for (int64_t t = c * tpc; t < std::min(st.n_tiles, (c + 1) * tpc); ++t) {
                    const int64_t base = (*words)[static_cast<size_t>(st.tile_off_pos + t * row_words + 2 + i)];
                    lo = std::min(lo, base);
                    hi = std::max(hi, base + span[i] + 1);
                }
                lo = lo / 4 * 4;
                const int64_t len = std::min(round_up(hi - lo, 4), size[i] - lo);
                rec.insert(rec.end(), {static_cast<int32_t>(lo), static_cast<int32_t>(len), static_cast<int32_t>(smem)});
                smem += len;
            }
            worst = std::max(worst, smem);
        }
        if (worst * 4 <= slice_budget()) {
            st.slice_pos = static_cast<int64_t>(words->size());
            words->insert(words->end(), rec.begin(), rec.end());
            st.slice_tpc = tpc;
            st.slice_smem = worst;
            return true;
        }
    }
    return false;
}

bool plan_slab(sbn_program *P, StepDesc &st, int T, std::vector<int32_t> *words) {
    (void)P;
    const int n_axes = static_cast<int>(st.cards.size());
    const int n_in = static_cast<int>(st.in.size());
    if (st.nc != 0 || st.na != 1 || st.nb != 1 || st.nu > 1 || n_in > 3 || n_axes < 3) return false;
    if (st.ecards.size() != 1) return false;
    if (!(st.cx == T || (T == 4 && st.cx == 8))) return false;  // needs the preload schedule
    const InDesc &A = st.in[st.order[st.nu]], &B = st.in[st.order[st.nu + 1]];
    if (!A.batched || !B.batched) return false;
    const int c0 = st.cards[0], c1 = st.cards[1];
    std::vector<int> pa, pb, sh;  // axes >= 2: private to A, private to B, shared
    int64_t n_pa = 1, n_pb = 1, n_sh = 1;
    for (int j = 2; j < n_axes; ++j) {
        const bool ha = A.strides[j] != 0, hb = B.strides[j] != 0;
        if (ha && !hb) { pa.push_back(j); n_pa *= st.cards[j]; }
        else if (hb && !ha) { pb.push_back(j); n_pb *= st.cards[j]; }
        else { sh.push_back(j); n_sh *= st.cards[j]; }
    }
    if (n_pa == 1 || n_pb == 1) return false;  // nothing is re-read: the plain tile walk is optimal
    // small operands are re-read from L2 anyway (measured: B125 x B125 is faster without the slab)
    if (static_cast<int64_t>(c0) * n_pa * st.cx < 512 || static_cast<int64_t>(c1) * n_pb * st.cx < 512) return false;
    const int64_t ma = static_cast<int64_t>(c0) * n_pa;
    const int64_t n_slab = ma * st.cx;
    if (n_slab * kSlabThreads * kRowsPerThread * 4 > kSlabSmemMax) return false;
    const int n_ta = (c0 + T - 1) / T, n_tb = (c1 + T - 1) / T;
    const int64_t tiles_per_super = n_pb * n_tb * n_pa * n_ta;
    if (n_sh * tiles_per_super * (n_in + 5) > kTileTableMax) return false;

    st.slab = true;
    st.slab_ma = static_cast<int>(ma);
    st.n_slab = static_cast<int>(n_slab);
    st.n_super = n_sh;
    st.tiles_per_super = tiles_per_super;
    // slab entry k = x * ma + (d0 + c0 * pa_index)  ->  element offset inside A (shared digits 0)
    st.slab_off_pos = static_cast<int64_t>(words->size());
    for (int x = 0; x < st.cx; ++x)
        for (int64_t ia = 0; ia < n_pa; ++ia)
            for (int d0 = 0; d0 < c0; ++d0) {
                int64_t off = static_cast<int64_t>(x) * A.sx + static_cast<int64_t>(d0) * A.strides[0];
                int64_t r = ia;
                for (int j : pa) {
                    off += (r % st.cards[j]) * A.strides[j];
                    r /= st.cards[j];
                }
                words->push_back(static_cast<int32_t>(off));
            }
    // NOTE the loop nest above emits (x, ia, d0) with d0 fastest: index = x*ma + ia*c0 + d0

    std::vector<int64_t> out_stride(n_axes, 1);
    for (int j = 1; j < n_axes; ++j) out_stride[j] = out_stride[j - 1] * st.cards[j - 1];
    st.slab_tile_off_pos = static_cast<int64_t>(words->size());
    std::vector<int> digit(n_axes, 0);
    for (int64_t is = 0; is < n_sh; ++is) {
        int64_t r = is;
        for (int j : sh) { digit[j] = static_cast<int>(r % st.cards[j]); r /= st.cards[j]; }
        int64_t a_super = 0;
        for (int j : sh) a_super += static_cast<int64_t>(digit[j]) * A.strides[j];
        for (int64_t ib = 0; ib < n_pb; ++ib) {
            r = ib;
            for (int j : pb) { digit[j] = static_cast<int>(r % st.cards[j]); r /= st.cards[j]; }
            for (int tb = 0; tb < n_tb; ++tb) {
                for (int64_t ia = 0; ia < n_pa; ++ia) {
                    r = ia;
                    for (int j : pa) { digit[j] = static_cast<int>(r % st.cards[j]); r /= st.cards[j]; }
                    for (int ta = 0; ta < n_ta; ++ta) {
                        const int na = std::min(T, c0 - ta * T), nb = std::min(T, c1 - tb * T);
                        int64_t o = static_cast<int64_t>(ta) * T + static_cast<int64_t>(tb) * T * c0;
                        for (int j = 2; j < n_axes; ++j) o += static_cast<int64_t>(digit[j]) * out_stride[j];
                        words->push_back(static_cast<int32_t>(o));
                        words->push_back(na | (nb << 8));
                        for (int i = 0; i < n_in; ++i) {
                            const InDesc &in = st.in[st.order[i]];
                            int64_t off = static_cast<int64_t>(ta) * T * in.strides[0] + static_cast<int64_t>(tb) * T * in.strides[1];
                            for (int j = 2; j < n_axes; ++j) off += static_cast<int64_t>(digit[j]) * in.strides[j];
                            words->push_back(static_cast<int32_t>(off));
                        }
                        words->push_back(static_cast<int32_t>(is));
                        words->push_back(static_cast<int32_t>(ta * T + static_cast<int64_t>(c0) * ia));
                        words->push_back(static_cast<int32_t>(a_super));
                    }
                }
            }
        }
    }
    return true;
}

// Host half of the tiled kernel: pick the tile edge and precompute, for every tile, the
// output entry and each input's element offset (the row-invariant mixed-radix
// decomposition, hoisted out of the kernel).
void plan_tiles(sbn_program *P, std::vector<int32_t> *words) {
    // joint-state offset tables of the steps that sum out several variables at once:
    // zoff[i][z] = sum_k digit_k(z) * estride_i[k], first eliminated variable fastest
    for (StepDesc &st : P->steps) {
        st.zoff_pos = -1;
        if (st.kind == 3 || st.kind == 7) {
            // count step and joint readout: soff[i][s] = sum_j digit_j(s) * strides_i[j]; count step:
            // coff[s] = sum_j digit_j(s) * cstrides[j]
            st.soff_pos = static_cast<int64_t>(words->size());
            for (const InDesc &in : st.in)
                for (int64_t s = 0; s < st.n_out; ++s) {
                    int64_t r = s, off = 0;
                    for (size_t j = 0; j < st.cards.size(); ++j) {
                        off += (r % st.cards[j]) * in.strides[j];
                        r /= st.cards[j];
                    }
                    words->push_back(static_cast<int32_t>(off));
                }
        }
        if (st.kind == 3) {
            st.coff_pos = static_cast<int64_t>(words->size());
            for (int64_t s = 0; s < st.n_out; ++s) {
                int64_t r = s, off = 0;
                for (size_t j = 0; j < st.cards.size(); ++j) {
                    off += (r % st.cards[j]) * st.cstrides[j];
                    r /= st.cards[j];
                }
                words->push_back(static_cast<int32_t>(off));
            }
        }
        if (st.ecards.size() < 2 && st.kind < 2) continue;
        st.zoff_pos = static_cast<int64_t>(words->size());
        for (const InDesc &in : st.in) {
            for (int z = 0; z < st.cx; ++z) {
                int r = z;
                int64_t off = 0;
                for (size_t k = 0; k < st.ecards.size(); ++k) {
                    off += static_cast<int64_t>(r % st.ecards[k]) * in.estrides[k];
                    r /= st.ecards[k];
                }
                words->push_back(static_cast<int32_t>(off));
            }
        }
    }
    for (StepDesc &st : P->steps) {
        st.tile = 0;
        // an MPE / MAP program's steps run on the log-domain kernels only (launch_step), which have no tiled variant
        if (st.kind != 1 || sbn_log_domain(P->kind) || st.in.size() > static_cast<size_t>(kTiledMaxIn)) continue;

        int64_t smem = 0;
        for (const InDesc &in : st.in)
            if (!in.batched) smem += in.is_slot ? P->slots[in.id].padded : P->table_padded[in.id];
        const bool over = smem * 4 > SBN_SMEM_BUDGET;
        st.big_tables = over && smem * 4 <= smem_big();
        const bool sliced = over && !st.big_tables;  // decided below, once the tiles are known
        const int n_axes = static_cast<int>(st.cards.size());
        const int c0 = n_axes > 0 ? st.cards[0] : 1;
        const int c1 = n_axes > 1 ? st.cards[1] : 1;
        if (c0 > 255 * 5 || c1 > 255 * 5) continue;
        // sort the inputs by the tile axes they carry
        std::vector<int> us, as, bs, cs;
        for (size_t i = 0; i < st.in.size(); ++i) {
            const bool h0 = n_axes > 0 && st.in[i].strides[0] != 0;
            const bool h1 = n_axes > 1 && st.in[i].strides[1] != 0;
            if (h0 && h1) cs.push_back(static_cast<int>(i));
            else if (h0) as.push_back(static_cast<int>(i));
            else if (h1) bs.push_back(static_cast<int>(i));
            else us.push_back(static_cast<int>(i));
        }
        if (cs.size() > 1) continue;  // two inputs span the whole tile: plain kernel
        if (cs.empty()) {
            // a factor without tile axes may ride on either side (stride 0 re-reads one entry)
            while (us.size() > 2 || (as.empty() && !us.empty())) {
                if (as.size() < 2) as.push_back(us.back());
                else if (n_axes > 1 && bs.size() < 2) bs.push_back(us.back());
                else break;
                us.pop_back();
            }
            if (us.size() > 2 || as.empty() || as.size() > 2 || bs.size() > 2) continue;
            if (n_axes > 1 && bs.empty()) continue;
        } else {
            // with a C-side input the instantiated combinations are NU, NA, NB <= 1
            if (us.size() > 1 || as.size() > 1 || bs.size() > 1) continue;
        }
        st.nu = static_cast<int>(us.size());
        st.na = static_cast<int>(as.size());
        st.nb = static_cast<int>(bs.size());
        st.nc = static_cast<int>(cs.size());
        st.order = us;
        st.order.insert(st.order.end(), as.begin(), as.end());
        st.order.insert(st.order.end(), bs.begin(), bs.end());
        st.order.insert(st.order.end(), cs.begin(), cs.end());
        if (st.zoff_pos >= 0) {
            // the tiled kernel sees its inputs in `order`: give it the offset rows in that order
            st.zoff_tiled_pos = static_cast<int64_t>(words->size());
            for (int slot : st.order)
                for (int z = 0; z < st.cx; ++z) {
                    const int32_t v = (*words)[static_cast<size_t>(st.zoff_pos) + static_cast<size_t>(slot) * st.cx + z];
                    words->push_back(v);
                }
        }
        // tile edge: least padding waste, ties to the larger tile
        int best_t = 2;
        double best_w = 1e30;
        for (int t = 2; t <= 5; ++t) {
            auto waste = [&](int c) { return static_cast<double>((c + t - 1) / t * t) / c; };
            // a single-axis output has a T x 1 tile: axis 1 wastes nothing
            const double w = waste(c0) * (n_axes > 1 ? waste(c1) : 1.0);
            if (w < best_w - 1e-9 || (w < best_w + 1e-9 && t > best_t)) {
                best_w = w;
                best_t = t;
            }
        }
        const int T = best_t;
        const int n_ta = (c0 + T - 1) / T, n_tb = (c1 + T - 1) / T;
        const int64_t rest = st.n_out / (static_cast<int64_t>(c0) * c1);
        const int64_t n_tiles = rest * n_ta * n_tb;
        const int n_in = static_cast<int>(st.in.size());
        if (n_tiles * (n_in + 2) > kTileTableMax) continue;
        st.tile = T;
        st.n_tiles = n_tiles;
        st.slab = false;
        if (!over) plan_slab(P, st, T, words);  // optional second tile table in slab order
        st.tile_off_pos = static_cast<int64_t>(words->size());
        std::vector<int64_t> off(n_in);
        for (int64_t r = 0; r < rest; ++r) {
            int64_t q = r;
            std::fill(off.begin(), off.end(), 0);
            for (int j = 2; j < n_axes; ++j) {
                const int d = static_cast<int>(q % st.cards[j]);
                q /= st.cards[j];
                for (int i = 0; i < n_in; ++i) off[i] += static_cast<int64_t>(d) * st.in[st.order[i]].strides[j];
            }
            for (int tb = 0; tb < n_tb; ++tb) {
                for (int ta = 0; ta < n_ta; ++ta) {
                    const int na = std::min(T, c0 - ta * T), nb = std::min(T, c1 - tb * T);
                    words->push_back(static_cast<int32_t>(r * c0 * c1 + static_cast<int64_t>(tb) * T * c0 + ta * T));
                    words->push_back(na | (nb << 8));
                    for (int i = 0; i < n_in; ++i) {
                        int64_t o = off[i];
                        if (n_axes > 0) o += static_cast<int64_t>(ta) * T * st.in[st.order[i]].strides[0];
                        if (n_axes > 1) o += static_cast<int64_t>(tb) * T * st.in[st.order[i]].strides[1];
                        words->push_back(static_cast<int32_t>(o));
                    }
                }
            }
        }
        if (sliced && !plan_slices(P, st, T, words)) st.tile = 0;  // plain kernel, tables from L1/L2
    }
}

void drop_graph(CachedGraph &g) {
    if (g.exec) cudaGraphExecDestroy(g.exec);
    g.exec = nullptr;
}

void drop_graphs(sbn_program *P) {
    // captured launches embed the kernel variants and pointers of the moment they were captured
    drop_graph(P->graph);
    drop_graph(P->pipe_graph);
    drop_graph(P->forward_graph);
}

void free_scratch(sbn_program *P) {
    drop_graphs(P);
    cudaFree(P->d_arena);
    cudaFree(P->d_ev);
    cudaFree(P->d_out);
    cudaFree(P->d_total);
    cudaFree(P->d_lik);
    cudaFree(P->d_log_max);
    cudaFree(P->d_weight);
    P->d_weight = nullptr;
    P->d_lik = nullptr;
    P->d_log_max = nullptr;
    P->d_total = nullptr;
    P->d_arena = nullptr;
    P->d_ev = nullptr;
    P->d_out = nullptr;
    P->reserved_rows = 0;
    P->ld = 0;
}

int64_t batched_floats_per_row(const sbn_program *P) {
    int64_t t = 0;
    for (const Slot &s : P->slots)
        if (s.batched) t += s.size;
    return t;
}

// Fill the kernel parameter block of one step.
void build_params(const sbn_program *P, const StepDesc &st, const uint8_t *ev, int64_t ld_ev, int64_t n_rows,
                  SbnStep *q) {
    memset(q, 0, sizeof *q);
    q->out = P->slots[st.out_slot].ptr;
    q->ev = ev;
    q->ld_ev = ld_ev;
    q->ld = P->ld;
    q->n_rows = static_cast<int32_t>(n_rows);
    q->n_in = static_cast<int32_t>(st.in.size());
    q->n_axes = static_cast<int32_t>(st.cards.size());
    q->cx = st.cx;
    q->cx_inner = st.ecards.empty() ? 1 : st.ecards[0];
    q->zoff = st.zoff_pos >= 0 ? P->d_tile_off + st.zoff_pos : nullptr;
    if (st.kind == 1 && st.tile > 0 && P->use_tiled && !P->f64 && st.zoff_tiled_pos >= 0) q->zoff = P->d_tile_off + st.zoff_tiled_pos;
    q->n_out = static_cast<int32_t>(st.n_out);
    for (size_t j = 0; j < st.cards.size(); ++j) q->card[j] = st.cards[j];
    int smem = 0;
    const bool tiled = st.kind == 1 && st.tile > 0 && P->use_tiled && !P->f64;
    for (size_t i = 0; i < st.in.size(); ++i) {
        const InDesc &in = st.in[tiled ? st.order[i] : i];
        SbnInput &d = q->in[i];
        int64_t padded;
        if (in.is_slot) {
            d.ptr = P->slots[in.id].ptr;
            padded = P->slots[in.id].padded;
        } else {
            d.ptr = reinterpret_cast<const float *>(reinterpret_cast<const char *>(P->d_tables) +
                                                    P->tables[in.id].first * (P->f64 ? 8 : 4));
            padded = P->table_padded[in.id];
        }
        d.batched = in.batched ? 1 : 0;
        d.sx = in.sx;
        d.n_ev = static_cast<int32_t>(in.ev.size());
        for (size_t k = 0; k < in.ev.size(); ++k) {
            d.ev_col[k] = in.ev[k].col;
            d.ev_stride[k] = in.ev[k].stride;
            d.ev_card[k] = in.ev[k].card;
        }
        for (size_t j = 0; j < in.strides.size(); ++j) d.stride[j] = in.strides[j];
        d.smem_off = -1;
        d.stage_floats = 0;
        if (tiled && st.slice_pos >= 0) {
            // sliced staging: the kernel reads (first float, floats, offset) per chunk from q->slices
            if (!in.batched) d.smem_off = 0;
        } else if (st.kind == 1 && !P->f64 && !in.batched && (smem + padded) * 4 <= (tiled ? smem_big() : SBN_SMEM_BUDGET)) {
            d.smem_off = smem;
            d.stage_floats = static_cast<int32_t>(padded);
            smem += static_cast<int>(padded);
        }
    }
    q->smem_floats = smem;
    q->slices = nullptr;
    if (tiled && st.slice_pos >= 0) {
        q->smem_floats = static_cast<int32_t>(st.slice_smem);
        q->slices = P->d_tile_off + st.slice_pos;
    }
    if (tiled) {
        const int64_t rows_per_cta = static_cast<int64_t>(tiled_threads()) * kRowsPerThread;
        const int64_t n_rblocks = (n_rows + rows_per_cta - 1) / rows_per_cta;
        // enough CTAs for ~8 waves (SMs x ~6 resident CTAs), otherwise as many
        // consecutive tiles per CTA as possible (neighbouring tiles share operands in L1)
        static const int64_t target_env = [] {
            const char *e = getenv("SOROBN_B200_TARGET_CTAS");
            return e ? atoll(e) : 0LL;
        }();
        const int64_t sms = P->n_sms;
        // big tables: one CTA per SM, so few CTAs that each amortise their 100+ KB of staging
        int64_t target = st.big_tables ? 4 * sms : (target_env > 0 ? target_env : 8 * sms * 6);
        static const int64_t small_env = [] {
            const char *e = getenv("SOROBN_B200_SMALL_WAVE");
            return e ? atoll(e) : 2000LL;
        }();
        // A launch with few tiles in total (at one tile per CTA: under ~4.5 waves) runs as ONE wave
        // of CTAs that each walk all their tiles: staging and the first loads are paid once per CTA,
        // not once per tile.
        if (small_env > 0 && !st.big_tables && st.n_tiles * n_rblocks <= small_env) target = 3 * sms;
        int64_t chunks = std::max<int64_t>(1, std::min<int64_t>(st.n_tiles, target / std::max<int64_t>(1, n_rblocks)));
        int64_t tpc = (st.n_tiles + chunks - 1) / chunks;
        if (st.slice_pos >= 0) tpc = st.slice_tpc;  // the slices were cut for this chunk size
        q->tiles_per_cta = static_cast<int32_t>(tpc);
        q->n_tiles = static_cast<int32_t>(st.n_tiles);
        q->n_chunks = static_cast<int32_t>((st.n_tiles + tpc - 1) / tpc);
        q->tile_off = P->d_tile_off + st.tile_off_pos;
        q->n_bblocks = static_cast<int32_t>(n_rblocks);
        q->tile1 = 0;
        q->n_tile1 = 0;
        if (st.slab && !st.big_tables && P->use_preload && P->use_slab) {
            // whole groups per CTA; 64-thread CTAs (128 rows) so that the slab fits shared memory
            const int64_t rows_slab = static_cast<int64_t>(kSlabThreads) * kRowsPerThread;
            const int64_t n_rb = (n_rows + rows_slab - 1) / rows_slab;
            const int64_t groups = std::max<int64_t>(1, std::min<int64_t>(st.n_super, target / std::max<int64_t>(1, n_rb)));
            const int64_t supers_per_cta = (st.n_super + groups - 1) / groups;
            q->tiles_per_cta = static_cast<int32_t>(supers_per_cta * st.tiles_per_super);
            q->n_chunks = static_cast<int32_t>((st.n_super + supers_per_cta - 1) / supers_per_cta);
            q->n_bblocks = static_cast<int32_t>(n_rb);
            q->tile_off = P->d_tile_off + st.slab_tile_off_pos;
            q->slab_off = P->d_tile_off + st.slab_off_pos;
            q->n_slab = st.n_slab;
            q->slab_ma = st.slab_ma;
            q->slab_smem_off = static_cast<int32_t>(round_up(q->smem_floats, 4));
        }
    } else if (st.kind == 1) {
        const int c0 = q->n_axes > 0 ? q->card[0] : 1;
        const int c1 = q->n_axes > 1 ? q->card[1] : 1;
        const int64_t rows_per_cta = P->f64 ? SBN_THREADS * 2 : SBN_ROWS_PER_CTA;  // double2 / float4 per thread
        const int64_t n_bblocks = (n_rows + rows_per_cta - 1) / rows_per_cta;
        const int64_t rest = st.n_out / (static_cast<int64_t>(c0) * c1);
        // Tile = axis 0 x tile1 digits of axis 1.  Start from ~32 outputs per thread and
        // shrink while the grid is below two full waves (SMs x 16 CTAs).
        int tile1 = std::max(1, std::min(c1, 32 / std::max(1, c0)));
        auto ctas = [&](int t1) { return n_bblocks * ((c1 + t1 - 1) / t1) * rest; };
        while (tile1 > 1 && ctas(tile1) < 2 * static_cast<int64_t>(P->n_sms) * 16) tile1 = (tile1 + 1) / 2;
        q->tile1 = tile1;
        q->n_tile1 = (c1 + tile1 - 1) / tile1;
        q->n_bblocks = static_cast<int32_t>(n_bblocks);
    }
}

cudaError_t launch_tiled(const StepDesc &st, const SbnStep &q, bool preload, int64_t grid, cudaStream_t stream) {
    // the kernel instantiations live in four translation units (sbn_tiled_*.cu), grouped by the number of
    // inputs without a tile axis / with a both-axes input
    if (q.slab_off != nullptr) return sbn_slab_launch(st.nu, q, st.tile, grid, stream);
    const int key = st.nu * 1000 + st.na * 100 + st.nb * 10 + st.nc;
    // the preload schedule keeps every operand of a tile, for one block of eliminated states, in
    // registers: only for <= 3 inputs, or 4 when two of them carry no tile axis (one value per state)
    preload = preload && (st.in.size() <= 3 || (st.nu == 2 && st.na == 1 && st.nb == 1));
    if (st.nc > 0) return sbn_tiled_c_launch(key, q, st.tile, preload, grid, stream);
    if (st.nu == 0) return sbn_tiled_u0_launch(key, q, st.tile, preload, grid, stream);
    if (st.nu == 1) return sbn_tiled_u1_launch(key, q, st.tile, preload, grid, stream);
    return sbn_tiled_u2_launch(key, q, st.tile, preload, grid, stream);
}

cudaError_t set_tiled_attrs() {
    cudaError_t e = sbn_tiled_u0_set_attrs();
    if (e == cudaSuccess) e = sbn_tiled_u1_set_attrs();
    if (e == cudaSuccess) e = sbn_tiled_u2_set_attrs();
    if (e == cudaSuccess) e = sbn_tiled_c_set_attrs();
    return e;
}

// A step of an MPE or marginal MAP program (log tables): the max-sum or, for a step that sums out (marginal MAP),
// the log-sum-exp instantiations of the flat and the plain batched kernel, whatever the program's switches say --
// the tiled, paired, TMA, join and on-chip kernels are sum-product only.
cudaError_t launch_log_domain(const StepDesc &st, const SbnStep &q, cudaStream_t stream) {
    if (st.kind == 0) {
        const int threads = 256;
        const int64_t grid = (st.n_out + threads - 1) / threads;
        if (st.logsumexp)
            sbn_launch(sbn_step_flat<float, SbnLogSumExp>, dim3(static_cast<unsigned>(grid)), dim3(threads), 0, stream, q);
        else
            sbn_launch(sbn_step_flat<float, SbnMaxSum>, dim3(static_cast<unsigned>(grid)), dim3(threads), 0, stream, q);
        return cudaGetLastError();
    }
    if (st.kind != 1 || q.tile_off != nullptr) return cudaErrorInvalidValue;
    const int64_t rest = st.n_out / (static_cast<int64_t>(q.n_axes > 0 ? q.card[0] : 1) * (q.n_axes > 1 ? q.card[1] : 1));
    const int64_t grid = static_cast<int64_t>(q.n_bblocks) * q.n_tile1 * rest;
    if (grid >= (1LL << 31)) return cudaErrorInvalidConfiguration;
    return st.logsumexp ? sbn_batched_logsumexp_launch(q, grid, stream) : sbn_batched_maxsum_launch(q, grid, stream);
}

cudaError_t launch_step(sbn_program *P, const StepDesc &st, const SbnStep &q, cudaStream_t stream) {
    P->launches++;
    if (sbn_log_domain(P->kind)) return launch_log_domain(st, q, stream);
    if (st.kind == 1 && q.tile_off != nullptr && P->kind != kMarginals && sbn_tma_eligible(P, st))
        return sbn_tma_launch(P, st, q.ev, q.ld_ev, q.n_rows, stream);
    if (st.kind == 1 && q.tile_off != nullptr && sbn_join_rows(P, st, q) > 0) return sbn_join_launch(P, st, q, stream);
    if (st.kind == 1 && q.tile_off != nullptr) {
        const int64_t chunks = (q.n_tiles + q.tiles_per_cta - 1) / q.tiles_per_cta;
        const int64_t grid = chunks * q.n_bblocks;
        if (grid >= (1LL << 31)) return cudaErrorInvalidConfiguration;
        return launch_tiled(st, q, P->use_preload, grid, stream);
    }
    if (st.kind == 0) {
        const int threads = 256;
        const int64_t grid = (st.n_out + threads - 1) / threads;
        if (P->f64) sbn_launch(sbn_step_flat<double>, dim3(static_cast<unsigned>(grid)), dim3(threads), 0, stream, q);
        else sbn_launch(sbn_step_flat<float>, dim3(static_cast<unsigned>(grid)), dim3(threads), 0, stream, q);
        return cudaGetLastError();
    }
    const int64_t rest = st.n_out / (static_cast<int64_t>(q.n_axes > 0 ? q.card[0] : 1) * (q.n_axes > 1 ? q.card[1] : 1));
    const int64_t grid = static_cast<int64_t>(q.n_bblocks) * q.n_tile1 * rest;
    if (grid >= (1LL << 31)) return cudaErrorInvalidConfiguration;
    if (P->f64) {
        const dim3 g(static_cast<unsigned>(grid)), b(SBN_THREADS);
        switch (q.n_in) {
            case 1: sbn_launch(sbn_step_batched_f64<1>, g, b, 0, stream, q); break;
            case 2: sbn_launch(sbn_step_batched_f64<2>, g, b, 0, stream, q); break;
            case 3: sbn_launch(sbn_step_batched_f64<3>, g, b, 0, stream, q); break;
            case 4: sbn_launch(sbn_step_batched_f64<4>, g, b, 0, stream, q); break;
            case 5: sbn_launch(sbn_step_batched_f64<5>, g, b, 0, stream, q); break;
            case 6: sbn_launch(sbn_step_batched_f64<6>, g, b, 0, stream, q); break;
            case 7: sbn_launch(sbn_step_batched_f64<7>, g, b, 0, stream, q); break;
            case 8: sbn_launch(sbn_step_batched_f64<8>, g, b, 0, stream, q); break;
            default: return cudaErrorInvalidValue;
        }
        return cudaGetLastError();
    }
    return sbn_batched_launch(q, grid, stream);
}

// The operands of a readout, count, sample or argmax step (SbnMargIn, SbnCountIn, SbnSampleIn): pointer, batched
// flag and (col stride card) gathers.  Tables are staged like the step kernels' (bulk-TMA, 16-byte aligned and
// sized), float programs only.  Returns the floats of shared memory they take.
template <typename In>
int64_t bind_operands(const sbn_program *P, const StepDesc &st, In *ins) {
    const int64_t elem = P->f64 ? 8 : 4;
    int64_t smem = 0;
    for (size_t i = 0; i < st.in.size(); ++i) {
        const InDesc &in = st.in[i];
        In &d = ins[i];
        int64_t padded;
        if (in.is_slot) {
            d.ptr = P->slots[in.id].ptr;
            padded = P->slots[in.id].padded;
        } else {
            d.ptr = reinterpret_cast<const char *>(P->d_tables) + P->tables[in.id].first * elem;
            padded = P->table_padded[in.id];
        }
        d.batched = in.batched ? 1 : 0;
        d.n_ev = static_cast<int32_t>(in.ev.size());
        for (size_t k = 0; k < in.ev.size(); ++k) {
            d.ev_col[k] = in.ev[k].col;
            d.ev_stride[k] = in.ev[k].stride;
            d.ev_card[k] = in.ev[k].card;
        }
        d.smem_off = -1;
        if (!P->f64 && !in.batched && (smem + padded) * 4 <= SBN_SMEM_BUDGET) {
            d.smem_off = static_cast<int32_t>(smem);
            d.stage_floats = static_cast<int32_t>(padded);
            smem += padded;
        }
    }
    return smem;
}

// Readout of one target (kind 2): its segment of the posterior, normalised, for rows 0 .. n_rows - 1.
cudaError_t launch_marginal(sbn_program *P, const StepDesc &st, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, float *d_out,
                            int64_t ld_out, cudaStream_t stream) {
    P->launches++;
    SbnMarginal m;
    memset(&m, 0, sizeof m);
    const size_t elem = P->f64 ? 8 : 4;
    m.out = reinterpret_cast<char *>(d_out) + st.q_offset * ld_out * static_cast<int64_t>(elem);
    m.ld_out = ld_out;
    m.ev = ev;
    m.ld_ev = ld_ev;
    m.ld = P->ld;
    m.zoff = P->d_tile_off + st.zoff_pos;
    m.min_total = P->f64 ? 1e-290 : static_cast<double>(SBN_MIN_TOTAL_F32);
    m.n_rows = static_cast<int32_t>(n_rows);
    m.n_in = static_cast<int32_t>(st.in.size());
    m.n_common = st.n_common;
    m.card = st.cards[0];
    m.cz = st.cx;
    const int64_t smem = bind_operands(P, st, m.in);
    for (size_t i = 0; i < st.in.size(); ++i) m.in[i].ts = st.in[i].strides[0];
    m.smem_floats = static_cast<int32_t>(smem);
    if (P->f64) return sbn_marginal_launch<double>(m, 0, stream);
    return sbn_marginal_launch<float>(m, static_cast<size_t>(smem) * 4, stream);
}

// Persistent CTAs of one count step: enough for 4 per SM, fewer when the per-warp partial tables of a large
// family would pass kCountPartialBytes.  Depends on the step, the device and n_rows only.
constexpr int64_t kCountPartialBytes = 64LL << 20;
int64_t count_grid(const sbn_program *P, const StepDesc &st, int64_t n_rows) {
    const int64_t blocks = (n_rows + SBN_COUNT_THREADS - 1) / SBN_COUNT_THREADS;
    const int64_t cap = std::max<int64_t>(1, kCountPartialBytes / (8 * SBN_COUNT_WARPS * st.span));
    return std::max<int64_t>(1, std::min<int64_t>({blocks, 4LL * P->n_sms, cap}));
}

// What one run reads and writes beyond its codes and output, for one host call only (the caller's device pointers
// live here, never on the program): the drawn-code buffer's draws and pitch (sample / MPE run: P->d_drawn holds
// codes [n_sampled][n_draws][ld_drawn], one draw for MPE, then one flag byte per row), the likelihoods the pack
// reads and their pitch (soft evidence), the row weights of a gradient program's count steps, whether the run is a
// gradient program's forward run (P(observed) only), and the per-warp partial count tables (counts / backward run).
struct RunInputs {
    int64_t n_draws = 1, ld_drawn = 0;
    const void *lik = nullptr;
    int64_t ld_lik = 0;
    const double *weight = nullptr;
    bool forward = false;
    double *partial = nullptr;
    uint8_t *flags(const sbn_program *P) const { return P->d_drawn + static_cast<int64_t>(P->n_sampled) * n_draws * ld_drawn; }
};

// Count step (kind 3): adds the family's expected counts of rows 0 .. n_rows - 1 into P->d_counts.
cudaError_t launch_count(sbn_program *P, const StepDesc &st, const uint8_t *ev, int64_t ld_ev, int64_t n_rows,
                         const RunInputs &in, cudaStream_t stream) {
    P->launches += 2;
    SbnCount c;
    memset(&c, 0, sizeof c);
    const int64_t grid = count_grid(P, st, n_rows);
    c.partial = in.partial;
    c.ev = ev;
    c.ld_ev = ld_ev;
    c.ld = P->ld;
    const Slot &ps = P->slots[P->post_slot];
    c.prob = ps.ptr;
    c.prob_batched = ps.batched ? 1 : 0;
    c.zoff = st.zoff_pos >= 0 ? P->d_tile_off + st.zoff_pos : nullptr;
    c.soff = P->d_tile_off + st.soff_pos;
    c.coff = P->d_tile_off + st.coff_pos;
    c.min_total = P->f64 ? 1e-290 : static_cast<double>(SBN_MIN_TOTAL_F32);
    c.n_rows = static_cast<int32_t>(n_rows);
    c.n_in = static_cast<int32_t>(st.in.size());
    c.n_common = st.n_common;
    c.cs = static_cast<int32_t>(st.n_out);
    c.cz = st.cx;
    c.n_entries = static_cast<int32_t>(st.span);
    c.n_key = static_cast<int32_t>(st.key.size());
    for (size_t k = 0; k < st.key.size(); ++k) {
        c.key_col[k] = st.key[k].col;
        c.key_stride[k] = st.key[k].stride;
        c.key_card[k] = st.key[k].card;
    }
    const int64_t smem = bind_operands(P, st, c.in);
    c.smem_floats = static_cast<int32_t>(smem);
    double *counts = P->d_counts + st.q_offset;
    const double *weight = P->kind == kGrad ? in.weight : nullptr;  // a gradient program's counts are weighted
    if (P->f64) return sbn_count_launch<double>(c, grid, 0, counts, stream, weight);
    return sbn_count_launch<float>(c, grid, static_cast<size_t>(smem) * 4, counts, stream, weight);
}

// Joint readout of a joint program (kind 7): the group's rows q_offset .. of the output, for rows 0 .. n_rows - 1,
// divided by P(observed)
cudaError_t launch_joint(sbn_program *P, const StepDesc &st, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, float *d_out,
                         int64_t ld_out, cudaStream_t stream) {
    P->launches++;
    SbnCount c;
    memset(&c, 0, sizeof c);
    c.ev = ev;
    c.ld_ev = ld_ev;
    c.ld = P->ld;
    const Slot &ps = P->slots[P->post_slot];
    c.prob = ps.ptr;
    c.prob_batched = ps.batched ? 1 : 0;
    c.zoff = st.zoff_pos >= 0 ? P->d_tile_off + st.zoff_pos : nullptr;
    c.soff = P->d_tile_off + st.soff_pos;
    c.min_total = P->f64 ? 1e-290 : static_cast<double>(SBN_MIN_TOTAL_F32);
    c.n_rows = static_cast<int32_t>(n_rows);
    c.n_in = static_cast<int32_t>(st.in.size());
    c.n_common = st.n_common;
    c.cs = static_cast<int32_t>(st.n_out);
    c.cz = st.cx;
    const int64_t smem = bind_operands(P, st, c.in);
    c.smem_floats = static_cast<int32_t>(smem);
    const int64_t first = st.q_offset * ld_out;
    if (P->f64) return sbn_joint_launch<double>(c, 0, reinterpret_cast<double *>(d_out) + first, ld_out, stream);
    return sbn_joint_launch<float>(c, static_cast<size_t>(smem) * 4, d_out + first, ld_out, stream);
}

// Derivative readout of a gradient program (kind 6): the soft variable's rows q_offset .. of the output, for rows
// 0 .. n_rows - 1, divided by P(observed).
cudaError_t launch_deriv(sbn_program *P, const StepDesc &st, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, float *d_out,
                         int64_t ld_out, cudaStream_t stream) {
    P->launches++;
    SbnDeriv d;
    memset(&d, 0, sizeof d);
    SbnMarginal &m = d.m;
    const size_t elem = P->f64 ? 8 : 4;
    m.out = reinterpret_cast<char *>(d_out) + st.q_offset * ld_out * static_cast<int64_t>(elem);
    m.ld_out = ld_out;
    m.ev = ev;
    m.ld_ev = ld_ev;
    m.ld = P->ld;
    m.zoff = P->d_tile_off + st.zoff_pos;
    m.min_total = P->f64 ? 1e-290 : static_cast<double>(SBN_MIN_TOTAL_F32);
    m.n_rows = static_cast<int32_t>(n_rows);
    m.n_in = static_cast<int32_t>(st.in.size());
    m.n_common = st.n_common;
    m.card = st.cards[0];
    m.cz = st.cx;
    const int64_t smem = bind_operands(P, st, m.in);
    for (size_t i = 0; i < st.in.size(); ++i) m.in[i].ts = st.in[i].strides[0];
    m.smem_floats = static_cast<int32_t>(smem);
    const Slot &ps = P->slots[P->post_slot];
    d.prob = ps.ptr;
    d.prob_batched = ps.batched ? 1 : 0;
    if (P->f64) return sbn_deriv_launch<double>(d, 0, stream);
    return sbn_deriv_launch<float>(d, static_cast<size_t>(smem) * 4, stream);
}

// Sample step (kind 4): draws its variables for rows 0 .. n_rows - 1 and draws 0 .. n_draws - 1 (`k`: its index
// among the sample steps).  Argmax step of an MPE program (kind 5, n_draws = 1): decodes them.
cudaError_t launch_sample(sbn_program *P, const StepDesc &st, int k, const uint8_t *ev, int64_t ld_ev, int64_t n_rows,
                          const RunInputs &in, cudaStream_t stream) {
    P->launches++;
    SbnSample m;
    memset(&m, 0, sizeof m);
    m.ev = ev;
    m.ld_ev = ld_ev;
    m.drawn = P->d_drawn;
    m.ld_drawn = in.ld_drawn;
    m.ld = P->ld;
    m.zoff = P->d_tile_off + st.zoff_pos;
    m.args = P->d_sample_args;
    m.flag = in.flags(P);
    m.min_total = P->f64 ? 1e-290 : static_cast<double>(SBN_MIN_TOTAL_F32);
    m.n_rows = static_cast<int32_t>(n_rows);
    m.n_draws = static_cast<int32_t>(in.n_draws);
    m.n_ev = P->n_ev;
    m.n_in = static_cast<int32_t>(st.in.size());
    m.cz = st.cx;
    m.n_x = static_cast<int32_t>(st.ecards.size());
    m.d_first = static_cast<int32_t>(st.q_offset);
    m.step = k;
    for (size_t j = 0; j < st.ecards.size(); ++j) m.x_card[j] = st.ecards[j];
    const int64_t smem = bind_operands(P, st, m.in);
    m.smem_floats = static_cast<int32_t>(smem);
    if (sbn_log_domain(P->kind)) return sbn_argmax_launch(m, static_cast<size_t>(smem) * 4, stream);
    if (P->f64) return sbn_sample_launch<double>(m, 0, stream);
    return sbn_sample_launch<float>(m, static_cast<size_t>(smem) * 4, stream);
}

// A readout, count, sample, argmax, derivative or joint step (kinds 2 .. 7) on its own launch; `k`: its index among the sample /
// argmax steps (Philox counter word 0 of a sample step)
cudaError_t launch_kind_step(sbn_program *P, const StepDesc &st, int k, const uint8_t *ev, int64_t ld_ev, int64_t n_rows,
                             float *d_out, int64_t ld_out, const RunInputs &in, cudaStream_t stream) {
    if (st.kind == 2) return launch_marginal(P, st, ev, ld_ev, n_rows, d_out, ld_out, stream);
    if (st.kind == 3) return launch_count(P, st, ev, ld_ev, n_rows, in, stream);
    if (st.kind == 6) return launch_deriv(P, st, ev, ld_ev, n_rows, d_out, ld_out, stream);
    if (st.kind == 7) return launch_joint(P, st, ev, ld_ev, n_rows, d_out, ld_out, stream);
    return launch_sample(P, st, k, ev, ld_ev, n_rows, in, stream);
}

// The per-row output of a counts or sample run: P(observed) out of the posterior slot, NaN where it is out of
// range (and, sample run, where a sample step flagged the row)
cudaError_t launch_prob(sbn_program *P, int64_t n_rows, void *d_prob, const uint8_t *flag, cudaStream_t stream) {
    P->launches++;
    const Slot &ps = P->slots[P->post_slot];
    const int threads = 256;
    const unsigned grid = static_cast<unsigned>((n_rows + threads - 1) / threads);
    const int32_t rows = static_cast<int32_t>(n_rows), batched = ps.batched ? 1 : 0;
    const double *p64 = reinterpret_cast<const double *>(ps.ptr);
    if (!flag && P->f64)
        sbn_count_prob<double><<<grid, threads, 0, stream>>>(p64, batched, rows, 1e-290, static_cast<double *>(d_prob));
    else if (!flag)
        sbn_count_prob<float><<<grid, threads, 0, stream>>>(ps.ptr, batched, rows, static_cast<double>(SBN_MIN_TOTAL_F32),
                                                            static_cast<float *>(d_prob));
    else if (P->f64)
        sbn_sample_prob<double><<<grid, threads, 0, stream>>>(p64, batched, flag, rows, 1e-290, static_cast<double *>(d_prob));
    else
        sbn_sample_prob<float><<<grid, threads, 0, stream>>>(ps.ptr, batched, flag, rows, static_cast<double>(SBN_MIN_TOTAL_F32),
                                                             static_cast<float *>(d_prob));
    return cudaGetLastError();
}

cudaError_t launch_normalise(sbn_program *P, float *d_out, int64_t ld_out, int64_t n_rows, cudaStream_t stream) {
    P->launches++;
    const int threads = 256;
    const int64_t grid = (n_rows + threads - 1) / threads;
    if (P->f64)
        sbn_normalise<double><<<static_cast<unsigned>(grid), threads, 0, stream>>>(
            reinterpret_cast<const double *>(P->slots[P->post_slot].ptr), P->ld, P->post_batched, P->Q,
            reinterpret_cast<double *>(d_out), ld_out, static_cast<int>(n_rows), 1e-290,
            reinterpret_cast<double *>(P->d_total));
    else
        sbn_normalise<float><<<static_cast<unsigned>(grid), threads, 0, stream>>>(
            P->slots[P->post_slot].ptr, P->ld, P->post_batched, P->Q, d_out, ld_out, static_cast<int>(n_rows),
            SBN_MIN_TOTAL_F32, P->d_total);
    return cudaGetLastError();
}

// Bytes per likelihood entry of a soft-evidence program: double for a float64 program and for the log-domain kinds,
// whose pack takes the log of each double ratio (their programs are float only, so the caller's scale must not
// pass through float32 first)
inline size_t lik_elem(const sbn_program *P) { return P->f64 || sbn_log_domain(P->kind) ? 8 : 4; }

// Soft-evidence program: fill the likelihood slots from in.lik (pitch in.ld_lik) and sum log(max) per row; the
// log-domain kinds store log(lik / max)
cudaError_t launch_soft_pack(sbn_program *P, int64_t n_rows, const RunInputs &in, cudaStream_t stream) {
    P->launches++;
    const int threads = 256;
    const unsigned grid = static_cast<unsigned>((n_rows + threads - 1) / threads);
    const int32_t rows = static_cast<int32_t>(n_rows), n_soft = static_cast<int32_t>(P->soft.size());
    if (sbn_log_domain(P->kind))  // MPE / MAP: log(lik / max) into the slots of a max-sum / log-sum-exp program
        sbn_soft_pack_log<<<grid, threads, 0, stream>>>(static_cast<const double *>(in.lik), in.ld_lik, rows, n_soft,
                                                        P->d_soft, P->d_arena, P->ld, P->d_log_max);
    else if (P->f64)
        sbn_soft_pack<double><<<grid, threads, 0, stream>>>(static_cast<const double *>(in.lik), in.ld_lik, rows, n_soft,
                                                            P->d_soft, reinterpret_cast<double *>(P->d_arena), P->ld,
                                                            P->d_log_max);
    else
        sbn_soft_pack<float><<<grid, threads, 0, stream>>>(static_cast<const float *>(in.lik), in.ld_lik, rows, n_soft,
                                                           P->d_soft, P->d_arena, P->ld, P->d_log_max);
    return cudaGetLastError();
}

// Evidence-independent steps of a batched program (products of CPTs, possibly keeping evidence
// variables as ordinary axes) depend on the tables only: they run once, in create_common, and
// every later run reads their outputs (19 of the 67 launches of the benchmark grid's step).
inline bool hoisted(const sbn_program *P, const StepDesc &st) { return P->mode == 1 && st.kind == 0; }

inline bool chain_on(const sbn_program *P) {
    return P->use_chain && P->chain_fits && P->use_tiled && !P->use_branches && !P->segments.empty();
}

inline bool pair_on(const sbn_program *P) {
    // with the on-chip segments running, only pairs that were planned around them (SOROBN_B200_CHAIN=1 at creation)
    return P->use_pair && P->use_tiled && !P->use_branches && (!chain_on(P) || P->pairs_avoid_segments) && !P->pairs.empty();
}

int run_table_steps(sbn_program *P) {
    if (P->mode != 1) return SBN_OK;
    SbnStep q;
    for (const StepDesc &st : P->steps) {
        if (!hoisted(P, st)) continue;
        build_params(P, st, nullptr, 0, 1, &q);
        SBN_CUDA(launch_step(P, st, q, P->stream));
    }
    SBN_CUDA(cudaStreamSynchronize(P->stream));
    P->setup_launches = P->launches;
    P->launches = 0;
    return SBN_OK;
}

// The normalisation can ride in the posterior step when that step runs on the tiled kernel (not the
// slab / TMA / plain variants) and its whole output is ONE tile (Q <= T x T joint query states).
inline bool fold_normalise(const sbn_program *P, const StepDesc &st, const SbnStep &q) {
#if !SBN_FOLD_NORMALISE
    // Compiled out by default (sbn_kernels.cuh): the extra epilogue lands in every instantiation of the
    // tiled kernel, so every launch pays for it to save one small normalisation launch.
    (void)P;
    (void)st;
    (void)q;
    return false;
#endif
    static const bool enabled = [] {
        const char *e = getenv("SOROBN_B200_FOLD_NORMALISE");
        return e ? atoi(e) != 0 : true;
    }();
    return enabled && P->kind == kPosterior && !P->f64 && P->post_batched && st.kind == 1 && q.tile_off != nullptr &&
           q.slab_off == nullptr && st.n_tiles == 1 && st.n_out == P->Q && !sbn_tma_eligible(P, st);
}

// Every launch of one run of rows 0 .. n_rows - 1, whatever the program's kind: its steps, then its epilogue.
// d_out is the posterior [Q][ld_out] of a posterior or marginals run, P(observed) [n_rows] of a counts or sample
// run; an MPE run leaves max log P(x, e) in the posterior slot.  `events` (profiling): one record per step, one
// after the steps, one after the epilogue.
int issue_all(sbn_program *P, const uint8_t *d_ev, int64_t ld_ev, int64_t n_rows, float *d_out, int64_t ld_out,
              cudaStream_t stream, cudaEvent_t *events, const RunInputs &in = {}) {
    // the flags of the sample steps start clear in every run, captured graph or not
    if (P->kind == kSample) SBN_CUDA(cudaMemsetAsync(in.flags(P), 0, static_cast<size_t>(n_rows), stream));
    if (!P->soft.empty()) SBN_CUDA(launch_soft_pack(P, n_rows, in, stream));
    SbnStep q;
    int k = 0;
    int n_decoded = 0;  // sample / argmax steps issued so far
    bool folded = false;
    bool skip_second = false;  // the pair launched last covers the next launched step
    for (const StepDesc &st : P->steps) {
        if (events) SBN_CUDA(cudaEventRecord(events[k], stream));
        ++k;
        if (hoisted(P, st)) continue;  // computed once, when the program was created
        if (in.forward && !P->forward[k - 1]) continue;  // a forward run of a gradient program: P(observed) only
        if (st.kind >= 2) {
            const int decoded = st.kind == 4 || st.kind == 5 ? n_decoded++ : 0;
            SBN_CUDA(launch_kind_step(P, st, decoded, d_ev, ld_ev, n_rows, d_out, ld_out, in, stream));
            continue;
        }
        const int seg = chain_on(P) ? P->seg_first[k - 1] : -1;
        if (seg == -2) continue;       // runs inside the segment launched at its first step
        if (seg >= 0) {
            P->launches++;
            SBN_CUDA(sbn_chain_launch(P, *P->segments[seg], d_ev, ld_ev, n_rows, d_out, ld_out, stream));
            continue;
        }
        int pair = pair_on(P) ? P->pair_first[k - 1] : -1;
        if (pair == -2 && !skip_second) pair = -1;  // its first step ran on its own (row pitch beyond 32-bit offsets)
        skip_second = false;
        if (pair == -2) continue;      // computed by the launch of the step that feeds it
        if (pair >= 0 && !sbn_pair_fits(P, *P->pairs[pair])) pair = -1;
        if (pair >= 0) {
            skip_second = true;
            P->launches++;
            SBN_CUDA(sbn_pair_launch(P, *P->pairs[pair], d_ev, ld_ev, n_rows, stream));
            continue;
        }
        build_params(P, st, d_ev, ld_ev, n_rows, &q);
        if (k == static_cast<int>(P->steps.size()) && fold_normalise(P, st, q)) {
            // the posterior step's whole output is one register tile: normalise there, skip the extra launch
            q.norm_out = d_out;
            q.norm_ld = ld_out;
            q.norm_totals = P->d_total;
            q.norm_min = SBN_MIN_TOTAL_F32;
            folded = true;
        }
        SBN_CUDA(launch_step(P, st, q, stream));
    }
    if (events) SBN_CUDA(cudaEventRecord(events[k], stream));
    switch (P->kind) {
        case kPosterior:
            if (!folded && !(chain_on(P) && P->segments.back()->ends_in_posterior))
                SBN_CUDA(launch_normalise(P, d_out, ld_out, n_rows, stream));
            break;
        case kCounts:
        case kGrad: SBN_CUDA(launch_prob(P, n_rows, d_out, nullptr, stream)); break;
        case kSample: SBN_CUDA(launch_prob(P, n_rows, d_out, in.flags(P), stream)); break;
        case kJoint: SBN_CUDA(launch_prob(P, n_rows, P->d_total, nullptr, stream)); break;  // d_out holds the readouts
        case kMarginals:  // the readouts normalise
        case kMpe:
        case kMap: break;
    }
    if (events) SBN_CUDA(cudaEventRecord(events[k + 1], stream));
    return SBN_OK;
}

// Capture-time variant of issue_all: steps are spread over the branch streams and ordered
// by events, so the instantiated graph carries exactly the true dependencies:
//   * read-after-write: a step waits for the producers of its slot inputs;
//   * slot reuse: a step that overwrites a slot waits for the slot's previous writer and
//     for every reader of the previous tenant.
// A step runs on the stream of the producer of its largest slot input (chains stay on one
// stream, no event needed); leaves take the branch streams round-robin.
int issue_branched(sbn_program *P, const uint8_t *d_ev, int64_t ld_ev, int64_t n_rows, float *d_out, int64_t ld_out,
                   cudaStream_t origin, const RunInputs &in) {
    const int n_steps = static_cast<int>(P->steps.size());
    const int n_slots = static_cast<int>(P->slots.size());
    std::vector<int> last_writer(n_slots, -1);
    std::vector<std::vector<int>> readers(n_slots);
    std::vector<int> stream_of(n_steps, 0);
    cudaEvent_t fork = P->step_done[n_steps];  // reused as the fork event before any step
    if (!P->soft.empty()) SBN_CUDA(launch_soft_pack(P, n_rows, in, origin));  // every branch forks after it
    SBN_CUDA(cudaEventRecord(fork, origin));
    bool joined[sbn_program::kBranches] = {false, false, false, false};
    int rr = 0;
    SbnStep q;
    for (int s = 0; s < n_steps; ++s) {
        const StepDesc &st = P->steps[s];
        if (hoisted(P, st)) continue;
        std::vector<int> deps;
        int home = -1;
        int64_t home_size = -1;
        for (const InDesc &in : st.in) {
            if (!in.is_slot) continue;
            const int w = last_writer[in.id];
            if (w >= 0 && !hoisted(P, P->steps[w])) {
                deps.push_back(w);
                if (P->slots[in.id].size > home_size) {
                    home_size = P->slots[in.id].size;
                    home = stream_of[w];
                }
            }
        }
        const bool readout = st.kind >= 2;  // writes the posterior (marginals program), no slot
        if (!readout && last_writer[st.out_slot] >= 0) deps.push_back(last_writer[st.out_slot]);
        if (!readout)
            for (int r : readers[st.out_slot]) deps.push_back(r);
        const int k = home >= 0 ? home : (rr++ % sbn_program::kBranches);
        stream_of[s] = k;
        cudaStream_t stream = P->branch[k];
        if (!joined[k]) {
            SBN_CUDA(cudaStreamWaitEvent(stream, fork, 0));
            joined[k] = true;
        }
        std::sort(deps.begin(), deps.end());
        deps.erase(std::unique(deps.begin(), deps.end()), deps.end());
        for (int d : deps)
            if (stream_of[d] != k) SBN_CUDA(cudaStreamWaitEvent(stream, P->step_done[d], 0));
        if (readout) {
            SBN_CUDA(launch_kind_step(P, st, 0, d_ev, ld_ev, n_rows, d_out, ld_out, in, stream));
        } else {
            build_params(P, st, d_ev, ld_ev, n_rows, &q);
            SBN_CUDA(launch_step(P, st, q, stream));
        }
        SBN_CUDA(cudaEventRecord(P->step_done[s], stream));
        for (const InDesc &in : st.in)
            if (in.is_slot) readers[in.id].push_back(s);
        if (readout) continue;
        last_writer[st.out_slot] = s;
        readers[st.out_slot].clear();
    }
    // join: the origin stream waits for the tail of every branch that was used, then normalises
    std::vector<int> tail(sbn_program::kBranches, -1);
    for (int s = 0; s < n_steps; ++s)
        if (!hoisted(P, P->steps[s])) tail[stream_of[s]] = s;
    for (int k = 0; k < sbn_program::kBranches; ++k)
        if (tail[k] >= 0) SBN_CUDA(cudaStreamWaitEvent(origin, P->step_done[tail[k]], 0));
    if (P->kind == kPosterior) SBN_CUDA(launch_normalise(P, d_out, ld_out, n_rows, origin));
    return SBN_OK;
}

// Per program kind: its name, and the host call of its programs without and with soft evidence
struct KindCalls {
    const char *name, *plain, *soft;
};
constexpr const char *kGradCalls = "sbn_program_grad_forward_host / sbn_program_grad_backward_host";
constexpr KindCalls kKindCalls[] = {
    {"posterior", "sbn_program_run_host", "sbn_program_run_soft_host"},
    {"marginals", "sbn_program_run_host", "sbn_program_run_soft_host"},
    {"counts", "sbn_program_counts_host", "sbn_program_counts_soft_host"},
    {"sample", "sbn_program_sample_host", "sbn_program_sample_soft_host"},
    {"MPE", "sbn_program_mpe_host", "sbn_program_mpe_soft_host"},
    {"MAP", "sbn_program_mpe_host", "sbn_program_mpe_soft_host"},
    {"gradient", kGradCalls, kGradCalls},
    {"joint", "sbn_program_joint_host", "sbn_program_joint_host"},
};

// The checks every run shares: the program is of the kind the entry point runs (kPosterior: the run, evidence and
// profile calls, which take posterior and marginals programs; kMpe: MPE and MAP programs) and has soft evidence
// exactly when the call is the kind's soft-evidence call (the gradient and joint calls take both), and the rows
// and their evidence are well formed
int check_rows(const sbn_program *P, ProgramKind kind, const void *ev, int64_t ld_ev, int64_t n_rows, bool soft = false) {
    if (!P) return fail(SBN_E_INVALID, "null program");
    const KindCalls &calls = kKindCalls[P->kind];
    const bool has_soft = !P->soft.empty();
    const char *own = has_soft ? calls.soft : calls.plain;
    if ((P->kind == kMarginals ? kPosterior : P->kind == kMap ? kMpe : P->kind) != kind)
        return fail(SBN_E_INVALID, "a %s program%s runs through %s", calls.name, has_soft ? " with soft evidence" : "", own);
    if (kind != kGrad && kind != kJoint && has_soft != soft)
        return fail(SBN_E_INVALID, "a %s program %s soft evidence runs through %s", calls.name, has_soft ? "with" : "without",
                    own);
    if (n_rows <= 0) return fail(SBN_E_INVALID, "n_rows must be positive");
    if (P->n_ev > 0 && !ev) return fail(SBN_E_INVALID, "null evidence");
    if (P->n_ev > 1 && ld_ev < n_rows) return fail(SBN_E_INVALID, "ld_ev < n_rows");
    if (P->mode == 0 && n_rows != 1) return fail(SBN_E_INVALID, "a flat program answers exactly one row");
    return SBN_OK;
}

// check_rows for the calls that write a posterior [Q][ld_out]
int check_run_args(const sbn_program *P, const void *ev, int64_t ld_ev, int64_t n_rows, const void *out, int64_t ld_out,
                   bool soft = false) {
    const int rc = check_rows(P, kPosterior, ev, ld_ev, n_rows, soft);
    if (rc != SBN_OK) return rc;
    if (!out) return fail(SBN_E_INVALID, "null output");
    if (P->Q > 1 && ld_out < n_rows) return fail(SBN_E_INVALID, "ld_out < n_rows");
    return SBN_OK;
}

// Make the program's device current and grow its scratch to n_rows (it never shrinks).  The reservation is capped
// by the free device memory, so it may stay below n_rows: the host paths then run in chunks.
int reserve_rows(sbn_program *P, int64_t n_rows) {
    SBN_CUDA(cudaSetDevice(P->device));
    return n_rows > P->reserved_rows ? sbn_program_reserve(P, n_rows) : SBN_OK;
}

// Rows per chunk of a host call: the reservation, capped by SOROBN_B200_CHUNK_ROWS (rounded down to a multiple of 32,
// at least 32) when it is set, so that a test can run a batch in several chunks.  Read on every call.
int64_t chunk_rows(const sbn_program *P) {
    const char *e = getenv("SOROBN_B200_CHUNK_ROWS");
    if (!e || !*e) return P->reserved_rows;
    return std::min(P->reserved_rows, std::max<int64_t>(32, atoll(e) / 32 * 32));
}

// Replay `g` on `stream`.  When `key` differs from the key it was captured for, capture it first: `issue()` issues
// one run on the capture stream `cap`, and the launches it counts are what every replay adds to P->launches.
template <typename Issue>
int replay(sbn_program *P, CachedGraph &g, const GraphKey &key, cudaStream_t cap, cudaStream_t stream, Issue &&issue) {
    if (!g.exec || !(g.key == key)) {
        drop_graph(g);
        SBN_CUDA(cudaStreamBeginCapture(cap, cudaStreamCaptureModeRelaxed));
        const int64_t before = P->launches;
        const int rc = issue();
        cudaGraph_t graph = nullptr;
        cudaError_t e = cudaStreamEndCapture(cap, &graph);
        g.launches = P->launches - before;
        P->launches = before;
        if (rc == SBN_OK && e == cudaSuccess) e = cudaGraphInstantiate(&g.exec, graph, 0);
        if (graph) cudaGraphDestroy(graph);
        if (rc != SBN_OK) return rc;
        if (e != cudaSuccess) {
            cudaGetLastError();
            g.exec = nullptr;
            return fail(SBN_E_CUDA, "graph capture failed: %s", cudaGetErrorString(e));
        }
        g.key = key;
    }
    SBN_CUDA(cudaGraphLaunch(g.exec, stream));
    P->launches += g.launches;
    return SBN_OK;
}

constexpr int64_t kSampleGraphMinRows = 4096;

// One run of rows already on the device: a replay of the program's graph (captured on the program's stream) when
// graphs are on, else plain launches on `stream`
int run_rows(sbn_program *P, const uint8_t *d_ev, int64_t ld_ev, int64_t n_rows, float *d_out, int64_t ld_out,
             cudaStream_t stream, const RunInputs &in = {}) {
    // a short sample / MPE chunk runs as plain launches: capturing and instantiating a graph costs more than it
    // saves, and the short runs of a pattern whose rows are scattered through a frame come in many lengths
    const bool short_chunk = (P->kind == kSample || sbn_log_domain(P->kind)) && n_rows < kSampleGraphMinRows;
    if (!P->use_graph || short_chunk) return issue_all(P, d_ev, ld_ev, n_rows, d_out, ld_out, stream, nullptr, in);
    const GraphKey key = {d_ev, ld_ev, n_rows, d_out, ld_out, in.partial, P->d_drawn, in.n_draws, in.ld_drawn, in.lik,
                          in.ld_lik, in.forward ? nullptr : in.weight};
    const bool branched = P->use_branches && P->kind <= kMarginals;
    // a gradient program's forward run issues a subset of its launches: it keeps a graph of its own
    return replay(P, in.forward ? P->forward_graph : P->graph, key, P->stream, stream, [&] {
        return branched ? issue_branched(P, d_ev, ld_ev, n_rows, d_out, ld_out, P->stream, in)
                        : issue_all(P, d_ev, ld_ev, n_rows, d_out, ld_out, P->stream, nullptr, in);
    });
}

// Walk a host batch in chunks of at most `cap` rows on the program's stream: upload each chunk's codes to
// P->d_ev, then `body(r0, rows)` runs the chunk and downloads its outputs
template <typename Body>
int for_each_chunk(sbn_program *P, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, int64_t cap, Body &&body) {
    for (int64_t r0 = 0; r0 < n_rows; r0 += cap) {
        const int64_t rows = std::min(cap, n_rows - r0);
        if (P->n_ev > 0)
            SBN_CUDA(cudaMemcpy2DAsync(P->d_ev, static_cast<size_t>(P->ld), ev + r0, static_cast<size_t>(ld_ev),
                                       static_cast<size_t>(rows), static_cast<size_t>(P->n_ev), cudaMemcpyHostToDevice,
                                       P->stream));
        const int rc = body(r0, rows);
        if (rc != SBN_OK) return rc;
    }
    return SBN_OK;
}

// Whether a posterior run of n_rows host rows in chunks of `cap` goes through run_pipelined
bool pipelined(const sbn_program *P, int64_t n_rows, int64_t cap, size_t elem) {
    // Transfer-bound programs (a handful of launches for megabytes of codes in and posteriors
    // out: Asia is ONE batched launch for 4 MB + 8 MB per million rows) are pipelined: the batch is
    // cut into column ranges of the same staging buffers, H2D / kernels / D2H run on three streams
    // chained by events, so a range's posteriors drain while the next range computes and the one
    // after uploads -- PCIe is full duplex.  Launch-heavy programs (the grid: 48 launches per run,
    // 5 MB of copies against milliseconds of kernels) keep the single CUDA-graph replay.
    int64_t launches_per_run = 1;
    for (size_t k = 0; k < P->steps.size(); ++k)
        if (!hoisted(P, P->steps[k])) ++launches_per_run;
    const int64_t bytes = n_rows * (P->n_ev + static_cast<int64_t>(P->Q) * static_cast<int64_t>(elem));
    static const int pipe_env = [] {
        const char *e = getenv("SOROBN_B200_PIPELINE");
        return e ? atoi(e) : 1;
    }();
    return pipe_env && n_rows <= cap && launches_per_run <= 8 && bytes >= (int64_t(2) << 20) && n_rows >= 4 * 32768;
}

// One posterior run of a whole host batch (n_rows <= the reservation), pipelined over column ranges
int run_pipelined(sbn_program *P, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, char *out, int64_t ld_out, size_t elem) {
    constexpr int kMaxRanges = 8;
    static const int kRanges = [] {
        const char *e = getenv("SOROBN_B200_PIPE_RANGES");
        // few ranges: each range adds copies and launches, and the copies are the bound
        const int v = e ? atoi(e) : 3;
        return v >= 2 && v <= kMaxRanges ? v : 3;
    }();
    if (P->pipe_events.empty()) {
        P->pipe_events.resize(3 + 2 * kMaxRanges);
        for (auto &e : P->pipe_events) SBN_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    }
    cudaStream_t s_in = P->branch[0], s_run = P->stream, s_out = P->branch[1];
    const int64_t range = round_up((n_rows + kRanges - 1) / kRanges, 32);
    // the side streams fork from s_run and join back into it; a few plain launches per range, nothing to
    // amortise inside
    auto issue_ranges = [&]() -> int {
        cudaEvent_t fork = P->pipe_events[0], j_in = P->pipe_events[1 + 2 * kMaxRanges], j_out = P->pipe_events[2 + 2 * kMaxRanges];
        SBN_CUDA(cudaEventRecord(fork, s_run));
        SBN_CUDA(cudaStreamWaitEvent(s_in, fork, 0));
        SBN_CUDA(cudaStreamWaitEvent(s_out, fork, 0));
        for (int64_t r0 = 0, k = 0; r0 < n_rows; r0 += range, ++k) {
            const int64_t rows = std::min(range, n_rows - r0);
            cudaEvent_t up = P->pipe_events[1 + 2 * k], done = P->pipe_events[2 + 2 * k];
            if (P->n_ev > 0) {
                SBN_CUDA(cudaMemcpy2DAsync(P->d_ev + r0, static_cast<size_t>(P->ld), ev + r0, static_cast<size_t>(ld_ev),
                                           static_cast<size_t>(rows), static_cast<size_t>(P->n_ev), cudaMemcpyHostToDevice, s_in));
                SBN_CUDA(cudaEventRecord(up, s_in));
                SBN_CUDA(cudaStreamWaitEvent(s_run, up, 0));
            }
            char *d_out = reinterpret_cast<char *>(P->d_out) + r0 * elem;
            const int rc = issue_all(P, P->d_ev + r0, P->ld, rows, reinterpret_cast<float *>(d_out), P->ld, s_run, nullptr);
            if (rc != SBN_OK) return rc;
            SBN_CUDA(cudaEventRecord(done, s_run));
            SBN_CUDA(cudaStreamWaitEvent(s_out, done, 0));
            SBN_CUDA(cudaMemcpy2DAsync(out + r0 * elem, static_cast<size_t>(ld_out) * elem, d_out, static_cast<size_t>(P->ld) * elem,
                                       static_cast<size_t>(rows) * elem, static_cast<size_t>(P->Q), cudaMemcpyDeviceToHost, s_out));
        }
        SBN_CUDA(cudaEventRecord(j_in, s_in));
        SBN_CUDA(cudaStreamWaitEvent(s_run, j_in, 0));
        SBN_CUDA(cudaEventRecord(j_out, s_out));
        SBN_CUDA(cudaStreamWaitEvent(s_run, j_out, 0));
        return SBN_OK;
    };
    // the whole fan-out is replayed as ONE graph launch when the host buffers are pinned (a dozen copies,
    // launches and event edges cost CPU time of the order of what they overlap); the graph is kept for the
    // (buffers, rows) it was built for
    auto pinned = [](const void *ptr) {
        cudaPointerAttributes a;
        if (cudaPointerGetAttributes(&a, ptr) != cudaSuccess) {
            cudaGetLastError();
            return false;
        }
        return a.type == cudaMemoryTypeHost;
    };
    int rc;
    if (P->use_graph && pinned(out) && (P->n_ev == 0 || pinned(ev)))
        rc = replay(P, P->pipe_graph, {ev, ld_ev, n_rows, out, ld_out}, s_run, s_run, issue_ranges);
    else
        rc = issue_ranges();
    if (rc != SBN_OK) {  // the side streams may not have joined s_run
        cudaStreamSynchronize(s_in);
        cudaStreamSynchronize(s_out);
    }
    const cudaError_t e = cudaStreamSynchronize(s_run);
    if (rc != SBN_OK) return rc;
    SBN_CUDA(e);
    return SBN_OK;
}

// One host call: the program kind it takes (as check_rows), whether it is the kind's soft-evidence call, its
// precision, the caller's rows and where each output goes.  The caller's pointers are read and written during the
// call only.
struct HostCall {
    HostCall(ProgramKind kind, bool f64, const uint8_t *ev, int64_t ld_ev, int64_t n_rows)
        : kind(kind), f64(f64), ev(ev), ld_ev(ld_ev), n_rows(n_rows) {}
    ProgramKind kind;
    bool soft = false;
    bool f64;
    const uint8_t *ev;  // codes [n_ev][ld_ev]
    int64_t ld_ev, n_rows;
    const void *lik = nullptr;  // soft evidence: [n_rows][ld_lik], host or (lik_on_device) device memory
    int64_t ld_lik = 0;
    int lik_on_device = 0;
    const double *weights = nullptr;  // gradient program: the row weights of a backward call (null: a forward call)
    int weights_on_device = 0;
    int64_t n_draws = 1;  // sample program: draws per row, seed, the caller's index of row 0
    uint64_t seed = 0;
    int64_t row_base = 0;
    // the readouts [Q][ld_out] of a posterior or joint run, the derivative readouts [n_lik][ld_out] of a backward
    // run, the drawn / decoded codes [n_sampled][n_draws][n_rows] of a sample / MPE run
    void *out = nullptr;
    int64_t ld_out = 0;
    // per row, in the program's type: P(event) of a posterior run, P(observed) of a counts, sample, gradient or
    // joint run, max log P of an MPE run
    void *prob = nullptr;
    double *log_prob = nullptr;  // per row: log of prob (MPE: prob) + sum log(max) of a soft-evidence row
    double *counts = nullptr;    // counts program / backward call: the count table [n_counts], added into
    int64_t n_counts = 0;
};

// Every host call but the pipelined posterior run: the checks, the reservation, the call's buffers, then per chunk
// the staged rows, one run and its downloads, and after one final sync the count table and log P of the batch.
int host_call(sbn_program *P, const HostCall &c) {
    int rc = check_rows(P, c.kind, c.ev, c.ld_ev, c.n_rows, c.soft);
    if (rc != SBN_OK) return rc;
    if (P->f64 != c.f64) return fail(SBN_E_INVALID, "program precision does not match the call");
    const int64_t n_rows = c.n_rows;
    const bool soft = !P->soft.empty(), mpe = c.kind == kMpe, decodes = mpe || c.kind == kSample;
    const bool backward = c.kind == kGrad && c.weights, counting = c.kind == kCounts || backward;
    const char *joint_call = c.f64 ? "sbn_program_joint_host_f64" : "sbn_program_joint_host";
    if (c.kind == kJoint && soft && !c.lik)
        return fail(SBN_E_INVALID, "a joint program with soft evidence needs its likelihoods: pass lik to %s", joint_call);
    if (c.kind == kJoint && !soft && c.lik)
        return fail(SBN_E_INVALID, "a joint program without soft evidence takes no likelihoods: pass lik = NULL to %s", joint_call);
    if (soft && !c.lik) return fail(SBN_E_INVALID, "null likelihoods");
    if (soft && c.ld_lik < P->n_lik)
        return fail(SBN_E_INVALID, "ld_lik %lld < the %d likelihood columns", (long long)c.ld_lik, P->n_lik);
    switch (c.kind) {  // the outputs
        case kPosterior:
            if (!c.out && !c.prob) return fail(SBN_E_INVALID, "null output");
            if (c.out && P->Q > 1 && c.ld_out < n_rows) return fail(SBN_E_INVALID, "ld_out < n_rows");
            if (P->kind == kMarginals && (c.prob || c.log_prob))
                return fail(SBN_E_INVALID, "a marginals program has no single normaliser; P(event) and log P(e, lik) come "
                                           "from a posterior program");
            break;
        case kJoint:
            if (!c.out || !c.prob) return fail(SBN_E_INVALID, "null output");
            if (c.ld_out < n_rows) return fail(SBN_E_INVALID, "ld_out < n_rows");
            break;
        case kSample:
            if (c.n_draws <= 0 || c.n_draws > INT32_MAX) return fail(SBN_E_INVALID, "n_draws must be in 1 .. 2^31 - 1");
            if (c.row_base < 0) return fail(SBN_E_INVALID, "row_base must not be negative");
            if ((P->n_sampled > 0 && !c.out) || !c.prob) return fail(SBN_E_INVALID, "null output");
            break;
        case kMpe:
            if ((P->n_sampled > 0 && !c.out) || (!c.prob && !c.log_prob)) return fail(SBN_E_INVALID, "null output");
            break;
        case kCounts:
            if (!c.counts || !c.prob) return fail(SBN_E_INVALID, "null output");
            break;
        case kGrad:
            if (backward && (!c.counts || (P->n_lik > 0 && !c.out))) return fail(SBN_E_INVALID, "null output");
            if (backward && P->n_lik > 0 && c.ld_out < n_rows) return fail(SBN_E_INVALID, "ld_deriv < n_rows");
            break;
        default: break;
    }
    if (counting && c.n_counts != P->n_counts)
        return fail(SBN_E_INVALID, "the count table has %lld entries, not %lld", (long long)P->n_counts, (long long)c.n_counts);
    // the chunk capacity follows the largest batch seen so far (a program first used for one row must not answer a
    // later million-row batch one row at a time)
    rc = reserve_rows(P, n_rows);
    if (rc != SBN_OK) return rc;
    int64_t cap = chunk_rows(P);
    const size_t elem = c.f64 ? 8 : 4;
    if (c.kind == kPosterior && c.out && !soft && pipelined(P, n_rows, cap, elem))
        return run_pipelined(P, c.ev, c.ld_ev, n_rows, static_cast<char *>(c.out), c.ld_out, elem);

    // from here on every return leaves nothing running on the program's stream and frees the partial tables
    struct Finish {
        sbn_program *P;
        double *partial;
        ~Finish() {
            cudaStreamSynchronize(P->stream);
            if (partial) cudaFree(partial);
        }
    } finish = {P, nullptr};
    RunInputs in;
    in.forward = c.kind == kGrad && !backward;
    if (counting) {
        // the per-warp partial tables live for this call only: a program that is not running holds none of them
        const cudaError_t e = cudaMalloc(&finish.partial, static_cast<size_t>(std::max<int64_t>(1, P->partial_doubles)) * 8);
        if (e != cudaSuccess) {
            cudaGetLastError();
            finish.partial = nullptr;
            return fail(SBN_E_NOMEM, "cudaMalloc of %lld bytes of partial count tables failed: %s",
                        (long long)(P->partial_doubles * 8), cudaGetErrorString(e));
        }
        in.partial = finish.partial;
        SBN_CUDA(cudaMemsetAsync(P->d_counts, 0, static_cast<size_t>(P->n_counts) * 8, P->stream));
    }
    if (decodes) {
        // the drawn codes of a chunk ([n_sampled][n_draws] bytes + one flag byte per row) take at most half of the
        // free device memory: larger batches run in more chunks
        const int64_t per_row = static_cast<int64_t>(P->n_sampled) * c.n_draws + 1;
        if (round_up(std::min(cap, n_rows), 32) * per_row > P->drawn_bytes) {  // the buffer of an earlier call may do
            size_t free_b = 0, total_b = 0;
            SBN_CUDA(cudaMemGetInfo(&free_b, &total_b));
            const int64_t budget = static_cast<int64_t>(free_b / 2) + P->drawn_bytes;
            if (round_up(cap, 32) * per_row > budget) cap = std::max<int64_t>(32, budget / per_row / 32 * 32);
        }
        in.n_draws = c.n_draws;
        in.ld_drawn = round_up(std::min(cap, n_rows), 32);
        const int64_t bytes = in.ld_drawn * per_row;
        if (bytes > P->drawn_bytes) {
            SBN_CUDA(cudaStreamSynchronize(P->stream));
            cudaFree(P->d_drawn);
            P->d_drawn = nullptr;
            P->drawn_bytes = 0;
            const cudaError_t e = cudaMalloc(&P->d_drawn, static_cast<size_t>(bytes));
            if (e != cudaSuccess) {
                cudaGetLastError();
                P->d_drawn = nullptr;
                return fail(SBN_E_NOMEM, "cudaMalloc of %lld bytes of drawn codes failed: %s", (long long)bytes, cudaGetErrorString(e));
            }
            P->drawn_bytes = bytes;
        }
        if (!mpe && !P->d_sample_args) SBN_CUDA(cudaMalloc(&P->d_sample_args, 4 * sizeof(uint32_t)));
    }
    // a chunk's readouts: rows first .. first + n_readouts - 1 of d_out (a gradient program's derivatives follow
    // its P(observed) row)
    const int64_t first = c.kind == kGrad ? 1 : 0;
    const int64_t n_readouts = !c.out || decodes ? 0 : c.kind == kGrad ? P->n_lik : P->Q;
    // a chunk's per-row value: the normaliser of a posterior or joint run, the maximum in the posterior slot of an
    // MPE run ([1][ld], or one value for every row), P(observed) in d_out otherwise; into the caller's prob, or into
    // a batch buffer of the call's own when only its log is asked for
    const bool one_value = mpe && !P->slots[P->post_slot].batched;
    const void *value = c.kind == kPosterior || c.kind == kJoint ? static_cast<const void *>(P->d_total)
                        : mpe                                    ? P->slots[P->post_slot].ptr
                                                                 : P->d_out;
    std::vector<char> own(!c.prob && c.log_prob ? static_cast<size_t>(n_rows) * elem : 0);
    char *prob = c.prob ? static_cast<char *>(c.prob) : own.empty() ? nullptr : own.data();
    std::vector<double> log_max(c.log_prob ? static_cast<size_t>(n_rows) : 0, 0.0);
    const size_t lik_bytes = lik_elem(P);
    rc = for_each_chunk(P, c.ev, c.ld_ev, n_rows, cap, [&](int64_t r0, int64_t rows) -> int {
        // the chunk's likelihoods and weights: device rows read in place, host rows staged on the program's stream
        const char *lik = static_cast<const char *>(c.lik) + r0 * c.ld_lik * static_cast<int64_t>(lik_bytes);
        if (soft && c.lik_on_device) {
            in.lik = lik;
            in.ld_lik = c.ld_lik;
        } else if (soft) {
            SBN_CUDA(cudaMemcpy2DAsync(P->d_lik, static_cast<size_t>(P->n_lik) * lik_bytes, lik, static_cast<size_t>(c.ld_lik) * lik_bytes,
                                       static_cast<size_t>(P->n_lik) * lik_bytes, static_cast<size_t>(rows), cudaMemcpyHostToDevice,
                                       P->stream));
            in.lik = P->d_lik;
            in.ld_lik = P->n_lik;
        }
        if (backward && c.weights_on_device) {
            in.weight = c.weights + r0;
        } else if (backward) {
            SBN_CUDA(cudaMemcpyAsync(P->d_weight, c.weights + r0, static_cast<size_t>(rows) * 8, cudaMemcpyHostToDevice, P->stream));
            in.weight = P->d_weight;
        }
        if (c.kind == kSample) {
            // read by the sample steps at run time, so that one captured graph serves every seed and chunk
            const uint64_t first_row = static_cast<uint64_t>(c.row_base + r0);
            const uint32_t args[4] = {static_cast<uint32_t>(c.seed), static_cast<uint32_t>(c.seed >> 32),
                                      static_cast<uint32_t>(first_row), static_cast<uint32_t>(first_row >> 32)};
            SBN_CUDA(cudaMemcpyAsync(P->d_sample_args, args, sizeof args, cudaMemcpyHostToDevice, P->stream));
        }
        // the graph reads the tables and the count table by address, so it replays the values sbn_program_set_tables uploads
        const int rc = run_rows(P, P->d_ev, P->ld, rows, P->d_out, P->ld, P->stream, in);
        if (rc != SBN_OK) return rc;
        if (decodes && P->n_sampled > 0)
            SBN_CUDA(cudaMemcpy2DAsync(static_cast<uint8_t *>(c.out) + r0, static_cast<size_t>(n_rows), P->d_drawn,
                                       static_cast<size_t>(in.ld_drawn), static_cast<size_t>(rows),
                                       static_cast<size_t>(P->n_sampled * c.n_draws), cudaMemcpyDeviceToHost, P->stream));
        if (n_readouts > 0)
            SBN_CUDA(cudaMemcpy2DAsync(static_cast<char *>(c.out) + r0 * elem, static_cast<size_t>(c.ld_out) * elem,
                                       reinterpret_cast<char *>(P->d_out) + first * P->ld * elem, static_cast<size_t>(P->ld) * elem,
                                       static_cast<size_t>(rows) * elem, static_cast<size_t>(n_readouts), cudaMemcpyDeviceToHost,
                                       P->stream));
        if (prob && !one_value)
            SBN_CUDA(cudaMemcpyAsync(prob + r0 * elem, value, static_cast<size_t>(rows) * elem, cudaMemcpyDeviceToHost, P->stream));
        else if (prob && r0 == 0)
            SBN_CUDA(cudaMemcpyAsync(prob, value, elem, cudaMemcpyDeviceToHost, P->stream));
        if (soft && c.log_prob)
            SBN_CUDA(cudaMemcpyAsync(log_max.data() + r0, P->d_log_max, static_cast<size_t>(rows) * 8, cudaMemcpyDeviceToHost, P->stream));
        return SBN_OK;
    });
    if (rc != SBN_OK) return rc;
    std::vector<double> table(counting ? static_cast<size_t>(P->n_counts) : 0);
    if (counting) SBN_CUDA(cudaMemcpyAsync(table.data(), P->d_counts, table.size() * 8, cudaMemcpyDeviceToHost, P->stream));
    SBN_CUDA(cudaStreamSynchronize(P->stream));
    for (size_t i = 0; i < table.size(); ++i) c.counts[i] += table[i];
    if (one_value && prob) std::fill(reinterpret_cast<float *>(prob) + 1, reinterpret_cast<float *>(prob) + n_rows, *reinterpret_cast<float *>(prob));
    // log P(observed, lik) = log P(observed, lik / max) + sum log(max) of the row, NaN where the row is flagged; an
    // MPE run's maximum is a log already
    for (int64_t i = 0; c.log_prob && i < n_rows; ++i) {
        const double p = c.f64 ? reinterpret_cast<const double *>(prob)[i] : reinterpret_cast<const float *>(prob)[i];
        c.log_prob[i] = (mpe ? p : std::log(p)) + log_max[static_cast<size_t>(i)];
    }
    return SBN_OK;
}

}  // namespace

// =========================================================================== C ABI
extern "C" {

int sbn_abi_version(void) { return SBN_ABI_VERSION; }
const char *sbn_last_error(void) { return g_err.c_str(); }

int sbn_device_count(int *count) {
    if (!count) return fail(SBN_E_INVALID, "null count");
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0) {
        *count = 0;
        return fail(SBN_E_NODEVICE, "no CUDA device: %s", cudaGetErrorString(e));
    }
    *count = n;
    return SBN_OK;
}

static int create_common(int device, const int32_t *words, int64_t n_words, const void *tables, int64_t n_table_floats,
                         bool f64, sbn_program **out) {
    if (!words || !out || (n_table_floats > 0 && !tables)) return fail(SBN_E_INVALID, "null argument");
    *out = nullptr;
    sbn_program *P = new sbn_program();
    P->device = device;
    P->f64 = f64;
    P->n_table_floats = n_table_floats;
    {
        const char *e = getenv("SOROBN_B200_CHAIN");
        P->use_chain = e && atoi(e) != 0;  // on-chip segments are opt-in (see sbn_chain.cu)
        e = getenv("SOROBN_B200_TMA");
        P->use_tma = e && atoi(e) != 0;    // so is the tensor-map TMA pipeline kernel (see sbn_tma.cu: no gain measured)
        e = getenv("SOROBN_B200_PAIR");
        P->use_pair = e ? atoi(e) != 0 : true;  // paired steps (sbn_pair.h)
    }
    const size_t elem = f64 ? 8 : 4;
    int rc = parse(P, words, n_words);

    if (rc != SBN_OK) {
        delete P;
        return rc;
    }
    if (sbn_log_domain(P->kind) && f64) {
        const char *what = P->kind == kMap ? "MAP" : "MPE";
        delete P;
        return fail(SBN_E_INVALID, "an %s program runs in float32 only (its tables are logs: nothing underflows)", what);
    }
    for (size_t t = 0; t < P->tables.size(); ++t) {
        if (P->tables[t].first + P->table_padded[t] > n_table_floats) {
            delete P;
            return fail(SBN_E_INVALID, "table %zu lies outside the table blob", t);
        }
    }
    int n_dev = 0;
    if (cudaGetDeviceCount(&n_dev) != cudaSuccess || n_dev == 0) {
        delete P;
        return fail(SBN_E_NODEVICE, "no CUDA device available");
    }
    if (device < 0 || device >= n_dev) {
        delete P;
        return fail(SBN_E_NODEVICE, "device %d out of range (%d visible)", device, n_dev);
    }
    auto bail = [&](int code) {
        sbn_program_destroy(P);
        return code;
    };
#define SBN_CUDA_P(call)                                                                                      \
    do {                                                                                                      \
        cudaError_t e_ = (call);                                                                              \
        if (e_ != cudaSuccess)                                                                                \
            return bail(fail(SBN_E_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__)); \
    } while (0)
    SBN_CUDA_P(cudaSetDevice(device));
    cudaDeviceProp prop;
    SBN_CUDA_P(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0)
        return bail(fail(SBN_E_NODEVICE, "device %d is sm_%d%d; this library is built for sm_90a only", device, prop.major,
                         prop.minor));
    P->n_sms = prop.multiProcessorCount;
    SBN_CUDA_P(cudaStreamCreateWithFlags(&P->stream, cudaStreamNonBlocking));
    for (int k = 0; k < sbn_program::kBranches; ++k)
        SBN_CUDA_P(cudaStreamCreateWithFlags(&P->branch[k], cudaStreamNonBlocking));
    P->step_done.resize(P->steps.size() + 1);
    for (auto &e : P->step_done) SBN_CUDA_P(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    if (n_table_floats > 0) {
        // All setup traffic goes through the program's own (non-blocking) stream and is
        // synchronised below: a NULL-stream cudaMemcpy from pageable memory may return before
        // the DMA lands and would not be ordered with later work on P->stream.
        SBN_CUDA_P(cudaMalloc(&P->d_tables, static_cast<size_t>(n_table_floats) * elem));
        SBN_CUDA_P(cudaMemcpyAsync(P->d_tables, tables, static_cast<size_t>(n_table_floats) * elem,
                                   cudaMemcpyHostToDevice, P->stream));
    }
    // evidence-independent scratch: one allocation, 256-byte aligned sub-buffers
    int64_t shared_floats = 0;
    for (Slot &s : P->slots)
        if (!s.batched) shared_floats += round_up(s.padded, 64);
    if (shared_floats > 0) {
        SBN_CUDA_P(cudaMalloc(&P->d_shared, static_cast<size_t>(shared_floats) * elem));
        SBN_CUDA_P(cudaMemsetAsync(P->d_shared, 0, static_cast<size_t>(shared_floats) * elem, P->stream));
        int64_t off = 0;
        for (Slot &s : P->slots)
            if (!s.batched) {
                s.ptr = reinterpret_cast<float *>(reinterpret_cast<char *>(P->d_shared) + off * elem);
                off += round_up(s.padded, 64);
            }
    }
    {
        std::vector<int32_t> &tile_words = P->h_tile_words;  // kept: sbn_chain_bind derives its byte tables from them
        tile_words.clear();
        plan_tiles(P, &tile_words);
        if (!tile_words.empty()) {
            SBN_CUDA_P(cudaMalloc(&P->d_tile_off, tile_words.size() * 4));
            SBN_CUDA_P(cudaMemcpyAsync(P->d_tile_off, tile_words.data(), tile_words.size() * 4,
                                       cudaMemcpyHostToDevice, P->stream));
        }
        SBN_CUDA_P(cudaStreamSynchronize(P->stream));
        // The on-chip segments and paired steps assume every intermediate has ONE consumer; the factors of the
        // other kinds' programs feed several launches, so they run on the classic per-step launches.
        // (nor do the likelihood slots of soft evidence fit them: no step writes those)
        if (P->kind == kPosterior && P->soft.empty()) sbn_chain_plan(P);
    }
    if (!P->soft.empty()) {
        // the pack's descriptors: (row offset of the slot in the batched arena, card) per likelihood
        P->use_tma = false;  // the TMA pipeline kernel is not planned for soft programs either
        std::vector<int32_t> desc;
        for (const auto &sv : P->soft) {
            int64_t off = 0;
            for (int s = 0; s < sv.first; ++s)
                if (P->slots[s].batched) off += P->slots[s].size;
            desc.push_back(static_cast<int32_t>(off));
            desc.push_back(sv.second);
        }
        SBN_CUDA_P(cudaMalloc(&P->d_soft, desc.size() * 4));
        SBN_CUDA_P(cudaMemcpyAsync(P->d_soft, desc.data(), desc.size() * 4, cudaMemcpyHostToDevice, P->stream));
        SBN_CUDA_P(cudaStreamSynchronize(P->stream));
    }
    {
        // opt every step-kernel instantiation into SBN_SMEM_BUDGET of dynamic shared memory
        // (once per device and process)
        static bool done[64] = {false};
        if (device < 64 && !done[device]) {
            SBN_CUDA_P(sbn_batched_set_attrs());
            SBN_CUDA_P(set_tiled_attrs());
            SBN_CUDA_P(sbn_chain_set_attrs());
            SBN_CUDA_P(sbn_tma_set_attrs());
            SBN_CUDA_P(sbn_join_set_attrs());
            SBN_CUDA_P(sbn_triple_rows_set_attrs());
            SBN_CUDA_P(sbn_contract_set_attrs());
            SBN_CUDA_P(sbn_marginal_set_attrs());
            SBN_CUDA_P(sbn_count_set_attrs());
            SBN_CUDA_P(sbn_deriv_set_attrs());
            SBN_CUDA_P(sbn_joint_set_attrs());
            SBN_CUDA_P(sbn_sample_set_attrs());
            SBN_CUDA_P(sbn_argmax_set_attrs());
            SBN_CUDA_P(sbn_batched_logdomain_set_attrs());
            done[device] = true;
        }
    }
    if (P->kind == kCounts || P->kind == kGrad) {
        // the count table; the largest step's per-warp partial tables (count_grid caps them) are sized here and
        // allocated by each counts call only for its duration, so idle programs hold no partial tables
        for (const StepDesc &st : P->steps)
            if (st.kind == 3)
                P->partial_doubles = std::max<int64_t>(P->partial_doubles, count_grid(P, st, INT32_MAX) * SBN_COUNT_WARPS * st.span);
        SBN_CUDA_P(cudaMalloc(&P->d_counts, static_cast<size_t>(P->n_counts) * 8));
    }
#undef SBN_CUDA_P
    rc = run_table_steps(P);
    if (rc != SBN_OK) return bail(rc);
    {
        // pairs multiply the tables of two steps on the host: needs the outputs of the table steps above
        cudaError_t e = P->kind == kPosterior ? sbn_pair_plan(P) : cudaSuccess;
        if (e != cudaSuccess) return bail(fail(SBN_E_CUDA, "planning the paired steps failed: %s", cudaGetErrorString(e)));
    }
    *out = P;
    return SBN_OK;
}

int sbn_program_create(int device, const int32_t *words, int64_t n_words, const float *tables, int64_t n_table_floats,
                       sbn_program **out) {
    return create_common(device, words, n_words, tables, n_table_floats, false, out);
}

int sbn_program_create_f64(int device, const int32_t *words, int64_t n_words, const double *tables,
                           int64_t n_table_doubles, sbn_program **out) {
    return create_common(device, words, n_words, tables, n_table_doubles, true, out);
}

void sbn_program_destroy(sbn_program *P) {
    if (!P) return;
    cudaSetDevice(P->device);
    free_scratch(P);
    sbn_chain_free(P);
    sbn_pair_free(P);
    cudaFree(P->d_shared);
    cudaFree(P->d_counts);
    cudaFree(P->d_drawn);
    cudaFree(P->d_sample_args);
    cudaFree(P->d_soft);
    cudaFree(P->d_tile_off);
    cudaFree(P->d_tables);
    if (P->stream) cudaStreamDestroy(P->stream);
    for (auto &b : P->branch)
        if (b) cudaStreamDestroy(b);
    for (auto &e : P->step_done)
        if (e) cudaEventDestroy(e);
    for (auto &e : P->pipe_events)
        if (e) cudaEventDestroy(e);
    delete P;
}

int sbn_program_reserve(sbn_program *P, int64_t max_rows) {
    if (!P) return fail(SBN_E_INVALID, "null program");
    if (max_rows <= 0) return fail(SBN_E_INVALID, "max_rows must be positive");
    if (P->mode == 0) max_rows = 1;
    if (max_rows <= P->reserved_rows) return SBN_OK;
    SBN_CUDA(cudaSetDevice(P->device));
    SBN_CUDA(cudaStreamSynchronize(P->stream));
    free_scratch(P);
    const int64_t elem = P->f64 ? 8 : 4;
    // (+ a soft program's staged likelihoods and sum log(max))
    const int64_t per_row = batched_floats_per_row(P) * elem + P->n_ev + static_cast<int64_t>(P->Q) * elem + elem +
                            (P->soft.empty() ? 0 : P->n_lik * static_cast<int64_t>(lik_elem(P)) + 8) +
                            (P->kind == kGrad ? 8 : 0);  // (+ a gradient program's staged weights)
    size_t free_b = 0, total_b = 0;
    SBN_CUDA(cudaMemGetInfo(&free_b, &total_b));
    const int64_t budget = static_cast<int64_t>(free_b * 0.85);
    int64_t rows = max_rows;
    if (per_row > 0 && round_up(rows, 32) * per_row > budget) rows = (budget / per_row) / 32 * 32;
    if (rows <= 0)
        return fail(SBN_E_NOMEM, "one evidence row needs %lld bytes of scratch; %lld free", (long long)per_row,
                    (long long)free_b);
    const int64_t ld = round_up(rows, 32);
    const int64_t arena = batched_floats_per_row(P) * ld;
    if (arena > 0) {
        cudaError_t e = cudaMalloc(&P->d_arena, static_cast<size_t>(arena) * elem);
        if (e != cudaSuccess) {
            cudaGetLastError();
            return fail(SBN_E_NOMEM, "cudaMalloc of %lld scratch bytes failed: %s", (long long)(arena * elem),
                        cudaGetErrorString(e));
        }
        int64_t off = 0;
        for (Slot &s : P->slots)
            if (s.batched) {
                s.ptr = reinterpret_cast<float *>(reinterpret_cast<char *>(P->d_arena) + off * elem);
                off += s.size * ld;
            }
    }
    if (P->n_ev > 0) {
        SBN_CUDA(cudaMalloc(&P->d_ev, static_cast<size_t>(P->n_ev) * ld));
        SBN_CUDA(cudaMemsetAsync(P->d_ev, 0, static_cast<size_t>(P->n_ev) * ld, P->stream));
    }
    SBN_CUDA(cudaMalloc(&P->d_out, static_cast<size_t>(P->Q) * ld * (P->f64 ? 8 : 4)));
    SBN_CUDA(cudaMalloc(&P->d_total, static_cast<size_t>(ld) * (P->f64 ? 8 : 4)));
    if (!P->soft.empty()) {
        SBN_CUDA(cudaMalloc(&P->d_lik, static_cast<size_t>(ld) * P->n_lik * lik_elem(P)));
        SBN_CUDA(cudaMalloc(&P->d_log_max, static_cast<size_t>(ld) * 8));
    }
    if (P->kind == kGrad) SBN_CUDA(cudaMalloc(&P->d_weight, static_cast<size_t>(ld) * 8));
    SBN_CUDA(cudaStreamSynchronize(P->stream));  // the memset must not race a caller's stream
    P->reserved_rows = rows;
    P->ld = ld;
    SBN_CUDA(sbn_chain_bind(P));  // segment descriptors point into the new arena
    return SBN_OK;
}

int sbn_program_run_device(sbn_program *P, const uint8_t *d_ev, int64_t ld_ev, int64_t n_rows, float *d_out,
                           int64_t ld_out, void *stream_) {
    int rc = check_run_args(P, d_ev, ld_ev, n_rows, d_out, ld_out);
    if (rc != SBN_OK) return rc;
    if (P->f64) return fail(SBN_E_INVALID, "float64 programs only run through sbn_program_run_host_f64");
    rc = reserve_rows(P, n_rows);
    if (rc != SBN_OK) return rc;
    if (n_rows > P->reserved_rows)
        return fail(SBN_E_NOMEM, "n_rows %lld exceeds the %lld rows of scratch that fit the device; use the host path "
                    "(it runs in chunks) or smaller batches", (long long)n_rows, (long long)P->reserved_rows);
    return run_rows(P, d_ev, ld_ev, n_rows, d_out, ld_out, static_cast<cudaStream_t>(stream_));
}

int sbn_program_run_host(sbn_program *P, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, float *out, int64_t ld_out) {
    HostCall c(kPosterior, false, ev, ld_ev, n_rows);
    c.out = out, c.ld_out = ld_out;
    return host_call(P, c);
}

int sbn_program_run_host_f64(sbn_program *P, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, double *out,
                             int64_t ld_out) {
    HostCall c(kPosterior, true, ev, ld_ev, n_rows);
    c.out = out, c.ld_out = ld_out;
    return host_call(P, c);
}

int sbn_program_evidence_host(sbn_program *P, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, float *prob) {
    HostCall c(kPosterior, false, ev, ld_ev, n_rows);
    c.prob = prob;
    return host_call(P, c);
}

int sbn_program_evidence_host_f64(sbn_program *P, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, double *prob) {
    HostCall c(kPosterior, true, ev, ld_ev, n_rows);
    c.prob = prob;
    return host_call(P, c);
}

// A posterior or marginals program with soft evidence: the pack fills the likelihood slots inside each chunk's run
// (captured graph or not); with `log_evidence`, log P(e, lik) = log(normaliser) + sum log(max).  Never pipelined.
int sbn_program_run_soft_host(sbn_program *P, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, const float *lik,
                              int64_t ld_lik, int lik_on_device, float *out, int64_t ld_out, double *log_evidence) {
    HostCall c(kPosterior, false, ev, ld_ev, n_rows);
    c.soft = true, c.lik = lik, c.ld_lik = ld_lik, c.lik_on_device = lik_on_device;
    c.out = out, c.ld_out = ld_out, c.log_prob = log_evidence;
    return host_call(P, c);
}

int sbn_program_run_soft_host_f64(sbn_program *P, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, const double *lik,
                                  int64_t ld_lik, int lik_on_device, double *out, int64_t ld_out, double *log_evidence) {
    HostCall c(kPosterior, true, ev, ld_ev, n_rows);
    c.soft = true, c.lik = lik, c.ld_lik = ld_lik, c.lik_on_device = lik_on_device;
    c.out = out, c.ld_out = ld_out, c.log_prob = log_evidence;
    return host_call(P, c);
}

int sbn_program_counts_soft_host(sbn_program *P, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, const float *lik,
                                 int64_t ld_lik, int lik_on_device, double *counts, int64_t n_counts, float *prob,
                                 double *log_evidence) {
    HostCall c(kCounts, false, ev, ld_ev, n_rows);
    c.soft = true, c.lik = lik, c.ld_lik = ld_lik, c.lik_on_device = lik_on_device;
    c.counts = counts, c.n_counts = n_counts, c.prob = prob, c.log_prob = log_evidence;
    return host_call(P, c);
}

int sbn_program_counts_soft_host_f64(sbn_program *P, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, const double *lik,
                                     int64_t ld_lik, int lik_on_device, double *counts, int64_t n_counts, double *prob,
                                     double *log_evidence) {
    HostCall c(kCounts, true, ev, ld_ev, n_rows);
    c.soft = true, c.lik = lik, c.ld_lik = ld_lik, c.lik_on_device = lik_on_device;
    c.counts = counts, c.n_counts = n_counts, c.prob = prob, c.log_prob = log_evidence;
    return host_call(P, c);
}

int sbn_program_counts_host(sbn_program *P, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, double *counts, int64_t n_counts,
                            float *prob) {
    HostCall c(kCounts, false, ev, ld_ev, n_rows);
    c.counts = counts, c.n_counts = n_counts, c.prob = prob;
    return host_call(P, c);
}

int sbn_program_counts_host_f64(sbn_program *P, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, double *counts,
                                int64_t n_counts, double *prob) {
    HostCall c(kCounts, true, ev, ld_ev, n_rows);
    c.counts = counts, c.n_counts = n_counts, c.prob = prob;
    return host_call(P, c);
}

// A gradient call: codes, likelihoods (when the program has soft variables) and, backward, the row weights are
// staged or read in place on the device; the forward run issues the upward closure of P(observed) only.  Out:
// P(observed, lik / max) and log P(observed, lik) [n_rows] (forward, both optional); backward the weighted counts
// added into `counts`, the derivative readouts [n_lik][ld_deriv] and P(observed, lik / max) (optional).
int sbn_program_grad_forward_host(sbn_program *P, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, const float *lik,
                                  int64_t ld_lik, int lik_on_device, float *prob, double *log_prob) {
    HostCall c(kGrad, false, ev, ld_ev, n_rows);
    c.lik = lik, c.ld_lik = ld_lik, c.lik_on_device = lik_on_device, c.prob = prob, c.log_prob = log_prob;
    return host_call(P, c);
}

int sbn_program_grad_forward_host_f64(sbn_program *P, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, const double *lik,
                                      int64_t ld_lik, int lik_on_device, double *prob, double *log_prob) {
    HostCall c(kGrad, true, ev, ld_ev, n_rows);
    c.lik = lik, c.ld_lik = ld_lik, c.lik_on_device = lik_on_device, c.prob = prob, c.log_prob = log_prob;
    return host_call(P, c);
}

int sbn_program_grad_backward_host(sbn_program *P, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, const float *lik,
                                   int64_t ld_lik, int lik_on_device, const double *weights, int weights_on_device,
                                   double *counts, int64_t n_counts, float *deriv, int64_t ld_deriv, float *prob) {
    if (!weights) return fail(SBN_E_INVALID, "null weights");
    HostCall c(kGrad, false, ev, ld_ev, n_rows);
    c.lik = lik, c.ld_lik = ld_lik, c.lik_on_device = lik_on_device, c.weights = weights, c.weights_on_device = weights_on_device;
    c.counts = counts, c.n_counts = n_counts, c.out = deriv, c.ld_out = ld_deriv, c.prob = prob;
    return host_call(P, c);
}

int sbn_program_grad_backward_host_f64(sbn_program *P, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, const double *lik,
                                       int64_t ld_lik, int lik_on_device, const double *weights, int weights_on_device,
                                       double *counts, int64_t n_counts, double *deriv, int64_t ld_deriv, double *prob) {
    if (!weights) return fail(SBN_E_INVALID, "null weights");
    HostCall c(kGrad, true, ev, ld_ev, n_rows);
    c.lik = lik, c.ld_lik = ld_lik, c.lik_on_device = lik_on_device, c.weights = weights, c.weights_on_device = weights_on_device;
    c.counts = counts, c.n_counts = n_counts, c.out = deriv, c.ld_out = ld_deriv, c.prob = prob;
    return host_call(P, c);
}

// A joint call: codes and (when the program has soft variables) likelihoods are staged, or read in place on the
// device; each chunk's readouts [Q][ld] and P(observed) come back.
int sbn_program_joint_host(sbn_program *P, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, const float *lik,
                           int64_t ld_lik, int lik_on_device, float *out, int64_t ld_out, float *prob) {
    HostCall c(kJoint, false, ev, ld_ev, n_rows);
    c.lik = lik, c.ld_lik = ld_lik, c.lik_on_device = lik_on_device, c.out = out, c.ld_out = ld_out, c.prob = prob;
    return host_call(P, c);
}

int sbn_program_joint_host_f64(sbn_program *P, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, const double *lik,
                               int64_t ld_lik, int lik_on_device, double *out, int64_t ld_out, double *prob) {
    HostCall c(kJoint, true, ev, ld_ev, n_rows);
    c.lik = lik, c.ld_lik = ld_lik, c.lik_on_device = lik_on_device, c.out = out, c.ld_out = ld_out, c.prob = prob;
    return host_call(P, c);
}

static int set_tables_common(sbn_program *P, const void *tables, int64_t n, bool f64) {
    if (!P) return fail(SBN_E_INVALID, "null program");
    if (P->kind != kCounts && P->kind != kGrad)
        return fail(SBN_E_INVALID, "only counts and gradient programs take new tables (other programs fold table products into "
                                   "their launches)");
    if (P->f64 != f64) return fail(SBN_E_INVALID, "program precision does not match the table call");
    if (n != P->n_table_floats || (n > 0 && !tables))
        return fail(SBN_E_INVALID, "the table blob has %lld entries, not %lld", (long long)P->n_table_floats, (long long)n);
    SBN_CUDA(cudaSetDevice(P->device));
    if (n > 0)
        SBN_CUDA(cudaMemcpyAsync(P->d_tables, tables, static_cast<size_t>(n) * (f64 ? 8 : 4), cudaMemcpyHostToDevice, P->stream));
    // the evidence-independent launches read the tables once, at creation: run them again
    const int64_t launches = P->launches, setup = P->setup_launches;
    const int rc = run_table_steps(P);
    P->setup_launches += setup;
    P->launches = launches;
    if (rc != SBN_OK) return rc;
    SBN_CUDA(cudaStreamSynchronize(P->stream));
    return SBN_OK;
}

int sbn_program_set_tables(sbn_program *P, const float *tables, int64_t n_table_floats) {
    return set_tables_common(P, tables, n_table_floats, false);
}

int sbn_program_set_tables_f64(sbn_program *P, const double *tables, int64_t n_table_doubles) {
    return set_tables_common(P, tables, n_table_doubles, true);
}

// The host path of sample programs and (kMpe, one draw, no seed) of MPE and marginal MAP programs: the decoded
// codes of a chunk are the drawn-code buffer, the per-row output is P(observed) (sample) or max log P(x, e) (MPE;
// max log P(x_MAP, e) for MAP).
int sbn_program_sample_host(sbn_program *P, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, int64_t n_draws, uint64_t seed,
                            int64_t row_base, uint8_t *out, float *prob) {
    HostCall c(kSample, false, ev, ld_ev, n_rows);
    c.n_draws = n_draws, c.seed = seed, c.row_base = row_base, c.out = out, c.prob = prob;
    return host_call(P, c);
}

int sbn_program_sample_host_f64(sbn_program *P, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, int64_t n_draws,
                                uint64_t seed, int64_t row_base, uint8_t *out, double *prob) {
    HostCall c(kSample, true, ev, ld_ev, n_rows);
    c.n_draws = n_draws, c.seed = seed, c.row_base = row_base, c.out = out, c.prob = prob;
    return host_call(P, c);
}

int sbn_program_mpe_host(sbn_program *P, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, uint8_t *codes, float *log_prob) {
    HostCall c(kMpe, false, ev, ld_ev, n_rows);
    c.out = codes, c.prob = log_prob;
    return host_call(P, c);
}

int sbn_program_sample_soft_host(sbn_program *P, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, const float *lik,
                                 int64_t ld_lik, int lik_on_device, int64_t n_draws, uint64_t seed, int64_t row_base,
                                 uint8_t *out, float *prob, double *log_evidence) {
    HostCall c(kSample, false, ev, ld_ev, n_rows);
    c.soft = true, c.lik = lik, c.ld_lik = ld_lik, c.lik_on_device = lik_on_device;
    c.n_draws = n_draws, c.seed = seed, c.row_base = row_base, c.out = out, c.prob = prob, c.log_prob = log_evidence;
    return host_call(P, c);
}

int sbn_program_sample_soft_host_f64(sbn_program *P, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, const double *lik,
                                     int64_t ld_lik, int lik_on_device, int64_t n_draws, uint64_t seed, int64_t row_base,
                                     uint8_t *out, double *prob, double *log_evidence) {
    HostCall c(kSample, true, ev, ld_ev, n_rows);
    c.soft = true, c.lik = lik, c.ld_lik = ld_lik, c.lik_on_device = lik_on_device;
    c.n_draws = n_draws, c.seed = seed, c.row_base = row_base, c.out = out, c.prob = prob, c.log_prob = log_evidence;
    return host_call(P, c);
}

// The program's float32 max log P(x, e, lik / max), then the double sum log(max) added back
int sbn_program_mpe_soft_host(sbn_program *P, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, const double *lik,
                              int64_t ld_lik, int lik_on_device, uint8_t *codes, double *log_prob) {
    HostCall c(kMpe, false, ev, ld_ev, n_rows);
    c.soft = true, c.lik = lik, c.ld_lik = ld_lik, c.lik_on_device = lik_on_device, c.out = codes, c.log_prob = log_prob;
    return host_call(P, c);
}

int sbn_program_profile(sbn_program *P, const uint8_t *d_ev, int64_t ld_ev, int64_t n_rows, float *d_out,
                        int64_t ld_out, void *stream_, float *step_ms, int64_t n_step_ms) {
    int rc = check_run_args(P, d_ev, ld_ev, n_rows, d_out, ld_out);
    if (rc != SBN_OK) return rc;
    if (P->f64) return fail(SBN_E_INVALID, "profiling is for float32 programs");
    const int64_t n = static_cast<int64_t>(P->steps.size()) + 1;
    if (!step_ms || n_step_ms < n) return fail(SBN_E_INVALID, "step_ms needs %lld entries", (long long)n);
    rc = reserve_rows(P, n_rows);
    if (rc != SBN_OK) return rc;
    if (n_rows > P->reserved_rows) return fail(SBN_E_NOMEM, "n_rows exceeds the scratch that fits the device");
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    std::vector<cudaEvent_t> ev(n + 1);
    for (auto &e : ev) SBN_CUDA(cudaEventCreate(&e));
    rc = issue_all(P, d_ev, ld_ev, n_rows, d_out, ld_out, stream, ev.data());
    if (rc == SBN_OK) {
        cudaError_t e = cudaStreamSynchronize(stream);
        if (e != cudaSuccess) rc = fail(SBN_E_CUDA, "profile run failed: %s", cudaGetErrorString(e));
    }
    if (rc == SBN_OK)
        for (int64_t i = 0; i < n; ++i) cudaEventElapsedTime(&step_ms[i], ev[i], ev[i + 1]);
    for (auto &e : ev) cudaEventDestroy(e);
    return rc;
}

int sbn_program_info(const sbn_program *P, int64_t *info, int64_t n_info) {
    if (!P || !info || n_info < 8) return fail(SBN_E_INVALID, "info needs at least 8 entries");
    if (n_info >= 12) {
        int64_t covered = 0, hbm = 0, scratch = 0;
        for (const SbnSegment *seg : P->segments) {
            covered += static_cast<int64_t>(seg->steps.size());
            hbm += seg->hbm_bytes_per_row;
            scratch = std::max(scratch, seg->scratch_floats);
        }
        info[8] = chain_on(P) ? static_cast<int64_t>(P->segments.size()) : 0;
        info[9] = chain_on(P) ? covered : 0;
        info[10] = chain_on(P) ? hbm : 0;
        info[11] = scratch;
    }
    if (n_info >= 14) {
        int64_t saved = 0;
        for (const SbnPair *pr : P->pairs) saved += 8 * P->steps[pr->step1].n_out;  // one fp32 write + one read per entry
        info[12] = pair_on(P) ? static_cast<int64_t>(P->pairs.size()) : 0;
        info[13] = pair_on(P) ? saved : 0;
    }
    info[0] = P->Q;
    info[1] = P->n_ev;
    info[2] = static_cast<int64_t>(P->steps.size());
    info[3] = batched_floats_per_row(P);
    info[4] = P->reserved_rows;
    info[5] = P->launches;
    info[6] = P->mode;
    int64_t shared = 0;
    for (const Slot &s : P->slots)
        if (!s.batched) shared += s.size;
    info[7] = shared;
    return SBN_OK;
}

int sbn_program_step_roles(const sbn_program *P, int32_t *roles, int64_t n_roles) {
    if (!P || !roles || n_roles < static_cast<int64_t>(P->steps.size())) return fail(SBN_E_INVALID, "roles needs n_steps entries");
    int first_kind = 0;
    bool second_follows = false;
    for (size_t i = 0; i < P->steps.size(); ++i) {
        const StepDesc &st = P->steps[i];
        if (P->mode != 1 || hoisted(P, st)) {
            roles[i] = 0;
            continue;
        }
        roles[i] = 1;
        if (chain_on(P) && P->seg_first[i] != -1) {
            roles[i] = 6;
            continue;
        }
        int pair = pair_on(P) ? P->pair_first[i] : -1;
        if (pair == -2 && !second_follows) pair = -1;
        second_follows = false;
        if (pair == -2) roles[i] = first_kind == 1 ? 5 : 3;
        if (pair >= 0 && sbn_pair_fits(P, *P->pairs[pair])) {
            first_kind = P->pairs[pair]->kind;
            roles[i] = first_kind == 1 ? 4 : 2;
            second_follows = true;
        }
    }
    return SBN_OK;
}

int sbn_program_set_graph(sbn_program *P, int enabled) {
    if (!P) return fail(SBN_E_INVALID, "null program");
    P->use_graph = enabled != 0;
    P->use_branches = enabled == 3;
    drop_graphs(P);
    return SBN_OK;
}

int sbn_program_set_tiled(sbn_program *P, int enabled) {
    if (!P) return fail(SBN_E_INVALID, "null program");
    drop_graphs(P);
    P->use_tiled = enabled != 0;
    P->use_preload = enabled != 4;
    P->use_slab = enabled != 5;
    if (enabled == 8) P->use_tma = false;
    if (enabled == 9) P->use_tma = P->soft.empty();  // not planned for soft-evidence programs
    if (enabled == 6) P->use_chain = false;
    if (enabled == 7) P->use_chain = true;
    if (enabled == 10) P->use_pair = false;
    if (enabled == 11) P->use_pair = true;
    return SBN_OK;
}

int sbn_host_alloc(void **ptr, int64_t bytes) {
    if (!ptr || bytes <= 0) return fail(SBN_E_INVALID, "bad host allocation request");
    SBN_CUDA(cudaHostAlloc(ptr, static_cast<size_t>(bytes), cudaHostAllocDefault));
    return SBN_OK;
}

int sbn_host_free(void *ptr) {
    if (ptr) SBN_CUDA(cudaFreeHost(ptr));
    return SBN_OK;
}

}  // extern "C"

// ================================================================== Gibbs sampling
struct sbn_sampler {
    int device = 0;
    int n_vars = 0, n_query = 0, n_ev = 0, n_cycle = 0, Q = 0;
    int32_t *d_ints = nullptr;  // one allocation for every int array
    float *d_tables = nullptr;
    const int32_t *card = nullptr, *cpt_off = nullptr, *par_ptr = nullptr, *par_idx = nullptr, *par_stride = nullptr,
                  *chi_ptr = nullptr, *chi_idx = nullptr, *chi_stride = nullptr, *cycle = nullptr, *query = nullptr,
                  *ev_var = nullptr, *prog = nullptr, *flat = nullptr;
    int prog_words = 0, flat_words = 0;
    int64_t table_floats = 0;
    int max_card = 1;
    std::vector<int32_t> h_cycle;   // host copies for sbn_gibbs_conditional
    std::vector<int32_t> h_card;
    uint8_t *d_ev = nullptr;
    float *d_out = nullptr;
    int64_t cap = 0;
    cudaStream_t stream = nullptr;
    int64_t launches = 0;
};

extern "C" {

int sbn_gibbs_create(int device, int32_t n_vars, const int32_t *card, const int32_t *par_ptr, const int32_t *par_idx,
                     const int32_t *cpt_off, const float *tables, int64_t n_table_floats, int32_t n_query,
                     const int32_t *query, int32_t n_ev, const int32_t *ev_vars, int32_t n_cycle, const int32_t *cycle,
                     sbn_sampler **out) {
    if (!card || !par_ptr || !cpt_off || !tables || !query || !cycle || !out || (n_ev > 0 && !ev_vars))
        return fail(SBN_E_INVALID, "null argument");
    *out = nullptr;
    if (n_vars <= 0 || n_query <= 0 || n_cycle <= 0 || n_ev < 0) return fail(SBN_E_INVALID, "bad counts");
    const int n_par = par_ptr[n_vars];
    if (n_par > 0 && !par_idx) return fail(SBN_E_INVALID, "null parent list");
    // parents precede children (ids are topological) and every CPT lies inside the blob
    std::vector<int32_t> par_stride(n_par), chi_ptr(n_vars + 1, 0), chi_idx(n_par), chi_stride(n_par);
    for (int v = 0; v < n_vars; ++v) {
        if (card[v] < 1 || card[v] > SBN_GIBBS_MAX_CARD) return fail(SBN_E_INVALID, "variable %d has %d states (max %d)", v, card[v], SBN_GIBBS_MAX_CARD);
        if (par_ptr[v] > par_ptr[v + 1]) return fail(SBN_E_INVALID, "bad parent CSR");
        int64_t stride = card[v];
        for (int k = par_ptr[v + 1] - 1; k >= par_ptr[v]; --k) {
            const int pv = par_idx[k];
            if (pv < 0 || pv >= v) return fail(SBN_E_INVALID, "variable ids must be topological (parent %d of %d)", pv, v);
            par_stride[k] = static_cast<int32_t>(stride);
            stride *= card[pv];
            if (stride >= (1LL << 31)) return fail(SBN_E_INVALID, "CPT of variable %d is too large", v);
            chi_ptr[pv + 1]++;
        }
        if (cpt_off[v] < 0 || cpt_off[v] + stride > n_table_floats) return fail(SBN_E_INVALID, "CPT %d outside the table blob", v);
    }
    for (int v = 0; v < n_vars; ++v) chi_ptr[v + 1] += chi_ptr[v];
    {
        std::vector<int32_t> fill(chi_ptr.begin(), chi_ptr.end() - 1);
        for (int v = 0; v < n_vars; ++v)
            for (int k = par_ptr[v]; k < par_ptr[v + 1]; ++k) {
                const int pv = par_idx[k];
                chi_idx[fill[pv]] = v;
                chi_stride[fill[pv]] = par_stride[k];
                fill[pv]++;
            }
    }
    int64_t Q = 1;
    for (int k = 0; k < n_query; ++k) {
        if (query[k] < 0 || query[k] >= n_vars) return fail(SBN_E_INVALID, "query id out of range");
        Q *= card[query[k]];
        if (Q > 4096) return fail(SBN_E_INVALID, "more than 4096 joint query states");
    }
    for (int k = 0; k < n_ev; ++k)
        if (ev_vars[k] < 0 || ev_vars[k] >= n_vars) return fail(SBN_E_INVALID, "evidence id out of range");
    for (int k = 0; k < n_cycle; ++k)
        if (cycle[k] < 0 || cycle[k] >= n_vars) return fail(SBN_E_INVALID, "cycle id out of range");
    // the resampling cycle compiled into one record per position (layout: sbn_gibbs.cuh)
    std::vector<int32_t> prog(n_cycle, 0);
    int max_card = 1;
    for (int i = 0; i < n_cycle; ++i) {
        const int v = cycle[i];
        prog[i] = static_cast<int32_t>(prog.size());
        max_card = std::max(max_card, card[v]);
        const int np = par_ptr[v + 1] - par_ptr[v], nc = chi_ptr[v + 1] - chi_ptr[v];
        if (np > 255 || nc > 255 || v > 0xffff) return fail(SBN_E_INVALID, "variable %d has too many parents / children for the sampler", v);
        prog.push_back(v | card[v] << 16);
        prog.push_back(cpt_off[v]);
        prog.push_back(np | nc << 8);
        for (int k = par_ptr[v]; k < par_ptr[v + 1]; ++k) {
            prog.push_back(par_idx[k]);
            prog.push_back(par_stride[k]);
        }
        for (int k = chi_ptr[v]; k < chi_ptr[v + 1]; ++k) {
            const int ch = chi_idx[k];
            prog.push_back(cpt_off[ch]);
            prog.push_back(ch);
            prog.push_back(chi_stride[k]);
            int others = 0;
            for (int j = par_ptr[ch]; j < par_ptr[ch + 1]; ++j) others += par_idx[j] != v;
            prog.push_back(others);
            for (int j = par_ptr[ch]; j < par_ptr[ch + 1]; ++j)
                if (par_idx[j] != v) {
                    prog.push_back(par_idx[j]);
                    prog.push_back(par_stride[j]);
                }
        }
    }
    // the straight-line variant (sbn_gibbs_flat_kernel): fixed-size records, when the network is small enough
    std::vector<int32_t> flat;
    bool flat_ok = max_card <= 8 && n_query <= 4 && n_vars < 0xffff;
    // The straight-line kernel multiplies its <= 5 factors without the rescaling of sbn_gibbs_weights.
    // It takes a cycle position only when the product of the smallest non-zero entries of those
    // tables stays far above float32's smallest normal, so that no weight can underflow and both
    // kernels pick the same states.
    std::vector<double> min_entry(n_vars, 1.0);
    if (flat_ok)
        for (int v = 0; v < n_vars; ++v) {
            int64_t size = card[v];
            for (int k = par_ptr[v]; k < par_ptr[v + 1]; ++k) size *= card[par_idx[k]];
            for (int64_t e = 0; e < size; ++e) {
                const float t = tables[cpt_off[v] + e];
                if (t > 0.f) min_entry[v] = std::min(min_entry[v], static_cast<double>(t));
            }
        }
    const int32_t ones_off = static_cast<int32_t>(n_table_floats);  // a 1.0f appended to the table blob
    for (int i = 0; i < n_cycle && flat_ok; ++i) {
        const int v = cycle[i];
        const int np = par_ptr[v + 1] - par_ptr[v], nc = chi_ptr[v + 1] - chi_ptr[v];
        if (np > SBN_GF_TERMS || nc > SBN_GF_GROUPS - 1) { flat_ok = false; break; }
        double smallest = min_entry[v];
        for (int k = chi_ptr[v]; k < chi_ptr[v + 1]; ++k) smallest *= min_entry[chi_idx[k]];
        if (smallest < 1e-30) { flat_ok = false; break; }
        std::vector<int32_t> rec(SBN_GF_WORDS, 0);
        rec[0] = v | card[v] << 16;
        auto group = [&](int g) { return rec.data() + 2 + g * (2 + 2 * SBN_GF_TERMS); };
        for (int g = 0; g < SBN_GF_GROUPS; ++g) {  // padding: the constant 1.0, terms on the dummy state
            int32_t *gw = group(g);
            gw[0] = ones_off;
            gw[1] = 0;
            for (int k = 0; k < SBN_GF_TERMS; ++k) { gw[2 + 2 * k] = n_vars; gw[3 + 2 * k] = 0; }
        }
        int32_t *g0 = group(0);
        g0[0] = cpt_off[v];
        g0[1] = 1;
        for (int k = par_ptr[v], t = 0; k < par_ptr[v + 1]; ++k, ++t) { g0[2 + 2 * t] = par_idx[k]; g0[3 + 2 * t] = par_stride[k]; }
        for (int k = chi_ptr[v], g = 1; k < chi_ptr[v + 1] && flat_ok; ++k, ++g) {
            const int ch = chi_idx[k];
            int32_t *gw = group(g);
            gw[0] = cpt_off[ch];
            gw[1] = chi_stride[k];
            int t = 0;
            gw[2] = ch;  // the child's own state, stride 1
            gw[3] = 1;
            ++t;
            for (int j = par_ptr[ch]; j < par_ptr[ch + 1]; ++j)
                if (par_idx[j] != v) {
                    if (t >= SBN_GF_TERMS) { flat_ok = false; break; }
                    gw[2 + 2 * t] = par_idx[j];
                    gw[3 + 2 * t] = par_stride[j];
                    ++t;
                }
        }
        flat.insert(flat.end(), rec.begin(), rec.end());
    }
    if (flat_ok) {
        const size_t need = flat.size() * 4 + ((static_cast<size_t>(n_table_floats) + 1 + 3) / 4) * 16 +
                            ((static_cast<size_t>(n_vars + 1) * SBN_GIBBS_CHAINS + 15) / 16) * 16 + static_cast<size_t>(Q) * SBN_GIBBS_CHAINS * 4;
        if (need > 100 * 1024) flat_ok = false;  // two CTAs per SM
    }
    const size_t smem_min = ((prog.size() + 3) / 4) * 16 + ((static_cast<size_t>(n_vars) * SBN_GIBBS_CHAINS + 15) / 16) * 16 +
                            static_cast<size_t>(Q) * SBN_GIBBS_CHAINS * 4;
    if (smem_min > 200 * 1024) return fail(SBN_E_INVALID, "chain state needs %zu bytes of shared memory per CTA", smem_min);

    int n_dev = 0;
    if (cudaGetDeviceCount(&n_dev) != cudaSuccess || n_dev == 0) return fail(SBN_E_NODEVICE, "no CUDA device available");
    if (device < 0 || device >= n_dev) return fail(SBN_E_NODEVICE, "device %d out of range", device);
    sbn_sampler *S = new sbn_sampler();
    S->device = device;
    S->n_vars = n_vars;
    S->n_query = n_query;
    S->n_ev = n_ev;
    S->n_cycle = n_cycle;
    S->Q = static_cast<int>(Q);
    auto bail = [&](int code) {
        sbn_gibbs_destroy(S);
        return code;
    };
#define SBN_CUDA_S(call)                                                                                   \
    do {                                                                                                   \
        cudaError_t e_ = (call);                                                                           \
        if (e_ != cudaSuccess) return bail(fail(SBN_E_CUDA, "%s failed: %s", #call, cudaGetErrorString(e_))); \
    } while (0)
    SBN_CUDA_S(cudaSetDevice(device));
    SBN_CUDA_S(cudaStreamCreateWithFlags(&S->stream, cudaStreamNonBlocking));
    std::vector<int32_t> ints;
    auto put = [&](const int32_t *src, size_t n) {
        const size_t at = ints.size();
        ints.insert(ints.end(), src, src + n);
        return at;
    };
    const size_t o_card = put(card, n_vars), o_off = put(cpt_off, n_vars), o_pp = put(par_ptr, n_vars + 1),
                 o_pi = put(par_idx ? par_idx : card, n_par), o_ps = put(par_stride.data(), n_par),
                 o_cp = put(chi_ptr.data(), n_vars + 1), o_ci = put(chi_idx.data(), n_par),
                 o_cs = put(chi_stride.data(), n_par), o_cy = put(cycle, n_cycle), o_q = put(query, n_query),
                 o_ev = put(ev_vars ? ev_vars : card, n_ev), o_prog = put(prog.data(), prog.size());
    while (ints.size() % 4) ints.push_back(0);  // the flat records are read as int4
    const size_t o_flat = put(flat.data(), flat_ok ? flat.size() : 0);
    SBN_CUDA_S(cudaMalloc(&S->d_ints, ints.size() * 4 + 4));
    SBN_CUDA_S(cudaMemcpyAsync(S->d_ints, ints.data(), ints.size() * 4, cudaMemcpyHostToDevice, S->stream));
    SBN_CUDA_S(cudaMalloc(&S->d_tables, static_cast<size_t>(n_table_floats + 1) * 4));
    SBN_CUDA_S(cudaMemcpyAsync(S->d_tables, tables, static_cast<size_t>(n_table_floats) * 4, cudaMemcpyHostToDevice, S->stream));
    {
        static const float one = 1.0f;  // the padding entry of the straight-line records
        SBN_CUDA_S(cudaMemcpyAsync(S->d_tables + n_table_floats, &one, 4, cudaMemcpyHostToDevice, S->stream));
    }
    SBN_CUDA_S(cudaStreamSynchronize(S->stream));
    S->card = S->d_ints + o_card;
    S->cpt_off = S->d_ints + o_off;
    S->par_ptr = S->d_ints + o_pp;
    S->par_idx = S->d_ints + o_pi;
    S->par_stride = S->d_ints + o_ps;
    S->chi_ptr = S->d_ints + o_cp;
    S->chi_idx = S->d_ints + o_ci;
    S->chi_stride = S->d_ints + o_cs;
    S->cycle = S->d_ints + o_cy;
    S->query = S->d_ints + o_q;
    S->ev_var = S->d_ints + o_ev;
    S->prog = S->d_ints + o_prog;
    S->prog_words = static_cast<int>(prog.size());
    S->flat = flat_ok ? S->d_ints + o_flat : nullptr;
    S->flat_words = flat_ok ? static_cast<int>(flat.size()) : 0;
    SBN_CUDA_S(cudaFuncSetAttribute(sbn_gibbs_flat_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
    S->table_floats = n_table_floats;
    S->max_card = max_card;
    S->h_cycle.assign(cycle, cycle + n_cycle);
    S->h_card.assign(card, card + n_vars);
    SBN_CUDA_S(cudaFuncSetAttribute(sbn_gibbs_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    SBN_CUDA_S(cudaFuncSetAttribute(sbn_gibbs_kernel<SBN_GIBBS_MAX_CARD>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    SBN_CUDA_S(cudaFuncSetAttribute(sbn_forward_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
#undef SBN_CUDA_S
    *out = S;
    return SBN_OK;
}

void sbn_gibbs_destroy(sbn_sampler *S) {
    if (!S) return;
    cudaSetDevice(S->device);
    cudaFree(S->d_ints);
    cudaFree(S->d_tables);
    cudaFree(S->d_ev);
    cudaFree(S->d_out);
    if (S->stream) cudaStreamDestroy(S->stream);
    delete S;
}

static int sampler_run(sbn_sampler *S, int algo, const uint8_t *ev, int64_t ld_ev, int64_t n_chains, int64_t n_iterations,
                       uint64_t seed, float *out, int64_t ld_out) {
    if (!S || !out) return fail(SBN_E_INVALID, "null argument");
    const bool force_generic = algo == 3;  // Gibbs through the generic kernel (cross-check of the straight-line one)
    if (algo == 3) algo = 0;
    if (algo < 0 || algo > 2) return fail(SBN_E_INVALID, "unknown sampling algorithm %d", algo);
    if (n_chains <= 0 || n_iterations <= 0) return fail(SBN_E_INVALID, "n_chains and n_iterations must be positive");
    if (S->n_ev > 0 && (!ev || (S->n_ev > 1 && ld_ev < n_chains))) return fail(SBN_E_INVALID, "bad evidence");
    if (S->Q > 1 && ld_out < n_chains) return fail(SBN_E_INVALID, "ld_out < n_chains");
    SBN_CUDA(cudaSetDevice(S->device));
    if (n_chains > S->cap) {
        cudaFree(S->d_ev);
        cudaFree(S->d_out);
        S->d_ev = nullptr;
        S->d_out = nullptr;
        if (S->n_ev > 0) SBN_CUDA(cudaMalloc(&S->d_ev, static_cast<size_t>(S->n_ev) * n_chains));
        SBN_CUDA(cudaMalloc(&S->d_out, static_cast<size_t>(S->Q) * n_chains * 4));
        S->cap = n_chains;
    }
    if (S->n_ev > 0)
        SBN_CUDA(cudaMemcpy2DAsync(S->d_ev, static_cast<size_t>(n_chains), ev, static_cast<size_t>(ld_ev),
                                   static_cast<size_t>(n_chains), static_cast<size_t>(S->n_ev), cudaMemcpyHostToDevice, S->stream));
    SbnGibbs g;
    memset(&g, 0, sizeof g);
    g.n_vars = S->n_vars;
    g.n_cycle = S->n_cycle;
    g.n_query = S->n_query;
    g.Q = S->Q;
    g.n_ev = S->n_ev;
    g.card = S->card;
    g.cpt_off = S->cpt_off;
    g.par_ptr = S->par_ptr;
    g.par_idx = S->par_idx;
    g.par_stride = S->par_stride;
    g.chi_ptr = S->chi_ptr;
    g.chi_idx = S->chi_idx;
    g.chi_stride = S->chi_stride;
    g.cycle = S->cycle;
    g.query = S->query;
    g.ev_var = S->ev_var;
    g.tables = S->d_tables;
    g.ev = S->d_ev;
    g.ld_ev = n_chains;
    g.out = S->d_out;
    g.ld_out = n_chains;
    g.n_chains = n_chains;
    g.n_iterations = n_iterations;
    g.seed = seed;
    g.prog = S->prog;
    g.prog_words = S->prog_words;
    g.table_floats = static_cast<int32_t>(S->table_floats);
    static const bool flat_env = [] {
        const char *e = getenv("SOROBN_B200_GIBBS_FLAT");
        return e ? atoi(e) != 0 : true;
    }();
    if (algo == 0 && S->flat && flat_env && !force_generic) {
        g.prog = S->flat;
        g.prog_words = S->flat_words;
        g.table_floats = static_cast<int32_t>(S->table_floats + 1);
        g.tables_in_smem = 1;
        const size_t smem = static_cast<size_t>(S->flat_words) * 4 + ((static_cast<size_t>(g.table_floats) + 3) / 4) * 16 +
                            ((static_cast<size_t>(S->n_vars + 1) * SBN_GIBBS_CHAINS + 15) / 16) * 16 + static_cast<size_t>(S->Q) * SBN_GIBBS_CHAINS * 4;
        const int64_t grid = (n_chains + SBN_GIBBS_CHAINS - 1) / SBN_GIBBS_CHAINS;
        sbn_gibbs_flat_kernel<<<static_cast<unsigned>(grid), SBN_GIBBS_CHAINS, smem, S->stream>>>(g);
    } else if (algo == 0) {
        const size_t base = ((static_cast<size_t>(S->prog_words) + 3) / 4) * 16 + ((static_cast<size_t>(S->n_vars) * SBN_GIBBS_CHAINS + 15) / 16) * 16 +
                            static_cast<size_t>(S->Q) * SBN_GIBBS_CHAINS * 4;
        const size_t tab = ((static_cast<size_t>(S->table_floats) + 3) / 4) * 16;
        // every CPT in shared memory when that still leaves two CTAs per SM
        g.tables_in_smem = base + tab <= 100 * 1024 ? 1 : 0;
        const size_t smem = base + (g.tables_in_smem ? tab : 0);
        const int64_t grid = (n_chains + SBN_GIBBS_CHAINS - 1) / SBN_GIBBS_CHAINS;
        if (S->max_card <= 8) sbn_gibbs_kernel<8><<<static_cast<unsigned>(grid), SBN_GIBBS_CHAINS, smem, S->stream>>>(g);
        else sbn_gibbs_kernel<SBN_GIBBS_MAX_CARD><<<static_cast<unsigned>(grid), SBN_GIBBS_CHAINS, smem, S->stream>>>(g);
    } else {
        // one CTA per evidence row; its threads share the row's n_iterations samples
        // (per joint query state: a double sum and a uint32 count)
        const size_t smem = ((static_cast<size_t>(S->n_vars) * (SBN_GIBBS_THREADS + 1) + 15) / 16) * 16 + static_cast<size_t>(S->Q) * 12;
        if (smem > 200 * 1024) return fail(SBN_E_INVALID, "sampler state needs %zu bytes of shared memory", smem);
        sbn_forward_kernel<<<static_cast<unsigned>(n_chains), SBN_GIBBS_THREADS, smem, S->stream>>>(g, algo);
    }
    SBN_CUDA(cudaGetLastError());
    S->launches++;
    SBN_CUDA(cudaMemcpy2DAsync(out, static_cast<size_t>(ld_out) * 4, S->d_out, static_cast<size_t>(n_chains) * 4,
                               static_cast<size_t>(n_chains) * 4, static_cast<size_t>(S->Q), cudaMemcpyDeviceToHost, S->stream));
    SBN_CUDA(cudaStreamSynchronize(S->stream));
    return SBN_OK;
}

int sbn_gibbs_conditional(sbn_sampler *S, int32_t var, const uint8_t *joint, float *out) {
    if (!S || !joint || !out) return fail(SBN_E_INVALID, "null argument");
    int pos = -1;
    for (size_t i = 0; i < S->h_cycle.size(); ++i)
        if (S->h_cycle[i] == var) pos = static_cast<int>(i);
    if (pos < 0) return fail(SBN_E_INVALID, "variable %d is not in the sampler's cycle", var);
    SBN_CUDA(cudaSetDevice(S->device));
    uint8_t *d_joint = nullptr;
    float *d_w = nullptr;
    SBN_CUDA(cudaMalloc(&d_joint, static_cast<size_t>(S->n_vars)));
    SBN_CUDA(cudaMalloc(&d_w, SBN_GIBBS_MAX_CARD * sizeof(float)));
    SBN_CUDA(cudaMemcpyAsync(d_joint, joint, static_cast<size_t>(S->n_vars), cudaMemcpyHostToDevice, S->stream));
    SbnGibbs g;
    memset(&g, 0, sizeof g);
    g.card = S->card;
    g.prog = S->prog;
    g.tables = S->d_tables;
    sbn_gibbs_conditional_kernel<<<1, 32, 0, S->stream>>>(g, pos, d_joint, d_w);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess)
        e = cudaMemcpyAsync(out, d_w, static_cast<size_t>(S->h_card[var]) * sizeof(float), cudaMemcpyDeviceToHost, S->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(S->stream);
    cudaFree(d_joint);
    cudaFree(d_w);
    if (e != cudaSuccess) return fail(SBN_E_CUDA, "sbn_gibbs_conditional failed: %s", cudaGetErrorString(e));
    return SBN_OK;
}

int sbn_gibbs_run_host(sbn_sampler *S, const uint8_t *ev, int64_t ld_ev, int64_t n_chains, int64_t n_iterations,
                       uint64_t seed, float *out, int64_t ld_out) {
    return sampler_run(S, 0, ev, ld_ev, n_chains, n_iterations, seed, out, ld_out);
}

int sbn_sampler_run_host(sbn_sampler *S, int algo, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, int64_t n_iterations,
                         uint64_t seed, float *out, int64_t ld_out) {
    return sampler_run(S, algo, ev, ld_ev, n_rows, n_iterations, seed, out, ld_out);
}

}  // extern "C"
