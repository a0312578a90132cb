/*
 * sorobn_b200 -- C ABI of the H100 (sm_90a) exact-inference engine.
 *
 * This is the drop-in boundary for the exact-inference path of MaxHalford/sorobn.
 * The reference has no native layer: the whole path is Python over pandas
 * (/root/reference/sorobn/bayes_net.py).  The entry points below are what a ctypes
 * binding inside the reference's `BayesNet` would call instead of
 *
 *   - `BayesNet._variable_elimination`      bayes_net.py:739-794  (the loop)
 *   - `pointwise_mul` / `pointwise_mul_two` bayes_net.py:106-256  (factor product)
 *   - `CDTAccessor.sum_out`                 bayes_net.py:54-103   (marginalisation)
 *   - the normalisation at                  bayes_net.py:789-790
 *
 * INTEGRATION.md shows that binding.  Plain pointers and sizes only: no torch,
 * numpy or pandas types cross this line.
 *
 * A *program* is the frozen form of one `(query variables, evidence variables)`
 * pair: the CPTs involved (dense fp32 tables) and the list of fused
 * "product of k factors -> sum out one variable" steps, one kernel launch each
 * (word layout: sorobn_b200/planner.py).  Running a program on B evidence rows
 * computes B posteriors, i.e. B calls of `BayesNet.query(..., algorithm="exact")`.
 *
 * Layouts (both "column-major" over rows so that device accesses coalesce):
 *   evidence : uint8 state codes, ev[c * ld_ev + b]   c < n_ev, b < n_rows
 *   posterior: float,             out[q * ld_out + b] q < Q,    b < n_rows
 * where q enumerates the joint states of the query variables, variables sorted by
 * name and the last one varying fastest -- the row order of the reference's answer
 * (`reorder_levels(sorted(...))`, `sort_index()`; bayes_net.py:872-875).
 * A row whose evidence has probability zero yields NaN (the reference returns an
 * empty Series there).  In float32 programs a row whose normaliser is below 1e-30 is also
 * NaN: float32 underflow may have dropped addends; re-run it with a float64 program.
 *
 * Every function returns 0 on success or a negative SBN_E_* code;
 * sbn_last_error() then describes the failure (thread-local string).
 */
#ifndef SOROBN_B200_H
#define SOROBN_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SBN_ABI_VERSION 22

#define SBN_OK 0
#define SBN_E_INVALID (-1)   /* malformed program / bad argument            */
#define SBN_E_CUDA (-2)      /* CUDA runtime error (see sbn_last_error)     */
#define SBN_E_NOMEM (-3)     /* scratch does not fit the device             */
#define SBN_E_NODEVICE (-4)  /* no usable sm_90 GPU                         */

typedef struct sbn_program sbn_program;

/* Fixed limits of the step kernel (also enforced by the planner). */
#define SBN_MAX_IN 8     /* factors multiplied in one launch   */
#define SBN_MAX_AXES 20  /* variables in one output factor     */
#define SBN_MAX_EV 8     /* evidence axes gathered per factor  */

int sbn_abi_version(void);
const char *sbn_last_error(void);

/* Number of CUDA devices visible; SBN_E_NODEVICE if none. */
int sbn_device_count(int *count);

/* Compile a program for `device`: validates `words` (planner.py layout), uploads the
 * CPT tables.  Replaces the per-query factor preparation of bayes_net.py:768-776. */
int sbn_program_create(int device, const int32_t *words, int64_t n_words, const float *tables,
                       int64_t n_table_floats, sbn_program **out);
void sbn_program_destroy(sbn_program *prog);

/* Same for a program evaluated in float64: tables, scratch and the posterior are doubles.
 * Single-event ("flat", mode 0) programs are what `BayesNet.query` uses; batched ones re-run
 * the rows a float32 program flagged.  One query is launch-latency bound, so it gets the
 * reference's own precision and range (float64, bayes_net.py throughout) for free; it is
 * also the fallback for evidence rows too unlikely for float32 (see run_host below). */
int sbn_program_create_f64(int device, const int32_t *words, int64_t n_words, const double *tables,
                           int64_t n_table_doubles, sbn_program **out);

/* Allocate scratch for chunks of up to `max_rows` evidence rows (larger batches are
 * processed in chunks).  Called implicitly by the run functions when needed. */
int sbn_program_reserve(sbn_program *prog, int64_t max_rows);

/* Answer `n_rows` queries with HOST buffers: copies the evidence codes to the device,
 * runs every step, copies the posteriors back and synchronises.  This is the call that
 * replaces `BayesNet._variable_elimination` (bayes_net.py:739) for a batch of events. */
int sbn_program_run_host(sbn_program *prog, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, float *out,
                         int64_t ld_out);

/* float64 programs: flat (n_rows must be 1) or batched (the robust fallback for rows that
 * the float32 program flagged; plain kernel in double, several times slower). */
int sbn_program_run_host_f64(sbn_program *prog, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, double *out,
                             int64_t ld_out);

/* P(event) of every evidence row: the normaliser the run divides by (bayes_net.py:790).  This is
 * what `BayesNet.predict_proba` returns (bayes_net.py:934-962: the full joint, marginalised over
 * the unobserved variables and looked up at the row) without ever building the joint.  The program
 * may have no query variable at all (planner: allow_empty_query).  prob[b], b < n_rows; NaN marks
 * a row below the float32 range (re-run it with a float64 program). */
int sbn_program_evidence_host(sbn_program *prog, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, float *prob);
int sbn_program_evidence_host_f64(sbn_program *prog, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, double *prob);

/* Soft (likelihood, virtual) evidence: a posterior or marginals program planned with soft variables
 * (planner.build_plan / build_marginals_plan `soft=`) runs through these calls only, and they refuse
 * every other program.  `lik` is [n_rows][ld_lik] row-major: one column per state of every soft
 * variable (variables sorted by name, states in domain order, ld_lik >= that count), non-negative; a
 * row's posterior is P(query | e) with every P(x) weighted by prod_v lik_v(x_v), which is unchanged
 * when a variable's row is scaled.  `lik` is host memory, or device memory of the program's device
 * when `lik_on_device` is non-zero (read on the program's stream: the caller's writes must be
 * complete).  Codes and `out` are host memory, as for run_host.  `log_evidence` (double [n_rows], or
 * null; posterior programs only) receives log P(e, lik) = log sum_x P(x, e) prod_v lik_v(x_v); NaN
 * where the float32 range rule flags the row, or for a row of probability zero (an all-zero lik_v
 * makes one). */
int sbn_program_run_soft_host(sbn_program *prog, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, const float *lik,
                              int64_t ld_lik, int lik_on_device, float *out, int64_t ld_out, double *log_evidence);
int sbn_program_run_soft_host_f64(sbn_program *prog, const uint8_t *ev, int64_t ld_ev, int64_t n_rows,
                                  const double *lik, int64_t ld_lik, int lik_on_device, double *out, int64_t ld_out,
                                  double *log_evidence);

/* Expected counts (the E-step of expectation-maximisation) of a counts program
 * (planner.build_counts_plan, version 6; the run and evidence calls refuse it, and these calls refuse
 * every other program).  For every row b and every node v, P(v, parents(v) | the row's observed cells)
 * is ADDED into counts[c_offset(v) + ...]: the dense [*parents, v] arrays of the CPTs in the network's
 * order, concatenated, n_counts entries in all.  prob[b] = P(observed cells of b), or NaN for a row below
 * the float32 range (1e-30; 1e-290 for the float64 twin) or of probability zero: such a row adds nothing,
 * re-run it with a float64 program.  The rows are reduced without floating-point atomics: two calls on
 * the same device and batch give bitwise the same counts.  Large batches run in chunks. */
int sbn_program_counts_host(sbn_program *prog, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, double *counts,
                            int64_t n_counts, float *prob);
int sbn_program_counts_host_f64(sbn_program *prog, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, double *counts,
                                int64_t n_counts, double *prob);

/* Replace a counts or gradient program's table blob in place (same size and layout: planner.refresh_tables) and
 * re-run its evidence-independent launches; later runs, graph replays included, use the new values.
 * An EM loop plans once and calls this every iteration.  Other programs are refused: their paired
 * steps fold table products into coefficients built on the host. */
int sbn_program_set_tables(sbn_program *prog, const float *tables, int64_t n_table_floats);
int sbn_program_set_tables_f64(sbn_program *prog, const double *tables, int64_t n_table_doubles);

/* Exact posterior draws of a sample program (planner.build_sample_plan, version 7; the run, evidence and
 * counts calls refuse it, and these calls refuse every other program).  For every row b and draw d,
 * out[(j * n_draws + d) * n_rows + b] is the code of the j-th sampled variable (Plan.sampled), drawn from
 * P(unobserved | the row's observed cells) by backward sampling over the bucket tree.  The draws depend only
 * on (seed, row_base + b, d): Philox-4x32-10, key (seed lo, seed hi), counter (sample step, d, row lo, row hi),
 * so a batch cut into pieces run with their row_base gives the same draws, and so do two calls.
 * prob[b] = P(observed cells of b), or NaN for a row below the float32 range (1e-30; 1e-290 for the float64
 * twin) or of probability zero: its draws are meaningless, re-run it with a float64 program and the same
 * row_base + b.  Large batches run in chunks. */
int sbn_program_sample_host(sbn_program *prog, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, int64_t n_draws,
                            uint64_t seed, int64_t row_base, uint8_t *out, float *prob);
int sbn_program_sample_host_f64(sbn_program *prog, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, int64_t n_draws,
                                uint64_t seed, int64_t row_base, uint8_t *out, double *prob);

/* Most probable explanation of an MPE program (planner.build_mpe_plan, version 8; the run, evidence, counts
 * and sample calls refuse it, this call refuses every other program, and it is created in float32 only).
 * For every row b, codes[j * n_rows + b] is the code of the j-th decoded variable (Plan.sampled) in the
 * argmax over every unobserved variable jointly of P(unobserved, the row's observed cells); ties go to the
 * first joint state of a bucket (first variable fastest).  log_prob[b] = that maximum, log P(x*, e), or
 * -inf for a row whose observed cells have probability zero (its codes are meaningless).  Large batches
 * run in chunks.
 * The same call runs a marginal MAP program (planner.build_map_plan, version 9; created in float32 only):
 * the decoded variables are its MAP variables, every other unobserved variable is summed out, and
 * log_prob[b] = max over the MAP variables of log P(x_MAP, the row's observed cells). */
int sbn_program_mpe_host(sbn_program *prog, const uint8_t *ev, int64_t ld_ev, int64_t n_rows,
                         uint8_t *codes /* [n_decoded][n_rows] */, float *log_prob /* [n_rows] */);

/* Soft evidence on counts, sample, MPE and marginal MAP programs planned with soft variables
 * (planner.build_pattern_plan `soft=`): these calls run them, the calls above refuse them, and these
 * refuse a program without soft variables.  `lik`, `ld_lik` and `lik_on_device` are those of
 * sbn_program_run_soft_host; a soft variable is unobserved, with its probabilities weighted by lik.
 * Counts and sample: the outputs of sbn_program_counts_host / sbn_program_sample_host given the observed
 * cells and lik, with prob[b] = P(observed, lik / max) (every row of lik divided by its maximum, so the
 * float32 range rule keeps its meaning) and `log_evidence` (double [n_rows], or null) = log P(observed,
 * lik) = log prob[b] + sum_v log max lik_v, NaN where prob[b] is flagged.  The sample streams are those of
 * sbn_program_sample_host: the draws depend only on (seed, row_base + b, d) and the program.
 * MPE and MAP (float32 programs; the likelihood slots hold log(lik / max)): `lik` is double, so that any
 * finite scale reaches the log intact; the codes of sbn_program_mpe_host, and log_prob[b] = the program's
 * float32 maximum plus the double sum_v log max lik_v, log P(x*, e, lik) on the caller's scale; -inf for a row
 * of probability zero (an all-zero lik_v makes one). */
int sbn_program_counts_soft_host(sbn_program *prog, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, const float *lik,
                                 int64_t ld_lik, int lik_on_device, double *counts, int64_t n_counts, float *prob,
                                 double *log_evidence);
int sbn_program_counts_soft_host_f64(sbn_program *prog, const uint8_t *ev, int64_t ld_ev, int64_t n_rows,
                                     const double *lik, int64_t ld_lik, int lik_on_device, double *counts,
                                     int64_t n_counts, double *prob, double *log_evidence);
int sbn_program_sample_soft_host(sbn_program *prog, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, const float *lik,
                                 int64_t ld_lik, int lik_on_device, int64_t n_draws, uint64_t seed, int64_t row_base,
                                 uint8_t *out, float *prob, double *log_evidence);
int sbn_program_sample_soft_host_f64(sbn_program *prog, const uint8_t *ev, int64_t ld_ev, int64_t n_rows,
                                     const double *lik, int64_t ld_lik, int lik_on_device, int64_t n_draws,
                                     uint64_t seed, int64_t row_base, uint8_t *out, double *prob, double *log_evidence);
int sbn_program_mpe_soft_host(sbn_program *prog, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, const double *lik,
                              int64_t ld_lik, int lik_on_device, uint8_t *codes /* [n_decoded][n_rows] */,
                              double *log_prob /* [n_rows] */);

/* Gradients of log P(observed cells, lik) of a gradient program (planner.build_pattern_plan kind "grad",
 * version 10; every other call refuses it, and these calls refuse every other program).  The program may have
 * soft variables or none; with none, lik may be NULL.  `lik`, `ld_lik` and `lik_on_device` are those of
 * sbn_program_run_soft_host.  prob[b] = P(observed, lik / max), NaN for a row below the float32 range (1e-30;
 * 1e-290 for the float64 twin) or of probability zero: re-run it with the float64 program.
 * Forward: prob and log_prob[b] = log P(observed, lik) (double; either may be NULL).  Only the launches
 * P(observed) depends on run: no count step and no readout.
 * Backward: `weights` [n_rows] double (host, or device memory of the program's device with weights_on_device);
 * counts[e] += sum_b w_b * P(family entry e | observed, lik) (the layout of sbn_program_counts_host; a fully
 * observed family adds w_b), which is sum_b w_b * theta_e * d log P_b / d theta_e; and
 * deriv[j * ld_deriv + b] = d log P(observed, lik / max) / d (lik / max)_j of likelihood column j, which is
 * max * d log P_b / d lik_j (divide by the row's maximum of that variable), exact where lik_j = 0.  A flagged
 * row adds nothing and reads NaN.  The counts are reduced without floating-point atomics: two calls give
 * bitwise the same results.  Large batches run in chunks. */
int sbn_program_grad_forward_host(sbn_program *prog, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, const float *lik,
                                  int64_t ld_lik, int lik_on_device, float *prob, double *log_prob);
int sbn_program_grad_forward_host_f64(sbn_program *prog, const uint8_t *ev, int64_t ld_ev, int64_t n_rows,
                                      const double *lik, int64_t ld_lik, int lik_on_device, double *prob,
                                      double *log_prob);
int sbn_program_grad_backward_host(sbn_program *prog, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, const float *lik,
                                   int64_t ld_lik, int lik_on_device, const double *weights, int weights_on_device,
                                   double *counts, int64_t n_counts, float *deriv, int64_t ld_deriv, float *prob);
int sbn_program_grad_backward_host_f64(sbn_program *prog, const uint8_t *ev, int64_t ld_ev, int64_t n_rows,
                                       const double *lik, int64_t ld_lik, int lik_on_device, const double *weights,
                                       int weights_on_device, double *counts, int64_t n_counts, double *deriv,
                                       int64_t ld_deriv, double *prob);

/* Per-row joint posteriors of a joint program (planner.build_joint_plan / build_pattern_plan kind "joint",
 * version 11; every other call refuses it, and these calls refuse every other program).  `lik` is NULL exactly
 * when the program has no soft variables; otherwise `lik`, `ld_lik` and `lik_on_device` are those of
 * sbn_program_run_soft_host.  out[q * ld_out + b] = row q of the program's output for row b: the joint posterior
 * of each group's unobserved members at its rows (planner: Plan.group_rows; the first member fastest), given
 * the row's observed cells and likelihoods.  prob[b] = P(observed, lik / max).  A row below the float32 range
 * (1e-30; 1e-290 for the float64 twin) or of probability zero reads NaN throughout: re-run it with the float64
 * program.  No atomics: two calls give bitwise the same results.  Large batches run in chunks. */
int sbn_program_joint_host(sbn_program *prog, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, const float *lik,
                           int64_t ld_lik, int lik_on_device, float *out, int64_t ld_out, float *prob);
int sbn_program_joint_host_f64(sbn_program *prog, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, const double *lik,
                               int64_t ld_lik, int lik_on_device, double *out, int64_t ld_out, double *prob);

/* Same with DEVICE buffers, asynchronous on `stream` (a cudaStream_t; NULL = default
 * stream).  n_rows must not exceed the reserved chunk size. */
int sbn_program_run_device(sbn_program *prog, const uint8_t *d_ev, int64_t ld_ev, int64_t n_rows, float *d_out,
                           int64_t ld_out, void *stream);

/* Per-step device time of one run on device buffers (CUDA events around every launch;
 * diagnostic, not the fast path).  step_ms has n_steps + 1 entries (last = normalise). */
int sbn_program_profile(sbn_program *prog, const uint8_t *d_ev, int64_t ld_ev, int64_t n_rows, float *d_out,
                        int64_t ld_out, void *stream, float *step_ms, int64_t n_step_ms);

/* info[0]=Q  [1]=n_ev  [2]=n_steps  [3]=scratch floats per row  [4]=reserved rows
 * [5]=kernel launches issued by this program so far  [6]=mode (0 flat, 1 batched)
 * [7]=unbatched scratch floats
 * with n_info >= 12 also: [8]=on-chip segments in use  [9]=steps they cover  [10]=bytes per row the
 * segments still move through the HBM slot arena  [11]=per-CTA private scratch floats
 * with n_info >= 14 also: [12]=paired launches in use (a step and its consumer as one kernel, csrc/sbn_pair.h)
 * [13]=bytes per row those pairs do not move (their intermediates stay in registers) */
int sbn_program_info(const sbn_program *prog, int64_t *info, int64_t n_info);

/* How every program step is executed with the current switches: roles[i] = 0 evidence-independent (ran once, at
 * creation; or any step of a flat program), 1 its own launch, 2 / 3 first / second step of a paired launch
 * (csrc/sbn_pair.h: table x frontier twice), 4 / 5 first / second step of an expanding product fused with its
 * consumer, 6 inside an on-chip segment.  n_roles >= n_steps. */
int sbn_program_step_roles(const sbn_program *prog, int32_t *roles, int64_t n_roles);

/* 0 = plain launches; 1 = CUDA-graph replay of the step sequence (default); 3 = graph replay
 * with independent sub-trees of the elimination as parallel branches (experimental: measured
 * no gain on the benchmark plans, which are one long dependency chain). */
int sbn_program_set_graph(sbn_program *prog, int enabled);

/* Select the step kernel: 0 = the plain one-output-per-iteration kernel (general
 * fallback, cross-check in tests); 1 or 2 = register-tiled kernel with the operand
 * preload schedule where available (default); 4 = tiled, x-loop schedule only; 5 = tiled
 * without the shared-memory slab variant for expanding products; 7 = run the on-chip segments
 * (csrc/sbn_chain.h: runs of steps executed by one persistent kernel with the intermediates in
 * shared memory / an L2-resident scratch; opt-in, also SOROBN_B200_CHAIN=1), 6 = back to one launch
 * per step; 9 = run the steps it covers through the tensor-map TMA pipeline kernel (csrc/sbn_tma.h: 2-D / 4-D
 * `cp.async.bulk.tensor` boxes into a shared-memory ring fed by a producer warp; opt-in, also SOROBN_B200_TMA=1:
 * parity-green but not faster than the register-preload kernel, see DESIGN.md), 8 = off again;
 * 10 = no paired steps (every step its own launch), 11 = paired steps where eligible (default; csrc/sbn_pair.h:
 * a step and its consumer run as ONE kernel that keeps the intermediate factor in registers; SOROBN_B200_PAIR=0
 * disables them at creation). */
int sbn_program_set_tiled(sbn_program *prog, int enabled);

/* ------------------------------------------------------------------ Gibbs sampling
 * `BayesNet._gibbs_sampling` (bayes_net.py:665-737) with one chain per evidence row.
 * Variables are numbered topologically (every parent id < its child's id); CPT `v` lives at
 * tables[cpt_off[v]] with axes [*parents(v), v], v fastest.  `query` lists the query
 * variables slowest first (the order of the posterior's rows); `cycle` is the resampling
 * order of the non-event variables (the reference: sorted by name).  out[q * ld_out + c] is
 * the fraction of chain c's iterations spent in joint query state q. */
typedef struct sbn_sampler sbn_sampler;
int sbn_gibbs_create(int device, int32_t n_vars, const int32_t *card, const int32_t *par_ptr, const int32_t *par_idx,
                     const int32_t *cpt_off, const float *tables, int64_t n_table_floats, int32_t n_query,
                     const int32_t *query, int32_t n_ev, const int32_t *ev_vars, int32_t n_cycle, const int32_t *cycle,
                     sbn_sampler **out);
int sbn_gibbs_run_host(sbn_sampler *sampler, const uint8_t *ev, int64_t ld_ev, int64_t n_chains, int64_t n_iterations,
                       uint64_t seed, float *out, int64_t ld_out);
void sbn_gibbs_destroy(sbn_sampler *sampler);

/* The conditional the chain resamples `var` from, P(var | Markov blanket) for ONE joint state
 * (joint[v] = state code of variable v, v < n_vars; only the blanket is read): out[x], x < card(var),
 * normalised.  It is the table `_gibbs_sampling` precomputes for every variable
 * (bayes_net.py:699-712), evaluated by the same device code the chains run -- deterministic, so the
 * tests pin it entry by entry to the reference's tables. */
int sbn_gibbs_conditional(sbn_sampler *sampler, int32_t var, const uint8_t *joint, float *out);

/* The other sampling algorithms of `BayesNet.query` on the same sampler object:
 * algo 0 = Gibbs (as above), 1 = likelihood weighting (bayes_net.py:621-663), 2 = rejection
 * sampling (bayes_net.py:577-619); both built on forward sampling (bayes_net.py:518-548),
 * n_iterations samples per evidence row.  A row of rejection sampling that keeps no sample
 * is NaN (the reference returns an empty Series). */
#define SBN_ALGO_GIBBS 0
#define SBN_ALGO_LIKELIHOOD 1
#define SBN_ALGO_REJECTION 2
#define SBN_ALGO_GIBBS_GENERIC 3  /* Gibbs through the generic kernel even when the straight-line one applies (tests) */
int sbn_sampler_run_host(sbn_sampler *sampler, int algo, const uint8_t *ev, int64_t ld_ev, int64_t n_rows,
                         int64_t n_iterations, uint64_t seed, float *out, int64_t ld_out);

/* ------------------------------------------------------------------ structure learning
 * A tally is a complete discrete data set resident on one device, for the counting passes of score-based
 * structure learning (sorobn_b200/structure.py).  `codes` is host memory, uint8 state codes
 * codes[v * ld + b] (v < n_vars, b < n_rows: one row of codes per column, rows innermost, as the evidence
 * layout), every code below cards[v] (1 <= cards[v] <= 256; checked); it is uploaded once, at creation.
 * A data set that does not fit the device fails with SBN_E_NOMEM.
 *
 * A batch of families is given by `words`: per family k, then its k distinct member columns, the child first
 * and its parents after it.  Family f's contingency table has T_f = prod cards entries, at most
 * SBN_TALLY_MAX_TABLE, laid out [parent k-1] .. [parent 1][child] with the child fastest (entry
 * sum_i code_i * prod_{l < i} cards[member l]); the tables of a batch are concatenated in family order.
 * Families whose tables fit SBN_TALLY_SMEM_BINS together are counted in shared memory, each code byte read
 * once per such group; a family with a larger table counts with global atomics.  Counts are exact.
 *
 * sbn_tally_counts: every table of the batch, counts[n_counts] (n_counts = sum_f T_f).
 * sbn_tally_scores: scores[f], the decomposable score of family f in double, with N = n_rows, N_jk the count of
 * child state k under parent configuration j (q = T_f / r configurations, r = cards[child], seen or not) and
 * N_j = sum_k N_jk:
 *   SBN_SCORE_BIC:  sum_jk N_jk ln(N_jk / N_j) - ln(N) q (r - 1) / 2, with 0 ln 0 = 0;
 *   SBN_SCORE_BDEU: sum_j [lgamma(a/q) - lgamma(N_j + a/q) + sum_k (lgamma(N_jk + a/(q r)) - lgamma(a/(q r)))],
 *                   a = ess > 0, the equivalent sample size (ignored by BIC).
 * sbn_tally_tests: conditional-independence tests X _|_ Y | S for constraint-based learning.  A test's words are
 * those of a family with x as the child and y as parent 1: k x y s1 .. s(k-2), k >= 2, so its table is
 * [s_(k-2)] .. [s_1][y][x], x fastest, and a configuration z of S is a stratum of r_x r_y contiguous entries.
 * out[3 t .. 3 t + 2] = statistic, degrees of freedom, p-value of test t, in double.  Per stratum, N_z is its rows,
 * N_xz = sum_y N_xyz and N_yz = sum_x N_xyz:
 *   SBN_TEST_G2:   G^2 = 2 sum N_xyz ln(N_xyz N_z / (N_xz N_yz)) over the non-zero cells;
 *   SBN_TEST_CHI2: X^2 = sum (N_xyz - E)^2 / E, E = N_xz N_yz / N_z, over the cells with E > 0.
 * dof = sum_z (a_z - 1)(b_z - 1), a_z (b_z) the states of x (y) with N_xz > 0 (N_yz > 0); an empty stratum adds 0.
 * p = Q(dof / 2, stat / 2), the regularised upper incomplete gamma function, and 1 when dof = 0.  k < 2 and an
 * unknown kind are SBN_E_INVALID; the words are checked as sbn_tally_counts checks them. */
typedef struct sbn_tally sbn_tally;
#define SBN_TALLY_MAX_TABLE (1 << 22)  /* entries of one family's table                         */
#define SBN_TALLY_SMEM_BINS 32768      /* shared-memory bins of one group; larger tables go global */
#define SBN_SCORE_BIC 0
#define SBN_SCORE_BDEU 1
#define SBN_TEST_G2 0    /* likelihood-ratio G^2 */
#define SBN_TEST_CHI2 1  /* Pearson X^2          */
int sbn_tally_create(int device, const uint8_t *codes, int64_t ld, int32_t n_vars, int64_t n_rows, const int32_t *cards,
                     sbn_tally **out);
int sbn_tally_counts(sbn_tally *tally, const int32_t *words, int64_t n_words, uint64_t *counts, int64_t n_counts);
int sbn_tally_scores(sbn_tally *tally, const int32_t *words, int64_t n_words, int kind, double ess, double *scores,
                     int64_t n_families);
int sbn_tally_tests(sbn_tally *tally, const int32_t *words, int64_t n_words, int kind, double *out, int64_t n_tests);
void sbn_tally_destroy(sbn_tally *tally);

/* ------------------------------------------------------------------ loopy belief propagation
 * Approximate posterior marginals of networks too wide to eliminate exactly: sum-product message passing on the
 * factor graph of the CPT families, synchronous flooding with damping (the algorithm, its zero and underflow
 * rules and the word layout: sorobn_b200/bp.py).  `words` and `tables` come from bp.compile_graph; every word is
 * bounds-checked here.  One thread runs one evidence row through every sweep; larger batches run in chunks, and a
 * row's result does not depend on the chunking.
 * sbn_bp_run_host: `ev` uint8 codes [n_ev][ld_ev] (host; a code past its variable's states reads as the last);
 * out[q * ld_out + b] = the belief of row b in state q of the targets' output (float, host); iterations[b] = the
 * sweep at which row b converged (its largest damped-message change fell below tol) or met a zero sum (its
 * beliefs are then NaN), or n_iterations + 1 when it did not converge.  1 <= n_iterations < 2^31 - 1,
 * 0 <= damping < 1, tol >= 0 (tol = 0 runs exactly n_iterations sweeps).
 * sbn_bp_mpe_host: max-product words of bp.compile_mpe_graph (version 2; sbn_bp_create takes either version, and
 * each run call refuses the other's words): the same sweep with a max in place of the sum, then, per row,
 * codes[k * ld_codes + b] = the decoded state of the k-th unobserved variable (var id order; codes may be NULL when
 * there is none), log_p[b] = log P(decode, observed cells) in double (-inf for a decode of probability 0, NaN for
 * a row that met a zero sum, whose codes are 0) and iterations[b] as above (0 when every node is observed).
 * Same argument rules as sbn_bp_run_host.
 * sbn_bp_counts_host: expected-counts words of bp.compile_counts_graph (version 3; bp.py "Expected counts"): the
 * sum-product sweep over every CPT, then per row the belief of every family, summed over the live rows into
 * counts[n_table_floats] (double, blob order: entry i counts the configuration of table entry i; bp.Graph.perm maps
 * it to the dense CPTs) without floating-point atomics, so two calls are bitwise equal; log_z[b] = the Bethe
 * log-likelihood of row b in double (NaN for a dead row, which adds nothing) and iterations[b] as above (0 for a row
 * dead before its first sweep and when every node is observed).  Same argument rules as sbn_bp_run_host.  Each run
 * call refuses the words of the others, naming the call that runs them.
 * sbn_bp_set_tables: new float32 tables of the same size for the handle's words (an EM iteration's CPTs). */
typedef struct sbn_bp sbn_bp;
int sbn_bp_create(int device, const int32_t *words, int64_t n_words, const float *tables, int64_t n_table_floats,
                  sbn_bp **out);
int sbn_bp_run_host(sbn_bp *bp, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, int32_t n_iterations, float damping,
                    float tol, float *out, int64_t ld_out, int32_t *iterations);
int sbn_bp_mpe_host(sbn_bp *bp, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, int32_t n_iterations,
                    float damping, float tol, uint8_t *codes, int64_t ld_codes, double *log_p, int32_t *iterations);
int sbn_bp_counts_host(sbn_bp *bp, const uint8_t *ev, int64_t ld_ev, int64_t n_rows, int32_t n_iterations,
                       float damping, float tol, double *counts, double *log_z, int32_t *iterations);
int sbn_bp_set_tables(sbn_bp *bp, const float *tables, int64_t n_table_floats);
void sbn_bp_destroy(sbn_bp *bp);

/* Pinned host memory for evidence / posterior staging buffers. */
int sbn_host_alloc(void **ptr, int64_t bytes);
int sbn_host_free(void *ptr);

#ifdef __cplusplus
}
#endif
#endif /* SOROBN_B200_H */
