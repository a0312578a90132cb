// sorobn_b200 -- row-block join kernel for the steps where two batched factors meet and several variables are
// summed out (e.g. `625 <- sum_25 t5e2 x B625 x B625 x t25e1` on the benchmark grid).
//
// The tiled kernel (sbn_kernels.cuh, MX schedule) gives each thread one 5 x 5 output tile and reads the operand
// entries it needs from global memory; the neighbouring tiles of the same rows read most of those entries again,
// through L2.  Here one CTA owns a block of R evidence rows and computes EVERY output entry of the step for them:
//   * the batched operands of the R rows travel to shared memory as one tensor-map TMA box per operand
//     ((R rows) x (all entries), entry-major), into a two-stage ring on `full` mbarriers, so the next block's
//     load overlaps the current block's arithmetic; persistent CTAs walk the row blocks;
//   * the step's tables are staged once per CTA by bulk TMA and gathered with the row's evidence offset;
//   * thread = (row, tile): the arithmetic reads shared memory only, every operand byte comes from HBM once,
//     the outputs go from registers to HBM with streaming stores.
// Each output entry is computed with the same fp32 operations, in the same order, as the tiled kernel's MX
// schedule (same products of the U / A / B operands, same fmaf order over the eliminated states), so the two
// kernels give bitwise equal results and the choice between them is invisible.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define SBN_JOIN_STAGES 2          // ring depth: 2 x (R rows x all batched entries) fits 227 KB at R = 16 / 32
#define SBN_JOIN_MAX_THREADS 512   // R x tiles
#define SBN_JOIN_MAX_BATCHED 2     // batched operands (one tensor map each)

struct sbn_program;
struct StepDesc;
struct SbnStep;
// Rows per CTA block the join kernel runs step `st` with, for the launch parameters `q` the tiled kernel would get,
// or 0 when the step is left to the tiled kernel: it takes the tiled kernel's MX steps (T = 5, several eliminated
// variables, whole tiles) with two batched operands, and only when the batch has enough row blocks to fill every SM.
int sbn_join_rows(const sbn_program *P, const StepDesc &st, const SbnStep &q);
cudaError_t sbn_join_launch(sbn_program *P, const StepDesc &st, const SbnStep &q, cudaStream_t stream);
cudaError_t sbn_join_set_attrs();
