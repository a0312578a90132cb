// sorobn_b200 -- tensor-map TMA pipeline for the HBM-bound elimination steps.
//
// The tiled kernel (sbn_kernels.cuh) keeps every operand of a tile in registers before the first
// FFMA (the "preload schedule"): ~100 of its 167-200 registers are loads in flight, which caps it
// at 12-17 % warps active and leaves the DRAM bus ~67 % busy -- a thread cannot fetch tile t + 1
// while it computes tile t.  Here the batched operands of a tile travel as 2-D TMA boxes
// (`cp.async.bulk.tensor.2d`, SASS UTMALDG): the factor `[entries][ld rows]` is one tensor map,
// a box is `256 rows x 1 entry` (1 KB), a producer warp issues the boxes of tile t + 2 into a
// shared-memory ring while four consumer warps compute tile t from shared memory and store it.
// Persistent CTAs walk (row block, tile) items, so the pipeline never drains inside a launch.
//
// Reference operators fused by one launch: `pointwise_mul` (bayes_net.py:253-256) over the
// step's factors + `sum_out` (bayes_net.py:54-103) of one variable + the evidence filter of
// bayes_net.py:772-774 -- the same contract as sbn_step_tiled.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/sorobn_b200.h"

#define SBN_TMA_ROWS 256          // rows per item = rows of one box (the TMA maximum per dimension)
#define SBN_TMA_CONSUMERS 4       // consumer warps: 32 lanes x 2 rows each
#define SBN_TMA_THREADS ((SBN_TMA_CONSUMERS + 1) * 32)
#define SBN_TMA_SLOTS 6           // U0 U1 | A0 A1 | B0 B1   (U0 / A0 / B0 may be batched, the others are tables)
#define SBN_TMA_MAX_STAGES 4

struct SbnTmaIn {
    int32_t kind;                 // 0 absent, 1 table (gathered from shared memory), 2 batched (TMA ring)
    int32_t col;                  // column of this input's element offset in a tile row
    int32_t sx, sd;               // element strides: eliminated variable, the tile axis of the slot's class
    int32_t off;                  // table: float offset inside the table area; batched: float offset inside a stage
    int32_t tmap;                 // batched: tensor map index
    int32_t tn;                   // batched: entries per eliminated state (T, or 1 for a U-class operand)
    int32_t n_ev;
    int32_t ev_col[SBN_MAX_EV];
    int32_t ev_stride[SBN_MAX_EV];
    int32_t ev_card[SBN_MAX_EV];
};

struct SbnTmaTable {
    const float *src;
    int32_t floats;               // multiple of 4
    int32_t off;                  // float offset inside the table area
};

struct SbnTmaParams {
    CUtensorMap tm[2];            // batched operands: 4-D view (rows, tile digit, eliminated state, entry), box (256, tn, CX, 1);
                                  // fallback: (rows, entries), box (256, 1)
    float *out;
    const uint8_t *ev;
    const int32_t *tile_off;      // [n_tiles][n_in + 2] (tiled-kernel table: out entry, na | nb << 8, input offsets)
    int64_t ld_ev;
    int64_t ld;
    int32_t n_rows;
    int32_t n_tiles;
    int32_t row_words;
    int32_t c0;                   // cardinality of output axis 0
    const int32_t *zoff;          // several eliminated variables: [n_in][cx] joint-state element offsets (tiled order), else nullptr
    int32_t cx;                   // joint states of the eliminated variables
    int32_t n_blocks;             // cx / CX: blocks of the first variable's states (one stage each)
    int64_t n_items;              // row blocks x tiles
    int32_t n_stages;
    int32_t stage_floats;         // floats of one stage (all batched operands of one tile)
    int32_t n_boxes;              // boxes (= entries) per stage
    int32_t nk0;                  // boxes of tensor map 0 (the rest belong to map 1)
    int32_t n_tables;
    int32_t table_floats;
    int32_t big_boxes;            // 1: 4-D tensor maps, one box per operand and stage; 0: (rows, entries) maps, one-entry boxes
    int32_t n_maps;
    SbnTmaTable tab[4];
    SbnTmaIn in[SBN_TMA_SLOTS];
};

struct sbn_program;
struct StepDesc;
// host side (sbn_tma.cu)
bool sbn_tma_eligible(const sbn_program *P, const StepDesc &st);
cudaError_t sbn_tma_launch(sbn_program *P, const StepDesc &st, const uint8_t *d_ev, int64_t ld_ev, int64_t n_rows,
                           cudaStream_t stream);
cudaError_t sbn_tma_set_attrs();
// Tensor map of the first n_rows rows of a batched factor [entries][ld] as the 3-D view
// (row, entry % e_lo, entry / e_lo), box = (box_rows, e_lo, entries / e_lo): one instruction copies the whole
// factor for box_rows rows, entry-major in shared memory.  Rows past n_rows arrive as zeros.  false when the
// driver has no encoder or refuses the view.
bool sbn_tma_encode_rows(CUtensorMap *map, const float *base, int64_t ld, int64_t n_rows, int64_t entries, int box_rows, int e_lo);
// Tensor map of the first n_rows rows of a batched factor [entries][ld] seen through `rank` (<= 4) entry axes of
// extents dims[] and entry strides strides[] (any order; an axis of extent 1 may have any stride): the view
// (row, axis 0, .., axis rank-1), box (box_rows, box[0], .., box[rank-1]), row-major in shared memory with the row
// fastest.  Rows past n_rows arrive as zeros.  false when the driver has no encoder or refuses the view.
bool sbn_tma_encode_view(CUtensorMap *map, const float *base, int64_t ld, int64_t n_rows, int rank, const int64_t *dims,
                         const int64_t *strides, const int *box, int box_rows);
