// Support kernels around the sweep: min-max initialisation, operand-image
// quantisation, per-step scale tables, deterministic score reduction, argmax +
// commit of the chosen candidate.  All HBM-bound streaming work.
#pragma once
#include "common.cuh"

struct P4VSeg {          // one K segment of an operand image
  int k0, klen;          // source column range
  int dst_off;           // byte offset of the segment inside the tile image ( = 128 * byte offset in the padded row )
  int didx;              // column index into the step-size table (block / chunk id)
  float fixed_delta;     // > 0: use this constant step size (twin-uniform negative part)
  float lo, hi;          // clamp range
  int sos_part;          // split-of-softmax twin quantizer (matmul.py:595-598): 1 = high part, 2 = low part, 0 = plain
  float qm1;             // qmax - 1 for the sos parts
  int split3;            // 1..3: no quantisation, emit the i-th bf16 term of the exact 3-way split of the fp32 value
  int square;            // with split3: split v*v*presc^2 instead of v (Gram operand g^2)
};

struct QuantImageArgs {
  const float* src; long long ld; long long prob_stride;   // [P][rows][K], transposed read if src_kmajor == 0
  int src_transposed;    // 1: element (row, k) lives at src[k * ld + row]  (MatMul B operand)
  int P, rows, tiles;    // tiles per problem
  uint8_t* dst; unsigned long long tile_bytes, plane_stride;
  int n_planes;          // candidate planes (1 for the current image)
  const float* factors;  // [n_planes] candidate factors or null (=> 1.0, no extra rounding)
  const float* delta;    // step-size table: delta[rb * d_stride + seg.didx]
  int rows_per_block;    // rb = (row / rows_per_block) (Linear W: crb_rows); 0 => rb = problem % d_mod
  int d_stride, d_mod;
  const P4VSeg* segs; int nseg;
  int is_int8;
  const float* split;    // sos: device scalar split point for the current image (candidate planes use factors[plane])
  const float* presc;    // optional device scalar multiplied into the source before `square`
  int ieee_div;          // filled by p4v_quant_image: Python-scalar step sizes divide the IEEE way (see keys_to_delta)
};
int p4v_quant_image(const QuantImageArgs& a, cudaStream_t st);

// max / absmax of blocks of a row-major matrix, written as order-preserving int keys
int p4v_block_max(const float* src, long long ld, int rows, int row_block, int n_row_blocks,
                  int col_block, int n_col_blocks, int use_abs, int* keys, cudaStream_t st);
// per-problem-group absmax of a [P][rows][cols] tensor: group = p % n_groups
int p4v_group_absmax(const float* src, long long prob_elems, int P, int n_groups, int* keys, cudaStream_t st);
int p4v_keys_reset(int* keys, int n, cudaStream_t st);
// delta[i] = key_to_float(keys[i]) / denom ; optionally copy to a second array
int p4v_keys_broadcast_max(int* keys, int n, cudaStream_t st);     // init_layerwise: all keys of the range := their maximum
int p4v_scalar_div_ieee();
int p4v_keys_to_delta(const int* keys, int n, float denom, float* d0, float* d1, cudaStream_t st);
// gscale = 2^-floor(log2(max|g|)) (1 if max is 0 / non-finite)
int p4v_make_gscale(const int* key, float* gscale, cudaStream_t st);

struct GroupMeta { short h, a; short neg; short pad; };   // neg: use the constant negative-part step size

struct StepTablesArgs {
  int kind;                  // 0: Linear W step, 1: Linear X step, 2: head-wise MatMul step, 3: MatMul step whose other operand has per-group uniform scales (sos)
  int target;                // h (W step) / a (X step)
  const float* dW; const float* dW0; int n_V, n_H, crb_rows;
  const float* dX; const float* dX0; int n_a; float d_neg;
  const float* factors; int n_cand;
  const GroupMeta* fixed_meta; int n_fixed_groups;
  const GroupMeta* cand_meta;  int n_cand_groups;
  int nsg;
  float* fix_scale; float* candA; float* candB;
};
int p4v_step_tables(const StepTablesArgs& a, cudaStream_t st);

struct ReduceArgs {
  const float* partial; int n_cand;
  int P, tiles_m, tiles_n, order;
  int mode;                  // P4V_SG_COLUMN: key = global 16-column group (tn*8+i) ; P4V_SG_PROBLEM: key = p % n_keys
  int n_keys;
  double* sums;              // [n_cand][n_keys]  fixed-order fp64 sums of the sweep partials
  int accumulate;            // 1: add to sums (later chunks of a chunked search) instead of overwriting them
};
int p4v_reduce_scores(const ReduceArgs& a, cudaStream_t st);

// One block: scores[c][g] = -norm * sum_{k in group g} sums[c][k]; argmax over c per group (first maximum, NaN wins,
// like torch.argmax); publishes the new step sizes, the score log and -- when has_next -- the scale tables of the
// next search step (which depend on the step sizes just chosen).
struct SelectArgs {
  const double* sums; int n_cand, n_keys, n_groups, keys_per_group;
  double inv_count; const float* gscale;
  const float* factors;
  const float* d0; float* d; int d_stride, d_col;    // d[g * d_stride + d_col] = fl(f[best_g] * d0[...])
  int* best;                                         // [n_groups]
  float* score_log;                                  // [n_cand][n_groups] fp32 (optional)
  float* d_prev;                                     // optional [n_groups]: the step sizes before this step
  int has_next; StepTablesArgs next;
};
int p4v_select_step(const SelectArgs& a, cudaStream_t st);

// Copy the winning candidate's image slabs into the current image.
struct CommitSeg { int src_off, dst_off, kb; };
struct CommitArgs {
  const int* best; int n_groups;
  // rows of group g = [g*rows_per_group, (g+1)*rows_per_group) ; rows_per_group==0 -> all rows group 0 ; problem mode: group = p % n_groups
  const uint8_t* cand; unsigned long long cand_plane_stride, cand_tile_bytes;
  uint8_t* cur; unsigned long long cur_tile_bytes;
  int P, tiles, rows_per_group, problem_groups;
  const CommitSeg* segs; int nseg;
  int commit_chunks;                                 // sum over segs of kb/16
};
int p4v_commit_step(const CommitArgs& a, cudaStream_t st);
