// Normal-equation form of the weight-step search (see gram.cu).
#pragma once
#include "common.cuh"

#ifndef GRAM_BM
#define GRAM_BM 64       // tokens per shared-memory chunk of the update pass
#endif
#ifndef GRAM_UN
#define GRAM_UN 4        // tokens per register group of the update pass (the next group is prefetched)
#endif

struct GramUpdateArgs {
  float* E; const float* G; const float* gscale;      // [M][O] residual (in/out), gradient, power-of-two scale
  const float* W; int M, O, K;
  const int8_t* XqT; int Mp;                           // [K][Mp] quantised activations, token-major
  const float* dX; int crb_acts;
  const float* dW; const float* dW_prev;               // current table [n_V][n_H]; step sizes of block h_prev before its search [n_V]
  int n_V, n_H, crb_rows;
  int h_prev, k_prev, k_next, ks;                      // h_prev < 0: no update, only accumulate
  float w_lo, w_hi;
  float* Upart; float* E2part;                         // [n_split][O][ks], [n_split][O]
  float* D; int n_split;                               // scratch [O][32 or 64] (weight deltas of the previous pick); token splits
};
int p4v_gram_update(const GramUpdateArgs& a, cudaStream_t st);
int p4v_gram_update_splits(int O, int M);

struct GramEvalArgs {
  const float* H; int ldH; int npairs;                 // [O][ldH] Gram of the integer activations (upper triangle, row-major pairs)
  const float* U; const float* E2;                     // [O][ks], [O] (reduced over the token blocks)
  const float* W; int O, K, k_first, ks;
  const float* dW; const float* dW0; int n_H, h;
  const float* dX; int crb_acts;
  const float* factors; int n_cand;
  int n_groups, rows_per_group;                        // row blocks v
  int osplit, rows_per_block;                          // each row block is evaluated by osplit thread blocks of rows_per_block channels
  float w_lo, w_hi;
  double* sums; int n_keys;                            // [n_cand][n_keys = n_groups*osplit]: positive error sums per thread block
  double* sums2;                                       // [n_cand][n_groups]: the same summed per row block
};
int p4v_gram_eval(const GramEvalArgs& a, cudaStream_t st);
// accumulate = 1: add to U and E2 (later row chunks of a chunked search) instead of overwriting them
int p4v_gram_reduce(const float* Upart, const float* E2part, int n_mblk, int O, int ks, float* U, float* E2, int accumulate,
                    cudaStream_t st);

int p4v_xq_transpose(const float* x, int M, int K, int Mp, const float* dX, int crb_acts, float qlo, float qhi, int8_t* out, cudaStream_t st);
// Z image of n_blocks column blocks starting at weight column k_first: row (b * npairs + pair) of 256-row tiles
int p4v_pair_image(const int8_t* XqT, int Mp, int M, int k_first, int ks, int npairs, int n_blocks, int tiles_p,
                   unsigned long long tile_bytes, unsigned int term_bytes, uint8_t* dst, cudaStream_t st);

#define GRAM_PT 256      // pair rows per tile of the Z image (= N of the Gram GEMM's MMA)
struct GramGemmArgs {
  const uint8_t* R; unsigned long long R_tile_bytes;   // (gs*g)^2 image: [tiles_o][2 terms][K chunk][128][16 B]
  const uint8_t* C; unsigned long long C_tile_bytes;   // pair image:     [tiles_p][2 terms][K chunk][256][16 B]
  unsigned int term_bytes;                             // bytes of K (tokens * 2, padded to 32) of one term
  int tiles_o, tiles_p, O;
  float* H; long long ldH;                             // [O][ldH], ldH >= tiles_p * 256
  int accumulate;                                      // 1: the running sum starts from the stored H (row chunks)
};
int p4v_gram_gemm(const GramGemmArgs& a, cudaStream_t st);
